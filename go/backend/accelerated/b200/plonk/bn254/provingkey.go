// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build b200

package plonk

import (
	"sync"

	plonk_bn254 "github.com/consensys/gnark/backend/plonk/bn254"
	cs "github.com/consensys/gnark/constraint/bn254"

	"github.com/consensys/gnark/backend/accelerated/b200/internal/cabi"
)

// deviceInfo is the device-resident form of the key: the trace (Ql, Qr, Qm, Qo, Qk, Qcp, the permutation) of ONE
// constraint system and the canonical KZG SRS, behind b200_plonk_pk_load; and, when the system has BSB22 commitments,
// pk.KzgLagrange.G1 as a plain table for the hint's commitment (b200_msm_indexed).
type deviceInfo struct {
	spr      *cs.SparseR1CS // the system the trace was built from
	device   int
	key      *cabi.PlonkKey
	trace    *plonk_bn254.Trace
	lagrange *cabi.Table // nil without BSB22 commitments
}

func (d *deviceInfo) free() {
	d.key.Free()
	d.lagrange.Free()
}

// ProvingKey embeds the native key so that WriteTo / ReadFrom are inherited and keys are wire compatible with the CPU
// backend (the construction of the accelerated Groth16 keys, backend/accelerated/icicle/groth16/bn254/provingkey.go:37-42).
type ProvingKey struct {
	plonk_bn254.ProvingKey
	*deviceInfo
	setupMu sync.Mutex
}

// FreeGPUResources releases the device-resident copy of the key. Safe to call more than once; the next Prove uploads
// the key again.
func (pk *ProvingKey) FreeGPUResources() {
	pk.setupMu.Lock()
	defer pk.setupMu.Unlock()
	if pk.deviceInfo != nil {
		pk.deviceInfo.free()
		pk.deviceInfo = nil
	}
}

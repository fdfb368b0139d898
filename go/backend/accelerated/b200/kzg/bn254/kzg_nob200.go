// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build !b200

package bn254

import (
	"hash"

	curve "github.com/consensys/gnark-crypto/ecc/bn254"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr"
	"github.com/consensys/gnark-crypto/ecc/bn254/kzg"
	"github.com/consensys/gnark/backend/accelerated/b200"
)

// ToLagrangeG1 is the GPU twin of gnark-crypto's kzg.ToLagrangeG1 (see the b200 build).
func ToLagrangeG1(coeffs []curve.G1Affine) ([]curve.G1Affine, error) {
	panic("b200 backend requested but program compiled without 'b200' build tag")
}

// DeviceKey is the device-resident KZG proving key of the b200 build.
type DeviceKey struct{}

const noTag = "b200 backend requested but program compiled without 'b200' build tag"

// NewDeviceKey is the b200 build's (see there).
func NewDeviceKey(pk kzg.ProvingKey, opts ...b200.Option) (*DeviceKey, error) { panic(noTag) }

func (k *DeviceKey) Free()                                               { panic(noTag) }
func (k *DeviceKey) Commit(p []fr.Element) (kzg.Digest, error)            { panic(noTag) }
func (k *DeviceKey) CommitBatch(ps [][]fr.Element) ([]kzg.Digest, error) { panic(noTag) }
func (k *DeviceKey) Open(p []fr.Element, point fr.Element) (kzg.OpeningProof, error) {
	panic(noTag)
}
func (k *DeviceKey) OpenBatch(ps [][]fr.Element, points []fr.Element) ([]kzg.OpeningProof, error) {
	panic(noTag)
}
func (k *DeviceKey) BatchOpenSinglePoint(polynomials [][]fr.Element, digests []kzg.Digest, point fr.Element, hf hash.Hash,
	dataTranscript ...[]byte) (kzg.BatchOpeningProof, error) {
	panic(noTag)
}

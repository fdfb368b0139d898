// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build b200

package bn254

import (
	"fmt"
	"math/big"
	"runtime"
	"slices"
	"sync"
	"time"
	"unsafe"

	"github.com/consensys/gnark-crypto/ecc"
	curve "github.com/consensys/gnark-crypto/ecc/bn254"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr/hash_to_field"
	"github.com/consensys/gnark/backend"
	"github.com/consensys/gnark/backend/accelerated/b200"
	"github.com/consensys/gnark/backend/accelerated/b200/internal/cabi"
	groth16_bn254 "github.com/consensys/gnark/backend/groth16/bn254"
	"github.com/consensys/gnark/backend/witness"
	"github.com/consensys/gnark/constraint"
	cs "github.com/consensys/gnark/constraint/bn254"
	"github.com/consensys/gnark/constraint/solver"
	fcs "github.com/consensys/gnark/frontend/cs"
	"github.com/consensys/gnark/internal"
	"github.com/consensys/gnark/logger"
)

const curveID = cabi.BN254

func boolsToBytes(b []bool) []byte { // InfinityA / InfinityB: one byte per wire on the C side
	out := make([]byte, len(b))
	for i, v := range b {
		if v {
			out[i] = 1
		}
	}
	return out
}

func ptrOf[T any](s []T) unsafe.Pointer { return unsafe.Pointer(unsafe.SliceData(s)) }

// setupDevicePointers uploads the key once per placement (setupDevicePointers, icicle.go:88-264). gnark's memory image
// of the point slices is the device table layout, so there is no conversion pass; every slice is borrowed for the
// duration of the C call only.
func (pk *ProvingKey) setupDevicePointers(r1cs *cs.R1CS, cfg *b200.Config) error {
	pk.setupMu.Lock()
	defer pk.setupMu.Unlock()
	devs := cfg.Devices()
	if pk.deviceInfo != nil {
		if slices.Equal(pk.deviceInfo.devices, devs) && pk.deviceInfo.precompute == cfg.Precompute {
			return nil
		}
		pk.freeLocked() // another placement: release the old one first
	}
	commitmentInfo := r1cs.CommitmentInfo.(constraint.Groth16Commitments)
	// wires that have no base in G1.K (prove.go:231-235): the private committed wires and the commitment wires
	toRemove := commitmentInfo.GetPrivateCommitted()
	toRemove = append(toRemove, commitmentInfo.CommitmentIndexes())
	removed := internal.ConcatAll(toRemove...)
	kRemoved := make([]uint32, len(removed))
	for i, w := range removed {
		kRemoved[i] = uint32(w)
	}
	slices.Sort(kRemoved)

	infA, infB := boolsToBytes(pk.InfinityA), boolsToBytes(pk.InfinityB)
	flags := int32(0)
	if cfg.Precompute {
		flags = cabi.TablePrecomp
	}
	info := &deviceInfo{devices: slices.Clone(devs), precompute: cfg.Precompute}
	release := func() {
		for _, k := range info.keys {
			k.Free()
		}
		for _, k := range info.commitment {
			k.Free()
		}
	}
	for shard, dev := range devs {
		d := cabi.Groth16KeyDesc{
			Curve:      curveID,
			DomainSize: pk.Domain.Cardinality,
			DomainGen:  unsafe.Pointer(&pk.Domain.Generator),
			CosetGen:   unsafe.Pointer(&pk.Domain.FrMultiplicativeGen),
			G1Alpha:    unsafe.Pointer(&pk.G1.Alpha),
			G1Beta:     unsafe.Pointer(&pk.G1.Beta),
			G1Delta:    unsafe.Pointer(&pk.G1.Delta),
			G2Beta:     unsafe.Pointer(&pk.G2.Beta),
			G2Delta:    unsafe.Pointer(&pk.G2.Delta),
			G1A:        ptrOf(pk.G1.A),
			NA:         len(pk.G1.A),
			G1B:        ptrOf(pk.G1.B),
			NB:         len(pk.G1.B),
			G1Z:        ptrOf(pk.G1.Z),
			NZ:         len(pk.G1.Z),
			G1K:        ptrOf(pk.G1.K),
			NK:         len(pk.G1.K),
			G2B:        ptrOf(pk.G2.B),
			NB2:        len(pk.G2.B),
			InfinityA:  infA,
			InfinityB:  infB,
			NbWires:    len(pk.InfinityA),
			NbPublic:   r1cs.GetNbPublicVariables(),
			Flags:      flags,
			ShardRank:  shard,
			ShardWorld: len(devs),
			KRemoved:   kRemoved,
			Pin: []any{&pk.Domain.Generator, &pk.Domain.FrMultiplicativeGen, &pk.G1.Alpha, &pk.G1.Beta, &pk.G1.Delta,
				&pk.G2.Beta, &pk.G2.Delta, unsafe.SliceData(pk.G1.A), unsafe.SliceData(pk.G1.B), unsafe.SliceData(pk.G1.Z),
				unsafe.SliceData(pk.G1.K), unsafe.SliceData(pk.G2.B)},
		}
		k, err := cabi.LoadGroth16Key(dev, &d)
		if err != nil {
			release()
			return err
		}
		info.keys = append(info.keys, k)
	}
	// Pedersen commitment keys (CommitmentKeys[i].Basis / BasisExpSigma) on the first device
	for i := range pk.CommitmentKeys {
		ck := &pk.CommitmentKeys[i]
		var pinner runtime.Pinner
		if len(ck.Basis) > 0 {
			pinner.Pin(unsafe.SliceData(ck.Basis))
			pinner.Pin(unsafe.SliceData(ck.BasisExpSigma))
		}
		k, err := cabi.LoadPedersenKey(devs[0], curveID, ptrOf(ck.Basis), ptrOf(ck.BasisExpSigma), len(ck.Basis))
		pinner.Unpin()
		if err != nil {
			release()
			return err
		}
		info.commitment = append(info.commitment, k)
	}
	pk.deviceInfo = info
	return nil
}

// Prove generates the proof of knowledge of a r1cs with full witness (secret + public part). Same signature and
// option handling as the ICICLE backend's per-curve Prove (icicle.go:784); the stage order follows
// backend/groth16/bn254/prove.go:52-315.
func Prove(r1cs *cs.R1CS, pk *ProvingKey, fullWitness witness.Witness, cfg *b200.Config) (*groth16_bn254.Proof, error) {
	log := logger.Logger().With().Str("curve", r1cs.CurveID().String()).Str("acceleration", "b200").Int("nbConstraints", r1cs.GetNbConstraints()).Str("backend", "groth16").Logger()
	if err := pk.setupDevicePointers(r1cs, cfg); err != nil {
		return nil, fmt.Errorf("setup device pointers: %w", err)
	}
	info := pk.deviceInfo
	proof, solution, err := solve(r1cs, pk, fullWitness, cfg, info)
	if err != nil {
		return nil, err
	}

	start := time.Now()

	// sample random r and s (prove.go:170-182)
	var r, s fr.Element
	if _, err := r.SetRandom(); err != nil {
		return nil, err
	}
	if _, err := s.SetRandom(); err != nil {
		return nil, err
	}

	// everything from here to the three proof points runs behind the C ABI: wire filtering (prove.go:147-168), computeH
	// (:346-389), the five MSMs (:194,207,227,237,283) and the assembly (:185,199-214,241-269,287-292)
	var pinner runtime.Pinner
	defer pinner.Unpin()
	for _, p := range []any{unsafe.SliceData(solution.W), unsafe.SliceData(solution.A), unsafe.SliceData(solution.B),
		unsafe.SliceData(solution.C), &r, &s, &proof.Ar, &proof.Bs, &proof.Krs} {
		pinner.Pin(p)
	}
	w, a, b, c := ptrOf(solution.W), ptrOf(solution.A), ptrOf(solution.B), ptrOf(solution.C)
	if len(info.keys) == 1 {
		if err := info.keys[0].Prove(w, a, b, c, len(solution.A), unsafe.Pointer(&r), unsafe.Pointer(&s),
			unsafe.Pointer(&proof.Ar), unsafe.Pointer(&proof.Bs), unsafe.Pointer(&proof.Krs)); err != nil {
			return nil, err
		}
	} else {
		// one goroutine per device: the device parts run concurrently (the library locks per device), the partial
		// sums are added here - the shape of the reference's own chunk loop (icicle.go:383-411)
		type partial struct {
			G1 [4]curve.G1Jac // A, B1, Z(h), K
			G2 curve.G2Jac    // B2
		}
		parts := make([]partial, len(info.keys))
		errs := make([]error, len(info.keys))
		pinner.Pin(unsafe.SliceData(parts))
		var wg sync.WaitGroup
		for d := range info.keys {
			wg.Add(1)
			go func(d int) {
				defer wg.Done()
				errs[d] = info.keys[d].MSMs(w, a, b, c, len(solution.A), unsafe.Pointer(&parts[d]))
			}(d)
		}
		wg.Wait()
		for _, e := range errs {
			if e != nil {
				return nil, e
			}
		}
		for d := 1; d < len(parts); d++ {
			for k := range parts[0].G1 {
				parts[0].G1[k].AddAssign(&parts[d].G1[k])
			}
			parts[0].G2.AddAssign(&parts[d].G2)
		}
		if err := info.keys[0].Assemble(unsafe.Pointer(&parts[0]), unsafe.Pointer(&r), unsafe.Pointer(&s),
			unsafe.Pointer(&proof.Ar), unsafe.Pointer(&proof.Bs), unsafe.Pointer(&proof.Krs)); err != nil {
			return nil, err
		}
	}
	runtime.KeepAlive(solution)
	log.Debug().Dur("took", time.Since(start)).Msg("prover done")
	return proof, nil
}

// solve runs the R1CS solver with the BSB22 commitment hint served by the device (prove.go:72-99) and folds the proofs of
// knowledge of the commitments (prove.go:118-129).  Every call has its own prover config, hint closure and proof, so
// several witnesses can be solved concurrently.
func solve(r1cs *cs.R1CS, pk *ProvingKey, fullWitness witness.Witness, cfg *b200.Config, info *deviceInfo) (*groth16_bn254.Proof, *cs.R1CSSolution, error) {
	opt, err := backend.NewProverConfig(cfg.ProverOpts...)
	if err != nil {
		return nil, nil, fmt.Errorf("new prover config: %w", err)
	}
	if opt.HashToFieldFn == nil {
		opt.HashToFieldFn = hash_to_field.New([]byte(constraint.CommitmentDst))
	}
	commitmentInfo := r1cs.CommitmentInfo.(constraint.Groth16Commitments)
	proof := &groth16_bn254.Proof{Commitments: make([]curve.G1Affine, len(commitmentInfo))}
	solverOpts := opt.SolverOpts[:len(opt.SolverOpts):len(opt.SolverOpts)]
	poks := make([]curve.G1Affine, len(pk.CommitmentKeys))
	// override hints (prove.go:72-99): Commit AND ProveKnowledge of commitment i are two MSMs of the same scalars, run
	// on the device over one upload; the proof of knowledge is kept for the fold below
	bsb22ID := solver.GetHintID(fcs.Bsb22CommitmentComputePlaceholder)
	solverOpts = append(solverOpts, solver.OverrideHint(bsb22ID, func(_ *big.Int, in []*big.Int, out []*big.Int) error {
		i := int(in[0].Int64())
		in = in[1:]
		values := make([]fr.Element, len(commitmentInfo[i].PrivateCommitted))
		hashed := in[:len(commitmentInfo[i].PublicAndCommitmentCommitted)]
		committed := in[+len(hashed):]
		for j, inJ := range committed {
			values[j].SetBigInt(inJ)
		}
		var pinner runtime.Pinner
		pinner.Pin(&proof.Commitments[i])
		pinner.Pin(&poks[i])
		if len(values) > 0 {
			pinner.Pin(unsafe.SliceData(values))
		}
		err := info.commitment[i].Commit(ptrOf(values), len(values), unsafe.Pointer(&proof.Commitments[i]), unsafe.Pointer(&poks[i]))
		pinner.Unpin()
		if err != nil {
			return err
		}

		opt.HashToFieldFn.Write(constraint.SerializeCommitment(proof.Commitments[i].Marshal(), hashed, (fr.Bits-1)/8+1))
		hashBts := opt.HashToFieldFn.Sum(nil)
		opt.HashToFieldFn.Reset()
		nbBuf := fr.Bytes
		if opt.HashToFieldFn.Size() < fr.Bytes {
			nbBuf = opt.HashToFieldFn.Size()
		}
		var res fr.Element
		res.SetBytes(hashBts[:nbBuf])
		res.BigInt(out[0])
		return nil
	}))

	_solution, err := r1cs.Solve(fullWitness, solverOpts...)
	if err != nil {
		return nil, nil, err
	}
	solution := _solution.(*cs.R1CSSolution)
	wireValues := []fr.Element(solution.W)

	// compute challenge for folding the PoKs from the commitments (prove.go:118-129)
	commitmentsSerialized := make([]byte, fr.Bytes*len(commitmentInfo))
	for i := range commitmentInfo {
		copy(commitmentsSerialized[fr.Bytes*i:], wireValues[commitmentInfo[i].CommitmentIndex].Marshal())
	}
	challenge, err := fr.Hash(commitmentsSerialized, []byte("G16-BSB22"), 1)
	if err != nil {
		return nil, nil, err
	}
	if _, err = proof.CommitmentPok.Fold(poks, challenge[0], ecc.MultiExpConfig{NbTasks: 1}); err != nil {
		return nil, nil, err
	}
	return proof, solution, nil
}


// ProveBatch proves several full witnesses of one circuit with one b200_groth16_prove_batch call: the witnesses are solved
// concurrently (each with its own hint closure, proof and proof-of-knowledge fold), then the device work of all of them
// runs as one launch sequence.  Proof i equals what Prove gives for witness i with the same r, s.  One device and an
// unsharded key only.
func ProveBatch(r1cs *cs.R1CS, pk *ProvingKey, fullWitnesses []witness.Witness, cfg *b200.Config) ([]*groth16_bn254.Proof, error) {
	if len(cfg.Devices()) > 1 {
		return nil, fmt.Errorf("ProveBatch: one device only (WithDevices lists %d)", len(cfg.Devices()))
	}
	if len(fullWitnesses) == 0 {
		return nil, nil
	}
	if err := pk.setupDevicePointers(r1cs, cfg); err != nil {
		return nil, fmt.Errorf("setup device pointers: %w", err)
	}
	info := pk.deviceInfo
	k := len(fullWitnesses)
	proofs := make([]*groth16_bn254.Proof, k)
	solutions := make([]*cs.R1CSSolution, k)
	errs := make([]error, k)
	var wg sync.WaitGroup
	for i := range fullWitnesses {
		wg.Add(1)
		go func(i int) {
			defer wg.Done()
			proofs[i], solutions[i], errs[i] = solve(r1cs, pk, fullWitnesses[i], cfg, info)
		}(i)
	}
	wg.Wait()
	for i, e := range errs {
		if e != nil {
			return nil, fmt.Errorf("witness %d: %w", i, e)
		}
	}
	// r_i, s_i item-major (prove.go:170-182); the outputs are written into the proofs through three staging arrays
	rs := make([]fr.Element, 2*k)
	for i := range rs {
		if _, err := rs[i].SetRandom(); err != nil {
			return nil, err
		}
	}
	r, s := make([]fr.Element, k), make([]fr.Element, k)
	for i := 0; i < k; i++ {
		r[i], s[i] = rs[2*i], rs[2*i+1]
	}
	ar, bs, krs := make([]curve.G1Affine, k), make([]curve.G2Affine, k), make([]curve.G1Affine, k)
	var pinner runtime.Pinner
	defer pinner.Unpin()
	w, a, b, c := make([]unsafe.Pointer, k), make([]unsafe.Pointer, k), make([]unsafe.Pointer, k), make([]unsafe.Pointer, k)
	for i, sol := range solutions {
		for _, p := range []any{unsafe.SliceData(sol.W), unsafe.SliceData(sol.A), unsafe.SliceData(sol.B), unsafe.SliceData(sol.C)} {
			pinner.Pin(p)
		}
		w[i], a[i], b[i], c[i] = ptrOf(sol.W), ptrOf(sol.A), ptrOf(sol.B), ptrOf(sol.C)
	}
	for _, p := range []any{unsafe.SliceData(r), unsafe.SliceData(s), unsafe.SliceData(ar), unsafe.SliceData(bs), unsafe.SliceData(krs)} {
		pinner.Pin(p)
	}
	if err := info.keys[0].ProveBatch(w, a, b, c, len(solutions[0].A), ptrOf(r), ptrOf(s), ptrOf(ar), ptrOf(bs), ptrOf(krs)); err != nil {
		return nil, err
	}
	for i := range proofs {
		proofs[i].Ar, proofs[i].Bs, proofs[i].Krs = ar[i], bs[i], krs[i]
	}
	runtime.KeepAlive(solutions)
	return proofs, nil
}

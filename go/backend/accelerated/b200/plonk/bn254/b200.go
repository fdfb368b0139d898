// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build b200

package plonk

import (
	"errors"
	"fmt"
	"hash"
	"math/big"
	"math/bits"
	"runtime"
	"time"
	"unsafe"

	curve "github.com/consensys/gnark-crypto/ecc/bn254"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr/fft"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr/hash_to_field"
	"github.com/consensys/gnark-crypto/ecc/bn254/kzg"
	fiatshamir "github.com/consensys/gnark-crypto/fiat-shamir"
	"github.com/consensys/gnark/backend"
	"github.com/consensys/gnark/backend/accelerated/b200"
	"github.com/consensys/gnark/backend/accelerated/b200/internal/cabi"
	plonk_bn254 "github.com/consensys/gnark/backend/plonk/bn254"
	"github.com/consensys/gnark/backend/witness"
	"github.com/consensys/gnark/constraint"
	cs "github.com/consensys/gnark/constraint/bn254"
	"github.com/consensys/gnark/constraint/solver"
	fcs "github.com/consensys/gnark/frontend/cs"
	"github.com/consensys/gnark/logger"
)

const curveID = cabi.BN254

// blinding orders of backend/plonk/bn254/prove.go:70-76 (order + 1 coefficients each)
const (
	orderBlindingL = 1
	orderBlindingR = 1
	orderBlindingO = 1
	orderBlindingZ = 2
)

func ptrOf[T any](s []T) unsafe.Pointer { return unsafe.Pointer(unsafe.SliceData(s)) }

// setupDevicePointers builds the trace of spr (NewTrace, setup.go:171-231) and uploads it together with the canonical
// SRS, once per (key, constraint system, device). The sigma polynomials are rebuilt on the library side from trace.S.
func (pk *ProvingKey) setupDevicePointers(spr *cs.SparseR1CS, domain0 *fft.Domain, cfg *b200.Config) error {
	pk.setupMu.Lock()
	defer pk.setupMu.Unlock()
	if pk.deviceInfo != nil {
		if pk.deviceInfo.spr == spr && pk.deviceInfo.device == cfg.DeviceID {
			return nil
		}
		pk.deviceInfo.free()
		pk.deviceInfo = nil
	}
	n := int(domain0.Cardinality)
	if len(pk.Kzg.G1) < n+3 {
		return fmt.Errorf("kzg srs too small: %d points, need %d", len(pk.Kzg.G1), n+3)
	}
	trace := plonk_bn254.NewTrace(spr, domain0)
	qcp := make([]unsafe.Pointer, len(trace.Qcp))
	pin := []any{unsafe.SliceData(trace.Ql.Coefficients()), unsafe.SliceData(trace.Qr.Coefficients()),
		unsafe.SliceData(trace.Qm.Coefficients()), unsafe.SliceData(trace.Qo.Coefficients()),
		unsafe.SliceData(trace.Qk.Coefficients()), unsafe.SliceData(pk.Kzg.G1)}
	for i := range trace.Qcp {
		qcp[i] = ptrOf(trace.Qcp[i].Coefficients())
		pin = append(pin, unsafe.SliceData(trace.Qcp[i].Coefficients()))
	}
	key, err := cabi.LoadPlonkKey(cfg.DeviceID, curveID, uint32(bits.TrailingZeros64(domain0.Cardinality)),
		ptrOf(trace.Ql.Coefficients()), ptrOf(trace.Qr.Coefficients()), ptrOf(trace.Qm.Coefficients()),
		ptrOf(trace.Qo.Coefficients()), ptrOf(trace.Qk.Coefficients()), trace.S, ptrOf(pk.Kzg.G1), qcp, pin)
	if err != nil {
		return err
	}
	// the BSB22 hint commits against the Lagrange SRS (kzg.Commit(values, pk.KzgLagrange), prove.go:300): a plain table
	// of exactly n points, as plonk.Setup requires; systems without commitments upload nothing more
	var lagrange *cabi.Table
	if len(trace.Qcp) > 0 {
		if len(pk.KzgLagrange.G1) != n {
			key.Free()
			return fmt.Errorf("kzg lagrange srs: %d points, need %d", len(pk.KzgLagrange.G1), n)
		}
		var pinner runtime.Pinner
		pinner.Pin(unsafe.SliceData(pk.KzgLagrange.G1))
		lagrange, err = cabi.UploadTable(cfg.DeviceID, curveID, 1, ptrOf(pk.KzgLagrange.G1), n, 0)
		pinner.Unpin()
		if err != nil {
			key.Free()
			return err
		}
	}
	pk.deviceInfo = &deviceInfo{spr: spr, device: cfg.DeviceID, key: key, trace: trace, lagrange: lagrange}
	return nil
}

// bindPublicData and deriveRandomness restate the transcript layout of backend/plonk/bn254/verify.go:325-366 and
// prove.go (deriveRandomness): what the verifier recomputes, so it cannot differ.
func bindPublicData(fs *fiatshamir.Transcript, challenge string, vk *plonk_bn254.VerifyingKey, publicInputs []fr.Element) error {
	for _, d := range []*kzg.Digest{&vk.S[0], &vk.S[1], &vk.S[2], &vk.Ql, &vk.Qr, &vk.Qm, &vk.Qo, &vk.Qk} {
		if err := fs.Bind(challenge, d.Marshal()); err != nil {
			return err
		}
	}
	for i := range vk.Qcp {
		if err := fs.Bind(challenge, vk.Qcp[i].Marshal()); err != nil {
			return err
		}
	}
	for i := range publicInputs {
		if err := fs.Bind(challenge, publicInputs[i].Marshal()); err != nil {
			return err
		}
	}
	return nil
}

func deriveRandomness(fs *fiatshamir.Transcript, challenge string, points ...*curve.G1Affine) (fr.Element, error) {
	var r fr.Element
	for _, p := range points {
		buf := p.RawBytes()
		if err := fs.Bind(challenge, buf[:]); err != nil {
			return r, err
		}
	}
	b, err := fs.ComputeChallenge(challenge)
	if err != nil {
		return r, err
	}
	r.SetBytes(b)
	return r, nil
}

// deriveFolding restates gnark-crypto's kzg.deriveGamma (ecc/bn254/kzg/kzg.go, unexported): the challenge that
// kzg.BatchOpenSinglePoint folds the opened polynomials with, bound to the point, the digests, the claimed values and
// the extra transcript data. kzg.BatchVerifySinglePoint recomputes it on the verifier's side.
func deriveFolding(point fr.Element, digests []kzg.Digest, claimedValues []fr.Element, hf hash.Hash, dataTranscript ...[]byte) (fr.Element, error) {
	var gamma fr.Element
	fs := fiatshamir.NewTranscript(hf, "gamma")
	if err := fs.Bind("gamma", point.Marshal()); err != nil {
		return gamma, err
	}
	for i := range digests {
		if err := fs.Bind("gamma", digests[i].Marshal()); err != nil {
			return gamma, err
		}
	}
	for i := range claimedValues {
		if err := fs.Bind("gamma", claimedValues[i].Marshal()); err != nil {
			return gamma, err
		}
	}
	for i := range dataTranscript {
		if err := fs.Bind("gamma", dataTranscript[i]); err != nil {
			return gamma, err
		}
	}
	b, err := fs.ComputeChallenge("gamma")
	if err != nil {
		return gamma, err
	}
	gamma.SetBytes(b)
	return gamma, nil
}

func randomCoefficients(order int) ([]fr.Element, error) { // getRandomPolynomial, prove.go:1239-1253
	a := make([]fr.Element, order+1)
	for i := range a {
		if _, err := a[i].SetRandom(); err != nil {
			return nil, err
		}
	}
	return a, nil
}

// Prove generates a PLONK proof (backend/plonk/bn254/prove.go:98-153). The solver, the BSB22 hint, hashing and the
// Fiat-Shamir transcript run in Go exactly as in the CPU prover; every polynomial operation between two challenges
// is one call into the library (b200_plonk_begin ... b200_plonk_batch_open), with all polynomials resident in HBM.
func Prove(spr *cs.SparseR1CS, pk *ProvingKey, fullWitness witness.Witness, cfg *b200.Config) (*plonk_bn254.Proof, error) {
	log := logger.Logger().With().Str("curve", spr.CurveID().String()).Str("acceleration", "b200").
		Int("nbConstraints", spr.GetNbConstraints()).Str("backend", "plonk").Logger()
	opt, err := backend.NewProverConfig(cfg.ProverOpts...)
	if err != nil {
		return nil, fmt.Errorf("get prover options: %w", err)
	}
	if opt.HashToFieldFn == nil {
		opt.HashToFieldFn = hash_to_field.New([]byte("BSB22-Plonk"))
	}
	start := time.Now()

	// fft domain of the circuit (newInstance, prove.go:236)
	sizeSystem := uint64(spr.GetNbConstraints() + len(spr.Public)) // len(spr.Public) is for the placeholder constraints
	domain0 := fft.NewDomain(sizeSystem)
	if domain0.Cardinality < 8 {
		return nil, errors.New("b200 plonk: circuits below 8 rows need the 8n quotient domain of the CPU prover (prove.go:248); use backend/plonk")
	}
	n := int(domain0.Cardinality)
	if err := pk.setupDevicePointers(spr, domain0, cfg); err != nil {
		return nil, fmt.Errorf("setup device pointers: %w", err)
	}
	info := pk.deviceInfo
	trace := info.trace

	wWitness, ok := fullWitness.Vector().(fr.Vector)
	if !ok {
		return nil, witness.ErrInvalidWitness
	}

	proof := &plonk_bn254.Proof{}
	fs := fiatshamir.NewTranscript(opt.ChallengeHash, "gamma", "beta", "alpha", "zeta")

	// BSB22 commitments (initBSB22Commitments + bsb22Hint, prove.go:268-318): the hint runs while solving, before
	// L, R, O exist, so its commitment is the Lagrange-SRS MSM of the reference - here one indexed MSM on the device over
	// the hint's few non-zero entries (b200_msm_indexed); the committed polynomials are kept and handed to the device
	// prover, which adds their gate term, their part of the linearised polynomial and the openings
	commitmentInfo := spr.CommitmentInfo.(constraint.PlonkCommitments)
	commitmentVal := make([]fr.Element, len(commitmentInfo))
	committed := make([][]fr.Element, len(commitmentInfo))
	proof.Bsb22Commitments = make([]kzg.Digest, len(commitmentInfo))
	bsb22ID := solver.GetHintID(fcs.Bsb22CommitmentComputePlaceholder)
	solverOpts := append(opt.SolverOpts[:len(opt.SolverOpts):len(opt.SolverOpts)], solver.OverrideHint(bsb22ID,
		func(_ *big.Int, ins, outs []*big.Int) error {
			commDepth := int(ins[0].Int64())
			ins = ins[1:]
			ci := commitmentInfo[commDepth]
			values := make([]fr.Element, n)
			offset := spr.GetNbPublicVariables()
			for i := range ins {
				values[offset+ci.Committed[i]].SetBigInt(ins[i])
			}
			// the commitment injection constraint and the last constraint have qcp = 0: safe to use for blinding
			if _, err := values[offset+ci.CommitmentIndex].SetRandom(); err != nil {
				return err
			}
			if _, err := values[offset+spr.GetNbConstraints()-1].SetRandom(); err != nil {
				return err
			}
			committed[commDepth] = values
			// kzg.Commit(values, pk.KzgLagrange) over the len(ins) + 2 entries the hint wrote (a position written twice
			// is taken once, with its last value, as in the dense vector)
			positions := append(append(make([]int, 0, len(ins)+2), ci.Committed[:len(ins)]...), ci.CommitmentIndex, spr.GetNbConstraints()-1)
			idx := make([]uint32, 0, len(positions))
			seen := make(map[int]bool, len(positions))
			for _, p := range positions {
				if !seen[p] {
					seen[p] = true
					idx = append(idx, uint32(offset+p))
				}
			}
			scalars := make([]fr.Element, len(idx))
			for j, p := range idx {
				scalars[j] = values[p]
			}
			var digest curve.G1Jac
			var pinner runtime.Pinner
			pinner.Pin(unsafe.SliceData(scalars))
			pinner.Pin(&digest)
			err := info.lagrange.MSMIndexed(idx, ptrOf(scalars), unsafe.Pointer(&digest))
			pinner.Unpin()
			if err != nil {
				return err
			}
			proof.Bsb22Commitments[commDepth].FromJacobian(&digest)
			opt.HashToFieldFn.Write(proof.Bsb22Commitments[commDepth].Marshal())
			hashBts := opt.HashToFieldFn.Sum(nil)
			opt.HashToFieldFn.Reset()
			nbBuf := fr.Bytes
			if opt.HashToFieldFn.Size() < fr.Bytes {
				nbBuf = opt.HashToFieldFn.Size()
			}
			commitmentVal[commDepth].SetBytes(hashBts[:nbBuf])
			commitmentVal[commDepth].BigInt(outs[0])
			return nil
		}))

	// solve constraints (solveConstraints, prove.go:320-350)
	_solution, err := spr.Solve(fullWitness, solverOpts...)
	if err != nil {
		return nil, err
	}
	solution := _solution.(*cs.SparseR1CSSolution)
	L, R, O := []fr.Element(solution.L), []fr.Element(solution.R), []fr.Element(solution.O)
	if len(L) != n || len(R) != n || len(O) != n {
		return nil, fmt.Errorf("b200 plonk: solution columns of %d rows on a domain of %d", len(L), n)
	}

	// complete qk (completeQk, prove.go:352-381)
	qk := make([]fr.Element, n)
	copy(qk, trace.Qk.Coefficients())
	copy(qk, wWitness[:len(spr.Public)])
	for i := range commitmentInfo {
		qk[spr.GetNbPublicVariables()+commitmentInfo[i].CommitmentIndex] = commitmentVal[i]
	}

	// blinding polynomials (initBlindingPolynomials, prove.go:259-266)
	bl, err := randomCoefficients(orderBlindingL)
	if err != nil {
		return nil, err
	}
	br, err := randomCoefficients(orderBlindingR)
	if err != nil {
		return nil, err
	}
	bo, err := randomCoefficients(orderBlindingO)
	if err != nil {
		return nil, err
	}
	bz, err := randomCoefficients(orderBlindingZ)
	if err != nil {
		return nil, err
	}

	var pinner runtime.Pinner
	defer pinner.Unpin()
	for _, s := range [][]fr.Element{L, R, O, qk, bl, br, bo, bz} {
		pinner.Pin(unsafe.SliceData(s))
	}
	pi2 := make([]unsafe.Pointer, len(committed))
	for i := range committed {
		pinner.Pin(unsafe.SliceData(committed[i]))
		pi2[i] = ptrOf(committed[i])
	}

	// round 1: [L], [R], [O] (commitToLRO, prove.go:404-489; the device commits the blinded canonical forms on the
	// canonical SRS: the same group elements as the reference's Lagrange-SRS MSM + commitBlindingFactor)
	var lro [3]curve.G1Jac
	bsbJac := make([]curve.G1Jac, len(committed))
	pinner.Pin(&lro)
	var bsbPtr unsafe.Pointer
	if len(bsbJac) > 0 {
		pinner.Pin(unsafe.SliceData(bsbJac))
		bsbPtr = ptrOf(bsbJac)
	}
	sess, err := info.key.Begin(ptrOf(L), ptrOf(R), ptrOf(O), ptrOf(bl), ptrOf(br), ptrOf(bo), pi2, bsbPtr, unsafe.Pointer(&lro))
	if err != nil {
		return nil, err
	}
	defer sess.End()
	for i := range lro {
		proof.LRO[i].FromJacobian(&lro[i])
	}
	for i := range bsbJac { // two independent device paths must agree: the hint's indexed Lagrange MSM and [PI2_i] of the canonical form
		var d kzg.Digest
		d.FromJacobian(&bsbJac[i])
		if !d.Equal(&proof.Bsb22Commitments[i]) {
			return nil, fmt.Errorf("b200 plonk: BSB22 commitment %d differs between the hint and the device", i)
		}
	}
	if err := sess.SetQk(ptrOf(qk)); err != nil {
		return nil, err
	}
	if opt.StatisticalZK { // quotientShardsRandomizers (newInstance, prove.go:239-242; h1(), h2(), h3() :689-722)
		hr, err := randomCoefficients(1)
		if err != nil {
			return nil, err
		}
		pinner.Pin(unsafe.SliceData(hr))
		if err := sess.SetQuotientRandomizers(ptrOf(hr)); err != nil {
			return nil, err
		}
	}

	// gamma, beta (deriveGammaAndBeta, prove.go:492-523)
	if err := bindPublicData(fs, "gamma", pk.Vk, wWitness[:len(spr.Public)]); err != nil {
		return nil, err
	}
	gamma, err := deriveRandomness(fs, "gamma", &proof.LRO[0], &proof.LRO[1], &proof.LRO[2])
	if err != nil {
		return nil, err
	}
	bbeta, err := fs.ComputeChallenge("beta")
	if err != nil {
		return nil, err
	}
	var beta fr.Element
	beta.SetBytes(bbeta)

	// round 2: [Z] (buildRatioCopyConstraint, prove.go:635-668)
	var zJac curve.G1Jac
	pinner.Pin(&zJac)
	pinner.Pin(&beta)
	pinner.Pin(&gamma)
	if err := sess.CommitZ(unsafe.Pointer(&beta), unsafe.Pointer(&gamma), ptrOf(bz), unsafe.Pointer(&zJac)); err != nil {
		return nil, err
	}
	proof.Z.FromJacobian(&zJac)

	// alpha (deriveAlpha, prove.go:541-550)
	alphaDeps := make([]*curve.G1Affine, len(proof.Bsb22Commitments)+1)
	for i := range proof.Bsb22Commitments {
		alphaDeps[i] = &proof.Bsb22Commitments[i]
	}
	alphaDeps[len(alphaDeps)-1] = &proof.Z
	alpha, err := deriveRandomness(fs, "alpha", alphaDeps...)
	if err != nil {
		return nil, err
	}

	// round 3: [H1], [H2], [H3] (computeQuotient, prove.go:558-633)
	var hJac [3]curve.G1Jac
	pinner.Pin(&hJac)
	pinner.Pin(&alpha)
	if err := sess.Quotient(unsafe.Pointer(&alpha), unsafe.Pointer(&hJac)); err != nil {
		return nil, err
	}
	for i := range hJac {
		proof.H[i].FromJacobian(&hJac[i])
	}

	// zeta (deriveZeta, prove.go:552-556)
	zeta, err := deriveRandomness(fs, "zeta", &proof.H[0], &proof.H[1], &proof.H[2])
	if err != nil {
		return nil, err
	}

	// round 4: Z opened at w*zeta, the linearised polynomial and its digest, the values opened at zeta
	// (openZ :670-687, computeLinearizedPolynomial :724-794)
	var two [2]curve.G1Jac
	values := make([]fr.Element, 7+len(commitmentInfo))
	pinner.Pin(&two)
	pinner.Pin(unsafe.SliceData(values))
	pinner.Pin(&zeta)
	if err := sess.Linearise(unsafe.Pointer(&zeta), unsafe.Pointer(&two), ptrOf(values)); err != nil {
		return nil, err
	}
	var linearizedDigest kzg.Digest
	linearizedDigest.FromJacobian(&two[0])
	proof.ZShiftedOpening.H.FromJacobian(&two[1])
	proof.ZShiftedOpening.ClaimedValue = values[6]
	claimed := make([]fr.Element, 0, 6+len(commitmentInfo))
	claimed = append(claimed, values[:6]...)
	claimed = append(claimed, values[7:]...)

	// round 5: batch opening at zeta (batchOpening, prove.go:796-837): the folding challenge of
	// kzg.BatchOpenSinglePoint, then the folded quotient on the device
	digestsToOpen := make([]kzg.Digest, 6+len(pk.Vk.Qcp))
	copy(digestsToOpen[6:], pk.Vk.Qcp)
	digestsToOpen[0] = linearizedDigest
	digestsToOpen[1], digestsToOpen[2], digestsToOpen[3] = proof.LRO[0], proof.LRO[1], proof.LRO[2]
	digestsToOpen[4], digestsToOpen[5] = pk.Vk.S[0], pk.Vk.S[1]
	v, err := deriveFolding(zeta, digestsToOpen, claimed, opt.KZGFoldingHash, proof.ZShiftedOpening.ClaimedValue.Marshal())
	if err != nil {
		return nil, err
	}
	var batchJac curve.G1Jac
	pinner.Pin(&batchJac)
	pinner.Pin(&v)
	if err := sess.BatchOpen(unsafe.Pointer(&v), unsafe.Pointer(&batchJac)); err != nil {
		return nil, err
	}
	proof.BatchedProof.H.FromJacobian(&batchJac)
	proof.BatchedProof.ClaimedValues = claimed

	runtime.KeepAlive(solution)
	log.Debug().Dur("took", time.Since(start)).Msg("prover done")
	return proof, nil
}

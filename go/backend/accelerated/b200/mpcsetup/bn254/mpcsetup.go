// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build b200

package bn254

import (
	"bytes"
	"crypto/sha256"
	"encoding/binary"
	"errors"
	"fmt"
	"io"
	"math/big"
	"slices"
	"unsafe"

	curve "github.com/consensys/gnark-crypto/ecc/bn254"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr"
	cmpc "github.com/consensys/gnark-crypto/ecc/bn254/mpcsetup"
	"github.com/consensys/gnark/backend/accelerated/b200/internal/cabi"
	"github.com/consensys/gnark/backend/groth16/bn254/mpcsetup"
	gIo "github.com/consensys/gnark/io"
)

const (
	curveID = cabi.BN254
	dev     = 0
)

// scaleG1 sets s[i] to (c * t^i) * s[i] on the device (t nil: t = 1).
func scaleG1(s []curve.G1Affine, c, t *fr.Element) error {
	if len(s) == 0 {
		return nil
	}
	return cabi.PointsScale(dev, curveID, 1, unsafe.Pointer(&s[0]), len(s), unsafe.Pointer(c), unsafe.Pointer(t))
}

// scaleG2 is scaleG1 on G2.
func scaleG2(s []curve.G2Affine, c, t *fr.Element) error {
	if len(s) == 0 {
		return nil
	}
	return cabi.PointsScale(dev, curveID, 2, unsafe.Pointer(&s[0]), len(s), unsafe.Pointer(c), unsafe.Pointer(t))
}

// ContributePhase2 is the twin of gnark's Phase2.Contribute (phase2.go:137-153) with the point vectors scaled on device 0:
// it sets p.Challenge to the sha256 of p.WriteTo, draws δ' and the σ_j with gnark-crypto's mpcsetup.UpdateValues (which
// also builds the update proofs), scales G1.Z and G1.PKK by 1/δ' and each G1.SigmaCKK[j] by σ_j on the device, and the
// single points G1.Delta, G2.Delta and G2.Sigma[j] on the host.  The new values are computed on copies and stored into p
// only once every step has succeeded: when an error is returned, p is unchanged.  p is otherwise trusted to be well
// formed, as by Contribute.
func ContributePhase2(p *mpcsetup.Phase2) error {
	nc := len(p.Parameters.G1.SigmaCKK)
	if nc > 255 {
		return errors.New("too many commitments") // DST collision
	}
	if len(p.Sigmas) != nc || len(p.Parameters.G2.Sigma) != nc {
		return errors.New("commitment counts of Sigmas, G1.SigmaCKK and G2.Sigma differ")
	}
	if err := cabi.Init([]int{dev}); err != nil {
		return err
	}
	h := sha256.New()
	if _, err := p.WriteTo(h); err != nil {
		return err
	}
	challenge := h.Sum(nil)

	var delta fr.Element
	deltaProof := cmpc.UpdateValues(&delta, challenge, mpcsetup.DST_DELTA)
	sigma := make([]fr.Element, nc)
	sigmaProofs := make([]cmpc.UpdateProof, nc)
	for i := range sigma {
		sigmaProofs[i] = cmpc.UpdateValues(&sigma[i], challenge, mpcsetup.DST_SIGMA+byte(i))
	}

	var I big.Int
	g2Sigma := slices.Clone(p.Parameters.G2.Sigma)
	sigmaCKK := make([][]curve.G1Affine, nc)
	for i := range sigma {
		sigma[i].BigInt(&I)
		g2Sigma[i].ScalarMultiplication(&g2Sigma[i], &I)
		sigmaCKK[i] = slices.Clone(p.Parameters.G1.SigmaCKK[i])
		if err := scaleG1(sigmaCKK[i], &sigma[i], nil); err != nil {
			return err
		}
	}
	delta.BigInt(&I)
	var g1Delta curve.G1Affine
	var g2Delta curve.G2Affine
	g1Delta.ScalarMultiplication(&p.Parameters.G1.Delta, &I)
	g2Delta.ScalarMultiplication(&p.Parameters.G2.Delta, &I)
	var deltaInv fr.Element
	deltaInv.Inverse(&delta)
	z := slices.Clone(p.Parameters.G1.Z)
	if err := scaleG1(z, &deltaInv, nil); err != nil {
		return err
	}
	pkk := slices.Clone(p.Parameters.G1.PKK)
	if err := scaleG1(pkk, &deltaInv, nil); err != nil {
		return err
	}

	p.Challenge = challenge
	p.Delta = deltaProof
	copy(p.Sigmas, sigmaProofs)
	p.Parameters.G1.Delta, p.Parameters.G2.Delta = g1Delta, g2Delta
	p.Parameters.G1.Z, p.Parameters.G1.PKK = z, pkk
	p.Parameters.G1.SigmaCKK, p.Parameters.G2.Sigma = sigmaCKK, g2Sigma
	return nil
}

// readRun reads n fixed-size encoded points of `size` bytes each.
func readRun(r io.Reader, n, size int) ([]byte, error) {
	b := make([]byte, n*size)
	_, err := io.ReadFull(r, b)
	return b, err
}

// decodeG1 decodes n compressed G1 points from r on the device into dst (len n).
func decodeG1(r io.Reader, dst []curve.G1Affine) error {
	if len(dst) == 0 {
		return nil
	}
	b, err := readRun(r, len(dst), curve.SizeOfG1AffineCompressed)
	if err != nil {
		return err
	}
	return cabi.PointsDecode(dev, curveID, 1, b, len(dst), cabi.PointsCompressed, unsafe.Pointer(&dst[0]))
}

// decodeG2 decodes n compressed G2 points from r on the device into dst (len n).
func decodeG2(r io.Reader, dst []curve.G2Affine) error {
	if len(dst) == 0 {
		return nil
	}
	b, err := readRun(r, len(dst), curve.SizeOfG2AffineCompressed)
	if err != nil {
		return err
	}
	return cabi.PointsDecode(dev, curveID, 2, b, len(dst), cabi.PointsCompressed, unsafe.Pointer(&dst[0]))
}

// ContributePhase1 reads a serialised Phase1 (what Phase1.WriteTo writes, marshal.go:19-57) from r and writes the next
// contribution to w, as Phase1.Contribute followed by WriteTo would, with the point work on device 0.  Phase 1's
// parameters are not exported, so the contribution goes through the serialised form:
//   - the challenge is the sha256 of the input bytes, which is the previous contribution's hash (its encoding is
//     canonical);
//   - the three previous update proofs are read with UpdateProof.ReadFrom and dropped;
//   - SrsCommons (SrsCommons.refsSlice, marshal.go:157-179: N, [β]₂, [τⁱ]₁ for 1 ≤ i ≤ 2N-2, [τⁱ]₂ for 1 ≤ i < N,
//     [βτⁱ]₁ and [ατⁱ]₁ for i < N) is decoded run by run on the device: a square root per compressed point would
//     dominate on the CPU.  Like UnsafeReadFrom, subgroup membership is not checked: the input is trusted to be well
//     formed, as by Contribute;
//   - τ', α', β' and their proofs come from gnark-crypto's mpcsetup.UpdateValues; the four vectors are scaled with
//     (c, t) = (τ', τ'), (τ', τ'), (α', τ'), (β', τ') on the device and [β]₂ on the host (phase1.go:104-147);
//   - the output is the three new proofs (UpdateProof.WriteTo), SrsCommons.WriteTo and the challenge
//     (io.WriteBytesShort).
func ContributePhase1(r io.Reader, w io.Writer) error {
	if err := cabi.Init([]int{dev}); err != nil {
		return err
	}
	in, err := io.ReadAll(r)
	if err != nil {
		return err
	}
	challenge := sha256.Sum256(in)
	rd := bytes.NewReader(in)
	var prev [3]cmpc.UpdateProof
	for i := range prev {
		if _, err := prev[i].ReadFrom(rd); err != nil {
			return fmt.Errorf("update proof %d: %w", i, err)
		}
	}
	var N uint64
	if err := binary.Read(rd, binary.BigEndian, &N); err != nil {
		return err
	}
	if N == 0 || N&(N-1) != 0 || N > 1<<31 {
		return fmt.Errorf("invalid domain size %d", N)
	}
	var c mpcsetup.SrsCommons
	c.G1.Tau = make([]curve.G1Affine, 2*N-1)
	c.G2.Tau = make([]curve.G2Affine, N)
	c.G1.AlphaTau = make([]curve.G1Affine, N)
	c.G1.BetaTau = make([]curve.G1Affine, N)
	_, _, c.G1.Tau[0], c.G2.Tau[0] = curve.Generators()
	b, err := readRun(rd, 1, curve.SizeOfG2AffineCompressed)
	if err != nil {
		return err
	}
	if _, err := c.G2.Beta.SetBytes(b); err != nil {
		return fmt.Errorf("[β]₂: %w", err)
	}
	for _, step := range []struct {
		name string
		run  func() error
	}{
		{"[τⁱ]₁", func() error { return decodeG1(rd, c.G1.Tau[1:]) }},
		{"[τⁱ]₂", func() error { return decodeG2(rd, c.G2.Tau[1:]) }},
		{"[βτⁱ]₁", func() error { return decodeG1(rd, c.G1.BetaTau) }},
		{"[ατⁱ]₁", func() error { return decodeG1(rd, c.G1.AlphaTau) }},
	} {
		if err := step.run(); err != nil {
			return fmt.Errorf("%s: %w", step.name, err)
		}
	}
	if _, _, err := gIo.ReadBytesShort(rd); err != nil {
		return fmt.Errorf("challenge: %w", err)
	}
	if rd.Len() != 0 {
		return errors.New("trailing bytes after the Phase1 object")
	}

	var tau, alpha, beta fr.Element
	proofs := [3]cmpc.UpdateProof{
		cmpc.UpdateValues(&tau, challenge[:], mpcsetup.DST_TAU),
		cmpc.UpdateValues(&alpha, challenge[:], mpcsetup.DST_ALPHA),
		cmpc.UpdateValues(&beta, challenge[:], mpcsetup.DST_BETA),
	}
	if err := scaleG1(c.G1.Tau[1:], &tau, &tau); err != nil {
		return err
	}
	if err := scaleG2(c.G2.Tau[1:], &tau, &tau); err != nil {
		return err
	}
	if err := scaleG1(c.G1.AlphaTau, &alpha, &tau); err != nil {
		return err
	}
	if err := scaleG1(c.G1.BetaTau, &beta, &tau); err != nil {
		return err
	}
	var I big.Int
	beta.BigInt(&I)
	c.G2.Beta.ScalarMultiplication(&c.G2.Beta, &I)

	for i := range proofs {
		if _, err := proofs[i].WriteTo(w); err != nil {
			return err
		}
	}
	if _, err := c.WriteTo(w); err != nil {
		return err
	}
	_, err = gIo.WriteBytesShort(challenge[:], w)
	return err
}

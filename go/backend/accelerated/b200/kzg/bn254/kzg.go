// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build b200

package bn254

import (
	"errors"
	"hash"
	"math/bits"
	"unsafe"

	curve "github.com/consensys/gnark-crypto/ecc/bn254"
	"github.com/consensys/gnark-crypto/ecc/bn254/fr"
	"github.com/consensys/gnark-crypto/ecc/bn254/kzg"
	fiatshamir "github.com/consensys/gnark-crypto/fiat-shamir"
	"github.com/consensys/gnark/backend/accelerated/b200"
	"github.com/consensys/gnark/backend/accelerated/b200/internal/cabi"
)

const curveID = cabi.BN254

// ToLagrangeG1 has the signature of gnark-crypto's kzg.ToLagrangeG1 and computes the same points on device 0: given the
// monomial SRS [tau^k]G1, k < n (n a power of two), it returns the Lagrange basis [L_i(tau)]G1 of the domain
// fft.NewDomain(n), in natural order (b200_points_ntt, inverse). coeffs is left unchanged.
func ToLagrangeG1(coeffs []curve.G1Affine) ([]curve.G1Affine, error) {
	n := len(coeffs)
	if n == 0 || n&(n-1) != 0 {
		return nil, errors.New("invalid input size")
	}
	if err := cabi.Init([]int{0}); err != nil {
		return nil, err
	}
	res := make([]curve.G1Affine, n)
	copy(res, coeffs)
	if err := cabi.PointsNTT(0, curveID, uint32(bits.TrailingZeros(uint(n))), unsafe.Pointer(&res[0]), true); err != nil {
		return nil, err
	}
	return res, nil
}

// DeviceKey is a KZG proving key whose G1 points live on one device: the GPU twin of gnark-crypto's kzg.Commit, Open
// and BatchOpenSinglePoint for that key.  Its results are gnark-crypto's own types, so kzg.Verify and
// kzg.BatchVerifySinglePoint accept them unchanged.
type DeviceKey struct {
	dev   int
	n     int
	table *cabi.Table
}

// NewDeviceKey uploads pk.G1 once to the device chosen by b200.WithDeviceID (device 0 by default).
func NewDeviceKey(pk kzg.ProvingKey, opts ...b200.Option) (*DeviceKey, error) {
	cfg, err := b200.NewConfig(opts...)
	if err != nil {
		return nil, err
	}
	dev := cfg.Devices()[0]
	if len(pk.G1) == 0 {
		return nil, kzg.ErrInvalidPolynomialSize
	}
	if err := cabi.Init([]int{dev}); err != nil {
		return nil, err
	}
	t, err := cabi.UploadTable(dev, curveID, 1, unsafe.Pointer(&pk.G1[0]), len(pk.G1), 0)
	if err != nil {
		return nil, err
	}
	return &DeviceKey{dev: dev, n: len(pk.G1), table: t}, nil
}

// Free releases the device points; safe more than once.
func (k *DeviceKey) Free() {
	if k != nil {
		k.table.Free()
	}
}

// rows packs polynomials into one item-major block of width n (the longest), zero-padded.
func rows(ps [][]fr.Element) ([]fr.Element, int) {
	n := 0
	for _, p := range ps {
		n = max(n, len(p))
	}
	buf := make([]fr.Element, len(ps)*n+1)
	for b, p := range ps {
		copy(buf[b*n:], p)
	}
	return buf, n
}

func affine(j []curve.G1Jac) []curve.G1Affine {
	out := make([]curve.G1Affine, len(j))
	for i := range j {
		out[i].FromJacobian(&j[i])
	}
	return out
}

// Commit is kzg.Commit(p, pk) on the device.
func (k *DeviceKey) Commit(p []fr.Element) (kzg.Digest, error) {
	d, err := k.CommitBatch([][]fr.Element{p})
	if err != nil {
		return kzg.Digest{}, err
	}
	return d[0], nil
}

// CommitBatch commits every polynomial in one batched MSM (b200_msm_batch over the key's points).
func (k *DeviceKey) CommitBatch(ps [][]fr.Element) ([]kzg.Digest, error) {
	for _, p := range ps {
		if len(p) == 0 || len(p) > k.n {
			return nil, kzg.ErrInvalidPolynomialSize
		}
	}
	if len(ps) == 0 {
		return nil, nil
	}
	buf, n := rows(ps)
	jac := make([]curve.G1Jac, len(ps))
	if err := k.table.MSMBatch(0, n, len(ps), unsafe.Pointer(&buf[0]), unsafe.Pointer(&jac[0])); err != nil {
		return nil, err
	}
	return affine(jac), nil
}

// Open is kzg.Open(p, point, pk) on the device.
func (k *DeviceKey) Open(p []fr.Element, point fr.Element) (kzg.OpeningProof, error) {
	o, err := k.OpenBatch([][]fr.Element{p}, []fr.Element{point})
	if err != nil {
		return kzg.OpeningProof{}, err
	}
	return o[0], nil
}

// OpenBatch opens ps[b] at points[b] for every b with one batched division and one batched MSM.
func (k *DeviceKey) OpenBatch(ps [][]fr.Element, points []fr.Element) ([]kzg.OpeningProof, error) {
	if len(ps) != len(points) {
		return nil, errors.New("OpenBatch: one point per polynomial is required")
	}
	for _, p := range ps {
		if len(p) == 0 || len(p)-1 > k.n {
			return nil, kzg.ErrInvalidPolynomialSize
		}
	}
	if len(ps) == 0 {
		return nil, nil
	}
	buf, n := rows(ps)
	values := make([]fr.Element, len(ps))
	jac := make([]curve.G1Jac, len(ps))
	if err := k.table.KZGOpenBatch(unsafe.Pointer(&buf[0]), n, len(ps), false, unsafe.Pointer(&points[0]),
		unsafe.Pointer(&values[0]), unsafe.Pointer(&jac[0])); err != nil {
		return nil, err
	}
	h := affine(jac)
	out := make([]kzg.OpeningProof, len(ps))
	for b := range out {
		out[b] = kzg.OpeningProof{H: h[b], ClaimedValue: values[b]}
	}
	return out, nil
}

// BatchOpenSinglePoint is kzg.BatchOpenSinglePoint(polynomials, digests, point, hf, pk, dataTranscript...) on the
// device: the polynomials go up once, their values at point come from b200_poly_eval_batch, gamma is derived from
// the transcript as gnark-crypto derives it, and H from b200_kzg_fold_open on the same device buffer.
func (k *DeviceKey) BatchOpenSinglePoint(polynomials [][]fr.Element, digests []kzg.Digest, point fr.Element, hf hash.Hash,
	dataTranscript ...[]byte) (kzg.BatchOpeningProof, error) {
	var res kzg.BatchOpeningProof
	if len(polynomials) != len(digests) {
		return res, kzg.ErrInvalidNbDigests
	}
	for _, p := range polynomials {
		if len(p) > k.n {
			return res, kzg.ErrInvalidPolynomialSize
		}
	}
	if len(polynomials) == 0 {
		return res, kzg.ErrInvalidNbDigests
	}
	buf, n := rows(polynomials)
	batch := len(polynomials)
	d, err := cabi.Upload(k.dev, unsafe.Pointer(&buf[0]), batch*n*fr.Bytes)
	if err != nil {
		return res, err
	}
	defer d.Free()
	res.ClaimedValues = make([]fr.Element, batch)
	pts := make([]fr.Element, batch)
	for b := range pts {
		pts[b] = point
	}
	if err := cabi.PolyEvalBatch(k.dev, curveID, d.P, n, batch, true, unsafe.Pointer(&pts[0]),
		unsafe.Pointer(&res.ClaimedValues[0])); err != nil {
		return res, err
	}
	gamma, err := deriveGamma(point, digests, res.ClaimedValues, hf, dataTranscript...)
	if err != nil {
		return res, err
	}
	var h curve.G1Jac
	if err := k.table.KZGFoldOpen(d.P, n, batch, true, unsafe.Pointer(&point), unsafe.Pointer(&gamma),
		unsafe.Pointer(&h)); err != nil {
		return res, err
	}
	res.H.FromJacobian(&h)
	return res, nil
}

// deriveGamma restates gnark-crypto's kzg deriveGamma: gamma binds the point, the digests, the claimed values and the
// caller's transcript data.
func deriveGamma(point fr.Element, digests []kzg.Digest, claimedValues []fr.Element, hf hash.Hash,
	dataTranscript ...[]byte) (fr.Element, error) {
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

// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build b200

package bn254

import (
	"errors"
	"math/bits"
	"unsafe"

	curve "github.com/consensys/gnark-crypto/ecc/bn254"
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

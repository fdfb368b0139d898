// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build !b200

package bn254

import (
	curve "github.com/consensys/gnark-crypto/ecc/bn254"
)

// ToLagrangeG1 is the GPU twin of gnark-crypto's kzg.ToLagrangeG1 (see the b200 build).
func ToLagrangeG1(coeffs []curve.G1Affine) ([]curve.G1Affine, error) {
	panic("b200 backend requested but program compiled without 'b200' build tag")
}

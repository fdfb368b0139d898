// Package bn254 converts a KZG SRS between monomial and Lagrange form on the GPU for the BLS12-381 curve: the drop-in twin of
// gnark-crypto's kzg.ToLagrangeG1 (in-tree statement: lagrangeCoeffsG1, backend/groth16/<curve>/mpcsetup/lagrange.go:21-41),
// which is how a ceremony SRS without a trapdoor gets the Lagrange basis that plonk.Setup takes as srsLagrange.  Its
// DeviceKey holds a KZG proving key on the GPU and gives kzg.Commit, Open and BatchOpenSinglePoint (and batches of the
// first two) in gnark-crypto's own types.
package bls12381

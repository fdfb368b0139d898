// Package bn254 runs the point work of a contribution to gnark's Groth16 MPC ceremony (backend/groth16/<curve>/mpcsetup)
// on the GPU for the BLS12-377 curve.  Every step of a contribution is out[i] = (c * t^i) * P[i] over long point vectors
// (phase1.go:104-147, phase2.go:110-135), which gnark runs one ScalarMultiplication at a time; here each vector is one
// b200_points_scale call, and phase 1's compressed point runs are decoded on the device (b200_points_decode).
package bls12377

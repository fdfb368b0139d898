// Package b200 implements accelerated prover backends for NVIDIA H100 (sm_90a) on top of libgnark_b200.so.
//
// The package layout, the function sets and the option handling follow
// [github.com/consensys/gnark/backend/accelerated/icicle] one to one, so that switching is an import change:
//
//	import b200_groth16 "github.com/consensys/gnark/backend/accelerated/b200/groth16"
//	...
//	pk := b200_groth16.NewProvingKey(ecc.BN254)
//	n, err = pk.ReadFrom(r)
//	...
//	proof, err := b200_groth16.Prove(ccs, pk, witness, b200.WithDeviceID(0))
//
// and, with no precedent in the reference (there is no accelerated PLONK upstream),
//
//	import b200_plonk "github.com/consensys/gnark/backend/accelerated/b200/plonk"
//	proof, err := b200_plonk.Prove(ccs, pk, witness, b200.WithDeviceID(0))
//
// Supported curves: BN254, BLS12-381, BLS12-377, BW6-761 (Groth16 and PLONK).
//
// # Build
//
// The shared library and its header come from the gnark_b200 repository (`python -c "import __graft_entry__ as g;
// g.build()"` or `make -C gnark_b200/csrc`). Point cgo at them and use the `b200` build tag:
//
//	export CGO_CFLAGS="-I$GNARK_B200/include"
//	export CGO_LDFLAGS="-L$GNARK_B200/gnark_b200/lib -lgnark_b200 -Wl,-rpath,$GNARK_B200/gnark_b200/lib"
//	go build -tags=b200 ./...
//
// Without the tag the packages compile to stubs that panic when called, exactly like the `icicle` tag.
//
// # Proving keys
//
// The accelerated proving keys embed the native ones, so `ReadFrom`, `WriteTo`, `ReadDump`, `WriteDump` are inherited
// and the serialised formats are identical. Point tables are copied to the device once per key and device (gnark's
// memory image is the device layout: no Montgomery conversion) and released by [ProvingKey.FreeGPUResources].
//
// # Several GPUs
//
// [WithDeviceIDs] shards every MSM table by point range over the listed devices of one box; a proof then runs one
// goroutine per device and the partial sums are added on the host (five points per device).
//
// # What stays in Go
//
// The constraint solver, the BSB22 hint (only its MSMs run on the device), hashing to the field, the Fiat-Shamir
// transcripts and the sampling of randomness stay in Go, byte for byte as in the CPU provers.
package b200

//go:build b200

// Package cabi is the cgo binding of include/gnark_b200.h shared by the per-curve packages.
//
// Rules the C ABI is designed around (INTEGRATION.md §3):
//   - host pointers are borrowed for the duration of a call only, nothing is retained;
//   - every entry point selects its device itself, so callers need not LockOSThread;
//   - errors are an int32 status plus a message; the message is thread local on the C side, so a failing call and
//     its b200_last_error must run on one OS thread: Call does that.
package cabi

/*
#cgo LDFLAGS: -lgnark_b200
#include <stdlib.h>
#include <gnark_b200.h>
*/
import "C"

import (
	"errors"
	"runtime"
	"sync"
	"unsafe"
)

// Curve identifiers of the C ABI.
const (
	BN254     = int32(C.B200_BN254)
	BLS12_381 = int32(C.B200_BLS12_381)
	BLS12_377 = int32(C.B200_BLS12_377)
	BW6_761   = int32(C.B200_BW6_761)
)

// TablePrecomp is B200_TABLE_PRECOMP.
const TablePrecomp = int32(C.B200_TABLE_PRECOMP)

// Call runs f (a closure around one C call returning the int32 status) on a locked OS thread and turns a non-zero
// status into an error carrying b200_last_error().
func Call(f func() int32) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	if rc := f(); rc != 0 {
		return errors.New(C.GoString(C.b200_last_error()))
	}
	return nil
}

var (
	initOnce sync.Once
	initErr  error
)

// Init is the twin of warmUpDevice (backend/accelerated/icicle/groth16/groth16_icicle.go:38-72): once per process,
// all listed devices.
func Init(devs []int) error {
	initOnce.Do(func() {
		ids := make([]C.int32_t, len(devs))
		for i, d := range devs {
			ids[i] = C.int32_t(d)
		}
		initErr = Call(func() int32 { return int32(C.b200_init(C.int32_t(len(ids)), (*C.int32_t)(unsafe.SliceData(ids)))) })
	})
	if initErr != nil {
		return initErr
	}
	// devices that were not part of the first call are initialised lazily by the library
	return nil
}

// Groth16Key is a device-resident Groth16 proving key (b200_pk_t).
type Groth16Key struct{ h C.b200_pk_t }

// Groth16KeyDesc mirrors b200_groth16_pk_desc with Go types; all pointers are borrowed for LoadGroth16Key only.
type Groth16KeyDesc struct {
	Curve                            int32
	DomainSize                       uint64
	DomainGen, CosetGen              unsafe.Pointer
	G1Alpha, G1Beta, G1Delta         unsafe.Pointer
	G2Beta, G2Delta                  unsafe.Pointer
	G1A, G1B, G1Z, G1K, G2B          unsafe.Pointer
	NA, NB, NZ, NK, NB2              int
	InfinityA, InfinityB             []byte
	NbWires, NbPublic                int
	Flags                            int32
	ShardRank, ShardWorld            int
	KRemoved                         []uint32
	Pin                              []any // everything the pointers above point into
}

// LoadGroth16Key is b200_groth16_pk_load (setupDevicePointers, icicle.go:88-264).
func LoadGroth16Key(dev int, d *Groth16KeyDesc) (*Groth16Key, error) {
	var cd C.b200_groth16_pk_desc
	cd.curve = C.int32_t(d.Curve)
	cd.domain_size = C.uint64_t(d.DomainSize)
	cd.domain_gen, cd.coset_gen = d.DomainGen, d.CosetGen
	cd.g1_alpha, cd.g1_beta, cd.g1_delta = d.G1Alpha, d.G1Beta, d.G1Delta
	cd.g2_beta, cd.g2_delta = d.G2Beta, d.G2Delta
	cd.g1_a, cd.n_a = d.G1A, C.size_t(d.NA)
	cd.g1_b, cd.n_b = d.G1B, C.size_t(d.NB)
	cd.g1_z, cd.n_z = d.G1Z, C.size_t(d.NZ)
	cd.g1_k, cd.n_k = d.G1K, C.size_t(d.NK)
	cd.g2_b, cd.n_b2 = d.G2B, C.size_t(d.NB2)
	cd.infinity_a = (*C.uint8_t)(unsafe.SliceData(d.InfinityA))
	cd.infinity_b = (*C.uint8_t)(unsafe.SliceData(d.InfinityB))
	cd.nb_wires, cd.nb_public = C.size_t(d.NbWires), C.size_t(d.NbPublic)
	cd.flags = C.int32_t(d.Flags)
	cd.shard_rank, cd.shard_world = C.int32_t(d.ShardRank), C.int32_t(d.ShardWorld)
	if len(d.KRemoved) > 0 {
		cd.k_removed = (*C.uint32_t)(unsafe.SliceData(d.KRemoved))
		cd.n_k_removed = C.size_t(len(d.KRemoved))
	}
	// the descriptor holds Go pointers to Go memory: pin them for the call (cgo pointer passing rules)
	var pinner runtime.Pinner
	defer pinner.Unpin()
	for _, p := range d.Pin {
		pinner.Pin(p)
	}
	if len(d.InfinityA) > 0 {
		pinner.Pin(unsafe.SliceData(d.InfinityA))
	}
	if len(d.InfinityB) > 0 {
		pinner.Pin(unsafe.SliceData(d.InfinityB))
	}
	if len(d.KRemoved) > 0 {
		pinner.Pin(unsafe.SliceData(d.KRemoved))
	}
	k := &Groth16Key{}
	if err := Call(func() int32 { return int32(C.b200_groth16_pk_load(C.int32_t(dev), &cd, &k.h)) }); err != nil {
		return nil, err
	}
	return k, nil
}

// Free is b200_groth16_pk_free; safe on a nil key and more than once.
func (k *Groth16Key) Free() {
	if k != nil && k.h != nil {
		C.b200_groth16_pk_free(k.h)
		k.h = nil
	}
}

// Prove is b200_groth16_prove: from the solver's vectors to the three proof points (prove.go:131-315).
// w, a, b, c: first elements of the fr.Vectors; r, s: the two random fr.Elements; ar, bs, krs: the proof's points.
func (k *Groth16Key) Prove(w, a, b, c unsafe.Pointer, nConstraints int, r, s, ar, bs, krs unsafe.Pointer) error {
	return Call(func() int32 {
		return int32(C.b200_groth16_prove(k.h, w, a, b, c, C.size_t(nConstraints), r, s, ar, bs, krs, nil))
	})
}

// ProveBatch is b200_groth16_prove_batch: len(w) proofs of one circuit in one call.  w, a, b, c: one pointer per item to
// the first element of its fr.Vectors (the C arrays of pointers are built here, as Begin does for pi2); r, s: len(w)
// fr.Elements each; ar, bs, krs: len(w) proof points each.
func (k *Groth16Key) ProveBatch(w, a, b, c []unsafe.Pointer, nConstraints int, r, s, ar, bs, krs unsafe.Pointer) error {
	n := len(w)
	if n == 0 {
		return nil
	}
	if len(a) != n || len(b) != n || len(c) != n {
		return errors.New("ProveBatch: w, a, b, c must have one pointer per item")
	}
	arrays := [4]*unsafe.Pointer{}
	for i, src := range [4][]unsafe.Pointer{w, a, b, c} {
		arrays[i] = (*unsafe.Pointer)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(uintptr(0)))))
		defer C.free(unsafe.Pointer(arrays[i]))
		copy(unsafe.Slice(arrays[i], n), src)
	}
	return Call(func() int32 {
		return int32(C.b200_groth16_prove_batch(k.h, C.size_t(n), arrays[0], arrays[1], arrays[2], arrays[3],
			C.size_t(nConstraints), r, s, ar, bs, krs, nil))
	})
}

// MSMs is b200_groth16_msms: this shard's partial sums, 4 G1Jac + 1 G2Jac into out.
func (k *Groth16Key) MSMs(w, a, b, c unsafe.Pointer, nConstraints int, out unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_groth16_msms(k.h, w, a, b, c, C.size_t(nConstraints), out)) })
}

// Assemble is b200_groth16_assemble: the proof from the five complete MSM results.
func (k *Groth16Key) Assemble(msm5, r, s, ar, bs, krs unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_groth16_assemble(k.h, msm5, r, s, ar, bs, krs)) })
}

// PedersenKey is a device-resident pedersen.ProvingKey{Basis, BasisExpSigma} (b200_pedersen_key_t).
type PedersenKey struct {
	h C.b200_pedersen_key_t
	N int
}

// LoadPedersenKey is b200_pedersen_key_load. basis, basisExpSigma: first elements of the G1Affine slices.
func LoadPedersenKey(dev int, curve int32, basis, basisExpSigma unsafe.Pointer, n int) (*PedersenKey, error) {
	k := &PedersenKey{N: n}
	err := Call(func() int32 {
		return int32(C.b200_pedersen_key_load(C.int32_t(dev), C.int32_t(curve), basis, basisExpSigma, C.size_t(n), &k.h))
	})
	if err != nil {
		return nil, err
	}
	return k, nil
}

// Commit is b200_pedersen_commit: Commit (prove.go:84) and ProveKnowledge (prove.go:114) over one upload of the values.
// commitment / pok: G1Affine destinations, either may be nil.
func (k *PedersenKey) Commit(values unsafe.Pointer, n int, commitment, pok unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_pedersen_commit(k.h, values, C.size_t(n), 0, commitment, pok)) })
}

// Free is b200_pedersen_key_free.
func (k *PedersenKey) Free() {
	if k != nil && k.h != nil {
		C.b200_pedersen_key_free(k.h)
		k.h = nil
	}
}

// PlonkKey is a device-resident PLONK proving key (b200_plonk_pk_t).
type PlonkKey struct {
	h    C.b200_plonk_pk_t
	NQcp int
}

// LoadPlonkKey is b200_plonk_pk_load. ql..qk: Lagrange/regular trace columns (n fr.Elements each), perm: trace.S (3n),
// srs: pk.Kzg.G1 (at least n+3 points), qcp: the BSB22 selectors. All pointers are borrowed for the call.
func LoadPlonkKey(dev int, curve int32, log2n uint32, ql, qr, qm, qo, qk unsafe.Pointer, perm []int64, srs unsafe.Pointer,
	qcp []unsafe.Pointer, pin []any) (*PlonkKey, error) {
	var d C.b200_plonk_pk_desc
	d.log2n = C.uint32_t(log2n)
	d.ql, d.qr, d.qm, d.qo, d.qk = ql, qr, qm, qo, qk
	d.perm = (*C.int64_t)(unsafe.SliceData(perm))
	d.srs_canonical = srs
	// the array of selector pointers is C memory: a Go slice of Go pointers may not be passed to C
	var arr *unsafe.Pointer
	if len(qcp) > 0 {
		arr = (*unsafe.Pointer)(C.malloc(C.size_t(len(qcp)) * C.size_t(unsafe.Sizeof(uintptr(0)))))
		defer C.free(unsafe.Pointer(arr))
		copy(unsafe.Slice(arr, len(qcp)), qcp)
		d.n_qcp = C.uint32_t(len(qcp))
		d.qcp = arr
	}
	var pinner runtime.Pinner
	defer pinner.Unpin()
	for _, p := range pin {
		pinner.Pin(p)
	}
	pinner.Pin(unsafe.SliceData(perm))
	k := &PlonkKey{NQcp: len(qcp)}
	if err := Call(func() int32 { return int32(C.b200_plonk_pk_load(C.int32_t(dev), C.int32_t(curve), &d, &k.h)) }); err != nil {
		return nil, err
	}
	return k, nil
}

// Free is b200_plonk_pk_free.
func (k *PlonkKey) Free() {
	if k != nil && k.h != nil {
		C.b200_plonk_pk_free(k.h)
		k.h = nil
	}
}

// PlonkSession is one proof in flight (b200_plonk_session_t), driven one Fiat-Shamir round at a time.
type PlonkSession struct{ h C.b200_plonk_session_t }

// Begin is b200_plonk_begin: commitToLRO (prove.go:404-489). l, r, o: the solved columns; bl, br, bo: 2 blinding
// coefficients each; pi2: the committed BSB22 polynomials (C memory array of pointers is built here); outBsb22: len(pi2)
// G1Jac; outLRO: 3 G1Jac.
func (k *PlonkKey) Begin(l, r, o, bl, br, bo unsafe.Pointer, pi2 []unsafe.Pointer, outBsb22, outLRO unsafe.Pointer) (*PlonkSession, error) {
	var arr *unsafe.Pointer
	if len(pi2) > 0 {
		arr = (*unsafe.Pointer)(C.malloc(C.size_t(len(pi2)) * C.size_t(unsafe.Sizeof(uintptr(0)))))
		defer C.free(unsafe.Pointer(arr))
		copy(unsafe.Slice(arr, len(pi2)), pi2)
	}
	s := &PlonkSession{}
	err := Call(func() int32 {
		return int32(C.b200_plonk_begin(k.h, l, r, o, bl, br, bo, arr, outBsb22, &s.h, outLRO))
	})
	if err != nil {
		return nil, err
	}
	return s, nil
}

// SetQk is b200_plonk_set_qk: this proof's complete Qk (completeQk, prove.go:349-373).
func (s *PlonkSession) SetQk(qk unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_plonk_set_qk(s.h, qk)) })
}

// SetQuotientRandomizers is b200_plonk_set_quotient_randomizers: StatisticalZK, the two quotientShardsRandomizers of
// newInstance (prove.go:239-242), 2 fr.Elements; to be called before Quotient.
func (s *PlonkSession) SetQuotientRandomizers(hr unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_plonk_set_quotient_randomizers(s.h, hr)) })
}

// CommitZ is b200_plonk_commit_z (buildRatioCopyConstraint, prove.go:635-668).
func (s *PlonkSession) CommitZ(beta, gamma, bz, outZ unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_plonk_commit_z(s.h, beta, gamma, bz, outZ)) })
}

// Quotient is b200_plonk_quotient (computeQuotient, prove.go:558-633): outH receives 3 G1Jac.
func (s *PlonkSession) Quotient(alpha, outH unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_plonk_quotient(s.h, alpha, outH)) })
}

// Linearise is b200_plonk_linearise (openZ + computeLinearizedPolynomial, prove.go:670-794): outPoints 2 G1Jac
// (linearised digest, Z-shifted opening quotient), outValues 7 + nQcp fr.Elements.
func (s *PlonkSession) Linearise(zeta, outPoints, outValues unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_plonk_linearise(s.h, zeta, outPoints, outValues)) })
}

// BatchOpen is b200_plonk_batch_open (batchOpening, prove.go:796-837): outPoint receives BatchedProof.H as G1Jac.
func (s *PlonkSession) BatchOpen(v, outPoint unsafe.Pointer) error {
	return Call(func() int32 { return int32(C.b200_plonk_batch_open(s.h, v, outPoint)) })
}

// End is b200_plonk_end; safe at any stage and more than once.
func (s *PlonkSession) End() {
	if s != nil && s.h != nil {
		C.b200_plonk_end(s.h)
		s.h = nil
	}
}

// PointsNTT is b200_points_ntt on a domain of 2^log2n points created for the call with gnark-crypto's fft.NewDomain
// generator: points (2^log2n G1Affine of `curve`, host memory, borrowed for the call) are transformed in place, natural
// order in and out; inverse = monomial SRS -> Lagrange basis (kzg.ToLagrangeG1), otherwise back.
func PointsNTT(dev int, curve int32, log2n uint32, points unsafe.Pointer, inverse bool) error {
	var d C.b200_domain_t
	err := Call(func() int32 {
		return int32(C.b200_ntt_domain_new(C.int32_t(dev), C.int32_t(curve), C.uint32_t(log2n), nil, nil, &d))
	})
	if err != nil {
		return err
	}
	defer C.b200_ntt_domain_free(d)
	inv := C.int32_t(0)
	if inverse {
		inv = 1
	}
	return Call(func() int32 { return int32(C.b200_points_ntt(d, 1, points, 0, inv)) })
}

// PointsScale is b200_points_scale: points[i] <- (c * t^i) * points[i], i < n, in place on n affine points of G1
// (group 1) or G2 (group 2) of `curve` in host memory; c and t point to one fr.Element each, t nil means t = 1.
func PointsScale(dev int, curve, group int32, points unsafe.Pointer, n int, c, t unsafe.Pointer) error {
	return Call(func() int32 {
		return int32(C.b200_points_scale(C.int32_t(dev), C.int32_t(curve), C.int32_t(group), points, C.size_t(n), 0, c, t))
	})
}

// Encodings of b200_points_decode.
const (
	PointsRaw        = int32(C.B200_POINTS_RAW)
	PointsCompressed = int32(C.B200_POINTS_COMPRESSED)
)

// PointsDecode is b200_points_decode: n points in gnark-crypto's fixed-size encoding (PointsRaw / PointsCompressed) to n
// affine points of G1 or G2 in host memory at out.
func PointsDecode(dev int, curve, group int32, data []byte, n int, encoding int32, out unsafe.Pointer) error {
	if n == 0 {
		return nil
	}
	return Call(func() int32 {
		return int32(C.b200_points_decode(C.int32_t(dev), C.int32_t(curve), C.int32_t(group), unsafe.Pointer(&data[0]),
			C.size_t(n), C.int32_t(encoding), out, 0))
	})
}

// Table is a device-resident MSM base table (b200_table_t).
type Table struct {
	h C.b200_table_t
	N int
}

// UploadTable is b200_table_upload: n affine points of `group` (1 or 2) from host memory (borrowed for the call).
// flags: 0 for a plain table, TablePrecomp for one with the precomputed window slabs.
func UploadTable(dev int, curve, group int32, points unsafe.Pointer, n int, flags int32) (*Table, error) {
	t := &Table{N: n}
	err := Call(func() int32 {
		return int32(C.b200_table_upload(C.int32_t(dev), C.int32_t(curve), C.int32_t(group), points, C.size_t(n), C.int32_t(flags), &t.h))
	})
	if err != nil {
		return nil, err
	}
	return t, nil
}

// MSMIndexed is b200_msm_indexed: sum_j scalars[j] * bases[idx[j]] into out (one G?Jac). idx and scalars (len(idx)
// fr.Elements) are host memory borrowed for the call; every index must be below the table's point count.
func (t *Table) MSMIndexed(idx []uint32, scalars, out unsafe.Pointer) error {
	var pinner runtime.Pinner
	defer pinner.Unpin()
	var ip *C.uint32_t
	if len(idx) > 0 {
		pinner.Pin(unsafe.SliceData(idx))
		ip = (*C.uint32_t)(unsafe.SliceData(idx))
	}
	return Call(func() int32 { return int32(C.b200_msm_indexed(t.h, ip, C.size_t(len(idx)), 0, scalars, 0, out)) })
}

// MSMBatch is b200_msm_batch: out[b] = sum_{i<n} scalars[b*n + i] * bases[off + i] for b < batch (batch G?Jac).
// scalars (batch*n fr.Elements, item-major) and out are host memory borrowed for the call.
func (t *Table) MSMBatch(off, n, batch int, scalars, out unsafe.Pointer) error {
	return Call(func() int32 {
		return int32(C.b200_msm_batch(t.h, C.size_t(off), C.size_t(n), C.size_t(batch), scalars, 0, out))
	})
}

// KZGOpenBatch is b200_kzg_open_batch on a G1 SRS table: kzg.Open of `batch` polynomials of n coefficients (polys,
// item-major, on the device when onDev, else host memory borrowed for the call) at points (batch fr.Elements); values
// (batch fr.Elements) and proofs (batch G1Jac) are host memory.
func (t *Table) KZGOpenBatch(polys unsafe.Pointer, n, batch int, onDev bool, points, values, proofs unsafe.Pointer) error {
	return Call(func() int32 {
		return int32(C.b200_kzg_open_batch(t.h, polys, C.size_t(n), C.size_t(batch), boolInt(onDev), points, values, proofs))
	})
}

// KZGFoldOpen is b200_kzg_fold_open: the H of kzg.BatchOpenSinglePoint (one G1Jac to proof) of `batch` polynomials of
// n coefficients folded with powers of gamma, opened at z.
func (t *Table) KZGFoldOpen(polys unsafe.Pointer, n, batch int, onDev bool, z, gamma, proof unsafe.Pointer) error {
	return Call(func() int32 {
		return int32(C.b200_kzg_fold_open(t.h, polys, C.size_t(n), C.size_t(batch), boolInt(onDev), z, gamma, proof))
	})
}

// PolyEvalBatch is b200_poly_eval_batch: values[b] = p_b(points[b]) for `batch` polynomials of n coefficients.
func PolyEvalBatch(dev int, curve int32, polys unsafe.Pointer, n, batch int, onDev bool, points, values unsafe.Pointer) error {
	return Call(func() int32 {
		return int32(C.b200_poly_eval_batch(C.int32_t(dev), C.int32_t(curve), polys, C.size_t(n), C.size_t(batch),
			boolInt(onDev), points, values))
	})
}

// DeviceBuffer is device memory from b200_alloc, filled from host memory with b200_h2d.
type DeviceBuffer struct {
	dev int
	P   unsafe.Pointer
}

// Upload copies `bytes` bytes of host memory (borrowed for the call) into a new device buffer on dev.
func Upload(dev int, src unsafe.Pointer, bytes int) (*DeviceBuffer, error) {
	b := &DeviceBuffer{dev: dev}
	if err := Call(func() int32 { return int32(C.b200_alloc(C.int32_t(dev), C.size_t(bytes), &b.P)) }); err != nil {
		return nil, err
	}
	if bytes > 0 {
		if err := Call(func() int32 { return int32(C.b200_h2d(C.int32_t(dev), b.P, src, C.size_t(bytes))) }); err != nil {
			b.Free()
			return nil, err
		}
	}
	return b, nil
}

// Free is b200_free; safe on a nil buffer and more than once.
func (b *DeviceBuffer) Free() {
	if b != nil && b.P != nil {
		C.b200_free(C.int32_t(b.dev), b.P)
		b.P = nil
	}
}

func boolInt(v bool) C.int32_t {
	if v {
		return 1
	}
	return 0
}

// Free is b200_table_free; safe on a nil table and more than once.
func (t *Table) Free() {
	if t != nil && t.h != nil {
		C.b200_table_free(t.h)
		t.h = nil
	}
}

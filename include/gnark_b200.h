/* libgnark_b200.so - C ABI of the H100 (sm_90a) prover-arithmetic backend for gnark.
 *
 * This is the drop-in boundary for the Groth16 / PLONK prover hot path: every
 * entry point below is what a cgo shim package backend/accelerated/b200/... would
 * bind, in place of the icicle-gnark cgo calls the reference makes from
 * backend/accelerated/icicle/groth16/<curve>/icicle.go (cited per function).
 * The Go-side binding is shown in INTEGRATION.md.
 *
 * Conventions
 *  - Every function returns int32_t: 0 = success, non-zero = failure with a
 *    thread-local message available from b200_last_error().  Nothing aborts or
 *    throws across the ABI (reference: EIcicleError.AsString(), panics in
 *    RunOnDevice closures icicle.go:122,164,200).
 *  - All field elements / points use gnark-crypto's in-memory layout, unchanged:
 *    fr.Element / fp.Element = [Limbs]uint64 little-endian, Montgomery form
 *    (R = 2^(64*Limbs)); G1Affine {X,Y}; G2Affine {X{A0,A1},Y{A0,A1}}; affine
 *    infinity = (0,0); G1Jac/G2Jac {X,Y,Z} with x = X/Z^2, y = Y/Z^3.
 *    No Montgomery conversion is ever required of the caller
 *    (reference: FromMontgomery/AffineFromMontgomery icicle.go:121,322,350,1008).
 *  - Host pointers are borrowed only for the duration of the call (cgo pointer
 *    rule); device pointers come from b200_alloc.
 *  - Every call takes a device id or a handle bound to one and selects the device
 *    itself (thread-local), so callers need not pin OS threads
 *    (reference: icicle_runtime.RunOnDevice).
 */
#ifndef GNARK_B200_H
#define GNARK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* curve ids (ecc.ID order used by backend/accelerated/icicle/groth16/groth16_icicle.go:85-96) */
enum {
  B200_BN254 = 0,
  B200_BLS12_381 = 1,
  B200_BLS12_377 = 2,
  B200_BW6_761 = 3
};

enum { B200_DIF = 0, B200_DIT = 1 }; /* fft.DIF / fft.DIT */

/* b200_table_upload flags */
enum {
  B200_TABLE_PRECOMP = 1,      /* also build 2^(c*w)*P slabs on device (one bucket set per MSM) */
  B200_TABLE_SRC_ON_DEVICE = 2 /* `points` is a device pointer */
};

typedef struct b200_table_s* b200_table_t;   /* device-resident MSM base table  */
typedef struct b200_domain_s* b200_domain_t; /* device-resident fft.Domain      */
typedef struct b200_pk_s* b200_pk_t;         /* device-resident Groth16 proving key */

/* ---- runtime (replaces warmUpDevice, groth16_icicle.go:38-72) ---------------- */
const char* b200_version(void);
const char* b200_last_error(void);
int32_t b200_device_count(int32_t* out_count);
int32_t b200_init(int32_t n_dev, const int32_t* dev_ids); /* idempotent; NULL/0 = device 0 */
int32_t b200_shutdown(void);
/* run subsequent work of `dev` on the caller's CUDA stream (cudaStream_t), NULL = library stream */
int32_t b200_set_stream(int32_t dev, void* cuda_stream);
int32_t b200_sync(int32_t dev);

/* ---- memory (replaces HostSlice.CopyToDevice / DeviceSlice.Free, ~70 sites) -- */
int32_t b200_alloc(int32_t dev, size_t bytes, void** out_dev_ptr);
int32_t b200_free(int32_t dev, void* dev_ptr);
int32_t b200_h2d(int32_t dev, void* dst_dev, const void* src_host, size_t bytes);
int32_t b200_d2h(int32_t dev, void* dst_host, const void* src_dev, size_t bytes);
int32_t b200_host_alloc(size_t bytes, void** out_pinned); /* C-owned pinned staging buffers */
int32_t b200_host_free(void* pinned);

/* ---- MSM base tables (replaces loadG1/loadG1Raw/loadG2 icicle.go:319-359,
 *      PinToGPU uploads :185-261, FreeGPUResources :1493-1549) ---------------- */
int32_t b200_table_upload(int32_t dev, int32_t curve, int32_t group /*1|2*/, const void* points_affine_mont,
                          size_t n, int32_t flags, b200_table_t* out);
/* Table straight from a file region: n affine points (gnark memory layout) starting at byte_offset of `path` - the payload
 * of one point slice of gnark's ProvingKey dump (ProvingKey.WriteDump / ReadDump, backend/groth16/bn254/marshal.go:375-539:
 * G1.A, G1.B, G1.Z, G1.K, G2.B and the commitment bases are written by unsafe.WriteSlice as raw memory images; SURVEY.md
 * §8f-1).  The file is read through two pinned slots while the previous chunk is copied to the device; no host copy of the
 * slice is ever made.  The caller (the Go shim, which reads the dump's header with gnark-crypto's decoder) supplies the
 * payload offset; a point-range shard supplies the offset and count of ITS range. */
int32_t b200_table_upload_file(int32_t dev, int32_t curve, int32_t group /*1|2*/, const char* path, uint64_t byte_offset,
                               size_t n, int32_t flags, b200_table_t* out);
/* Table from a point slice in gnark-crypto's SERIALISED encoding - what backend/plonk/<curve>/marshal.go:96-129 writes
 * for pk.Kzg / pk.KzgLagrange and backend/groth16/<curve>/marshal.go:136-214 for the Groth16 slices outside the dump
 * format: after the encoder's uint32 length, n points of fixed size, big-endian canonical coordinates with metadata
 * bits in the first byte (B200_POINTS_COMPRESSED = what WriteTo emits, x only, sizeof(fp) bytes per G1 point;
 * B200_POINTS_RAW = what WriteRawTo emits, x || y).  The bytes are uploaded as they are and decoded on the device, one
 * thread per point: byte order, Montgomery form, and for compressed points the square root that dominates ReadFrom on the
 * CPU.  Compressed and raw: G1 and G2 of every curve (square roots by exponentiation where p = 3 mod 4, Tonelli-Shanks
 * for BLS12-377; in Fp2 by the norm).  Each point is
 * checked to be canonical and on the curve (G1); subgroup membership is not checked, as with UnsafeReadFrom.  An
 * invalid point fails the call and names its index. */
enum { B200_POINTS_RAW = 1, B200_POINTS_COMPRESSED = 2 };
int32_t b200_table_upload_encoded(int32_t dev, int32_t curve, int32_t group, const void* bytes, size_t n,
                                  int32_t encoding, int32_t flags, b200_table_t* out);
int32_t b200_table_free(b200_table_t t);
int32_t b200_table_info(b200_table_t t, size_t* n, int32_t* window_bits, int32_t* n_windows, int32_t* precomp,
                        size_t* device_bytes);

/* ---- MSM (replaces msmChunkedG1/G2 icicle.go:362-467 + projectiveToGnarkAffine
 *      :266-315; CPU twin G1Jac/G2Jac.MultiExp prove.go:194,207,227,237,283) ---
 * out = sum_{i<n} scalars[i] * bases[off+i] as ONE Jacobian point (gnark layout).
 * Handles n = 0, zero scalars, (0,0) bases, repeated and opposite points. */
int32_t b200_msm(b200_table_t bases, size_t off, size_t n, const void* scalars_mont, int32_t scalars_on_dev,
                 void* out_jac_host);
int32_t b200_msm_g1(b200_table_t bases, size_t off, size_t n, const void* scalars_mont, int32_t scalars_on_dev,
                    void* out_g1jac_host);
int32_t b200_msm_g2(b200_table_t bases, size_t off, size_t n, const void* scalars_mont, int32_t scalars_on_dev,
                    void* out_g2jac_host);
/* stream-ordered variant: all pointers on device, no synchronisation */
int32_t b200_msm_async(b200_table_t bases, size_t off, size_t n, const void* d_scalars_mont, void* d_out_jac);

/* pipelined variant: as b200_msm_async, but the reduction tail of this MSM is placed on a second
 * stream so it overlaps the NEXT b200_msm_pipelined call (a Groth16 proof issues five MSMs back
 * to back; the reference overlaps its four G1 MSMs on CPU cores, prove.go:296-304).  d_out_jac is
 * valid on the device stream only after b200_msm_join (or b200_sync). */
int32_t b200_msm_pipelined(b200_table_t bases, size_t off, size_t n, const void* d_scalars_mont, void* d_out_jac);
int32_t b200_msm_join(int32_t dev);

/* Asynchronous MSM from HOST buffers, for a stream of MSMs (the reference issues its MSMs from concurrent
 * goroutines, prove.go:186-292): scalar upload, compute, reduction tail and result download of consecutive
 * calls overlap.  scalars_host (n fr.Elements) and out_jac_host (one G?Jac) must be b200_host_alloc memory
 * and stay untouched until b200_sync(dev) returns; results are valid after b200_sync. */
int32_t b200_msm_submit(b200_table_t bases, size_t off, size_t n, const void* scalars_host, void* out_jac_host);
/* the same with the result left on the device (valid on the device stream after b200_msm_join): what a sharded MSM
 * needs, whose partial results pass through b200_points_allreduce before one download of the totals */
int32_t b200_msm_submit_dev(b200_table_t bases, size_t off, size_t n, const void* scalars_host, void* d_out_jac);

/* step profile (the reference's ICICLE_STEP_PROFILE timers, icicle.go:72-75,1088-1094):
 * device milliseconds of the 7 pipeline stages of one MSM - decompose, sort,
 * offsets+task scan, accumulate, combine, reduce chunks, set sum+finish. */
int32_t b200_msm_profile(b200_table_t bases, size_t off, size_t n, const void* d_scalars_mont, void* d_out_jac,
                         float* stage_ms /* [7] */);

/* host-side group helpers for combining partial results (the reference sums its
 * per-chunk MSM results on the host in Go, icicle.go:383-411; multi-GPU shards are
 * combined the same way).  Pure CPU, no device needed. */
int32_t b200_point_add_jac(int32_t curve, int32_t group, void* acc_jac, const void* q_jac);
int32_t b200_point_to_affine(int32_t curve, int32_t group, const void* p_jac, void* out_affine);

/* ---- multi-GPU (SURVEY.md 8b "NCCL comm when n_dev>1", 8e) ---------------------------------------------------
 * The path shards by point range: every device owns the table shard of its range and produces one partial point per
 * MSM; the only exchange is a gather of `world` points followed by world-1 group additions - the multi-device twin of
 * the reference's host-side chunk loop (icicle.go:383-411; the reference itself drives one device per proof,
 * opts.go:68-77).  The library owns one NCCL communicator per device (bound at run time: without NCCL everything
 * single-GPU still works) and does gather + additions on the device, on the device's stream.
 *   one process per GPU : rank 0 calls b200_comm_unique_id, ships the 128 bytes to the other ranks by any means
 *                         (the Go shim: its own RPC; the Python harness: torch.distributed broadcast), every rank
 *                         calls b200_comm_init(dev, world, rank, id).
 *   one process, N GPUs : b200_comm_init_all(n, dev_ids); afterwards each device's calls come from its own thread
 *                         (goroutine), as NCCL requires for collectives issued without a group. */
#define B200_COMM_ID_BYTES 128
int32_t b200_comm_unique_id(void* out_id128);
int32_t b200_comm_init(int32_t dev, int32_t world, int32_t rank, const void* id128);
int32_t b200_comm_init_all(int32_t n_dev, const int32_t* dev_ids);
int32_t b200_comm_destroy(int32_t dev);
int32_t b200_comm_info(int32_t dev, int32_t* out_world, int32_t* out_rank);
/* d_totals[k] = sum over ranks of that rank's d_partials[k], k < count (G?Jac, device memory, may alias): one
 * ncclAllGather of world*count points + one fold kernel, stream-ordered, no host synchronisation.  count is the
 * number of results combined at once (5 for a Groth16 proof, K for a stream of MSMs).  No communicator: a copy. */
int32_t b200_points_allreduce(int32_t dev, int32_t curve, int32_t group, const void* d_partials_jac, size_t count,
                              void* d_totals_jac);
/* the reduction half alone: d_gathered = world rows of count G?Jac points (row r = source r), d_totals[k] = sum over
 * rows of d_gathered[r][k]; for callers that move the partial points themselves */
int32_t b200_points_fold(int32_t dev, int32_t curve, int32_t group, const void* d_gathered_jac, uint32_t world,
                         uint32_t count, void* d_totals_jac);
/* b200_msm of this rank's shard + the combine: out_jac_host = the full sum, on every rank */
int32_t b200_msm_allreduce(b200_table_t bases, size_t off, size_t n, const void* scalars_mont, int32_t scalars_on_device,
                           void* out_jac_host);

/* ---- witness-side MSMs (SURVEY.md 8a-a8, 8f-4) ----------------------------------------------------------------
 * gather-index MSM: sum_j scalars[idx[j]] * bases[off + j], j < n_idx.  The table holds the bases that are not the
 * point at infinity; idx lists the wires they belong to, so the solver's wire vector is used as is - replaces the
 * filtered copies of backend/groth16/bn254/prove.go:147-168 ("worst memory allocation offender", :232; GPU twin
 * icicle.go:1018-1070).  idx / scalars: host or device memory. */
int32_t b200_msm_gather(b200_table_t bases, size_t off, const uint32_t* idx, size_t n_idx, int32_t idx_on_device,
                        const void* scalars_mont, size_t n_scalars, int32_t scalars_on_device, void* out_jac_host);
/* sum_{j<n} scalars[j] * bases[idx[j]]: bases picked from the table by index (any order, repeats allowed, each < the
 * table's point count); idx / scalars host or device; out: one G?Jac on the host.  The sparse twin of b200_msm
 * (e.g. kzg.Commit of a mostly-zero Lagrange-form vector, the BSB22 hint) - cost follows n, not the table size.
 * b200_msm_gather indexes the other side: there the scalars are picked (scalars[idx[j]]) and the bases are a
 * contiguous range.  On a plain table the window comes from n; a precomputed table keeps the window its slabs were
 * built for.  Every index is checked before a point is read: host indices on the host, device indices by a check
 * kernel whose verdict is downloaded (one synchronisation) before the MSM runs.  An index out of range fails the call,
 * names its position and leaves out_jac_host untouched.  n = 0 gives the point at infinity. */
int32_t b200_msm_indexed(b200_table_t bases, const uint32_t* idx, size_t n, int32_t idx_on_device,
                         const void* scalars_mont, int32_t scalars_on_device, void* out_jac_host);
/* out[b] = sum_{i<n} scalars[b*n + i] * bases[off + i], b < batch: `batch` MSMs over ONE base range of one table
 * (ICICLE's BatchSize with ArePointsSharedInBatch).  scalars: batch*n fr.Elements (Montgomery), item-major, host or
 * device; out_jac_host: batch G?Jac (the table's group) in gnark layout.  The batch runs as one MSM pipeline whose bucket
 * sets are the items' sets side by side: one sort, one accumulate and one reduction tail for all items.  On a plain table
 * the window comes from n; a precomputed table keeps the window its slabs were built for.  Limits, checked before anything
 * is allocated or launched (a violation fails the call, names the limit and leaves out_jac_host untouched):
 * off + n <= the table's point count, batch * n * windows < 2^31, batch * bucket sets * 2^(c-1) < 2^31 - 1.
 * batch = 0 writes nothing; n = 0 writes `batch` points at infinity.  Joins pending pipelined MSMs first. */
int32_t b200_msm_batch(b200_table_t bases, size_t off, size_t n, size_t batch, const void* scalars_mont,
                       int32_t scalars_on_dev, void* out_jac_host);

/* Pedersen / BSB22 commitment keys (gnark-crypto pedersen.ProvingKey{Basis, BasisExpSigma}, one per commitment:
 * ProvingKey.CommitmentKeys, backend/groth16/bn254/setup.go:46).  b200_pedersen_commit runs
 *   commitment = sum_i values[i] * Basis[i]            (pk.CommitmentKeys[i].Commit,         prove.go:84, inside the solver hint)
 *   pok        = sum_i values[i] * BasisExpSigma[i]    (pk.CommitmentKeys[i].ProveKnowledge, prove.go:114)
 * over ONE upload of the values (either output may be NULL); results are G1Affine in gnark layout.  n must equal the
 * basis length (gnark-crypto returns an error otherwise).  b200_pedersen_fold is ProofOfKnowledge.Fold (prove.go:127):
 * sum_i challenge^i * poks[i], host CPU.  Hashing the commitment into the hint's output (prove.go:90-98) stays in Go. */
typedef struct b200_pedersen_key_s* b200_pedersen_key_t;
int32_t b200_pedersen_key_load(int32_t dev, int32_t curve, const void* basis_affine, const void* basis_exp_sigma_affine,
                               size_t n, b200_pedersen_key_t* out);
int32_t b200_pedersen_key_free(b200_pedersen_key_t key);
int32_t b200_pedersen_commit(b200_pedersen_key_t key, const void* values_mont, size_t n, int32_t values_on_device,
                             void* out_commitment_affine, void* out_pok_affine);
int32_t b200_pedersen_fold(int32_t curve, const void* poks_affine, size_t count, const void* challenge_mont,
                           void* out_affine);

/* fixed-base batch: out[i] = scalars[i] * base, n affine points in gnark layout (replaces gnark-crypto's
 * curve.BatchScalarMultiplicationG1/G2 as called by Groth16 Setup, backend/groth16/bn254/setup.go:233,302,
 * and by the SRS generators test/unsafekzg/kzgsrs.go:198 - SURVEY.md §8(f)-3).  base_affine: ONE point on the
 * host; scalars: n fr.Elements (Montgomery), host or device; out: n G?Affine, host or device.  Windowed table
 * of the base built on the device per call (window by batch size), results converted to affine with batched
 * inversions. */
int32_t b200_fixed_base_batch(int32_t dev, int32_t curve, int32_t group, const void* base_affine,
                              const void* scalars_mont, int32_t scalars_on_device, size_t n, void* out_affine,
                              int32_t out_on_device);

/* ---- NTT (replaces icicle_ntt.InitDomain/ReleaseDomain icicle.go:151,163 and
 *      Ntt :1425,1428,1474; CPU twin fft.Domain.FFT/FFTInverse prove.go:362-386) -
 * generator / coset_gen: one fr.Element (Montgomery) each, NULL = gnark-crypto's
 * fft.NewDomain defaults (Generator of order 2^log2n, FrMultiplicativeGen).
 * One domain per handle: no process-global NTT state (the reference serialises all
 * proofs on nttDomainMu / deviceProveMu, icicle.go:53-60). */
int32_t b200_ntt_domain_new(int32_t dev, int32_t curve, uint32_t log2n, const void* generator_mont,
                            const void* coset_gen_mont, b200_domain_t* out);
int32_t b200_ntt_domain_free(b200_domain_t d);
/* in place on `data` (2^log2n fr.Elements).  DIF: natural -> bit-reversed; DIT:
 * bit-reversed -> natural; inverse scales by 1/n; on_coset as fft.OnCoset(). */
int32_t b200_ntt(b200_domain_t d, void* data, int32_t data_on_dev, int32_t inverse, int32_t decimation,
                 int32_t on_coset);
int32_t b200_ntt_async(b200_domain_t d, void* d_data, int32_t inverse, int32_t decimation, int32_t on_coset);
/* `batch` transforms of the domain's size in one call (ICICLE's NTTConfig.BatchSize): data holds batch * 2^log2n
 * fr.Elements item-major, each vector transformed as b200_ntt would.  batch = 0 does nothing. */
int32_t b200_ntt_batch(b200_domain_t d, void* data, size_t batch, int32_t data_on_dev, int32_t inverse,
                       int32_t decimation, int32_t on_coset);
/* Group-element NTT: a KZG SRS between monomial form [tau^k]G and the Lagrange basis [L_i(tau)]G (SURVEY.md §8(f)-3).
 * Replaces gnark-crypto's kzg.ToLagrangeG1 (as used at std/recursion/plonk/verifier_test.go:370; in-tree statement
 * lagrangeCoeffsG1, backend/groth16/<curve>/mpcsetup/lagrange.go:21-41), the route of a ceremony SRS without a trapdoor;
 * test/unsafekzg/kzgsrs.go:184 takes the trapdoor shortcut instead.  points_affine: 2^log2n G1Affine of the domain's
 * curve, host or device, transformed in place with the domain's generator w (its coset is not used):
 *   inverse = 1 (monomial -> Lagrange): out[i] = (1/n) sum_k w^(-ik) in[k]
 *   inverse = 0 (Lagrange -> monomial): out[k] = sum_i w^(ik) in[i]
 * Natural order in and out; results are canonical affine points ((0,0) = infinity); n = 1 leaves the input unchanged.
 * Synchronous.  group must be 1: G2 is not supported. */
int32_t b200_points_ntt(b200_domain_t d, int32_t group, void* points_affine, int32_t points_on_dev, int32_t inverse);

/* ---- Groth16 MPC contributions (SURVEY.md §8(f)-3) ----------------------------------------------------------------
 * Every step of a contribution to gnark's ceremony (backend/groth16/<curve>/mpcsetup) is out[i] = (c * t^i) * P[i]:
 *   phase 1, SrsCommons.update (phase1.go:104-147), domain size N:
 *     G1.Tau[1 .. 2N-2] and G2.Tau[1 .. N-1]   (c, t) = (tau', tau')
 *     G1.AlphaTau[0 .. N-1]                     (c, t) = (alpha', tau')
 *     G1.BetaTau[0 .. N-1]                      (c, t) = (beta', tau')     (and the single point G2.Beta *= beta')
 *   phase 2, Phase2.update (phase2.go:110-135):
 *     G1.Z, G1.PKK                              c = 1/delta', t = 1
 *     G1.SigmaCKK[j]                            c = sigma_j, t = 1         (and G1.Delta, G2.Delta, G2.Sigma[j])
 * b200_points_scale: points[i] <- (c * t^i) * points[i], i < n (t^0 = 1; t = NULL means t = 1), in place on n affine
 * points of G1 or G2 of `curve` (group 1 or 2; BW6-761's G2 is over Fp), host or device buffer.  c, t: one fr.Element
 * each (Montgomery) on the host.  The scalars are built on the device (b200_vec_scale_powers' kernel on a vector of
 * ones); one thread per point runs a double-and-add with mixed additions over the canonical scalar, and the
 * results are canonical affine points ((0,0) = infinity).  Points are not checked to be on the curve, as with gnark's
 * ScalarMultiplication.  n = 0 does nothing; c = 0 gives n points at infinity.  Synchronous; joins pending pipelined
 * MSMs first.  Refused before anything is launched, with the argument named and the buffer untouched: an unknown curve or
 * group, a null c, null points with n > 0, n >= 2^32. */
int32_t b200_points_scale(int32_t dev, int32_t curve, int32_t group, void* points_affine, size_t n, int32_t points_on_dev,
                          const void* c_mont, const void* t_mont);
/* n points in gnark-crypto's serialised encoding (B200_POINTS_RAW / B200_POINTS_COMPRESSED, as for
 * b200_table_upload_encoded: what the Encoder writes for each point of SrsCommons and Phase2, marshal.go:19-57,157-179)
 * -> n affine points in gnark layout, out_affine on the host or the device.  bytes: n * (point size) bytes on the host.
 * The decoder of b200_table_upload_encoded, with its checks: canonical coordinates and, except for raw G2, on the curve;
 * subgroup membership is not checked, as with UnsafeReadFrom.  An invalid point fails the call, names its index and
 * leaves out_affine untouched.  Refused before anything is launched: an unknown curve, group or encoding, null
 * bytes or out with n > 0, n >= 2^32.  n = 0 does nothing.  Synchronous. */
int32_t b200_points_decode(int32_t dev, int32_t curve, int32_t group, const void* bytes, size_t n, int32_t encoding,
                           void* out_affine, int32_t out_on_dev);

/* ---- Groth16 quotient (replaces computeH icicle.go:1391-1488; CPU twin
 *      prove.go:346-389).  a,b,c: `len` fr.Elements each (len <= n, zero padded
 *      internally); h_out: n elements, BIT-REVERSED order, Montgomery - directly
 *      usable as the scalars of MSM(G1.Z, h[:n-1]). */
int32_t b200_groth16_compute_h(b200_domain_t d, const void* a, const void* b, const void* c, size_t len,
                               int32_t inputs_on_dev, void* h_out, int32_t out_on_dev);

/* ---- element-wise vector ops on device vectors (replaces icicle_vecops.VecOp
 *      icicle.go:1455-1461 and the PLONK pointwise loops plonk/bn254/prove.go:
 *      953-1076,1312-1317) ---------------------------------------------------- */
enum { B200_VEC_MUL = 0, B200_VEC_ADD = 1, B200_VEC_SUB = 2 };
int32_t b200_vec_op(int32_t dev, int32_t curve, int32_t op, void* d_out, const void* d_a, const void* d_b, size_t n);
int32_t b200_vec_bit_reverse(int32_t dev, int32_t curve, void* d_data, uint32_t log2n);
/* out[i] = a[i] * s * g^i */
int32_t b200_vec_scale_powers(int32_t dev, int32_t curve, void* d_data, size_t n, const void* s_mont,
                              const void* g_mont);

int32_t b200_vec_batch_invert(int32_t dev, int32_t curve, void* d_data, size_t n); /* 0 stays 0 */
/* y[i] += a * x[i]  (linear combinations: linearised polynomial plonk/bn254/prove.go:1431-1480, opening folds) */
int32_t b200_vec_axpy(int32_t dev, int32_t curve, void* d_y, const void* a_mont, const void* d_x, size_t n);

/* ---- PLONK quotient building blocks (no accelerated PLONK exists in the reference; these are
 *      the device twins of backend/plonk/bn254/prove.go computeNumerator :841-1123 and
 *      divideByZH :1287-1324).  One call evaluates gate + alpha*permutation + alpha^2*L1
 *      constraints on ONE coset of the small domain and scatters the n values into the
 *      bit-reversed rho*n result vector (cres[bitrev(rho*j+i)], :1070-1076).
 *      Inputs are the 12 polynomials already evaluated on that coset (iFFT-DIF, then FFT-DIT
 *      on the coset through b200_ntt with the matching coset generator, as :1035-1057). */
typedef struct {
  const void *l, *r, *o, *z, *s1, *s2, *s3, *ql, *qr, *qm, *qo, *qk; /* device, n fr.Elements each */
  const void *alpha, *beta, *gamma;                                  /* host, one fr.Element each */
  const void *bl, *br, *bo, *bz;                                     /* host, blinding poly coeffs */
  int32_t nbl, nbr, nbo, nbz;                                        /* their lengths (<= 4)       */
  uint32_t coset_index;                                              /* i in [0, rho)              */
  uint32_t rho;                                                      /* |domain1| / |domain0|      */
  void* out;                                                         /* device, rho*n elements     */
} b200_plonk_coset_args;
int32_t b200_plonk_constraints_coset(b200_domain_t domain0, const void* domain1_coset_gen_mont,
                                     const void* domain1_gen_mont, const b200_plonk_coset_args* args);
/* BSB22 commitment gates (gateConstraint :881-884: + sum_i Qcp_i * PI2_i): after b200_plonk_constraints_coset has
 * written coset `coset_index`, one call per commitment adds qcp[j] * pi2[j] (both already ON that coset, regular
 * layout, n elements) to the slot of point j. */
int32_t b200_plonk_bsb22_coset(b200_domain_t domain0, const void* d_qcp, const void* d_pi2, uint32_t coset_index,
                               uint32_t rho, void* d_out);
/* r[i] *= 1/(X^n-1) on the big coset (indexing rule of :1312-1317), then
 * FFTInverse(DIT, OnCoset) on domain1: LagrangeCoset/BitReverse -> Canonical/Regular, in place. */
int32_t b200_plonk_divide_by_zh(b200_domain_t domain1, uint32_t domain0_log2n, void* d_data);

/* ---- O(n) scans of the PLONK prover (SURVEY.md §8 a11): keep every polynomial device-resident
 *      between the MSM / NTT stages.  */
enum { B200_SCAN_PRODUCT = 0, B200_SCAN_SUM = 1 };
int32_t b200_vec_scan(int32_t dev, int32_t curve, int32_t op, void* d_data, size_t n, int32_t exclusive);
/* iop.BuildRatioCopyConstraint (plonk/bn254/prove.go:645-656): Z[0] = 1,
 * Z[i+1] = Z[i] * prod_j (f_j[i] + beta*id_j[i] + gamma) / (f_j[i] + beta*supp[S[j*n+i]] + gamma), f = (L, R, O)
 * in Lagrange/regular form on domain0; S = the trace permutation (int64[3n], plonk/bn254/setup.go:289-392);
 * supp = <w> || g<w> || g^2<w> (getSupportPermutation :377-392), g = domain0's coset generator. */
int32_t b200_plonk_build_z(b200_domain_t domain0, const void* d_l, const void* d_r, const void* d_o,
                           const int64_t* d_perm, const void* beta_mont, const void* gamma_mont, void* d_z_out);
/* Polynomial.Evaluate (Horner) of n canonical coefficients at x; result (one fr.Element) on the host */
int32_t b200_poly_eval(int32_t dev, int32_t curve, const void* d_coeffs, size_t n, const void* x_mont, void* out_host);
/* kzg.Open's quotient: coeffs <- (p(X) - p(z)) / (X - z) in place (degree n-2, top coefficient zeroed);
 * the claimed value p(z) is returned on the host */
int32_t b200_poly_div_by_linear(int32_t dev, int32_t curve, void* d_coeffs, size_t n, const void* z_mont,
                                void* claimed_value_host);

/* ---- KZG over a G1 SRS table (kzg_host.cu; gnark-crypto's kzg.Commit / Open / BatchOpenSinglePoint) ----
 * A commitment needs no entry point of its own: kzg.Commit(p) is b200_msm on the SRS table, and a batch of commitments
 * is ONE b200_msm_batch on it (off = 0, n = the longest polynomial, the shorter ones zero-padded).
 * The three calls below are synchronous, synchronise once at the end and join pending pipelined MSMs first.  polys:
 * batch * n fr.Elements (Montgomery), item-major, on the host or the device (polys_on_dev); they are only read.  The
 * caller zero-pads shorter polynomials to n, which changes no commitment, value or quotient.  points / z / gamma: on the
 * host; a point may be 0.  Refusals, each checked before anything is allocated, naming the argument or the limit, with
 * every output untouched: a null pointer, a G2 table, n - 1 above the table's point count, batch * n overflowing, and the
 * quotient MSM's limits (batch * (n - 1) * windows < 2^31, batch * bucket sets * 2^(c-1) < 2^31 - 1; the message names the
 * largest batch that fits).  batch = 0 writes nothing; n = 0 gives value 0 and the point at infinity, n = 1 value c_0 and
 * the point at infinity. */
/* values[b] = p_b(points[b]), b < batch: batch fr.Elements to values_host */
int32_t b200_poly_eval_batch(int32_t dev, int32_t curve, const void* polys, size_t n, size_t batch, int32_t polys_on_dev,
                             const void* points_mont, void* values_host);
/* kzg.Open of every item: values[b] = p_b(z_b), proofs[b] = sum_{i<n-1} q_b[i] * srs[i] (G1Jac, gnark layout) with
 * q_b = (p_b - p_b(z_b)) / (X - z_b).  One batched division and one batched MSM over srs[0, n - 1): an SRS of exactly
 * n - 1 points is enough, as for kzg.Open.  The MSM window is a precomputed table's own, else that of an n-point MSM. */
int32_t b200_kzg_open_batch(b200_table_t srs, const void* polys, size_t n, size_t batch, int32_t polys_on_dev,
                            const void* points_mont, void* values_host, void* proofs_jac_host);
/* kzg.BatchOpenSinglePoint's H: f = sum_b gamma^b p_b (gamma^0 = 1), proof = Commit((f - f(z)) / (X - z)) over
 * srs[0, n - 1), one G1Jac.  The claimed values come from b200_poly_eval_batch on the same polynomials. */
int32_t b200_kzg_fold_open(b200_table_t srs, const void* polys, size_t n, size_t batch, int32_t polys_on_dev,
                           const void* z_mont, const void* gamma_mont, void* proof_jac_host);

/* ---- PLONK prover (host orchestration in C++, plonk_host.cu; the reference has no accelerated PLONK - this is
 *      the device-resident twin of backend/plonk/bn254/prove.go:98-837 behind one call, for a Go package
 *      backend/accelerated/b200/plonk mirroring backend/plonk/plonk.go:94-135).
 *      Key = the Trace (setup.go:67-86: Ql, Qr, Qm, Qo, Qk in Lagrange/regular form, the permutation S) and the
 *      canonical KZG SRS (pk.Kzg.G1, n + 3 points); sigma polynomials are rebuilt from S (setup.go:289-392).
 *      Challenges and blinding coefficients are INPUTS: the Go shim derives gamma, beta, alpha, zeta, v from its
 *      Fiat-Shamir transcript exactly as prove.go:492-555 and samples the blinding polynomials (:1211-1220);
 *      passing them in also makes every intermediate result reproducible.  BSB22 commitment gates are supported
 *      (n_qcp / qcp in the key, the committed polynomials in b200_plonk_challenges.pi2 / b200_plonk_begin), and so is
 *      StatisticalZK (b200_plonk_challenges.hr / b200_plonk_set_quotient_randomizers).  Domains below 2^3 are refused (the CPU prover switches to an 8n quotient domain there,
 *      prove.go:248).  All scalars are fr.Elements (Montgomery) on the host. */
typedef struct b200_plonk_pk_s* b200_plonk_pk_t;
typedef struct {
  uint32_t log2n;                        /* domain0 = 2^log2n rows */
  const void *ql, *qr, *qm, *qo, *qk;    /* n fr.Elements each, Lagrange/regular */
  const int64_t* perm;                   /* trace.S, 3n entries */
  const void* srs_canonical;             /* n + 3 G1Affine */
  uint32_t n_qcp;                        /* BSB22 commitment gates (len(trace.Qcp)), 0 = none */
  const void* const* qcp;                /* n_qcp selectors Qcp_j, n fr.Elements each, Lagrange/regular */
} b200_plonk_pk_desc;
typedef struct {
  const void *gamma, *beta, *alpha, *zeta, *v; /* one fr.Element each */
  const void *bl, *br, *bo;                    /* blinding of L, R, O: 2 coefficients each */
  const void* bz;                              /* blinding of Z: 3 coefficients */
  /* BSB22 (keys with n_qcp > 0, else NULL): the committed polynomials PI2_j produced by the solver hint
   * (prove.go:280-318), n fr.Elements each, Lagrange/regular; out_bsb22 receives [PI2_j] (n_qcp G1Jac) */
  const void* const* pi2;
  void* out_bsb22;
  /* this proof's complete Qk (completeQk, prove.go:349-373: public inputs and BSB22 commitment values folded into the
   * trace's Qk), n fr.Elements, Lagrange/regular; NULL = the Qk the key was loaded with */
  const void* qk;
  /* StatisticalZK (backend.WithStatisticalZeroKnowledge, backend/backend.go:141-147): the two
   * quotientShardsRandomizers of newInstance (prove.go:239-242), 2 fr.Elements; NULL = off.  [H1], [H2], [H3] become the
   * commitments of h1 + b1 X^(n+2), h2 - b1 + b2 X^(n+2), h3 - b2 (prove.go:689-722) and the linearised polynomial
   * follows (prove.go:1466-1481); the verifier is unchanged. */
  const void* hr;
} b200_plonk_challenges;
int32_t b200_plonk_pk_load(int32_t dev, int32_t curve, const b200_plonk_pk_desc* desc, b200_plonk_pk_t* out);
int32_t b200_plonk_pk_free(b200_plonk_pk_t pk);
/* l, r, o: the solved wire columns (SparseR1CSSolution{L,R,O}, constraint/bn254/system.go:208-210), n fr.Elements
 * each on the host.  out_points: 10 G1Jac in gnark layout - [L], [R], [O], [Z], [H1], [H2], [H3], linearised digest,
 * batched opening quotient, Z-shifted opening quotient (Proof fields, prove.go:77-96).  out_values: 7 + n_qcp
 * fr.Elements - the claimed values at zeta of {linearised polynomial, l, r, o, s1, s2}, then Z(w*zeta), then
 * Qcp_j(zeta) (BatchedProof.ClaimedValues = values 0-5 followed by values 7..). */
int32_t b200_plonk_prove(b200_plonk_pk_t pk, const void* l, const void* r, const void* o,
                         const b200_plonk_challenges* ch, void* out_points, void* out_values);
/* wall-clock milliseconds of the five stages of the last successful b200_plonk_prove on this key (begin = L,R,O
 * canonical forms + 3 commitments; commit_z; quotient; linearise; batch_open) - the step profile of the PLONK prover,
 * like b200_msm_profile for the MSM (the reference times its stages with the same granularity in debug logs,
 * backend/plonk/bn254/prove.go:155-233 "instance.*" goroutine stages) */
int32_t b200_plonk_last_stage_ms(b200_plonk_pk_t pk, double* out_ms5);
/* The same proof, one entry point per Fiat-Shamir round, so that a caller can derive each challenge from the digests
 * of the previous round exactly as prove.go:492-555 (gamma, beta <- [L],[R],[O]; alpha <- [Z]; zeta <- [H1..3];
 * v <- linearised digest + opened values).  Stages must be called in this order; b200_plonk_end releases the
 * session at any point.
 *   begin       commitToLRO :404-489            out_lro: [L], [R], [O]                         (3 G1Jac)
 *   commit_z    buildRatioCopyConstraint :635   out_z: [Z]
 *   quotient    computeQuotient :558-633        out_h: [H1], [H2], [H3]
 *   linearise   openZ :670-687 + computeLinearizedPolynomial :724-794
 *               out_points: linearised digest, Z-shifted opening quotient (2 G1Jac);
 *               out_values: p(zeta) of {linearised, l, r, o, s1, s2}, then Z(w*zeta), then Qcp_j(zeta)
 *                                                                                       (7 + n_qcp fr.Elements)
 *   batch_open  batchOpening :796-837           out_point: BatchedProof.H */
typedef struct b200_plonk_session_s* b200_plonk_session_t;
int32_t b200_plonk_begin(b200_plonk_pk_t pk, const void* l, const void* r, const void* o, const void* bl /*2*/,
                         const void* br /*2*/, const void* bo /*2*/, const void* const* pi2 /* n_qcp or NULL */,
                         void* out_bsb22 /* n_qcp G1Jac or NULL */, b200_plonk_session_t* out, void* out_lro);
/* optional, between begin and quotient: this proof's complete Qk (see b200_plonk_challenges.qk) */
int32_t b200_plonk_set_qk(b200_plonk_session_t s, const void* qk_lagrange);
/* optional, between begin and quotient: StatisticalZK, the two quotientShardsRandomizers (see b200_plonk_challenges.hr) */
int32_t b200_plonk_set_quotient_randomizers(b200_plonk_session_t s, const void* hr /*2*/);
int32_t b200_plonk_commit_z(b200_plonk_session_t s, const void* beta, const void* gamma, const void* bz /*3*/,
                            void* out_z);
int32_t b200_plonk_quotient(b200_plonk_session_t s, const void* alpha, void* out_h);
int32_t b200_plonk_linearise(b200_plonk_session_t s, const void* zeta, void* out_points, void* out_values);
int32_t b200_plonk_batch_open(b200_plonk_session_t s, const void* v, void* out_point);
int32_t b200_plonk_end(b200_plonk_session_t s);

/* ---- Groth16 prover (host layer mirroring backend/accelerated/icicle/groth16/
 *      bn254/icicle.go:784-1360 Prove + setupDevicePointers :88-264) ------------
 * Builds the device-resident key from the gnark ProvingKey fields
 * (backend/groth16/bn254/setup.go:25-48).  infinity_a/b: one byte per wire. */
typedef struct {
  int32_t curve;
  uint64_t domain_size;       /* pk.Domain.Cardinality */
  const void* domain_gen;     /* pk.Domain.Generator (fr, Montgomery) or NULL */
  const void* coset_gen;      /* pk.Domain.FrMultiplicativeGen or NULL */
  const void* g1_alpha;       /* G1Affine */
  const void* g1_beta;
  const void* g1_delta;
  const void* g2_beta;        /* G2Affine */
  const void* g2_delta;
  const void* g1_a; size_t n_a;   /* []G1Affine, infinities already removed */
  const void* g1_b; size_t n_b;
  const void* g1_z; size_t n_z;   /* n-1 entries, bit-reversed order */
  const void* g1_k; size_t n_k;   /* private wires */
  const void* g2_b; size_t n_b2;
  const uint8_t* infinity_a;  /* nb_wires flags */
  const uint8_t* infinity_b;
  size_t nb_wires;
  size_t nb_public;           /* r1cs.GetNbPublicVariables() (K covers wires[nb_public:]) */
  int32_t flags;              /* B200_TABLE_PRECOMP */
  /* multi-GPU: this process keeps only shard `shard_rank` of `shard_world` contiguous point-range
   * shards of every table (SURVEY.md §8e); 0/0 or world <= 1 = the whole key. */
  int32_t shard_rank;
  int32_t shard_world;
  /* BSB22 commitments: the wires that have no base in G1.K are excluded from the Krs MSM (filterHeap,
   * backend/groth16/bn254/prove.go:231-239,321-344): sorted absolute wire indices of
   * internal.ConcatAll(commitmentInfo.GetPrivateCommitted()..., commitmentInfo.CommitmentIndexes()), i.e. the private
   * committed wires AND the commitment wires themselves; n_k then equals nb_wires - nb_public - n_k_removed.
   * NULL / 0 = no commitments.  The commitment MSMs themselves (CommitmentKeys[i].Commit / ProveKnowledge,
   * prove.go:84,114) are b200_pedersen_commit. */
  const uint32_t* k_removed;
  size_t n_k_removed;
  /* Key tables from gnark's dump file instead of host memory (SURVEY.md §8f-1): when dump_path is not NULL the five
   * pointers g1_a, g1_b, g1_z, g1_k, g2_b are ignored and every table (or this process's shard of it) is read with
   * b200_table_upload_file from the payload offsets below (the byte position of element 0 of each slice, i.e. just
   * after the slice's length prefix); n_a .. n_b2 still give the slice lengths. */
  const char* dump_path;
  uint64_t dump_off_a, dump_off_b, dump_off_z, dump_off_k, dump_off_b2;
} b200_groth16_pk_desc;

int32_t b200_groth16_pk_load(int32_t dev, const b200_groth16_pk_desc* desc, b200_pk_t* out);
int32_t b200_groth16_pk_free(b200_pk_t pk);

/* One proof from a solved witness (R1CSSolution{W,A,B,C}, constraint/bn254/system.go:162-165).
 * r, s: the prover's randomness as fr.Elements (Montgomery); the Go shim samples
 * them exactly as prove.go:170-182 does.  Outputs are gnark affine points:
 * ar, krs: G1Affine; bs: G2Affine.  msm_out (optional, may be NULL): the five raw
 * MSM results as Jacobian points in the order A, B1, Z(h), K, B2 - the
 * deterministic sub-results parity tests pin.  Sharded keys (shard_world > 1): the call works when the device has a
 * communicator of the same world size (b200_comm_init / b200_comm_init_all) - the five partial sums are gathered and
 * added on the device, every rank returns the same proof; without one it is refused (use the two halves below). */
int32_t b200_groth16_prove(b200_pk_t pk, const void* wires, const void* a, const void* b, const void* c,
                           size_t n_constraints, const void* r, const void* s, void* ar_out, void* bs_out,
                           void* krs_out, void* msm_out);
/* The two halves of b200_groth16_prove, for sharded keys (one process per GPU, or one thread per GPU inside one
 * process - entry points lock per device, INTEGRATION.md §3b):
 *  - b200_groth16_msms: device part.  computeH + this shard's slice of the five MSMs; msm_out
 *    receives 4 G1Jac + 1 G2Jac partial sums (order A, B1, Z(h), K, B2).  With a communicator of the key's
 *    world size on the device the sums are already COMPLETE (b200_points_allreduce inside the call); without one
 *    the caller adds the shards' partial sums (b200_point_add_jac, or its own group arithmetic).
 *  - b200_groth16_assemble: host part (prove.go:185,199-214,241-269,287-292) from the five
 *    complete MSM results. */
int32_t b200_groth16_msms(b200_pk_t pk, const void* wires, const void* a, const void* b, const void* c,
                          size_t n_constraints, void* msm_out);
int32_t b200_groth16_assemble(b200_pk_t pk, const void* msm5, const void* r, const void* s, void* ar_out,
                              void* bs_out, void* krs_out);
/* `batch` proofs of one circuit in one call: the device work of all items runs as one launch sequence (batched
 * wire filters, one batched MSM per key table, computeH as batched NTTs), then the proofs are assembled on host threads.
 * wires / a / b / c: one host pointer per item (nb_wires and n_constraints fr.Elements, as b200_groth16_prove takes);
 * r, s: batch fr.Elements each, item-major.  Outputs: batch affine points each in ar_out, bs_out, krs_out; msm_out
 * (optional) batch x (4 G1Jac + 1 G2Jac), each item laid out as b200_groth16_prove's.  Every proof equals what
 * b200_groth16_prove gives for the same item and r, s.  Refused, with every output untouched: sharded keys, a null
 * argument, n_constraints above the domain, and a batch larger than the device indices allow (the message names the
 * largest batch the key takes).  batch = 0 writes nothing. */
int32_t b200_groth16_prove_batch(b200_pk_t pk, size_t batch, const void* const* wires, const void* const* a,
                                 const void* const* b, const void* const* c, size_t n_constraints,
                                 const void* r, const void* s, void* ar_out, void* bs_out, void* krs_out, void* msm_out);

#ifdef __cplusplus
}
#endif
#endif /* GNARK_B200_H */

// Type-erased per-(curve, group) operation tables.  Each inst_<curve>.cu translation
// unit instantiates the templates for its field types and registers the function
// pointers here; capi.cu / groth16_host.cu dispatch through them.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

#include "host_fr.h"

namespace gb200 {

// Stream-ordered device buffer that cannot leak on an early return: freed on its allocation stream by the destructor
// unless it was handed back with release_on() (success paths free on the stream of the LAST user).
struct AsyncBuf {
  void* p = nullptr;
  cudaStream_t st = nullptr;
  AsyncBuf() = default;
  AsyncBuf(const AsyncBuf&) = delete;
  AsyncBuf& operator=(const AsyncBuf&) = delete;
  ~AsyncBuf() { if (p) cudaFreeAsync(p, st); }
  cudaError_t alloc(size_t bytes, cudaStream_t s) { st = s; return cudaMallocAsync(&p, bytes ? bytes : 1, s); }
  cudaError_t release_on(cudaStream_t s) {
    if (!p) return cudaSuccess;
    void* q = p; p = nullptr;
    return cudaFreeAsync(q, s);
  }
};

// Streams of a pipelined MSM (null members: that stage stays on the call's stream).  The front (decompose, sort,
// offsets: DRAM-bound) stays on the caller's stream; the accumulate kernel (integer-multiplier-bound) runs on `acc`;
// the latency-bound reduction tail on `tail` - so MSM i+1's front overlaps MSM i's accumulate, and MSM i's tail overlaps both.
struct MsmPipe {
  cudaStream_t acc = nullptr;
  cudaStream_t tail = nullptr;
  cudaEvent_t front_ev = nullptr;  // recorded on the call's stream after the front
  cudaEvent_t acc_ev = nullptr;    // recorded on `acc` (or the call's stream) after the accumulate kernel
};

struct MsmOps {
  int scalar_bits;      // Fr bit length
  size_t fr_bytes;      // sizeof(fr.Element)
  size_t affine_bytes;  // sizeof(G?Affine)
  size_t jac_bytes;     // sizeof(G?Jac)
  // workspace bytes for `batch` MSMs of n scalars each (1: a single MSM) with the given parameters
  cudaError_t (*ws_bytes)(uint32_t n, uint32_t batch, uint32_t stride, int c, int precomp, uint32_t task_len, uint32_t chunk,
                          size_t* out);
  // enqueue a full MSM (all pointers on device); d_idx null: bases off + i, else bases d_idx[i] (indices checked
  // against the table's point count by the caller).  batch > 1: d_scalars holds batch * n scalars (item-major), d_out_jac
  // batch points, and d_idx must be null
  // item b's scalars start at d_scalars + b * scalar_stride (0: n, the items back to back)
  cudaError_t (*run)(cudaStream_t st, uint32_t n, uint32_t batch, uint32_t stride, uint32_t off, int c, int precomp,
                     uint32_t task_len, uint32_t chunk, const void* d_table, const void* d_scalars, void* d_out_jac,
                     void* ws, cudaEvent_t* stage_events /* nullable, 8 entries */,
                     const MsmPipe* pipe /* nullable: everything on st */, const uint32_t* d_idx, uint32_t scalar_stride);
  // fill slabs 1..nwin-1 of a [nwin][n] table whose slab 0 holds the bases
  cudaError_t (*precompute)(cudaStream_t st, uint32_t n, int nwin, int c, void* d_table);
  // resident 128-thread blocks of the accumulate kernel per SM (occupancy API): the task length is chosen so that the
  // accumulate grid is close to a whole number of waves
  int (*acc_blocks_per_sm)();
  // fixed-base batch (fixed_base.cuh): d_out[i] = scalars[i] * base; h_base is ONE affine point on the host
  cudaError_t (*fixed_base)(cudaStream_t st, const void* h_base, const void* d_scalars, size_t n, int c, void* d_out_affine);
  // multi-GPU combine: d_out[k] = sum_r d_gathered[r * count + k] (Jacobian points, k_points_fold)
  cudaError_t (*fold)(cudaStream_t st, const void* d_gathered, uint32_t world, uint32_t count, void* d_out_jac);
  // serialised point slices (gnark-crypto encodings, points_decode.cuh): bytes per point of an encoding (0 = not
  // supported for this group), and the decode kernel.  curve / group: which curve coefficient (or twist coefficient) applies;
  // d_status: two uint32 (DECODE_* code, index), zeroed by the caller
  size_t (*encoded_bytes)(int encoding);
  cudaError_t (*decode)(cudaStream_t st, const void* d_bytes, size_t n, int encoding, int curve, int group, void* d_out_affine,
                        uint32_t* d_status);
  // group-element NTT (points_ntt.cuh) in place on the 2^logn device points of d_points, on the NttDomainDev of the same
  // curve's Fr behind `dom`; G1 only (null for G2)
  cudaError_t (*points_ntt)(cudaStream_t st, void* dom, void* d_points, int inverse);
  // variable-base scaling (points_scale.cuh) in place on n <= PS_MAX_POINTS device points: d_points[i] <- (c * t^i) *
  // d_points[i]; c, t: one Fr element each on the host (Montgomery), t null means t = 1
  cudaError_t (*points_scale)(cudaStream_t st, void* d_points, size_t n, const void* c_mont, const void* t_mont);
};

struct NttOps {
  size_t fr_bytes;
  int two_adicity;
  void* (*domain_new)(cudaStream_t st, int logn, const void* gen_mont, const void* coset_mont, cudaError_t* err);
  void (*domain_free)(void* dom);
  size_t (*domain_bytes)(void* dom);
  cudaError_t (*ntt)(cudaStream_t st, void* dom, void* d_data, int inverse, int decimation, int on_coset);
  cudaError_t (*compute_h)(cudaStream_t st, void* dom, void* d_a, void* d_b, void* d_c);
  cudaError_t (*vec_op)(cudaStream_t st, int op, void* d_out, const void* d_a, const void* d_b, size_t n);
  cudaError_t (*bit_reverse)(cudaStream_t st, void* d_data, uint32_t logn);
  cudaError_t (*scale_powers)(cudaStream_t st, void* d_data, size_t n, const void* s_mont, const void* g_mont);
  cudaError_t (*batch_invert)(cudaStream_t st, void* d_data, size_t n);
  // PLONK (see plonk.cuh); `args` is a const b200_plonk_coset_args*
  cudaError_t (*plonk_coset)(cudaStream_t st, void* dom0, const void* big_coset_gen, const void* big_gen,
                             const void* args);
  cudaError_t (*plonk_divide_by_zh)(cudaStream_t st, void* dom1, uint32_t log_n0, void* d_data);
  cudaError_t (*axpy)(cudaStream_t st, void* d_y, const void* a_mont, const void* d_x, size_t n);   // y += a*x
  // O(n) scans (plonk.cuh)
  cudaError_t (*scan)(cudaStream_t st, int op /*0 product, 1 sum*/, void* d_data, size_t n, int exclusive);
  cudaError_t (*plonk_build_z)(cudaStream_t st, void* dom0, const void* d_l, const void* d_r, const void* d_o,
                               const int64_t* d_perm, const void* beta, const void* gamma, void* d_z);
  cudaError_t (*poly_eval)(cudaStream_t st, const void* d_coeffs, size_t n, const void* x_mont, void* out_host);
  cudaError_t (*poly_div_linear)(cudaStream_t st, void* d_coeffs, size_t n, const void* z_mont, void* rem_host);
  // out[j] = src[idx[j]] (wire filtering, backend/groth16/bn254/prove.go:147-168)
  cudaError_t (*gather)(cudaStream_t st, void* d_out, const void* d_src, const uint32_t* d_idx, size_t n);
  // host-side Fr constants and arithmetic (host_fr.h) for the scalar work between device stages
  const HostFrCtx* (*host_fr)();
  // BSB22 commitment gate: out[scatter(j)] += qcp[j] * pi2[j] on one coset (plonk.cuh)
  cudaError_t (*plonk_bsb22)(cudaStream_t st, void* dom0, const void* d_qcp, const void* d_pi2, uint32_t coset_index,
                             uint32_t rho, void* d_out);
  // `batch` transforms of the domain's size on batch * n item-major elements (ntt_enqueue with a batch)
  cudaError_t (*ntt_batch)(cudaStream_t st, void* dom, void* d_data, size_t batch, int inverse, int decimation, int on_coset);
  // computeH of `batch` proofs: d_abc is [3][batch][n] (A, B, C); h of item b ends at d_abc + b * n (compute_h_batch_enqueue)
  cudaError_t (*compute_h_batch)(cudaStream_t st, void* dom, void* d_abc, size_t batch);
  // gather over a batch: out[b * out_stride + j] = src[b * src_stride + idx[j]], j < n, b < batch
  cudaError_t (*gather_batch)(cudaStream_t st, void* d_out, const void* d_src, const uint32_t* d_idx, size_t n, size_t batch,
                              size_t src_stride, size_t out_stride);
  // batches of `batch` polynomials of n coefficients, item-major on the device, points on the host; enqueued on st with
  // no host synchronisation (plonk.cuh): d_values[b] = p_b(points[b]) ...
  cudaError_t (*poly_eval_batch)(cudaStream_t st, const void* d_polys, size_t n, size_t batch, const void* points_host,
                                 void* d_values);
  // ... row b of d_q (batch * n) = (p_b - p_b(z_b)) / (X - z_b) with its top coefficient 0, d_values[b] = p_b(z_b) ...
  cudaError_t (*poly_div_linear_batch)(cudaStream_t st, const void* d_polys, size_t n, size_t batch, const void* points_host,
                                       void* d_q, void* d_values);
  // ... d_out[j] = sum_b gamma^b p_b[j] (n coefficients; gamma on the host)
  cudaError_t (*poly_fold)(cudaStream_t st, const void* d_polys, size_t n, size_t batch, const void* gamma_mont, void* d_out);
};

// Host-side group arithmetic for proof assembly (backend/groth16/bn254/prove.go:
// 185,199-200,212-214,241-269,287-292): a handful of scalar multiplications and
// additions that the reference also keeps on the CPU (in Go).
struct HostGroupOps {
  size_t affine_bytes, jac_bytes, fr_bytes;
  // out_jac = k * p_affine   (k: fr.Element Montgomery)
  void (*scalar_mul_affine)(const void* p_affine, const void* k_mont, void* out_jac);
  void (*scalar_mul_jac)(const void* p_jac, const void* k_mont, void* out_jac);
  void (*add_jac)(void* acc_jac, const void* q_jac);            // acc += q
  void (*add_mixed)(void* acc_jac, const void* q_affine);       // acc += q
  void (*to_affine)(const void* p_jac, void* out_affine);
  // fr helpers: out = -(a*b)
  void (*fr_neg_mul)(const void* a_mont, const void* b_mont, void* out_mont);
};

const MsmOps* get_msm_ops(int curve, int group);
const NttOps* get_ntt_ops(int curve);
const HostGroupOps* get_host_group_ops(int curve, int group);

// registration (called from static initialisers in inst_*.cu)
void register_msm_ops(int curve, int group, const MsmOps* ops);
void register_ntt_ops(int curve, const NttOps* ops);
void register_host_group_ops(int curve, int group, const HostGroupOps* ops);

}  // namespace gb200

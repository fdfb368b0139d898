// shared between capi.cu and groth16_host.cu
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>
#include <cstring>
#include <exception>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/gnark_b200.h"
#include "internal.h"
#include "msm.cuh"

#define GB200_MAX_DEVICES 16

namespace gb200 {

struct DeviceCtx {
  // Host-side state of a device (current stream, fork/join events, pending tail) is shared by every entry point:
  // each extern "C" function holds this lock from its device_ctx() lookup to its return, so concurrent callers
  // (goroutines) on ONE device are serialised here instead of by a process-global mutex (the reference:
  // deviceProveMu, icicle.go:53-60); different devices do not contend.  Recursive: entry points call one another.
  std::recursive_mutex mu;
  bool ready = false;
  int dev = 0;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;  // own_stream or the caller's (b200_set_stream)
  // pipelined MSMs (MsmPipe, internal.h): the accumulate kernel of MSM i runs on acc_stream and its reduction tail on
  // tail_stream while MSM i+1 decomposes and sorts on `stream`
  cudaStream_t acc_stream = nullptr;
  cudaStream_t tail_stream = nullptr;
  cudaStream_t copy_stream = nullptr;  // H2D of later-needed inputs overlaps compute on `stream`
  cudaEvent_t copy_ev = nullptr;
  cudaEvent_t front_ev = nullptr;  // front done (recorded on stream)
  cudaEvent_t acc_ev[2] = {nullptr, nullptr};   // accumulate of pipelined MSM k done (recorded on acc_stream), slot k & 1
  uint64_t pipe_seq = 0;           // pipelined MSMs enqueued since the last join
  cudaEvent_t tail_ev = nullptr;   // tail done (recorded on tail_stream)
  bool tail_pending = false;
  // multi-GPU (comm.cu): NCCL communicator of this device (ncclComm_t), nullptr = single device
  void* comm = nullptr;
  int comm_world = 1, comm_rank = 0;
};
void comm_teardown(DeviceCtx& c);   // comm.cu
int32_t points_allreduce_on_stream(DeviceCtx* ctx, const MsmOps* ops, const void* d_partials, size_t count, void* d_totals);

int32_t set_error(const std::string& msg);
int32_t cuda_fail(const char* what, cudaError_t e);
int32_t device_ctx(int dev, DeviceCtx** out);
int msm_window_for(size_t n);
// task length and reduction chunk of `batch` MSMs of n scalars each (1: a single MSM), sized by their total entries and buckets
void msm_tuning(size_t n, size_t batch, int nwin, int c, int precomp, int acc_blocks_per_sm, uint32_t* task_len, uint32_t* chunk);

}  // namespace gb200

struct b200_table_s {
  int dev, curve, group;
  size_t n;          // bases
  int c, nwin, precomp;
  size_t bytes;
  void* d_points = nullptr;
  const gb200::MsmOps* ops;
  // owns its device buffer: a table that fails half way through its construction does not leak it
  ~b200_table_s() { if (d_points) cudaFree(d_points); }
};

struct b200_domain_s {
  int dev, curve, logn;
  const gb200::NttOps* ops;
  void* impl;
};

namespace gb200 {
// stream-ordered scratch memory for the host orchestrations (plonk_host.cu): cudaMallocAsync / cudaFreeAsync on the
// device's stream, served from the never-shrinking pool - a proof allocates and releases GiBs of temporaries, and
// cudaMalloc / cudaFree (b200_alloc / b200_free: synchronous, unmap on free) were a visible part of its wall time
int32_t scratch_alloc(int dev, size_t bytes, void** out);
int32_t scratch_free(int dev, void* p);
// d_idx (optional, device): n table indices already checked against t->n; scalar i then multiplies base d_idx[i]
// (off must be 0).  On a plain table an indexed MSM takes its window from n, not from the table's size.
// batch > 1: `batch` MSMs over the same bases in one pipeline (msm_make_batch_plan), item b's n scalars at
// d_scalars + b * stride (0: n), one Jacobian result per item at d_out; the window is the table's, as for a single MSM.
// The caller checks msm_batch_fits() first.
int32_t msm_on_stream(DeviceCtx* ctx, b200_table_s* t, size_t off, size_t n, const void* d_scalars, void* d_out,
                      cudaEvent_t* stage_events = nullptr, bool pipelined = false, const uint32_t* d_idx = nullptr,
                      size_t batch = 1, size_t stride = 0);
// largest batch of n-scalar MSMs with window c on t that the pipeline can index: batch * n * windows entries below 2^31
// and batch * bucket sets * 2^(c-1) bucket keys below 2^31 - 1 (what b200_msm_batch checks)
size_t msm_max_batch(const b200_table_s* t, size_t n, int c);
// window of an MSM of n scalars on a table of `scalar_bits`-bit scalars: msm_window_for(n), raised until the scalar has
// at most 64 windows (MSM_MAX_WINDOWS of the table precompute)
int msm_window_with_limit(size_t n, int scalar_bits);
int32_t msm_join(DeviceCtx* ctx);  // make ctx->stream wait for the pipelined tails

// Buffers of one synchronous entry point, all on ctx->stream.  Host pointers are borrowed for the call only: host
// inputs are uploaded into pool buffers now, host outputs are downloaded by finish(), which also frees every buffer
// (before the sync, so that the pool can reuse them) and synchronises - nothing is read after the call returns.
// Device-resident and zero-byte buffers are used in place.  An early return frees the buffers without a sync.
class Staging {
 public:
  explicit Staging(DeviceCtx* ctx) : ctx_(ctx) {}
  ~Staging();
  Staging(const Staging&) = delete;
  Staging& operator=(const Staging&) = delete;

  // *d = the device copy of src (read by the operation), of dst (written by it) or of p (both)
  cudaError_t in(const void* src, size_t bytes, bool on_dev, const void** d) {
    return stage(const_cast<void*>(src), bytes, on_dev, true, false, const_cast<void**>(d));
  }
  cudaError_t out(void* dst, size_t bytes, bool on_dev, void** d) { return stage(dst, bytes, on_dev, false, true, d); }
  cudaError_t inout(void* p, size_t bytes, bool on_dev, void** d) { return stage(p, bytes, on_dev, true, true, d); }
  cudaError_t scratch(size_t bytes, void** d);
  // copy src (device or host) into the device buffer d_dst now
  cudaError_t upload(void* d_dst, const void* src, size_t bytes, bool src_on_dev);
  // copy the device buffer d_src to dst (device or host) in finish(), once the operation has succeeded
  void download(void* dst, const void* d_src, size_t bytes, bool dst_on_dev);
  // downloads (when rc == 0 and e == cudaSuccess), frees, synchronises; returns the first error of: rc, e, a
  // download, the sync.  `what` labels the CUDA failures.
  int32_t finish(const char* what, int32_t rc, cudaError_t e = cudaSuccess);
  int32_t finish(const char* what, cudaError_t e) { return finish(what, 0, e); }

 private:
  struct Copy { void* dst; const void* src; size_t bytes; cudaMemcpyKind kind; };
  cudaError_t stage(void* p, size_t bytes, bool on_dev, bool up, bool down, void** d);
  DeviceCtx* ctx_;
  std::vector<void*> bufs_;
  std::vector<Copy> downloads_;
};
}

#define CK(x)                                                        \
  do {                                                               \
    cudaError_t e_ = (x);                                            \
    if (e_ != cudaSuccess) return gb200::cuda_fail(#x, e_);          \
  } while (0)

// device_ctx() + the per-device lock for the rest of the enclosing scope
#define GB_DEVICE(ctxvar, dev)                                        \
  gb200::DeviceCtx* ctxvar;                                           \
  {                                                                   \
    int32_t rc_dev_ = gb200::device_ctx((dev), &ctxvar);              \
    if (rc_dev_) return rc_dev_;                                      \
  }                                                                   \
  std::lock_guard<std::recursive_mutex> lock_##ctxvar(ctxvar->mu)

#define GUARD_BEGIN try {
#define GUARD_END                                                               \
  }                                                                             \
  catch (const std::exception& ex) { return gb200::set_error(std::string("exception: ") + ex.what()); } \
  catch (...) { return gb200::set_error("unknown exception"); }

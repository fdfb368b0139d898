// C ABI of libgnark_b200.so (declared in include/gnark_b200.h): runtime, memory,
// MSM base tables, MSM, NTT, vector ops.  The Groth16 host layer lives in
// groth16_host.cu.  Requires a CUDA device: there is no CPU fallback.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include "capi_common.h"
#include "file_stage.h"
#include "fixed_base.cuh"
#include "points_scale.cuh"

namespace gb200 {

// ---- registries ------------------------------------------------------------
static const MsmOps* g_msm_ops[4][3];
static const NttOps* g_ntt_ops[4];
static const HostGroupOps* g_host_ops[4][3];
void register_msm_ops(int curve, int group, const MsmOps* ops) { g_msm_ops[curve][group] = ops; }
void register_ntt_ops(int curve, const NttOps* ops) { g_ntt_ops[curve] = ops; }
void register_host_group_ops(int curve, int group, const HostGroupOps* ops) { g_host_ops[curve][group] = ops; }
const MsmOps* get_msm_ops(int curve, int group) {
  if (curve < 0 || curve > 3 || group < 1 || group > 2) return nullptr;
  return g_msm_ops[curve][group];
}
const NttOps* get_ntt_ops(int curve) { return (curve < 0 || curve > 3) ? nullptr : g_ntt_ops[curve]; }
const HostGroupOps* get_host_group_ops(int curve, int group) {
  if (curve < 0 || curve > 3 || group < 1 || group > 2) return nullptr;
  return g_host_ops[curve][group];
}

// ---- error + device context --------------------------------------------------
thread_local std::string g_last_error;
int32_t set_error(const std::string& msg) { g_last_error = msg; return 1; }
int32_t cuda_fail(const char* what, cudaError_t e) {
  g_last_error = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  return 2;
}

// MSM tuning (mirrors the reference's env knob ICICLE_MSM_MAX_WINDOW, icicle.go:586-598)
static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}
static std::mutex g_ctx_mu;
static DeviceCtx g_ctx[GB200_MAX_DEVICES];

int32_t device_ctx(int dev, DeviceCtx** out) {
  if (dev < 0 || dev >= GB200_MAX_DEVICES) return set_error("invalid device id " + std::to_string(dev));
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  DeviceCtx& c = g_ctx[dev];
  if (!c.ready) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess) return cuda_fail("cudaGetDeviceCount (a CUDA device is required; no CPU fallback)", e);
    if (dev >= count) return set_error("device " + std::to_string(dev) + " not present (" + std::to_string(count) + " visible)");
    CK(cudaSetDevice(dev));
    // priorities: reduction tail (latency-bound, few blocks) > the library's main stream (MSM fronts, NTTs) > accumulate
    // (fills the machine for milliseconds; the next MSM's sort slips into the SM slots its blocks free)
    int lo_prio = 0, hi_prio = 0;
    CK(cudaDeviceGetStreamPriorityRange(&lo_prio, &hi_prio));
    CK(cudaStreamCreateWithPriority(&c.own_stream, cudaStreamNonBlocking, (lo_prio + hi_prio) / 2));
    c.stream = c.own_stream;
    CK(cudaStreamCreateWithPriority(&c.tail_stream, cudaStreamNonBlocking, hi_prio));
    CK(cudaStreamCreateWithPriority(&c.acc_stream, cudaStreamNonBlocking, lo_prio));
    CK(cudaEventCreateWithFlags(&c.front_ev, cudaEventDisableTiming));
    for (int k = 0; k < 2; k++) CK(cudaEventCreateWithFlags(&c.acc_ev[k], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&c.tail_ev, cudaEventDisableTiming));
    CK(cudaStreamCreateWithFlags(&c.copy_stream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&c.copy_ev, cudaEventDisableTiming));
    cudaMemPool_t pool;
    CK(cudaDeviceGetDefaultMemPool(&pool, dev));
    uint64_t thr = UINT64_MAX;  // keep freed workspace cached in the pool
    CK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    // L2 fill granularity on a miss: 64 bytes.  The bucket accumulate gathers 64-byte (BN254 G1) / 96..192-byte points at
    // random from a table far larger than L2; with the driver's default (128) every 64-byte gather drags a second sector
    // in with it.  The kernels are multiplier-bound, so the time does not move - this removes wasted HBM traffic, nothing
    // else.  GB200_L2_FETCH=32|64|128 overrides, 0 leaves the device limit alone.
    if (const int g = env_int("GB200_L2_FETCH", 64)) CK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)g));
    c.dev = dev;
    c.ready = true;
  }
  cudaError_t e = cudaSetDevice(dev);
  if (e != cudaSuccess) return cuda_fail("cudaSetDevice", e);
  *out = &c;
  return 0;
}

int msm_window_for(size_t n) {
  int c = env_int("GB200_MSM_WINDOW", 0);
  if (c > 0) return c < 2 ? 2 : (c > 24 ? 24 : c);
  int lg = 0;
  while ((1ull << (lg + 1)) <= n) lg++;
  c = lg - 4;
  if (c < 4) c = 4;
  if (c > 16) c = 16;
  return c;
}
void msm_tuning(size_t n, size_t batch, int nwin, int c, int precomp, int acc_blocks_per_sm, uint32_t* task_len,
                uint32_t* chunk) {
  const size_t m = n * batch * (size_t)nwin;
  const size_t buckets = batch * (precomp ? (size_t)1 : (size_t)nwin) << (c - 1);
  // Task length.  One thread adds a task's entries; a bucket of k entries is cut into ceil(k / task_len) tasks.  Short
  // tasks fill the machine evenly (the accumulate grid is many waves deep, the short last task of every bucket idles its
  // lane for less) at the price of more partial sums for the combine kernel.  Within [24, 40] ([48, 64] for grids of a
  // dozen waves and more) the length is picked so that the grid is as close as possible to a whole number of waves of
  // resident blocks (the device's SMs - 132 on H100 SXM - x blocks per SM from the occupancy API): the last, partly
  // filled wave is the other loss (a grid of 3.04 waves spends a quarter of the kernel's time on 4 % of its work).
  int sms = 132;
  { int dev = 0; if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  const double resident = (double)sms * (acc_blocks_per_sm > 0 ? acc_blocks_per_sm : 1);
  // a grid a dozen waves deep loses little to its last wave: there the longer task wins again, because every partial
  // costs the combine kernel one full addition
  const double waves64 = ((double)m / 64.0 + 0.5 * (double)buckets) / 128.0 / resident;
  size_t lo = waves64 >= 12.0 ? 48 : 24, hi = waves64 >= 12.0 ? 64 : 40;
  const size_t per_bucket = m / (buckets ? buckets : 1);
  if (per_bucket < 2 * hi) { lo = 8; hi = per_bucket / 2 > 8 ? per_bucket / 2 : 8; }     // small problems: >= 2 tasks per bucket
  if (hi > 64) hi = 64;
  if (lo > hi) lo = hi;
  size_t best = hi;
  double best_waste = 2.0;
  for (size_t tl = hi; tl >= lo; tl--) {
    const double blocks = ((double)m / (double)tl + 0.5 * (double)buckets) / 128.0;    // expected tasks / threads per block
    const double waves = blocks / resident;
    const double full = waves <= 1.0 ? 1.0 : (double)(size_t)(waves + 0.999999);
    const double waste = (full - waves) / full;
    if (waste < best_waste - 0.005) { best_waste = waste; best = tl; }                 // ties: the longer task
    if (tl == lo) break;
  }
  // Overrides (tools/sweep_msm.py).  Both are clamped here, the one place that fixes the plan, so that the workspace size
  // and the run always agree.  A task length below 1 divides by zero on the host; above 2^30 the kernel's rounded-up
  // task count (entries + task_len - 1, 32-bit) wraps and a bucket gets no task at all.  A chunk below 1 divides by zero;
  // more than a set's 2^(c-1) buckets only leaves one chunk per set.  An override out of range keeps the default.
  const int tl_env = env_int("GB200_MSM_TASK_LEN", 0);
  *task_len = tl_env >= 1 ? (uint32_t)(tl_env < (1 << 30) ? tl_env : (1 << 30)) : (uint32_t)best;
  const int ch_env = env_int("GB200_MSM_CHUNK", 0);
  const uint32_t set_size = 1u << (c - 1);
  *chunk = ch_env >= 1 ? ((uint32_t)ch_env < set_size ? (uint32_t)ch_env : set_size) : (c >= 12 ? 8u : 4u);
}

int32_t scratch_alloc(int dev, size_t bytes, void** out) {
  GB_DEVICE(ctx, dev);
  CK(cudaMallocAsync(out, bytes ? bytes : 1, ctx->stream));
  return 0;
}
int32_t scratch_free(int dev, void* p) {
  if (!p) return 0;
  GB_DEVICE(ctx, dev);
  int32_t rc = msm_join(ctx);          // pipelined MSM tails may still read the buffer on the tail stream
  if (rc) return rc;
  CK(cudaFreeAsync(p, ctx->stream));
  return 0;
}

int32_t msm_join(DeviceCtx* ctx) {
  if (ctx->tail_pending) {
    CK(cudaStreamWaitEvent(ctx->stream, ctx->tail_ev, 0));
    ctx->tail_pending = false;
    ctx->pipe_seq = 0;
  }
  return 0;
}

int msm_window_with_limit(size_t n, int scalar_bits) {
  int c = msm_window_for(n ? n : 1);
  while (msm_num_windows(scalar_bits, c) > 64) c++;   // MSM_MAX_WINDOWS of the table precompute
  return c;
}

size_t msm_max_batch(const b200_table_s* t, size_t n, int c) {
  const size_t nwin = (size_t)msm_num_windows(t->ops->scalar_bits, c);
  const size_t by_entries = n ? (((size_t)1 << 31) - 1) / (n * nwin) : SIZE_MAX;
  const size_t by_keys = (((size_t)1 << 31) - 2) / ((t->precomp ? (size_t)1 : nwin) << (c - 1));
  return by_entries < by_keys ? by_entries : by_keys;
}

int32_t msm_on_stream(DeviceCtx* ctx, b200_table_s* t, size_t off, size_t n, const void* d_scalars, void* d_out,
                      cudaEvent_t* stage_events, bool pipelined, const uint32_t* d_idx, size_t batch, size_t stride) {
  if (d_idx ? off != 0 : off + n > t->n) return set_error("msm: range [off, off+n) exceeds the table");
  if (batch > 1 && (d_idx || batch > msm_max_batch(t, n, t->c))) return set_error("msm: batch exceeds the pipeline's indices");
  // a precomputed table's slabs fix its window; an indexed MSM on a plain table sizes its bucket sets by its own n
  // (a few hundred indices into a 2^22-point table must not pay for 2^15-bucket sets)
  const int c = (d_idx && !t->precomp) ? msm_window_with_limit(n, t->ops->scalar_bits) : t->c;
  const int nwin = msm_num_windows(t->ops->scalar_bits, c);
  // the pipeline indexes its n * nwin (scalar, window) entries with 31-bit counts (radix sort, offsets, tasks)
  if ((size_t)n * (size_t)nwin >= ((size_t)1 << 31))
    return set_error("msm: n * windows exceeds 2^31 entries - split the call into point ranges (or shard the table) and add the results");
  if (stage_events || n == 0) pipelined = false;
  if (!pipelined) { int32_t rc = msm_join(ctx); if (rc) return rc; }
  uint32_t task_len, chunk;
  msm_tuning(n, batch, nwin, c, t->precomp, t->ops->acc_blocks_per_sm(), &task_len, &chunk);
  size_t ws_bytes = 0;
  CK(t->ops->ws_bytes((uint32_t)n, (uint32_t)batch, (uint32_t)t->n, c, t->precomp, task_len, chunk, &ws_bytes));
  AsyncBuf ws_buf;
  CK(ws_buf.alloc(ws_bytes, ctx->stream));
  void* ws = ws_buf.p;
  MsmPipe pipe;
  if (pipelined) {
    // at most one front ahead of the accumulate stream (bounds the live workspaces): the front of MSM k waits for the
    // accumulate of MSM k - 2, whose event slot it then reuses
    const int slot = (int)(ctx->pipe_seq & 1);
    if (ctx->pipe_seq >= 2) CK(cudaStreamWaitEvent(ctx->stream, ctx->acc_ev[slot], 0));
    pipe.acc = env_int("GB200_MSM_ACC_STREAM", 1) ? ctx->acc_stream : nullptr;
    pipe.tail = ctx->tail_stream;
    pipe.front_ev = ctx->front_ev;
    pipe.acc_ev = ctx->acc_ev[slot];
    ctx->pipe_seq++;
  }
  cudaError_t e = t->ops->run(ctx->stream, (uint32_t)n, (uint32_t)batch, (uint32_t)t->n, (uint32_t)off, c, t->precomp,
                              task_len, chunk, t->d_points, d_scalars, d_out, ws, stage_events, pipelined ? &pipe : nullptr,
                              d_idx, (uint32_t)stride);
  // the workspace is last used by the tail kernels
  cudaError_t e2 = ws_buf.release_on(pipelined ? ctx->tail_stream : ctx->stream);
  if (pipelined && e == cudaSuccess) {
    cudaError_t e3 = cudaEventRecord(ctx->tail_ev, ctx->tail_stream);
    if (e3 != cudaSuccess) return cuda_fail("cudaEventRecord", e3);
    ctx->tail_pending = true;
  }
  if (e != cudaSuccess) return cuda_fail("msm enqueue", e);
  if (e2 != cudaSuccess) return cuda_fail("cudaFreeAsync", e2);
  return 0;
}

Staging::~Staging() { for (void* p : bufs_) cudaFreeAsync(p, ctx_->stream); }

cudaError_t Staging::scratch(size_t bytes, void** d) {
  cudaError_t e = cudaMallocAsync(d, bytes ? bytes : 1, ctx_->stream);
  if (e == cudaSuccess) bufs_.push_back(*d);
  return e;
}

cudaError_t Staging::upload(void* d_dst, const void* src, size_t bytes, bool src_on_dev) {
  return cudaMemcpyAsync(d_dst, src, bytes, src_on_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx_->stream);
}

void Staging::download(void* dst, const void* d_src, size_t bytes, bool dst_on_dev) {
  downloads_.push_back({dst, d_src, bytes, dst_on_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost});
}

cudaError_t Staging::stage(void* p, size_t bytes, bool on_dev, bool up, bool down, void** d) {
  *d = p;
  if (on_dev || bytes == 0) return cudaSuccess;
  cudaError_t e = scratch(bytes, d);
  if (e == cudaSuccess && up) e = upload(*d, p, bytes, false);
  if (e == cudaSuccess && down) download(p, *d, bytes, false);
  return e;
}

int32_t Staging::finish(const char* what, int32_t rc, cudaError_t e) {
  if (rc == 0 && e == cudaSuccess)
    for (const Copy& c : downloads_)
      if ((e = cudaMemcpyAsync(c.dst, c.src, c.bytes, c.kind, ctx_->stream)) != cudaSuccess) break;
  for (void* p : bufs_) cudaFreeAsync(p, ctx_->stream);
  bufs_.clear();
  const cudaError_t e_sync = cudaStreamSynchronize(ctx_->stream);
  if (rc) return rc;
  if (e != cudaSuccess) return cuda_fail(what, e);
  if (e_sync != cudaSuccess) return cuda_fail(what, e_sync);
  return 0;
}

// b200_msm_submit / b200_msm_submit_dev: the scalars go up on the copy stream (overlapping the MSM before), the MSM is
// pipelined; out_host == nullptr leaves the result in d_out, otherwise it is downloaded where the MSM produced it
static int32_t msm_submit(DeviceCtx* ctx, b200_table_s* t, size_t off, size_t n, const void* scalars_host, void* d_out,
                          void* out_host) {
  AsyncBuf d_sc, out_buf;
  if (out_host) {
    CK(out_buf.alloc(t->ops->jac_bytes, ctx->stream));
    d_out = out_buf.p;
  }
  if (n) {
    CK(d_sc.alloc(n * t->ops->fr_bytes, ctx->copy_stream));
    CK(cudaMemcpyAsync(d_sc.p, scalars_host, n * t->ops->fr_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    CK(cudaEventRecord(ctx->copy_ev, ctx->copy_stream));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->copy_ev, 0));
  }
  int32_t rc = msm_on_stream(ctx, t, off, n, d_sc.p, d_out, nullptr, /*pipelined=*/true);
  // the result is produced on the tail stream when the call was pipelined (n > 0), else on the main stream
  cudaStream_t res_stream = (n > 0) ? ctx->tail_stream : ctx->stream;
  if (rc == 0 && out_host) {
    cudaError_t e = cudaMemcpyAsync(out_host, d_out, t->ops->jac_bytes, cudaMemcpyDeviceToHost, res_stream);
    if (e != cudaSuccess) rc = cuda_fail("msm_submit result copy", e);
    if (rc == 0 && n > 0) {   // the join point must cover the download too
      e = cudaEventRecord(ctx->tail_ev, ctx->tail_stream);
      if (e != cudaSuccess) rc = cuda_fail("cudaEventRecord", e);
    }
  }
  d_sc.release_on(ctx->stream);       // last read by the decompose kernel on the main stream
  out_buf.release_on(res_stream);
  return rc;
}

}  // namespace gb200

using namespace gb200;

extern "C" {

const char* b200_version(void) { return "gnark_b200 0.1.0 (sm_90a)"; }
const char* b200_last_error(void) { return g_last_error.c_str(); }

int32_t b200_device_count(int32_t* out) {
  GUARD_BEGIN
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess) return cuda_fail("cudaGetDeviceCount", e);
  *out = count;
  return 0;
  GUARD_END
}

int32_t b200_init(int32_t n_dev, const int32_t* dev_ids) {
  GUARD_BEGIN
  if (n_dev <= 0 || !dev_ids) { DeviceCtx* c; return device_ctx(0, &c); }
  for (int i = 0; i < n_dev; i++) { GB_DEVICE(c, dev_ids[i]); }
  return 0;
  GUARD_END
}

int32_t b200_shutdown(void) {
  GUARD_BEGIN
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  for (int d = 0; d < GB200_MAX_DEVICES; d++) {
    DeviceCtx& c = g_ctx[d];
    if (!c.ready) continue;
    cudaSetDevice(d);
    cudaStreamSynchronize(c.stream);
    cudaStreamSynchronize(c.acc_stream);
    cudaStreamSynchronize(c.tail_stream);
    comm_teardown(c);
    cudaStreamDestroy(c.own_stream);
    cudaStreamDestroy(c.acc_stream);
    cudaStreamDestroy(c.tail_stream);
    cudaStreamDestroy(c.copy_stream);
    cudaEventDestroy(c.copy_ev);
    cudaEventDestroy(c.front_ev);
    cudaEventDestroy(c.acc_ev[0]);
    cudaEventDestroy(c.acc_ev[1]);
    cudaEventDestroy(c.tail_ev);
    // back to the initial state (the lock itself stays)
    c.ready = false; c.tail_pending = false; c.pipe_seq = 0;
    c.own_stream = c.stream = c.acc_stream = c.tail_stream = c.copy_stream = nullptr;
    c.copy_ev = c.front_ev = c.acc_ev[0] = c.acc_ev[1] = c.tail_ev = nullptr;
  }
  return 0;
  GUARD_END
}

int32_t b200_set_stream(int32_t dev, void* stream) {
  GUARD_BEGIN
  GB_DEVICE(c, dev);
  c->stream = stream ? reinterpret_cast<cudaStream_t>(stream) : c->own_stream;
  return 0;
  GUARD_END
}

int32_t b200_sync(int32_t dev) {
  GUARD_BEGIN
  GB_DEVICE(c, dev);
  int32_t rc = msm_join(c); if (rc) return rc;
  CK(cudaStreamSynchronize(c->stream));
  return 0;
  GUARD_END
}

int32_t b200_alloc(int32_t dev, size_t bytes, void** out) {
  GUARD_BEGIN
  GB_DEVICE(c, dev);
  CK(cudaMalloc(out, bytes ? bytes : 1));
  return 0;
  GUARD_END
}
int32_t b200_free(int32_t dev, void* p) {
  GUARD_BEGIN
  GB_DEVICE(c, dev);
  CK(cudaStreamSynchronize(c->stream));
  CK(cudaFree(p));
  return 0;
  GUARD_END
}
int32_t b200_h2d(int32_t dev, void* dst, const void* src, size_t bytes) {
  GUARD_BEGIN
  GB_DEVICE(c, dev);
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));  // host pointer is only borrowed for the call
  return 0;
  GUARD_END
}
int32_t b200_d2h(int32_t dev, void* dst, const void* src, size_t bytes) {
  GUARD_BEGIN
  GB_DEVICE(c, dev);
  int32_t rc = msm_join(c); if (rc) return rc;
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
  GUARD_END
}
int32_t b200_host_alloc(size_t bytes, void** out) {
  GUARD_BEGIN
  CK(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return 0;
  GUARD_END
}
int32_t b200_host_free(void* p) {
  GUARD_BEGIN
  CK(cudaFreeHost(p));
  return 0;
  GUARD_END
}

// ---- tables ------------------------------------------------------------------
}  // extern "C"

namespace gb200 {
// device table of n points with room for the precomputed slabs; slab 0 (= the first n entries of d_points) is filled by
// the caller - from host / device memory, from a file region, or by the point decoder - and table_finish builds the rest
static int32_t table_new(int dev, int curve, int group, size_t n, int flags, std::unique_ptr<b200_table_s>& t) {
  const MsmOps* ops = get_msm_ops(curve, group);
  if (!ops) return set_error("table_upload: unsupported curve/group");
  t.reset(new b200_table_s());
  t->dev = dev; t->curve = curve; t->group = group; t->n = n; t->ops = ops;
  t->c = msm_window_with_limit(n, ops->scalar_bits);
  t->nwin = msm_num_windows(ops->scalar_bits, t->c);
  t->precomp = (flags & B200_TABLE_PRECOMP) ? 1 : 0;
  if (env_int("GB200_MSM_PRECOMP", -1) >= 0) t->precomp = env_int("GB200_MSM_PRECOMP", 0) ? 1 : 0;
  const size_t slabs = t->precomp ? (size_t)t->nwin : 1;
  if (slabs * n >= (1ull << 31)) return set_error("table_upload: table too large for 31-bit point indices; shard it");
  t->bytes = slabs * (n ? n : 1) * ops->affine_bytes;
  CK(cudaMalloc(&t->d_points, t->bytes));
  return 0;
}
static int32_t table_finish(DeviceCtx* ctx, b200_table_s* t) {
  if (t->precomp) CK(t->ops->precompute(ctx->stream, (uint32_t)t->n, t->nwin, t->c, t->d_points));
  CK(cudaStreamSynchronize(ctx->stream));
  return 0;
}
// the error of a failed point decode: status = {DECODE_* code, index of the point}
static int32_t decode_failure(const char* what, const uint32_t status[2]) {
  static const char* why[] = {"", "invalid metadata bits", "coordinate not reduced modulo p", "point not on the curve"};
  return set_error(std::string(what) + ": point " + std::to_string(status[1]) + ": " + why[status[0] < 4 ? status[0] : 0]);
}
}  // namespace gb200

extern "C" {

int32_t b200_table_upload(int32_t dev, int32_t curve, int32_t group, const void* points, size_t n, int32_t flags,
                          b200_table_t* out) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  if (!out) return set_error("table_upload: null argument");
  if (n && !points) return set_error("table_upload: null points");
  std::unique_ptr<b200_table_s> t;
  int32_t rc = table_new(dev, curve, group, n, flags, t); if (rc) return rc;
  const cudaMemcpyKind kind = (flags & B200_TABLE_SRC_ON_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (n) CK(cudaMemcpyAsync(t->d_points, points, n * t->ops->affine_bytes, kind, ctx->stream));
  rc = table_finish(ctx, t.get()); if (rc) return rc;
  *out = t.release();
  return 0;
  GUARD_END
}

// Table from a slice in gnark-crypto's SERIALISED point encoding (points_decode.cuh): what backend/plonk/<curve>/marshal.go
// writes for pk.Kzg / pk.KzgLagrange (compressed with WriteTo, uncompressed with WriteRawTo) after the slice's uint32
// length.  The bytes go up as they are; one thread per point decodes (a square root per compressed point) straight into
// the table.  Every point is checked (canonical coordinates, on the curve); subgroup membership is not, as with
// gnark's UnsafeReadFrom.  An invalid point fails the call with its index.
int32_t b200_table_upload_encoded(int32_t dev, int32_t curve, int32_t group, const void* bytes, size_t n, int32_t encoding,
                                  int32_t flags, b200_table_t* out) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  if (!out || (n && !bytes)) return set_error("table_upload_encoded: null argument");
  if (flags & B200_TABLE_SRC_ON_DEVICE) return set_error("table_upload_encoded: the encoded slice is read from host memory");
  if (curve < 0 || curve > 3) return set_error("table_upload_encoded: unsupported curve");
  std::unique_ptr<b200_table_s> t;
  int32_t rc = table_new(dev, curve, group, n, flags, t); if (rc) return rc;
  const size_t per = t->ops->encoded_bytes(encoding);
  if (per == 0) return set_error("table_upload_encoded: unknown encoding (1 = raw, 2 = compressed)");
  if (n) {
    Staging st(ctx);
    uint32_t status[2] = {0, 0};
    const void* d_bytes;
    void* d_status;
    CK(st.in(bytes, n * per, false, &d_bytes));
    CK(st.out(status, sizeof(status), false, &d_status));
    CK(cudaMemsetAsync(d_status, 0, sizeof(status), ctx->stream));
    cudaError_t e = t->ops->decode(ctx->stream, d_bytes, n, encoding, curve, group, t->d_points, (uint32_t*)d_status);
    if (e == cudaErrorNotSupported) return set_error("table_upload_encoded: encoding not supported for this group");
    if (e != cudaSuccess) return cuda_fail("points decode", e);
    rc = st.finish("table_upload_encoded", 0);
    if (rc) return rc;
    if (status[0]) return decode_failure("table_upload_encoded", status);
  }
  rc = table_finish(ctx, t.get()); if (rc) return rc;
  *out = t.release();
  return 0;
  GUARD_END
}

// Table straight from a file region (SURVEY.md §8f-1): the point slices of gnark's ProvingKey dump
// (backend/groth16/bn254/marshal.go:375-539: G1.A, G1.B, G1.Z, G1.K, G2.B written by unsafe.WriteSlice as raw memory
// images, i.e. exactly the device table layout) are read chunk by chunk into two pinned slots and copied to the device
// while the next chunk is being read, then handed to b200_table_upload as a device-resident source.  The Go shim reads
// the dump's header with gnark-crypto's own decoder and passes the byte offset of each slice's payload; a shard passes
// the offset of ITS point range, so that no process ever holds the whole key in host memory.
int32_t b200_table_upload_file(int32_t dev, int32_t curve, int32_t group, const char* path, uint64_t byte_offset, size_t n,
                               int32_t flags, b200_table_t* out) {
  GUARD_BEGIN
  if (!path || !out) return set_error("table_upload_file: null argument");
  if (flags & B200_TABLE_SRC_ON_DEVICE) return set_error("table_upload_file: the source is a file");
  GB_DEVICE(ctx, dev);
  const MsmOps* ops = get_msm_ops(curve, group);
  if (!ops) return set_error("table_upload_file: unsupported curve/group");
  const size_t bytes = n * ops->affine_bytes;
  struct Fd { int fd = -1; ~Fd() { if (fd >= 0) close(fd); } } f;
  f.fd = open(path, O_RDONLY | O_CLOEXEC);
  if (f.fd < 0) return set_error(std::string("table_upload_file: cannot open ") + path + ": " + strerror(errno));
  struct stat st;
  if (fstat(f.fd, &st) != 0) return set_error(std::string("table_upload_file: fstat: ") + strerror(errno));
  if ((uint64_t)st.st_size < byte_offset || (uint64_t)st.st_size - byte_offset < bytes)
    return set_error("table_upload_file: [offset, offset + n * sizeof(point)) exceeds the file");
  std::unique_ptr<b200_table_s> t;
  int32_t rc = table_new(dev, curve, group, n, flags, t); if (rc) return rc;
  if (n) {
    // the file region goes through two pinned slots straight into slab 0 of the table: no second device copy of the
    // slice, peak HBM = the table itself
    const size_t slot_bytes = bytes < ((size_t)32 << 20) ? bytes : ((size_t)32 << 20);
    struct Pinned { void* p[2] = {nullptr, nullptr}; cudaEvent_t ev[2] = {nullptr, nullptr};
                    ~Pinned() { for (int i = 0; i < 2; i++) { if (p[i]) cudaFreeHost(p[i]); if (ev[i]) cudaEventDestroy(ev[i]); } } } pin;
    for (int i = 0; i < 2; i++) {
      CK(cudaHostAlloc(&pin.p[i], slot_bytes, cudaHostAllocDefault));
      CK(cudaEventCreateWithFlags(&pin.ev[i], cudaEventDisableTiming));
    }
    bool used[2] = {false, false};
    cudaError_t ce = cudaSuccess;
    std::string err;
    char* dst = reinterpret_cast<char*>(t->d_points);
    const int r = stage_file_region(
        f.fd, byte_offset, bytes, pin.p, slot_bytes,
        [&](int slot, const void* data, size_t pos, size_t len) {
          ce = cudaMemcpyAsync(dst + pos, data, len, cudaMemcpyHostToDevice, ctx->copy_stream);
          if (ce == cudaSuccess) ce = cudaEventRecord(pin.ev[slot], ctx->copy_stream);
          used[slot] = true;
          return ce == cudaSuccess ? 0 : 1;
        },
        [&](int slot) {
          if (!used[slot]) return 0;
          ce = cudaEventSynchronize(pin.ev[slot]);
          return ce == cudaSuccess ? 0 : 1;
        },
        &err);
    cudaError_t ce2 = cudaStreamSynchronize(ctx->copy_stream);
    if (ce != cudaSuccess) return cuda_fail("table_upload_file", ce);
    if (r != 0) return set_error("table_upload_file: " + err);
    if (ce2 != cudaSuccess) return cuda_fail("table_upload_file", ce2);
  }
  rc = table_finish(ctx, t.get()); if (rc) return rc;
  *out = t.release();
  return 0;
  GUARD_END
}

int32_t b200_table_free(b200_table_t t) {
  GUARD_BEGIN
  if (!t) return 0;
  GB_DEVICE(ctx, t->dev);
  CK(cudaStreamSynchronize(ctx->stream));
  delete t;       // ~b200_table_s releases the device buffers
  return 0;
  GUARD_END
}

int32_t b200_table_info(b200_table_t t, size_t* n, int32_t* c, int32_t* nwin, int32_t* precomp, size_t* bytes) {
  GUARD_BEGIN
  if (!t) return set_error("table_info: null table");
  if (n) *n = t->n;
  if (c) *c = t->c;
  if (nwin) *nwin = t->nwin;
  if (precomp) *precomp = t->precomp;
  if (bytes) *bytes = t->bytes;
  return 0;
  GUARD_END
}

// ---- MSM -----------------------------------------------------------------------
int32_t b200_msm_async(b200_table_t t, size_t off, size_t n, const void* d_scalars, void* d_out) {
  GUARD_BEGIN
  if (!t) return set_error("msm: null table");
  GB_DEVICE(ctx, t->dev);
  return msm_on_stream(ctx, t, off, n, d_scalars, d_out);
  GUARD_END
}

int32_t b200_fixed_base_batch(int32_t dev, int32_t curve, int32_t group, const void* base_affine,
                              const void* scalars, int32_t scalars_on_device, size_t n, void* out_affine,
                              int32_t out_on_device) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const MsmOps* ops = get_msm_ops(curve, group);
  if (!ops) return set_error("fixed_base_batch: unsupported curve/group");
  if (!base_affine || (n && (!scalars || !out_affine))) return set_error("fixed_base_batch: null argument");
  if (n == 0) return 0;
  int32_t rc = msm_join(ctx); if (rc) return rc;
  Staging st(ctx);
  const void* d_sc;
  void* d_out;
  CK(st.in(scalars, n * ops->fr_bytes, scalars_on_device, &d_sc));
  CK(st.out(out_affine, n * ops->affine_bytes, out_on_device, &d_out));
  int c = env_int("GB200_FIXED_BASE_WINDOW", 0);
  if (c < 2 || c > 16) c = fixed_base_window_for(n);
  return st.finish("fixed_base_batch", ops->fixed_base(ctx->stream, base_affine, d_sc, n, c, d_out));
  GUARD_END
}

// step profile: device time of each pipeline stage of one MSM (ms), stages =
// {decompose, sort, offsets+task scan, accumulate, combine, reduce chunks, set sum+finish}
int32_t b200_msm_profile(b200_table_t t, size_t off, size_t n, const void* d_scalars, void* d_out, float* stage_ms) {
  GUARD_BEGIN
  if (!t || !stage_ms) return set_error("msm_profile: null argument");
  GB_DEVICE(ctx, t->dev);
  cudaEvent_t ev[8];
  for (int k = 0; k < 8; k++) CK(cudaEventCreate(&ev[k]));
  int32_t rc = msm_on_stream(ctx, t, off, n, d_scalars, d_out, ev);
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (rc == 0 && e == cudaSuccess && n > 0)
    for (int k = 0; k < 7; k++) cudaEventElapsedTime(&stage_ms[k], ev[k], ev[k + 1]);
  for (int k = 0; k < 8; k++) cudaEventDestroy(ev[k]);
  if (rc) return rc;
  if (e != cudaSuccess) return cuda_fail("msm_profile", e);
  return 0;
  GUARD_END
}

int32_t b200_msm_pipelined(b200_table_t t, size_t off, size_t n, const void* d_scalars, void* d_out) {
  GUARD_BEGIN
  if (!t) return set_error("msm: null table");
  GB_DEVICE(ctx, t->dev);
  return msm_on_stream(ctx, t, off, n, d_scalars, d_out, nullptr, true);
  GUARD_END
}
int32_t b200_msm_join(int32_t dev) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  return msm_join(ctx);
  GUARD_END
}

int32_t b200_msm(b200_table_t t, size_t off, size_t n, const void* scalars, int32_t on_dev, void* out_host) {
  GUARD_BEGIN
  if (!t) return set_error("msm: null table");
  if (n && !scalars) return set_error("msm: null scalars");
  GB_DEVICE(ctx, t->dev);
  Staging st(ctx);
  void* d_out;
  const void* sc;
  CK(st.out(out_host, t->ops->jac_bytes, false, &d_out));
  CK(st.in(scalars, n * t->ops->fr_bytes, on_dev, &sc));
  return st.finish("msm", msm_on_stream(ctx, t, off, n, sc, d_out));
  GUARD_END
}

// out[b] = sum_i scalars[b * n + i] * bases[off + i], b < batch: the batch runs as ONE MSM whose bucket sets are the
// items' sets side by side (msm_make_batch_plan) - one decompose, sort and accumulate, one reduction tail whose finish
// runs the items' Horner sums in parallel - instead of `batch` calls that each pay the latency-bound tail and a sync.
int32_t b200_msm_batch(b200_table_t t, size_t off, size_t n, size_t batch, const void* scalars, int32_t on_dev,
                       void* out_host) {
  GUARD_BEGIN
  if (!t) return set_error("msm_batch: null table");
  if (!out_host || (batch && n && !scalars)) return set_error("msm_batch: null argument");
  if (off > t->n || n > t->n - off) return set_error("msm_batch: range [off, off+n) exceeds the table");
  if (batch == 0) return 0;
  // a precomputed table's slabs fix its window; on a plain table the window follows n, as for an indexed MSM (a batch of
  // short vectors against a long SRS must not pay for the table's 2^15-bucket sets)
  const int bits = t->ops->scalar_bits;
  const int c = t->precomp ? t->c : msm_window_with_limit(n, bits);
  const int nwin = msm_num_windows(bits, c);
  const unsigned __int128 entries = (unsigned __int128)batch * n * (unsigned)nwin;
  if (entries >= ((unsigned __int128)1 << 31))
    return set_error("msm_batch: batch * n * windows exceeds 2^31 entries - split the batch into smaller ones");
  // bucket keys are 32-bit with the batch's bucket count as the "no entry" key, and the bucket scan counts them in an int
  const unsigned __int128 buckets = ((unsigned __int128)batch * (t->precomp ? 1u : (unsigned)nwin)) << (c - 1);
  if (buckets >= ((unsigned __int128)1 << 31) - 1)
    return set_error("msm_batch: batch * bucket sets * 2^(c-1) exceeds 2^31 - 2 bucket keys - split the batch into "
                     "smaller ones");
  GB_DEVICE(ctx, t->dev);
  int32_t rc = msm_join(ctx); if (rc) return rc;
  uint32_t task_len, chunk;
  msm_tuning(n, batch, nwin, c, t->precomp, t->ops->acc_blocks_per_sm(), &task_len, &chunk);
  size_t ws_bytes = 0;   // n = 0 writes `batch` points at infinity and needs no workspace
  if (n) CK(t->ops->ws_bytes((uint32_t)n, (uint32_t)batch, (uint32_t)t->n, c, t->precomp, task_len, chunk, &ws_bytes));
  Staging st(ctx);
  void *d_out, *ws;
  const void* sc;
  CK(st.out(out_host, batch * t->ops->jac_bytes, false, &d_out));
  CK(st.in(scalars, batch * n * t->ops->fr_bytes, on_dev, &sc));
  CK(st.scratch(ws_bytes, &ws));
  return st.finish("msm_batch", t->ops->run(ctx->stream, (uint32_t)n, (uint32_t)batch, (uint32_t)t->n, (uint32_t)off, c,
                                            t->precomp, task_len, chunk, t->d_points, sc, d_out, ws, nullptr, nullptr,
                                            nullptr, 0));
  GUARD_END
}

// Asynchronous twin of b200_msm for a STREAM of MSMs from host buffers: the scalar upload of call i+1 (copy
// stream) and the reduction tail + result download of call i (tail stream) overlap the sort/accumulate of the
// calls around them.  Both host buffers must stay valid until b200_sync(dev) returns - use b200_host_alloc
// memory (pinned, C-owned: legal to hold across cgo calls), never Go memory.
int32_t b200_msm_submit(b200_table_t t, size_t off, size_t n, const void* scalars_host, void* out_host) {
  GUARD_BEGIN
  if (!t) return set_error("msm_submit: null table");
  if (!out_host || (n && !scalars_host)) return set_error("msm_submit: null argument");
  GB_DEVICE(ctx, t->dev);
  return msm_submit(ctx, t, off, n, scalars_host, nullptr, out_host);
  GUARD_END
}

// b200_msm_submit with the result left on the DEVICE (d_out_jac, valid after b200_msm_join / b200_sync): the form a
// sharded MSM needs, whose partial results go through b200_points_allreduce before anything is downloaded.
int32_t b200_msm_submit_dev(b200_table_t t, size_t off, size_t n, const void* scalars_host, void* d_out_jac) {
  GUARD_BEGIN
  if (!t) return set_error("msm_submit_dev: null table");
  if (!d_out_jac || (n && !scalars_host)) return set_error("msm_submit_dev: null argument");
  GB_DEVICE(ctx, t->dev);
  return msm_submit(ctx, t, off, n, scalars_host, d_out_jac, nullptr);
  GUARD_END
}

int32_t b200_msm_g1(b200_table_t t, size_t off, size_t n, const void* s, int32_t on_dev, void* out) {
  if (t && t->group != 1) return set_error("msm_g1: table holds G2 points");
  return b200_msm(t, off, n, s, on_dev, out);
}
int32_t b200_msm_g2(b200_table_t t, size_t off, size_t n, const void* s, int32_t on_dev, void* out) {
  if (t && t->group != 2) return set_error("msm_g2: table holds G1 points");
  return b200_msm(t, off, n, s, on_dev, out);
}

// ---- NTT -----------------------------------------------------------------------
int32_t b200_ntt_domain_new(int32_t dev, int32_t curve, uint32_t log2n, const void* gen, const void* coset,
                            b200_domain_t* out) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("ntt_domain_new: unsupported curve");
  if ((int)log2n > ops->two_adicity || log2n > 30)
    return set_error("ntt_domain_new: log2n exceeds the field's 2-adicity / supported size");
  cudaError_t e = cudaSuccess;
  void* impl = ops->domain_new(ctx->stream, (int)log2n, gen, coset, &e);
  if (!impl) return cuda_fail("ntt_domain_new", e);
  b200_domain_s* d = new b200_domain_s();
  d->dev = dev; d->curve = curve; d->logn = (int)log2n; d->ops = ops; d->impl = impl;
  *out = d;
  return 0;
  GUARD_END
}

int32_t b200_ntt_domain_free(b200_domain_t d) {
  GUARD_BEGIN
  if (!d) return 0;
  GB_DEVICE(ctx, d->dev);
  CK(cudaStreamSynchronize(ctx->stream));
  d->ops->domain_free(d->impl);
  delete d;
  return 0;
  GUARD_END
}

int32_t b200_ntt_async(b200_domain_t d, void* d_data, int32_t inverse, int32_t decimation, int32_t on_coset) {
  GUARD_BEGIN
  if (!d) return set_error("ntt: null domain");
  if (decimation != B200_DIF && decimation != B200_DIT) return set_error("ntt: decimation must be DIF or DIT");
  GB_DEVICE(ctx, d->dev);
  CK(d->ops->ntt(ctx->stream, d->impl, d_data, inverse, decimation, on_coset));
  return 0;
  GUARD_END
}

int32_t b200_ntt(b200_domain_t d, void* data, int32_t on_dev, int32_t inverse, int32_t decimation, int32_t on_coset) {
  GUARD_BEGIN
  if (!d) return set_error("ntt: null domain");
  if (decimation != B200_DIF && decimation != B200_DIT) return set_error("ntt: decimation must be DIF or DIT");
  GB_DEVICE(ctx, d->dev);
  Staging st(ctx);
  void* buf;
  CK(st.inout(data, ((size_t)1 << d->logn) * d->ops->fr_bytes, on_dev, &buf));
  return st.finish("ntt", d->ops->ntt(ctx->stream, d->impl, buf, inverse, decimation, on_coset));
  GUARD_END
}

int32_t b200_ntt_batch(b200_domain_t d, void* data, size_t batch, int32_t on_dev, int32_t inverse, int32_t decimation,
                       int32_t on_coset) {
  GUARD_BEGIN
  if (!d) return set_error("ntt_batch: null domain");
  if (decimation != B200_DIF && decimation != B200_DIT) return set_error("ntt_batch: decimation must be DIF or DIT");
  if (batch == 0) return 0;
  if (!data) return set_error("ntt_batch: null data");
  GB_DEVICE(ctx, d->dev);
  Staging st(ctx);
  void* buf;
  CK(st.inout(data, batch * ((size_t)1 << d->logn) * d->ops->fr_bytes, on_dev, &buf));
  return st.finish("ntt_batch", d->ops->ntt_batch(ctx->stream, d->impl, buf, batch, inverse, decimation, on_coset));
  GUARD_END
}

// group-element NTT of the domain's size on G1 points of the domain's curve (points_ntt.cuh), host or device buffer
int32_t b200_points_ntt(b200_domain_t d, int32_t group, void* points_affine, int32_t points_on_dev, int32_t inverse) {
  GUARD_BEGIN
  if (!d) return set_error("points_ntt: null domain");
  if (!points_affine) return set_error("points_ntt: null points");
  if (group != 1) return set_error("points_ntt: only G1 is supported (group must be 1; G2 is not supported)");
  const MsmOps* ops = get_msm_ops(d->curve, group);
  if (!ops || !ops->points_ntt) return set_error("points_ntt: unsupported curve");
  GB_DEVICE(ctx, d->dev);
  int32_t rc = msm_join(ctx); if (rc) return rc;
  Staging st(ctx);
  void* buf;
  CK(st.inout(points_affine, ((size_t)1 << d->logn) * ops->affine_bytes, points_on_dev, &buf));
  return st.finish("points_ntt", ops->points_ntt(ctx->stream, d->impl, buf, inverse));
  GUARD_END
}

// points[i] <- (c * t^i) * points[i] (points_scale.cuh): the point vectors of a Groth16 MPC contribution
int32_t b200_points_scale(int32_t dev, int32_t curve, int32_t group, void* points_affine, size_t n, int32_t points_on_dev,
                          const void* c_mont, const void* t_mont) {
  GUARD_BEGIN
  if (curve < 0 || curve > 3) return set_error("points_scale: unknown curve " + std::to_string(curve));
  if (group != 1 && group != 2) return set_error("points_scale: unknown group " + std::to_string(group) + " (1 = G1, 2 = G2)");
  if (!c_mont) return set_error("points_scale: null c");
  if (n && !points_affine) return set_error("points_scale: null points");
  if (n > PS_MAX_POINTS) return set_error("points_scale: n = " + std::to_string(n) + " exceeds the kernel's 32-bit point indices");
  GB_DEVICE(ctx, dev);
  const MsmOps* ops = get_msm_ops(curve, group);
  if (!ops || !ops->points_scale) return set_error("points_scale: unsupported curve/group");
  if (n == 0) return 0;
  int32_t rc = msm_join(ctx); if (rc) return rc;
  Staging st(ctx);
  void* buf;
  CK(st.inout(points_affine, n * ops->affine_bytes, points_on_dev, &buf));
  return st.finish("points_scale", ops->points_scale(ctx->stream, buf, n, c_mont, t_mont));
  GUARD_END
}

// n encoded points -> n affine points (the decoder of b200_table_upload_encoded).  The points are decoded into a scratch
// buffer and copied out only when every one of them is valid, so a failure leaves out_affine untouched.
int32_t b200_points_decode(int32_t dev, int32_t curve, int32_t group, const void* bytes, size_t n, int32_t encoding,
                           void* out_affine, int32_t out_on_dev) {
  GUARD_BEGIN
  if (curve < 0 || curve > 3) return set_error("points_decode: unknown curve " + std::to_string(curve));
  if (group != 1 && group != 2) return set_error("points_decode: unknown group " + std::to_string(group) + " (1 = G1, 2 = G2)");
  if (encoding != B200_POINTS_RAW && encoding != B200_POINTS_COMPRESSED)
    return set_error("points_decode: unknown encoding " + std::to_string(encoding) + " (1 = raw, 2 = compressed)");
  if (n && !bytes) return set_error("points_decode: null bytes");
  if (n && !out_affine) return set_error("points_decode: null out");
  if (n > 0xffffffffull) return set_error("points_decode: n = " + std::to_string(n) + " exceeds the decoder's 32-bit point indices");
  GB_DEVICE(ctx, dev);
  const MsmOps* ops = get_msm_ops(curve, group);
  if (!ops) return set_error("points_decode: unsupported curve/group");
  const size_t per = ops->encoded_bytes(encoding);
  if (per == 0) return set_error("points_decode: encoding not supported for this group");
  if (n == 0) return 0;
  Staging st(ctx);
  uint32_t status[2] = {0, 0};
  const void* d_bytes;
  void *d_pts, *d_status;
  CK(st.in(bytes, n * per, false, &d_bytes));
  CK(st.scratch(n * ops->affine_bytes, &d_pts));
  CK(st.scratch(sizeof(status), &d_status));
  CK(cudaMemsetAsync(d_status, 0, sizeof(status), ctx->stream));
  cudaError_t e = ops->decode(ctx->stream, d_bytes, n, encoding, curve, group, d_pts, (uint32_t*)d_status);
  if (e == cudaSuccess) e = cudaMemcpyAsync(status, d_status, sizeof(status), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) return st.finish("points_decode", e);
  if (status[0]) return st.finish("points_decode", decode_failure("points_decode", status));
  st.download(out_affine, d_pts, n * ops->affine_bytes, out_on_dev);
  return st.finish("points_decode", 0);
  GUARD_END
}

int32_t b200_groth16_compute_h(b200_domain_t d, const void* a, const void* b, const void* c, size_t len,
                               int32_t in_dev, void* h_out, int32_t out_dev) {
  GUARD_BEGIN
  if (!d) return set_error("compute_h: null domain");
  GB_DEVICE(ctx, d->dev);
  const size_t n = (size_t)1 << d->logn;
  if (len > n) return set_error("compute_h: len exceeds the domain");
  const size_t fb = d->ops->fr_bytes;
  // the transform works in place: device inputs are copied too, into buffers zero-padded to the domain
  Staging st(ctx);
  void* v[3];
  const void* src[3] = {a, b, c};
  for (int k = 0; k < 3; k++) {
    CK(st.scratch(n * fb, &v[k]));
    if (len) CK(st.upload(v[k], src[k], len * fb, in_dev));
    if (len < n) CK(cudaMemsetAsync((char*)v[k] + len * fb, 0, (n - len) * fb, ctx->stream));
  }
  st.download(h_out, v[0], n * fb, out_dev);
  return st.finish("compute_h", d->ops->compute_h(ctx->stream, d->impl, v[0], v[1], v[2]));
  GUARD_END
}

// ---- vector ops -----------------------------------------------------------------
int32_t b200_vec_op(int32_t dev, int32_t curve, int32_t op, void* out, const void* a, const void* b, size_t n) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("vec_op: unsupported curve");
  if (op < 0 || op > 2) return set_error("vec_op: unknown op");
  CK(ops->vec_op(ctx->stream, op, out, a, b, n));
  return 0;
  GUARD_END
}
int32_t b200_vec_bit_reverse(int32_t dev, int32_t curve, void* data, uint32_t log2n) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("vec_bit_reverse: unsupported curve");
  CK(ops->bit_reverse(ctx->stream, data, log2n));
  return 0;
  GUARD_END
}
int32_t b200_vec_scale_powers(int32_t dev, int32_t curve, void* data, size_t n, const void* s, const void* g) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("vec_scale_powers: unsupported curve");
  CK(ops->scale_powers(ctx->stream, data, n, s, g));
  return 0;
  GUARD_END
}

int32_t b200_vec_batch_invert(int32_t dev, int32_t curve, void* data, size_t n) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("vec_batch_invert: unsupported curve");
  CK(ops->batch_invert(ctx->stream, data, n));
  return 0;
  GUARD_END
}

int32_t b200_vec_axpy(int32_t dev, int32_t curve, void* y, const void* a, const void* x, size_t n) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("vec_axpy: unsupported curve");
  if (!a || (n && (!y || !x))) return set_error("vec_axpy: null argument");
  CK(ops->axpy(ctx->stream, y, a, x, n));
  return 0;
  GUARD_END
}
int32_t b200_vec_scan(int32_t dev, int32_t curve, int32_t op, void* data, size_t n, int32_t exclusive) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("vec_scan: unsupported curve");
  if (op != B200_SCAN_PRODUCT && op != B200_SCAN_SUM) return set_error("vec_scan: unknown op");
  CK(ops->scan(ctx->stream, op, data, n, exclusive));
  return 0;
  GUARD_END
}
int32_t b200_plonk_build_z(b200_domain_t d0, const void* l, const void* r, const void* o, const int64_t* perm,
                           const void* beta, const void* gamma, void* z) {
  GUARD_BEGIN
  if (!d0 || !l || !r || !o || !perm || !beta || !gamma || !z) return set_error("plonk_build_z: null argument");
  GB_DEVICE(ctx, d0->dev);
  CK(d0->ops->plonk_build_z(ctx->stream, d0->impl, l, r, o, perm, beta, gamma, z));
  return 0;
  GUARD_END
}
int32_t b200_poly_eval(int32_t dev, int32_t curve, const void* c, size_t n, const void* x, void* out) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("poly_eval: unsupported curve");
  if (!x || !out || (n && !c)) return set_error("poly_eval: null argument");
  CK(ops->poly_eval(ctx->stream, c, n, x, out));
  return 0;
  GUARD_END
}
int32_t b200_poly_div_by_linear(int32_t dev, int32_t curve, void* c, size_t n, const void* z, void* rem) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("poly_div_by_linear: unsupported curve");
  if (!z || !rem || (n && !c)) return set_error("poly_div_by_linear: null argument");
  CK(ops->poly_div_linear(ctx->stream, c, n, z, rem));
  return 0;
  GUARD_END
}

// ---- PLONK ------------------------------------------------------------------------
int32_t b200_plonk_constraints_coset(b200_domain_t d0, const void* big_coset_gen, const void* big_gen,
                                     const b200_plonk_coset_args* args) {
  GUARD_BEGIN
  if (!d0 || !big_coset_gen || !big_gen || !args) return set_error("plonk_constraints_coset: null argument");
  GB_DEVICE(ctx, d0->dev);
  cudaError_t e = d0->ops->plonk_coset(ctx->stream, d0->impl, big_coset_gen, big_gen, args);
  if (e == cudaErrorInvalidValue) return set_error("plonk_constraints_coset: invalid rho / coset index / blinding length");
  if (e != cudaSuccess) return cuda_fail("plonk_constraints_coset", e);
  return 0;
  GUARD_END
}
int32_t b200_plonk_bsb22_coset(b200_domain_t d0, const void* d_qcp, const void* d_pi2, uint32_t coset_index, uint32_t rho,
                               void* d_out) {
  GUARD_BEGIN
  if (!d0 || !d_qcp || !d_pi2 || !d_out) return set_error("plonk_bsb22_coset: null argument");
  GB_DEVICE(ctx, d0->dev);
  cudaError_t e = d0->ops->plonk_bsb22(ctx->stream, d0->impl, d_qcp, d_pi2, coset_index, rho, d_out);
  if (e == cudaErrorInvalidValue) return set_error("plonk_bsb22_coset: invalid rho / coset index");
  if (e != cudaSuccess) return cuda_fail("plonk_bsb22_coset", e);
  return 0;
  GUARD_END
}
int32_t b200_plonk_divide_by_zh(b200_domain_t d1, uint32_t log_n0, void* d_data) {
  GUARD_BEGIN
  if (!d1 || !d_data) return set_error("plonk_divide_by_zh: null argument");
  GB_DEVICE(ctx, d1->dev);
  cudaError_t e = d1->ops->plonk_divide_by_zh(ctx->stream, d1->impl, log_n0, d_data);
  if (e == cudaErrorInvalidValue) return set_error("plonk_divide_by_zh: invalid domain ratio");
  if (e != cudaSuccess) return cuda_fail("plonk_divide_by_zh", e);
  return 0;
  GUARD_END
}

}  // extern "C"

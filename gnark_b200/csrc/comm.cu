// Multi-GPU plumbing of the C ABI (SURVEY.md 8b: "b200_init ... NCCL comm when n_dev>1", 8e): one NCCL communicator
// per device context, owned by the library, and the one exchange the path has - a gather of `world` partial points
// followed by world-1 group additions, done on the device (ncclAllGather + k_points_fold on the device's stream, no
// host round trip).  The reference sums its per-chunk MSM results on the host (icicle.go:383-411) and supports one
// device per proof (opts.go:68-77); this is the multi-device twin of that loop.
//
// NCCL is bound at run time (dlopen "libnccl.so.2"): the library still loads, and every single-GPU entry point still
// works, on a machine without NCCL; in a PyTorch process the already loaded NCCL is picked up.  Group addition is not
// an NCCL reduction operator, so the collective is an all-gather and the reduction is our own kernel.
#include <dlfcn.h>
#include <nccl.h>

#include "capi_common.h"

namespace gb200 {

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string error;
};

static NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      api.handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) { api.error = std::string("NCCL not available: ") + dlerror(); return; }
    auto sym = [&](const char* n) -> void* {
      void* p = dlsym(api.handle, n);
      if (!p && api.error.empty()) api.error = std::string("NCCL symbol missing: ") + n;
      return p;
    };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.CommInitAll = reinterpret_cast<decltype(api.CommInitAll)>(sym("ncclCommInitAll"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
  });
  return &api;
}

static int32_t nccl_fail(const NcclApi* api, const char* what, ncclResult_t r) {
  return set_error(std::string(what) + ": " + (api->GetErrorString ? api->GetErrorString(r) : "NCCL error"));
}

#define NCK(api, x)                                             \
  do {                                                          \
    ncclResult_t r_ = (x);                                      \
    if (r_ != ncclSuccess) return nccl_fail(api, #x, r_);       \
  } while (0)

void comm_teardown(DeviceCtx& c) {
  if (c.comm) {
    NcclApi* api = nccl_api();
    if (api->CommDestroy) api->CommDestroy(reinterpret_cast<ncclComm_t>(c.comm));
    c.comm = nullptr;
  }
  c.comm_world = 1;
  c.comm_rank = 0;
}

// gather + fold of `count` Jacobian points on ctx->stream; d_partials and d_totals may alias
int32_t points_allreduce_on_stream(DeviceCtx* ctx, const MsmOps* ops, const void* d_partials, size_t count, void* d_totals) {
  if (count == 0) return 0;
  int32_t rc = msm_join(ctx);           // partial results may still be in flight on the tail stream
  if (rc) return rc;
  if (!ctx->comm || ctx->comm_world <= 1) {
    if (d_totals != d_partials)
      CK(cudaMemcpyAsync(d_totals, d_partials, count * ops->jac_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return 0;
  }
  NcclApi* api = nccl_api();
  AsyncBuf gathered;
  CK(gathered.alloc((size_t)ctx->comm_world * count * ops->jac_bytes, ctx->stream));
  NCK(api, api->AllGather(d_partials, gathered.p, count * ops->jac_bytes, ncclUint8, reinterpret_cast<ncclComm_t>(ctx->comm),
                          ctx->stream));
  cudaError_t e = ops->fold(ctx->stream, gathered.p, (uint32_t)ctx->comm_world, (uint32_t)count, d_totals);
  cudaError_t e2 = gathered.release_on(ctx->stream);
  if (e != cudaSuccess) return cuda_fail("points fold", e);
  if (e2 != cudaSuccess) return cuda_fail("cudaFreeAsync", e2);
  return 0;
}

}  // namespace gb200

using namespace gb200;

extern "C" {

int32_t b200_comm_unique_id(void* out_id128) {
  GUARD_BEGIN
  if (!out_id128) return set_error("comm_unique_id: null argument");
  NcclApi* api = nccl_api();
  if (!api->error.empty()) return set_error(api->error);
  static_assert(sizeof(ncclUniqueId) == B200_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  NCK(api, api->GetUniqueId(&id));
  memcpy(out_id128, &id, sizeof(id));
  return 0;
  GUARD_END
}

int32_t b200_comm_init(int32_t dev, int32_t world, int32_t rank, const void* id128) {
  GUARD_BEGIN
  if (world < 1 || rank < 0 || rank >= world) return set_error("comm_init: need 0 <= rank < world");
  GB_DEVICE(ctx, dev);
  comm_teardown(*ctx);
  if (world == 1) return 0;
  if (!id128) return set_error("comm_init: null unique id");
  NcclApi* api = nccl_api();
  if (!api->error.empty()) return set_error(api->error);
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t comm = nullptr;
  NCK(api, api->CommInitRank(&comm, world, id, rank));
  ctx->comm = comm;
  ctx->comm_world = world;
  ctx->comm_rank = rank;
  return 0;
  GUARD_END
}

// one process driving several devices (a goroutine / thread per device): all communicators in one call
int32_t b200_comm_init_all(int32_t n_dev, const int32_t* dev_ids) {
  GUARD_BEGIN
  if (n_dev < 1 || !dev_ids || n_dev > GB200_MAX_DEVICES) return set_error("comm_init_all: invalid device list");
  std::vector<DeviceCtx*> ctxs(n_dev);
  for (int i = 0; i < n_dev; i++) {
    int32_t rc = device_ctx(dev_ids[i], &ctxs[i]);
    if (rc) return rc;
    std::lock_guard<std::recursive_mutex> lk(ctxs[i]->mu);
    comm_teardown(*ctxs[i]);
  }
  if (n_dev == 1) return 0;
  NcclApi* api = nccl_api();
  if (!api->error.empty()) return set_error(api->error);
  std::vector<ncclComm_t> comms(n_dev, nullptr);
  std::vector<int> ids(dev_ids, dev_ids + n_dev);
  NCK(api, api->CommInitAll(comms.data(), n_dev, ids.data()));
  for (int i = 0; i < n_dev; i++) {
    std::lock_guard<std::recursive_mutex> lk(ctxs[i]->mu);
    ctxs[i]->comm = comms[i];
    ctxs[i]->comm_world = n_dev;
    ctxs[i]->comm_rank = i;
  }
  return 0;
  GUARD_END
}

int32_t b200_comm_destroy(int32_t dev) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  if (ctx->comm) {
    int32_t rc = msm_join(ctx); if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
  }
  comm_teardown(*ctx);
  return 0;
  GUARD_END
}

int32_t b200_comm_info(int32_t dev, int32_t* world, int32_t* rank) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  if (world) *world = ctx->comm ? ctx->comm_world : 1;
  if (rank) *rank = ctx->comm ? ctx->comm_rank : 0;
  return 0;
  GUARD_END
}

int32_t b200_points_allreduce(int32_t dev, int32_t curve, int32_t group, const void* d_partials, size_t count,
                              void* d_totals) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const MsmOps* ops = get_msm_ops(curve, group);
  if (!ops) return set_error("points_allreduce: unsupported curve/group");
  if (count && (!d_partials || !d_totals)) return set_error("points_allreduce: null argument");
  return points_allreduce_on_stream(ctx, ops, d_partials, count, d_totals);
  GUARD_END
}

// the kernel half on its own: for callers that gather the partial points themselves (one process driving several
// devices with peer copies, or results collected from another transport)
int32_t b200_points_fold(int32_t dev, int32_t curve, int32_t group, const void* d_gathered, uint32_t world, uint32_t count,
                         void* d_totals) {
  GUARD_BEGIN
  GB_DEVICE(ctx, dev);
  const MsmOps* ops = get_msm_ops(curve, group);
  if (!ops) return set_error("points_fold: unsupported curve/group");
  if (count && world && (!d_gathered || !d_totals)) return set_error("points_fold: null argument");
  if (world == 0) return set_error("points_fold: world must be at least 1");
  int32_t rc = msm_join(ctx); if (rc) return rc;
  CK(ops->fold(ctx->stream, d_gathered, world, count, d_totals));
  return 0;
  GUARD_END
}

// b200_msm on a point-range shard + the combine: every rank passes ITS scalars for ITS table shard; out_host receives
// the sum over all ranks (on every rank).  Without a communicator this is b200_msm.
int32_t b200_msm_allreduce(b200_table_t t, size_t off, size_t n, const void* scalars, int32_t on_dev, void* out_host) {
  GUARD_BEGIN
  if (!t) return set_error("msm_allreduce: null table");
  if (!out_host || (n && !scalars)) return set_error("msm_allreduce: null argument");
  GB_DEVICE(ctx, t->dev);
  Staging st(ctx);
  void* d_out;
  const void* sc;
  CK(st.out(out_host, t->ops->jac_bytes, false, &d_out));
  CK(st.in(scalars, n * t->ops->fr_bytes, on_dev, &sc));
  int32_t rc = msm_on_stream(ctx, t, off, n, sc, d_out);
  if (rc == 0) rc = points_allreduce_on_stream(ctx, t->ops, d_out, 1, d_out);
  return st.finish("msm_allreduce", rc);
  GUARD_END
}

}  // extern "C"

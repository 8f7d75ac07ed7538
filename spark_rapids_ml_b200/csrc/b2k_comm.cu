// NCCL communicator lifecycle + the per-iteration allreduce of the fused [k*d sums | k counts | cost]
// buffer (reference: common/cuml_context.py:75-81,123-131,158-175 and the two raft::comms allreduce calls
// inside cuML's KMeansMG — SURVEY.md §8a a-8, a-11).  libnccl is resolved at run time, once per process: the
// library named by B2K_NCCL_LIB when that is set (a failure to load it is an error, never a fall-back), else the
// copy torch already mapped or the system one.  So the library has no link-time NCCL dependency and single-GPU
// users never touch it.
#include <dlfcn.h>
#include <string.h>

#include "b2k_internal.cuh"

namespace {
// Minimal NCCL ABI (stable since 2.x): opaque comm, 128-byte unique id, enum values below.
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess_ = 0 };
enum { ncclUint8_ = 1, ncclInt64_ = 4, ncclUint64_ = 5, ncclFloat32_ = 7, ncclFloat64_ = 8 };  // ncclDataType_t
enum { ncclSum_ = 0 };                                                        // ncclRedOp_t

struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*CommAbort)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  int (*GetVersion)(int*) = nullptr;
  std::string load_err;
};

NcclApi* nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return &api;
  tried = true;
  // The override is loaded first: once torch is imported, libnccl.so.2 is already mapped, so a dlopen of that name
  // always succeeds and an override consulted only after it would never take effect.  RTLD_LOCAL keeps the override's
  // nccl* symbols out of the global namespace, where torch's NCCL resolves its own.
  const char* env = getenv("B2K_NCCL_LIB");
  if (env && *env) {
    api.h = dlopen(env, RTLD_NOW | RTLD_LOCAL);
    if (!api.h) {
      const char* e = dlerror();
      api.load_err = std::string("cannot dlopen B2K_NCCL_LIB=") + env + ": " + (e ? e : "");
      return &api;
    }
  } else {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      api.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (api.h) break;
    }
    if (!api.h) {
      const char* e = dlerror();
      api.load_err = std::string("cannot dlopen libnccl.so.2 (set B2K_NCCL_LIB): ") + (e ? e : "");
      return &api;
    }
  }
#define B2K_SYM(field, name)                                               \
  *(void**)(&api.field) = dlsym(api.h, name);                              \
  if (!api.field) api.load_err += std::string("missing symbol ") + name + "; ";
  B2K_SYM(GetUniqueId, "ncclGetUniqueId");
  B2K_SYM(CommInitRank, "ncclCommInitRank");
  B2K_SYM(CommDestroy, "ncclCommDestroy");
  B2K_SYM(CommAbort, "ncclCommAbort");
  B2K_SYM(AllReduce, "ncclAllReduce");
  B2K_SYM(AllGather, "ncclAllGather");
  B2K_SYM(GetErrorString, "ncclGetErrorString");
  B2K_SYM(GetVersion, "ncclGetVersion");
#undef B2K_SYM
  return &api;
}
}  // namespace

struct B2kNccl {
  ncclComm_t comm = nullptr;
};

static int nccl_fail(b2k_ctx* ctx, const char* what, int rc) {
  NcclApi* a = nccl_api();
  std::string m = std::string(what) + ": NCCL error " + std::to_string(rc);
  if (a->GetErrorString) m += std::string(" (") + a->GetErrorString(rc) + ")";
  return b2k_fail(ctx, B2K_ERR_NCCL, m);
}

extern "C" int b2k_comm_unique_id(char out[B2K_UNIQUE_ID_BYTES]) {
  if (!out) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_comm_unique_id: out is NULL");
  NcclApi* a = nccl_api();
  if (!a->h || !a->load_err.empty()) return b2k_fail(nullptr, B2K_ERR_NCCL, a->load_err);
  ncclUniqueId id;
  int rc = a->GetUniqueId(&id);
  if (rc != ncclSuccess_) return nccl_fail(nullptr, "ncclGetUniqueId", rc);
  static_assert(sizeof(ncclUniqueId) == B2K_UNIQUE_ID_BYTES, "uid size");
  memcpy(out, id.internal, B2K_UNIQUE_ID_BYTES);
  return B2K_OK;
}

extern "C" int b2k_comm_init(b2k_ctx* ctx, int nranks, int rank, const char uid[B2K_UNIQUE_ID_BYTES]) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_comm_init: ctx is NULL");
  if (nranks < 1 || rank < 0 || rank >= nranks || !uid)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_comm_init: bad nranks/rank/uid");
  if (ctx->nccl) return b2k_fail(ctx, B2K_ERR_STATE, "b2k_comm_init: communicator already initialised");
  NcclApi* a = nccl_api();
  if (!a->h || !a->load_err.empty()) return b2k_fail(ctx, B2K_ERR_NCCL, a->load_err);
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  ncclUniqueId id;
  memcpy(id.internal, uid, B2K_UNIQUE_ID_BYTES);
  B2kNccl* n = new B2kNccl();
  int rc = a->CommInitRank(&n->comm, nranks, id, rank);
  if (rc != ncclSuccess_) {
    delete n;
    return nccl_fail(ctx, "ncclCommInitRank", rc);
  }
  ctx->nccl = n;
  ctx->nranks = nranks;
  ctx->rank = rank;
  return B2K_OK;
}

extern "C" int b2k_comm_destroy(b2k_ctx* ctx) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_comm_destroy: ctx is NULL");
  if (!ctx->nccl) return B2K_OK;
  NcclApi* a = nccl_api();
  int rc = a->CommDestroy(ctx->nccl->comm);
  delete ctx->nccl;
  ctx->nccl = nullptr;
  ctx->nranks = 1;
  ctx->rank = 0;
  if (rc != ncclSuccess_) return nccl_fail(ctx, "ncclCommDestroy", rc);
  return B2K_OK;
}

extern "C" int b2k_comm_abort(b2k_ctx* ctx) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_comm_abort: ctx is NULL");
  if (!ctx->nccl) return B2K_OK;
  NcclApi* a = nccl_api();
  int rc = a->CommAbort(ctx->nccl->comm);
  delete ctx->nccl;
  ctx->nccl = nullptr;
  ctx->nranks = 1;
  ctx->rank = 0;
  if (rc != ncclSuccess_) return nccl_fail(ctx, "ncclCommAbort", rc);
  return B2K_OK;
}

int b2k_comm_allreduce_f64(b2k_ctx* ctx, double* buf, size_t count, cudaStream_t s) {
  if (!ctx->nccl || ctx->nranks == 1) return B2K_OK;
  int rc = nccl_api()->AllReduce(buf, buf, count, ncclFloat64_, ncclSum_, ctx->nccl->comm, s);
  ctx->stats.nccl_allreduces++;
  if (rc != ncclSuccess_) return nccl_fail(ctx, "ncclAllReduce(f64)", rc);
  return B2K_OK;
}

int b2k_comm_allreduce_f32(b2k_ctx* ctx, float* buf, size_t count, cudaStream_t s) {
  if (!ctx->nccl || ctx->nranks == 1) return B2K_OK;
  int rc = nccl_api()->AllReduce(buf, buf, count, ncclFloat32_, ncclSum_, ctx->nccl->comm, s);
  ctx->stats.nccl_allreduces++;
  if (rc != ncclSuccess_) return nccl_fail(ctx, "ncclAllReduce(f32)", rc);
  return B2K_OK;
}

int b2k_comm_allreduce_i64(b2k_ctx* ctx, int64_t* buf, size_t count, cudaStream_t s) {
  if (!ctx->nccl || ctx->nranks == 1) return B2K_OK;
  int rc = nccl_api()->AllReduce(buf, buf, count, ncclInt64_, ncclSum_, ctx->nccl->comm, s);
  ctx->stats.nccl_allreduces++;
  if (rc != ncclSuccess_) return nccl_fail(ctx, "ncclAllReduce(i64)", rc);
  return B2K_OK;
}

int b2k_comm_allgather_i64(b2k_ctx* ctx, const int64_t* send_dev, int64_t* recv_dev, size_t count_per_rank,
                           cudaStream_t s) {
  if (!ctx->nccl || ctx->nranks == 1) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(recv_dev, send_dev, count_per_rank * sizeof(int64_t),
                                     cudaMemcpyDeviceToDevice, s));
    return B2K_OK;
  }
  int rc = nccl_api()->AllGather(send_dev, recv_dev, count_per_rank, ncclInt64_, ctx->nccl->comm, s);
  if (rc != ncclSuccess_) return nccl_fail(ctx, "ncclAllGather(i64)", rc);
  return B2K_OK;
}

int b2k_comm_allgather_bytes(b2k_ctx* ctx, const void* send_dev, void* recv_dev, size_t bytes_per_rank,
                             cudaStream_t s) {
  if (!ctx->nccl || ctx->nranks == 1) {
    if (send_dev != recv_dev)
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(recv_dev, send_dev, bytes_per_rank, cudaMemcpyDeviceToDevice, s));
    return B2K_OK;
  }
  int rc = nccl_api()->AllGather(send_dev, recv_dev, bytes_per_rank, ncclUint8_, ctx->nccl->comm, s);
  if (rc != ncclSuccess_) return nccl_fail(ctx, "ncclAllGather(u8)", rc);
  return B2K_OK;
}

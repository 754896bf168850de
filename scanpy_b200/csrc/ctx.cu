// ctx.cu — context, error text, device info, NCCL attachment.
#include <string.h>
#include <dlfcn.h>

#include "common.cuh"

static thread_local char g_err[1024] = "";

void sb2_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" {

int32_t sb2_version(void) { return 100; }
const char* sb2_last_error(void) { return g_err; }

int32_t sb2_ctx_create(int32_t device, void* stream, uint32_t flags, sb2_ctx** out) {
  SB2_CHECK_ARG(out != nullptr, "out");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    sb2_set_error("no CUDA device available (%s): libscanpy_b200 has no CPU path", cudaGetErrorString(e));
    return SB2_E_CUDA;
  }
  SB2_CHECK_ARG(device >= 0 && device < ndev, "device index");
  SB2_CUDA(cudaSetDevice(device));
  sb2_ctx* c = new sb2_ctx();
  c->device = device;
  SB2_CUDA(cudaGetDeviceProperties(&c->prop, device));
  if (c->prop.major != 9 || c->prop.minor != 0) {
    sb2_set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, c->prop.major,
                  c->prop.minor);
    delete c;
    return SB2_E_UNSUPPORTED;
  }
  if (!(flags & SB2_CTX_PRIVATE_STREAM)) {
    c->stream = reinterpret_cast<cudaStream_t>(stream);  // NULL = legacy default stream
  } else {
    SB2_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  // keep freed scratch in the pool: the same sizes come back every call
  cudaMemPool_t pool;
  SB2_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
  uint64_t thr = UINT64_MAX;
  SB2_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
  *out = c;
  return SB2_OK;
}

int32_t sb2_ctx_sync(sb2_ctx* ctx) {
  SB2_CHECK_ARG(ctx, "ctx");
  SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  return SB2_OK;
}

int64_t sb2_ctx_launch_count(sb2_ctx* ctx) { return ctx ? ctx->launches : -1; }

int32_t sb2_device_info_get(sb2_ctx* ctx, sb2_device_info* o) {
  SB2_CHECK_ARG(ctx && o, "ctx/out");
  memset(o, 0, sizeof(*o));
  o->device = ctx->device;
  o->sm_count = ctx->prop.multiProcessorCount;
  o->cc_major = ctx->prop.major;
  o->cc_minor = ctx->prop.minor;
  int v = 0;
  cudaDeviceGetAttribute(&v, cudaDevAttrClockRate, ctx->device);
  o->clock_khz = v;
  cudaDeviceGetAttribute(&v, cudaDevAttrMemoryClockRate, ctx->device);
  o->mem_clock_khz = v;
  o->l2_bytes = ctx->prop.l2CacheSize;
  o->smem_per_block_optin = (int32_t)ctx->prop.sharedMemPerBlockOptin;
  o->total_mem = (int64_t)ctx->prop.totalGlobalMem;
  strncpy(o->name, ctx->prop.name, sizeof(o->name) - 1);
  return SB2_OK;
}

// ---------------------------------------------------------------------------------------------
// NCCL is bound at run time with dlopen/dlsym so that the library loads (and every single-GPU entry
// point works) on a machine without libnccl, and so that we share the libnccl.so.2 torch already
// mapped into the process instead of pulling in a second copy.
// ---------------------------------------------------------------------------------------------
typedef struct { char internal[128]; } nccl_uid_t;
typedef int (*p_ncclGetUniqueId)(nccl_uid_t*);
typedef int (*p_ncclCommInitRank)(void**, int, nccl_uid_t, int);
typedef int (*p_ncclCommDestroy)(void*);
typedef int (*p_ncclAllGather)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef int (*p_ncclAllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef const char* (*p_ncclGetErrorString)(int);
static struct {
  void* h = nullptr;
  p_ncclGetUniqueId GetUniqueId;
  p_ncclCommInitRank CommInitRank;
  p_ncclCommDestroy CommDestroy;
  p_ncclAllGather AllGather;
  p_ncclAllReduce AllReduce;
  p_ncclGetErrorString GetErrorString;
} g_nccl;

static int32_t nccl_load() {
  if (g_nccl.h) return SB2_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    sb2_set_error("cannot dlopen libnccl.so.2: %s", dlerror());
    return SB2_E_NCCL;
  }
#define LOADSYM(name)                                              \
  g_nccl.name = (p_nccl##name)dlsym(h, "nccl" #name);              \
  if (!g_nccl.name) {                                              \
    sb2_set_error("libnccl.so.2 lacks symbol nccl" #name);         \
    return SB2_E_NCCL;                                             \
  }
  LOADSYM(GetUniqueId) LOADSYM(CommInitRank) LOADSYM(CommDestroy) LOADSYM(AllGather) LOADSYM(AllReduce)
  LOADSYM(GetErrorString)
#undef LOADSYM
  g_nccl.h = h;
  return SB2_OK;
}
#define SB2_NCCL(expr)                                                                \
  do {                                                                                \
    int _r = (expr);                                                                  \
    if (_r != 0) {                                                                    \
      sb2_set_error("NCCL error %d at %s:%d: %s", _r, __FILE__, __LINE__,             \
                    g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?");         \
      return SB2_E_NCCL;                                                              \
    }                                                                                 \
  } while (0)

int32_t sb2_comm_unique_id(void* h_id128) {
  SB2_CHECK_ARG(h_id128, "id buffer");
  SB2_TRY(nccl_load());
  nccl_uid_t id;
  SB2_NCCL(g_nccl.GetUniqueId(&id));
  memcpy(h_id128, &id, sizeof(id));
  return SB2_OK;
}

int32_t sb2_comm_init(sb2_ctx* ctx, int32_t n_ranks, int32_t rank, const void* h_id128) {
  SB2_CHECK_ARG(ctx && h_id128, "ctx/id");
  SB2_CHECK_ARG(n_ranks >= 1 && rank >= 0 && rank < n_ranks, "rank/n_ranks");
  SB2_TRY(nccl_load());
  SB2_CUDA(cudaSetDevice(ctx->device));
  nccl_uid_t id;
  memcpy(&id, h_id128, sizeof(id));
  void* comm = nullptr;
  SB2_NCCL(g_nccl.CommInitRank(&comm, n_ranks, id, rank));
  ctx->nccl_comm = comm;
  ctx->n_ranks = n_ranks;
  ctx->rank = rank;
  return SB2_OK;
}

int32_t sb2_comm_allgather(sb2_ctx* ctx, const void* d_send, void* d_recv, int64_t bytes_per_rank) {
  SB2_CHECK_ARG(ctx && ctx->nccl_comm, "ctx has no communicator");
  SB2_NCCL(g_nccl.AllGather(d_send, d_recv, (size_t)bytes_per_rank, /*ncclInt8*/ 0, ctx->nccl_comm, ctx->stream));
  return SB2_OK;
}

int32_t sb2_comm_allreduce_f64(sb2_ctx* ctx, double* d_buf, int64_t count) {
  SB2_CHECK_ARG(ctx, "ctx");
  if (!ctx->nccl_comm || ctx->n_ranks == 1) return SB2_OK;
  SB2_NCCL(g_nccl.AllReduce(d_buf, d_buf, (size_t)count, /*ncclFloat64*/ 8, /*ncclSum*/ 0, ctx->nccl_comm,
                            ctx->stream));
  return SB2_OK;
}

int32_t sb2_ctx_destroy(sb2_ctx* ctx) {
  if (!ctx) return SB2_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->nccl_comm && g_nccl.h) g_nccl.CommDestroy(ctx->nccl_comm);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return SB2_OK;
}

}  // extern "C"

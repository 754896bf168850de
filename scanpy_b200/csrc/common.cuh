// common.cuh — shared host/device helpers for libscanpy_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string>
#include <vector>

#include "../../include/scanpy_b200.h"

void sb2_set_error(const char* fmt, ...);

#define SB2_CUDA(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      sb2_set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__,   \
                    cudaGetErrorString(_e));                                                  \
      return _e == cudaErrorMemoryAllocation ? SB2_E_OOM : SB2_E_CUDA;                        \
    }                                                                                         \
  } while (0)

#define SB2_CHECK_ARG(cond, msg)                         \
  do {                                                   \
    if (!(cond)) {                                       \
      sb2_set_error("bad argument: %s (%s)", msg, #cond); \
      return SB2_E_BADARG;                               \
    }                                                    \
  } while (0)

#define SB2_TRY(expr)            \
  do {                           \
    int32_t _r = (expr);         \
    if (_r != SB2_OK) return _r; \
  } while (0)

struct sb2_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaDeviceProp prop{};
  int64_t launches = 0;
  void* nccl_comm = nullptr;  // ncclComm_t
  int n_ranks = 1, rank = 0;
  std::vector<void*> scratch;  // stream-ordered allocations owned by the current call
};

// Stream-ordered scratch: freed (stream-ordered) by ScratchScope's destructor.
struct ScratchScope {
  sb2_ctx* ctx;
  std::vector<void*> ptrs;
  explicit ScratchScope(sb2_ctx* c) : ctx(c) {}
  ~ScratchScope() {
    for (void* p : ptrs) cudaFreeAsync(p, ctx->stream);
  }
  template <typename T>
  int32_t alloc(T** out, size_t count) {
    void* p = nullptr;
    size_t bytes = count * sizeof(T);
    if (bytes == 0) bytes = 16;
    cudaError_t e = cudaMallocAsync(&p, bytes, ctx->stream);
    if (e != cudaSuccess) {
      sb2_set_error("cudaMallocAsync(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
      *out = nullptr;
      return e == cudaErrorMemoryAllocation ? SB2_E_OOM : SB2_E_CUDA;
    }
    ptrs.push_back(p);
    *out = reinterpret_cast<T*>(p);
    return SB2_OK;
  }
};

#define SB2_LAUNCH_CHECK(ctx)            \
  do {                                   \
    (ctx)->launches++;                   \
    SB2_CUDA(cudaPeekAtLastError());     \
  } while (0)

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// debug-only phase timing (SB2_TIMING=1): synchronises the stream, so never enabled in measured runs
#include <chrono>
#include <stdlib.h>
struct PhaseTimer {
  bool on;
  cudaStream_t st;
  std::chrono::steady_clock::time_point t0;
  explicit PhaseTimer(cudaStream_t s) : on(getenv("SB2_TIMING") != nullptr), st(s) { reset(); }
  void reset() {
    if (on) { cudaStreamSynchronize(st); t0 = std::chrono::steady_clock::now(); }
  }
  // adds the time since the last reset()/lap() to *acc (milliseconds)
  void lap(double* acc) {
    if (!on) return;
    cudaStreamSynchronize(st);
    auto t1 = std::chrono::steady_clock::now();
    *acc += std::chrono::duration<double, std::milli>(t1 - t0).count();
    t0 = t1;
  }
};

#ifdef __CUDACC__
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// sum over the CTA of one value per thread, in a fixed order (warp tree, then warps in order); result on thread 0
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  T s = 0;
  if (threadIdx.x == 0)
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  __syncthreads();
  return s;
}
#endif

// ---- util.cu ----
// out[0..n] (int64) = exclusive prefix sum of in[0..n) (int32 counts); out[n] = total
int32_t sb2_scan_i32_to_i64(sb2_ctx* ctx, const int32_t* d_in, int64_t n, int64_t* d_out);
// host cyclic Jacobi: A (m x m symmetric, row-major, destroyed) -> eigenvalues w, eigenvectors V (columns)
void jacobi_eigh(std::vector<double>& A, int m, std::vector<double>& w, std::vector<double>& V);

// ---- eigs.cu ----
// sb2_eigsh_csr_scaled with the search for missed copies of the wanted eigenvalues made optional: without it, the first
// set whose residuals converge is returned (the UMAP spectral initialisation, which lays out a disconnected graph as one)
int32_t eigsh_csr_scaled(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices, const float* d_weights,
                         const double* d_scale, int32_t nev, int32_t which, int32_t ncv, double tol, int32_t max_restarts,
                         const double* d_v0, double* h_evals, double* d_evecs, sb2_eigs_info* info, bool lock_and_search);

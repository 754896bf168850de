// umap.cu — sc.tl.umap's layout optimisation on the device (SURVEY.md 8f row f1).
//
// Replaces `umap.umap_.simplicial_set_embedding(...)` as called at src/scanpy/tools/_umap.py:196-215 (umap-learn is a
// third-party dependency, not vendored in the reference; algorithm restated from umap/umap_.py `simplicial_set_embedding`,
// `make_epochs_per_sample` and umap/layouts.py `_optimize_layout_euclidean_single_epoch`):
//   * edges with weight < max/n_epochs are dropped; edge e is sampled every eps_e = max_w / w_e epochs;
//   * a sampled edge (j,k) pulls j towards k with  -2ab d^(2(b-1)) / (a d^(2b) + 1), every coordinate of the step clipped to
//     [-4, 4], and pushes j away from ~negative_sample_rate random vertices with  2 gamma b / ((0.001 + d^2)(a d^(2b) + 1));
//   * learning rate alpha = initial_alpha (1 - epoch / n_epochs).
// Schedule: umap walks the COO edge list sequentially (or hogwild with parallel=True, which is what scanpy selects when
// no seed is given) and moves both end points of a sampled edge.  Here a THREAD OWNS A VERTEX: it walks its CSR row,
// keeps its own position in registers and updates it edge after edge (Gauss-Seidel inside the vertex, exactly umap's
// order within one head vertex), reading the other end points from the previous epoch's snapshot (double buffer).  The
// graph is symmetric, so the "move the other end" half of edge (k,j) is applied by j's owner as a second pull along
// (j,k) in the same epoch: same forces, same clipping, same schedule, no write races, and the result is a
// deterministic function of (graph, init, seed) whatever the launch geometry.
// Sampling epochs are closed forms of umap's running counters (cnt-th sample of an edge at epoch ceil(cnt * eps)), so no
// per-edge state is kept: one epoch reads 8 B per stored arc + the L2-resident embedding (8 B per vertex for 2-D).
#include <math.h>

#include "common.cuh"

namespace {

__device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ float clip4(float v) { return fminf(4.0f, fmaxf(-4.0f, v)); }

// weights -> epochs_per_sample (fp32, 0 = never sampled): eps = max_w / w for w >= max_w / n_epochs
__global__ void umap_eps_kernel(int64_t nnz, const float* __restrict__ w, const float* __restrict__ wmax_p, int n_epochs,
                                float* __restrict__ eps) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nnz) return;
  const float wmax = *wmax_p;
  const float x = w[i];
  eps[i] = (wmax > 0.0f && x > 0.0f && x >= wmax / (float)n_epochs) ? wmax / x : 0.0f;
}
__global__ void umap_wmax_kernel(int64_t nnz, const float* __restrict__ w, float* __restrict__ wmax) {
  float m = 0.0f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, w[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(wmax), __float_as_int(m));  // w >= 0: int order == float order
}

template <int DIM>
__global__ void __launch_bounds__(128)
umap_epoch_kernel(int32_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                  const float* __restrict__ eps, const float* __restrict__ pos_in, float* __restrict__ pos_out, int epoch,
                  float alpha, float a, float b, float gamma, int neg_rate, uint32_t seed) {
  const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  float cur[DIM];
#pragma unroll
  for (int d = 0; d < DIM; ++d) cur[d] = pos_in[(size_t)j * DIM + d];
  const double nd = (double)epoch;
  for (int64_t e = indptr[j]; e < indptr[j + 1]; ++e) {
    const float ep = eps[e];
    if (ep <= 0.0f) continue;
    // cnt = number of samples of this edge up to and including this epoch; sampled now iff the count just went up
    const double epd = (double)ep;
    const int64_t cnt = (int64_t)floor(nd / epd);
    if (cnt < 1 || (int64_t)floor((nd - 1.0) / epd) >= cnt) continue;
    const int32_t k = indices[e];
    float oth[DIM];
#pragma unroll
    for (int d = 0; d < DIM; ++d) oth[d] = pos_in[(size_t)k * DIM + d];
    // two pulls: edge (j,k) moving its head j, and edge (k,j) moving its tail j (move_other=True)
#pragma unroll
    for (int rep = 0; rep < 2; ++rep) {
      float d2 = 0.0f;
#pragma unroll
      for (int d = 0; d < DIM; ++d) { const float t = cur[d] - oth[d]; d2 += t * t; }
      if (d2 > 0.0f) {
        const float pb = __powf(d2, b);
        const float gc = -2.0f * a * b * (pb / d2) / (a * pb + 1.0f);
#pragma unroll
        for (int d = 0; d < DIM; ++d) cur[d] += clip4(gc * (cur[d] - oth[d])) * alpha;
      }
    }
    // negative samples owed since the previous sample of this edge (umap's epoch_of_next_negative_sample bookkeeping):
    // floor(epoch * rate / eps) with the integer product divided last, so that it is exact when eps divides it
    const double rate = (double)neg_rate;
    const int64_t c_now = (int64_t)floor(nd * rate / epd);
    int64_t c_prev = 1;
    if (cnt > 1) c_prev = (int64_t)floor(ceil((double)(cnt - 1) * epd) * rate / epd);
    if (c_prev < 1) c_prev = 1;
    const int n_neg = (int)min((int64_t)64, max((int64_t)0, c_now - c_prev));
    uint32_t h = hash32(seed ^ hash32((uint32_t)epoch * 0x9E3779B9U + (uint32_t)(e & 0xffffffffu)));
    for (int p = 0; p < n_neg; ++p) {
      h = hash32(h + 0x6D2B79F5U * (uint32_t)(p + 1));
      const int32_t kk = (int32_t)(((uint64_t)h * (uint64_t)n) >> 32);
      if (kk == j) continue;
      float d2 = 0.0f;
      float df[DIM];
#pragma unroll
      for (int d = 0; d < DIM; ++d) { df[d] = cur[d] - pos_in[(size_t)kk * DIM + d]; d2 += df[d] * df[d]; }
      if (d2 > 0.0f) {
        const float gc = 2.0f * gamma * b / ((0.001f + d2) * (a * __powf(d2, b) + 1.0f));
        if (gc > 0.0f) {
#pragma unroll
          for (int d = 0; d < DIM; ++d) cur[d] += clip4(gc * df[d]) * alpha;
        }
      }
    }
  }
#pragma unroll
  for (int d = 0; d < DIM; ++d) pos_out[(size_t)j * DIM + d] = cur[d];
}


// The kernel above is divergence-bound (one vertex per lane, each lane in its own edge).  Giving a vertex EIGHT LANES -
// lane 0 the double pull, lanes 1..7 the negative samples of a sampled edge, displacements summed by a shuffle tree - does
// not remove that: the four groups of a warp still sit in different edges, so the divergence only moves from lanes to
// groups; removing it needs forces that are simultaneous across a vertex's edges (a different optimiser), not a different
// thread mapping.

// per-dimension min / max (float atomics through the ordered-int trick)
__device__ __forceinline__ int f2ord(float f) { const int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }
__global__ void umap_minmax_kernel(int64_t n, int dim, const float* __restrict__ x, int* __restrict__ mn, int* __restrict__ mx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * dim; i += (int64_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % dim);
    const float v = x[i];
    if (isfinite(v)) { atomicMin(&mn[d], f2ord(v)); atomicMax(&mx[d], f2ord(v)); }
  }
}
// mode 0: x = 10 (x - min_d) / (max_d - min_d)   (simplicial_set_embedding's final rescale of the initialisation)
// mode 1: x = x * (10 / max|x|) + N(0, 1e-4)     (expansion + jitter of the spectral initialisation)
__global__ void umap_rescale_kernel(int64_t n, int dim, float* __restrict__ x, const int* __restrict__ mn, const int* __restrict__ mx,
                                    int mode, uint32_t seed) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * dim) return;
  const int d = (int)(i % dim);
  if (mode == 0) {
    const float lo = ord2f(mn[d]), hi = ord2f(mx[d]);
    x[i] = hi > lo ? 10.0f * (x[i] - lo) / (hi - lo) : 0.0f;
  } else {
    float amax = 0.0f;
    for (int q = 0; q < dim; ++q) amax = fmaxf(amax, fmaxf(fabsf(ord2f(mn[q])), fabsf(ord2f(mx[q]))));
    const uint32_t h1 = hash32(seed ^ hash32((uint32_t)i * 2u + 1u)), h2 = hash32(seed + 0x9E3779B9U + hash32((uint32_t)i * 2u));
    const float u1 = ((float)(h1 >> 8) + 1.0f) * (1.0f / 16777217.0f), u2 = (float)(h2 >> 8) * (1.0f / 16777216.0f);
    const float g = sqrtf(-2.0f * __logf(u1)) * __cosf(6.2831853f * u2);
    x[i] = x[i] * (amax > 0.0f ? 10.0f / amax : 1.0f) + 1e-4f * g;
  }
}
// evecs fp64 [nev x n] (ascending eigenvalues) -> init fp32 [n x dim]: component c = eigenvector nev-2-c (the top one, the
// trivial eigenvector of the normalised adjacency, is skipped like umap's `order[1:k+1]`)
__global__ void umap_spectral_pick_kernel(int64_t n, int dim, int nev, const double* __restrict__ evecs, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * dim) return;
  const int64_t r = i / dim;
  const int c = (int)(i - r * dim);
  out[i] = (float)evecs[(size_t)(nev - 2 - c) * n + r];
}
// s = 1 / sqrt(degree), degree = row sum of weights
__global__ void umap_invsqrt_deg_kernel(int64_t n, const int64_t* __restrict__ indptr, const float* __restrict__ w, double* __restrict__ s) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  double acc = 0.0;
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32) acc += (double)w[e];
  acc = warp_sum(acc);
  if (lane == 0) s[row] = acc > 0.0 ? 1.0 / sqrt(acc) : 0.0;
}
__global__ void umap_v0_kernel(int64_t n, double* __restrict__ v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = 1.0 + 1e-3 * (double)(hash32((uint32_t)i) >> 8) * (1.0 / 16777216.0);  // ~ umap's v0 = ones, off the exact eigenvector
}

template <int DIM>
int32_t run_epochs(sb2_ctx* ctx, int32_t n, const int64_t* indptr, const int32_t* indices, const float* eps, float* pos,
                   float* tmp, int n_epochs, float alpha0, float a, float b, float gamma, int neg_rate, uint32_t seed) {
  float *in = pos, *out = tmp;
  for (int ep = 0; ep < n_epochs; ++ep) {
    const float alpha = alpha0 * (1.0f - (float)ep / (float)n_epochs);
    umap_epoch_kernel<DIM><<<(unsigned)ceil_div64(n, 128), 128, 0, ctx->stream>>>(n, indptr, indices, eps, in, out, ep, alpha, a, b,
                                                                                gamma, neg_rate, seed);
    SB2_LAUNCH_CHECK(ctx);
    std::swap(in, out);
  }
  if (in != pos) SB2_CUDA(cudaMemcpyAsync(pos, in, sizeof(float) * (size_t)n * DIM, cudaMemcpyDeviceToDevice, ctx->stream));
  return SB2_OK;
}

}  // namespace

extern "C" {

// spectral initialisation: d_init fp32 [n x dim] = eigenvectors 2..dim+1 of D^-1/2 A D^-1/2 (largest eigenvalues), expanded
// to max|x| = 10 and jittered with N(0, 1e-4) like umap's `init='spectral'` branch
int32_t sb2_umap_spectral_init_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                   const float* d_weights, int32_t dim, uint64_t seed, float* d_init) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_weights && d_init, "null pointer");
  SB2_CHECK_ARG(dim >= 1 && dim <= 16 && n > dim + 1, "dim must be in [1,16] and < n - 1");
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  const int nev = dim + 1;
  double *s, *v0, *evecs;
  int* mm;
  SB2_TRY(scr.alloc(&s, (size_t)n));
  SB2_TRY(scr.alloc(&v0, (size_t)n));
  SB2_TRY(scr.alloc(&evecs, (size_t)nev * n));
  SB2_TRY(scr.alloc(&mm, 32));
  umap_invsqrt_deg_kernel<<<(unsigned)ceil_div64(n, 8), 256, 0, st>>>(n, d_indptr, d_weights, s);
  SB2_LAUNCH_CHECK(ctx);
  umap_v0_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(n, v0);
  SB2_LAUNCH_CHECK(ctx);
  double evals[17];
  sb2_eigs_info inf{};
  // umap: eigsh(L, k+1, which='SM', ncv=max(2k+1, sqrt(n)), tol=1e-4); an initialisation does not need more.  No search
  // for missed copies of eigenvalue 1: on a disconnected graph they would collapse each component to a point
  int32_t rc = eigsh_csr_scaled(ctx, n, d_indptr, d_indices, d_weights, s, nev, 0, std::max(2 * nev + 16, 40), 1e-5, 60, v0,
                                evals, evecs, &inf, false);
  if (rc != SB2_OK) return rc;
  const unsigned ge = (unsigned)ceil_div64(n * dim, 256);
  umap_spectral_pick_kernel<<<ge, 256, 0, st>>>(n, dim, nev, evecs, d_init);
  SB2_LAUNCH_CHECK(ctx);
  SB2_CUDA(cudaMemsetAsync(mm, 0x7f, sizeof(int) * 16, st));        // min slots: large positive ordered ints
  SB2_CUDA(cudaMemsetAsync(mm + 16, 0x80, sizeof(int) * 16, st));   // max slots: large negative
  umap_minmax_kernel<<<ctx->prop.multiProcessorCount * 4, 256, 0, st>>>(n, dim, d_init, mm, mm + 16);
  SB2_LAUNCH_CHECK(ctx);
  umap_rescale_kernel<<<ge, 256, 0, st>>>(n, dim, d_init, mm, mm + 16, 1, (uint32_t)(seed ^ (seed >> 32)));
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

// d_embedding fp32 [n x dim]: the initialisation on entry (any scale: it is mapped to [0, 10]^dim first, as
// simplicial_set_embedding does), the optimised layout on return.
int32_t sb2_umap_layout_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices, const float* d_weights,
                            int32_t dim, int32_t n_epochs, double a, double b, double gamma, double initial_alpha,
                            int32_t negative_sample_rate, uint64_t seed, float* d_embedding) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_weights && d_embedding, "null pointer");
  SB2_CHECK_ARG(n >= 1 && n < INT32_MAX, "n");
  SB2_CHECK_ARG(dim >= 1 && dim <= 16, "n_components must be in [1,16]");
  SB2_CHECK_ARG(n_epochs >= 0 && negative_sample_rate >= 0, "n_epochs / negative_sample_rate");
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  int64_t nnz = 0;
  SB2_CUDA(cudaMemcpyAsync(&nnz, d_indptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  float *eps, *tmp, *wmax;
  int* mm;
  SB2_TRY(scr.alloc(&eps, (size_t)std::max<int64_t>(nnz, 1)));
  SB2_TRY(scr.alloc(&tmp, (size_t)n * dim));
  SB2_TRY(scr.alloc(&wmax, 4));
  SB2_TRY(scr.alloc(&mm, 32));
  const unsigned ge = (unsigned)ceil_div64(n * dim, 256);
  SB2_CUDA(cudaMemsetAsync(mm, 0x7f, sizeof(int) * 16, st));
  SB2_CUDA(cudaMemsetAsync(mm + 16, 0x80, sizeof(int) * 16, st));
  umap_minmax_kernel<<<ctx->prop.multiProcessorCount * 4, 256, 0, st>>>(n, dim, d_embedding, mm, mm + 16);
  SB2_LAUNCH_CHECK(ctx);
  umap_rescale_kernel<<<ge, 256, 0, st>>>(n, dim, d_embedding, mm, mm + 16, 0, 0u);
  SB2_LAUNCH_CHECK(ctx);
  if (nnz == 0 || n_epochs == 0) return SB2_OK;
  SB2_CUDA(cudaMemsetAsync(wmax, 0, 16, st));
  umap_wmax_kernel<<<ctx->prop.multiProcessorCount * 4, 256, 0, st>>>(nnz, d_weights, wmax);
  SB2_LAUNCH_CHECK(ctx);
  // n_epochs <= 10 keeps the reference's pruning threshold of the DEFAULT epoch count (umap_.py: `if n_epochs > 10 ... else`)
  const int prune_epochs = n_epochs > 10 ? n_epochs : (n <= 10000 ? 500 : 200);
  umap_eps_kernel<<<(unsigned)ceil_div64(nnz, 256), 256, 0, st>>>(nnz, d_weights, wmax, prune_epochs, eps);
  SB2_LAUNCH_CHECK(ctx);
  const uint32_t sd = (uint32_t)(seed ^ (seed >> 32)) * 2654435761u + 12345u;
  const int32_t nn = (int32_t)n;
#define SB2_UMAP_DIM(D) \
  case D: return run_epochs<D>(ctx, nn, d_indptr, d_indices, eps, d_embedding, tmp, n_epochs, (float)initial_alpha, (float)a, \
                               (float)b, (float)gamma, negative_sample_rate, sd);
  switch (dim) {
    SB2_UMAP_DIM(1) SB2_UMAP_DIM(2) SB2_UMAP_DIM(3) SB2_UMAP_DIM(4) SB2_UMAP_DIM(5) SB2_UMAP_DIM(6) SB2_UMAP_DIM(7) SB2_UMAP_DIM(8)
    SB2_UMAP_DIM(9) SB2_UMAP_DIM(10) SB2_UMAP_DIM(11) SB2_UMAP_DIM(12) SB2_UMAP_DIM(13) SB2_UMAP_DIM(14) SB2_UMAP_DIM(15)
    SB2_UMAP_DIM(16)
  }
#undef SB2_UMAP_DIM
  return SB2_E_BADARG;
}

}  // extern "C"

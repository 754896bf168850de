// combat.cu — the passes over X of
//   sc.pp.combat  (src/scanpy/preprocessing/_combat.py:71-289)
// that are not the design-matrix product DᵀX (that one is sb2_regress_col_sums).
//
// With the fitted coefficients, stand_mean[i, j] = grand[j] + sum_k cov[i, k] beta[k, j] (cov: the design's covariate
// columns, beta: their rows of b_hat) and r = x - stand_mean.  Every zero of a sparse X has an r too, so both passes walk
// the implicit dense matrix: one CTA per 256-gene slab, one thread per gene, CSR rows scattered into a zeroed
// shared-memory tile (slab.cuh).  All arithmetic is fp64.
//
// Moments: the count, mean and M2 (sum of squared deviations) of r over the rows of one batch.  One CTA per
// (SLAB_TILE-row subtile, slab) accumulates shifted sums (shift = the subtile's first r) and writes the subtile's (mean,
// M2); the subtiles are then merged into the caller's accumulators with Chan's formula in subtile order.  The caller
// passes one batch at a time in blocks that start on a subtile boundary of the batch, so results are bit-identical
// across runs and block sizes.  From these the host derives the pooled variance, gamma_hat, delta_hat and every sum of
// squares the empirical-Bayes iteration needs.
//
// Adjust: the dense corrected block ((s - gamma*_b) / sqrt(delta*_b)) * sqrt(vp) + stand_mean, s = r / sqrt(vp) (0 where
// vp == 0), in the reference's expression order, rounded once to float64; HBM-bound.
#include <math.h>

#include "common.cuh"
#include "slab.cuh"

namespace {

constexpr int CB_MAXP = 32;

// sum_k cov[k] * beta[k], then + grand: the order of `grand_mean + np.dot(tmp, b_hat)`
template <int KMAX>
__device__ __forceinline__ double stand_mean(const double* __restrict__ cr, const double (&bk)[KMAX], int p, double gm) {
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
    if (k < p) s += cr[k] * bk[k];
  return gm + s;
}

// grid (subtiles, slabs); part[sub][k][j]: k = 0 the subtile's mean r, 1 its M2.  Row k of the call is X row order[k]
// (order NULL: row k of the block); cov is indexed by the call's row.
template <typename T, bool CSR, int KMAX>
__global__ void __launch_bounds__(SLAB_THREADS, 1)
moments_kernel(int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
               const int32_t* __restrict__ indices, const T* __restrict__ data, const int64_t* __restrict__ order,
               const double* __restrict__ cov, int p, const double* __restrict__ grand,
               const double* __restrict__ beta, double* __restrict__ part) {
  __shared__ T tile[CSR ? SLAB_ROWS : 1][SLAB_THREADS];
  __shared__ int64_t rid[SLAB_ROWS], lo[SLAB_ROWS], hi[SLAB_ROWS];
  const int64_t sub = blockIdx.x;
  const int c0 = blockIdx.y * SLAB_THREADS, c = c0 + threadIdx.x;
  const int c1 = min(g, c0 + SLAB_THREADS);
  const int64_t s0 = sub * SLAB_TILE, s1 = min(rows, s0 + SLAB_TILE);
  double bk[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) bk[k] = (c < g && k < p) ? beta[(int64_t)k * g + c] : 0.0;
  const double gm = c < g ? grand[c] : 0.0;
  double shift = 0.0, a1 = 0.0, a2 = 0.0;
  if (CSR)
    for (int r = 0; r < SLAB_ROWS; ++r) tile[r][threadIdx.x] = T(0);
  for (int64_t b = s0; b < s1; b += SLAB_ROWS) {
    const int m = (int)min((int64_t)SLAB_ROWS, s1 - b);
    if ((int)threadIdx.x < m) rid[threadIdx.x] = order ? order[b + threadIdx.x] : b + threadIdx.x;
    if (CSR) stage_csr(indptr, indices, data, rid, m, c0, c1, tile, lo, hi);
    else __syncthreads();
    if (c < g) {
      for (int r = 0; r < m; ++r) {
        double v;
        if (CSR) {
          v = (double)tile[r][threadIdx.x];
          tile[r][threadIdx.x] = T(0);
        } else {
          v = (double)x[rid[r] * g + c];
        }
        const double d = v - stand_mean<KMAX>(cov + (b + r) * p, bk, p, gm);
        if (b == s0 && r == 0) shift = d;
        const double e = d - shift;
        a1 += e;
        a2 += e * e;
      }
    }
    __syncthreads();
  }
  if (c >= g) return;
  const double m = (double)(s1 - s0);
  double* out = part + sub * 2 * (int64_t)g;
  out[c] = shift + a1 / m;
  out[g + c] = a2 - a1 * a1 / m;
}

// grid (row tiles of SLAB_ROWS, slabs)
template <typename T, bool CSR, int KMAX>
__global__ void __launch_bounds__(SLAB_THREADS)
adjust_kernel(int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
              const int32_t* __restrict__ indices, const T* __restrict__ data, const int32_t* __restrict__ batch,
              const double* __restrict__ cov, int p, const double* __restrict__ grand, const double* __restrict__ beta,
              const double* __restrict__ sqrt_vp, const double* __restrict__ gamma, const double* __restrict__ dsq,
              double* __restrict__ out) {
  __shared__ T tile[CSR ? SLAB_ROWS : 1][SLAB_THREADS];
  __shared__ int64_t rid[SLAB_ROWS], lo[SLAB_ROWS], hi[SLAB_ROWS];
  const int64_t r0 = (int64_t)blockIdx.x * SLAB_ROWS;
  const int m = (int)min((int64_t)SLAB_ROWS, rows - r0);
  const int c0 = blockIdx.y * SLAB_THREADS, c = c0 + threadIdx.x;
  const int c1 = min(g, c0 + SLAB_THREADS);
  if (CSR) {
    for (int r = 0; r < SLAB_ROWS; ++r) tile[r][threadIdx.x] = T(0);
    if ((int)threadIdx.x < m) rid[threadIdx.x] = r0 + threadIdx.x;
    stage_csr(indptr, indices, data, rid, m, c0, c1, tile, lo, hi);
  }
  if (c >= g) return;
  double bk[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) bk[k] = k < p ? beta[(int64_t)k * g + c] : 0.0;
  const double gm = grand[c], sv = sqrt_vp[c];
  for (int r = 0; r < m; ++r) {
    const int64_t row = r0 + r;
    const double v = CSR ? (double)tile[r][threadIdx.x] : (double)x[row * g + c];
    const double sm = stand_mean<KMAX>(cov + row * p, bk, p, gm);
    const double s = sv == 0.0 ? 0.0 : (v - sm) / sv;
    const int64_t bj = (int64_t)batch[row] * g + c;
    out[row * g + c] = ((s - gamma[bj]) / dsq[bj]) * sv + sm;
  }
}

}  // namespace

extern "C" {

int32_t sb2_combat_moments(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                           const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                           const int64_t* d_order, const double* d_cov, int32_t p, const double* d_grand,
                           const double* d_beta, double* d_acc) {
  SB2_CHECK_ARG(ctx && d_grand && d_acc && g >= 1 && rows >= 0, "null pointer");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CHECK_ARG(p >= 0 && p <= CB_MAXP && (p == 0 || (d_cov && d_beta)), "covariates");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  const int64_t nsub = ceil_div64(rows, SLAB_TILE), slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(nsub < INT32_MAX && slabs <= 65535, "shape");
  ScratchScope scr(ctx);
  double* part;
  SB2_TRY(scr.alloc(&part, (size_t)(nsub * 2 * g)));
  const dim3 grid((unsigned)nsub, (unsigned)slabs);
  with_types(is_f64, d_x, [&](auto t, auto csr) {
    using T = decltype(t);
    with_kmax(p > 4, [&](auto kmax) {
      moments_kernel<T, decltype(csr)::value, kmax><<<grid, SLAB_THREADS, 0, ctx->stream>>>(
          rows, g, static_cast<const T*>(d_x), d_indptr, d_indices, static_cast<const T*>(d_data), d_order, d_cov, p,
          d_grand, d_beta, part);
    });
  });
  SB2_LAUNCH_CHECK(ctx);
  moments_fold_kernel<false><<<(unsigned)ceil_div64(g, 256), 256, 0, ctx->stream>>>(nsub, rows, g, part, d_acc);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_combat_adjust(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                          const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                          const int32_t* d_batch, const double* d_cov, int32_t p, const double* d_grand,
                          const double* d_beta, const double* d_sqrt_vp, const double* d_gamma, const double* d_dsq,
                          double* d_out) {
  SB2_CHECK_ARG(ctx && d_batch && d_grand && d_sqrt_vp && d_gamma && d_dsq && d_out && g >= 1 && rows >= 0,
                "null pointer");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CHECK_ARG(p >= 0 && p <= CB_MAXP && (p == 0 || (d_cov && d_beta)), "covariates");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  const int64_t tiles = ceil_div64(rows, SLAB_ROWS), slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(tiles < INT32_MAX && slabs <= 65535, "shape");
  const dim3 grid((unsigned)tiles, (unsigned)slabs);
  with_types(is_f64, d_x, [&](auto t, auto csr) {
    using T = decltype(t);
    with_kmax(p > 4, [&](auto kmax) {
      adjust_kernel<T, decltype(csr)::value, kmax><<<grid, SLAB_THREADS, 0, ctx->stream>>>(
          rows, g, static_cast<const T*>(d_x), d_indptr, d_indices, static_cast<const T*>(d_data), d_batch, d_cov, p,
          d_grand, d_beta, d_sqrt_vp, d_gamma, d_dsq, d_out);
    });
  });
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

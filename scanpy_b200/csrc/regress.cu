// regress.cu — the two passes over X of
//   sc.pp.regress_out  (src/scanpy/preprocessing/_simple.py:468-681)
//
// Pass 1 (column sums): for every gene j, acc[k, j] = sum_i W[i, k] x[i, j] (weighted: W = the regressors A for the
// numpy shortcut, or an orthonormal basis Q of range(A) for the GLM fallback), or acc[c, j] = sum of x[i, j] over the
// rows of group c (categorical), plus the per-gene min / max / NaN flag that decide `not (col != col[0]).any()`.
// One CTA owns a 256-column slab of a fixed SLAB_TILE-row subtile and each thread one column; it walks the subtile's rows
// in a fixed order (by group, then by row), so every partial is a sequential fp64 sum.  The subtiles' partials are
// then folded into the accumulators in subtile order.  Sums therefore do not depend on the launch shape or on how the
// caller splits the rows into blocks, as long as every block but the last is a multiple of SLAB_TILE rows: results are
// bit-identical across runs and chunk sizes.
//
// Pass 2 (residual): out[i, j] = x[i, j] - fit[i, j] computed in fp64 and rounded once to the output type, with
// fit = sum_k W[i, k] B[k, j] or b0[j] + b1[j] * means[code_i, j] (b0[j] for code -1); genes flagged in `pass` are
// copied.  Writes the dense row block; HBM-bound.
//
// A CSR input is read in place in both passes (slab.cuh: `stage_csr`), so implicit zeros enter the sums and the min /
// max as zeros.
#include <math.h>

#include "common.cuh"
#include "slab.cuh"

namespace {

constexpr int RG_MAXP = 32;

// grid (subtiles, slabs).  Weighted (w != NULL): part[sub][k][j], k < p.  Categorical: part[sub][group][j], the groups a
// subtile lacks stay as the caller zeroed them; `order` lists each subtile's rows sorted by (group, row).
template <typename T, bool CSR, int KMAX>
__global__ void __launch_bounds__(SLAB_THREADS)
col_sums_kernel(int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
                const int32_t* __restrict__ indices, const T* __restrict__ data, const double* __restrict__ w, int p,
                const int32_t* __restrict__ group, const int32_t* __restrict__ order, int n_groups,
                double* __restrict__ part, double* __restrict__ pmin, double* __restrict__ pmax, int32_t* __restrict__ pnan) {
  __shared__ T tile[CSR ? SLAB_ROWS : 1][SLAB_THREADS];
  __shared__ int64_t rid[SLAB_ROWS], lo[SLAB_ROWS], hi[SLAB_ROWS];
  const int64_t sub = blockIdx.x;
  const int c0 = blockIdx.y * SLAB_THREADS, c = c0 + threadIdx.x;
  const int c1 = min(g, c0 + SLAB_THREADS);
  const int64_t s0 = sub * SLAB_TILE, s1 = min(rows, s0 + SLAB_TILE);
  const int64_t width = (int64_t)(w ? p : n_groups) * g;
  double* out = part + sub * width;
  double acc[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) acc[k] = 0.0;
  double mn = INFINITY, mx = -INFINITY;
  int32_t nan = 0;
  int cur = -1;
  if (CSR)
    for (int r = 0; r < SLAB_ROWS; ++r) tile[r][threadIdx.x] = T(0);
  for (int64_t b = s0; b < s1; b += SLAB_ROWS) {
    const int m = (int)min((int64_t)SLAB_ROWS, s1 - b);
    if (CSR) {
      if ((int)threadIdx.x < m) rid[threadIdx.x] = order ? order[b + threadIdx.x] : b + threadIdx.x;
      stage_csr(indptr, indices, data, rid, m, c0, c1, tile, lo, hi);
    }
    for (int r = 0; r < m; ++r) {
      const int64_t row = CSR ? rid[r] : (order ? order[b + r] : b + r);
      double v = 0.0;
      if (c < g) {
        if (CSR) {
          v = (double)tile[r][threadIdx.x];
          tile[r][threadIdx.x] = T(0);
        } else {
          v = (double)x[row * g + c];
        }
      }
      if (w) {
        const double* wr = w + row * p;
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
          if (k < p) acc[k] += wr[k] * v;
      } else {
        const int grp = group[row];
        if (grp != cur) {
          if (cur >= 0 && c < g) out[(int64_t)cur * g + c] = acc[0];
          acc[0] = 0.0;
          cur = grp;
        }
        acc[0] += v;
      }
      nan |= v != v;
      mn = fmin(mn, v);
      mx = fmax(mx, v);
    }
    if (CSR) __syncthreads();
  }
  if (c >= g) return;
  if (w) {
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
      if (k < p) out[(int64_t)k * g + c] = acc[k];
  } else if (cur >= 0) {
    out[(int64_t)cur * g + c] = acc[0];
  }
  pmin[sub * g + c] = mn;
  pmax[sub * g + c] = mx;
  pnan[sub * g + c] = nan;
}

// grid (row tiles of SLAB_ROWS, slabs)
template <typename T, typename O, bool CSR, int KMAX>
__global__ void __launch_bounds__(SLAB_THREADS)
residual_kernel(int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
                const int32_t* __restrict__ indices, const T* __restrict__ data, const double* __restrict__ w, int p,
                const double* __restrict__ coef, const int32_t* __restrict__ code, const double* __restrict__ means,
                const double* __restrict__ b0, const double* __restrict__ b1, const uint8_t* __restrict__ pass,
                O* __restrict__ out) {
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
  double a0 = 0.0, a1 = 0.0;
  if (w) {
#pragma unroll
    for (int k = 0; k < KMAX; ++k) bk[k] = k < p ? coef[(int64_t)k * g + c] : 0.0;
  } else {
    a0 = b0[c];
    a1 = b1[c];
  }
  const bool copy = pass && pass[c];
  for (int r = 0; r < m; ++r) {
    const int64_t row = r0 + r;
    const double v = CSR ? (double)tile[r][threadIdx.x] : (double)x[row * g + c];
    double fit;
    if (w) {
      const double* wr = w + row * p;
      fit = 0.0;
#pragma unroll
      for (int k = 0; k < KMAX; ++k)
        if (k < p) fit += wr[k] * bk[k];
    } else {
      const int cc = code[row];
      fit = cc >= 0 ? a0 + a1 * means[(int64_t)cc * g + c] : a0;
    }
    out[row * g + c] = copy ? (O)v : (O)(v - fit);
  }
}

}  // namespace

extern "C" {

int32_t sb2_regress_col_sums(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                             const int64_t* d_indptr, const int32_t* d_indices, const void* d_data, const double* d_w,
                             int32_t p, const int32_t* d_group, const int32_t* d_order, int32_t n_groups, double* d_acc,
                             double* d_min, double* d_max, int32_t* d_nan) {
  SB2_CHECK_ARG(ctx && d_acc && d_min && d_max && d_nan && g >= 1 && rows >= 0, "null pointer");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CHECK_ARG(d_w ? (p >= 1 && p <= RG_MAXP) : (d_group && d_order && n_groups >= 1), "weights or groups");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  const int64_t nsub = ceil_div64(rows, SLAB_TILE), slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(nsub < INT32_MAX && slabs <= 65535, "shape");
  const int64_t width = (int64_t)(d_w ? p : n_groups) * g;
  ScratchScope scr(ctx);
  double *part, *pmin, *pmax;
  int32_t* pnan;
  SB2_TRY(scr.alloc(&part, (size_t)(nsub * width)));
  SB2_TRY(scr.alloc(&pmin, (size_t)(nsub * g)));
  SB2_TRY(scr.alloc(&pmax, (size_t)(nsub * g)));
  SB2_TRY(scr.alloc(&pnan, (size_t)(nsub * g)));
  if (!d_w) SB2_CUDA(cudaMemsetAsync(part, 0, sizeof(double) * (size_t)(nsub * width), ctx->stream));
  const dim3 grid((unsigned)nsub, (unsigned)slabs);
  const int32_t* order = d_w ? nullptr : d_order;
  const int32_t* group = d_w ? nullptr : d_group;
  with_types(is_f64, d_x, [&](auto t, auto csr) {
    using T = decltype(t);
    with_kmax(d_w && p > 4, [&](auto kmax) {
      col_sums_kernel<T, decltype(csr)::value, kmax><<<grid, SLAB_THREADS, 0, ctx->stream>>>(
          rows, g, static_cast<const T*>(d_x), d_indptr, d_indices, static_cast<const T*>(d_data), d_w, p, group, order,
          n_groups, part, pmin, pmax, pnan);
    });
  });
  SB2_LAUNCH_CHECK(ctx);
  const int64_t span = width > g ? width : g;
  fold_kernel<><<<(unsigned)ceil_div64(span, 256), 256, 0, ctx->stream>>>(nsub, width, g, part, pmin, pmax, pnan, d_acc,
                                                                         d_min, d_max, d_nan);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_regress_residual(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                             const int64_t* d_indptr, const int32_t* d_indices, const void* d_data, const double* d_w,
                             int32_t p, const double* d_coef, const int32_t* d_code, const double* d_means,
                             const double* d_b0, const double* d_b1, const uint8_t* d_pass, int32_t out_f64,
                             void* d_out) {
  SB2_CHECK_ARG(ctx && d_out && g >= 1 && rows >= 0, "null pointer");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CHECK_ARG(d_w ? (p >= 1 && p <= RG_MAXP && d_coef) : (d_code && d_means && d_b0 && d_b1), "fit");
  SB2_CHECK_ARG(is_f64 ? out_f64 : 1, "a float64 X needs a float64 output");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  const int64_t tiles = ceil_div64(rows, SLAB_ROWS), slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(tiles < INT32_MAX && slabs <= 65535, "shape");
  const dim3 grid((unsigned)tiles, (unsigned)slabs);
  with_types(is_f64, out_f64, d_x, [&](auto t, auto o, auto csr) {
    using T = decltype(t);
    using O = decltype(o);
    with_kmax(d_w && p > 4, [&](auto kmax) {
      residual_kernel<T, O, decltype(csr)::value, kmax><<<grid, SLAB_THREADS, 0, ctx->stream>>>(
          rows, g, static_cast<const T*>(d_x), d_indptr, d_indices, static_cast<const T*>(d_data), d_w, p, d_coef, d_code,
          d_means, d_b0, d_b1, d_pass, static_cast<O*>(d_out));
    });
  });
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

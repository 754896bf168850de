// pearson.cu — the passes over X of analytic Pearson residuals (Lause et al. 2021):
//   sc.experimental.pp.highly_variable_genes(flavor="pearson_residuals")
//       (src/scanpy/experimental/pp/_highly_variable_genes.py:35-126,129-287)
//   sc.experimental.pp.normalize_pearson_residuals  (src/scanpy/experimental/pp/_normalization.py:36-75)
//
// The residual of count x[i, j] is r = clip((x - mu) / sqrt(mu + mu^2 / theta)), mu = s_i s_j / S, with the cell total
// s_i, the gene total s_j and the grand total S; theta = inf gives mu^2 / theta = 0.  Every zero of a sparse X has a
// residual too, so both passes walk the implicit dense matrix: one CTA per 256-gene slab, one thread per gene, CSR rows
// scattered into a zeroed shared-memory tile (slab.cuh).  All arithmetic is fp64.
//
// Row totals: one warp per row, a fixed-order lane-strided sum and a butterfly reduction.
//
// Residual variance: the population variance of r over the rows of one batch.  One CTA per (PR_TILE-row subtile,
// slab) accumulates shifted sums (shift = the subtile's first residual) and writes the subtile's (mean, M2); the
// per-gene Σx² rides along.  The subtiles are then merged into the caller's accumulators with Chan's formula in subtile
// order.  The caller passes one batch at a time in blocks that start on a subtile boundary of the batch, so results
// are bit-identical across runs and block sizes.
//
// Residuals: the dense row block, each value in fp64 rounded once to the output type; HBM-bound.
//
// The clip is written with comparisons, as np.clip and numba's min(max(r, -c), c) are: a NaN residual (a zero-total
// cell or gene: 0 / 0) stays NaN, where fmin / fmax would return the bound.
#include <math.h>

#include "common.cuh"
#include "slab.cuh"

namespace {

constexpr int PR_TILE = SB2_PEARSON_TILE_ROWS;
static_assert(PR_TILE % SLAB_ROWS == 0, "subtile");

__device__ __forceinline__ double pearson_residual(double v, double sg, double sc, double total, double clip,
                                                   double theta) {
  const double mu = sg * sc / total;
  const double r = (v - mu) / sqrt(mu + mu * mu / theta);
  const double lo = r < -clip ? -clip : r;
  return lo > clip ? clip : lo;
}

// one warp per row
template <typename T, bool CSR>
__global__ void __launch_bounds__(256)
row_sums_kernel(int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
                const T* __restrict__ data, double* __restrict__ out) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  double s = 0.0;
  if (CSR) {
    for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32) s += (double)data[e];
  } else {
    const T* xr = x + row * g;
    for (int c = lane; c < g; c += 32) s += (double)xr[c];
  }
  s = warp_sum(s);
  if (lane == 0) out[row] = s;
}

// grid (subtiles, slabs); part[sub][k][j]: k = 0 the subtile's mean residual, 1 its M2, 2 its Σx²
template <typename T, bool CSR>
__global__ void __launch_bounds__(SLAB_THREADS, 4)
resvar_kernel(int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
              const int32_t* __restrict__ indices, const T* __restrict__ data, const int64_t* __restrict__ order,
              const double* __restrict__ gene, const double* __restrict__ cell, double total, double clip, double theta,
              double* __restrict__ part) {
  __shared__ T tile[CSR ? SLAB_ROWS : 1][SLAB_THREADS];
  __shared__ int64_t rid[SLAB_ROWS], lo[SLAB_ROWS], hi[SLAB_ROWS];
  __shared__ double sc[SLAB_ROWS];
  const int64_t sub = blockIdx.x;
  const int c0 = blockIdx.y * SLAB_THREADS, c = c0 + threadIdx.x;
  const int c1 = min(g, c0 + SLAB_THREADS);
  const int64_t s0 = sub * PR_TILE, s1 = min(rows, s0 + PR_TILE);
  const double sg = c < g ? gene[c] : 0.0;
  double shift = 0.0, a1 = 0.0, a2 = 0.0, sq = 0.0;
  if (CSR)
    for (int r = 0; r < SLAB_ROWS; ++r) tile[r][threadIdx.x] = T(0);
  for (int64_t b = s0; b < s1; b += SLAB_ROWS) {
    const int m = (int)min((int64_t)SLAB_ROWS, s1 - b);
    if ((int)threadIdx.x < m) {
      rid[threadIdx.x] = order ? order[b + threadIdx.x] : b + threadIdx.x;
      sc[threadIdx.x] = cell[b + threadIdx.x];
    }
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
        const double res = pearson_residual(v, sg, sc[r], total, clip, theta);
        if (b == s0 && r == 0) shift = res;
        const double d = res - shift;
        a1 += d;
        a2 += d * d;
        sq += v * v;
      }
    }
    __syncthreads();
  }
  if (c >= g) return;
  const double m = (double)(s1 - s0);
  double* out = part + sub * 3 * (int64_t)g;
  out[c] = shift + a1 / m;
  out[g + c] = a2 - a1 * a1 / m;
  out[2 * (int64_t)g + c] = sq;
}

// acc[k][j] (k = 0 count, 1 mean, 2 M2, 3 Σx²) merged with the subtiles' partials in subtile order (Chan et al.)
__global__ void resvar_fold_kernel(int64_t nsub, int64_t rows, int g, const double* __restrict__ part,
                                   double* __restrict__ acc) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g) return;
  double n = acc[j], mean = acc[g + j], m2 = acc[2 * (int64_t)g + j], sq = acc[3 * (int64_t)g + j];
  for (int64_t t = 0; t < nsub; ++t) {
    const double* p = part + t * 3 * (int64_t)g;
    const double nb = (double)min((int64_t)PR_TILE, rows - t * PR_TILE);
    const double mb = p[j], m2b = p[g + j];
    if (n == 0.0) {
      mean = mb;
      m2 = m2b;
    } else {
      const double nn = n + nb, d = mb - mean;
      mean += d * (nb / nn);
      m2 += m2b + d * d * (n * nb / nn);
    }
    n += nb;
    sq += p[2 * (int64_t)g + j];
  }
  acc[j] = n;
  acc[g + j] = mean;
  acc[2 * (int64_t)g + j] = m2;
  acc[3 * (int64_t)g + j] = sq;
}

// grid (row tiles of SLAB_ROWS, slabs)
template <typename T, typename O, bool CSR>
__global__ void __launch_bounds__(SLAB_THREADS, 4)
residual_kernel(int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
                const int32_t* __restrict__ indices, const T* __restrict__ data, const double* __restrict__ gene,
                const double* __restrict__ cell, double total, double clip, double theta, O* __restrict__ out) {
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
  const double sg = gene[c];
  for (int r = 0; r < m; ++r) {
    const int64_t row = r0 + r;
    const double v = CSR ? (double)tile[r][threadIdx.x] : (double)x[row * g + c];
    out[row * g + c] = (O)pearson_residual(v, sg, cell[row], total, clip, theta);
  }
}

template <typename T>
void launch_row_sums(sb2_ctx* ctx, int64_t rows, int g, const void* x, const int64_t* indptr, const void* data,
                     double* out) {
  const unsigned blocks = (unsigned)ceil_div64(rows * 32, 256);
  if (x) row_sums_kernel<T, false><<<blocks, 256, 0, ctx->stream>>>(rows, g, static_cast<const T*>(x), nullptr,
                                                                     nullptr, out);
  else row_sums_kernel<T, true><<<blocks, 256, 0, ctx->stream>>>(rows, g, nullptr, indptr,
                                                                  static_cast<const T*>(data), out);
}

template <typename T, bool CSR>
void launch_resvar(sb2_ctx* ctx, dim3 grid, int64_t rows, int g, const void* x, const int64_t* indptr,
                   const int32_t* indices, const void* data, const int64_t* order, const double* gene,
                   const double* cell, double total, double clip, double theta, double* part) {
  resvar_kernel<T, CSR><<<grid, SLAB_THREADS, 0, ctx->stream>>>(rows, g, static_cast<const T*>(x), indptr, indices,
                                                                 static_cast<const T*>(data), order, gene, cell, total,
                                                                 clip, theta, part);
}

template <typename T, typename O, bool CSR>
void launch_residual(sb2_ctx* ctx, dim3 grid, int64_t rows, int g, const void* x, const int64_t* indptr,
                     const int32_t* indices, const void* data, const double* gene, const double* cell, double total,
                     double clip, double theta, void* out) {
  residual_kernel<T, O, CSR><<<grid, SLAB_THREADS, 0, ctx->stream>>>(rows, g, static_cast<const T*>(x), indptr,
                                                                      indices, static_cast<const T*>(data), gene, cell,
                                                                      total, clip, theta, static_cast<O*>(out));
}

}  // namespace

extern "C" {

int32_t sb2_pearson_row_sums(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                             const int64_t* d_indptr, const void* d_data, double* d_out) {
  SB2_CHECK_ARG(ctx && d_out && g >= 1 && rows >= 0, "null pointer");
  SB2_CHECK_ARG(d_x || (d_indptr && d_data), "X: dense block or CSR arrays");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  SB2_CHECK_ARG(ceil_div64(rows * 32, 256) < INT32_MAX, "shape");
  if (is_f64) launch_row_sums<double>(ctx, rows, g, d_x, d_indptr, d_data, d_out);
  else launch_row_sums<float>(ctx, rows, g, d_x, d_indptr, d_data, d_out);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_pearson_residual_var(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                                 const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                                 const int64_t* d_order, const double* d_gene, const double* d_cell, double total,
                                 double clip, double theta, double* d_acc) {
  SB2_CHECK_ARG(ctx && d_gene && d_cell && d_acc && g >= 1 && rows >= 0, "null pointer");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CHECK_ARG(theta > 0 && clip >= 0, "theta > 0, clip >= 0");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  const int64_t nsub = ceil_div64(rows, PR_TILE), slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(nsub < INT32_MAX && slabs <= 65535, "shape");
  ScratchScope scr(ctx);
  double* part;
  SB2_TRY(scr.alloc(&part, (size_t)(nsub * 3 * g)));
  const dim3 grid((unsigned)nsub, (unsigned)slabs);
  if (d_x) {
    if (is_f64) launch_resvar<double, false>(ctx, grid, rows, g, d_x, nullptr, nullptr, nullptr, d_order, d_gene, d_cell,
                                             total, clip, theta, part);
    else launch_resvar<float, false>(ctx, grid, rows, g, d_x, nullptr, nullptr, nullptr, d_order, d_gene, d_cell, total,
                                     clip, theta, part);
  } else {
    if (is_f64) launch_resvar<double, true>(ctx, grid, rows, g, nullptr, d_indptr, d_indices, d_data, d_order, d_gene,
                                            d_cell, total, clip, theta, part);
    else launch_resvar<float, true>(ctx, grid, rows, g, nullptr, d_indptr, d_indices, d_data, d_order, d_gene, d_cell,
                                    total, clip, theta, part);
  }
  SB2_LAUNCH_CHECK(ctx);
  resvar_fold_kernel<<<(unsigned)ceil_div64(g, 256), 256, 0, ctx->stream>>>(nsub, rows, g, part, d_acc);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_pearson_residuals(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                              const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                              const double* d_gene, const double* d_cell, double total, double clip, double theta,
                              int32_t out_f64, void* d_out) {
  SB2_CHECK_ARG(ctx && d_gene && d_cell && d_out && g >= 1 && rows >= 0, "null pointer");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CHECK_ARG(theta > 0 && clip >= 0, "theta > 0, clip >= 0");
  SB2_CHECK_ARG(is_f64 ? out_f64 : 1, "a float64 X needs a float64 output");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  const int64_t tiles = ceil_div64(rows, SLAB_ROWS), slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(tiles < INT32_MAX && slabs <= 65535, "shape");
  const dim3 grid((unsigned)tiles, (unsigned)slabs);
  const bool csr = d_x == nullptr;
#define SB2_PEARSON(T, O, C)                                                                                  \
  launch_residual<T, O, C>(ctx, grid, rows, g, d_x, d_indptr, d_indices, d_data, d_gene, d_cell, total, clip, \
                           theta, d_out)
  if (is_f64) {
    if (csr) SB2_PEARSON(double, double, true); else SB2_PEARSON(double, double, false);
  } else if (out_f64) {
    if (csr) SB2_PEARSON(float, double, true); else SB2_PEARSON(float, double, false);
  } else {
    if (csr) SB2_PEARSON(float, float, true); else SB2_PEARSON(float, float, false);
  }
#undef SB2_PEARSON
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

// preprocess.cu — the CSR passes in front of the hot path (SURVEY.md 8f row f2), kept on the device:
//   sc.pp.normalize_total  (src/scanpy/preprocessing/_normalization.py:29-66 numba `_normalize_csr`, :69-125, :127-306)
//   sc.pp.log1p            (src/scanpy/preprocessing/_simple.py:310-425)
//   per-gene mean/variance of expm1(X) for sc.pp.highly_variable_genes(flavor='seurat')
//                          (src/scanpy/preprocessing/_highly_variable_genes.py:300-385)
// All of them are single-pass streaming kernels over the CSR arrays: HBM-bound, 4..8 bytes per non-zero.
#include <math.h>

#include "common.cuh"

namespace {

// counts_per_cell[i] = sum_j data[j]  (accumulated in fp64 like numba's `count = 0.0`, stored as float32);
// with `skip_cols` given, entries whose column is flagged (counts_per_cols[col] != 0) are left out
__global__ void __launch_bounds__(256)
row_sums_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                const float* __restrict__ data, const int32_t* __restrict__ skip_cols, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  double s = 0.0;
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32)
    if (!skip_cols || skip_cols[indices[e]] == 0) s += (double)data[e];
  s = warp_sum(s);
  if (lane == 0) out[row] = (float)s;
}
// counts_per_cols[c] += 1 for every entry with data > max_fraction * counts_per_cell[row]
__global__ void __launch_bounds__(256)
hiexpr_count_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                    const float* __restrict__ data, const float* __restrict__ row_sums, double max_fraction,
                    int32_t* __restrict__ counts_per_col) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const double thr = max_fraction * (double)row_sums[row];
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32)
    if ((double)data[e] > thr) atomicAdd(&counts_per_col[indices[e]], 1);
}
// data[j] /= scale[row]   (scale == 0 -> divide by 1: `allow_divide_by_zero=False`, _utils/__init__.py:638-639)
__global__ void __launch_bounds__(256)
scale_rows_kernel(int64_t n, const int64_t* __restrict__ indptr, float* __restrict__ data, const float* __restrict__ scale) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  float s = scale[row];
  if (s == 0.0f) s = 1.0f;
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32) data[e] = data[e] / s;
}
__global__ void log1p_kernel(int64_t nnz, float* __restrict__ data, double log_base) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nnz) return;
  float v = log1pf(data[i]);
  if (log_base != 0.0) v = (float)((double)v / log_base);  // np.divide(x, np.log(base)) (_simple.py:359-380)
  data[i] = v;
}
// per-gene sum and sum of squares of f(x), f = expm1(x * log_scale) (EXPM1) or identity; fp64 REDs into replicated copies.
// The product is taken in fp64 and rounded once to float32, as the reference's `x *= np.log(base)` on float32 data does
// (a float32 multiply by the rounded log_scale is 1 ulp off for a few percent of x, which expm1 amplifies by ~x·ln b)
constexpr int MV_COPIES = 32;
template <bool EXPM1>
__global__ void col_sums_transformed_kernel(int64_t nnz, const int32_t* __restrict__ indices, const float* __restrict__ data,
                                            int g, double* __restrict__ acc, double log_scale) {
  double* mine = acc + (size_t)(blockIdx.x % MV_COPIES) * 2 * g;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    float x = data[i];
    if (EXPM1) {
      if (log_scale != 1.0) x = (float)((double)x * log_scale);
      x = expm1f(x);
    }
    const double v = (double)x;
    atomicAdd(&mine[indices[i]], v);
    atomicAdd(&mine[g + indices[i]], v * v);
  }
}
__global__ void reduce_copies_kernel(const double* __restrict__ src, int copies, int64_t len, double* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= len) return;
  double s = 0.0;
  for (int c = 0; c < copies; ++c) s += src[(size_t)c * len + i];
  dst[i] = s;
}


// ---- sc.pp.scale (src/scanpy/preprocessing/_scale.py:150-296) ---------------------------------------------------------
// per-gene sum / sum of squares over the rows with mask != 0 (mask == nullptr: all rows): warp per row, fp64 REDs into
// MV_COPIES replicated accumulators (mean_var(x[mask_obs, :], axis=0, correction=1) without materialising the subset)
__global__ void __launch_bounds__(256)
col_stats_rows_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                      const float* __restrict__ data, const uint8_t* __restrict__ mask, int g, double* __restrict__ acc) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n || (mask && !mask[row])) return;
  double* mine = acc + (size_t)(blockIdx.x % MV_COPIES) * 2 * g;
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32) {
    const double v = (double)data[e];
    atomicAdd(&mine[indices[e]], v);
    atomicAdd(&mine[g + indices[e]], v * v);
  }
}
// numba `scale_and_clip_csr` (_scale.py:267-283): data[j] = min(max_value, data[j] / std[col]) on the masked rows
__global__ void __launch_bounds__(256)
scale_cols_csr_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                      float* __restrict__ data, const double* __restrict__ stdv, const uint8_t* __restrict__ mask,
                      int has_max, double max_value) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n || (mask && !mask[row])) return;
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32) {
    double v = (double)data[e] / stdv[indices[e]];
    if (has_max) v = fmin(max_value, v);
    data[e] = (float)v;
  }
}
// zero_center=True on a CSR densifies it (`x -= mean` -> float64 dense, then / std, then clip to [-max, max]): CTA per
// row writes the row's background (0 - mean)/std and then the stored entries; the dense row is written once (the
// background pass skips nothing - a second write of ~5 % of the columns is cheaper than a per-column search)
__device__ __forceinline__ double clip_sym(double v, int has_max, double mx) {
  if (has_max) { if (v > mx) v = mx; else if (v < -mx) v = -mx; }
  return v;
}
__global__ void __launch_bounds__(256)
scale_csr_to_dense_kernel(int64_t n, int g, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                          const float* __restrict__ data, const double* __restrict__ mean, const double* __restrict__ stdv,
                          const uint8_t* __restrict__ mask, int has_max, double max_value, double* __restrict__ out) {
  const int64_t row = blockIdx.x;
  double* o = out + (size_t)row * g;
  const bool on = !mask || mask[row];   // rows outside mask_obs keep their values (`x[mask_obs, :] = scaled`)
  for (int c = threadIdx.x; c < g; c += blockDim.x) o[c] = on ? clip_sym((0.0 - mean[c]) / stdv[c], has_max, max_value) : 0.0;
  __syncthreads();
  for (int64_t e = indptr[row] + threadIdx.x; e < indptr[row + 1]; e += blockDim.x) {
    const int c = indices[e];
    o[c] = on ? clip_sym(((double)data[e] - mean[c]) / stdv[c], has_max, max_value) : (double)data[e];
  }
}
// dense input: column sums over the masked rows; a CTA owns DS_ROWS rows, thread t the columns t, t+256, ...
constexpr int DS_ROWS = 64;
template <typename T>
__global__ void __launch_bounds__(256)
dense_col_stats_kernel(int64_t n, int g, const T* __restrict__ x, const uint8_t* __restrict__ mask, double* __restrict__ acc) {
  const int64_t r0 = (int64_t)blockIdx.x * DS_ROWS;
  const int64_t r1 = r0 + DS_ROWS < n ? r0 + DS_ROWS : n;
  double* mine = acc + (size_t)(blockIdx.x % MV_COPIES) * 2 * g;
  for (int c = threadIdx.x; c < g; c += blockDim.x) {
    double s = 0.0, q = 0.0;
    for (int64_t r = r0; r < r1; ++r) {
      if (mask && !mask[r]) continue;
      const double v = (double)x[(size_t)r * g + c];
      s += v;
      q += v * v;
    }
    atomicAdd(&mine[c], s);
    atomicAdd(&mine[g + c], q);
  }
}
// dense input, in place: `x -= mean` (rounded to T), `x /= std` (rounded to T), clip_array (_scale.py:52-69): the lower
// bound only applies with zero_center
template <typename T>
__global__ void dense_scale_kernel(int64_t n, int g, T* __restrict__ x, const double* __restrict__ mean,
                                   const double* __restrict__ stdv, const uint8_t* __restrict__ mask, int has_max, double max_value) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * g) return;
  const int64_t r = i / g;
  const int c = (int)(i - r * g);
  if (mask && !mask[r]) return;
  T v = x[i];
  if (mean) v = (T)((double)v - mean[c]);
  v = (T)((double)v / stdv[c]);
  if (has_max) {
    const T mx = (T)max_value;
    if (v > mx) v = mx; else if (mean && v < -mx) v = -mx;
  }
  x[i] = v;
}

inline unsigned gridw(int64_t n) { return (unsigned)ceil_div64(n, 8); }

// zeroed [MV_COPIES][2][g] accumulators for the column-stats kernels, and the [2][g] buffer finish_col_stats sums them into
int32_t alloc_col_stats(sb2_ctx* ctx, ScratchScope& scr, int32_t g, double** acc, double** both) {
  SB2_TRY(scr.alloc(acc, (size_t)MV_COPIES * 2 * g));
  SB2_TRY(scr.alloc(both, (size_t)2 * g));
  SB2_CUDA(cudaMemsetAsync(*acc, 0, sizeof(double) * MV_COPIES * 2 * g, ctx->stream));
  return SB2_OK;
}
int32_t finish_col_stats(sb2_ctx* ctx, const double* acc, double* both, int32_t g, double* d_sum, double* d_sumsq) {
  reduce_copies_kernel<<<(unsigned)ceil_div64(2 * g, 256), 256, 0, ctx->stream>>>(acc, MV_COPIES, 2 * (int64_t)g, both);
  SB2_LAUNCH_CHECK(ctx);
  SB2_CUDA(cudaMemcpyAsync(d_sum, both, sizeof(double) * g, cudaMemcpyDeviceToDevice, ctx->stream));
  SB2_CUDA(cudaMemcpyAsync(d_sumsq, both + g, sizeof(double) * g, cudaMemcpyDeviceToDevice, ctx->stream));
  return SB2_OK;
}

}  // namespace

extern "C" {

int32_t sb2_csr_row_sums_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                             const float* d_data, const int32_t* d_skip_cols, float* d_out) {
  SB2_CHECK_ARG(ctx && d_indptr && d_out, "null pointer");
  SB2_CHECK_ARG(!d_skip_cols || d_indices, "indices needed with skip_cols");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  row_sums_kernel<<<gridw(n), 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_data, d_skip_cols, d_out);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_csr_hiexpr_count_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                                 const float* d_data, const float* d_row_sums, double max_fraction,
                                 int32_t* d_counts_per_col) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_row_sums && d_counts_per_col, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  SB2_CUDA(cudaMemsetAsync(d_counts_per_col, 0, sizeof(int32_t) * (size_t)g, ctx->stream));
  if (n == 0) return SB2_OK;
  hiexpr_count_kernel<<<gridw(n), 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_data, d_row_sums, max_fraction,
                                                        d_counts_per_col);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_csr_scale_rows_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, float* d_data, const float* d_scale) {
  SB2_CHECK_ARG(ctx && d_indptr && d_scale, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  scale_rows_kernel<<<gridw(n), 256, 0, ctx->stream>>>(n, d_indptr, d_data, d_scale);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_log1p_f32(sb2_ctx* ctx, int64_t nnz, float* d_data, double base) {
  SB2_CHECK_ARG(ctx && (d_data || nnz == 0), "null pointer");
  SB2_CHECK_ARG(base == 0.0 || (base > 0.0 && base != 1.0), "base");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (nnz == 0) return SB2_OK;
  log1p_kernel<<<(unsigned)ceil_div64(nnz, 256), 256, 0, ctx->stream>>>(nnz, d_data, base == 0.0 ? 0.0 : log(base));
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_csr_col_sums_f32(sb2_ctx* ctx, int64_t nnz, int32_t g, const int32_t* d_indices, const float* d_data,
                             int32_t apply_expm1, double log_scale, double* d_sum, double* d_sumsq) {
  SB2_CHECK_ARG(ctx && d_sum && d_sumsq && g >= 1, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  double *acc, *both;
  SB2_TRY(alloc_col_stats(ctx, scr, g, &acc, &both));
  if (nnz > 0) {
    const unsigned grid = ctx->prop.multiProcessorCount * 8;
    if (apply_expm1)
      col_sums_transformed_kernel<true><<<grid, 256, 0, ctx->stream>>>(nnz, d_indices, d_data, g, acc, log_scale);
    else
      col_sums_transformed_kernel<false><<<grid, 256, 0, ctx->stream>>>(nnz, d_indices, d_data, g, acc, log_scale);
    SB2_LAUNCH_CHECK(ctx);
  }
  return finish_col_stats(ctx, acc, both, g, d_sum, d_sumsq);
}

int32_t sb2_csr_col_stats_rows_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                                   const float* d_data, const uint8_t* d_mask, double* d_sum, double* d_sumsq) {
  SB2_CHECK_ARG(ctx && d_indptr && d_sum && d_sumsq && g >= 1, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  double *acc, *both;
  SB2_TRY(alloc_col_stats(ctx, scr, g, &acc, &both));
  if (n > 0) {
    col_stats_rows_kernel<<<gridw(n), 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_data, d_mask, g, acc);
    SB2_LAUNCH_CHECK(ctx);
  }
  return finish_col_stats(ctx, acc, both, g, d_sum, d_sumsq);
}

int32_t sb2_csr_scale_cols_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices, float* d_data,
                               const double* d_std, const uint8_t* d_mask, int32_t has_max, double max_value) {
  SB2_CHECK_ARG(ctx && d_indptr && d_std, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  scale_cols_csr_kernel<<<gridw(n), 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_data, d_std, d_mask, has_max, max_value);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_csr_scale_dense_f64(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                                const float* d_data, const double* d_mean, const double* d_std, const uint8_t* d_mask,
                                int32_t has_max, double max_value, double* d_out) {
  SB2_CHECK_ARG(ctx && d_indptr && d_mean && d_std && d_out && g >= 1, "null pointer");
  SB2_CHECK_ARG(n < INT32_MAX, "n");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  scale_csr_to_dense_kernel<<<(unsigned)n, 256, 0, ctx->stream>>>(n, g, d_indptr, d_indices, d_data, d_mean, d_std, d_mask,
                                                                 has_max, max_value, d_out);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_dense_col_stats(sb2_ctx* ctx, int64_t n, int32_t g, const void* d_x, int32_t is_f64, const uint8_t* d_mask,
                            double* d_sum, double* d_sumsq) {
  SB2_CHECK_ARG(ctx && d_x && d_sum && d_sumsq && g >= 1, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  double *acc, *both;
  SB2_TRY(alloc_col_stats(ctx, scr, g, &acc, &both));
  if (n > 0) {
    const unsigned grid = (unsigned)ceil_div64(n, DS_ROWS);
    if (is_f64) dense_col_stats_kernel<double><<<grid, 256, 0, ctx->stream>>>(n, g, (const double*)d_x, d_mask, acc);
    else dense_col_stats_kernel<float><<<grid, 256, 0, ctx->stream>>>(n, g, (const float*)d_x, d_mask, acc);
    SB2_LAUNCH_CHECK(ctx);
  }
  return finish_col_stats(ctx, acc, both, g, d_sum, d_sumsq);
}

int32_t sb2_dense_scale(sb2_ctx* ctx, int64_t n, int32_t g, void* d_x, int32_t is_f64, const double* d_mean,
                        const double* d_std, const uint8_t* d_mask, int32_t has_max, double max_value) {
  SB2_CHECK_ARG(ctx && d_x && d_std && g >= 1, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  const unsigned grid = (unsigned)ceil_div64(n * g, 256);
  if (is_f64) dense_scale_kernel<double><<<grid, 256, 0, ctx->stream>>>(n, g, (double*)d_x, d_mean, d_std, d_mask, has_max, max_value);
  else dense_scale_kernel<float><<<grid, 256, 0, ctx->stream>>>(n, g, (float*)d_x, d_mean, d_std, d_mask, has_max, max_value);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

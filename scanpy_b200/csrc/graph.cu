// graph.cu — UMAP fuzzy simplicial set -> symmetric connectivities CSR (sm_90a).
//
// Replaces umap.umap_.fuzzy_simplicial_set(...).tocsr() as called by the reference at
// src/scanpy/neighbors/_connectivity.py:124-138 (arithmetic spec: SURVEY.md Appendix A2;
// umap-learn's smooth_knn_dist / compute_membership_strengths / fuzzy union).
//
//   fuzzy_rows_kernel     thread per cell: rho = first non-zero distance, 64-step sigma bisection
//                         (fp64 scalars like umap's numba code, fp32 storage), fp32 membership
//                         strengths.  Pure streaming: 12*n*k B in, 4*n*k B out.
//   sym_count_kernel      thread per directed edge (i -> j): looks i up in j's k-list (k <= 32
//                         entries, L2 hits), forms c = mix*(a+b-ab) + (1-mix)*ab, counts row
//                         lengths of the union pattern; edges whose reverse is absent from j's
//                         list also count towards row j ("in-only").
//   (prefix sum)          row pointers (util.cu)
//   sym_fill_kernel       scatters values: out-edges in list order, in-only edges via a per-row
//                         atomic cursor
//   sym_sort_rows_kernel  warp per row: sorts each row by column (bitonic in registers for
//                         <= 32 entries, rank sort for hubs) -> deterministic CSR, no explicit zeros
// No global sort and no COO materialisation: the transpose-merge R + R^T - R*R^T of the reference
// is resolved with the k-list lookup because every stored entry of R^T is a k-list entry.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int MAXK = 64;   // k-lists up to 64 entries (the kNN kernel serves k <= 56); kernels are instantiated for 32 and 64

__global__ void sum_f32cast_kernel(const double* __restrict__ x, int64_t n, double* __restrict__ out) {
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s += (double)(float)x[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, s);
}

template <int MK>   // MK >= k: length of the thread's register-resident k-list
__global__ void __launch_bounds__(128)
fuzzy_rows_kernel(int64_t n, int k, const int32_t* __restrict__ knn_idx, const double* __restrict__ knn_dist,
                  float local_connectivity, const double* __restrict__ dist_sum, float* __restrict__ w_out,
                  float* __restrict__ sigmas, float* __restrict__ rhos) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float d[MK];
  double row_sum = 0.0;
#pragma unroll
  for (int j = 0; j < MK; ++j) {
    d[j] = j < k ? (float)knn_dist[i * k + j] : 0.0f;
    if (j < k) row_sum += (double)d[j];
  }
  // rho (umap_.py smooth_knn_dist: the non_zero_dists block)
  const int index = (int)floorf(local_connectivity);
  const float interpolation = local_connectivity - (float)index;
  int nnz = 0;
  float nz_im1 = 0.0f, nz_i = 0.0f, nz_0 = 0.0f, nz_max = 0.0f;
#pragma unroll
  for (int j = 0; j < MK; ++j) {
    if (j < k && d[j] > 0.0f) {
      if (nnz == 0) nz_0 = d[j];
      if (nnz == index - 1) nz_im1 = d[j];
      if (nnz == index) nz_i = d[j];
      nz_max = fmaxf(nz_max, d[j]);
      ++nnz;
    }
  }
  float rho = 0.0f;
  if ((float)nnz >= local_connectivity) {
    if (index > 0) {
      rho = nz_im1;
      if (interpolation > 1e-5f) rho += interpolation * (nz_i - nz_im1);
    } else {
      rho = interpolation * nz_0;
    }
  } else if (nnz > 0) {
    rho = nz_max;
  }
  // sigma: bisection so that sum_j exp(-(d_j - rho)/sigma) = log2(k)
  const double target = log2((double)k);
  double lo = 0.0, hi = INFINITY, mid = 1.0;
  for (int it = 0; it < 64; ++it) {
    double psum = 0.0;
#pragma unroll
    for (int j = 1; j < MK; ++j) {
      if (j < k) {
        const float dd = d[j] - rho;
        psum += dd > 0.0f ? exp(-((double)dd / mid)) : 1.0;
      }
    }
    if (fabs(psum - target) < 1e-5) break;
    if (psum > target) {
      hi = mid;
      mid = (lo + hi) / 2.0;
    } else {
      lo = mid;
      if (isinf(hi)) mid *= 2.0;
      else mid = (lo + hi) / 2.0;
    }
  }
  float sigma = (float)mid;
  {
    const double mean_ith = row_sum / (double)k;
    const double mean_all = *dist_sum / ((double)n * (double)k);
    const double fl = 1e-3 * (rho > 0.0f ? mean_ith : mean_all);
    if ((double)sigma < fl) sigma = (float)fl;
  }
  sigmas[i] = sigma;
  rhos[i] = rho;
  // membership strengths (compute_membership_strengths), float32
#pragma unroll
  for (int j = 0; j < MK; ++j) {
    if (j < k) {
      const int32_t nb = knn_idx[i * k + j];
      float val;
      if (nb < 0) val = 0.0f;
      else if (nb == (int32_t)i) val = 0.0f;
      else if (d[j] - rho <= 0.0f || sigma == 0.0f) val = 1.0f;
      else val = expf(-((d[j] - rho) / sigma));
      w_out[i * k + j] = val;
    }
  }
}

// how the directed weight a = W[i,j] and its reverse b = W[j,i] (0 if absent) combine into C[i,j] = C[j,i]
enum SymOp { SYM_FUZZY_UNION = 0, SYM_AVERAGE = 1, SYM_COPY_MISSING = 2 };
template <typename T>
__device__ __forceinline__ T sym_combine(T a, T b, int op, T mix) {
  if (op == SYM_AVERAGE) return (a + b) / (T)2;         // jaccard: (J + J^T) / 2   (_connectivity.py:183-184)
  if (op == SYM_COPY_MISSING) return a != (T)0 ? a : b;  // gauss: w[j,i] = w[i,j] where missing (:93-97)
  const T p = a * b;                                     // umap: mix (a + b - ab) + (1 - mix) ab
  return mix * (a + b - p) + ((T)1 - mix) * p;
}

// one thread per (i, m): value of C[i, idx[i][m]] and in-only bookkeeping
template <typename T>
__global__ void sym_count_kernel(int64_t n, int k, const int32_t* __restrict__ knn_idx, const T* __restrict__ w,
                                 int op, T mix, T* __restrict__ cval, uint8_t* __restrict__ inonly,
                                 int32_t* __restrict__ n_out, int32_t* __restrict__ n_in) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * k) return;
  const int64_t i = t / k;
  const int32_t j = knn_idx[t];
  T c = (T)0;
  bool in_only = false;
  if (j >= 0) {  // a self entry (j == i) finds itself, so b = a: the fuzzy kernel's 0 stays 0, gauss / jaccard keep C[i,i]
    const T a = w[t];
    T b = (T)0;
    bool found = false;
    const int32_t* lj = knn_idx + (int64_t)j * k;
    for (int m = 0; m < k; ++m) {
      if (lj[m] == (int32_t)i) { found = true; b = w[(int64_t)j * k + m]; break; }
    }
    c = sym_combine<T>(a, b, op, mix);
    in_only = !found && c != (T)0;
  }
  cval[t] = c;
  inonly[t] = in_only ? 1 : 0;
  if (c != (T)0) atomicAdd(&n_out[i], 1);
  if (in_only) atomicAdd(&n_in[j], 1);
}
__global__ void add_i32_kernel(const int32_t* __restrict__ a, const int32_t* __restrict__ b, int32_t* __restrict__ c, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) c[i] = a[i] + b[i];
}
template <typename T>
__global__ void sym_fill_kernel(int64_t n, int k, const int32_t* __restrict__ knn_idx, const T* __restrict__ cval,
                                const uint8_t* __restrict__ inonly, const int64_t* __restrict__ indptr,
                                const int32_t* __restrict__ n_out, int32_t* __restrict__ cursor,
                                int32_t* __restrict__ t_indices, T* __restrict__ t_data) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t p = indptr[i];
  for (int m = 0; m < k; ++m) {
    const int64_t t = i * k + m;
    const T c = cval[t];
    if (c != (T)0) {
      t_indices[p] = knn_idx[t];
      t_data[p] = c;
      ++p;
    }
    if (inonly[t]) {
      const int32_t j = knn_idx[t];
      const int64_t q = indptr[j] + n_out[j] + atomicAdd(&cursor[j], 1);
      t_indices[q] = (int32_t)i;
      t_data[q] = c;
    }
  }
}
template <typename T>
__global__ void __launch_bounds__(256)
sym_sort_rows_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ t_indices,
                     const T* __restrict__ t_data, int32_t* __restrict__ indices, T* __restrict__ data) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int64_t p0 = indptr[row];
  const int len = (int)(indptr[row + 1] - p0);
  if (len <= 32) {
    int32_t key = lane < len ? t_indices[p0 + lane] : INT32_MAX;
    T val = lane < len ? t_data[p0 + lane] : (T)0;
#pragma unroll
    for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
      for (int j = kk >> 1; j > 0; j >>= 1) {
        const int32_t ok = __shfl_xor_sync(0xffffffffu, key, j);
        const T ov = __shfl_xor_sync(0xffffffffu, val, j);
        const bool want_min = ((lane & j) == 0) == ((lane & kk) == 0);
        const bool take = want_min ? (ok < key) : (ok > key);
        if (take) { key = ok; val = ov; }
      }
    }
    if (lane < len) { indices[p0 + lane] = key; data[p0 + lane] = val; }
  } else {
    for (int a = lane; a < len; a += 32) {
      const int32_t key = t_indices[p0 + a];
      int rank = 0;
      for (int b = 0; b < len; ++b) rank += t_indices[p0 + b] < key;
      indices[p0 + rank] = key;
      data[p0 + rank] = t_data[p0 + a];
    }
  }
}

// ---- method='jaccard' / 'gauss' directed weights (SURVEY 8f row f3), fp64 like the reference ----
// jaccard (src/scanpy/neighbors/_connectivity.py:141-186): |N(i) & N(j)| / (2(k-1) - |N(i) & N(j)|), where N(i) is the
// list without its column 0.  Column 0 is normally self; when it is not (a duplicate cell came first), self sits in
// N(i) and gets J[i,i] = 1, as in the reference.
__global__ void jaccard_rows_kernel(int64_t n, int k, const int32_t* __restrict__ knn_idx, double* __restrict__ w) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * k) return;
  const int64_t i = t / k;
  const int m = (int)(t % k);
  const int32_t j = knn_idx[t];
  double val = 0.0;
  if (m > 0 && j >= 0) {
    const int32_t* li = knn_idx + i * k;
    const int32_t* lj = knn_idx + (int64_t)j * k;
    int shared = 0;
    for (int a = 1; a < k; ++a) {
      const int32_t x = li[a];
      for (int b = 1; b < k; ++b) shared += (lj[b] == x);
    }
    val = (double)shared / (double)(2 * (k - 1) - shared);
  }
  w[t] = val;
}
// gauss, sparse kNN branch (:17-100): sigma_i^2 = median of the k-1 squared neighbour distances; every entry after
// column 0 is weighted, self included when it is not first (its weight is exp(-d^2 / (2 sigma_i^2)))
template <int MK>
__global__ void gauss_sigma_kernel(int64_t n, int k, const double* __restrict__ knn_dist, double* __restrict__ sig_sq) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double d[MK];
  const int m = k - 1;
  for (int j = 0; j < m; ++j) { const double x = knn_dist[i * k + 1 + j]; d[j] = x * x; }
  for (int a = 1; a < m; ++a) {  // insertion sort (rows arrive ascending already)
    const double x = d[a];
    int b = a - 1;
    while (b >= 0 && d[b] > x) { d[b + 1] = d[b]; --b; }
    d[b + 1] = x;
  }
  sig_sq[i] = (m & 1) ? d[m / 2] : 0.5 * (d[m / 2 - 1] + d[m / 2]);  // np.median
}
__global__ void gauss_rows_kernel(int64_t n, int k, const int32_t* __restrict__ knn_idx, const double* __restrict__ knn_dist,
                                  const double* __restrict__ sig_sq, double* __restrict__ w) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * k) return;
  const int64_t i = t / k;
  const int m = (int)(t % k);
  const int32_t j = knn_idx[t];
  double val = 0.0;
  if (m > 0 && j >= 0) {
    const double si2 = sig_sq[i], sj2 = sig_sq[j];
    const double num = 2.0 * sqrt(si2) * sqrt(sj2), den = si2 + sj2;
    const double d = knn_dist[t];
    val = sqrt(num / den) * exp(-(d * d) / den);
  }
  w[t] = val;
}

// directed k-list weights w[n x k] -> symmetric CSR (sorted rows, no explicit zeros); syncs the stream
template <typename T>
int32_t symmetrize(sb2_ctx* ctx, ScratchScope& scr, int64_t n, int32_t k, const int32_t* d_knn_idx, const T* w, int op, T mix,
                   int64_t* d_indptr, int32_t* d_indices, T* d_data, int64_t cap, int64_t* h_nnz) {
  cudaStream_t st = ctx->stream;
  const int64_t nk = n * k;
  T *cval, *t_data;
  uint8_t* inonly;
  int32_t *n_out, *n_in, *len, *cursor, *t_indices;
  SB2_TRY(scr.alloc(&cval, (size_t)nk));
  SB2_TRY(scr.alloc(&inonly, (size_t)nk));
  SB2_TRY(scr.alloc(&n_out, (size_t)n * 4));
  n_in = n_out + n; len = n_in + n; cursor = len + n;
  SB2_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int32_t) * 4 * n, st));
  sym_count_kernel<T><<<(unsigned)ceil_div64(nk, 256), 256, 0, st>>>(n, k, d_knn_idx, w, op, mix, cval, inonly, n_out, n_in);
  SB2_LAUNCH_CHECK(ctx);
  add_i32_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(n_out, n_in, len, n);
  SB2_LAUNCH_CHECK(ctx);
  SB2_TRY(sb2_scan_i32_to_i64(ctx, len, n, d_indptr));
  int64_t nnz = 0;
  SB2_CUDA(cudaMemcpyAsync(&nnz, d_indptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  *h_nnz = nnz;
  if (nnz > cap) {
    sb2_set_error("connectivities need %lld entries but cap is %lld", (long long)nnz, (long long)cap);
    return SB2_E_BADARG;
  }
  SB2_TRY(scr.alloc(&t_indices, (size_t)nnz));
  SB2_TRY(scr.alloc(&t_data, (size_t)nnz));
  sym_fill_kernel<T><<<(unsigned)ceil_div64(n, 128), 128, 0, st>>>(n, k, d_knn_idx, cval, inonly, d_indptr, n_out, cursor, t_indices, t_data);
  SB2_LAUNCH_CHECK(ctx);
  sym_sort_rows_kernel<T><<<(unsigned)ceil_div64(n, 8), 256, 0, st>>>(n, d_indptr, t_indices, t_data, d_indices, d_data);
  SB2_LAUNCH_CHECK(ctx);
  SB2_CUDA(cudaStreamSynchronize(st));
  return SB2_OK;
}

}  // namespace

extern "C" int32_t sb2_knn_connectivities_f64(sb2_ctx* ctx, int64_t n, int32_t k, const int32_t* d_knn_idx,
                                              const double* d_knn_dist, int32_t method, int64_t* d_indptr,
                                              int32_t* d_indices, double* d_data, int64_t cap, int64_t* h_nnz) {
  SB2_CHECK_ARG(ctx && d_knn_idx && d_indptr && d_indices && d_data && h_nnz, "null pointer");
  SB2_CHECK_ARG(n >= 1 && k >= 2 && k <= MAXK, "k must be in [2,64]");
  SB2_CHECK_ARG(method == 1 || method == 2, "method: 1 = gauss, 2 = jaccard");
  SB2_CHECK_ARG(method == 2 || d_knn_dist, "gauss needs distances");
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  const int64_t nk = n * k;
  double* w;
  SB2_TRY(scr.alloc(&w, (size_t)nk));
  if (method == 2) {
    jaccard_rows_kernel<<<(unsigned)ceil_div64(nk, 256), 256, 0, st>>>(n, k, d_knn_idx, w);
    SB2_LAUNCH_CHECK(ctx);
    return symmetrize<double>(ctx, scr, n, k, d_knn_idx, w, SYM_AVERAGE, 1.0, d_indptr, d_indices, d_data, cap, h_nnz);
  }
  double* sig_sq;
  SB2_TRY(scr.alloc(&sig_sq, (size_t)n));
  if (k <= 32) gauss_sigma_kernel<32><<<(unsigned)ceil_div64(n, 128), 128, 0, st>>>(n, k, d_knn_dist, sig_sq);
  else gauss_sigma_kernel<64><<<(unsigned)ceil_div64(n, 128), 128, 0, st>>>(n, k, d_knn_dist, sig_sq);
  SB2_LAUNCH_CHECK(ctx);
  gauss_rows_kernel<<<(unsigned)ceil_div64(nk, 256), 256, 0, st>>>(n, k, d_knn_idx, d_knn_dist, sig_sq, w);
  SB2_LAUNCH_CHECK(ctx);
  return symmetrize<double>(ctx, scr, n, k, d_knn_idx, w, SYM_COPY_MISSING, 1.0, d_indptr, d_indices, d_data, cap, h_nnz);
}

extern "C" int32_t sb2_fuzzy_simplicial_set_f32(sb2_ctx* ctx, int64_t n, int32_t k, const int32_t* d_knn_idx,
                                                const double* d_knn_dist, float set_op_mix_ratio,
                                                float local_connectivity, int64_t* d_indptr, int32_t* d_indices,
                                                float* d_data, int64_t cap, int64_t* h_nnz, float* d_sigmas,
                                                float* d_rhos) {
  SB2_CHECK_ARG(ctx && d_knn_idx && d_knn_dist && d_indptr && d_indices && d_data && h_nnz, "null pointer");
  SB2_CHECK_ARG(n >= 1 && k >= 2 && k <= MAXK, "k must be in [2,64]");
  SB2_CHECK_ARG(set_op_mix_ratio >= 0.0f && set_op_mix_ratio <= 1.0f, "set_op_mix_ratio in [0,1]");
  SB2_CHECK_ARG(local_connectivity >= 0.0f && local_connectivity < (float)k, "local_connectivity");
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  const int64_t nk = n * k;
  float *w, *sig, *rho;
  double* dsum;
  SB2_TRY(scr.alloc(&w, (size_t)nk));
  SB2_TRY(scr.alloc(&dsum, 2));
  SB2_TRY(scr.alloc(&sig, (size_t)n));
  SB2_TRY(scr.alloc(&rho, (size_t)n));
  SB2_CUDA(cudaMemsetAsync(dsum, 0, 16, st));
  sum_f32cast_kernel<<<ctx->prop.multiProcessorCount * 4, 256, 0, st>>>(d_knn_dist, nk, dsum);
  SB2_LAUNCH_CHECK(ctx);
  if (k <= 32)
    fuzzy_rows_kernel<32><<<(unsigned)ceil_div64(n, 128), 128, 0, st>>>(n, k, d_knn_idx, d_knn_dist, local_connectivity, dsum, w,
                                                                        d_sigmas ? d_sigmas : sig, d_rhos ? d_rhos : rho);
  else
    fuzzy_rows_kernel<64><<<(unsigned)ceil_div64(n, 128), 128, 0, st>>>(n, k, d_knn_idx, d_knn_dist, local_connectivity, dsum, w,
                                                                        d_sigmas ? d_sigmas : sig, d_rhos ? d_rhos : rho);
  SB2_LAUNCH_CHECK(ctx);
  return symmetrize<float>(ctx, scr, n, k, d_knn_idx, w, SYM_FUZZY_UNION, set_op_mix_ratio, d_indptr, d_indices, d_data, cap,
                           h_nnz);
}


// ---- sc.tl.paga aggregation (SURVEY.md 8f row f3) ----------------------------------------------------------------------
// counts[gi * G + gj] = number of stored arcs i -> j with group[i] = gi, group[j] = gj: what igraph's
// `VertexClustering.cluster_graph(combine_edges="sum")` + `subgraph(i).ecount()` give PAGA on the all-ones distances graph
// (src/scanpy/tools/_paga.py:177-208).  Warp per row: the lanes' target groups are merged with MATCH.ANY, so a row whose
// neighbours sit in one or two groups issues one or two atomics.
namespace {
__global__ void __launch_bounds__(256)
group_arc_counts_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                        const int32_t* __restrict__ group, int G, unsigned long long* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int gi = group[row];
  const int64_t e0 = indptr[row], e1 = indptr[row + 1];
  for (int64_t base = e0; base < e1; base += 32) {
    const int64_t e = base + lane;
    const bool on = e < e1;
    const int gj = on ? group[indices[e]] : -1;
    const unsigned act = __ballot_sync(0xffffffffu, on);
    if (on) {
      const unsigned same = __match_any_sync(act, gj);
      if ((int)(__ffs(same) - 1) == lane && gi >= 0 && gi < G && gj >= 0 && gj < G)
        atomicAdd(&counts[(size_t)gi * G + gj], (unsigned long long)__popc(same));
    }
  }
}
}  // namespace

extern "C" int32_t sb2_group_arc_counts(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                        const int32_t* d_group, int32_t n_groups, int64_t* d_counts) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_group && d_counts, "null pointer");
  SB2_CHECK_ARG(n_groups >= 1 && n_groups <= 46340, "n_groups");
  SB2_CUDA(cudaSetDevice(ctx->device));
  SB2_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(int64_t) * (size_t)n_groups * n_groups, ctx->stream));
  if (n == 0) return SB2_OK;
  group_arc_counts_kernel<<<(unsigned)ceil_div64(n, 8), 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_group, n_groups,
                                                                            reinterpret_cast<unsigned long long*>(d_counts));
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

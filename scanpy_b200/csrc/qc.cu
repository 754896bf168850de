// qc.cu — the per-cell and per-gene passes of
//   sc.pp.calculate_qc_metrics  (src/scanpy/preprocessing/_qc.py:41-307; the top-n shares follow the numba
//                               `top_segment_proportions_sparse_csr`, :430-457)
//   sc.pp.filter_cells / sc.pp.filter_genes  (src/scanpy/preprocessing/_simple.py:53-306)
//
// Row pass: one CTA per row reduces the count, the fp64 total and the fp64 totals over up to 32 gene masks.  For the
// top-n sums the set S is the row's NON-ZERO stored values (explicit zeros are ignored, so the result is what the
// reference computes after `eliminate_zeros()`), m = max(ns), k = min(|S|, m) and z = max(0, m - |S|) zero pads:
//   top(n) = sum of the n largest of S ∪ {z zeros} = P[n] (n <= q), P[q] (q < n <= q + z), P[n - z] (otherwise),
// with P the prefix sums of S sorted descending and q = #{s in S : s > 0}.  So every row only needs its k largest
// values sorted.  Rows of at most SHORT_CAP stored values are staged in shared memory and bitonic-sorted whole; longer
// rows are queued and a second kernel radix-selects the k-th largest order-preserving 32-bit key over the row (read
// from L2), gathers the k candidates (ties filled with the threshold) and sorts only those.  The prefix sums are taken
// in a fixed order over the sorted values (16-value segments summed in order, then the segment sums in order), so a
// top-n sum depends only on the multiset S: bit-identical across runs, launch shapes and the two paths.  HBM traffic is
// one read of the row (8 B per stored value, +4 B with gene masks for the column index).
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int QC_THREADS = 128;    // row pass: one CTA per row
constexpr int SHORT_CAP = 2048;    // stored values per row staged by the row pass (8 KB of keys)
constexpr int LONG_THREADS = 512;  // long rows: one CTA per queued row
constexpr int SEG = 16;            // prefix sums: fixed 16-value segments
constexpr int MAX_QC = 32;

// order-preserving float -> uint32 (a > b  <=>  key(a) > key(b)); key 0 is a NaN bit pattern and serves as "empty"
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__host__ __device__ __forceinline__ int pow2_ceil(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// s[0..p) sorted descending in place (p a power of two); the caller synchronises before
__device__ void bitonic_desc(uint32_t* s, int p) {
  for (int k = 2; k <= p; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < p; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint32_t a = s[i], b = s[ixj];
          if ((i & k) == 0 ? a < b : a > b) { s[i] = b; s[ixj] = a; }
        }
      }
      __syncthreads();
    }
}

// s[0..k): the k largest values of S as keys, sorted descending; nz = |S|, q = #positive values in S.
// out[i] = sum of the ns[i] largest values of S padded with max(0, m - nz) zeros.  seg: k / SEG + 1 doubles.
__device__ void top_sums(const uint32_t* s, int k, int64_t nz, int64_t q, int m, const int32_t* ns, int n_ns,
                         double* seg, double* out) {
  const int nseg = (k + SEG - 1) / SEG;
  for (int t = threadIdx.x; t < nseg; t += blockDim.x) {
    const int e1 = min(k, (t + 1) * SEG);
    double a = 0.0;
    for (int e = t * SEG; e < e1; ++e) a += (double)key2f(s[e]);
    seg[t + 1] = a;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    seg[0] = 0.0;
    for (int t = 1; t <= nseg; ++t) seg[t] += seg[t - 1];
  }
  __syncthreads();
  const int64_t z = nz < m ? m - nz : 0;
  for (int i = threadIdx.x; i < n_ns; i += blockDim.x) {
    const int64_t n = ns[i];
    const int64_t j = n <= q ? n : (n <= q + z ? q : n - z);
    double p = seg[j / SEG];
    for (int64_t e = j / SEG * SEG; e < j; ++e) p += (double)key2f(s[e]);
    out[i] = p;
  }
  __syncthreads();
}

struct RowStats {
  int64_t nz, pos;
};

template <bool HAS_QC>
__global__ void __launch_bounds__(QC_THREADS)
qc_rows_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
               const float* __restrict__ data, int positive_only, const uint32_t* __restrict__ qc_bits, int n_qc,
               const int32_t* __restrict__ ns, int n_ns, int m, int64_t* __restrict__ count, double* __restrict__ total,
               double* __restrict__ qc_total, double* __restrict__ top, int64_t* __restrict__ long_rows,
               unsigned long long* __restrict__ n_long) {
  __shared__ uint32_t keys[SHORT_CAP];
  __shared__ double seg[SHORT_CAP / SEG + 1];
  __shared__ double red_d[QC_THREADS / 32];
  __shared__ int64_t red_i[QC_THREADS / 32];
  __shared__ RowStats rs;
  const int64_t row = blockIdx.x;
  const int64_t e0 = indptr[row], len = indptr[row + 1] - e0;
  const bool stage = n_ns > 0 && len <= SHORT_CAP;
  int64_t cnt = 0, nz = 0, pos = 0;
  double tot = 0.0;
  double acc[HAS_QC ? MAX_QC : 1];
#pragma unroll
  for (int b = 0; b < (HAS_QC ? MAX_QC : 1); ++b) acc[b] = 0.0;
  for (int64_t i = threadIdx.x; i < len; i += QC_THREADS) {
    const float v = data[e0 + i];
    cnt += positive_only ? v > 0.0f : v != 0.0f;
    nz += v != 0.0f;
    pos += v > 0.0f;
    tot += (double)v;
    if (HAS_QC) {
      const uint32_t bits = qc_bits[indices[e0 + i]];
#pragma unroll
      for (int b = 0; b < MAX_QC; ++b)
        if ((bits >> b) & 1u) acc[b] += (double)v;
    }
    if (stage) keys[i] = v != 0.0f ? f2key(v) : 0u;
  }
  cnt = block_sum(cnt, red_i);
  nz = block_sum(nz, red_i);
  pos = block_sum(pos, red_i);
  tot = block_sum(tot, red_d);
  if (threadIdx.x == 0) {
    count[row] = cnt;
    total[row] = tot;
    rs.nz = nz;
    rs.pos = pos;
  }
  if (HAS_QC) {
#pragma unroll
    for (int b = 0; b < MAX_QC; ++b) {
      if (b >= n_qc) break;
      const double s = block_sum(acc[b], red_d);
      if (threadIdx.x == 0) qc_total[row * n_qc + b] = s;
    }
  }
  if (n_ns == 0) return;
  if (!stage) {
    if (threadIdx.x == 0) long_rows[atomicAdd(n_long, 1ull)] = row;
    return;
  }
  const int p = pow2_ceil((int)len);
  for (int i = (int)len + threadIdx.x; i < p; i += QC_THREADS) keys[i] = 0u;
  __syncthreads();
  bitonic_desc(keys, p);
  const int64_t rnz = rs.nz;
  top_sums(keys, (int)(rnz < m ? rnz : m), rnz, rs.pos, m, ns, n_ns, seg, top + row * n_ns);
}

// the queued long rows: radix-select the k-th largest non-zero key (4 passes of 8 bits over the row), gather the k
// candidates into shared memory, sort them, then the same top_sums as the row pass
__global__ void __launch_bounds__(LONG_THREADS)
qc_long_rows_kernel(const int64_t* __restrict__ indptr, const float* __restrict__ data, const int32_t* __restrict__ ns,
                    int n_ns, int m, int cap, const int64_t* __restrict__ long_rows,
                    const unsigned long long* __restrict__ n_long, double* __restrict__ top) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint32_t* keys = reinterpret_cast<uint32_t*>(smem);
  double* seg = reinterpret_cast<double*>(smem + sizeof(uint32_t) * (size_t)cap);
  __shared__ int64_t red_i[LONG_THREADS / 32];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel_prefix, sel_mask, n_gt;
  __shared__ int64_t sel_left, row_nz, row_pos;
  const int64_t nl = (int64_t)*n_long;
  for (int64_t r = blockIdx.x; r < nl; r += gridDim.x) {
    const int64_t row = long_rows[r];
    const int64_t e0 = indptr[row], e1 = indptr[row + 1];
    int64_t nz = 0, pos = 0;
    for (int64_t e = e0 + threadIdx.x; e < e1; e += LONG_THREADS) {
      const float v = data[e];
      nz += v != 0.0f;
      pos += v > 0.0f;
    }
    nz = block_sum(nz, red_i);
    pos = block_sum(pos, red_i);
    if (threadIdx.x == 0) {
      row_nz = nz;
      row_pos = pos;
      sel_prefix = 0u;
      sel_mask = 0u;
      sel_left = nz < m ? nz : m;
      n_gt = 0u;
    }
    __syncthreads();
    const int64_t k = row_nz < m ? row_nz : m;
    if (k > cap) {  // excluded by the entry point's row-length check
      for (int i = threadIdx.x; i < n_ns; i += LONG_THREADS) top[row * n_ns + i] = nan("");
      __syncthreads();
      continue;
    }
    for (int shift = 24; shift >= 0 && k > 0; shift -= 8) {
      for (int i = threadIdx.x; i < 256; i += LONG_THREADS) hist[i] = 0u;
      __syncthreads();
      const uint32_t pre = sel_prefix, msk = sel_mask;
      for (int64_t e = e0 + threadIdx.x; e < e1; e += LONG_THREADS) {
        const float v = data[e];
        if (v == 0.0f) continue;
        const uint32_t key = f2key(v);
        if ((key & msk) == pre) atomicAdd(&hist[(key >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int64_t above = 0, left = sel_left;
        int b = 255;
        for (; b > 0; --b) {
          if (above + hist[b] >= left) break;
          above += hist[b];
        }
        sel_left = left - above;
        sel_prefix = pre | ((uint32_t)b << shift);
        sel_mask = msk | (255u << shift);
      }
      __syncthreads();
    }
    // keys > threshold, then (k - #greater) copies of the threshold: the k largest as a multiset
    const uint32_t thr = sel_prefix;
    if (k > 0)
      for (int64_t e = e0 + threadIdx.x; e < e1; e += LONG_THREADS) {
        const float v = data[e];
        if (v == 0.0f) continue;
        const uint32_t key = f2key(v);
        if (key > thr) keys[atomicAdd(&n_gt, 1u)] = key;
      }
    __syncthreads();
    const int p = pow2_ceil((int)k);
    for (int i = (int)n_gt + threadIdx.x; i < p; i += LONG_THREADS) keys[i] = i < k ? thr : 0u;
    __syncthreads();
    bitonic_desc(keys, p);
    top_sums(keys, (int)k, row_nz, row_pos, m, ns, n_ns, seg, top + row * n_ns);
  }
}

__global__ void max_row_len_kernel(int64_t n, const int64_t* __restrict__ indptr, unsigned long long* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicMax(out, (unsigned long long)(indptr[i + 1] - indptr[i]));
}

__global__ void col_counts_kernel(int64_t nnz, const int32_t* __restrict__ indices, const float* __restrict__ data,
                                  int positive_only, unsigned long long* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = data[i];
    if (positive_only ? v > 0.0f : v != 0.0f) atomicAdd(&out[indices[i]], 1ull);
  }
}

size_t long_smem(int cap) { return sizeof(uint32_t) * (size_t)cap + sizeof(double) * (size_t)(cap / SEG + 1); }

}  // namespace

extern "C" {

int32_t sb2_csr_qc_rows_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                            const float* d_data, int32_t positive_only, const uint32_t* d_qc_bits, int32_t n_qc,
                            const int32_t* h_ns, int32_t n_ns, int64_t* d_count, double* d_total, double* d_qc_total,
                            double* d_top) {
  SB2_CHECK_ARG(ctx && d_indptr && d_count && d_total && g >= 1, "null pointer");
  SB2_CHECK_ARG(n_qc >= 0 && n_qc <= MAX_QC, "n_qc must be in [0, 32]");
  SB2_CHECK_ARG(n_qc == 0 || (d_qc_bits && d_indices && d_qc_total), "qc masks need indices and an output");
  SB2_CHECK_ARG(n_ns >= 0 && (n_ns == 0 || (h_ns && d_top)), "ns");
  for (int i = 0; i < n_ns; ++i) {
    SB2_CHECK_ARG(h_ns[i] >= 1 && h_ns[i] <= g, "ns must lie in [1, g]");
    SB2_CHECK_ARG(i == 0 || h_ns[i] >= h_ns[i - 1], "ns must be sorted ascending");
  }
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  SB2_CHECK_ARG(n < INT32_MAX, "n");
  const int m = n_ns > 0 ? h_ns[n_ns - 1] : 0;
  int cap = 0;
  ScratchScope scr(ctx);
  int32_t* d_ns = nullptr;
  int64_t* long_rows = nullptr;
  unsigned long long* n_long = nullptr;
  if (n_ns > 0) {
    // the largest power-of-two candidate count whose keys and segment sums fit the opt-in shared memory
    const size_t lim = ctx->prop.sharedMemPerBlockOptin - 8192;
    cap = SHORT_CAP;
    while (long_smem(cap * 2) <= lim) cap *= 2;
    SB2_TRY(scr.alloc(&d_ns, (size_t)n_ns));
    SB2_TRY(scr.alloc(&long_rows, (size_t)n));
    SB2_TRY(scr.alloc(&n_long, 1));
    SB2_CUDA(cudaMemcpyAsync(d_ns, h_ns, sizeof(int32_t) * (size_t)n_ns, cudaMemcpyHostToDevice, ctx->stream));
    SB2_CUDA(cudaMemsetAsync(n_long, 0, sizeof(unsigned long long), ctx->stream));
    if (m > cap) {  // k = min(|S|, m) candidates must fit in shared memory: check the longest row
      unsigned long long h_max = 0;
      SB2_CUDA(cudaMemcpyAsync(n_long, &h_max, sizeof(h_max), cudaMemcpyHostToDevice, ctx->stream));
      max_row_len_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, ctx->stream>>>(n, d_indptr, n_long);
      SB2_LAUNCH_CHECK(ctx);
      SB2_CUDA(cudaMemcpyAsync(&h_max, n_long, sizeof(h_max), cudaMemcpyDeviceToHost, ctx->stream));
      SB2_CUDA(cudaStreamSynchronize(ctx->stream));
      SB2_CUDA(cudaMemsetAsync(n_long, 0, sizeof(unsigned long long), ctx->stream));
      if (h_max > (unsigned long long)cap) {
        sb2_set_error("bad argument: top-n shares with max(ns) = %d > %d need rows of at most %d stored values (a row "
                      "has %llu)", m, cap, cap, h_max);
        return SB2_E_BADARG;
      }
    }
  }
  if (n_qc > 0)
    qc_rows_kernel<true><<<(unsigned)n, QC_THREADS, 0, ctx->stream>>>(
        n, d_indptr, d_indices, d_data, positive_only, d_qc_bits, n_qc, d_ns, n_ns, m, d_count, d_total, d_qc_total, d_top,
        long_rows, n_long);
  else
    qc_rows_kernel<false><<<(unsigned)n, QC_THREADS, 0, ctx->stream>>>(
        n, d_indptr, d_indices, d_data, positive_only, nullptr, 0, d_ns, n_ns, m, d_count, d_total, nullptr, d_top,
        long_rows, n_long);
  SB2_LAUNCH_CHECK(ctx);
  if (n_ns > 0) {
    const size_t smem = long_smem(cap);
    SB2_CUDA(cudaFuncSetAttribute(qc_long_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    qc_long_rows_kernel<<<(unsigned)ctx->prop.multiProcessorCount, LONG_THREADS, smem, ctx->stream>>>(
        d_indptr, d_data, d_ns, n_ns, m, cap, long_rows, n_long, d_top);
    SB2_LAUNCH_CHECK(ctx);
  }
  return SB2_OK;
}

int32_t sb2_csr_col_counts_f32(sb2_ctx* ctx, int64_t nnz, int32_t g, const int32_t* d_indices, const float* d_data,
                               int32_t positive_only, int64_t* d_counts) {
  SB2_CHECK_ARG(ctx && d_counts && g >= 1 && (nnz == 0 || (d_indices && d_data)), "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  SB2_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(int64_t) * (size_t)g, ctx->stream));
  if (nnz == 0) return SB2_OK;
  const int64_t grid = std::min<int64_t>(ceil_div64(nnz, 256), (int64_t)ctx->prop.multiProcessorCount * 16);
  col_counts_kernel<<<(unsigned)grid, 256, 0, ctx->stream>>>(nnz, d_indices, d_data, positive_only,
                                                             reinterpret_cast<unsigned long long*>(d_counts));
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

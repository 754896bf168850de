// aggregate.cu — the per-group passes over X of
//   sc.get.aggregate  (src/scanpy/get/_aggregated.py:47-190, 663-698)
//
// Group order: a stable counting sort of the kept rows by their int32 group code (-1: no group).  Rows are cut into
// tiles; one pass counts each group's rows per tile, a per-group walk over the tiles turns the counts into each tile's
// first slot in the group, and one warp per tile places its rows in row order (match_any ranks equal codes within a
// warp step).  No placement depends on timing, so the order is the same on every call.
//
// Moments: the call's rows are segments, each a run of consecutive rows of one group (the caller groups them with the
// order above).  One CTA per (SLAB_TILE-row subtile of a segment, 256-gene slab) reads the subtile's rows (CSR rows
// through stage_csr, dense rows in place) and keeps, per gene, Welford's mean and M2, Σx and the count of x != 0, all
// in fp64 (implicit zeros are values; stored zeros are not non-zero).  A group whose rows fit one subtile is written
// straight to the outputs; longer groups write per-subtile partials that a fold merges into the outputs in subtile
// order with Chan's formula.  Subtiles start at the group's first row, so the bits depend only on the group's rows and
// their order, not on how the caller splits X into blocks.
//
// Median: np.median per (group, gene), the mean of the order statistics ⌊(n-1)/2⌋ and ⌊n/2⌋ over all n values of the
// group, zeros included.  One CTA per (group, MED_GENES genes) runs a radix selection on order-preserving integer keys
// (8-bit digits: 4 passes for float32, 8 for float64), re-reading the group's rows in every pass.  For a CSR the
// group's implicit zeros (n minus the stored count) are added to the bucket of the key of 0.0, so zeros are never
// materialised; NaN sorts above +inf, as in sklearn's csc_median_axis_0.  A dense X gives NaN when the group holds a
// NaN, as np.median does.  The upper statistic comes from the last digit histogram, or, when the lower one ends its
// bucket run, from one more pass taking the least key above it.
#include <math.h>

#include "common.cuh"
#include "slab.cuh"

namespace {

constexpr int GO_TILE = 4096;        // rows per tile of the group order
constexpr int GO_WARPS = 4;          // tiles (warps) per CTA of the placement
constexpr int64_t GO_HIST_BYTES = int64_t(1) << 28;  // cap of the per-tile count table
constexpr int64_t AG_PARTIAL_BYTES = int64_t(1) << 28;  // scratch for the moments' per-subtile partials per launch
constexpr int MED_GENES = 64;        // genes per median CTA
constexpr int MED_THREADS = 512;
constexpr int MED_WARPS = MED_THREADS / 32;
constexpr int MED_BINS = 256;        // 8-bit digits
constexpr int MED_SMEM = MED_GENES * MED_BINS * 4;

// ------------------------------------------------------------------------------------------ group order
__global__ void order_count_kernel(int64_t n, int64_t tile, int ng, const int32_t* __restrict__ codes,
                                   int32_t* __restrict__ hist) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = codes[i];
    if (c >= 0) atomicAdd(&hist[(i / tile) * ng + c], 1);
  }
}

// hist[t][c] -> the number of group c's rows in tiles before t; counts[c] = the group's rows
__global__ void order_base_kernel(int64_t ntiles, int ng, int32_t* __restrict__ hist, int32_t* __restrict__ counts) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ng) return;
  int32_t run = 0;
  for (int64_t t = 0; t < ntiles; ++t) {
    const int32_t h = hist[t * ng + c];
    hist[t * ng + c] = run;
    run += h;
  }
  counts[c] = run;
}

// one warp per tile, 32 rows per step in row order: a row's slot is its group's start, plus the group's rows in
// earlier tiles and earlier steps (base, advanced by the step's last lane of the group), plus its rank in the step
__global__ void __launch_bounds__(GO_WARPS * 32)
order_place_kernel(int64_t n, int64_t tile, int ng, const int32_t* __restrict__ codes,
                   const int64_t* __restrict__ offsets, int32_t* __restrict__ base, int64_t* __restrict__ order) {
  const int64_t t = (int64_t)blockIdx.x * GO_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t r0 = t * tile, r1 = min(n, r0 + tile);
  if (r0 >= n) return;
  int32_t* b = base + t * ng;
  for (int64_t s = r0; s < r1; s += 32) {
    const int64_t i = s + lane;
    const int c = i < r1 ? codes[i] : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    if (c >= 0) {
      const int rank = __popc(peers & ((1u << lane) - 1));
      order[offsets[c] + b[c] + rank] = i;
    }
    __syncwarp();
    if (c >= 0 && lane == 31 - __clz(peers)) b[c] += __popc(peers);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------ moments
// items[k] = {first call row, rows, group, partial slot or -1: the group's only subtile, written to the outputs}
struct Item {
  int64_t r0;
  int32_t m, group, slot, pad;
};

// grid (items, slabs); part[slot][k][j]: k = 0 mean, 1 M2, 2 Σx, 3 count of x != 0
template <typename T, bool CSR>
__global__ void __launch_bounds__(SLAB_THREADS, 1)
moments_kernel(int g, const T* __restrict__ x, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
               const T* __restrict__ data, const int64_t* __restrict__ order, const Item* __restrict__ items,
               double* __restrict__ part, double* __restrict__ sum, double* __restrict__ mean,
               double* __restrict__ m2, int64_t* __restrict__ nnz) {
  __shared__ T tile[CSR ? SLAB_ROWS : 1][SLAB_THREADS];
  __shared__ int64_t rid[SLAB_ROWS], lo[SLAB_ROWS], hi[SLAB_ROWS];
  const Item it = items[blockIdx.x];
  const int c0 = blockIdx.y * SLAB_THREADS, c = c0 + threadIdx.x;
  const int c1 = min(g, c0 + SLAB_THREADS);
  double mu = 0.0, q = 0.0, s = 0.0, k = 0.0;
  int nz = 0;  // at most SLAB_TILE
  if (CSR)
    for (int r = 0; r < SLAB_ROWS; ++r) tile[r][threadIdx.x] = T(0);
  for (int b = 0; b < it.m; b += SLAB_ROWS) {
    const int m = min(SLAB_ROWS, it.m - b);
    if ((int)threadIdx.x < m) {
      const int64_t p = it.r0 + b + threadIdx.x;
      rid[threadIdx.x] = order ? order[p] : p;
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
        k += 1.0;
        const double d = v - mu;
        mu += d / k;
        q += d * (v - mu);
        s += v;
        nz += v != 0.0;
      }
    }
    __syncthreads();
  }
  if (c >= g) return;
  if (it.slot < 0) {
    const int64_t o = (int64_t)it.group * g + c;
    sum[o] = s;
    mean[o] = mu;
    m2[o] = q;
    nnz[o] = nz;
  } else {
    double* p = part + (int64_t)it.slot * 4 * g;
    p[c] = mu;
    p[g + c] = q;
    p[2 * (int64_t)g + c] = s;
    p[3 * (int64_t)g + c] = (double)nz;
  }
}

// folds[f] = {first slot, end slot, group, rows of the group merged before}: the slots of one group, in subtile order
struct Fold {
  int64_t s0, s1, n0;
  int32_t group, pad;
};

// grid (folds, gene blocks); slot_rows[s] = rows of slot s's subtile
__global__ void fold_kernel(int g, const Fold* __restrict__ folds, const int32_t* __restrict__ slot_rows,
                            const double* __restrict__ part, double* __restrict__ sum, double* __restrict__ mean,
                            double* __restrict__ m2, int64_t* __restrict__ nnz) {
  const int j = blockIdx.y * blockDim.x + threadIdx.x;
  if (j >= g) return;
  const Fold f = folds[blockIdx.x];
  const int64_t o = (int64_t)f.group * g + j;
  double n = (double)f.n0, mu = mean[o], q = m2[o], s = sum[o];
  int64_t nz = nnz[o];
  for (int64_t t = f.s0; t < f.s1; ++t) {
    const double* p = part + t * 4 * (int64_t)g;
    const double nb = (double)slot_rows[t];
    const double mb = p[j], qb = p[g + j];
    if (n == 0.0) {
      mu = mb;
      q = qb;
    } else {
      const double nn = n + nb, d = mb - mu;
      mu += d * (nb / nn);
      q += qb + d * d * (n * nb / nn);
    }
    n += nb;
    s += p[2 * (int64_t)g + j];
    nz += (int64_t)p[3 * (int64_t)g + j];
  }
  sum[o] = s;
  mean[o] = mu;
  m2[o] = q;
  nnz[o] = nz;
}

// ------------------------------------------------------------------------------------------ median
template <typename T>
struct KeyOf;
template <>
struct KeyOf<float> {
  using K = uint32_t;
  static constexpr int BITS = 32;
};
template <>
struct KeyOf<double> {
  using K = unsigned long long;
  static constexpr int BITS = 64;
};

// order-preserving key: -0.0 maps to +0.0 and every NaN to one NaN above +inf
template <typename T>
__device__ __forceinline__ typename KeyOf<T>::K to_key(T v) {
  using K = typename KeyOf<T>::K;
  constexpr K SIGN = K(1) << (KeyOf<T>::BITS - 1);
  K u;
  if (v == T(0)) u = 0;
  else if (v != v) u = sizeof(T) == 4 ? K(0x7FC00000u) : K(0x7FF8000000000000ull);
  else if constexpr (sizeof(T) == 4) u = __float_as_uint(v);
  else u = (K)__double_as_longlong(v);
  return (u & SIGN) ? ~u : (u | SIGN);
}

template <typename T>
__device__ __forceinline__ T from_key(typename KeyOf<T>::K k) {
  using K = typename KeyOf<T>::K;
  constexpr K SIGN = K(1) << (KeyOf<T>::BITS - 1);
  const K u = (k & SIGN) ? (k & ~SIGN) : ~k;
  if constexpr (sizeof(T) == 4) return __uint_as_float(u);
  else return __longlong_as_double((long long)u);
}

// calls f(j, v) for the group's values in genes [c0, c0 + w), row by row, a warp per row.  A CSR row gives its stored
// values only: all lanes search the row for c0, then lane l takes entries l, l + 32, ... while they stay below c0 + w.
template <typename T, bool CSR, typename F>
__device__ __forceinline__ void walk_group(int g, const T* __restrict__ x, const int64_t* __restrict__ indptr,
                                           const int32_t* __restrict__ indices, const T* __restrict__ data,
                                           const int64_t* __restrict__ order, int64_t r0, int64_t n, int c0, int w,
                                           F&& f) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t i = warp; i < n; i += MED_WARPS) {
    const int64_t row = order ? order[r0 + i] : r0 + i;
    if (CSR) {
      int64_t a = indptr[row], b = indptr[row + 1];
      const int64_t e1 = b;
      while (a < b) {
        const int64_t mid = (a + b) >> 1;
        if (indices[mid] < c0) a = mid + 1; else b = mid;
      }
      for (int64_t e = a + lane; e < e1; e += 32) {
        const int col = indices[e] - c0;
        if (col >= w) break;
        f(col, data[e]);
      }
    } else {
      for (int j = lane; j < w; j += 32) f(j, x[row * g + c0 + j]);
    }
  }
}

// grid (segments, gene blocks); segment s = call rows [seg[s], seg[s + 1]), all the rows of group seg_group[s]
template <typename T, bool CSR>
__global__ void __launch_bounds__(MED_THREADS)
median_kernel(int g, const T* __restrict__ x, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
              const T* __restrict__ data, const int64_t* __restrict__ order, const int64_t* __restrict__ seg,
              const int32_t* __restrict__ seg_group, T* __restrict__ out) {
  using K = typename KeyOf<T>::K;
  constexpr int BITS = KeyOf<T>::BITS, PASSES = BITS / 8;
  extern __shared__ uint32_t hist[];  // [MED_GENES][MED_BINS]
  __shared__ K prefix[MED_GENES], upper[MED_GENES];
  __shared__ uint32_t rank[MED_GENES], zeros[MED_GENES];
  __shared__ int nan_seen[MED_GENES], need_upper[MED_GENES], any_upper;
  const int64_t r0 = seg[blockIdx.x], n = seg[blockIdx.x + 1] - r0;
  const int c0 = blockIdx.y * MED_GENES, w = min(MED_GENES, g - c0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const K key0 = to_key(T(0));
  if ((int)threadIdx.x < MED_GENES) {
    prefix[threadIdx.x] = 0;
    rank[threadIdx.x] = (uint32_t)((n - 1) / 2);
    zeros[threadIdx.x] = 0;
    nan_seen[threadIdx.x] = 0;
    need_upper[threadIdx.x] = 0;
  }
  if (threadIdx.x == 0) any_upper = 0;
  for (int p = 0; p < PASSES; ++p) {
    const int shift = BITS - 8 * (p + 1);
    for (int i = threadIdx.x; i < MED_GENES * MED_BINS; i += MED_THREADS) hist[i] = 0;
    __syncthreads();
    walk_group<T, CSR>(g, x, indptr, indices, data, order, r0, n, c0, w, [&](int j, T v) {
      const K k = to_key(v);
      if (!CSR && p == 0 && v != v) nan_seen[j] = 1;
      if (p == 0 || ((k ^ prefix[j]) >> (shift + 8)) == 0) atomicAdd(&hist[j * MED_BINS + ((k >> shift) & 255)], 1u);
    });
    __syncthreads();
    // a warp per gene: lane l owns bins 8l .. 8l + 7
    for (int j = warp; j < w; j += MED_WARPS) {
      uint32_t h[8], local = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        h[q] = hist[j * MED_BINS + lane * 8 + q];
        local += h[q];
      }
      if (CSR) {
        if (p == 0) {
          const uint32_t stored = warp_sum(local);
          if (lane == 0) zeros[j] = (uint32_t)n - stored;
          __syncwarp();
        }
        const uint32_t z = zeros[j];
        const int zb = (int)((key0 >> shift) & 255);
        if (z && (p == 0 || ((key0 ^ prefix[j]) >> (shift + 8)) == 0) && (zb >> 3) == lane) {
#pragma unroll
          for (int q = 0; q < 8; ++q)
            if (q == (zb & 7)) h[q] += z;
          local += z;
        }
      }
      uint32_t incl = local;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      const uint32_t r = rank[j], excl = incl - local;
      const unsigned hit = __ballot_sync(0xffffffffu, excl <= r && r < incl);
      if (!hit) continue;  // only when X changed under the call
      const int src = __ffs(hit) - 1;
      const unsigned later = __ballot_sync(0xffffffffu, local > 0) & ~((2u << src) - 1);
      const int first_later = later ? __ffs(later) - 1 : 0;
      int nb = -1;  // the first non-empty bin of the first non-empty lane above src
#pragma unroll
      for (int q = 7; q >= 0; --q)
        if (h[q]) nb = lane * 8 + q;
      nb = __shfl_sync(0xffffffffu, nb, first_later);
      if (lane == src) {
        uint32_t cum = excl, in_bin = 0;
        int b = -1;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (b < 0) {
            if (r < cum + h[q]) {
              b = q;
              in_bin = h[q];
            } else {
              cum += h[q];
            }
          }
        }
        int next = -1;
#pragma unroll
        for (int q = 7; q >= 0; --q)
          if (q > b && h[q]) next = lane * 8 + q;
        if (next < 0 && later) next = nb;
        prefix[j] |= K(lane * 8 + b) << shift;
        rank[j] = r - cum;
        if (p == PASSES - 1 && (n & 1) == 0) {
          if (r - cum + 1 < in_bin) {
            upper[j] = prefix[j];
          } else if (next >= 0) {
            upper[j] = (prefix[j] & ~K(255)) | K(next);
          } else {
            need_upper[j] = 1;
            any_upper = 1;
          }
        }
      }
    }
    __syncthreads();
  }
  if (any_upper) {  // the least key above the lower statistic, for the genes whose upper one is in no later bucket
    if ((int)threadIdx.x < w && need_upper[threadIdx.x])
      upper[threadIdx.x] = (CSR && zeros[threadIdx.x] && key0 > prefix[threadIdx.x]) ? key0 : ~K(0);
    __syncthreads();
    walk_group<T, CSR>(g, x, indptr, indices, data, order, r0, n, c0, w, [&](int j, T v) {
      const K k = to_key(v);
      if (need_upper[j] && k > prefix[j]) atomicMin(&upper[j], k);
    });
    __syncthreads();
  }
  if ((int)threadIdx.x >= w) return;
  const int j = threadIdx.x;
  const T lo = from_key<T>(prefix[j]);
  T med = (n & 1) ? lo : (lo + from_key<T>(upper[j])) / T(2);
  if (!CSR && nan_seen[j]) med = T(NAN);
  out[(int64_t)seg_group[blockIdx.x] * g + c0 + j] = med;
}

template <typename T>
int32_t upload(sb2_ctx* ctx, ScratchScope& scr, const std::vector<T>& h, T** d) {
  SB2_TRY(scr.alloc(d, h.size()));
  if (!h.empty()) SB2_CUDA(cudaMemcpyAsync(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  return SB2_OK;
}

}  // namespace

extern "C" {

int32_t sb2_aggregate_group_order(sb2_ctx* ctx, int64_t n, const int32_t* d_codes, int32_t n_groups,
                                  int64_t* d_order, int64_t* d_offsets) {
  SB2_CHECK_ARG(ctx && d_codes && d_order && d_offsets && n >= 0 && n_groups >= 1, "null pointer");
  SB2_CHECK_ARG(n < INT32_MAX, "at most 2^31 - 1 rows");
  SB2_CUDA(cudaSetDevice(ctx->device));
  // the tile grows until the count table fits its cap
  int64_t tile = GO_TILE;
  while (ceil_div64(n, tile) * n_groups * 4 > GO_HIST_BYTES) tile *= 2;
  const int64_t ntiles = std::max<int64_t>(1, ceil_div64(n, tile));
  ScratchScope scr(ctx);
  int32_t *hist, *counts;
  SB2_TRY(scr.alloc(&hist, (size_t)(ntiles * n_groups)));
  SB2_TRY(scr.alloc(&counts, (size_t)n_groups));
  SB2_CUDA(cudaMemsetAsync(hist, 0, (size_t)(ntiles * n_groups) * 4, ctx->stream));
  if (n > 0) {
    order_count_kernel<<<(unsigned)std::min<int64_t>(ceil_div64(n, 256), 4096), 256, 0, ctx->stream>>>(
        n, tile, n_groups, d_codes, hist);
    SB2_LAUNCH_CHECK(ctx);
  }
  order_base_kernel<<<(unsigned)ceil_div64(n_groups, 256), 256, 0, ctx->stream>>>(ntiles, n_groups, hist, counts);
  SB2_LAUNCH_CHECK(ctx);
  SB2_TRY(sb2_scan_i32_to_i64(ctx, counts, n_groups, d_offsets));
  if (n > 0) {
    order_place_kernel<<<(unsigned)ceil_div64(ntiles, GO_WARPS), GO_WARPS * 32, 0, ctx->stream>>>(
        n, tile, n_groups, d_codes, d_offsets, hist, d_order);
    SB2_LAUNCH_CHECK(ctx);
  }
  return SB2_OK;
}

int32_t sb2_aggregate_moments(sb2_ctx* ctx, int32_t n_seg, const int64_t* h_seg_row, const int32_t* h_seg_group,
                              const int64_t* h_seg_n0, int32_t g, int32_t is_f64, const void* d_x,
                              const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                              const int64_t* d_order, double* d_sum, double* d_mean, double* d_m2, int64_t* d_nnz) {
  SB2_CHECK_ARG(ctx && d_sum && d_mean && d_m2 && d_nnz && g >= 1 && n_seg >= 0, "null pointer");
  SB2_CHECK_ARG(n_seg == 0 || (h_seg_row && h_seg_group && h_seg_n0), "segments");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n_seg == 0) return SB2_OK;
  const int64_t slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(slabs <= 65535, "shape");
  // items of whole subtiles; the partial slots of one launch stay below the scratch cap, and a group whose slots span
  // launches is folded in each launch in turn, so its subtiles still merge in order
  const int64_t max_slots = std::max<int64_t>(1, AG_PARTIAL_BYTES / (4 * 8 * (int64_t)g));
  std::vector<Item> items;
  std::vector<Fold> folds;
  std::vector<int32_t> slot_rows;
  const auto flush = [&]() -> int32_t {
    if (items.empty()) return SB2_OK;
    ScratchScope scr(ctx);
    Item* d_items;
    Fold* d_folds = nullptr;
    int32_t* d_rows = nullptr;
    double* part = nullptr;
    SB2_TRY(upload(ctx, scr, items, &d_items));
    if (!slot_rows.empty()) {
      SB2_TRY(upload(ctx, scr, folds, &d_folds));
      SB2_TRY(upload(ctx, scr, slot_rows, &d_rows));
      SB2_TRY(scr.alloc(&part, slot_rows.size() * 4 * (size_t)g));
    }
    SB2_CHECK_ARG(items.size() < INT32_MAX && folds.size() <= 65535 * 1024, "shape");
    with_types(is_f64, d_x, [&](auto t, auto csr) {
      using T = decltype(t);
      moments_kernel<T, decltype(csr)::value><<<dim3((unsigned)items.size(), (unsigned)slabs), SLAB_THREADS, 0,
                                                 ctx->stream>>>(
          g, static_cast<const T*>(d_x), d_indptr, d_indices, static_cast<const T*>(d_data), d_order, d_items, part,
          d_sum, d_mean, d_m2, d_nnz);
    });
    SB2_LAUNCH_CHECK(ctx);
    if (!folds.empty()) {
      fold_kernel<<<dim3((unsigned)folds.size(), (unsigned)ceil_div64(g, 256)), 256, 0, ctx->stream>>>(
          g, d_folds, d_rows, part, d_sum, d_mean, d_m2, d_nnz);
      SB2_LAUNCH_CHECK(ctx);
    }
    items.clear();
    folds.clear();
    slot_rows.clear();
    return SB2_OK;
  };
  for (int32_t s = 0; s < n_seg; ++s) {
    const int64_t a = h_seg_row[s], e = h_seg_row[s + 1], n0 = h_seg_n0[s];
    const int32_t grp = h_seg_group[s];
    SB2_CHECK_ARG(e > a && n0 >= 0 && n0 % SLAB_TILE == 0 && grp >= 0, "segment rows");
    if (n0 == 0 && e - a <= SLAB_TILE) {
      items.push_back(Item{a, (int32_t)(e - a), grp, -1, 0});
      continue;
    }
    int64_t first = (int64_t)slot_rows.size(), done = n0;
    for (int64_t r = a; r < e; r += SLAB_TILE) {
      if ((int64_t)slot_rows.size() == max_slots) {
        if ((int64_t)slot_rows.size() > first) folds.push_back(Fold{first, (int64_t)slot_rows.size(), done, grp, 0});
        done = n0 + (r - a);
        SB2_TRY(flush());
        first = 0;
      }
      const int32_t m = (int32_t)std::min<int64_t>(SLAB_TILE, e - r);
      items.push_back(Item{r, m, grp, (int32_t)slot_rows.size(), 0});
      slot_rows.push_back(m);
    }
    folds.push_back(Fold{first, (int64_t)slot_rows.size(), done, grp, 0});
  }
  return flush();
}

int32_t sb2_aggregate_median(sb2_ctx* ctx, int32_t n_seg, const int64_t* h_seg_row, const int32_t* h_seg_group,
                             int32_t g, int32_t is_f64, const void* d_x, const int64_t* d_indptr,
                             const int32_t* d_indices, const void* d_data, const int64_t* d_order, void* d_out) {
  SB2_CHECK_ARG(ctx && d_out && g >= 1 && n_seg >= 0, "null pointer");
  SB2_CHECK_ARG(n_seg == 0 || (h_seg_row && h_seg_group), "segments");
  SB2_CHECK_ARG(d_x || (d_indptr && d_indices && d_data), "X: dense block or CSR arrays");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n_seg == 0) return SB2_OK;
  std::vector<int64_t> seg(h_seg_row, h_seg_row + n_seg + 1);
  std::vector<int32_t> grp(h_seg_group, h_seg_group + n_seg);
  for (int32_t s = 0; s < n_seg; ++s)
    SB2_CHECK_ARG(seg[s + 1] > seg[s] && seg[s + 1] - seg[s] < INT32_MAX && grp[s] >= 0, "segment rows");
  const int64_t blocks = ceil_div64(g, MED_GENES);
  SB2_CHECK_ARG(blocks <= 65535, "shape");
  ScratchScope scr(ctx);
  int64_t* d_seg;
  int32_t* d_grp;
  SB2_TRY(upload(ctx, scr, seg, &d_seg));
  SB2_TRY(upload(ctx, scr, grp, &d_grp));
  int32_t rc = SB2_OK;
  with_types(is_f64, d_x, [&](auto t, auto csr) {
    using T = decltype(t);
    const auto kernel = median_kernel<T, decltype(csr)::value>;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MED_SMEM) != cudaSuccess) {
      rc = SB2_E_CUDA;
      return;
    }
    kernel<<<dim3((unsigned)n_seg, (unsigned)blocks), MED_THREADS, MED_SMEM, ctx->stream>>>(
        g, static_cast<const T*>(d_x), d_indptr, d_indices, static_cast<const T*>(d_data), d_order, d_seg, d_grp,
        static_cast<T*>(d_out));
  });
  SB2_CUDA(rc == SB2_OK ? cudaSuccess : cudaGetLastError());
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

// scrublet.cu — the two per-cell passes of
//   sc.pp.scrublet / sc.pp.scrublet_simulate_doublets  (src/scanpy/preprocessing/_scrublet/core.py:188-238, 313-386)
//
// Pair sums: simulated doublet s is the sum of observed rows p0 = pairs[s][0] and p1 = pairs[s][1] of a CSR with sorted,
// unique column indices, as scipy's canonical `x[p0] + x[p1]` forms it: the union of the two index sets in ascending
// order, a fp32 sum where both rows store the column, and entries whose result is 0 dropped (NaN is kept).  One warp
// walks the union of a row pair 32 items at a time: lane l takes item base + l of the merge of the two index lists (ties
// put p0's entry first) by a merge-path binary search, so a column stored in both rows is two adjacent items; the first
// of them emits the sum and the second nothing.  Pass 1 counts the kept entries per row, a scan makes the indptr, pass 2
// writes them at ballot-ranked positions.  Nothing depends on timing, and (i, i) pairs and empty rows need no branch.
//
// Label count: for every point i of d_x [n x d], its neighbour set is i itself plus the k - 1 nearest other points in
// (fp64 squared distance, id) order, where the fp64 squared distance is Σ_j (x_ij - x_cj)² summed over j in order, each
// difference, square and sum rounded separately (no FMA), as a numpy loop over the columns computes it.  The kernel
// returns how many of the k have id >= n_first, the fp64 distance of the (k - 1)-th other neighbour, and optionally the
// set.
//   select: one CTA per 32 query rows (lane = row, so each lane's histogram atomics hit its own row's 256 bins) streams
//           all points through shared memory in tiles of 64 and finds the (k - 1)-th smallest fp32 squared distance key
//           T of each row with four 8-bit radix passes, recomputing the distances in every pass.
//   band:   one more pass counts the points whose fp32 key lies below the band [lo, hi] around T (certainly inside the
//           set) and collects the ids inside the band into a per-row buffer of SC_BAND entries.  DESIGN.md §4 proves
//           that every point of the set lies below hi and every point below lo belongs to the set.
//   resolve: one warp per row re-scores the band in fp64 from the coordinates and takes the missing members by
//           (distance, id).
//   exact:  a row whose band overflows the buffer is redone by the same select kernel on the 96-bit key (fp64 distance
//           bits, id): twelve radix passes find the (k - 1)-th other neighbour itself.
// fp32 squared distances are sums of squared differences (no |q|² + |c|² - 2 q·c cancellation), so the band is a
// relative one, a few units of 1e-5 wide; rows fall back to the exact path only where many points tie at the threshold.
#include <math.h>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------ pair sums
constexpr int PS_WARPS = 8;

// the split of the first p items of the merge of a[0, la) and b[0, lb) (a's entry first on equal values)
__device__ __forceinline__ int merge_split(int64_t p, const int32_t* __restrict__ a, int64_t la,
                                           const int32_t* __restrict__ b, int64_t lb) {
  int64_t lo = p > lb ? p - lb : 0, hi = p < la ? p : la;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] <= b[p - mid - 1]) lo = mid + 1;
    else hi = mid;
  }
  return (int)lo;
}

template <bool FILL>
__global__ void __launch_bounds__(PS_WARPS * 32)
pair_sums_kernel(int64_t n_sim, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                 const float* __restrict__ data, const int64_t* __restrict__ pairs, int32_t* __restrict__ counts,
                 const int64_t* __restrict__ out_indptr, int32_t* __restrict__ out_indices, float* __restrict__ out_data) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * PS_WARPS;
  for (int64_t s = (int64_t)blockIdx.x * PS_WARPS + (threadIdx.x >> 5); s < n_sim; s += warps) {
    const int64_t r0 = pairs[2 * s], r1 = pairs[2 * s + 1];
    const int32_t* a = indices + indptr[r0];
    const int32_t* b = indices + indptr[r1];
    const float* va = data + indptr[r0];
    const float* vb = data + indptr[r1];
    const int64_t la = indptr[r0 + 1] - indptr[r0], lb = indptr[r1 + 1] - indptr[r1];
    int64_t done = 0;
    for (int64_t base = 0; base < la + lb; base += 32) {
      const int64_t p = base + lane;
      bool keep = false;
      int32_t col = 0;
      float v = 0.f;
      if (p < la + lb) {
        const int64_t ia = merge_split(p, a, la, b, lb), ib = p - ia;
        if (ia < la && (ib >= lb || a[ia] <= b[ib])) {  // item p is a[ia]; a following equal b[ib] is added here
          col = a[ia];
          v = (ib < lb && b[ib] == col) ? __fadd_rn(va[ia], vb[ib]) : va[ia];
          keep = v != 0.f;
        } else {  // item p is b[ib]; it was added to a[ia - 1] if that holds the same column
          col = b[ib];
          v = vb[ib];
          keep = !(ia > 0 && a[ia - 1] == col) && v != 0.f;
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (FILL && keep) {
        const int64_t o = out_indptr[s] + done + __popc(m & ((1u << lane) - 1u));
        out_indices[o] = col;
        out_data[o] = v;
      }
      done += __popc(m);
    }
    if (!FILL && lane == 0) counts[s] = (int32_t)done;
  }
}

// ------------------------------------------------------------------------------------------ label count
constexpr int SC_ROWS = 32;                 // query rows per CTA: one per lane
constexpr int SC_WARPS = 8;
constexpr int SC_THREADS = SC_WARPS * 32;
constexpr int SC_CPW = 8;                   // candidates per warp per tile
constexpr int SC_TILE = SC_WARPS * SC_CPW;  // candidates per tile
constexpr int SC_BINS = 256;
constexpr int SC_HSTRIDE = SC_BINS + 1;     // lane l's bin b sits in bank (l + b) % 32
constexpr int SC_BAND = 128;                // band entries kept per row
constexpr int SC_MAX_D = 256;
constexpr int SC_RES_WARPS = 4;             // rows per CTA of the resolve

// fp64 squared distance: differences, squares and sums each rounded (the order a numpy column loop uses)
__device__ __forceinline__ double dist64(const float* __restrict__ q, const float* __restrict__ c, int d) {
  double acc = 0.0;
  for (int j = 0; j < d; ++j) {
    const double t = __dsub_rn((double)q[j], (double)c[j]);
    acc = __dadd_rn(acc, __dmul_rn(t, t));
  }
  return acc;
}

// the 64-bit high part of a row's key to each of the warp's SC_CPW candidates of the tile in shared memory:
// fp32 distance bits << 32 (EXACT = false), or the fp64 distance bits (EXACT = true; the id is the low part)
template <bool EXACT>
__device__ __forceinline__ void tile_keys(const float* __restrict__ q, const float* __restrict__ cs, int d,
                                          uint64_t (&key)[SC_CPW]) {
  if constexpr (EXACT) {
    double acc[SC_CPW];
#pragma unroll
    for (int u = 0; u < SC_CPW; ++u) acc[u] = 0.0;
    for (int j = 0; j < d; ++j) {
      const double qv = (double)q[j];
#pragma unroll
      for (int u = 0; u < SC_CPW; ++u) {
        const double t = __dsub_rn(qv, (double)cs[u * d + j]);
        acc[u] = __dadd_rn(acc[u], __dmul_rn(t, t));
      }
    }
#pragma unroll
    for (int u = 0; u < SC_CPW; ++u) key[u] = (uint64_t)__double_as_longlong(acc[u]);
  } else {
    float acc[SC_CPW];
#pragma unroll
    for (int u = 0; u < SC_CPW; ++u) acc[u] = 0.f;
    for (int j = 0; j < d; ++j) {
      const float qv = q[j];
#pragma unroll
      for (int u = 0; u < SC_CPW; ++u) {
        const float t = __fsub_rn(qv, cs[u * d + j]);
        acc[u] = __fmaf_rn(t, t, acc[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < SC_CPW; ++u) key[u] = (uint64_t)__float_as_uint(acc[u]) << 32;
  }
}

// does (hi, id) share the first 8p bits of the selected prefix (hp, ip)?  p counts 8-bit digits, hi first.
__device__ __forceinline__ bool prefix_match(int p, uint64_t hi, uint32_t id, uint64_t hp, uint32_t ip) {
  if (p == 0) return true;
  if (p <= 8) return (hi >> (64 - 8 * p)) == (hp >> (64 - 8 * p));
  return hi == hp && (p == 8 || (id >> (32 - 8 * (p - 8))) == (ip >> (32 - 8 * (p - 8))));
}
__device__ __forceinline__ int digit(int p, uint64_t hi, uint32_t id) {
  return p < 8 ? (int)((hi >> (56 - 8 * p)) & 255u) : (int)((id >> (24 - 8 * (p - 8))) & 255u);
}

struct SelectOut {
  // fp32 mode: the rows' certain-inside counts and band lists
  int32_t* in_cnt;
  int32_t* in_lab;
  int32_t* band_cnt;
  int32_t* band;
  // exact mode: the final results
  int32_t* count;
  double* kth;
};

// One CTA per SC_ROWS query rows (rows[] maps CTA rows to points; NULL: the identity).  EXACT = false: four passes on the
// fp32 keys, then the band pass.  EXACT = true: twelve passes on (fp64 key, id), then the membership pass.
template <bool EXACT>
__global__ void __launch_bounds__(SC_THREADS)
select_kernel(int64_t n, int d, const float* __restrict__ x, const int32_t* __restrict__ rows, int64_t n_rows,
              int64_t n_first, int k, SelectOut out, int32_t* __restrict__ ids) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int qstride = d | 1;  // odd: lane l's reads of column j fall in distinct banks
  uint32_t* hist = reinterpret_cast<uint32_t*>(smem);
  uint64_t* pref_hi = reinterpret_cast<uint64_t*>(hist + SC_ROWS * SC_HSTRIDE);  // SC_ROWS * SC_HSTRIDE is even
  double* lo = reinterpret_cast<double*>(pref_hi + SC_ROWS);
  double* hi = lo + SC_ROWS;
  uint32_t* pref_id = reinterpret_cast<uint32_t*>(hi + SC_ROWS);
  int32_t* want = reinterpret_cast<int32_t*>(pref_id + SC_ROWS);
  int32_t* cnt_in = want + SC_ROWS;
  int32_t* cnt_lab = cnt_in + SC_ROWS;
  int32_t* cnt_band = cnt_lab + SC_ROWS;
  float* qs = reinterpret_cast<float*>(cnt_band + SC_ROWS);
  float* cs = qs + SC_ROWS * qstride;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * SC_ROWS;
  const bool valid = r0 + lane < n_rows;
  const int64_t me = valid ? (rows ? (int64_t)rows[r0 + lane] : r0 + lane) : -1;
  for (int i = threadIdx.x; i < SC_ROWS * d; i += SC_THREADS) {
    const int r = i / d, j = i % d;
    const int64_t pr = r0 + r < n_rows ? (rows ? (int64_t)rows[r0 + r] : r0 + r) : 0;
    qs[r * qstride + j] = x[pr * d + j];
  }
  if (threadIdx.x < SC_ROWS) {
    pref_hi[threadIdx.x] = 0;
    pref_id[threadIdx.x] = 0;
    want[threadIdx.x] = k - 1;
    cnt_in[threadIdx.x] = cnt_lab[threadIdx.x] = cnt_band[threadIdx.x] = 0;
  }
  const float* q = qs + lane * qstride;
  const int passes = EXACT ? 12 : 4;

  // passes 0 .. passes-1 select a digit each; the last trip (p == passes) classifies the points
  for (int p = 0; p <= passes; ++p) {
    for (int i = threadIdx.x; i < SC_ROWS * SC_HSTRIDE; i += SC_THREADS) hist[i] = 0;
    __syncthreads();
    const uint64_t hp = pref_hi[lane];
    const uint32_t ip = pref_id[lane];
    if (!EXACT && p == passes && warp == 0) {
      // the band around T (DESIGN.md §4): E = 2 (d + 2) u / (1 - (d + 2) u) with u = 2^-24, A = 2^-140 for underflow;
      // the factors 1 -+ 2^-50 cover the rounding of these few fp64 operations
      const double T = (double)__uint_as_float((uint32_t)(hp >> 32));
      const double u = ldexp(1.0, -24), E = 2.0 * (d + 2) * u / (1.0 - (d + 2) * u), A = ldexp(1.0, -140);
      lo[lane] = ((T - A) * (1.0 - E) - A) * (1.0 - E) * (1.0 - ldexp(1.0, -50));
      hi[lane] = ((1.0 + E) * ((1.0 + E) * T + A) + A) * (1.0 + ldexp(1.0, -50));
    }
    __syncthreads();
    const double my_lo = lo[lane], my_hi = hi[lane];
    int my_in = 0, my_lab = 0;
    for (int64_t t0 = 0; t0 < n; t0 += SC_TILE) {
      const int tn = n - t0 < SC_TILE ? (int)(n - t0) : SC_TILE;
      __syncthreads();
      for (int i = threadIdx.x; i < tn * d; i += SC_THREADS) cs[i] = x[t0 * d + i];
      __syncthreads();
      if (!valid) continue;
      const int c0 = warp * SC_CPW;
      if (c0 >= tn) continue;
      uint64_t key[SC_CPW];
      tile_keys<EXACT>(q, cs + c0 * d, d, key);
#pragma unroll
      for (int u = 0; u < SC_CPW; ++u) {
        const int64_t c = t0 + c0 + u;
        if (c0 + u >= tn || c == me) continue;
        const uint32_t cid = (uint32_t)c;
        if (p < passes) {
          if (prefix_match(p, key[u], cid, hp, ip)) atomicAdd(&hist[lane * SC_HSTRIDE + digit(p, key[u], cid)], 1u);
        } else if (EXACT) {
          if (key[u] < hp || (key[u] == hp && cid <= ip)) {  // (distance, id) <= the (k-1)-th: inside
            const int slot = atomicAdd(&cnt_in[lane], 1);
            my_lab += c >= n_first;
            if (ids) ids[me * (int64_t)k + 1 + slot] = (int32_t)c;
          }
        } else {
          const double v = (double)__uint_as_float((uint32_t)(key[u] >> 32));
          if (v < my_lo) {
            ++my_in;
            my_lab += c >= n_first;
            if (ids) ids[me * (int64_t)k + 1 + atomicAdd(&cnt_in[lane], 1)] = (int32_t)c;
          } else if (v <= my_hi) {
            const int slot = atomicAdd(&cnt_band[lane], 1);
            if (slot < SC_BAND) out.band[me * (int64_t)SC_BAND + slot] = (int32_t)c;
          }
        }
      }
    }
    if (p == passes) {
      if (valid) atomicAdd(&cnt_lab[lane], my_lab);
      if (!EXACT && valid && !ids) atomicAdd(&cnt_in[lane], my_in);
      break;
    }
    __syncthreads();
    if (threadIdx.x < SC_ROWS && valid) {  // the digit holding the want-th smallest key among the prefix's points
      const uint32_t* h = hist + threadIdx.x * SC_HSTRIDE;
      int w = want[threadIdx.x], b = 0;
      while (b < SC_BINS - 1 && (int)h[b] < w) w -= (int)h[b++];
      want[threadIdx.x] = w;
      if (p < 8) pref_hi[threadIdx.x] |= (uint64_t)b << (56 - 8 * p);
      else pref_id[threadIdx.x] |= (uint32_t)b << (24 - 8 * (p - 8));
    }
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x < SC_ROWS && valid) {
    if (EXACT) {
      out.count[me] = cnt_lab[threadIdx.x] + (me >= n_first);
      out.kth[me] = sqrt(__longlong_as_double((long long)pref_hi[threadIdx.x]));
      if (ids) ids[me * (int64_t)k] = (int32_t)me;
    } else {
      out.in_cnt[me] = cnt_in[threadIdx.x];
      out.in_lab[me] = cnt_lab[threadIdx.x];
      out.band_cnt[me] = cnt_band[threadIdx.x];
    }
  }
}

// One warp per row: the band's members by (fp64 distance, id) complete the set; rows whose band overflowed (or, which
// the bound excludes, does not hold the missing members) go to the exact list.
__global__ void __launch_bounds__(SC_RES_WARPS * 32)
resolve_kernel(int64_t n, int d, const float* __restrict__ x, int64_t n_first, int k, SelectOut out,
               int32_t* __restrict__ ids, int32_t* __restrict__ exact_rows, int32_t* __restrict__ n_exact) {
  __shared__ double bd[SC_RES_WARPS][SC_BAND];
  __shared__ int32_t bi[SC_RES_WARPS][SC_BAND];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * SC_RES_WARPS + warp;
  if (i >= n) return;
  const int c_in = out.in_cnt[i], m = out.band_cnt[i], need = k - 1 - c_in;
  if (m > SC_BAND || need < 1 || need > m) {
    if (lane == 0) exact_rows[atomicAdd(n_exact, 1)] = (int32_t)i;
    return;
  }
  for (int e = lane; e < m; e += 32) {
    const int32_t c = out.band[i * SC_BAND + e];
    bi[warp][e] = c;
    bd[warp][e] = dist64(x + i * d, x + (int64_t)c * d, d);
  }
  __syncwarp();
  int lab = 0;
  for (int e = lane; e < m; e += 32) {
    const double de = bd[warp][e];
    const int32_t ce = bi[warp][e];
    int rank = 0;
    for (int f = 0; f < m; ++f) {
      const double df = bd[warp][f];
      rank += df < de || (df == de && bi[warp][f] < ce);
    }
    if (rank < need) {
      lab += ce >= n_first;
      if (ids) ids[i * (int64_t)k + 1 + c_in + rank] = ce;
    }
    if (rank == need - 1) out.kth[i] = sqrt(de);
  }
  lab = warp_sum(lab);
  if (lane == 0) {
    out.count[i] = (i >= n_first) + out.in_lab[i] + lab;
    if (ids) ids[i * (int64_t)k] = (int32_t)i;
  }
}

// k == 1: the set is the point itself
__global__ void self_only_kernel(int64_t n, int64_t n_first, int32_t* __restrict__ count, double* __restrict__ kth,
                                 int32_t* __restrict__ ids) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    count[i] = i >= n_first;
    kth[i] = 0.0;
    if (ids) ids[i] = (int32_t)i;
  }
}

// flags a coordinate that is not finite or exceeds 2^55 in magnitude (the fp32 squared distances must not overflow)
__global__ void range_kernel(int64_t m, const float* __restrict__ x, int32_t* __restrict__ bad) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x)
    if (!(fabsf(x[i]) <= 0x1p55f)) *bad = 1;
}

size_t select_smem(int d) {
  return (size_t)(SC_ROWS * SC_HSTRIDE) * 4 + SC_ROWS * (8 + 8 + 8 + 4 + 4 * 4) +
         (size_t)(SC_ROWS * (d | 1) + SC_TILE * d) * 4;
}

template <bool EXACT>
int32_t launch_select(sb2_ctx* ctx, int64_t n, int d, const float* d_x, const int32_t* rows, int64_t n_rows,
                      int64_t n_first, int k, const SelectOut& out, int32_t* ids) {
  const size_t smem = select_smem(d);
  SB2_CUDA(cudaFuncSetAttribute(select_kernel<EXACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  select_kernel<EXACT><<<(unsigned)ceil_div64(n_rows, SC_ROWS), SC_THREADS, smem, ctx->stream>>>(
      n, d, d_x, rows, n_rows, n_first, k, out, ids);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // namespace

extern "C" {

int32_t sb2_scrublet_pair_sums(sb2_ctx* ctx, int64_t n_obs, const int64_t* d_indptr, const int32_t* d_indices,
                               const float* d_data, int64_t n_sim, const int64_t* d_pairs, int64_t* d_out_indptr,
                               int32_t* d_out_indices, float* d_out_data) {
  SB2_CHECK_ARG(ctx && d_indptr && d_pairs && d_out_indptr && n_obs >= 1 && n_sim >= 0, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  int32_t* counts;
  SB2_TRY(scr.alloc(&counts, (size_t)n_sim));
  const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(n_sim, PS_WARPS), 65536));
  if (n_sim > 0) {
    pair_sums_kernel<false><<<grid, PS_WARPS * 32, 0, ctx->stream>>>(n_sim, d_indptr, d_indices, d_data, d_pairs,
                                                                     counts, nullptr, nullptr, nullptr);
    SB2_LAUNCH_CHECK(ctx);
  }
  SB2_TRY(sb2_scan_i32_to_i64(ctx, counts, n_sim, d_out_indptr));
  if (n_sim > 0) {
    pair_sums_kernel<true><<<grid, PS_WARPS * 32, 0, ctx->stream>>>(n_sim, d_indptr, d_indices, d_data, d_pairs,
                                                                    nullptr, d_out_indptr, d_out_indices, d_out_data);
    SB2_LAUNCH_CHECK(ctx);
  }
  return SB2_OK;
}

int32_t sb2_knn_label_count_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int64_t n_first,
                                int32_t k, int32_t* d_count, double* d_kth, int32_t* d_ids) {
  SB2_CHECK_ARG(ctx && d_x && d_count && d_kth, "null pointer");
  SB2_CHECK_ARG(n_points >= 1 && n_points < INT32_MAX, "1 <= n_points < 2^31");
  SB2_CHECK_ARG(d >= 1 && d <= SC_MAX_D, "1 <= d <= 256");
  SB2_CHECK_ARG(k >= 1 && k <= n_points, "1 <= k <= n_points");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  int32_t* flags;  // [0]: out-of-range coordinate, [1]: rows on the exact path
  SB2_TRY(scr.alloc(&flags, 2));
  SB2_CUDA(cudaMemsetAsync(flags, 0, 8, ctx->stream));
  range_kernel<<<(unsigned)std::min<int64_t>(ceil_div64(n_points * d, 256), 4096), 256, 0, ctx->stream>>>(
      n_points * d, d_x, flags);
  SB2_LAUNCH_CHECK(ctx);
  int32_t h_bad = 0;
  SB2_CUDA(cudaMemcpyAsync(&h_bad, flags, 4, cudaMemcpyDeviceToHost, ctx->stream));
  SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  SB2_CHECK_ARG(h_bad == 0, "coordinates must be finite and at most 2^55 in magnitude");
  if (k == 1) {
    self_only_kernel<<<(unsigned)std::min<int64_t>(ceil_div64(n_points, 256), 4096), 256, 0, ctx->stream>>>(
        n_points, n_first, d_count, d_kth, d_ids);
    SB2_LAUNCH_CHECK(ctx);
    return SB2_OK;
  }
  SelectOut out{};
  SB2_TRY(scr.alloc(&out.in_cnt, (size_t)n_points));
  SB2_TRY(scr.alloc(&out.in_lab, (size_t)n_points));
  SB2_TRY(scr.alloc(&out.band_cnt, (size_t)n_points));
  SB2_TRY(scr.alloc(&out.band, (size_t)n_points * SC_BAND));
  int32_t* exact_rows;
  SB2_TRY(scr.alloc(&exact_rows, (size_t)n_points));
  out.count = d_count;
  out.kth = d_kth;
  SB2_TRY(launch_select<false>(ctx, n_points, d, d_x, nullptr, n_points, n_first, k, out, d_ids));
  resolve_kernel<<<(unsigned)ceil_div64(n_points, SC_RES_WARPS), SC_RES_WARPS * 32, 0, ctx->stream>>>(
      n_points, d, d_x, n_first, k, out, d_ids, exact_rows, flags + 1);
  SB2_LAUNCH_CHECK(ctx);
  int32_t h_exact = 0;
  SB2_CUDA(cudaMemcpyAsync(&h_exact, flags + 1, 4, cudaMemcpyDeviceToHost, ctx->stream));
  SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  if (h_exact > 0) SB2_TRY(launch_select<true>(ctx, n_points, d, d_x, exact_rows, h_exact, n_first, k, out, d_ids));
  return SB2_OK;
}

}  // extern "C"

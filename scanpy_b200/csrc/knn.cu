// knn.cu — exact brute-force euclidean kNN on the n x d float32 embedding (sm_90a).
//
// Replaces sklearn's KNeighborsTransformer(algorithm='brute') as built by the reference at
// src/scanpy/neighbors/__init__.py:754-768 (ArgKmin: GEMM-shaped middle term with fp64
// accumulation + per-row heaps).  Pipeline:
//
//   knn_prep_kernel     X[n,d] row-major  ->  Xt: tiles of 128 points, k-major [d+1][128]; the extra
//                       row holds hn_j = -|x_j|^2/2, so one 1-D bulk (TMA) copy stages a whole tile.
//   knn_pass1_kernel    CTA = 128 queries, sweeps all candidate tiles through a 3-stage
//                       cp.async.bulk + mbarrier ring.  8 compute warps, each owns 16 query rows
//                       exclusively; a lane's register micro-tile is 16 queries x 4 candidates
//                       (64 FFMA per k-step).  score = q.c - |c|^2/2 (larger = closer; d^2 = |q|^2 - 2 score)
//                       lands in the accumulators with no epilogue arithmetic (accumulators start
//                       at hn).  Per query row the warp keeps the best 32 scores as a sorted list
//                       distributed over its lanes (one entry per lane, in registers); a candidate
//                       is examined only if it beats the row's current 32nd best (one FSETP per
//                       element + one ballot per row and tile; insertions are O(32 ln n) per row).
//   knn_rescore_kernel  warp per query: exact fp64 |q-c|^2 of the 32 proposals, warp bitonic sort by
//                       (d^2, id), self forced to column 0, top-k out.  Certificate: every point
//                       not proposed has fp32 score <= s32, hence true d^2 >= |q|^2 - 2 (s32 + eps);
//                       if the exact k-th d^2 is below that bound the row is provably exact.
//   knn_fallback_kernel rows without a certificate (ties, duplicates, pathological scales) are
//                       recomputed exactly in fp64 against all points.
#include <float.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "knn_internal.cuh"

namespace {

constexpr int TILE = 128;      // points per tile (queries per CTA, candidates per stage)
constexpr int LISTM = 32;      // proposals kept per query (one per lane)
constexpr int NWARP_C = 8;     // compute warps
constexpr int PASS1_THREADS = (NWARP_C + 1) * 32;

// ------------------------------------------------------------------------------------------------
__global__ void knn_prep_kernel(const float* __restrict__ X, int64_t n, int d, float* __restrict__ Xt,
                                unsigned int* __restrict__ maxnorm_bits) {
  extern __shared__ float s[];  // [128][d] staged chunk
  const int64_t t = blockIdx.x;
  const int64_t p0 = t * TILE;
  const int rows = (n - p0 < TILE) ? (int)(n - p0) : TILE;
  const float* src = X + p0 * d;
  for (int i = threadIdx.x; i < TILE * d; i += blockDim.x) s[i] = (i < rows * d) ? src[i] : 0.0f;
  __syncthreads();
  float* dst = Xt + t * (int64_t)(d + 1) * TILE;
  for (int i = threadIdx.x; i < TILE * d; i += blockDim.x) {
    int k = i / TILE, j = i % TILE;
    dst[i] = s[j * d + k];
  }
  if (threadIdx.x < TILE) {
    int j = threadIdx.x;
    double acc = 0.0;
    for (int k = 0; k < d; ++k) {
      double v = s[j * d + k];
      acc += v * v;
    }
    float hn = (j < rows) ? (float)(-0.5 * acc) : -INFINITY;
    dst[d * TILE + j] = hn;
    if (j < rows) atomicMax(maxnorm_bits, __float_as_uint((float)acc * (1.0f + 1e-6f)));
  }
}

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D bulk async copy global -> shared (TMA engine, SASS UBLKCP), completion on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

template <int NST>
__global__ void __launch_bounds__(PASS1_THREADS, 1)
knn_pass1_kernel(const float* __restrict__ Xt, int d, int64_t n_tiles, int64_t qtile0, int64_t n_query,
                 float* __restrict__ cand_score, int32_t* __restrict__ cand_idx) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int chunk_f = (d + 1) * TILE;              // floats per tile chunk
  const uint32_t chunk_b = (uint32_t)chunk_f * 4u;  // bytes (multiple of 512)
  float* As = reinterpret_cast<float*>(smem_raw);
  float* Bs0 = As + chunk_f;
  uint64_t* bars = reinterpret_cast<uint64_t*>(Bs0 + (size_t)NST * chunk_f);
  uint64_t* full = bars;            // [NST]
  uint64_t* empty = bars + NST;     // [NST]
  uint64_t* afull = bars + 2 * NST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NST; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NWARP_C);
    }
    mbar_init(afull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int64_t qt = qtile0 + blockIdx.x;
  if (warp == NWARP_C) {
    // ---------------- producer warp: one elected lane drives the bulk-copy ring ----------------
    if (lane == 0) {
      mbar_expect_tx(afull, chunk_b);
      bulk_g2s(As, Xt + qt * chunk_f, chunk_b, afull);
      for (int64_t c = 0; c < n_tiles; ++c) {
        const int s = (int)(c % NST);
        const int64_t use = c / NST;
        if (use > 0) mbar_wait(&empty[s], (uint32_t)((use - 1) & 1));
        mbar_expect_tx(&full[s], chunk_b);
        bulk_g2s(Bs0 + (size_t)s * chunk_f, Xt + c * chunk_f, chunk_b, &full[s]);
      }
    }
    return;
  }

  // ---------------- compute warps ----------------
  float lv[16];
  int32_t li[16];
  float th[16];
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    lv[r] = -INFINITY;
    li[r] = -1;
    th[r] = -INFINITY;
  }
  mbar_wait(afull, 0);
  const float* Aw = As + 16 * warp;

  for (int64_t c = 0; c < n_tiles; ++c) {
    const int s = (int)(c % NST);
    mbar_wait(&full[s], (uint32_t)((c / NST) & 1));
    const float* Bs = Bs0 + (size_t)s * chunk_f + 4 * lane;

    float acc[16][4];
    {
      const float4 h = *reinterpret_cast<const float4*>(Bs + d * TILE);
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        acc[r][0] = h.x; acc[r][1] = h.y; acc[r][2] = h.z; acc[r][3] = h.w;
      }
    }
#pragma unroll 2
    for (int k = 0; k < d; ++k) {
      const float4 b = *reinterpret_cast<const float4*>(Bs + k * TILE);
      const float4 a0 = *reinterpret_cast<const float4*>(Aw + k * TILE);
      const float4 a1 = *reinterpret_cast<const float4*>(Aw + k * TILE + 4);
      const float4 a2 = *reinterpret_cast<const float4*>(Aw + k * TILE + 8);
      const float4 a3 = *reinterpret_cast<const float4*>(Aw + k * TILE + 12);
      const float a[16] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w,
                           a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        acc[r][0] = fmaf(a[r], b.x, acc[r][0]);
        acc[r][1] = fmaf(a[r], b.y, acc[r][1]);
        acc[r][2] = fmaf(a[r], b.z, acc[r][2]);
        acc[r][3] = fmaf(a[r], b.w, acc[r][3]);
      }
    }
    // release the stage as early as possible (all smem reads of this stage are done)
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);

    const int32_t base = (int32_t)(c * TILE);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const bool any = (acc[r][0] > th[r]) | (acc[r][1] > th[r]) | (acc[r][2] > th[r]) | (acc[r][3] > th[r]);
      if (__ballot_sync(0xffffffffu, any)) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          unsigned mj = __ballot_sync(0xffffffffu, acc[r][j] > th[r]);
          while (mj) {
            const int src = __ffs(mj) - 1;
            mj &= mj - 1;
            const float v = __shfl_sync(0xffffffffu, acc[r][j], src);
            if (v > th[r]) {  // warp-uniform: th may have risen since the ballot
              const int32_t id = base + 4 * src + j;
              const int pos = __popc(__ballot_sync(0xffffffffu, lv[r] >= v));
              const float up_v = __shfl_up_sync(0xffffffffu, lv[r], 1);
              const int32_t up_i = __shfl_up_sync(0xffffffffu, li[r], 1);
              if (lane > pos) { lv[r] = up_v; li[r] = up_i; }
              else if (lane == pos) { lv[r] = v; li[r] = id; }
              th[r] = __shfl_sync(0xffffffffu, lv[r], 31);
            }
          }
        }
      }
    }
  }

  // proposals out: row-major [n_query][32], lane = rank (0 = best)
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    const int64_t q = (int64_t)blockIdx.x * TILE + 16 * warp + r;
    if (q < n_query) {
      cand_score[q * LISTM + lane] = lv[r];
      cand_idx[q * LISTM + lane] = li[r];
    }
  }
}

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool lex_less(double ka, int ia, double kb, int ib) {
  return ka < kb || (ka == kb && ia < ib);
}

// R = proposals per lane: the list has 32*R entries.  The list is made of sub-lists of `sub` consecutive slots (sub = 32*R
// for a single list; the second-generation tensor sweep keeps four sub-lists per row, one per column quarter of a
// tile).  Every sub-list covers a disjoint part of the candidates and its smallest stored score (a real proposal or
// the sentinel it started from) bounds the score of every candidate of that part that is NOT in it; hence no
// unproposed candidate scored above tau = max over sub-lists of their minima.
template <int R>
__global__ void knn_rescore_kernel(const float* __restrict__ X, int64_t n_points, int d, int64_t q0, int64_t ql_base,
                                   const int32_t* __restrict__ row_map, int64_t n_rows,
                                   int k, int sub, const float* __restrict__ cand_score, const int32_t* __restrict__ cand_idx,
                                   const unsigned int* __restrict__ maxnorm_bits, const float* __restrict__ inv_s2,
                                   double c_q, double c_n, const float* __restrict__ dnorm,
                                   const unsigned int* __restrict__ dmax_bits, const int32_t* __restrict__ cand_map,
                                   const float* __restrict__ ubound, int32_t* __restrict__ idx_out,
                                   double* __restrict__ dist_out, int32_t* __restrict__ work_q,
                                   double* __restrict__ work_ub, unsigned long long* __restrict__ work_cnt) {
  constexpr int LM = 32 * R;
  const int lane = threadIdx.x & 31;
  // launch row i holds the proposals of local query ql (= row_map[i] for a gathered re-sweep, else ql_base + i);
  // outputs and queue entries are indexed by ql, the point itself is q0 + ql
  const int64_t li = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (li >= n_rows) return;
  const int64_t ql = row_map ? (int64_t)row_map[li] : ql_base + li;
  const int64_t q = q0 + ql;
  const float* xq = X + q * d;
  double key[R];
  int32_t id[R];
  float cs[R];
  double qn = 0.0;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    int32_t ci = cand_idx[li * LM + r * 32 + lane];
    if (cand_map && ci >= 0) ci = cand_map[ci];   // image position -> point
    cs[r] = cand_score[li * LM + r * 32 + lane];  // unused slots hold the sweep's starting threshold (-inf for a cold start)
    const float* xc = X + (int64_t)(ci < 0 ? 0 : ci) * d;
    double acc = 0.0, qq = 0.0;
    for (int j = 0; j < d; ++j) {
      const double a = xq[j];
      const double df = a - (double)xc[j];
      acc = fma(df, df, acc);
      qq = fma(a, a, qq);
    }
    qn = qq;
    key[r] = ci < 0 ? DBL_MAX : ((ci == q) ? -1.0 : acc);
    id[r] = ci < 0 ? INT32_MAX : ci;
  }
  // tau = max over sub-lists of (min over the sub-list's slots)
  float tau = -INFINITY;
  if (sub >= 32) {
    const int regs_per = sub >> 5;
#pragma unroll
    for (int r0 = 0; r0 < R; ++r0) {
      if (r0 % regs_per == 0) {
        float m = INFINITY;
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (r >= r0 && r < r0 + regs_per) m = fminf(m, cs[r]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
        tau = fmaxf(tau, m);
      }
    }
  } else {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float m = cs[r];
      for (int o = sub >> 1; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));   // min inside the sub-list's lanes
      for (int o = 16; o >= sub; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));      // max across the sub-lists of this register
      tau = fmaxf(tau, m);
    }
  }
  // bitonic sort of the 32*R elements (element e = r*32 + lane) ascending by (key, id)
#pragma unroll
  for (int kk = 2; kk <= LM; kk <<= 1) {
#pragma unroll
    for (int j = kk >> 1; j > 0; j >>= 1) {
      if (j >= 32) {  // partner lives in the same lane, register r ^ (j / 32)
        const int rj = j >> 5;
#pragma unroll
        for (int r = 0; r < R; ++r) {
          if ((r & rj) == 0 && (r | rj) < R) {
            const int r2 = r | rj;
            const bool asc = ((r * 32) & kk) == 0;
            const bool swap = asc ? lex_less(key[r2], id[r2], key[r], id[r]) : lex_less(key[r], id[r], key[r2], id[r2]);
            if (swap) {
              const double tk = key[r]; key[r] = key[r2]; key[r2] = tk;
              const int32_t ti = id[r]; id[r] = id[r2]; id[r2] = ti;
            }
          }
        }
      } else {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int e = r * 32 + lane;
          const double ok = __shfl_xor_sync(0xffffffffu, key[r], j);
          const int32_t oi = __shfl_xor_sync(0xffffffffu, id[r], j);
          const bool want_min = ((e & j) == 0) == ((e & kk) == 0);
          const bool other_less = lex_less(ok, oi, key[r], id[r]);
          const bool take = want_min ? other_less : lex_less(key[r], id[r], ok, oi);
          if (take) { key[r] = ok; id[r] = oi; }
        }
      }
    }
  }
  // the query itself must sit in column 0 (src/scanpy/neighbors/_common.py:74-98); if it was not proposed at
  // all (a flood of exact duplicates can push it out of the list) the row is not certified.
  const bool self_first = __shfl_sync(0xffffffffu, id[0], 0) == (int32_t)q;
  double kth = 0.0;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const double t = __shfl_sync(0xffffffffu, key[r], (k - 1) & 31);
    if (r == ((k - 1) >> 5)) kth = t;
  }
  bool certified;
  if (tau == -INFINITY) {
    certified = true;  // cold start and no sub-list ever filled: the proposal list is the whole data set
  } else {
    const double Rn = sqrt((double)__uint_as_float(*maxnorm_bits));
    double eps = c_n * 0.5 * Rn * Rn + c_q * sqrt(qn) * Rn;
    if (dnorm) {  // fp16 tier: |q.c - q_hi.c_hi| <= |dq| R + (|q| + |dq|) max|dc|
      const double dq = (double)dnorm[q], dc = (double)__uint_as_float(*dmax_bits);
      eps += (dq * Rn + (sqrt(qn) + dq) * dc) * (1.0 + 1e-6);
    }
    const double bound = qn - 2.0 * ((double)tau * (inv_s2 ? (double)*inv_s2 : 1.0) + eps);
    certified = self_first && (kth < bound);
    if (inv_s2) {
      // the tensor-path bounds are derived for a scaled largest norm in [100, 200) (the prep kernel's power-of-two
      // scale); data so tiny or so huge that the clamped scale cannot reach it (largest norm below ~1e-16 or above
      // ~2e20) is left to the exact scan.  Also catches non-finite scores.
      const double r2s2 = Rn * Rn / (double)*inv_s2;
      if (!(r2s2 >= 9801.0 && r2s2 <= 67600.0)) certified = false;
    }
  }
  // tile screen: the sweep skipped tiles with no point within ubound[li] of the row, so the row's k-th distance must be
  // below it (with a margin far above the fp64 rounding of any squared distance)
  if (ubound) {
    const double u = (double)ubound[li];
    certified = certified && kth <= u * u * (1.0 - 1e-9);
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int e = r * 32 + lane;
    if (e < k) {
      idx_out[ql * k + e] = id[r];
      dist_out[ql * k + e] = key[r] < 0.0 ? 0.0 : sqrt(key[r]);
    }
  }
  if (!certified && lane == 0) {
    const unsigned long long w = atomicAdd(work_cnt, 1ull);
    work_q[w] = (int32_t)ql;
    work_ub[w] = self_first ? kth : DBL_MAX;
  }
}


// Tile screen, per launch row li (local row row_map[li]) after the short sweep of its block's own neighbourhood: at
// least k proposals scored s_k or more, each with a true score >= s_k - eps (the fp16 tier's bound), so
//   u^2 = |q|^2 - 2 (s_k - eps) >= d_k^2                                          -> ub[li] (rounded up)
//   seed[li] = ((|q|^2 - u^2) / 2 - eps) / inv_s2: every point within u scores above it  (scaled units, rounded down)
//   rowp[li] = (qlb, u s): qlb = (|q|^2 - 2 eps_c - slack) s^2, eps_c the bound for the centre image (exact fp16 centres:
//              no |dc| term), slack 2^-19 (|q| + R)^2 s^2 covers the screen's fp32 arithmetic
// Fewer than k proposals: u = +inf.  Rows n_rows <= li < n_pad (padding of the last block): rowp = (+inf, 0).
template <int R>
__global__ void knn_row_bound_kernel(const float* __restrict__ X, int d, int64_t q0, const int32_t* __restrict__ row_map, int64_t n_rows,
                                     int64_t n_pad, int k, const float* __restrict__ cand_score, const int32_t* __restrict__ cand_idx,
                                     const unsigned int* __restrict__ maxnorm_bits, const float* __restrict__ inv_s2, double c_q,
                                     double c_n, const float* __restrict__ dnorm, const unsigned int* __restrict__ dmax_bits,
                                     float* __restrict__ ub, float* __restrict__ seed, float2* __restrict__ rowp) {
  constexpr int LM = 32 * R;
  const int lane = threadIdx.x & 31;
  const int64_t li = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (li >= n_pad) return;
  if (li >= n_rows) {
    if (lane == 0) rowp[li] = make_float2(INFINITY, 0.0f);
    return;
  }
  const int64_t q = q0 + row_map[li];
  double qq = 0.0;
  for (int j = lane; j < d; j += 32) {
    const double a = X[q * d + j];
    qq = fma(a, a, qq);
  }
  const double qn = warp_sum(qq);
  uint32_t kb[R];
  int valid = 0;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const bool ok = cand_idx[li * LM + r * 32 + lane] >= 0;
    kb[r] = ok ? ord_bits(cand_score[li * LM + r * 32 + lane]) : 0u;
    valid += ok;
  }
  valid = __reduce_add_sync(0xffffffffu, (unsigned)valid);
  // the k-th largest proposal score: the largest t with #{kb >= t} >= k
  uint32_t t = 0u;
  for (int bit = 31; bit >= 0; --bit) {
    const uint32_t cand = t | (1u << bit);
    int c = 0;
#pragma unroll
    for (int r = 0; r < R; ++r) c += kb[r] >= cand;
    if ((int)__reduce_add_sync(0xffffffffu, (unsigned)c) >= k) t = cand;
  }
  const double s2inv = (double)*inv_s2, s2 = 1.0 / s2inv;
  const double Rn = sqrt((double)__uint_as_float(*maxnorm_bits)), qnorm = sqrt(qn);
  const double dq = (double)dnorm[q], dc = (double)__uint_as_float(*dmax_bits);
  const double eps_c = c_n * 0.5 * Rn * Rn + c_q * qnorm * Rn + dq * Rn * (1.0 + 1e-6);
  const double eps = eps_c + (qnorm + dq) * dc * (1.0 + 1e-6);
  const float sk = from_ord_bits(t);
  float u = INFINITY, sd = -INFINITY;
  if (valid >= k && isfinite(sk) && isfinite(qn)) {
    const double u2 = qn - 2.0 * ((double)sk * s2inv - eps);
    u = __double2float_ru(sqrt(fmax(u2, 0.0)) * (1.0 + 1e-7));
    const double sdd = ((qn - (double)u * (double)u) * 0.5 - eps) * s2;
    sd = __double2float_rd(sdd - fabs(sdd) * 1e-6);
  }
  if (lane == 0) {
    ub[li] = u;
    seed[li] = sd;
    const double slack = 1.9073486328125e-06 * (qnorm + Rn) * (qnorm + Rn);   // 2^-19
    rowp[li] = make_float2(__double2float_rd((qn - 2.0 * eps_c - slack) * s2), u * sqrtf((float)s2));
  }
}

// a handful of open rows is cheaper to scan exactly than to sweep again: move queue 1 behind queue 2
__global__ void knn_append_queue_kernel(const int32_t* __restrict__ q_src, const double* __restrict__ ub_src, int64_t n,
                                        int32_t* __restrict__ q_dst, double* __restrict__ ub_dst,
                                        unsigned long long* __restrict__ cnt_dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long w = atomicAdd(cnt_dst, 1ull);
  q_dst[w] = q_src[i];
  ub_dst[w] = ub_src[i];
}

// exact fallback: one CTA per uncertified query, fp64 distances to every point
constexpr int FB_THREADS = 256;
constexpr int FB_BUF = 2048;

__device__ void block_bitonic_sort(double* keys, int32_t* ids, int n_pow2) {
  for (int kk = 2; kk <= n_pow2; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool asc = (i & kk) == 0;
          const bool gt = lex_less(keys[ixj], ids[ixj], keys[i], ids[i]);
          if (gt == asc) {
            double tk = keys[i]; keys[i] = keys[ixj]; keys[ixj] = tk;
            int32_t ti = ids[i]; ids[i] = ids[ixj]; ids[ixj] = ti;
          }
        }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(FB_THREADS)
knn_fallback_kernel(const float* __restrict__ X, const float* __restrict__ Xt, int64_t n_points, int d, int64_t q0,
                    int k, const int32_t* __restrict__ work_q, const double* __restrict__ work_ub,
                    const unsigned long long* __restrict__ work_cnt, int32_t* __restrict__ idx_out,
                    double* __restrict__ dist_out) {
  __shared__ double keys[FB_BUF];
  __shared__ int32_t ids[FB_BUF];
  __shared__ double qx[256];
  __shared__ int cnt;
  __shared__ double thr_key;
  __shared__ int32_t thr_id;
  const unsigned long long nwork = *work_cnt;
  for (unsigned long long w = blockIdx.x; w < nwork; w += gridDim.x) {
    const int64_t ql = work_q[w];
    const int64_t q = q0 + ql;
    __syncthreads();
    for (int j = threadIdx.x; j < d; j += blockDim.x) qx[j] = X[q * d + j];
    if (threadIdx.x == 0) {
      cnt = 0;
      thr_key = work_ub[w];
      thr_id = INT32_MAX;
    }
    __syncthreads();
    for (int64_t base = 0; base < n_points; base += FB_THREADS) {
      const int64_t p = base + threadIdx.x;
      if (p < n_points) {
        const float* col = Xt + (p / TILE) * (int64_t)(d + 1) * TILE + (p % TILE);
        double acc = 0.0;
        for (int j = 0; j < d; ++j) {
          const double df = qx[j] - (double)col[(int64_t)j * TILE];
          acc = fma(df, df, acc);
        }
        const double key = (p == q) ? -1.0 : acc;
        if (key < thr_key || (key == thr_key && (int32_t)p <= thr_id)) {
          const int pos = atomicAdd(&cnt, 1);
          keys[pos] = key;
          ids[pos] = (int32_t)p;
        }
      }
      __syncthreads();
      const bool compact = cnt > FB_BUF - FB_THREADS;  // snapshot: every thread takes the same branch
      __syncthreads();                                 // ... before anybody's next atomicAdd can change cnt
      if (compact) {
        const int c0 = cnt;
        for (int i = c0 + threadIdx.x; i < FB_BUF; i += blockDim.x) { keys[i] = DBL_MAX; ids[i] = INT32_MAX; }
        __syncthreads();
        block_bitonic_sort(keys, ids, FB_BUF);
        if (threadIdx.x == 0) {
          cnt = k;
          thr_key = keys[k - 1];
          thr_id = ids[k - 1];
        }
        __syncthreads();
      }
    }
    const int c0 = cnt;
    for (int i = c0 + threadIdx.x; i < FB_BUF; i += blockDim.x) { keys[i] = DBL_MAX; ids[i] = INT32_MAX; }
    __syncthreads();
    block_bitonic_sort(keys, ids, FB_BUF);
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
      idx_out[ql * k + i] = ids[i];
      dist_out[ql * k + i] = keys[i] < 0.0 ? 0.0 : sqrt(keys[i]);
    }
  }
}

}  // namespace

namespace {

struct EventPairs {  // CUDA-event brackets around the sweep kernels of one call (info != NULL only)
  cudaEvent_t ev[8][2];
  int n = 0;
  bool on = false;
  cudaStream_t st = nullptr;
  int32_t begin() {
    if (!on || n >= 8) return SB2_OK;
    SB2_CUDA(cudaEventCreate(&ev[n][0]));
    SB2_CUDA(cudaEventCreate(&ev[n][1]));
    SB2_CUDA(cudaEventRecord(ev[n][0], st));
    return SB2_OK;
  }
  int32_t end() {
    if (!on || n >= 8) return SB2_OK;
    SB2_CUDA(cudaEventRecord(ev[n][1], st));
    ++n;
    return SB2_OK;
  }
  float total_ms() {
    float t = 0.0f;
    for (int i = 0; i < n; ++i) {
      float ms = 0.0f;
      if (cudaEventElapsedTime(&ms, ev[i][0], ev[i][1]) == cudaSuccess) t += ms;
    }
    return t;
  }
  ~EventPairs() {
    for (int i = 0; i < n; ++i) { cudaEventDestroy(ev[i][0]); cudaEventDestroy(ev[i][1]); }
  }
};

// Every run-time switch of the kNN, parsed on every call (the tests change them between calls)
KnnSwitches knn_switches() {
  const auto is = [](const char* name, const char* value) {
    const char* e = getenv(name);
    return e && strcmp(e, value) == 0;
  };
  KnnSwitches s;
  s.ffma = is("SB2_KNN_PASS1", "ffma");
  s.split_only = is("SB2_KNN_TIERS", "3");
  s.big_list = is("SB2_KNN_LIST", "64") || is("SB2_KNN_LIST", "128");
  if (const char* e = getenv("SB2_KNN_EST")) {
    if (atoi(e) > 0) s.est_stride = atoi(e);
    else s.cold = true;
  }
  if (const char* e = getenv("SB2_KNN_EST_RANK"); e && atoi(e) >= 1 && atoi(e) <= EST_R) s.est_rank = atoi(e);
  if (const char* e = getenv("SB2_KNN_SCAN_SLOTS")) s.scan_slots = atoll(e);
  s.pipe = !is("SB2_KNN_PIPE", "0");
  s.stamps = is("SB2_KNN_STAMPS", "1");
  s.int_scan = !is("SB2_KNN_SCAN", "float");
  if (is("SB2_KNN_SCREEN", "0")) s.screen = 0;
  else if (is("SB2_KNN_SCREEN", "1")) s.screen = 1;
  if (const char* e = getenv("SB2_KNN_NEAR")) {   // anything but 1..KNN_MAX_NEAR fails the screened call (screen_prep)
    char* end = nullptr;
    const long v = strtol(e, &end, 10);
    s.near_tiles = (end != e && *end == '\0' && v >= 1 && v <= KNN_MAX_NEAR) ? (int)v : 0;
  }
  if (const char* e = getenv("SB2_KNN_SPLIT")) s.split = strcmp(e, "principal") == 0 ? 1 : strcmp(e, "coord") == 0 ? 0 : -1;
  if (const char* e = getenv("SB2_KNN_KD_WIDE")) {
    char* end = nullptr;
    const long long v = strtoll(e, &end, 10);
    s.kd_wide = (end != e && *end == '\0' && v >= 1) ? (int64_t)v : 0;
  }
  return s;
}

// Xt: the points in tiles of 128, k-major, with the row of -|x|^2/2; maxnorm[4]: [0] the bits of the largest squared
// norm, the rest zeroed for the fp16 tier
int32_t prep_points(sb2_ctx* ctx, ScratchScope& scr, const float* d_x, int64_t n_points, int d, float** Xt,
                    unsigned int** maxnorm) {
  const int64_t n_tiles = ceil_div64(n_points, TILE);
  SB2_TRY(scr.alloc(Xt, (size_t)(n_tiles * (d + 1) * TILE)));
  SB2_TRY(scr.alloc(maxnorm, 4));
  SB2_CUDA(cudaMemsetAsync(*maxnorm, 0, 16, ctx->stream));
  const size_t smem = (size_t)TILE * d * sizeof(float);
  SB2_CUDA(cudaFuncSetAttribute(knn_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  knn_prep_kernel<<<(unsigned)n_tiles, 256, smem, ctx->stream>>>(d_x, n_points, d, *Xt, *maxnorm);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

// what the passes of one sb2_knn_l2_f32 call share
struct KnnCall {
  sb2_ctx* ctx;
  ScratchScope* scr;
  KnnSwitches sw;
  const float* d_x;
  int64_t n_points, q0, n_query;
  int d, k;
  int32_t* d_idx;
  double* d_dist;
  float* Xt = nullptr;
  unsigned int* maxnorm = nullptr;   // bits of [0] the largest squared norm, [1] the fp16 tier's largest |x - fp16(x)|
  int32_t* wq[2] = {};               // local rows left open: [0] by tier 1, [1] for the exact scan
  double* wub[2] = {};               // their bounds on the k-th squared distance
  unsigned long long* wcnt = nullptr;  // [2] the two queues' lengths
  int list_m = 0, sub = 0;           // proposals per row, in sub-lists of sub
  float* cand_score = nullptr;       // [n_query][list_m]
  int32_t* cand_idx = nullptr;
  double issued_flops = 0.0;
  int64_t n_resweep = 0;
  EventPairs evs;
};

// how a pass's proposals are certified: |s_computed - s_true| <= c_q |q| R + c_n R^2 / 2 (scores in units of inv_s2 on
// the tensor path), plus the measured |x - fp16(x)| term of the fp16 tier; the rows it cannot certify join queue `queue`
struct Bound {
  double c_q, c_n;
  const float* inv_s2;
  const float* dnorm;
  const unsigned int* dmax;
  int queue;
};

// fp64 re-score + certificate of n_rows proposal lists (those of launch rows ql0 + i): launch row i is local row ql0 + i,
// or row_map[i]; cand_map maps proposal ids (image positions) to points, ubound[i] is row i's tile-screen bound
int32_t launch_rescore(KnnCall& c, const Bound& b, int64_t ql0, const int32_t* row_map, int64_t n_rows,
                       const int32_t* cand_map = nullptr, const float* ubound = nullptr) {
  if (n_rows == 0) return SB2_OK;
  const int wpb = 8;
  const unsigned grid = (unsigned)ceil_div64(n_rows, wpb);
  const auto launch = [&](auto r) {
    knn_rescore_kernel<r><<<grid, wpb * 32, 0, c.ctx->stream>>>(
        c.d_x, c.n_points, c.d, c.q0, ql0, row_map, n_rows, c.k, c.sub, c.cand_score + ql0 * c.list_m,
        c.cand_idx + ql0 * c.list_m, c.maxnorm, b.inv_s2, b.c_q, b.c_n, b.dnorm, b.dmax, cand_map, ubound, c.d_idx, c.d_dist, c.wq[b.queue],
        c.wub[b.queue], c.wcnt + b.queue);
  };
  if (c.list_m == 32) launch(std::integral_constant<int, 1>());
  else if (c.list_m == 64) launch(std::integral_constant<int, 2>());
  else launch(std::integral_constant<int, 4>());
  SB2_LAUNCH_CHECK(c.ctx);
  return SB2_OK;
}

int32_t read_count(sb2_ctx* ctx, const unsigned long long* d_cnt, int64_t* out) {
  unsigned long long h = 0;
  SB2_CUDA(cudaMemcpyAsync(&h, d_cnt, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = (int64_t)h;
  return SB2_OK;
}

// The tile screen of tier 1 (knn_tc2.cu): both images in the kd order, and per 128-row query block the candidate tiles
// that may hold a neighbour of one of its rows.  Launch row i (query image row i) is local row qloc[i].
struct Screen {
  int32_t* perm = nullptr;    // [n_points] image position -> point
  int32_t* qloc = nullptr;    // [n_query]
  int32_t* qpos = nullptr;    // [n_query] position of launch row i in perm (nullptr: i itself)
  int32_t* lists = nullptr;   // block b's ascending tiles at lists[off[b] ..]; nullptr: every block sweeps every tile
  int64_t* off = nullptr;     // [blocks]
  int32_t* len = nullptr;     // [blocks]
  std::vector<int32_t> h_len;
  std::vector<int64_t> h_off;
  float* ub = nullptr;        // [n_query] bound on the k-th neighbour distance
  float* seed = nullptr;      // [n_query] starting threshold of the sweep (scaled score units)
};

// one precision tier of the tensor path (knn_tc2.cu): its sweep shape, its candidate image and its certificate
struct Tier {
  KnnTc2Shape sh;
  __half* B = nullptr;
  Bound bound;
  const Screen* scr = nullptr;   // tier 1 with the tile screen: B and the query image in the kd order
};

// one sweep of a tier, bracketed by the call's events, and the re-score of its proposals (launch rows [ql0, ql0 + n_rows)):
// local rows [ql0, ql0 + n_rows) held by the query image A from its tile a_tile0 on, or the rows row_map[0, n_rows) that
// A holds gathered in that order.  With the screen, row_map is the kd order's and each block walks its tile list.
int32_t sweep_and_certify(KnnCall& c, const Tier& t, const __half* A, int64_t a_tile0, int64_t ql0, const int32_t* row_map,
                          int64_t n_rows) {
  KnnTc2Lists L{}, *lp = nullptr;
  const bool lists = t.scr && t.scr->lists;   // without lists: the full sweep with the sampled estimate, in the kd order
  if (t.scr) {
    const Screen& S = *t.scr;
    const int64_t b0 = ql0 / TILE, nb = ceil_div64(n_rows, TILE);
    if (lists) {
      int64_t total = 0;
      for (int64_t b = b0; b < b0 + nb; ++b) total += S.h_len[b];
      L = KnnTc2Lists{S.lists, 0, S.off + b0, S.len + b0, total, c.sw.cold ? nullptr : S.seed + ql0, c.sw.stamps};
      lp = &L;
    }
    row_map = S.qloc + ql0;
  }
  SB2_TRY(c.evs.begin());
  SB2_TRY(knn_tc2_sweep(c.ctx, c.sw, t.sh, A, a_tile0, t.B, c.n_points, n_rows, c.list_m, c.cand_score + ql0 * c.list_m,
                        c.cand_idx + ql0 * c.list_m, &c.issued_flops, lp));
  SB2_TRY(c.evs.end());
  return launch_rescore(c, t.bound, ql0, row_map, n_rows, t.scr ? t.scr->perm : nullptr, lists ? t.scr->ub + ql0 : nullptr);
}

// Above this share of kept (block, tile) pairs the screen's lists are dropped for the full sweep (SB2_KNN_SCREEN=1 keeps
// them): see DESIGN.md §4 for the measurement behind it.
constexpr double SCREEN_MAX_KEPT = 0.9;
constexpr int NEAR_COLD = 8;   // tiles of the screen's cold short sweep (the rest of the near tiles are swept seeded)

// Tier 1's images in the kd order and the tile screen: the order, the per-tile centres and radii, a short sweep of each
// block's own neighbourhood (SB2_KNN_NEAR consecutive tiles, 64 by default: a cold pass over the middle NEAR_COLD of
// them, then a pass over all of them seeded from its bound) whose proposals bound every row's k-th distance (knn_row_bound_kernel),
// then the screen of every row against every tile centre (knn_screen_kernel).  Bracketed by the call's events, so the
// reported sweep time includes it; SB2_KNN_STAMPS=1 reports its parts.  The lists are kept (S.lists) when they skip
// enough tiles (SCREEN_MAX_KEPT) and fit in device memory, or always with `force`; otherwise S.lists stays nullptr and
// tier 1 sweeps every tile of the kd-ordered images from the sampled estimate, as without the screen.
struct EventSet {   // CUDA events created on demand, destroyed on every exit
  cudaEvent_t e[3] = {};
  ~EventSet() {
    for (cudaEvent_t x : e)
      if (x) cudaEventDestroy(x);
  }
};
int32_t screen_prep(KnnCall& c, Tier& t1, __half* A1, float* inv_s2, float* dnorm, bool force, Screen& S) {
  sb2_ctx* ctx = c.ctx;
  ScratchScope& scr = *c.scr;
  cudaStream_t st = ctx->stream;
  const int64_t n_points = c.n_points, n_query = c.n_query, n_tiles = ceil_div64(n_points, TILE);
  const int64_t n_blocks = ceil_div64(n_query, TILE);
  const int d = c.d;
  EventSet evset;
  cudaEvent_t* ev = evset.e;
  if (c.sw.stamps)
    for (int i = 0; i < 3; ++i) SB2_CUDA(cudaEventCreate(&ev[i]));
  SB2_TRY(c.evs.begin());
  if (ev[0]) SB2_CUDA(cudaEventRecord(ev[0], st));
  SB2_CHECK_ARG(c.sw.split >= 0, "SB2_KNN_SPLIT must be principal or coord");
  SB2_CHECK_ARG(c.sw.kd_wide >= 1, "SB2_KNN_KD_WIDE must be an integer >= 1");
  SB2_TRY(scr.alloc(&S.perm, (size_t)n_points));
  SB2_TRY(knn_tc2_kd_order(ctx, c.d_x, n_points, d, c.sw.split == 0, c.sw.kd_wide, S.perm));
  if (c.q0 == 0 && n_query == n_points) {
    S.qloc = S.perm;
  } else {
    SB2_TRY(scr.alloc(&S.qloc, (size_t)n_query));
    SB2_TRY(scr.alloc(&S.qpos, (size_t)n_query));
    SB2_TRY(knn_tc2_restrict(ctx, S.perm, n_points, c.q0, n_query, S.qloc, S.qpos));
  }
  if (ev[1]) SB2_CUDA(cudaEventRecord(ev[1], st));
  // images in the kd order (dnorm stays indexed by point)
  SB2_TRY(knn_tc2_build_images(ctx, t1.sh, c.d_x, n_points, d, c.maxnorm, S.perm, 0, nullptr, t1.B, inv_s2, dnorm, c.maxnorm + 1));
  SB2_TRY(knn_tc2_build_images(ctx, t1.sh, c.d_x, n_query, d, c.maxnorm, S.qloc, c.q0, A1, nullptr, inv_s2));
  float *cent, *rad;
  __half* Cimg;
  SB2_TRY(scr.alloc(&cent, (size_t)n_tiles * d));
  SB2_TRY(scr.alloc(&rad, (size_t)n_tiles));
  SB2_TRY(scr.alloc(&Cimg, knn_tc2_b_halves(t1.sh, n_tiles)));
  SB2_TRY(knn_tc2_tile_stats(ctx, c.d_x, n_points, d, S.perm, c.maxnorm, cent, rad));
  SB2_TRY(knn_tc2_build_images(ctx, t1.sh, cent, n_tiles, d, c.maxnorm, nullptr, 0, nullptr, Cimg, inv_s2));
  // the short sweep over each block's own neighbourhood, nt consecutive tiles of the order (64 by default, not 8: a
  // block at a split boundary has its neighbours across the split, far away in the order; DESIGN.md §4).  A cold
  // sweep inserts on nearly every tile, so it covers only the middle NEAR_COLD tiles; its bound u1 seeds a second
  // sweep over all nt.  Every point within u1 scores above the seed, so the second sweep's sub-lists keep every
  // proposal a cold sweep of the nt tiles would rank in the top k (the k from the first sweep among them): its u is
  // the cold sweep's, at the cost of a warm sweep.
  const int nt = c.sw.near_tiles;
  SB2_CHECK_ARG(nt >= 1 && nt <= KNN_MAX_NEAR, "SB2_KNN_NEAR must be an integer in 1..64");
  float2* rowp;
  SB2_TRY(scr.alloc(&S.ub, (size_t)n_query));
  SB2_TRY(scr.alloc(&S.seed, (size_t)n_query));
  SB2_TRY(scr.alloc(&rowp, (size_t)n_blocks * TILE));
  int32_t *near, *near_len;
  SB2_TRY(scr.alloc(&near, (size_t)n_blocks * nt));
  SB2_TRY(scr.alloc(&near_len, (size_t)n_blocks));
  const auto short_sweep = [&](int w, const float* seed) -> int32_t {
    SB2_TRY(knn_tc2_near_lists(ctx, n_blocks, n_tiles, w, S.qpos, near, near_len));
    const KnnTc2Lists NL{near, w, nullptr, near_len, n_blocks * (w < n_tiles ? w : n_tiles), seed, false};
    SB2_TRY(knn_tc2_sweep(ctx, c.sw, t1.sh, A1, 0, t1.B, n_points, n_query, c.list_m, c.cand_score, c.cand_idx, &c.issued_flops, &NL));
    const int wpb = 8;
    const int64_t n_pad = n_blocks * TILE;
    const unsigned grid = (unsigned)ceil_div64(n_pad, wpb);
    const Bound& b = t1.bound;
    const auto launch = [&](auto r) {
      knn_row_bound_kernel<r><<<grid, wpb * 32, 0, st>>>(c.d_x, d, c.q0, S.qloc, n_query, n_pad, c.k, c.cand_score, c.cand_idx,
                                                         c.maxnorm, inv_s2, b.c_q, b.c_n, dnorm, c.maxnorm + 1, S.ub, S.seed, rowp);
    };
    if (c.list_m == 64) launch(std::integral_constant<int, 2>());
    else launch(std::integral_constant<int, 4>());
    SB2_LAUNCH_CHECK(ctx);
    return SB2_OK;
  };
  SB2_TRY(short_sweep(nt < NEAR_COLD ? nt : NEAR_COLD, nullptr));
  if (nt > NEAR_COLD) SB2_TRY(short_sweep(nt, S.seed));
  // the screen writes a bitmap per block (n_tiles / 8 bytes) and its count; only the kept tiles become list entries
  uint32_t* words;
  SB2_TRY(scr.alloc(&words, (size_t)n_blocks * knn_tc2_screen_words(n_tiles)));
  SB2_TRY(scr.alloc(&S.len, (size_t)n_blocks));
  SB2_TRY(knn_tc2_screen(ctx, t1.sh, A1, Cimg, n_blocks, n_tiles, rowp, rad, c.maxnorm, words, S.len));
  if (ev[2]) SB2_CUDA(cudaEventRecord(ev[2], st));
  SB2_TRY(c.evs.end());
  S.h_len.resize((size_t)n_blocks);
  SB2_CUDA(cudaMemcpyAsync(S.h_len.data(), S.len, (size_t)n_blocks * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  S.h_off.resize((size_t)n_blocks);
  int64_t total = 0;
  for (int64_t b = 0; b < n_blocks; ++b) {
    S.h_off[b] = total;
    total += S.h_len[b];
  }
  const double kept = (double)total / ((double)n_blocks * (double)n_tiles);
  size_t free_b = 0, total_b = 0;
  SB2_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const bool fits = (size_t)total * sizeof(int32_t) + (size_t)n_blocks * sizeof(int64_t) <= free_b / 4;
  if (force || (kept <= SCREEN_MAX_KEPT && fits)) {
    SB2_TRY(c.evs.begin());
    SB2_TRY(scr.alloc(&S.off, (size_t)n_blocks));
    SB2_TRY(scr.alloc(&S.lists, (size_t)total));
    SB2_CUDA(cudaMemcpyAsync(S.off, S.h_off.data(), (size_t)n_blocks * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    SB2_TRY(knn_tc2_expand_lists(ctx, words, n_blocks, n_tiles, S.off, S.lists));
    SB2_TRY(c.evs.end());
  }
  if (ev[0]) {
    float ms_order = 0.0f, ms_screen = 0.0f;
    SB2_CUDA(cudaEventElapsedTime(&ms_order, ev[0], ev[1]));
    SB2_CUDA(cudaEventElapsedTime(&ms_screen, ev[1], ev[2]));
    std::vector<int32_t> v = S.h_len;
    std::sort(v.begin(), v.end());
    fprintf(stderr, "[sb2 knn screen] %lld blocks x %lld tiles: surviving %.4f, list length min %d median %d max %d; kd order %.2f ms, "
            "images + short sweep (%d near tiles) + screen %.2f ms; %s\n", (long long)n_blocks, (long long)n_tiles, kept, v.front(),
            v[v.size() / 2], v.back(), ms_order, nt, ms_screen, S.lists ? "tile lists" : "full sweep (too few tiles skipped, or lists do not fit)");
  }
  return SB2_OK;
}

// Tensor path, in tiers that each end in the same fp64 re-score + certificate:
//   tier 1  one fp16 sweep (K = d+3): proposals whose rounding bound (2^-10 |q| R) still certifies the exact top-k are final
//   tier 2  rows tier 1 could not certify are gathered and swept again in split precision (K = 3d+3, bound ~2^-16 |q| R)
//   tier 3  rows still open (exact ties at the k-th distance, floods of duplicates): fp64 scan of every point (caller)
// A pilot of one wave of CTAs measures tier 1's certification rate; if most rows fail (data far from the origin,
// tiny neighbour gaps) the remaining rows go straight to the split-precision sweep.
int32_t tensor_tiers(KnnCall& c) {
  sb2_ctx* ctx = c.ctx;
  ScratchScope& scr = *c.scr;
  const int64_t n_points = c.n_points, n_query = c.n_query;
  const int d = c.d;
  // only tier 1 starts from a sampled threshold: a row the re-sweep gathers may have failed because its sampled
  // threshold was too tight (fewer than k candidates beat it), and must not fail twice
  Tier t1, t3;
  SB2_CHECK_ARG(knn_tc2_shape(ctx, d, 1, true, &t1.sh) && knn_tc2_shape(ctx, d, 3, false, &t3.sh),
                "tensor-core kNN tile does not fit shared memory");
  c.list_m = (c.k > 24 || c.sw.big_list) ? 128 : 64;
  c.sub = c.list_m / 4;  // four sub-lists per row
  SB2_TRY(scr.alloc(&c.cand_score, (size_t)n_query * c.list_m));
  SB2_TRY(scr.alloc(&c.cand_idx, (size_t)n_query * c.list_m));
  float* inv_s2;
  SB2_TRY(scr.alloc(&inv_s2, 4));
  t1.bound = {0.0, 0.0, inv_s2, nullptr, nullptr, 0};  // tier 1's open rows wait for the re-sweep,
  t3.bound = {0.0, 0.0, inv_s2, nullptr, nullptr, 1};  // the split tier's for the exact scan
  knn_tc2_error_coefs(t1.sh, &t1.bound.c_q, &t1.bound.c_n);
  knn_tc2_error_coefs(t3.sh, &t3.bound.c_q, &t3.bound.c_n);
  // the tile screen (SB2_KNN_SCREEN): by default from 512 candidate tiles on, below which the short sweep and the screen
  // cost more than the tiles they can skip
  const int64_t n_tiles = ceil_div64(n_points, TILE);
  bool screen = !c.sw.split_only && t1.sh.nsplit == 1 && (c.sw.screen == 1 || (c.sw.screen < 0 && n_tiles >= 512));
  if (screen) {   // the screen's bitmaps (n_q/128 x n/128 bits) must fit comfortably; otherwise the unscreened sweep
    size_t free_b = 0, total_b = 0;
    SB2_CUDA(cudaMemGetInfo(&free_b, &total_b));
    screen = (size_t)ceil_div64(n_query, TILE) * (size_t)knn_tc2_screen_words(n_tiles) * 4 <= free_b / 8;
  }
  Screen S;
  int64_t done = 0;  // launch rows [0, done) have been through their first sweep
  if (!c.sw.split_only) {
    __half* A1;
    float* dnorm;  // |x - fp16(x)| per point; its maximum lives in maxnorm[1]
    SB2_TRY(scr.alloc(&A1, knn_tc2_a_halves(t1.sh, n_points)));
    SB2_TRY(scr.alloc(&t1.B, knn_tc2_b_halves(t1.sh, n_points)));
    SB2_TRY(scr.alloc(&dnorm, (size_t)n_points));
    t1.bound.dnorm = dnorm;
    t1.bound.dmax = c.maxnorm + 1;
    if (screen) {
      SB2_TRY(screen_prep(c, t1, A1, inv_s2, dnorm, c.sw.screen == 1, S));
      t1.scr = &S;
    } else {
      SB2_TRY(knn_tc2_build_images(ctx, t1.sh, c.d_x, n_points, d, c.maxnorm, nullptr, 0, A1, t1.B, inv_s2, dnorm, c.maxnorm + 1));
    }
    const auto tile0 = [&](int64_t ql0) { return screen ? ql0 / TILE : (c.q0 + ql0) / TILE; };
    // pilot: one wave of CTAs.  With the screen that wave is one contiguous region of the kd order, not a sample of the
    // whole data set; what it decides (fp16 tier 1 for the rest, or split precision straight away) changes only the
    // speed, every row is certified either way, and what makes the fp16 tier fail (the data's distance from the origin,
    // relative to its neighbour gaps) is mostly a property of the whole embedding rather than of one region
    const int64_t wave = (int64_t)ctx->prop.multiProcessorCount * TILE;
    const int64_t first = n_query >= 4 * wave ? wave : n_query;
    SB2_TRY(sweep_and_certify(c, t1, A1, tile0(0), 0, nullptr, first));
    done = first;
    if (first < n_query) {
      int64_t open1 = 0;
      SB2_TRY(read_count(ctx, c.wcnt, &open1));
      if (open1 * 2 <= first) {  // most pilot rows certified: tier 1 for the rest too
        SB2_TRY(sweep_and_certify(c, t1, A1, tile0(done), done, nullptr, n_query - done));
        done = n_query;
      }
    }
  }
  if (done < n_query) {
    // split-precision sweep of the remaining rows, straight from the full image arrays (with the screen: the remaining
    // launch rows, gathered, against the candidates in storage order)
    __half* A3;
    SB2_TRY(scr.alloc(&A3, knn_tc2_a_halves(t3.sh, n_points)));
    SB2_TRY(scr.alloc(&t3.B, knn_tc2_b_halves(t3.sh, n_points)));
    if (screen) {
      SB2_TRY(knn_tc2_build_images(ctx, t3.sh, c.d_x, n_points, d, c.maxnorm, nullptr, 0, nullptr, t3.B, inv_s2));
      SB2_TRY(knn_tc2_build_images(ctx, t3.sh, c.d_x, n_query - done, d, c.maxnorm, S.qloc + done, c.q0, A3, nullptr, inv_s2));
      SB2_TRY(sweep_and_certify(c, t3, A3, 0, done, S.qloc + done, n_query - done));
    } else {
      SB2_TRY(knn_tc2_build_images(ctx, t3.sh, c.d_x, n_points, d, c.maxnorm, nullptr, 0, A3, t3.B, inv_s2));
      SB2_TRY(sweep_and_certify(c, t3, A3, (c.q0 + done) / TILE, done, nullptr, n_query - done));
    }
  }
  if (c.sw.split_only) return SB2_OK;
  // tier 2: gather the rows tier 1 left open and sweep them in split precision
  SB2_TRY(read_count(ctx, c.wcnt, &c.n_resweep));
  // a re-sweep occupies one CTA per 128 open rows for a whole pass over the candidates (9.4 ms at 1.3M x 50, however
  // few rows there are); the exact scan gives each ROW one CTA that streams the whole data set, 21 ms for a single row
  // at 1.3M x 50 (H100 80GB HBM3, 700 W): it only pays off as a bulk pass, so by default every open row is re-swept and
  // the scan takes what the re-sweep leaves open (SB2_KNN_SCAN_SLOTS=n sends up to n rows straight to the scan)
  const int64_t n_resweep = c.n_resweep;
  if (n_resweep > 0 && n_resweep <= c.sw.scan_slots) {
    knn_append_queue_kernel<<<(unsigned)ceil_div64(n_resweep, 256), 256, 0, ctx->stream>>>(c.wq[0], c.wub[0], n_resweep, c.wq[1],
                                                                                            c.wub[1], c.wcnt + 1);
    SB2_LAUNCH_CHECK(ctx);
  } else if (n_resweep > 0) {
    if (!t3.B) {
      SB2_TRY(scr.alloc(&t3.B, knn_tc2_b_halves(t3.sh, n_points)));
      SB2_TRY(knn_tc2_build_images(ctx, t3.sh, c.d_x, n_points, d, c.maxnorm, nullptr, 0, nullptr, t3.B, inv_s2));
    }
    __half* Ag;
    SB2_TRY(scr.alloc(&Ag, knn_tc2_a_halves(t3.sh, n_resweep)));
    SB2_TRY(knn_tc2_build_images(ctx, t3.sh, c.d_x, n_resweep, d, c.maxnorm, c.wq[0], c.q0, Ag, nullptr, inv_s2));
    SB2_TRY(sweep_and_certify(c, t3, Ag, 0, 0, c.wq[0], n_resweep));
  }
  return SB2_OK;
}

// The fp32 CUDA-core first pass (SB2_KNN_PASS1=ffma): 32 proposals per row; rows it cannot certify go to the exact scan
int32_t ffma_pass(KnnCall& c) {
  sb2_ctx* ctx = c.ctx;
  cudaStream_t st = ctx->stream;
  c.list_m = c.sub = LISTM;
  SB2_TRY(c.scr->alloc(&c.cand_score, (size_t)c.n_query * LISTM));
  SB2_TRY(c.scr->alloc(&c.cand_idx, (size_t)c.n_query * LISTM));
  c.issued_flops = 2.0 * (double)c.n_query * (double)c.n_points * (double)c.d;
  const double e = 1.5 * (double)(c.d + 2) * 5.9604644775390625e-08;
  const int64_t n_tiles = ceil_div64(c.n_points, TILE), q_tiles = ceil_div64(c.n_query, TILE);
  const size_t chunk_b = (size_t)(c.d + 1) * TILE * 4;
  const size_t smem3 = chunk_b * 4 + 64, smem2 = chunk_b * 3 + 64;
  const size_t lim = ctx->prop.sharedMemPerBlockOptin;
  SB2_TRY(c.evs.begin());
  if (smem3 <= lim) {
    SB2_CUDA(cudaFuncSetAttribute(knn_pass1_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem3));
    knn_pass1_kernel<3><<<(unsigned)q_tiles, PASS1_THREADS, smem3, st>>>(c.Xt, c.d, n_tiles, c.q0 / TILE, c.n_query,
                                                                         c.cand_score, c.cand_idx);
  } else {
    SB2_CHECK_ARG(smem2 <= lim, "d too large for shared memory");
    SB2_CUDA(cudaFuncSetAttribute(knn_pass1_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    knn_pass1_kernel<2><<<(unsigned)q_tiles, PASS1_THREADS, smem2, st>>>(c.Xt, c.d, n_tiles, c.q0 / TILE, c.n_query,
                                                                         c.cand_score, c.cand_idx);
  }
  SB2_LAUNCH_CHECK(ctx);
  SB2_TRY(c.evs.end());
  return launch_rescore(c, Bound{e, e, nullptr, nullptr, nullptr, 1}, 0, nullptr, c.n_query);
}

}  // namespace

// Exact kNN: a fast first pass proposes candidates per query, an fp64 re-score certifies the top-k against a rigorous
// rounding-error bound, rows without a certificate are recomputed exactly.  First pass: the tensor-core tiers above
// (knn_tc2.cu) or the fp32 CUDA-core sweep (SB2_KNN_PASS1=ffma).
extern "C" int32_t sb2_knn_l2_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int64_t q0,
                                  int64_t n_query, int32_t k, int32_t* d_idx, double* d_dist, sb2_knn_info* info) {
  SB2_CHECK_ARG(ctx && d_x && d_idx && d_dist, "null pointer");
  SB2_CHECK_ARG(n_points >= 1 && n_points < (int64_t)INT32_MAX - 2 * TILE, "n_points");
  SB2_CHECK_ARG(d >= 1 && d <= 150, "d must be in [1,150]");
  SB2_CHECK_ARG(k >= 1 && k <= 56 && k <= n_points, "k must be in [1,56] and <= n_points");
  SB2_CHECK_ARG(q0 >= 0 && n_query >= 0 && q0 + n_query <= n_points, "query range");
  SB2_CHECK_ARG(q0 % TILE == 0, "q0 must be a multiple of 128");
  if (n_query == 0) return SB2_OK;
  const KnnSwitches sw = knn_switches();
  const bool use_tc = knn_tc2_supported(d) && !sw.ffma;
  SB2_CHECK_ARG(use_tc || k <= LISTM - 2, "k > 30 needs the tensor-core pass (SB2_KNN_PASS1=ffma limits k to 30)");
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  KnnCall c{ctx, &scr, sw, d_x, n_points, q0, n_query, d, k, d_idx, d_dist};
  SB2_TRY(prep_points(ctx, scr, d_x, n_points, d, &c.Xt, &c.maxnorm));
  for (int i = 0; i < 2; ++i) {
    SB2_TRY(scr.alloc(&c.wq[i], (size_t)n_query));
    SB2_TRY(scr.alloc(&c.wub[i], (size_t)n_query));
  }
  SB2_TRY(scr.alloc(&c.wcnt, 2));
  SB2_CUDA(cudaMemsetAsync(c.wcnt, 0, 16, st));
  c.evs.on = info != nullptr;
  c.evs.st = st;
  SB2_TRY(use_tc ? tensor_tiers(c) : ffma_pass(c));
  {
    const int grid = ctx->prop.multiProcessorCount * 4;
    knn_fallback_kernel<<<grid, FB_THREADS, 0, st>>>(d_x, c.Xt, n_points, d, q0, k, c.wq[1], c.wub[1], c.wcnt + 1, d_idx, d_dist);
    SB2_LAUNCH_CHECK(ctx);
  }
  if (info) {
    unsigned long long h_cnt = 0;
    unsigned int h_bits = 0;
    SB2_CUDA(cudaMemcpyAsync(&h_cnt, c.wcnt + 1, sizeof(h_cnt), cudaMemcpyDeviceToHost, st));
    SB2_CUDA(cudaMemcpyAsync(&h_bits, c.maxnorm, sizeof(h_bits), cudaMemcpyDeviceToHost, st));
    SB2_CUDA(cudaStreamSynchronize(st));
    info->n_uncertified = (int64_t)h_cnt;
    float f;
    memcpy(&f, &h_bits, 4);
    info->max_norm = sqrtf(f);
    info->pass1_ms = c.evs.total_ms();
    info->pass1_flops = 2.0 * (double)n_query * (double)n_points * (double)d;
    info->pass1_issued_flops = c.issued_flops;
    info->pass1_tensor = use_tc ? 2 : 0;
    info->n_resweep = c.n_resweep;
  }
  return SB2_OK;
}

// Debug / test entry: the tile screen of a whole-data-set call (see include/scanpy_b200.h)
extern "C" int32_t sb2_knn_debug_screen_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int32_t k, int32_t* d_perm,
                                            int32_t* d_lists, int32_t* d_len, float* d_ub) {
  SB2_CHECK_ARG(ctx && d_x && d_perm && d_lists && d_len && d_ub, "null pointer");
  SB2_CHECK_ARG(n_points >= 1 && n_points < (int64_t)INT32_MAX - 2 * TILE && d >= 1 && d <= 150, "n_points / d");
  SB2_CHECK_ARG(k >= 1 && k <= 56 && k <= n_points, "k must be in [1,56] and <= n_points");
  const KnnSwitches sw = knn_switches();
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  KnnCall c{ctx, &scr, sw, d_x, n_points, 0, n_points, d, k, nullptr, nullptr};
  SB2_TRY(prep_points(ctx, scr, d_x, n_points, d, &c.Xt, &c.maxnorm));
  Tier t1;
  SB2_CHECK_ARG(knn_tc2_shape(ctx, d, 1, true, &t1.sh) && t1.sh.nsplit == 1, "tile does not fit shared memory");
  c.list_m = (k > 24 || sw.big_list) ? 128 : 64;
  c.sub = c.list_m / 4;
  SB2_TRY(scr.alloc(&c.cand_score, (size_t)n_points * c.list_m));
  SB2_TRY(scr.alloc(&c.cand_idx, (size_t)n_points * c.list_m));
  float *inv_s2, *dnorm;
  __half* A1;
  SB2_TRY(scr.alloc(&inv_s2, 4));
  SB2_TRY(scr.alloc(&dnorm, (size_t)n_points));
  SB2_TRY(scr.alloc(&A1, knn_tc2_a_halves(t1.sh, n_points)));
  SB2_TRY(scr.alloc(&t1.B, knn_tc2_b_halves(t1.sh, n_points)));
  t1.bound = {0.0, 0.0, inv_s2, dnorm, c.maxnorm + 1, 0};
  knn_tc2_error_coefs(t1.sh, &t1.bound.c_q, &t1.bound.c_n);
  Screen S;
  SB2_TRY(screen_prep(c, t1, A1, inv_s2, dnorm, true, S));
  const int64_t n_blocks = ceil_div64(n_points, TILE), n_tiles = ceil_div64(n_points, TILE);
  SB2_CUDA(cudaMemcpyAsync(d_perm, S.perm, (size_t)n_points * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  for (int64_t b = 0; b < n_blocks; ++b)
    SB2_CUDA(cudaMemcpyAsync(d_lists + b * n_tiles, S.lists + S.h_off[b], (size_t)S.h_len[b] * sizeof(int32_t),
                             cudaMemcpyDeviceToDevice, st));
  SB2_CUDA(cudaMemcpyAsync(d_len, S.len, (size_t)n_blocks * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  SB2_CUDA(cudaMemcpyAsync(d_ub, S.ub, (size_t)n_points * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  return SB2_OK;
}

// Debug / test entry: the raw proposals of ONE cold-start tensor sweep in the chosen operand format, with
// everything the rounding-error certificate is computed from, so that a test can MEASURE |s_tensor - s_exact| on the
// hardware against the bound knn_rescore_kernel uses (tests/test_gpu_parity.py::test_knn_tensor_score_error_within_bound).
//   d_score / d_idx [n_points x list_m]: proposal scores in the kernel's scaled units and their point ids (-1: unused)
//   d_dnorm [n_points]: |x - fp16(x)| per point (terms = 1 only, else untouched)
//   h_meta[6] = { inv_s2 (score_true = score * inv_s2), R^2 (largest squared norm), max_p dnorm[p], c_q, c_n, list_m }
extern "C" int32_t sb2_knn_debug_proposals_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int32_t terms,
                                               float* d_score, int32_t* d_idx, float* d_dnorm, double* h_meta) {
  SB2_CHECK_ARG(ctx && d_x && d_score && d_idx && h_meta, "null pointer");
  SB2_CHECK_ARG(terms == 1 || terms == 3, "terms must be 1 (fp16) or 3 (split fp16)");
  SB2_CHECK_ARG(n_points >= 1 && d >= 1 && d <= 150, "n_points / d");
  const KnnSwitches sw = knn_switches();
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  float* Xt;
  unsigned int* maxnorm;
  SB2_TRY(prep_points(ctx, scr, d_x, n_points, d, &Xt, &maxnorm));
  float* inv_s2;
  SB2_TRY(scr.alloc(&inv_s2, 4));
  KnnTc2Shape sh;
  SB2_CHECK_ARG(knn_tc2_shape(ctx, d, terms, false, &sh), "tile does not fit shared memory");
  __half *A, *B;
  SB2_TRY(scr.alloc(&A, knn_tc2_a_halves(sh, n_points)));
  SB2_TRY(scr.alloc(&B, knn_tc2_b_halves(sh, n_points)));
  float* dn = d_dnorm;
  if (!dn) SB2_TRY(scr.alloc(&dn, (size_t)n_points));
  SB2_TRY(knn_tc2_build_images(ctx, sh, d_x, n_points, d, maxnorm, nullptr, 0, A, B, inv_s2, terms == 1 ? dn : nullptr,
                               terms == 1 ? maxnorm + 1 : nullptr));
  const int list_m = 64;
  double fl = 0.0;
  SB2_TRY(knn_tc2_sweep(ctx, sw, sh, A, 0, B, n_points, n_points, list_m, d_score, d_idx, &fl));
  float h_inv = 0.0f;
  unsigned int h_bits[2] = {0, 0};
  SB2_CUDA(cudaMemcpyAsync(&h_inv, inv_s2, 4, cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaMemcpyAsync(h_bits, maxnorm, 8, cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  float r2, dmax;
  memcpy(&r2, &h_bits[0], 4);
  memcpy(&dmax, &h_bits[1], 4);
  double cq, cn;
  knn_tc2_error_coefs(sh, &cq, &cn);
  h_meta[0] = h_inv; h_meta[1] = r2; h_meta[2] = terms == 1 ? dmax : 0.0; h_meta[3] = cq; h_meta[4] = cn; h_meta[5] = list_m;
  return SB2_OK;
}

// knn_tc2.cu — tensor-core sweep of the exact kNN (sm_90a: wgmma m64n128k16 from shared memory + bulk-copy ring).
//
// Per query keep the proposals whose score
//     s(q,c) = q.c - |c|^2/2        (d^2 = |q|^2 - 2 s)
// is largest, plus a rigorous bound on the rounding error of s, so that knn_rescore_kernel can certify the exact fp64
// top-k.  Operand formats (coordinates scaled by a power of two so that max|x| is in [100, 200)):
//   terms = 1  fp16 operands            A = [q_hi | 1 1 1],               B = [c_hi | h0 h1 h2]              K = d+3
//   terms = 3  split fp16 (22 bits)     A = [q_hi | q_hi | q_lo | 1 1 1], B = [c_hi | c_lo | c_hi | h0 h1 h2]  K = 3d+3
// with hi = fp16(x), lo = fp16(x - hi) and h0+h1+h2 = -|c|^2/2 (three-way fp16 split); K is padded to a multiple of 16
// (d = 50: 64 and 160).  knn.cu runs terms = 1 first and re-sweeps the rows it cannot certify with terms = 3.
//
// Shape (one CTA per SM, 9 warps, or 12 in the pipelined loop):
//   CTA = 128 queries x the candidate tiles of 128 points on its list (all of them without the tile screen, below).
//     warps 0-7   two consumer warpgroups; warpgroup g owns query rows 64g..64g+63 and issues, per tile, the k-steps of
//                 wgmma.m64n128k16 (A = its 64 query rows, B = the staged candidate tile, both from shared memory, fp32
//                 accumulators in registers) and examines the 64 x 128 scores in registers.  Pipelined loop (K = 64 and
//                 K = 160 with whole tiles per ring stage): two accumulator sets, tile c+1's MMAs are issued before
//                 the warpgroup examines tile c, so each warpgroup's own MMAs run under its scan.  Otherwise: issue,
//                 wait, hand the stage back, examine (only the other warpgroup's MMAs can overlap).  In the accumulator
//                 fragment a thread holds two rows and, of each, the 32 columns with (column / 2) % 4 = lane % 4; every
//                 (row, lane % 4) keeps its OWN register-resident proposal sub-list (16 or 32 scores in groups of 8 with
//                 group minima; ids write-only to global memory): four disjoint sub-lists per row, no cross-thread
//                 traffic in the loop.  A point outside all four sub-lists of a row scored at most max(tau_0..tau_3),
//                 which is what the re-score certificate uses.
//     warp 8      producer: 1-D cp.async.bulk of pre-arranged candidate images (or K-slices of them) into an mbarrier
//                 ring that takes the shared memory left after the query image (pipelined loop: warps 8-11, so that
//                 setmaxnreg can hand their registers to the consumers)
//   Starting threshold: with the tile screen a per-row seed from its bound u(q); otherwise the first n/16 visits sweep
//   every 16th tile and keep the 6 largest chunk maxima per (row, sub-list); the four sub-lists of a row (four lanes of
//   one warp) are merged by shuffles once and the 6th largest of the 24 seeds all four (rank ~96 of the row;
//   SB2_KNN_EST_RANK picks another of the six).
//   Sweep front: CTAs walk their tile lists cyclically, starting where the running CTAs currently are (g_knn2_front).
#include <cuda_fp16.h>
#include <float.h>

#include <type_traits>
#include <utility>
#include <vector>

#include "common.cuh"
#include "knn_internal.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace tcptx;

constexpr int QM = 128;            // queries per CTA (two warpgroups of M = 64)
constexpr int CN = 128;            // candidates per tile (wgmma N)
constexpr int MAXST = 8;           // upper bound of the ring depth
constexpr int BAR_BYTES = 1024;    // mbarriers IN FRONT of the operand images
constexpr int NCONS = 8;           // consumer warps (two warpgroups)
constexpr int THREADS = (NCONS + 1) * 32;
constexpr int W_PROD = NCONS;
// pipelined loop: the producer gets a warpgroup of its own so that setmaxnreg can move registers from it to the
// consumers (two accumulator sets do not fit the 168 registers a thread gets when 288 or 384 threads share the file)
constexpr int THREADS_PIPE = (NCONS + 4) * 32;
constexpr int PROD_REGS = 40, CONS_REGS = 232;
// k-steps the pipelined loop is compiled for: K = 64 (fp16 operands, d <= 61) and K = 160 (fp16 up to d = 157, split
// fp16 at d = 50); other K axes take the single-buffer loop
constexpr int PIPE_NKS0 = 4, PIPE_NKS1 = 10;
static_assert(128 * PROD_REGS + 256 * CONS_REGS <= 65536 / THREADS_PIPE / 8 * 8 * THREADS_PIPE, "register file");
constexpr int NSUB = 4;            // sub-lists per query row (EST_R, EST_STRIDE: knn_internal.cuh)
constexpr uint32_t SBO = 128;              // bytes between 8-row groups (core matrices contiguous)
constexpr uint32_t LBO = QM * 16;          // bytes between K-chunks of a 128-row image  [kc][row-group][8][8]
static_assert(QM == CN, "query and candidate images share one layout");

// scale: power of two s with s*R in [100, 200]  ->  fp16 range is safe for coordinates and for s^2 R^2/2
__device__ __forceinline__ float tc_scale_from_maxnorm(unsigned int maxnorm_bits) {
  const float R = sqrtf(__uint_as_float(maxnorm_bits));
  if (!(R > 0.0f) || !isfinite(R)) return 1.0f;
  int e = (int)floorf(log2f(200.0f / R));
  e = max(-60, min(60, e));
  return exp2f((float)e);
}

// X[n,d] -> operand images of `tile_rows` points each (128 for query and candidate images), stored exactly as the
// wgmma "no-swizzle, K-major" shared-memory layout wants them (8x8 fp16 core matrices, K-chunk-major), so a tile
// (or a K-slice of it) is staged by ONE 1-D bulk copy.
//   is_a = 1: A = [hi | hi | lo | 1 1 1]  (terms = 3)   or  [hi | 1 1 1]      (terms = 1)
//   is_a = 0: B = [hi | lo | hi | h0 h1 h2]             or  [hi | h0 h1 h2]   with h0+h1+h2 = -|x|^2 s^2 / 2
// gather != nullptr: image row r of tile t is point gather_base + gather[t*tile_rows + r]; rows past n are zero rows
// (A) or score -60000 candidates (B).  dnorm[ps] (optional) = |x_ps - fp16(x_ps)| in the units of X, rounded up, indexed
// by the point ps itself (not its image row); *dmax_bits = its maximum (float bits).
__global__ void __launch_bounds__(256)
knn_tc2_prep_kernel(const float* __restrict__ X, int64_t n, int d, int kpad, int terms, int tile_rows, int is_a,
                    const unsigned int* __restrict__ maxnorm_bits, const int32_t* __restrict__ gather, int64_t gather_base,
                    __half* __restrict__ img, float* __restrict__ inv_s2, float* __restrict__ dnorm,
                    unsigned int* __restrict__ dmax_bits) {
  const int64_t t = blockIdx.x;
  const float s = tc_scale_from_maxnorm(*maxnorm_bits);
  if (t == 0 && threadIdx.x == 0 && inv_s2) *inv_s2 = 1.0f / (s * s);
  __shared__ __half hn3[256][3];
  const int kd = terms * d;  // coordinates on the K axis before the three norm slots
  if ((int)threadIdx.x < tile_rows) {
    const int64_t p = t * tile_rows + threadIdx.x;
    __half h0 = __float2half_rn(-60000.0f), h1 = __float2half_rn(0.0f), h2 = __float2half_rn(0.0f);
    if (p < n) {
      double acc = 0.0, dacc = 0.0;
      const int64_t ps = gather ? gather_base + gather[p] : p;
      for (int k = 0; k < d; ++k) {
        const float xs = X[ps * d + k] * s;
        const double v = (double)xs;
        acc += v * v;
        const double dl = v - (double)__half2float(__float2half_rn(xs));
        dacc += dl * dl;
      }
      if (dnorm) {
        const float dn = __double2float_ru(sqrt(dacc) * (1.0 + 1e-12) / (double)s);
        dnorm[ps] = dn;
        atomicMax(dmax_bits, __float_as_uint(dn));
      }
      const double hn = -0.5 * acc;
      h0 = __float2half_rn((float)hn);
      const double r1 = hn - (double)__half2float(h0);
      h1 = __float2half_rn((float)r1);
      h2 = __float2half_rn((float)(r1 - (double)__half2float(h1)));
    }
    hn3[threadIdx.x][0] = h0; hn3[threadIdx.x][1] = h1; hn3[threadIdx.x][2] = h2;
  }
  __syncthreads();
  const int nkc = kpad / 8;
  __half* out = img + (size_t)t * tile_rows * kpad;
  const size_t lbo = (size_t)tile_rows * 16;
  for (int i = threadIdx.x; i < tile_rows * nkc; i += blockDim.x) {
    const int kc = i / tile_rows, r = i % tile_rows;
    const int64_t p = t * tile_rows + r;
    const int64_t ps = (gather && p < n) ? gather_base + gather[p] : p;
    __align__(16) __half o8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = kc * 8 + j;
      __half v = __float2half_rn(0.0f);
      if (p < n) {
        if (e < kd) {
          const int seg = e / d, k = e - seg * d;
          const float xs = X[ps * d + k] * s;
          const __half hi = __float2half_rn(xs);
          const __half lo = __float2half_rn(xs - __half2float(hi));
          v = is_a ? (seg == 2 ? lo : hi) : (seg == 1 ? lo : hi);   // A = [hi | hi | lo], B = [hi | lo | hi]
        } else if (e < kd + 3) {
          v = is_a ? __float2half_rn(1.0f) : hn3[r][e - kd];
        }
      } else if (e == kd && !is_a) {
        v = hn3[r][0];  // padding candidates: score -60000 (padding queries are all-zero rows)
      }
      o8[j] = v;
    }
    const size_t off = ((size_t)kc * lbo + (size_t)(r >> 3) * SBO + (size_t)(r & 7) * 16) / 2;  // in halves
    *reinterpret_cast<uint4*>(out + off) = *reinterpret_cast<const uint4*>(o8);
  }
}

// ------------------------------------------------------------------------------------------------
// Per-(row, column quarter) proposal sub-list: 8*NG scores in REGISTERS (groups of 8 with a running minimum per
// group), ids in global memory (write-only).  tau = min of the sub-list = the score a candidate must beat.  All
// indexing is static (macro-expanded), so nothing spills and an insertion never waits on memory.
template <int NG>
struct SubList {
  float ls[8 * NG];
  float gm[NG];
  float tau;
};
__device__ __forceinline__ float min8(const float* x) {
  return fminf(fminf(fminf(x[0], x[1]), fminf(x[2], x[3])), fminf(fminf(x[4], x[5]), fminf(x[6], x[7])));
}
#define SB2_GROUP_INSERT2(G)                                                  \
  {                                                                           \
    bool placed = false;                                                      \
    _Pragma("unroll") for (int i = 0; i < 8; ++i) {                           \
      const bool hset = !placed && (L.ls[(G) * 8 + i] == L.tau);              \
      L.ls[(G) * 8 + i] = hset ? v : L.ls[(G) * 8 + i];                       \
      pos = hset ? ((G) * 8 + i) : pos;                                       \
      placed |= hset;                                                         \
    }                                                                         \
    L.gm[(G)] = min8(&L.ls[(G) * 8]);                                         \
  }
template <int NG>
__device__ __forceinline__ void list_insert(SubList<NG>& L, int32_t* __restrict__ id, float v, int32_t cand) {
  static_assert(NG == 2 || NG == 4, "sub-lists hold 16 or 32 proposals");
  int pos = 0;
  if (L.gm[0] == L.tau) SB2_GROUP_INSERT2(0)
  else if (NG == 2 || L.gm[1] == L.tau) SB2_GROUP_INSERT2(1)
  else if (L.gm[2 % NG] == L.tau) SB2_GROUP_INSERT2(2 % NG)
  else SB2_GROUP_INSERT2(3 % NG)
  id[pos] = cand;
  float t = L.gm[0];
#pragma unroll
  for (int g = 1; g < NG; ++g) t = fminf(t, L.gm[g]);
  L.tau = t;
}
__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float max8u(const uint32_t* v) {
  return fmax3(fmax3(__uint_as_float(v[0]), __uint_as_float(v[1]), __uint_as_float(v[2])),
               fmax3(__uint_as_float(v[3]), __uint_as_float(v[4]), __uint_as_float(v[5])),
               fmaxf(__uint_as_float(v[6]), __uint_as_float(v[7])));
}
// A thread examines one 32-value chunk of each of its two rows per tile (values already in registers; value m is
// candidate cand0 + 8 (m / 2) + m % 2, the columns one thread holds in the wgmma accumulator fragment).
// Fast path: "does anything in the chunk beat tau", one max tree and one compare per row.
//   chunk_imax (ISCAN, the default): the signed-integer maximum of the 32 raw bit patterns, a ternary tree of Hopper's
//     three-input integer max (VIMNMX3: 15 of them and one VIMNMX, against 31 FMNMX), compared with tau's bit pattern.
//     Exact whenever tau's sign bit is clear: a float above a non-negative tau is positive, positive floats order like
//     their patterns, and a negative value's pattern is a negative integer, below every non-negative pattern, so where
//     the negative values fall among themselves never matters.  Scores are finite (padding candidates score -60000),
//     and tau = +inf (rows past n_query) is above every finite pattern.
//   chunk_max: the float maximum, a tree of four independent quarter maxima.  The estimate phase needs the value itself,
//     and the hit test needs it while tau's sign bit is set (a cold start begins at -inf; rows near the origin keep a
//     negative tau): a warp with such a row takes the rare branch and redoes the test of both rows in floats there, so
//     the fast path pays one OR and one compare for the rule.
// Rare path (insert_hits), entered by the whole warp when any of its 64 (row, sub-list) pairs has a hit: a 32-bit mask
// of the values above tau (one compare each), walked lowest bit first with __ffs; each set bit's value is picked out of
// the registers by a five-level select tree and inserted if it still beats tau (every insertion raises tau).  So the
// values of a chunk go in column by column, not largest first: the scores a sub-list ends with do not depend on that
// order, only which of several EQUAL scores at tau it keeps, and those lie below every score the certificate accepts
// (a row whose k-th score ties tau is re-swept or scanned exactly), so the final (idx, dist) do not either.
// stamp(PH_SCAN) / stamp(PH_INSERT) bracket the rare path for the opt-in phase stamps (no-ops when they are off).
enum { PH_WAIT = 0, PH_MMA, PH_SCAN, PH_INSERT, PH_N };
// per (CTA, warpgroup) the stamps buffer holds the PH_N phase totals and two counters of the STAMPS instantiation:
// warp-tiles of the sweep proper on which a warp took the rare path, and insertions into the warpgroup's sub-lists
enum { CNT_RARE = PH_N, CNT_INSERT, ST_N };
__device__ __forceinline__ float chunk_max(const uint32_t (&v)[32]) {
  return fmaxf(fmax3(max8u(&v[0]), max8u(&v[8]), max8u(&v[16])), max8u(&v[24]));
}
__device__ __forceinline__ int chunk_imax(const uint32_t (&v)[32]) {
  int a[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) a[i] = __vimax3_s32((int)v[3 * i], (int)v[3 * i + 1], (int)v[3 * i + 2]);
  const int b0 = __vimax3_s32(a[0], a[1], a[2]), b1 = __vimax3_s32(a[3], a[4], a[5]), b2 = __vimax3_s32(a[6], a[7], a[8]);
  const int b3 = __vimax3_s32(a[9], (int)v[30], (int)v[31]);
  return max(__vimax3_s32(b0, b1, b2), b3);
}
template <int NG, bool COUNT>
__device__ __forceinline__ void insert_hits(SubList<NG>& L, int32_t* __restrict__ id, const uint32_t (&v)[32], int32_t cand0,
                                            int32_t n_points, unsigned& n_ins) {
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 32; ++i) m |= (__uint_as_float(v[i]) > L.tau ? 1u : 0u) << i;
  while (m) {
    const int j = __ffs(m) - 1;
    m &= m - 1;
    uint32_t s[16];   // v[j]: registers cannot be indexed at run time
#pragma unroll
    for (int i = 0; i < 16; ++i) s[i] = (j & 1) ? v[2 * i + 1] : v[2 * i];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = (j & 2) ? s[2 * i + 1] : s[2 * i];
#pragma unroll
    for (int i = 0; i < 4; ++i) s[i] = (j & 4) ? s[2 * i + 1] : s[2 * i];
#pragma unroll
    for (int i = 0; i < 2; ++i) s[i] = (j & 8) ? s[2 * i + 1] : s[2 * i];
    const float x = __uint_as_float((j & 16) ? s[1] : s[0]);
    const int32_t cand = cand0 + ((j >> 1) << 3) + (j & 1);
    if (x > L.tau && cand < n_points) {
      list_insert(L, id, x, cand);
      if (COUNT) ++n_ins;
    }
  }
}
// estimate phase: keep the EST_R largest values seen (sorted descending), branch-free
template <int LEN>
__device__ __forceinline__ void est_push(float (&est)[LEN], float cm) {
#pragma unroll
  for (int i = 0; i < EST_R; ++i) {
    const float hi = fmaxf(est[i], cm);
    cm = fminf(est[i], cm);
    est[i] = hi;
  }
}
template <int LEN>
__device__ __forceinline__ void est_chunk(float (&est)[LEN], const uint32_t (&v)[32]) {
  est_push(est, chunk_max(v));
}

// nks = k-steps (16 columns of the K axis) per staged slice, nsplit = slices per candidate image.  lists / list_len:
// the ascending candidate tiles of each CTA, from lists[list_off[cta]] or lists[cta * list_stride] (list_stride = 0 and
// list_len = nullptr: one list of all n_btiles tiles);
// seed (optional): each launch row's starting threshold in place of the sampled estimate.
// Sweep front: CTAs walk their lists cyclically, each starting at the first entry at or after the tile where the CTAs
// already running currently are (the order of the candidates is irrelevant to the result).  All resident CTAs then stream the same few tiles at the
// same time and the candidate images (166 MB at 1.3M x 50, more than the L2) are read from HBM about once per wave of
// CTAs instead of once per CTA.  "Where the running CTAs are" is the MEAN position of the pack, (sweep visits so far) /
// (resident CTAs): starting a new CTA at the position last published by ANY running CTA lets the spread of the pack
// grow from wave to wave; re-centring every new CTA on the mean bounds it by the drift of a single lap.  Progress is
// counted in tiles advanced along the walk (not visits), so that CTAs with short lists keep pace in tile space.
__device__ unsigned long long g_knn2_front;   // tiles the sweep-proper walks of all CTAs of this launch have advanced
// PNKS = 0: single-buffer loop.  Per tile, a warpgroup issues its nks k-steps, waits for all of them, releases the stage
//   and scans; the only overlap is whatever the other warpgroup's MMAs happen to do meanwhile.  Any nsplit / nstage.
// PNKS > 0: pipelined loop, nks = PNKS.  Two accumulator sets; tile c+1's MMAs are issued (and run) while the warpgroup
//   scans tile c, so every warpgroup keeps the tensor pipe fed on its own.  A warpgroup then holds two ring stages at a
//   time: needs nsplit = 1 and nstage >= 3 (knn_tc2_shape sets KnnTc2Shape::pipe), and 384 threads (THREADS_PIPE,
//   registers rebalanced).  The k-step count is a template argument because ptxas serialises every wgmma of the kernel
//   when a loop with a run-time trip count issues them while another group is in flight.
// STAMPS: lane 0 of warp 0 of each consumer warpgroup adds up clock64() per phase (PH_WAIT on full[s], PH_MMA issue to
//   end of the wgmma wait, PH_SCAN examination incl. estimate / seeding / release, PH_INSERT the rare path,
//   insert_hits) in shared memory and writes stamps[(cta * 2 + warpgroup) * ST_N + phase] at the end; every warp adds
//   its rare-path tiles and insertions to the CNT_RARE / CNT_INSERT slots.  A template
//   argument, not a run-time test: even never-taken uniform branches inside the scan cost the single-buffer loop 8 %
//   (they split the examination into blocks the scheduler cannot interleave).
// ISCAN: the fast path's hit test on the bit patterns (chunk_imax); false keeps the float max tree (SB2_KNN_SCAN=float).
template <int NG, int PNKS, bool STAMPS, bool ISCAN>
__global__ void __launch_bounds__(PNKS > 0 ? THREADS_PIPE : THREADS, 1)
knn_sweep2_kernel(const __half* __restrict__ Aimg, const __half* __restrict__ Bimg, int nks, int nsplit, int nstage,
                  int64_t n_btiles, int64_t n_est, int64_t est_stride, int est_rank, int64_t qtile0, int64_t n_query,
                  int32_t n_points, const int32_t* __restrict__ lists, int64_t list_stride, const int64_t* __restrict__ list_off,
                  const int32_t* __restrict__ list_len,
                  const float* __restrict__ seed, float* __restrict__ cand_score, int32_t* __restrict__ cand_idx,
                  unsigned long long* __restrict__ stamps) {
  constexpr bool PIPE = PNKS > 0;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t part_b = (uint32_t)(CN * 16 * 2) * (uint32_t)nks;     // bytes per staged K-slice of a candidate image
  const uint32_t tile_b = part_b * (uint32_t)nsplit;                    // bytes per 128-row image (query or candidate)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
  unsigned char* As = smem_raw + BAR_BYTES;
  unsigned char* Bs0 = As + tile_b;
  uint64_t* full = bars;                  // [MAXST] producer -> consumers
  uint64_t* empty = bars + MAXST;         // [MAXST] consumer warps -> producer
  uint64_t* afull = bars + 2 * MAXST;     // [1]
  int32_t* start_pos = reinterpret_cast<int32_t*>(bars + 2 * MAXST + 1);
  unsigned long long* stamp_sm = reinterpret_cast<unsigned long long*>(bars + 2 * MAXST + 2);  // [2][PH_N + 1]
  static_assert((2 * MAXST + 2 + 2 * (PH_N + 1)) * 8 <= BAR_BYTES, "barrier block");

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  // the candidate tiles this CTA visits after its estimate: lst[0, len), ascending
  const int32_t* lst = lists + (list_off ? list_off[blockIdx.x] : (int64_t)blockIdx.x * list_stride);
  const int32_t len = list_len ? list_len[blockIdx.x] : (int32_t)n_btiles;
  if (threadIdx.x == 0) {
    for (int s = 0; s < nstage; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NCONS); }
    mbar_init(afull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const unsigned long long f = *reinterpret_cast<volatile unsigned long long*>(&g_knn2_front);
    unsigned int nsm;
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsm));
    const unsigned long long resident = min((unsigned long long)gridDim.x, (unsigned long long)max(nsm, 1u));
    // mean tile of the pack now, plus the n_est visits this CTA spends on its threshold estimate before it joins; the
    // walk starts at the first list entry at or after it
    const int32_t pos = (int32_t)((f / resident + (unsigned long long)n_est) % (unsigned long long)n_btiles);
    int32_t lo = 0, hi = len;
    while (lo < hi) {
      const int32_t mid = (lo + hi) >> 1;
      if (lst[mid] < pos) lo = mid + 1;
      else hi = mid;
    }
    *start_pos = lo == len ? 0 : lo;
  }
  __syncthreads();

  if (warp >= W_PROD) {
    // ---------------- producer ----------------
    if constexpr (PIPE) setmaxnreg_dec<PROD_REGS>();
    if (warp == W_PROD && lane == 0) {
      mbar_expect_tx(afull, tile_b);
      bulk_g2s(As, reinterpret_cast<const unsigned char*>(Aimg) + (size_t)(qtile0 + (int64_t)blockIdx.x) * tile_b, tile_b, afull);
      // visit order: n_est sample tiles (every est_stride-th) for the threshold estimate, then every tile
      int s = 0;
      uint32_t use_phase = 1;  // parity of the previous use of stage s (first lap: nothing to wait for)
      bool first_lap = true;
      int32_t cs = *start_pos;   // cyclic walk of the list
      for (int64_t v = 0; v < n_est + len; ++v) {
        int64_t c = v * est_stride;
        if (v >= n_est) { c = lst[cs]; if (++cs == len) cs = 0; }
        for (int p = 0; p < nsplit; ++p) {
          if (!first_lap) mbar_wait(&empty[s], use_phase);
          mbar_expect_tx(&full[s], part_b);
          bulk_g2s(Bs0 + (size_t)s * part_b, reinterpret_cast<const unsigned char*>(Bimg) + (size_t)c * tile_b + (size_t)p * part_b,
                   part_b, &full[s]);
          if (++s == nstage) { s = 0; use_phase ^= 1u; first_lap = false; }
        }
      }
    }
    return;
  }

  // ---------------- consumers: thread <-> (two query rows, sub-list lane % 4) ----------------
  if constexpr (PIPE) setmaxnreg_inc<CONS_REGS>();
  const int g = warp >> 2;                                   // warpgroup: query rows 64g .. 64g+63
  const int sl = lane & 3;                                   // sub-list = column class of the fragment
  const int row0 = 64 * g + 16 * (warp & 3) + (lane >> 2);   // rows row0 and row0 + 8
  const int64_t ql0 = (int64_t)blockIdx.x * QM + row0, ql1 = ql0 + 8;
  const bool valid0 = ql0 < n_query, valid1 = ql1 < n_query;
  constexpr int LS = 8 * NG, LM = NSUB * LS;
  float* sc0 = cand_score + (valid0 ? ql0 : 0) * LM + sl * LS;
  float* sc1 = cand_score + (valid1 ? ql1 : 0) * LM + sl * LS;
  int32_t* id0 = cand_idx + (valid0 ? ql0 : 0) * LM + sl * LS;
  int32_t* id1 = cand_idx + (valid1 ? ql1 : 0) * LM + sl * LS;
  SubList<NG> L0, L1;
  L0.tau = INFINITY;
  L1.tau = INFINITY;
#pragma unroll
  for (int i = 0; i < LS; ++i) {
    if (valid0) id0[i] = -1;
    if (valid1) id1[i] = -1;
  }
  // During the estimate phase the EST_R running chunk maxima live in L.ls[0..EST_R) (the sub-list proper does not exist
  // yet): one register array serves both phases.
  static_assert(EST_R <= LS, "estimate aliases the list registers");
#pragma unroll
  for (int i = 0; i < LS; ++i) { L0.ls[i] = -INFINITY; L1.ls[i] = -INFINITY; }
  // descriptors: A = this warpgroup's 64 rows of the query image, B = ring stage 0; one k-step (two 8-column K-chunks)
  // advances the start address by 2 * LBO bytes (the address field counts 16-byte units)
  const uint64_t da0 = wgmma_desc(smem_u32(As) + (uint32_t)g * 8u * SBO, LBO, SBO);
  const uint64_t db0 = wgmma_desc(smem_u32(Bs0), LBO, SBO);
  constexpr uint32_t KSTEP16 = (2u * LBO) >> 4;
  const uint32_t part16 = part_b >> 4;
  const int n_visit = (int)(n_est + len), n_est_i = (int)n_est;
  int32_t lpos = *start_pos;                   // list position of the current sweep visit (cyclic walk)
  int32_t ctile = lst[lpos];                   // its candidate tile
  int32_t cbase = ctile * CN + 2 * sl;
  const int32_t n_bt = (int32_t)n_btiles;
  uint32_t adv = 0;                            // warp 0 lane 0: tiles the walk advanced since the last front update

  // phase stamps (opt-in): no code at all without STAMPS
  const bool stamp_on = STAMPS && (warp & 3) == 0;
  unsigned long long* my_st = stamp_sm + g * (PH_N + 1);   // [PH_N] totals, [PH_N] clock of the previous stamp
  const auto stamp = [&](int ph) {
    if (stamp_on) {
      __syncwarp();
      if (lane == 0) {
        const unsigned long long now = (unsigned long long)clock64();
        my_st[ph] += now - my_st[PH_N];
        my_st[PH_N] = now;
      }
    }
  };

  unsigned n_ins = 0, n_rare = 0;   // STAMPS: this thread's insertions, this warp's rare-path tiles

  // everything a warpgroup does with the scores of visit c once they are in acc
  const auto examine = [&](const float (&acc)[64], int c) {
    if (c == n_est_i) {
      // start of the sweep proper: seed the sub-lists.  With an estimate phase the four sub-lists of a row (lanes
      // lane ^ 1, ^ 2, ^ 3) are merged: the 6th largest of their 24 chunk maxima sits at about rank 6 * est_stride = 96
      // of the row; without one the lists start cold (-inf).  Any value is safe: the certificate uses the final tau.
      if (n_est_i > 0) {
        float o0[EST_R], o1[EST_R];
#pragma unroll
        for (int i = 0; i < EST_R; ++i) { o0[i] = L0.ls[i]; o1[i] = L1.ls[i]; }
#pragma unroll
        for (int o = 1; o < NSUB; ++o) {
#pragma unroll
          for (int i = 0; i < EST_R; ++i) {
            est_push(L0.ls, __shfl_xor_sync(0xffffffffu, o0[i], o));
            est_push(L1.ls, __shfl_xor_sync(0xffffffffu, o1[i], o));
          }
        }
      }
      float e0 = L0.ls[0], e1 = L1.ls[0];    // the est_rank-th largest of the merged chunk maxima
#pragma unroll
      for (int i = 1; i < EST_R; ++i) {
        e0 = i < est_rank ? L0.ls[i] : e0;
        e1 = i < est_rank ? L1.ls[i] : e1;
      }
      // rows past n_query never accept anything; a per-row seed (from the tile screen's bound) replaces the estimate
      const float t0 = valid0 ? (seed ? seed[ql0] : e0) : INFINITY;
      const float t1 = valid1 ? (seed ? seed[ql1] : e1) : INFINITY;
#pragma unroll
      for (int i = 0; i < LS; ++i) { L0.ls[i] = t0; L1.ls[i] = t1; }
#pragma unroll
      for (int gi = 0; gi < NG; ++gi) { L0.gm[gi] = t0; L1.gm[gi] = t1; }
      L0.tau = t0;
      L1.tau = t1;
    }
    uint32_t v0[32], v1[32];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      v0[2 * i] = __float_as_uint(acc[4 * i]);
      v0[2 * i + 1] = __float_as_uint(acc[4 * i + 1]);
      v1[2 * i] = __float_as_uint(acc[4 * i + 2]);
      v1[2 * i + 1] = __float_as_uint(acc[4 * i + 3]);
    }
    if (c < n_est_i) {
      est_chunk(L0.ls, v0);
      est_chunk(L1.ls, v1);
    } else {
      const int32_t npos = lpos + 1 == len ? 0 : lpos + 1;
      const int32_t ntile = lst[npos];   // the next visit's tile, loaded under the scan
      bool hit0, hit1, redo = false;
      if constexpr (ISCAN) {
        const int t0 = __float_as_int(L0.tau), t1 = __float_as_int(L1.tau);
        hit0 = chunk_imax(v0) > t0;
        hit1 = chunk_imax(v1) > t1;
        redo = (t0 | t1) < 0;   // a sign bit is set: the integer test of this thread's rows proves nothing
      } else {
        hit0 = chunk_max(v0) > L0.tau;
        hit1 = chunk_max(v1) > L1.tau;
      }
      stamp(PH_SCAN);
      if (__builtin_expect(__any_sync(0xffffffffu, hit0 || hit1 || redo), 0)) {
        bool rare = true;
        if constexpr (ISCAN) {
          if (__any_sync(0xffffffffu, redo)) {
            hit0 = chunk_max(v0) > L0.tau;
            hit1 = chunk_max(v1) > L1.tau;
            rare = __any_sync(0xffffffffu, hit0 || hit1);
          }
        }
        if (rare) {
          if (STAMPS) ++n_rare;
          if (hit0) insert_hits<NG, STAMPS>(L0, id0, v0, cbase, n_points, n_ins);
          if (hit1) insert_hits<NG, STAMPS>(L1, id1, v1, cbase, n_points, n_ins);
        }
      }
      stamp(PH_INSERT);
      if (warp == 0 && lane == 0) {   // the pack's front, in tiles, published every 16 visits
        adv += (uint32_t)(ntile > ctile ? ntile - ctile : ntile - ctile + n_bt);
        if ((c & 15) == 0) { atomicAdd(&g_knn2_front, (unsigned long long)adv); adv = 0; }
      }
      lpos = npos;
      ctile = ntile;
      cbase = ntile * CN + 2 * sl;
    }
  };

  mbar_wait(afull, 0);
  if (stamp_on && lane == 0) {
    for (int ph = 0; ph < PH_N; ++ph) my_st[ph] = 0ull;
    my_st[PH_N] = (unsigned long long)clock64();
  }
  if constexpr (PIPE) {
    // steady state per warpgroup: wait full[stage(c+1)], issue tile c+1 into the other accumulator set, wait until
    // only that group is in flight, release stage(c), examine tile c under tile c+1's MMAs.  The loop is unrolled by
    // two so that both accumulator sets keep static register indices.
    float accA[64], accB[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { accA[i] = 0.0f; accB[i] = 0.0f; }
    int s_iss = 0, s_rel = 0;     // ring stage of the next tile to issue / of the tile to examine next
    uint32_t ph_iss = 0;
    const auto issue = [&](float (&acc)[64]) {
      mbar_wait(&full[s_iss], ph_iss);
      stamp(PH_WAIT);
      wgmma_fence_operand(acc);
      wgmma_fence();
      const uint64_t db = db0 + (uint64_t)((uint32_t)s_iss * part16);
#pragma unroll
      for (int j = 0; j < PNKS; ++j)
        wgmma_m64n128k16_f16(acc, da0 + (uint64_t)((uint32_t)j * KSTEP16), db + (uint64_t)((uint32_t)j * KSTEP16), j != 0);
      wgmma_commit();
      if (++s_iss == nstage) { s_iss = 0; ph_iss ^= 1u; }
    };
    const auto release = [&]() {
      // this warp's reads of the stage are complete: the eighth arrival lets the producer refill it
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s_rel]);
      if (++s_rel == nstage) s_rel = 0;
    };
    // tile c is in flight in cur: issue tile c+1 into nxt, examine tile c
    const auto step = [&](float (&cur)[64], float (&nxt)[64], int c) {
      issue(nxt);
      wgmma_wait<1>();     // tile c's group is complete, tile c+1's still runs
      wgmma_fence_operand(cur);
      stamp(PH_MMA);
      release();
      examine(cur, c);
      stamp(PH_SCAN);
    };
    // the last tile, in flight in cur
    const auto last = [&](float (&cur)[64], int c) {
      wgmma_wait<0>();
      wgmma_fence_operand(cur);
      stamp(PH_MMA);
      release();
      examine(cur, c);
      stamp(PH_SCAN);
    };
    // each exit has its own epilogue: merging the two sets after the loop (or testing "is there a next tile" apart
    // from the loop exit) makes ptxas see accumulator copies while a group is in flight and serialise every wgmma
    issue(accA);
    stamp(PH_MMA);
    for (int c = 0;; c += 2) {
      if (c + 1 == n_visit) { last(accA, c); break; }
      step(accA, accB, c);
      if (c + 2 == n_visit) { last(accB, c + 1); break; }
      step(accB, accA, c + 1);
    }
  } else {
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
    int s = 0;
    uint32_t ring_phase = 0;
    for (int c = 0; c < n_visit; ++c) {
      for (int p = 0; p < nsplit; ++p) {
        mbar_wait(&full[s], ring_phase);
        stamp(PH_WAIT);
        wgmma_fence();
        const uint64_t da = da0 + (uint64_t)((uint32_t)(p * nks) * KSTEP16);
        const uint64_t db = db0 + (uint64_t)((uint32_t)s * part16);
        for (int j = 0; j < nks; ++j)
          wgmma_m64n128k16_f16(acc, da + (uint64_t)((uint32_t)j * KSTEP16), db + (uint64_t)((uint32_t)j * KSTEP16), (p | j) != 0);
        wgmma_commit();
        wgmma_wait_all();
        stamp(PH_MMA);
        // this warp's reads of the stage are complete: the eighth arrival lets the producer refill it
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        if (++s == nstage) { s = 0; ring_phase ^= 1u; }
      }
      examine(acc, c);
      stamp(PH_SCAN);
    }
  }
  if (STAMPS) {
    unsigned long long* st = stamps + ((size_t)blockIdx.x * 2 + g) * ST_N;   // zeroed by the host
    const unsigned ins = __reduce_add_sync(0xffffffffu, n_ins);
    if (lane == 0) {
      atomicAdd(&st[CNT_RARE], (unsigned long long)n_rare);
      atomicAdd(&st[CNT_INSERT], (unsigned long long)ins);
    }
    if (stamp_on && lane == 0) {
      for (int ph = 0; ph < PH_N; ++ph) st[ph] = my_st[ph];
    }
  }
  if (valid0) {
#pragma unroll
    for (int i = 0; i < LS; ++i) sc0[i] = L0.ls[i];
  }
  if (valid1) {
#pragma unroll
    for (int i = 0; i < LS; ++i) sc1[i] = L1.ls[i];
  }
}


// ------------------------------------------------------------------------------------------------
// Tile-compact order and tile screen (SB2_KNN_SCREEN, on by default from 512 candidate tiles).
//
// kd order: the points are split recursively, each segment at a multiple of 128 points along its (sampled) principal
// direction, until every segment is one tile; knn.cu builds the fp16 images in that order, so each 128-point
// candidate tile and each 128-row query block is spatially compact.  Per tile a centre mu_t and a radius r_t bound every
// point of the tile: |q - x| >= |q - mu_t| - r_t.  The screen scores every query row against every centre on the tensor
// cores (the centres go through the same image builder) and keeps, per query block, the tiles for which some row has
// |q - mu_t| - r_t <= u(q), where u(q) >= d_k(q) comes from a short sweep of the block's own neighbourhood.  A skipped
// tile holds no point within u(q) of any row of the block; the re-score checks d_k(q) <= u(q) before it certifies a row.
constexpr int KD_SAMPLES = 512;   // points per segment the split direction is chosen from
constexpr int KD_THREADS = 1024;
constexpr int KD_POWER_ITERS = 12;                // power iterations of the split direction
constexpr int KD_SAMPLE_SMEM = 200 * 1024;        // bytes of shared memory the direction's fp32 sample may take
constexpr int KD_MAX_D = 150;                     // the kNN's largest d

// Points in the sample of the direction kernel: KD_SAMPLES, fewer for d > 100 so the sample fits KD_SAMPLE_SMEM.
constexpr int KD_DIR_PARTS = 256;   // the direction kernel's threads: partial sums of its scatter product, parts x d <= 256
int kd_dir_samples(int d) { return std::min(KD_SAMPLES, KD_SAMPLE_SMEM / (4 * (d | 1))); }
size_t kd_dir_smem(int d, int ns) { return (size_t)(3 * d + KD_DIR_PARTS + ns) * sizeof(double) + (size_t)ns * (d | 1) * sizeof(float); }

// segment s of a level = [seg[3s], seg[3s+2]), split at seg[3s+1]: dir[s * (d + 1) ..] = its principal direction v (unit,
// largest |v_j| positive) and the offset mu . v, from an evenly spaced sample of ns_max (or all) of its points, all in
// fp64 and in a fixed order.  The sample is centred; KD_POWER_ITERS power iterations on its scatter start from the
// coordinate of largest variance (a sample without spread keeps that coordinate).  Any direction is correct: it only
// makes the tiles tight.
__global__ void __launch_bounds__(256) kd_dir_kernel(const float* __restrict__ X, int d, const int32_t* __restrict__ P,
                                                     const int32_t* __restrict__ seg, int ns_max, double* __restrict__ dir) {
  extern __shared__ double kd_sm[];
  const int ds = d | 1;   // odd row stride: a thread per sample row reads without bank conflicts
  double* mu = kd_sm;     // [d]
  double* v = mu + d;     // [d]
  double* u = v + d;      // [d]
  const int np = max(1, (int)blockDim.x / d);   // parts of the sample the scatter product is summed in
  double* part = u + d;                         // [np][d], np d <= KD_DIR_PARTS
  double* w = part + KD_DIR_PARTS;              // [ns]
  const int64_t a = seg[3 * blockIdx.x], len = seg[3 * blockIdx.x + 2] - a;
  const int ns = (int)min(len, (int64_t)ns_max);
  float* xs = reinterpret_cast<float*>(w + ns);   // [ns][ds]
  __shared__ double s_norm;
  __shared__ int s_best;
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = tid >> 5, nwarps = blockDim.x >> 5;
  for (int t0 = warp; t0 < ns; t0 += 4 * nwarps) {   // a warp per sample row, four rows in flight
    int64_t row[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int t = t0 + r * nwarps;
      row[r] = t < ns ? (int64_t)P[a + t * len / ns] * d : -1;
    }
    for (int j = lane; j < d; j += 32)
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (row[r] >= 0) xs[(t0 + r * nwarps) * ds + j] = X[row[r] + j];
  }
  __syncthreads();
  for (int j = tid; j < d; j += blockDim.x) {
    double s = 0.0;
    for (int t = 0; t < ns; ++t) s += xs[t * ds + j];
    mu[j] = s / ns;
  }
  __syncthreads();
  for (int j = tid; j < d; j += blockDim.x) {
    double s2 = 0.0;
    for (int t = 0; t < ns; ++t) {
      const double c = xs[t * ds + j] - mu[j];
      s2 = fma(c, c, s2);
    }
    u[j] = s2;
  }
  __syncthreads();
  if (tid == 0) {
    int best = 0;
    for (int j = 1; j < d; ++j)
      if (u[j] > u[best]) best = j;
    s_best = best;
  }
  __syncthreads();
  for (int j = tid; j < d; j += blockDim.x) v[j] = j == s_best ? 1.0 : 0.0;
  __syncthreads();
  for (int it = 0; it < KD_POWER_ITERS; ++it) {
    for (int t = tid; t < ns; t += blockDim.x) {   // w = (X_s - mu) v
      double acc = 0.0;
      for (int j = 0; j < d; ++j) acc = fma(xs[t * ds + j] - mu[j], v[j], acc);
      w[t] = acc;
    }
    __syncthreads();
    for (int e = tid; e < np * d; e += blockDim.x) {   // u = (X_s - mu)^T w, in np parts of the sample
      const int h = e / d, j = e - h * d;
      double acc = 0.0;
      for (int t = h * ns / np; t < (h + 1) * ns / np; ++t) acc = fma(xs[t * ds + j] - mu[j], w[t], acc);
      part[e] = acc;
    }
    __syncthreads();
    if (tid < 32) {
      double s2 = 0.0;
      for (int j = lane; j < d; j += 32) {
        double x = part[j];
        for (int h = 1; h < np; ++h) x += part[h * d + j];
        u[j] = x;
        s2 = fma(x, x, s2);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      if (lane == 0) s_norm = sqrt(s2);
    }
    __syncthreads();
    const double nrm = s_norm;
    if (!(nrm > 0.0) || !isfinite(nrm)) break;   // no spread in the sample: keep the current direction
    for (int j = tid; j < d; j += blockDim.x) v[j] = u[j] / nrm;
    __syncthreads();
  }
  if (tid == 0) {   // the sign: the largest |v_j| (the first of equals) positive
    int best = 0;
    for (int j = 1; j < d; ++j)
      if (fabs(v[j]) > fabs(v[best])) best = j;
    const double sg = v[best] < 0.0 ? -1.0 : 1.0;
    double off = 0.0;
    for (int j = 0; j < d; ++j) {
      const double vj = sg * v[j];
      dir[(int64_t)blockIdx.x * (d + 1) + j] = vj;
      off = fma(mu[j], vj, off);
    }
    dir[(int64_t)blockIdx.x * (d + 1) + d] = off;
  }
}

// SB2_KNN_SPLIT=coord: the segment's coordinate of largest variance over the same evenly spaced sample
__global__ void __launch_bounds__(256) kd_axis_kernel(const float* __restrict__ X, int d, const int32_t* __restrict__ P,
                                                      const int32_t* __restrict__ seg, int32_t* __restrict__ axis) {
  __shared__ double var[256];
  const int64_t a = seg[3 * blockIdx.x], len = seg[3 * blockIdx.x + 2] - a;
  const int64_t ns = min(len, (int64_t)KD_SAMPLES);
  const int j = threadIdx.x;
  if (j < d) {
    double s = 0.0, s2 = 0.0;
    for (int64_t t = 0; t < ns; ++t) {
      const double v = X[(int64_t)P[a + t * len / ns] * d + j];
      s += v;
      s2 += v * v;
    }
    var[j] = s2 - s * s / (double)ns;
  }
  __syncthreads();
  if (j == 0) {
    int best = 0;
    for (int i = 1; i < d; ++i)
      if (var[i] > var[best]) best = i;
    axis[blockIdx.x] = best;
  }
}

// the split keys: ord_bits(fp32(x . v - mu . v)) (the dot in fp64, in coordinate order), or with axis the coordinate itself
__global__ void __launch_bounds__(256) kd_keys_kernel(const float* __restrict__ X, int d, const int32_t* __restrict__ P,
                                                      const int32_t* __restrict__ seg, const double* __restrict__ dir,
                                                      const int32_t* __restrict__ axis, uint32_t* __restrict__ key) {
  __shared__ double v[KD_MAX_D + 1];
  const int64_t a = seg[3 * blockIdx.x], b = seg[3 * blockIdx.x + 2];
  if (axis) {
    const int ax = axis[blockIdx.x];
    for (int64_t i = a + (int64_t)blockIdx.y * blockDim.x + threadIdx.x; i < b; i += (int64_t)gridDim.y * blockDim.x)
      key[i] = ord_bits(X[(int64_t)P[i] * d + ax]);
    return;
  }
  // a warp stages its 32 rows in shared memory, each row read whole by the warp, then a thread takes a row
  extern __shared__ float kd_rows[];
  const int lane = threadIdx.x & 31, ds = d | 1;
  float* rows = kd_rows + (threadIdx.x >> 5) * 32 * ds;
  for (int j = threadIdx.x; j <= d; j += blockDim.x) v[j] = dir[(int64_t)blockIdx.x * (d + 1) + j];
  __syncthreads();
  for (int64_t base = a + ((int64_t)blockIdx.y * blockDim.x + (threadIdx.x & ~31)); base < b; base += (int64_t)gridDim.y * blockDim.x) {
    const int64_t i = base + lane;
    const int32_t p = i < b ? P[i] : -1;
#pragma unroll 8
    for (int r = 0; r < 32; ++r) {
      const int32_t pr = __shfl_sync(0xffffffffu, p, r);
      if (pr >= 0)
        for (int j = lane; j < d; j += 32) rows[r * ds + j] = X[(int64_t)pr * d + j];
    }
    __syncwarp();
    if (i < b) {
      double acc = 0.0;
      for (int j = 0; j < d; ++j) acc = fma((double)rows[lane * ds + j], v[j], acc);
      key[i] = ord_bits((float)(acc - v[d]));
    }
    __syncwarp();
  }
}
size_t kd_keys_smem(int d) { return (size_t)256 * (d | 1) * sizeof(float); }   // a row per thread of 256

// inclusive prefix sum of one value per thread over the CTA (in thread order); *total = the sum
__device__ __forceinline__ int block_scan_incl(int v, int* wsum, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) wsum[w] = v;
  __syncthreads();
  if (w == 0) {
    int s = lane < nw ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    wsum[lane] = s;
  }
  __syncthreads();
  const int r = v + (w > 0 ? wsum[w - 1] : 0);
  *total = wsum[nw - 1];
  __syncthreads();
  return r;
}

// A split sends the m - a smallest keys of [a, b) (equal keys in position order) to [a, m), the rest to [m, b), both
// in position order.  The pivot is found by a 4-pass radix select over the 32-bit keys (histogram counts aggregated per
// warp: the top byte of nearby floats is nearly constant); the partition takes KD_PER consecutive keys per thread.
// kd_split_kernel does a whole segment in one CTA; a wide level (segments longer than the wide threshold) spreads each
// segment over CTAs of KD_CHUNK keys with the same arithmetic, so both give the same permutation.
constexpr int KD_PER = 4;
constexpr int KD_WIDE_THREADS = 256;
constexpr int KD_CHUNK = KD_WIDE_THREADS * KD_PER * 4;   // keys per CTA of a wide level

// adds to hist[bin] the keys of [lo, hi) that match prefix above `byte`, binned by `byte`
__device__ __forceinline__ void kd_hist(const uint32_t* __restrict__ key, int64_t lo, int64_t hi, uint32_t prefix, int byte,
                                        unsigned* hist) {
  const int lane = threadIdx.x & 31;
  const uint32_t hmask = byte == 3 ? 0u : (0xffffffffu << (8 * (byte + 1)));
  for (int64_t base = lo; base < hi; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const uint32_t k = i < hi ? key[i] : 0u;
    const unsigned bin = (i < hi && (k & hmask) == prefix) ? (k >> (8 * byte)) & 255u : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin < 256u && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], (unsigned)__popc(peers));
  }
}

// the bin of `byte` that holds sorted index *rank; *rank becomes the index within that bin
__device__ __forceinline__ uint32_t kd_pick(const unsigned* hist, int byte, uint32_t prefix, int* rank) {
  int r = *rank, bin = 0;
  for (; bin < 255; ++bin) {
    if (r < (int)hist[bin]) break;
    r -= (int)hist[bin];
  }
  *rank = r;
  return prefix | ((uint32_t)bin << (8 * byte));
}

// the partition of the keys [lo, hi) of segment [a, m, b) around pivot, given the keys equal to the pivot before lo
// (eq_before) and the keys sent left before lo (left_before); eq_take of the equal keys go left
__device__ __forceinline__ void kd_partition(const uint32_t* __restrict__ key, const int32_t* __restrict__ P, int32_t* __restrict__ Pout,
                                             int64_t a, int64_t m, int64_t lo, int64_t hi, uint32_t pivot, int eq_take, int eq_before,
                                             int left_before, int* wsum) {
  for (int64_t base = lo; base < hi; base += (int64_t)blockDim.x * KD_PER) {
    const int64_t i0 = base + (int64_t)threadIdx.x * KD_PER;
    uint32_t k[KD_PER];
    int e_cnt = 0;
#pragma unroll
    for (int j = 0; j < KD_PER; ++j) {
      k[j] = i0 + j < hi ? key[i0 + j] : 0u;
      e_cnt += i0 + j < hi && k[j] == pivot;
    }
    int tot;
    int eq_rank = eq_before + block_scan_incl(e_cnt, wsum, &tot) - e_cnt;
    eq_before += tot;
    unsigned lf = 0u;
#pragma unroll
    for (int j = 0; j < KD_PER; ++j) {
      const bool in = i0 + j < hi, e = in && k[j] == pivot;
      lf |= (unsigned)(in && (k[j] < pivot || (e && eq_rank < eq_take))) << j;
      eq_rank += e;
    }
    const int l_cnt = __popc(lf);
    int64_t left_ex = left_before + block_scan_incl(l_cnt, wsum, &tot) - l_cnt;
    left_before += tot;
#pragma unroll
    for (int j = 0; j < KD_PER; ++j) {
      const int64_t i = i0 + j;
      if (i < hi) {
        const bool l = (lf >> j) & 1u;
        Pout[l ? a + left_ex : m + (i - a - left_ex)] = P[i];
        left_ex += l;
      }
    }
  }
}

// one CTA per segment
__global__ void __launch_bounds__(KD_THREADS) kd_split_kernel(const int32_t* __restrict__ seg, const uint32_t* __restrict__ key,
                                                              const int32_t* __restrict__ P, int32_t* __restrict__ Pout) {
  __shared__ unsigned hist[256];
  __shared__ uint32_t s_prefix;
  __shared__ int s_rank;
  __shared__ int wsum[32];
  const int64_t a = seg[3 * blockIdx.x], m = seg[3 * blockIdx.x + 1], b = seg[3 * blockIdx.x + 2];
  uint32_t prefix = 0;
  int rank = (int)(m - a) - 1;   // sorted index of the pivot
  for (int byte = 3; byte >= 0; --byte) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
    kd_hist(key, a, b, prefix, byte, hist);
    __syncthreads();
    if (threadIdx.x == 0) {
      s_prefix = kd_pick(hist, byte, prefix, &rank);
      s_rank = rank;
    }
    __syncthreads();
    prefix = s_prefix;
    rank = s_rank;
    __syncthreads();
  }
  kd_partition(key, P, Pout, a, m, a, b, prefix, rank + 1, 0, 0, wsum);
}

// A wide level: CTA (c, s) holds the keys [a + c KD_CHUNK, a + (c + 1) KD_CHUNK) of segment s (gridDim.x covers the
// longest segment; CTAs past the end return).  sel[2s] = the pivot's prefix so far, sel[2s + 1] = its rank within it;
// hist [segments][256] is zero before each kd_wide_hist_kernel.
__global__ void __launch_bounds__(KD_WIDE_THREADS) kd_wide_hist_kernel(const int32_t* __restrict__ seg, const uint32_t* __restrict__ key,
                                                                       int byte, const uint32_t* __restrict__ sel, unsigned* __restrict__ hist) {
  __shared__ unsigned h[256];
  const int64_t a = seg[3 * blockIdx.y], b = seg[3 * blockIdx.y + 2];
  const int64_t lo = a + (int64_t)blockIdx.x * KD_CHUNK;
  if (lo >= b) return;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0u;
  __syncthreads();
  kd_hist(key, lo, min(b, lo + KD_CHUNK), byte == 3 ? 0u : sel[2 * blockIdx.y], byte, h);
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (h[i]) atomicAdd(&hist[(int64_t)blockIdx.y * 256 + i], h[i]);
}

// one CTA of 256 threads per segment: the pivot's next byte, then the histogram zeroed for the next pass
__global__ void __launch_bounds__(256) kd_wide_pick_kernel(const int32_t* __restrict__ seg, int byte, uint32_t* __restrict__ sel,
                                                           unsigned* __restrict__ hist) {
  unsigned* hs = hist + (int64_t)blockIdx.x * 256;
  if (threadIdx.x == 0) {
    int rank = byte == 3 ? seg[3 * blockIdx.x + 1] - seg[3 * blockIdx.x] - 1 : (int)sel[2 * blockIdx.x + 1];
    sel[2 * blockIdx.x] = kd_pick(hs, byte, byte == 3 ? 0u : sel[2 * blockIdx.x], &rank);
    sel[2 * blockIdx.x + 1] = (uint32_t)rank;
  }
  __syncthreads();
  hs[threadIdx.x] = 0u;
}

// per CTA of a wide level: cnt[2 (s gridDim.x + c)] = its keys below the pivot, [.. + 1] = its keys equal to it
__global__ void __launch_bounds__(KD_WIDE_THREADS) kd_wide_count_kernel(const int32_t* __restrict__ seg, const uint32_t* __restrict__ key,
                                                                        const uint32_t* __restrict__ sel, int* __restrict__ cnt) {
  __shared__ int wsum[32];
  const int64_t a = seg[3 * blockIdx.y], b = seg[3 * blockIdx.y + 2];
  const int64_t lo = a + (int64_t)blockIdx.x * KD_CHUNK, hi = min(b, lo + KD_CHUNK);
  if (lo >= b) return;
  const uint32_t pivot = sel[2 * blockIdx.y];
  int lt = 0, eq = 0;
  for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const uint32_t k = key[i];
    lt += k < pivot;
    eq += k == pivot;
  }
  int tot_lt, tot_eq;
  block_scan_incl(lt, wsum, &tot_lt);
  block_scan_incl(eq, wsum, &tot_eq);
  if (threadIdx.x == 0) {
    int* c = cnt + 2 * ((int64_t)blockIdx.y * gridDim.x + blockIdx.x);
    c[0] = tot_lt;
    c[1] = tot_eq;
  }
}

// one thread per segment: each CTA's keys equal to the pivot before it and keys sent left before it, in place of cnt
__global__ void kd_wide_scan_kernel(const int32_t* __restrict__ seg, int n_seg, int chunks, const uint32_t* __restrict__ sel,
                                    int* __restrict__ cnt) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg) return;
  const int64_t a = seg[3 * s], b = seg[3 * s + 2];
  const int used = (int)((b - a + KD_CHUNK - 1) / KD_CHUNK);
  const int eq_take = (int)sel[2 * s + 1] + 1;
  int eq_before = 0, left_before = 0;
  for (int c = 0; c < used; ++c) {
    int* p = cnt + 2 * ((int64_t)s * chunks + c);
    const int lt = p[0], eq = p[1];
    p[0] = eq_before;
    p[1] = left_before;
    left_before += lt + max(0, min(eq, eq_take - eq_before));
    eq_before += eq;
  }
}

__global__ void __launch_bounds__(KD_WIDE_THREADS) kd_wide_scatter_kernel(const int32_t* __restrict__ seg, const uint32_t* __restrict__ key,
                                                                          const uint32_t* __restrict__ sel, const int* __restrict__ cnt,
                                                                          const int32_t* __restrict__ P, int32_t* __restrict__ Pout) {
  __shared__ int wsum[32];
  const int64_t a = seg[3 * blockIdx.y], m = seg[3 * blockIdx.y + 1], b = seg[3 * blockIdx.y + 2];
  const int64_t lo = a + (int64_t)blockIdx.x * KD_CHUNK;
  if (lo >= b) return;
  const int* c = cnt + 2 * ((int64_t)blockIdx.y * gridDim.x + blockIdx.x);
  kd_partition(key, P, Pout, a, m, lo, min(b, lo + KD_CHUNK), sel[2 * blockIdx.y], (int)sel[2 * blockIdx.y + 1] + 1, c[0], c[1], wsum);
}

__global__ void kd_iota_kernel(int32_t* __restrict__ P, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) P[i] = (int32_t)i;
}

// the call's query rows [q0, q0 + nq) in the order P puts them: qloc[j] = local row, qpos[j] = its position in P
__global__ void __launch_bounds__(KD_THREADS) kd_restrict_kernel(const int32_t* __restrict__ P, int64_t n, int64_t q0, int64_t nq,
                                                                 int32_t* __restrict__ qloc, int32_t* __restrict__ qpos) {
  __shared__ int wsum[32];
  int before = 0;
  for (int64_t base = 0; base < n; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const int64_t ql = i < n ? (int64_t)P[i] - q0 : -1;
    const int f = ql >= 0 && ql < nq;
    int tot;
    const int incl = block_scan_incl(f, wsum, &tot);
    if (f) {
      qloc[before + incl - 1] = (int32_t)ql;
      qpos[before + incl - 1] = (int32_t)i;
    }
    before += tot;
  }
}

// per tile t of the order P: the centre mu_t (the tile mean, rounded so that s * mu_t is an fp16 number, which the
// candidate image then holds exactly) and rad[t] >= max |x - mu_t| over the tile's points (fp64, rounded up)
__global__ void __launch_bounds__(256) kd_tile_stats_kernel(const float* __restrict__ X, int64_t n, int d, const int32_t* __restrict__ P,
                                                            const unsigned int* __restrict__ maxnorm_bits, float* __restrict__ cent,
                                                            float* __restrict__ rad) {
  __shared__ float mu[256];
  __shared__ unsigned int rmax;
  const int64_t t = blockIdx.x, p0 = t * CN;
  const int rows = (int)min((int64_t)CN, n - p0);
  const float s = tc_scale_from_maxnorm(*maxnorm_bits);
  if (threadIdx.x == 0) rmax = 0u;
  if ((int)threadIdx.x < d) {
    double acc = 0.0;
    for (int r = 0; r < rows; ++r) acc += X[(int64_t)P[p0 + r] * d + threadIdx.x];
    const float m = __half2float(__float2half_rn((float)(acc / rows) * s)) / s;
    mu[threadIdx.x] = m;
    cent[t * d + threadIdx.x] = m;
  }
  __syncthreads();
  if ((int)threadIdx.x < rows) {
    const float* x = X + (int64_t)P[p0 + threadIdx.x] * d;
    double acc = 0.0;
    for (int j = 0; j < d; ++j) {
      const double df = (double)x[j] - (double)mu[j];
      acc = fma(df, df, acc);
    }
    atomicMax(&rmax, __float_as_uint(__double2float_ru(sqrt(acc) * (1.0 + 1e-12))));
  }
  __syncthreads();
  if (threadIdx.x == 0) rad[t] = __uint_as_float(rmax);
}

// the short sweep's lists: nt consecutive tiles of the order around the tile of the block's first row
__global__ void knn_near_lists_kernel(int64_t n_blocks, int64_t n_tiles, int nt, const int32_t* __restrict__ qpos,
                                      int32_t* __restrict__ lists, int32_t* __restrict__ len) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_blocks) return;
  const int64_t own = (qpos ? (int64_t)qpos[b * QM] : b * QM) / CN;
  const int64_t cnt = min((int64_t)nt, n_tiles);
  const int64_t first = max((int64_t)0, min(own - (nt - 1) / 2, n_tiles - cnt));
  for (int64_t i = 0; i < cnt; ++i) lists[b * nt + i] = (int32_t)(first + i);
  len[b] = (int32_t)cnt;
}

// The screen: CTA = one 128-row query block, two warpgroups score it against 128 tile centres at a time (wgmma from
// shared memory, plain loads: the centre image is small and stays in L2).  rowp[row] = (qlb, us) in the images' scaled
// units: qlb <= |q|^2 - 2 eps_c - (fp32 slack), so |q - mu|^2 >= qlb - 2 score for the computed score; us >= u(q)
// (qlb = +inf: a padding row, which keeps nothing; us = +inf keeps everything).  Tile t survives if some row has
// qlb - 2 score <= (us + s r_t)^2 (1 + 2^-16), tested as !(>) so that a NaN keeps it.  Output: the surviving tiles of
// the block as a bitmap (bit t of words[block * n_words + t / 32]) and their count; knn_expand_lists_kernel turns the
// bitmaps into compact lists once the counts are known, so the lists take 4 B per kept (block, tile) pair.
__global__ void __launch_bounds__(256) knn_screen_kernel(const __half* __restrict__ Aimg, const __half* __restrict__ Cimg, int nks,
                                                         int64_t n_tiles, const float2* __restrict__ rowp, const float* __restrict__ rad,
                                                         const unsigned int* __restrict__ maxnorm_bits, uint32_t* __restrict__ words,
                                                         int64_t n_words, int32_t* __restrict__ list_len) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ float rs[CN];
  __shared__ uint32_t surv[NSUB];
  const uint32_t tile_b = (uint32_t)(CN * 16 * 2) * (uint32_t)nks;
  unsigned char* As = smem_raw;
  unsigned char* Bs = smem_raw + tile_b;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = warp >> 2, sl = lane & 3;
  const float s = tc_scale_from_maxnorm(*maxnorm_bits);
  {
    const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(Aimg) + (size_t)blockIdx.x * tile_b);
    uint4* dst = reinterpret_cast<uint4*>(As);
    for (uint32_t i = threadIdx.x; i < tile_b / 16; i += blockDim.x) dst[i] = src[i];
  }
  if (threadIdx.x < NSUB) surv[threadIdx.x] = 0u;
  const int row0 = 64 * g + 16 * (warp & 3) + (lane >> 2);
  const float2 p0 = rowp[(int64_t)blockIdx.x * QM + row0], p1 = rowp[(int64_t)blockIdx.x * QM + row0 + 8];
  const uint64_t da0 = wgmma_desc(smem_u32(As) + (uint32_t)g * 8u * SBO, LBO, SBO);
  const uint64_t db0 = wgmma_desc(smem_u32(Bs), LBO, SBO);
  constexpr uint32_t KSTEP16 = (2u * LBO) >> 4;
  constexpr float C = 1.0f + 1.0f / 65536.0f;
  uint32_t* out = words + (int64_t)blockIdx.x * n_words;
  int32_t cnt = 0;   // warp 0: tiles kept so far
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
  const int64_t n_ct = (n_tiles + CN - 1) / CN;
  for (int64_t ct = 0; ct < n_ct; ++ct) {
    __syncthreads();   // the previous centre tile is no longer read
    {
      const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(Cimg) + (size_t)ct * tile_b);
      uint4* dst = reinterpret_cast<uint4*>(Bs);
      for (uint32_t i = threadIdx.x; i < tile_b / 16; i += blockDim.x) dst[i] = src[i];
      if (threadIdx.x < CN) rs[threadIdx.x] = ct * CN + threadIdx.x < n_tiles ? rad[ct * CN + threadIdx.x] * s : 0.0f;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic stores -> wgmma operand reads
    __syncthreads();
    wgmma_fence_operand(acc);
    wgmma_fence();
    for (int j = 0; j < nks; ++j)
      wgmma_m64n128k16_f16(acc, da0 + (uint64_t)((uint32_t)j * KSTEP16), db0 + (uint64_t)((uint32_t)j * KSTEP16), j != 0);
    wgmma_commit();
    wgmma_wait_all();
    wgmma_fence_operand(acc);
    uint32_t keep = 0u;   // bit 2i + e: column 8i + 2 sl + e
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float r = rs[8 * i + 2 * sl + e];
        const float t0 = p0.y + r, t1 = p1.y + r;
        const bool k0 = !(fmaf(-2.0f, acc[4 * i + e], p0.x) > t0 * t0 * C);
        const bool k1 = !(fmaf(-2.0f, acc[4 * i + 2 + e], p1.x) > t1 * t1 * C);
        keep |= (uint32_t)(k0 || k1) << (2 * i + e);
      }
    }
    keep |= __shfl_xor_sync(0xffffffffu, keep, 4);
    keep |= __shfl_xor_sync(0xffffffffu, keep, 8);
    keep |= __shfl_xor_sync(0xffffffffu, keep, 16);
    if (lane < NSUB) atomicOr(&surv[lane], keep);
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = lane + 32 * e;
        const int64_t tile = ct * CN + col;
        const bool f = tile < n_tiles && ((surv[(col >> 1) & 3] >> (2 * (col >> 3) + (col & 1))) & 1u);
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0 && ct * 4 + e < n_words) out[ct * 4 + e] = bal;
        cnt += __popc(bal);
      }
    }
    __syncthreads();
    if (threadIdx.x < NSUB) surv[threadIdx.x] = 0u;
  }
  if (threadIdx.x == 0) {
    if (cnt == 0) { out[0] |= 1u; cnt = 1; }   // only padding rows: the sweep needs one visit
    list_len[blockIdx.x] = cnt;
  }
}

// one warp per block: the set bits of its bitmap, ascending, to lists[off[block] ..]
__global__ void knn_expand_lists_kernel(const uint32_t* __restrict__ words, int64_t n_words, int64_t n_blocks,
                                        const int64_t* __restrict__ off, int32_t* __restrict__ lists) {
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= n_blocks) return;
  const int lane = threadIdx.x & 31;
  int32_t* out = lists + off[b];
  int64_t base = 0;
  for (int64_t w0 = 0; w0 < n_words; w0 += 32) {
    uint32_t w = w0 + lane < n_words ? words[b * n_words + w0 + lane] : 0u;
    const int c = __popc(w);
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    int64_t pos = base + incl - c;
    while (w) {
      out[pos++] = (int32_t)((w0 + lane) * 32 + __ffs(w) - 1);
      w &= w - 1;
    }
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
}

}  // namespace

bool knn_tc2_supported(int d) { return 3 * d + 3 <= 512; }

bool knn_tc2_shape(const sb2_ctx* ctx, int d, int terms, bool want_estimate, KnnTc2Shape* out) {
  // one 128-row query image + a ring of candidate-image K-slices (128 rows each) in the opt-in shared memory of a
  // block; the K axis is staged in 1, 2, 4 or 8 slices, fewest first; at least 3 ring stages (2 when nothing else fits)
  const size_t cap = ctx->prop.sharedMemPerBlockOptin;
  for (int min_st = 3; min_st >= 2; --min_st) {
    for (int ns = 1; ns <= 8; ns *= 2) {
      const int unit = 16 * ns;
      const int kp = ((terms * d + 3 + unit - 1) / unit) * unit;
      const size_t ta = (size_t)QM * kp * 2, part = (size_t)CN * kp * 2 / ns;
      const size_t fixed = BAR_BYTES + ta;
      if (fixed + (size_t)min_st * part > cap) continue;
      int nst = (int)((cap - fixed) / part);
      if (nst > MAXST) nst = MAXST;
      out->nsplit = ns; out->nstage = nst; out->kpad = kp; out->terms = terms; out->est = want_estimate ? 1 : 0;
      // the pipelined loop holds two stages per warpgroup (the one it examines, the one its MMAs read): whole tiles
      // per stage, and a third stage so that the producer can run ahead; compiled for K = 64 and K = 160
      out->pipe = (ns == 1 && nst >= 3 && (kp == 16 * PIPE_NKS0 || kp == 16 * PIPE_NKS1)) ? 1 : 0;
      out->smem = fixed + (size_t)nst * part;
      return true;
    }
  }
  return false;
}

size_t knn_tc2_a_halves(const KnnTc2Shape& sh, int64_t n_rows) { return (size_t)(ceil_div64(n_rows, QM) + 1) * QM * sh.kpad; }
size_t knn_tc2_b_halves(const KnnTc2Shape& sh, int64_t n_rows) { return (size_t)(ceil_div64(n_rows, CN) + 1) * CN * sh.kpad; }

int32_t knn_tc2_build_images(sb2_ctx* ctx, const KnnTc2Shape& sh, const float* d_x, int64_t n_rows, int d,
                             const unsigned int* d_maxnorm_bits, const int32_t* d_gather, int64_t gather_base,
                             __half* Aimg, __half* Bimg, float* d_inv_s2, float* d_dnorm, unsigned int* d_dmax_bits) {
  if (Aimg) {
    const int64_t nt = ceil_div64(n_rows, QM) + 1;
    knn_tc2_prep_kernel<<<(unsigned)nt, 256, 0, ctx->stream>>>(d_x, n_rows, d, sh.kpad, sh.terms, QM, 1, d_maxnorm_bits, d_gather,
                                                                gather_base, Aimg, d_inv_s2, Bimg ? nullptr : d_dnorm,
                                                                Bimg ? nullptr : d_dmax_bits);
    SB2_LAUNCH_CHECK(ctx);
  }
  if (Bimg) {
    const int64_t nt = ceil_div64(n_rows, CN) + 1;
    knn_tc2_prep_kernel<<<(unsigned)nt, 256, 0, ctx->stream>>>(d_x, n_rows, d, sh.kpad, sh.terms, CN, 0, d_maxnorm_bits, d_gather,
                                                                gather_base, Bimg, d_inv_s2, d_dnorm, d_dmax_bits);
    SB2_LAUNCH_CHECK(ctx);
  }
  return SB2_OK;
}


int32_t knn_tc2_kd_order(sb2_ctx* ctx, const float* d_x, int64_t n, int d, bool coord, int64_t wide_min, int32_t* perm) {
  SB2_CHECK_ARG(d >= 1 && d <= KD_MAX_D, "kd order: d");
  cudaStream_t st = ctx->stream;
  // the segments of every level depend on n alone: [a, b) splits at a + 128 * floor(tiles / 2)
  std::vector<int32_t> segs;
  struct Level {
    size_t first;   // first segment
    int cnt;        // segments
    int64_t len;    // the longest
  };
  std::vector<Level> levels;
  std::vector<std::pair<int64_t, int64_t>> cur{{0, n}}, nxt;
  int max_seg = 0;
  int64_t wide_chunks = 0;   // largest segments x chunks of a wide level
  for (;;) {
    nxt.clear();
    const size_t first = segs.size() / 3;
    int64_t len = 0;
    for (const auto& ab : cur) {
      if (ab.second - ab.first <= CN) continue;
      const int64_t m = ab.first + CN * (ceil_div64(ab.second - ab.first, CN) / 2);
      segs.insert(segs.end(), {(int32_t)ab.first, (int32_t)m, (int32_t)ab.second});
      nxt.push_back({ab.first, m});
      nxt.push_back({m, ab.second});
      len = std::max(len, ab.second - ab.first);
    }
    const int cnt = (int)(segs.size() / 3 - first);
    if (cnt == 0) break;
    levels.push_back({first, cnt, len});
    max_seg = max_seg > cnt ? max_seg : cnt;
    if (len >= wide_min) wide_chunks = std::max(wide_chunks, (int64_t)cnt * ceil_div64(len, KD_CHUNK));
    cur.swap(nxt);
  }
  kd_iota_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(perm, n);
  SB2_LAUNCH_CHECK(ctx);
  if (levels.empty()) return SB2_OK;
  ScratchScope scr(ctx);
  int32_t *d_segs, *axis = nullptr, *other;
  double* dir = nullptr;
  uint32_t *key, *sel = nullptr;
  unsigned* hist = nullptr;
  int* cnt = nullptr;
  SB2_TRY(scr.alloc(&d_segs, segs.size()));
  if (coord) SB2_TRY(scr.alloc(&axis, (size_t)max_seg));
  else SB2_TRY(scr.alloc(&dir, (size_t)max_seg * (d + 1)));
  SB2_TRY(scr.alloc(&other, (size_t)n));
  SB2_TRY(scr.alloc(&key, (size_t)n));
  if (wide_chunks) {
    SB2_TRY(scr.alloc(&sel, (size_t)max_seg * 2));
    SB2_TRY(scr.alloc(&hist, (size_t)max_seg * 256));
    SB2_TRY(scr.alloc(&cnt, (size_t)wide_chunks * 2));
    SB2_CUDA(cudaMemsetAsync(hist, 0, (size_t)max_seg * 256 * sizeof(unsigned), st));   // each pick re-zeroes its own
  }
  const int ns_dir = kd_dir_samples(d);
  if (!coord) {
    SB2_CUDA(cudaFuncSetAttribute(kd_dir_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kd_dir_smem(d, ns_dir)));
    SB2_CUDA(cudaFuncSetAttribute(kd_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kd_keys_smem(d)));
  }
  SB2_CUDA(cudaMemcpyAsync(d_segs, segs.data(), segs.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  int32_t *src = perm, *dst = other;
  for (const auto& lv : levels) {
    const int32_t* sg = d_segs + lv.first * 3;
    const unsigned ns = (unsigned)lv.cnt;
    SB2_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));   // unsplit segments
    if (coord) {
      kd_axis_kernel<<<ns, 256, 0, st>>>(d_x, d, src, sg, axis);
    } else {
      const int ns_lv = (int)std::min<int64_t>(lv.len, ns_dir);
      kd_dir_kernel<<<ns, 256, kd_dir_smem(d, ns_lv), st>>>(d_x, d, src, sg, ns_dir, dir);
    }
    SB2_LAUNCH_CHECK(ctx);
    kd_keys_kernel<<<dim3(ns, (unsigned)ceil_div64(2048, ns)), 256, coord ? 0 : kd_keys_smem(d), st>>>(d_x, d, src, sg, dir, axis, key);
    SB2_LAUNCH_CHECK(ctx);
    if (lv.len >= wide_min) {
      const dim3 grid((unsigned)ceil_div64(lv.len, KD_CHUNK), ns);
      for (int byte = 3; byte >= 0; --byte) {
        kd_wide_hist_kernel<<<grid, KD_WIDE_THREADS, 0, st>>>(sg, key, byte, sel, hist);
        SB2_LAUNCH_CHECK(ctx);
        kd_wide_pick_kernel<<<ns, 256, 0, st>>>(sg, byte, sel, hist);
        SB2_LAUNCH_CHECK(ctx);
      }
      kd_wide_count_kernel<<<grid, KD_WIDE_THREADS, 0, st>>>(sg, key, sel, cnt);
      SB2_LAUNCH_CHECK(ctx);
      kd_wide_scan_kernel<<<(unsigned)ceil_div64(ns, 128), 128, 0, st>>>(sg, (int)ns, (int)grid.x, sel, cnt);
      SB2_LAUNCH_CHECK(ctx);
      kd_wide_scatter_kernel<<<grid, KD_WIDE_THREADS, 0, st>>>(sg, key, sel, cnt, src, dst);
    } else {
      kd_split_kernel<<<ns, KD_THREADS, 0, st>>>(sg, key, src, dst);
    }
    SB2_LAUNCH_CHECK(ctx);
    int32_t* t = src; src = dst; dst = t;
  }
  if (src != perm) SB2_CUDA(cudaMemcpyAsync(perm, src, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return SB2_OK;
}

int32_t knn_tc2_restrict(sb2_ctx* ctx, const int32_t* perm, int64_t n, int64_t q0, int64_t n_query, int32_t* qloc, int32_t* qpos) {
  kd_restrict_kernel<<<1, KD_THREADS, 0, ctx->stream>>>(perm, n, q0, n_query, qloc, qpos);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t knn_tc2_tile_stats(sb2_ctx* ctx, const float* d_x, int64_t n, int d, const int32_t* perm, const unsigned int* d_maxnorm_bits,
                           float* cent, float* rad) {
  kd_tile_stats_kernel<<<(unsigned)ceil_div64(n, CN), 256, 0, ctx->stream>>>(d_x, n, d, perm, d_maxnorm_bits, cent, rad);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t knn_tc2_near_lists(sb2_ctx* ctx, int64_t n_blocks, int64_t n_tiles, int nt, const int32_t* qpos, int32_t* lists, int32_t* len) {
  SB2_CHECK_ARG(nt >= 1 && nt <= KNN_MAX_NEAR, "near tiles");
  knn_near_lists_kernel<<<(unsigned)ceil_div64(n_blocks, 256), 256, 0, ctx->stream>>>(n_blocks, n_tiles, nt, qpos, lists, len);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int64_t knn_tc2_screen_words(int64_t n_tiles) { return ceil_div64(n_tiles, 32); }

int32_t knn_tc2_screen(sb2_ctx* ctx, const KnnTc2Shape& sh, const __half* Aimg, const __half* Cimg, int64_t n_blocks, int64_t n_tiles,
                       const float2* rowp, const float* rad, const unsigned int* d_maxnorm_bits, uint32_t* words, int32_t* list_len) {
  SB2_CHECK_ARG(sh.nsplit == 1, "the tile screen needs whole images in shared memory");
  const size_t smem = (size_t)2 * QM * sh.kpad * 2;
  SB2_CUDA(cudaFuncSetAttribute(knn_screen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  knn_screen_kernel<<<(unsigned)n_blocks, 256, smem, ctx->stream>>>(Aimg, Cimg, sh.kpad / 16, n_tiles, rowp, rad, d_maxnorm_bits,
                                                                    words, knn_tc2_screen_words(n_tiles), list_len);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t knn_tc2_expand_lists(sb2_ctx* ctx, const uint32_t* words, int64_t n_blocks, int64_t n_tiles, const int64_t* off, int32_t* lists) {
  knn_expand_lists_kernel<<<(unsigned)ceil_div64(n_blocks, 8), 256, 0, ctx->stream>>>(words, knn_tc2_screen_words(n_tiles), n_blocks,
                                                                                      off, lists);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

namespace {
// f(NG, PNKS, STAMPS, ISCAN) as std::integral_constants, the template arguments of knn_sweep2_kernel: NG = 2 for lists of
// 64 proposals, 4 for 128; PNKS the pipelined loop's k-steps when pipe (knn_tc2_shape only sets it for nsplit = 1 and
// these two K axes), else 0
template <typename F>
void with_sweep2(int list_m, bool iscan, bool pipe, int kpad, bool stamps, F&& f) {
  using std::integral_constant;
  const auto with_stamps = [&](auto ng, auto is, auto pnks) {
    if (stamps) f(ng, pnks, std::true_type(), is);
    else f(ng, pnks, std::false_type(), is);
  };
  const auto with_pnks = [&](auto ng, auto is) {
    const int nks = pipe ? kpad / 16 : 0;
    if (nks == PIPE_NKS0) with_stamps(ng, is, integral_constant<int, PIPE_NKS0>());
    else if (nks == PIPE_NKS1) with_stamps(ng, is, integral_constant<int, PIPE_NKS1>());
    else with_stamps(ng, is, integral_constant<int, 0>());
  };
  const auto with_scan = [&](auto ng) {
    if (iscan) with_pnks(ng, std::true_type());
    else with_pnks(ng, std::false_type());
  };
  if (list_m == 64) with_scan(integral_constant<int, 2>());
  else with_scan(integral_constant<int, 4>());
}

// SB2_KNN_STAMPS=1: where the consumer warpgroups of one sweep spent their cycles, summed over all of them, and how
// often they left the fast path, on stderr
int32_t report_stamps(sb2_ctx* ctx, const KnnTc2Shape& sh, bool pipe, unsigned grid, double visits, double est_visits, int64_t n_query,
                      int list_m, const unsigned long long* d_stamps) {
  std::vector<unsigned long long> h((size_t)grid * 2 * ST_N);
  SB2_CUDA(cudaMemcpyAsync(h.data(), d_stamps, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  double tot[ST_N] = {}, all = 0.0;
  for (size_t i = 0; i < h.size(); ++i) {
    tot[i % ST_N] += (double)h[i];
    if (i % ST_N < PH_N) all += (double)h[i];
  }
  const double tiles = 2.0 * visits;   // tiles examined (all CTAs), counted per warpgroup
  static const char* names[PH_N] = {"wait full", "mma", "scan", "insert"};
  fprintf(stderr, "[sb2 knn stamps] %s loop, K=%d nsplit=%d nstage=%d list=%d, %u CTAs x %.1f visits: %.0f cycles/tile",
          pipe ? "pipelined" : "single-buffer", sh.kpad, sh.nsplit, sh.nstage, list_m, grid, grid ? visits / grid : 0.0,
          tiles > 0 ? all / tiles : 0.0);
  for (int ph = 0; ph < PH_N; ++ph)
    fprintf(stderr, ", %s %.1f%% (%.0f)", names[ph], all > 0 ? 100.0 * tot[ph] / all : 0.0, tiles > 0 ? tot[ph] / tiles : 0.0);
  // the rare path: share of the sweep proper's warp-tiles (8 consumer warps per CTA) on which a warp took it, and the
  // insertions per query row (four sub-lists)
  const double warp_tiles = NCONS * (visits - est_visits);
  fprintf(stderr, ", rare-path tiles %.2f%%, insertions/row %.1f\n", warp_tiles > 0 ? 100.0 * tot[CNT_RARE] / warp_tiles : 0.0,
          n_query > 0 ? tot[CNT_INSERT] / (double)n_query : 0.0);
  return SB2_OK;
}
}  // namespace

int32_t knn_tc2_sweep(sb2_ctx* ctx, const KnnSwitches& sw, const KnnTc2Shape& sh, const __half* Aimg, int64_t a_tile0,
                      const __half* Bimg, int64_t n_points, int64_t n_query, int list_m, float* cand_score, int32_t* cand_idx,
                      double* issued_flops, const KnnTc2Lists* lists) {
  cudaStream_t st = ctx->stream;
  const int64_t n_tiles = ceil_div64(n_points, CN);
  const int64_t q_ctas = ceil_div64(n_query, QM);
  SB2_CHECK_ARG(list_m == 64 || list_m == 128, "list_m must be 64 or 128 (four sub-lists of 16 or 32)");
  // threshold estimate: the est_rank-th largest of the row's chunk maxima over every est_stride-th tile sits at about
  // rank est_rank * est_stride of the row
  const int64_t est_stride = sw.est_stride;
  int64_t n_est = sw.cold ? 0 : n_tiles / est_stride;
  if (n_tiles < 32 * est_stride || !sh.est || lists) n_est = 0;  // small problems / split-precision sweeps / tile lists
  // the sub-lists start at the est_rank-th largest of the row's sampled chunk maxima, rank ~96 of the row by default:
  // on the 1.3M x 50 benchmark (k = 15) every rank below 6 sends more rows to the split-precision re-sweep (rank 5:
  // 7x as many, rank 4: 46x) than it saves in insertions.  SB2_KNN_EST_RANK=1..6 picks another (tests, A/B timing).
  const int est_rank = sw.est_rank;
  const unsigned grid = (unsigned)q_ctas;
  ScratchScope scr(ctx);
  // without tile lists every CTA walks all tiles: one shared identity list
  KnnTc2Lists all{nullptr, 0, nullptr, nullptr, q_ctas * n_tiles, nullptr, sw.stamps};
  if (!lists) {
    int32_t* ident;
    SB2_TRY(scr.alloc(&ident, (size_t)n_tiles));
    kd_iota_kernel<<<(unsigned)ceil_div64(n_tiles, 256), 256, 0, st>>>(ident, n_tiles);
    SB2_LAUNCH_CHECK(ctx);
    all.idx = ident;
    lists = &all;
  }
  const double visits = (double)lists->total + (double)q_ctas * (double)n_est;
  if (issued_flops) *issued_flops += 2.0 * QM * visits * CN * (double)sh.kpad;
  const int32_t np = (int32_t)n_points;
  {
    void* fp = nullptr;
    SB2_CUDA(cudaGetSymbolAddress(&fp, g_knn2_front));
    SB2_CUDA(cudaMemsetAsync(fp, 0, sizeof(unsigned long long), st));
  }
  // SB2_KNN_PIPE=0 and SB2_KNN_SCAN=float give the same results (A/B timing)
  const bool pipe = sh.pipe && sw.pipe;
  unsigned long long* stamps = nullptr;
  if (lists->stamps) {
    SB2_TRY(scr.alloc(&stamps, (size_t)grid * 2 * ST_N));
    SB2_CUDA(cudaMemsetAsync(stamps, 0, (size_t)grid * 2 * ST_N * sizeof(unsigned long long), st));
  }
  cudaError_t le = cudaSuccess;
  with_sweep2(list_m, sw.int_scan, pipe, sh.kpad, lists->stamps, [&](auto ng, auto pnks, auto st_on, auto iscan) {
    le = cudaFuncSetAttribute(knn_sweep2_kernel<ng, pnks, st_on, iscan>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh.smem);
    if (le != cudaSuccess) return;
    const int nks = sh.kpad / 16 / sh.nsplit;
    knn_sweep2_kernel<ng, pnks, st_on, iscan><<<grid, pnks > 0 ? THREADS_PIPE : THREADS, sh.smem, st>>>(
        Aimg, Bimg, nks, sh.nsplit, sh.nstage, n_tiles, n_est, est_stride, est_rank, a_tile0, n_query, np, lists->idx, lists->stride,
        lists->off, lists->len, lists->seed, cand_score, cand_idx, stamps);
  });
  SB2_CUDA(le);
  SB2_LAUNCH_CHECK(ctx);
  if (stamps) SB2_TRY(report_stamps(ctx, sh, pipe, grid, visits, (double)q_ctas * (double)n_est, n_query, list_m, stamps));
  return SB2_OK;
}

void knn_tc2_error_coefs(const KnnTc2Shape& sh, double* c_q, double* c_n) {
  // |s_computed - s_true| <= c_q |q| R + c_n R^2 / 2   (R = largest norm in the data set, everything after scaling)
  //   fp32 accumulation in the tensor pipe: kpad/16 accumulator updates of one ulp each plus the alignment loss
  //   inside a 16-product group, bounded by 1.6 * kpad * 2^-24 of sum |a_i b_i| <= |q| R + R^2 / 2;
  //   three-way fp16 split of the norm: 2^-33 R^2/2; sub-normal halves: < 2^-27 R^2/2 since R >= 100 after scaling
  //   terms = 3: operand split 3 * 2^-24 |q| R, dropped lo*lo term 2^-22 * 2^-2 |q| R
  //   terms = 1: |q.c - q_hi.c_hi| <= |q - q_hi| |c| + |q_hi| |c - c_hi|: the re-score kernel adds this term from
  //              the measured residual norms (dnorm / dmax of knn_tc2_build_images), not from the 2^-11 worst case
  // tests/test_gpu_parity.py::test_knn_tensor_score_error_within_bound measures the actual error against this bound.
  const double u24 = 5.9604644775390625e-08;
  const double acc = 1.6 * sh.kpad * u24;
  *c_n = acc + 8.0 * u24;
  *c_q = acc + (sh.terms == 3 ? 8.0 * u24 : 0.0);
}

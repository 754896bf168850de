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
//   CTA = 128 queries x all candidate tiles of 128 points.
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
//   Starting threshold: the first n/16 visits sweep every 16th tile and keep the 6 largest chunk maxima per (row,
//   sub-list); the four sub-lists of a row (four lanes of one warp) are merged by shuffles once and the 6th largest of
//   the 24 seeds all four (rank ~96 of the row; SB2_KNN_EST_RANK picks another of the six).
//   Sweep front: CTAs walk the candidate tiles cyclically, starting where the running CTAs currently are (g_knn2_front).
#include <cuda_fp16.h>
#include <float.h>

#include <type_traits>

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
// (A) or score -60000 candidates (B).  dnorm[p] (optional) = |x_p - fp16(x_p)| in the units of X, rounded up;
// *dmax_bits = its maximum (float bits).
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
        dnorm[p] = dn;
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

// nks = k-steps (16 columns of the K axis) per staged slice, nsplit = slices per candidate image.
// Sweep front: CTAs walk the candidate tiles cyclically, each starting where the CTAs already running currently are
// (the order of the candidates is irrelevant to the result).  All resident CTAs then stream the same few tiles at the
// same time and the candidate images (166 MB at 1.3M x 50, more than the L2) are read from HBM about once per wave of
// CTAs instead of once per CTA.  "Where the running CTAs are" is the MEAN position of the pack, (sweep visits so far) /
// (resident CTAs): starting a new CTA at the position last published by ANY running CTA lets the spread of the pack
// grow from wave to wave; re-centring every new CTA on the mean bounds it by the drift of a single lap.
__device__ unsigned long long g_knn2_front;   // sweep-proper visits of all CTAs of this launch, in units of 16 tiles
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
                  int32_t n_points, float* __restrict__ cand_score, int32_t* __restrict__ cand_idx,
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
  int32_t* start_tile = reinterpret_cast<int32_t*>(bars + 2 * MAXST + 1);
  unsigned long long* stamp_sm = reinterpret_cast<unsigned long long*>(bars + 2 * MAXST + 2);  // [2][PH_N + 1]
  static_assert((2 * MAXST + 2 + 2 * (PH_N + 1)) * 8 <= BAR_BYTES, "barrier block");

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < nstage; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NCONS); }
    mbar_init(afull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const unsigned long long f = *reinterpret_cast<volatile unsigned long long*>(&g_knn2_front);
    unsigned int nsm;
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsm));
    const unsigned long long resident = min((unsigned long long)gridDim.x, (unsigned long long)max(nsm, 1u));
    // mean tile of the pack now, plus the n_est visits this CTA spends on its threshold estimate before it joins
    *start_tile = (int32_t)((f * 16ull / resident + (unsigned long long)n_est) % (unsigned long long)n_btiles);
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
      int64_t cs = *start_tile;   // cyclic walk of the sweep proper
      for (int64_t v = 0; v < n_est + n_btiles; ++v) {
        int64_t c = v * est_stride;
        if (v >= n_est) { c = cs; if (++cs == n_btiles) cs = 0; }
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
  const int n_visit = (int)(n_est + n_btiles), n_est_i = (int)n_est;
  int32_t ctile = *start_tile;                 // candidate tile of the current sweep visit (cyclic walk)
  int32_t cbase = ctile * CN + 2 * sl;
  const int32_t n_bt = (int32_t)n_btiles;

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
      const float t0 = valid0 ? e0 : INFINITY;  // rows past n_query never accept anything
      const float t1 = valid1 ? e1 : INFINITY;
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
      if ((c & 15) == 0 && warp == 0 && lane == 0) atomicAdd(&g_knn2_front, 1ull);   // 16 more visits of the pack
      cbase += CN;
      if (++ctile == n_bt) { ctile = 0; cbase = 2 * sl; }
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
int32_t report_stamps(sb2_ctx* ctx, const KnnTc2Shape& sh, bool pipe, unsigned grid, int64_t n_visit, int64_t n_est, int64_t n_query,
                      int list_m, const unsigned long long* d_stamps) {
  std::vector<unsigned long long> h((size_t)grid * 2 * ST_N);
  SB2_CUDA(cudaMemcpyAsync(h.data(), d_stamps, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  double tot[ST_N] = {}, all = 0.0;
  for (size_t i = 0; i < h.size(); ++i) {
    tot[i % ST_N] += (double)h[i];
    if (i % ST_N < PH_N) all += (double)h[i];
  }
  const double tiles = (double)grid * 2.0 * (double)n_visit;   // tiles examined, counted per warpgroup
  static const char* names[PH_N] = {"wait full", "mma", "scan", "insert"};
  fprintf(stderr, "[sb2 knn stamps] %s loop, K=%d nsplit=%d nstage=%d list=%d, %u CTAs x %lld visits: %.0f cycles/tile",
          pipe ? "pipelined" : "single-buffer", sh.kpad, sh.nsplit, sh.nstage, list_m, grid, (long long)n_visit,
          tiles > 0 ? all / tiles : 0.0);
  for (int ph = 0; ph < PH_N; ++ph)
    fprintf(stderr, ", %s %.1f%% (%.0f)", names[ph], all > 0 ? 100.0 * tot[ph] / all : 0.0, tiles > 0 ? tot[ph] / tiles : 0.0);
  // the rare path: share of the sweep proper's warp-tiles (8 consumer warps per CTA) on which a warp took it, and the
  // insertions per query row (four sub-lists)
  const double warp_tiles = (double)grid * NCONS * (double)(n_visit - n_est);
  fprintf(stderr, ", rare-path tiles %.2f%%, insertions/row %.1f\n", warp_tiles > 0 ? 100.0 * tot[CNT_RARE] / warp_tiles : 0.0,
          n_query > 0 ? tot[CNT_INSERT] / (double)n_query : 0.0);
  return SB2_OK;
}
}  // namespace

int32_t knn_tc2_sweep(sb2_ctx* ctx, const KnnSwitches& sw, const KnnTc2Shape& sh, const __half* Aimg, int64_t a_tile0,
                      const __half* Bimg, int64_t n_points, int64_t n_query, int list_m, float* cand_score, int32_t* cand_idx,
                      double* issued_flops) {
  cudaStream_t st = ctx->stream;
  const int64_t n_tiles = ceil_div64(n_points, CN);
  const int64_t q_ctas = ceil_div64(n_query, QM);
  SB2_CHECK_ARG(list_m == 64 || list_m == 128, "list_m must be 64 or 128 (four sub-lists of 16 or 32)");
  // threshold estimate: the est_rank-th largest of the row's chunk maxima over every est_stride-th tile sits at about
  // rank est_rank * est_stride of the row
  const int64_t est_stride = sw.est_stride;
  int64_t n_est = sw.cold ? 0 : n_tiles / est_stride;
  if (n_tiles < 32 * est_stride || !sh.est) n_est = 0;  // small problems / split-precision sweeps: cold start
  // the sub-lists start at the est_rank-th largest of the row's sampled chunk maxima, rank ~96 of the row by default:
  // on the 1.3M x 50 benchmark (k = 15) every rank below 6 sends more rows to the split-precision re-sweep (rank 5:
  // 7x as many, rank 4: 46x) than it saves in insertions.  SB2_KNN_EST_RANK=1..6 picks another (tests, A/B timing).
  const int est_rank = sw.est_rank;
  if (issued_flops) *issued_flops += 2.0 * (double)(q_ctas * QM) * (double)((n_tiles + n_est) * CN) * (double)sh.kpad;
  const unsigned grid = (unsigned)q_ctas;
  const int32_t np = (int32_t)n_points;
  {
    void* fp = nullptr;
    SB2_CUDA(cudaGetSymbolAddress(&fp, g_knn2_front));
    SB2_CUDA(cudaMemsetAsync(fp, 0, sizeof(unsigned long long), st));
  }
  // SB2_KNN_PIPE=0 and SB2_KNN_SCAN=float give the same results (A/B timing)
  const bool pipe = sh.pipe && sw.pipe;
  ScratchScope scr(ctx);
  unsigned long long* stamps = nullptr;
  if (sw.stamps) {
    SB2_TRY(scr.alloc(&stamps, (size_t)grid * 2 * ST_N));
    SB2_CUDA(cudaMemsetAsync(stamps, 0, (size_t)grid * 2 * ST_N * sizeof(unsigned long long), st));
  }
  cudaError_t le = cudaSuccess;
  with_sweep2(list_m, sw.int_scan, pipe, sh.kpad, sw.stamps, [&](auto ng, auto pnks, auto st_on, auto iscan) {
    le = cudaFuncSetAttribute(knn_sweep2_kernel<ng, pnks, st_on, iscan>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh.smem);
    if (le != cudaSuccess) return;
    const int nks = sh.kpad / 16 / sh.nsplit;
    knn_sweep2_kernel<ng, pnks, st_on, iscan><<<grid, pnks > 0 ? THREADS_PIPE : THREADS, sh.smem, st>>>(
        Aimg, Bimg, nks, sh.nsplit, sh.nstage, n_tiles, n_est, est_stride, est_rank, a_tile0, n_query, np, cand_score, cand_idx,
        stamps);
  });
  SB2_CUDA(le);
  SB2_LAUNCH_CHECK(ctx);
  if (stamps) SB2_TRY(report_stamps(ctx, sh, pipe, grid, n_tiles + n_est, n_est, n_query, list_m, stamps));
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

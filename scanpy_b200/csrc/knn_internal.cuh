// knn_internal.cuh — interface between knn.cu (host entry, re-score, fallback) and knn_tc2.cu (tensor-core sweep)
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

constexpr int EST_R = 6;           // chunk maxima an estimate keeps per (row, sub-list)
constexpr int EST_STRIDE = 16;     // the estimate samples every 16th candidate tile
constexpr int KNN_MAX_NEAR = 64;   // longest near list of the tile screen's short sweep (SB2_KNN_NEAR)
constexpr int64_t KD_WIDE_MIN = 16384;   // kd order: segments from this length on are split by many CTAs each

// float <-> unsigned with the same order (the kd order's radix select, the k-th largest proposal score)
__device__ __forceinline__ uint32_t ord_bits(float x) {
  const uint32_t u = __float_as_uint(x);
  return u ^ ((u & 0x80000000u) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float from_ord_bits(uint32_t u) { return __uint_as_float(u ^ ((u & 0x80000000u) ? 0x80000000u : 0xffffffffu)); }

// The kNN's run-time switches, read from the environment on every call by knn_switches (knn.cu).  The defaults are
// what bench.py measures; every other setting gives the same neighbours.
struct KnnSwitches {
  bool ffma = false;            // SB2_KNN_PASS1=ffma: the fp32 CUDA-core first pass instead of the tensor-core tiers
  bool split_only = false;      // SB2_KNN_TIERS=3: every row goes straight to the split-precision tier
  bool big_list = false;        // SB2_KNN_LIST=64 or 128: 128-proposal lists for every k
  bool cold = false;            // SB2_KNN_EST set to a value <= 0: every sweep starts cold
  int est_stride = EST_STRIDE;  // SB2_KNN_EST=n > 0: the threshold estimate samples every n-th candidate tile
  int est_rank = EST_R;         // SB2_KNN_EST_RANK=1..EST_R: which of the sampled chunk maxima seeds the sub-lists
  int64_t scan_slots = 0;       // SB2_KNN_SCAN_SLOTS=n: up to n rows tier 1 leaves open go straight to the exact scan
  bool pipe = true;             // SB2_KNN_PIPE=0 (false): the single-buffer consumer loop where the pipelined one could run
  bool stamps = false;          // SB2_KNN_STAMPS=1: each sweep launch reports its consumers' cycle split on stderr
  bool int_scan = true;         // SB2_KNN_SCAN=float (false): the float max tree in the fast path of the sweep's examination
  int screen = -1;              // SB2_KNN_SCREEN=0: no tile screen; =1: screen at every size; unset: from 512 candidate tiles
  int near_tiles = 64;          // SB2_KNN_NEAR=1..KNN_MAX_NEAR: consecutive tiles of the kd order in the screen's short sweep
  int split = 1;                // SB2_KNN_SPLIT=coord (0): the kd order splits on the coordinate of largest variance, not
                                // the principal direction (=principal, 1); -1: an unknown value, which fails the screened call
  int64_t kd_wide = KD_WIDE_MIN;   // SB2_KNN_KD_WIDE=n >= 1: the kd order's segment length from which many CTAs split one
                                   // segment (the same permutation; tests force either path); 0: not an integer >= 1
};

// ---- tensor-core sweep (knn_tc2.cu): 128-query CTAs x 128-candidate tiles (wgmma N = 128), two consumer warpgroups,
// four register-resident sub-lists per query row (one per column class of the accumulator fragment) ----
struct KnnTc2Shape {
  int nsplit;   // slices the K axis of a candidate image is staged in (1, 2, 4, 8)
  int nstage;   // depth of the candidate ring
  int kpad;     // padded K axis (terms*d + 3 rounded up to 16*nsplit)
  int terms;
  int est;      // 1: the sweep may start from a sampled threshold
  int pipe;     // 1: the shape allows the pipelined consumer loop (nsplit == 1, nstage >= 3)
  size_t smem;
};
bool knn_tc2_supported(int d);
bool knn_tc2_shape(const sb2_ctx* ctx, int d, int terms, bool want_estimate, KnnTc2Shape* out);
size_t knn_tc2_a_halves(const KnnTc2Shape& sh, int64_t n_rows);   // query images: tiles of 128 rows
size_t knn_tc2_b_halves(const KnnTc2Shape& sh, int64_t n_rows);   // candidate images: tiles of 128 rows
int32_t knn_tc2_build_images(sb2_ctx* ctx, const KnnTc2Shape& sh, const float* d_x, int64_t n_rows, int d,
                             const unsigned int* d_maxnorm_bits, const int32_t* d_gather, int64_t gather_base,
                             __half* Aimg, __half* Bimg, float* d_inv_s2, float* d_dnorm = nullptr,
                             unsigned int* d_dmax_bits = nullptr);
// proposals: list_m (64 or 128) per query = four sub-lists of list_m/4, sub-list j in slots [j*list_m/4, (j+1)*list_m/4);
// unused slots hold the sub-list's starting threshold (-inf for a cold start) and id -1.  Only a shape made with
// want_estimate starts from a sampled threshold.
// Per query block (CTA) the ascending candidate tiles it visits: idx[off[b] + i] (off == nullptr: idx[b * stride + i]),
// i < len[b]; total = the sum of len over the launch.  seed (optional): the starting threshold of each launch row (scaled score units) instead of the
// sampled estimate.  stamps: the launch may report SB2_KNN_STAMPS.
struct KnnTc2Lists {
  const int32_t* idx;
  int64_t stride;
  const int64_t* off;
  const int32_t* len;
  int64_t total;
  const float* seed;
  bool stamps;
};
// lists == nullptr: every CTA walks all candidate tiles
int32_t knn_tc2_sweep(sb2_ctx* ctx, const KnnSwitches& sw, const KnnTc2Shape& sh, const __half* Aimg, int64_t a_tile0,
                      const __half* Bimg, int64_t n_points, int64_t n_query, int list_m, float* cand_score, int32_t* cand_idx,
                      double* issued_flops, const KnnTc2Lists* lists = nullptr);
// ---- tile-compact order and tile screen (knn_tc2.cu) ----
// perm[i] = the point at position i of the kd order (deterministic, depends on X alone); coord: split on coordinates
// instead of principal directions; segments of wide_min points or more are split by many CTAs each
int32_t knn_tc2_kd_order(sb2_ctx* ctx, const float* d_x, int64_t n, int d, bool coord, int64_t wide_min, int32_t* perm);
// the query rows [q0, q0 + n_query) in perm's order: qloc[j] = local row, qpos[j] = its position in perm
int32_t knn_tc2_restrict(sb2_ctx* ctx, const int32_t* perm, int64_t n, int64_t q0, int64_t n_query, int32_t* qloc, int32_t* qpos);
// per tile of perm: cent[t * d ..] the centre (fp16-exact in the images' scale), rad[t] >= max |x - cent_t|
int32_t knn_tc2_tile_stats(sb2_ctx* ctx, const float* d_x, int64_t n, int d, const int32_t* perm, const unsigned int* d_maxnorm_bits,
                           float* cent, float* rad);
// lists [n_blocks][nt]: the nt consecutive tiles around the tile of each block's first row (qpos == nullptr: row = position)
int32_t knn_tc2_near_lists(sb2_ctx* ctx, int64_t n_blocks, int64_t n_tiles, int nt, const int32_t* qpos, int32_t* lists, int32_t* len);
// per query block of Aimg the tiles some row may need (rowp: see knn_screen_kernel): a bitmap of
// knn_tc2_screen_words(n_tiles) words per block and the count of its set bits
int64_t knn_tc2_screen_words(int64_t n_tiles);
int32_t knn_tc2_screen(sb2_ctx* ctx, const KnnTc2Shape& sh, const __half* Aimg, const __half* Cimg, int64_t n_blocks, int64_t n_tiles,
                       const float2* rowp, const float* rad, const unsigned int* d_maxnorm_bits, uint32_t* words, int32_t* list_len);
// the bitmaps as ascending tile lists: block b's at lists[off[b] ..]
int32_t knn_tc2_expand_lists(sb2_ctx* ctx, const uint32_t* words, int64_t n_blocks, int64_t n_tiles, const int64_t* off, int32_t* lists);
void knn_tc2_error_coefs(const KnnTc2Shape& sh, double* c_q, double* c_n);

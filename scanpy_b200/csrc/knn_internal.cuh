// knn_internal.cuh — interface between knn.cu (host entry, re-score, fallback) and knn_tc2.cu (tensor-core sweep)
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

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
// unused slots hold the sub-list's starting threshold (-inf for a cold start) and id -1
int32_t knn_tc2_sweep(sb2_ctx* ctx, const KnnTc2Shape& sh, const __half* Aimg, int64_t a_tile0, const __half* Bimg,
                      int64_t n_points, int64_t n_query, int list_m, float* cand_score, int32_t* cand_idx, double* issued_flops,
                      bool estimate = true);
void knn_tc2_error_coefs(const KnnTc2Shape& sh, double* c_q, double* c_n);

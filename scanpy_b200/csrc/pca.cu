// pca.cu — PCA of an implicitly centred CSR matrix (sm_90a).
//
// Replaces sklearn PCA(svd_solver='arpack') -> scipy svds -> ARPACK as called by the reference at
// src/scanpy/preprocessing/_pca/__init__.py:282-291,308 (arithmetic spec: SURVEY.md Appendix A1),
// and the `covariance_eigh` Gram route of src/scanpy/preprocessing/_pca/_dask.py:143-213 +
// _pca/_kernels.py:14-58.
//
// Kernels (all HBM/L2-bound integer+fp32 streaming work; no tensor cores):
//   csr_col_stats_kernel   one CSR pass: per-gene sum and sum of squares (fp64 REDs into replicated
//                          accumulators)                                   bytes: 8*nnz + 8*(n+1)
//   spmm_csr_kernel        Y = X*B - 1*shift^T, warp per row, lanes own l/32 columns of B;
//                          coalesced column-index loads, shuffle-broadcast of (col,val), B rows are
//                          read as one 128..512 B segment per non-zero     bytes: 8*nnz + 4*n*l
//   spmm_csr_t_kernel      Z += X^T*Y, warp per row, (l/4) lanes per non-zero issue one
//                          RED.ADD.F32x4 each into one of 8 replicated fp32 copies of Z (L2 resident)
//   csr_gram_kernel        G += x_r x_r^T (upper triangle), warp per row, fp64 REDs into L2-resident G
//   small dense fp64 helpers (g x l blocks, l <= 128): A^T B, A*M, C*V, residual norms.
//   rr_jacobi_kernel       the l x l Rayleigh-Ritz eigenproblem for l <= 64, one CTA (fp64).
// Host side (C++ in this file): the block subspace iteration, CholeskyQR2 with an eigen-based
// fallback for rank-deficient blocks, and a cyclic-Jacobi eigensolver for the l = 128 Rayleigh-Ritz
// problem (fp64).  Centering never densifies X:  X_c B = X B - 1 (mu^T B) and, because
// the columns of that product sum to zero, X_c^T (X_c B) = X^T (X B - 1 mu^T B).
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace {

constexpr int STAT_COPIES = 32;
constexpr int ZT_COPIES = 8;

// ---------------------------------------------------------------------------------------------
__global__ void csr_col_stats_kernel(int64_t nnz, const int32_t* __restrict__ indices, const float* __restrict__ data,
                                     int g, double* __restrict__ acc /* [COPIES][2][g] */) {
  double* mine = acc + (size_t)(blockIdx.x % STAT_COPIES) * 2 * g;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = indices[i];
    const double v = data[i];
    atomicAdd(&mine[c], v);
    atomicAdd(&mine[g + c], v * v);
  }
}
__global__ void reduce_copies_f64_kernel(const double* __restrict__ src, int copies, int64_t len, double* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= len) return;
  double s = 0.0;
  for (int c = 0; c < copies; ++c) s += src[(size_t)c * len + i];
  dst[i] = s;
}
__global__ void reduce_copies_f32_to_f64_kernel(const float* __restrict__ src, int copies, int64_t len,
                                                double* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= len) return;
  double s = 0.0;
  for (int c = 0; c < copies; ++c) s += (double)src[(size_t)c * len + i];
  dst[i] = s;
}

// ---------------------------------------------------------------------------------------------
// Y[r, 0:ncols_out] = sum_e data[e] * B[indices[e], :] - shift     (row stride of Y = ldy)
template <int LPT>  // columns of B per lane: l = 32*LPT
__global__ void __launch_bounds__(256)
spmm_csr_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                const float* __restrict__ data, const float* __restrict__ B, const float* __restrict__ shift,
                float* __restrict__ Y, int ldy, int ncols_out) {
  constexpr int L = 32 * LPT;
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int64_t e0 = indptr[row], e1 = indptr[row + 1];
  float acc[LPT];
#pragma unroll
  for (int j = 0; j < LPT; ++j) acc[j] = 0.0f;
  for (int64_t e = e0; e < e1; e += 32) {
    const int cnt = (int)min((int64_t)32, e1 - e);
    int c = 0;
    float v = 0.0f;
    if (lane < cnt) {
      c = indices[e + lane];
      v = data[e + lane];
    }
    for (int j = 0; j < cnt; ++j) {
      const int cj = __shfl_sync(0xffffffffu, c, j);
      const float vj = __shfl_sync(0xffffffffu, v, j);
      const float* b = B + (size_t)cj * L + lane * LPT;
      if (LPT == 1) {
        acc[0] = fmaf(vj, b[0], acc[0]);
      } else if (LPT == 2) {
        const float2 bb = *reinterpret_cast<const float2*>(b);
        acc[0] = fmaf(vj, bb.x, acc[0]);
        acc[1] = fmaf(vj, bb.y, acc[1]);
      } else {
        const float4 bb = *reinterpret_cast<const float4*>(b);
        acc[0] = fmaf(vj, bb.x, acc[0]);
        acc[1] = fmaf(vj, bb.y, acc[1]);
        acc[2] = fmaf(vj, bb.z, acc[2]);
        acc[3] = fmaf(vj, bb.w, acc[3]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < LPT; ++j) {
    const int col = lane * LPT + j;
    if (col < ncols_out) Y[row * (int64_t)ldy + col] = acc[j] - (shift ? shift[col] : 0.0f);
  }
}

// Z_copy[c, :] += data[e] * Y[r, :] for every non-zero (r, c); l in {32, 64, 128}
template <int L>
__global__ void __launch_bounds__(256)
spmm_csr_t_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                  const float* __restrict__ data, const float* __restrict__ Y, float* __restrict__ Zc, int g) {
  constexpr int LANES = L / 4;       // lanes per non-zero
  constexpr int GROUPS = 32 / LANES;  // non-zeros per warp instruction
  const int lane = threadIdx.x & 31;
  const int sub = lane % LANES, grp = lane / LANES;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  float* Z = Zc + (size_t)(blockIdx.x % ZT_COPIES) * g * L;
  const float4 y = *reinterpret_cast<const float4*>(Y + row * (int64_t)L + 4 * sub);
  const int64_t e0 = indptr[row], e1 = indptr[row + 1];
  for (int64_t e = e0; e < e1; e += 32) {
    const int cnt = (int)min((int64_t)32, e1 - e);
    int c = 0;
    float v = 0.0f;
    if (lane < cnt) {
      c = indices[e + lane];
      v = data[e + lane];
    }
    for (int j = 0; j < cnt; j += GROUPS) {
      const int jj = j + grp;
      const int cj = __shfl_sync(0xffffffffu, c, jj & 31);
      const float vj = __shfl_sync(0xffffffffu, v, jj & 31);
      if (jj < cnt) {
        float4* dst = reinterpret_cast<float4*>(Z + (size_t)cj * L + 4 * sub);
        atomicAdd(dst, make_float4(vj * y.x, vj * y.y, vj * y.z, vj * y.w));
      }
    }
  }
}

// G[ci, cj] += vi*vj for i <= j within a row (columns ascending within a CSR row => upper triangle
// when the row is sorted; unsorted rows are handled by ordering the pair)
__global__ void __launch_bounds__(256)
csr_gram_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                const float* __restrict__ data, double* __restrict__ G, int g) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int64_t e0 = indptr[row], e1 = indptr[row + 1];
  for (int64_t i = e0; i < e1; ++i) {
    const int ci = indices[i];
    const double vi = data[i];
    for (int64_t j = i + lane; j < e1; j += 32) {
      const int cj = indices[j];
      const double p = vi * (double)data[j];
      const int a = min(ci, cj), b = max(ci, cj);
      atomicAdd(&G[(size_t)a * g + b], p);
    }
  }
}

// ---- Gram matrix, tiled variant (opt-in, SB2_GRAM_TILED=1; measured slower than the kernel above, see sb2_csr_gram) ----------
// The kernel above issues one global fp64 RED per product (6.5e9 at 1.3M x 2000, ~195 G RED/s = 33 ms).
// Here the g columns are cut into NB blocks of GT_W; a CTA owns one tile pair (bi <= bj) of G for a contiguous range of
// rows and keeps that GT_W x GT_W fp64 tile in shared memory (128 KB): for every row, the entries falling into blocks bi
// and bj (contiguous, rows are column-sorted; their positions come from a per-row block-offset table built once) are
// multiplied pairwise and added with shared-memory atomics; the tile is flushed to G with one global RED per non-zero
// tile entry at the end.  CTAs are ordered row-range-major, so the CTAs resident at any time walk the same rows and the
// CSR streams through the L2 once per wave instead of once per tile pair.
constexpr int GT_W = 128;
constexpr int GT_THREADS = 512;
// boff[row * (NB+1) + b] = number of entries of the row with column < b * GT_W (uint16: a row holds < 65536 entries);
// *flag |= 1 if a row is not column-sorted or too long (the caller then falls back to the first-generation kernel)
__global__ void __launch_bounds__(256)
gram_block_offsets_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int NB,
                          uint16_t* __restrict__ boff, int* __restrict__ flag) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int64_t e0 = indptr[row], e1 = indptr[row + 1];
  if (e1 - e0 >= 65536) { if (lane == 0) atomicOr(flag, 1); }
  int lo = 0, hi = 0;  // counts for b = lane and b = lane + 32
  int prev_last = -1;
  bool bad = false;
  for (int64_t e = e0; e < e1; e += 32) {
    const bool on = e + lane < e1;
    const int c = on ? indices[e + lane] : 0x7fffffff;
    int pc = __shfl_up_sync(0xffffffffu, c, 1);
    if (lane == 0) pc = prev_last;
    if (on && pc > c) bad = true;
    prev_last = __shfl_sync(0xffffffffu, c, 31);
    const int blk = on ? c / GT_W : 0x7fffffff;
    for (int b = 1; b <= NB; ++b) {
      const int x = __popc(__ballot_sync(0xffffffffu, on && blk < b));
      if (b == lane) lo += x;
      if (b == lane + 32) hi += x;
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(flag, 1);
  uint16_t* o = boff + (size_t)row * (NB + 1);
  if (lane <= NB) o[lane] = (uint16_t)lo;
  if (lane + 32 <= NB) o[lane + 32] = (uint16_t)hi;
}
__global__ void __launch_bounds__(GT_THREADS, 1)
csr_gram_tiles_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                      const float* __restrict__ data, const uint16_t* __restrict__ boff, int NB, int n_pairs,
                      const int2* __restrict__ pair_tab, int64_t rows_per_range, double* __restrict__ G, int g) {
  extern __shared__ double tile[];  // [GT_W][GT_W]
  const int pair = blockIdx.x % n_pairs;
  const int64_t range = blockIdx.x / n_pairs;
  const int bi = pair_tab[pair].x, bj = pair_tab[pair].y;
  for (int t = threadIdx.x; t < GT_W * GT_W; t += GT_THREADS) tile[t] = 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = range * rows_per_range, r1 = min(n, r0 + rows_per_range);
  const bool diag = bi == bj;
  for (int64_t row = r0 + warp; row < r1; row += GT_THREADS / 32) {
    const uint16_t* bo = boff + (size_t)row * (NB + 1);
    const int a0 = bo[bi], p = (int)bo[bi + 1] - a0;
    const int b0 = bo[bj], q = (int)bo[bj + 1] - b0;
    if (p <= 0 || q <= 0) continue;
    const int64_t base = indptr[row];
    for (int ia = 0; ia < p; ia += 32) {
      const int na = min(32, p - ia);
      int ca = 0;
      double va = 0.0;
      if (lane < na) { ca = indices[base + a0 + ia + lane] - bi * GT_W; va = (double)data[base + a0 + ia + lane]; }
      for (int ib = 0; ib < q; ib += 32) {
        if (diag && ib + 31 < ia) continue;  // every (i, j) of this chunk pair has j < i
        const int nb = min(32, q - ib);
        int cb = 0;
        double vb = 0.0;
        if (lane < nb) { cb = indices[base + b0 + ib + lane] - bj * GT_W; vb = (double)data[base + b0 + ib + lane]; }
        const int np = na * nb;
        for (int t0 = 0; t0 < np; t0 += 32) {
          const int t = t0 + lane;
          const bool on = t < np;
          const int i = on ? t / nb : 0, j = on ? t - i * nb : 0;
          const int ci = __shfl_sync(0xffffffffu, ca, i), cj = __shfl_sync(0xffffffffu, cb, j);
          const double vi = __shfl_sync(0xffffffffu, va, i), vj = __shfl_sync(0xffffffffu, vb, j);
          // diagonal tiles: each unordered pair of entries once (positions i <= j; sorted columns => ci <= cj)
          if (on && (!diag || ia + i <= ib + j)) atomicAdd(&tile[ci * GT_W + cj], vi * vj);
        }
      }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < GT_W * GT_W; t += GT_THREADS) {
    const double v = tile[t];
    if (v != 0.0) {
      const int r = bi * GT_W + t / GT_W, c = bj * GT_W + t % GT_W;
      if (r < g && c < g) atomicAdd(&G[(size_t)r * g + c], v);
    }
  }
}
__global__ void mirror_upper_kernel(double* __restrict__ G, int g) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)g * g) return;
  const int r = (int)(i / g), c = (int)(i % g);
  if (r > c) G[i] = G[(size_t)c * g + r];
}
// C = G - n * mu mu^T   (in place)
__global__ void center_gram_kernel(double* __restrict__ G, const double* __restrict__ mu, double n_total, int g) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)g * g) return;
  const int r = (int)(i / g), c = (int)(i % g);
  G[i] -= n_total * mu[r] * mu[c];
}

// ---------------------------------------------------------------------------------------------
// small dense fp64 helpers on g x l blocks (row-major, leading dimension l)
// S[l x l] += A^T B over a chunk of rows (grid.x chunks); S must be zeroed first
__global__ void __launch_bounds__(256)
tsmm_tn_kernel(const double* __restrict__ A, const double* __restrict__ B, int g, int l, double* __restrict__ S) {
  extern __shared__ double sm[];  // [2][ROWS][l]
  constexpr int ROWS = 32;
  double* sa = sm;
  double* sb = sm + ROWS * l;
  const int r0 = blockIdx.x * ROWS;
  const int rows = min(ROWS, g - r0);
  for (int i = threadIdx.x; i < ROWS * l; i += blockDim.x) {
    const int r = i / l;
    sa[i] = r < rows ? A[(size_t)(r0 + r) * l + (i % l)] : 0.0;
    sb[i] = r < rows ? B[(size_t)(r0 + r) * l + (i % l)] : 0.0;
  }
  __syncthreads();
  for (int o = threadIdx.x; o < l * l; o += blockDim.x) {
    const int i = o / l, j = o % l;
    double s = 0.0;
#pragma unroll 8
    for (int r = 0; r < ROWS; ++r) s = fma(sa[r * l + i], sb[r * l + j], s);
    atomicAdd(&S[o], s);
  }
}
// C[g x lo] = A[g x l] * M[l x lo]
__global__ void __launch_bounds__(256)
right_mult_kernel(const double* __restrict__ A, const double* __restrict__ M, int g, int l, int lo,
                  double* __restrict__ C) {
  extern __shared__ double sm[];  // M
  for (int i = threadIdx.x; i < l * lo; i += blockDim.x) sm[i] = M[i];
  __syncthreads();
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (int64_t)g * lo) return;
  const int r = (int)(o / lo), c = (int)(o % lo);
  double s = 0.0;
  for (int k = 0; k < l; ++k) s = fma(A[(size_t)r * l + k], sm[k * lo + c], s);
  C[o] = s;
}
// Z[g x l] += C[g x g] * V[g x l]   (C symmetric, dense fp64; Z zeroed by the caller)
// 64 x 64 output tile per CTA, 4 x 4 per thread (16 FMA per 4 LDS.128), the K axis split over gridDim.y CTAs that
// merge with fp64 REDs: 256 CTAs for g = 2000, l = 64 instead of 125 LDS-bound ones.
constexpr int DSA_T = 64, DSA_K = 16, DSA_PAD = 66;
__global__ void __launch_bounds__(256)
dense_sym_apply_kernel(const double* __restrict__ C, const double* __restrict__ V, int g, int l, int k_per_split,
                       double* __restrict__ Z) {
  __shared__ __align__(16) double Cs[DSA_K][DSA_PAD];  // k-major: Cs[k][row]
  __shared__ __align__(16) double Vs[DSA_K][DSA_T];
  const int r0 = blockIdx.x * DSA_T, c0 = blockIdx.z * DSA_T;
  const int kb = blockIdx.y * k_per_split, ke = min(g, kb + k_per_split);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
  for (int k0 = kb; k0 < ke; k0 += DSA_K) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int i = threadIdx.x + it * 256;
      const int r = i >> 4, k = i & 15;  // 16 consecutive k of one row: 128 B per half-warp
      Cs[k][r] = (r0 + r < g && k0 + k < ke) ? C[(size_t)(r0 + r) * g + k0 + k] : 0.0;
      const int vk = i >> 6, vc = i & 63;
      Vs[vk][vc] = (k0 + vk < ke && c0 + vc < l) ? V[(size_t)(k0 + vk) * l + c0 + vc] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < DSA_K; ++k) {
      const double2 a01 = *reinterpret_cast<const double2*>(&Cs[k][ty * 4]);
      const double2 a23 = *reinterpret_cast<const double2*>(&Cs[k][ty * 4 + 2]);
      const double2 b01 = *reinterpret_cast<const double2*>(&Vs[k][tx * 4]);
      const double2 b23 = *reinterpret_cast<const double2*>(&Vs[k][tx * 4 + 2]);
      const double a[4] = {a01.x, a01.y, a23.x, a23.y};
      const double bb[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty * 4 + i;
    if (r >= g) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + tx * 4 + j;
      if (c < l) atomicAdd(&Z[(size_t)r * l + c], acc[i][j]);
    }
  }
}
// res2[j] += sum_r (Z[r,j] - theta[j] * V[r,j])^2 ; res2 zeroed first
__global__ void residual_kernel(const double* __restrict__ Z, const double* __restrict__ V,
                                const double* __restrict__ theta, int g, int l, double* __restrict__ res2) {
  const int j = threadIdx.x % l;
  const int rstep = blockDim.x / l;
  double s = 0.0;
  for (int r = blockIdx.x * rstep + threadIdx.x / l; r < g; r += gridDim.x * rstep) {
    const double d = Z[(size_t)r * l + j] - theta[j] * V[(size_t)r * l + j];
    s = fma(d, d, s);
  }
  if (threadIdx.x < rstep * l) atomicAdd(&res2[j], s);
}
// out = a*Z + b*Y + c*W  (elementwise; W may alias nothing when c == 0)
__global__ void lincomb3_kernel(int64_t n, double a, const double* __restrict__ Z, double b, const double* __restrict__ Y,
                                double c, const double* __restrict__ W, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a * Z[i] + b * Y[i] + (c != 0.0 ? c * W[i] : 0.0);
}
__global__ void f64_to_f32_kernel(const double* __restrict__ s, float* __restrict__ d, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = (float)s[i];
}
// components[k x g] (float32) = first k columns of U[g x l], transposed, times sign[j]
__global__ void components_out_kernel(const double* __restrict__ U, const double* __restrict__ sign, int g, int l, int k,
                                      float* __restrict__ comp) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)k * g) return;
  const int j = (int)(i / g), r = (int)(i % g);
  comp[i] = (float)(U[(size_t)r * l + j] * sign[j]);
}
// per column j < l: value with max |.| (first occurrence); one block per column
__global__ void col_absmax_kernel(const double* __restrict__ U, int g, int l, double* __restrict__ out) {
  __shared__ double sv[256];
  __shared__ int si[256];
  const int j = blockIdx.x;
  double best = -1.0;
  int bi = 0x7fffffff;
  for (int r = threadIdx.x; r < g; r += blockDim.x) {
    const double a = fabs(U[(size_t)r * l + j]);
    if (a > best) { best = a; bi = r; }
  }
  sv[threadIdx.x] = best;
  si[threadIdx.x] = bi;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const double o = sv[threadIdx.x + s];
      const int oi = si[threadIdx.x + s];
      if (o > sv[threadIdx.x] || (o == sv[threadIdx.x] && oi < si[threadIdx.x])) { sv[threadIdx.x] = o; si[threadIdx.x] = oi; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[j] = U[(size_t)si[0] * l + j];
}

// 1024 threads: a Jacobi step updates 2 x (m/2) x m = 2 x 2048 entries (m = 64) between barriers - two per thread; with 256
// threads the kernel took 0.73 ms per call (19 calls = 14 ms of the 62 ms PCA at 1.3M x 2000)
constexpr int RRJ_THREADS = 1024;
// ---------------------------------------------------------------------------------------------
// Rayleigh-Ritz eigenproblem on the device: S (m x m, m = block width <= 64, symmetrised on load) -> eigenvalues in
// descending order and the matching eigenvectors (columns of W).  One CTA, two-sided Jacobi with the round-robin
// ("tournament") ordering: every step rotates m/2 disjoint index pairs at once - rotation angles, column update of A and
// V, row update of A - so a sweep is m-1 steps of three barriers instead of m(m-1)/2 sequential rotations.  Replaces the
// host-side cyclic Jacobi (a few milliseconds of single-threaded CPU work and a device round trip per Rayleigh-Ritz step,
// replicated on every rank).
__global__ void __launch_bounds__(RRJ_THREADS)
rr_jacobi_kernel(const double* __restrict__ S, int m, double* __restrict__ W, double* __restrict__ theta) {
  extern __shared__ double sm[];
  const int ld = m + 1;
  double* A = sm;                 // [m][ld]
  double* V = A + (size_t)m * ld;  // [m][ld]
  double* cs = V + (size_t)m * ld;  // [m/2]
  double* sn = cs + m / 2;         // [m/2]
  double* red = sn + m / 2;        // [RRJ_THREADS] reduction scratch, then eigenvalues
  int* top = reinterpret_cast<int*>(red + RRJ_THREADS);  // [m/2]
  int* bot = top + m / 2;                        // [m/2]
  __shared__ int done;
  const int tid = threadIdx.x, nt = blockDim.x, half = m / 2;
  for (int i = tid; i < m * m; i += nt) {
    const int r = i / m, c = i % m;
    A[r * ld + c] = 0.5 * (S[r * m + c] + S[c * m + r]);
    V[r * ld + c] = r == c ? 1.0 : 0.0;
  }
  for (int p = tid; p < half; p += nt) { top[p] = 2 * p; bot[p] = 2 * p + 1; }
  __syncthreads();
  for (int sweep = 0; sweep < 40; ++sweep) {
    double off = 0.0, dg = 0.0;
    for (int i = tid; i < m * m; i += nt) {
      const int r = i / m, c = i % m;
      const double a = A[r * ld + c];
      if (r == c) dg += a * a; else if (c > r) off += a * a;
    }
    red[tid] = off;
    __syncthreads();
    for (int k = nt / 2; k > 0; k >>= 1) { if (tid < k) red[tid] += red[tid + k]; __syncthreads(); }
    const double offs = red[0];
    __syncthreads();
    red[tid] = dg;
    __syncthreads();
    for (int k = nt / 2; k > 0; k >>= 1) { if (tid < k) red[tid] += red[tid + k]; __syncthreads(); }
    if (tid == 0) done = (offs <= 1e-30 * (red[0] + offs) || offs == 0.0) ? 1 : 0;
    __syncthreads();
    if (done) break;
    for (int step = 0; step < m - 1; ++step) {
      if (tid < half) {
        const int a = top[tid], b = bot[tid];
        const int i = min(a, b), j = max(a, b);
        const double apq = A[i * ld + j];
        double c = 1.0, sv = 0.0;
        if (fabs(apq) >= 1e-300) {
          const double tau = (A[j * ld + j] - A[i * ld + i]) / (2.0 * apq);
          const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
          c = 1.0 / sqrt(1.0 + t * t);
          sv = t * c;
        }
        cs[tid] = c; sn[tid] = sv;
      }
      __syncthreads();
      for (int it = tid; it < half * m; it += nt) {   // columns i, j of A and V
        const int p = it / m, k = it % m;
        const int a = top[p], b = bot[p];
        const int i = min(a, b), j = max(a, b);
        const double c = cs[p], sv = sn[p];
        const double aki = A[k * ld + i], akj = A[k * ld + j];
        A[k * ld + i] = c * aki - sv * akj;
        A[k * ld + j] = sv * aki + c * akj;
        const double vki = V[k * ld + i], vkj = V[k * ld + j];
        V[k * ld + i] = c * vki - sv * vkj;
        V[k * ld + j] = sv * vki + c * vkj;
      }
      __syncthreads();
      for (int it = tid; it < half * m; it += nt) {   // rows i, j of A
        const int p = it / m, k = it % m;
        const int a = top[p], b = bot[p];
        const int i = min(a, b), j = max(a, b);
        const double c = cs[p], sv = sn[p];
        const double aik = A[i * ld + k], ajk = A[j * ld + k];
        A[i * ld + k] = c * aik - sv * ajk;
        A[j * ld + k] = sv * aik + c * ajk;
      }
      __syncthreads();
      if (tid == 0) {   // rotate the tournament: top[0] stays, everybody else moves one seat
        const int last_top = top[half - 1], first_bot = bot[0];
        for (int p = half - 1; p > 1; --p) top[p] = top[p - 1];
        if (half > 1) top[1] = first_bot;
        for (int p = 0; p < half - 1; ++p) bot[p] = bot[p + 1];
        bot[half - 1] = half > 1 ? last_top : first_bot;
      }
      __syncthreads();
    }
  }
  // eigenvalues, sorted descending (ties: smaller index first), eigenvectors permuted accordingly
  for (int i = tid; i < m; i += nt) red[i] = A[i * ld + i];
  __syncthreads();
  for (int i = tid; i < m; i += nt) {
    const double wi = red[i];
    int rank = 0;
    for (int j = 0; j < m; ++j) rank += (red[j] > wi || (red[j] == wi && j < i)) ? 1 : 0;
    theta[rank] = wi;
    for (int k = 0; k < m; ++k) W[(size_t)k * m + rank] = V[k * ld + i];
  }
}

// ---------------------------------------------------------------------------------------------
// host fp64 small dense algebra
// cyclic Jacobi: A (m x m symmetric, row-major, destroyed) -> eigenvalues w, eigenvectors V (columns)
void jacobi_eigh(std::vector<double>& A, int m, std::vector<double>& w, std::vector<double>& V) {
  V.assign((size_t)m * m, 0.0);
  for (int i = 0; i < m; ++i) V[(size_t)i * m + i] = 1.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < m; ++i) {
      diag += A[(size_t)i * m + i] * A[(size_t)i * m + i];
      for (int j = i + 1; j < m; ++j) off += A[(size_t)i * m + j] * A[(size_t)i * m + j];
    }
    if (off <= 1e-30 * (diag + off) || off == 0.0) break;
    for (int p = 0; p < m - 1; ++p) {
      for (int q = p + 1; q < m; ++q) {
        const double apq = A[(size_t)p * m + q];
        if (apq == 0.0) continue;
        const double app = A[(size_t)p * m + p], aqq = A[(size_t)q * m + q];
        if (fabs(apq) < 1e-300) continue;
        const double tau = (aqq - app) / (2.0 * apq);
        const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
        const double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
        for (int k = 0; k < m; ++k) {  // columns p,q
          const double akp = A[(size_t)k * m + p], akq = A[(size_t)k * m + q];
          A[(size_t)k * m + p] = c * akp - s * akq;
          A[(size_t)k * m + q] = s * akp + c * akq;
        }
        for (int k = 0; k < m; ++k) {  // rows p,q
          const double apk = A[(size_t)p * m + k], aqk = A[(size_t)q * m + k];
          A[(size_t)p * m + k] = c * apk - s * aqk;
          A[(size_t)q * m + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < m; ++k) {
          const double vkp = V[(size_t)k * m + p], vkq = V[(size_t)k * m + q];
          V[(size_t)k * m + p] = c * vkp - s * vkq;
          V[(size_t)k * m + q] = s * vkp + c * vkq;
        }
      }
    }
  }
  w.resize(m);
  for (int i = 0; i < m; ++i) w[i] = A[(size_t)i * m + i];
}
// sort eigenpairs descending
void sort_desc(std::vector<double>& w, std::vector<double>& V, int m) {
  std::vector<int> ord(m);
  for (int i = 0; i < m; ++i) ord[i] = i;
  std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return w[a] > w[b]; });
  std::vector<double> w2(m), V2((size_t)m * m);
  for (int j = 0; j < m; ++j) {
    w2[j] = w[ord[j]];
    for (int i = 0; i < m; ++i) V2[(size_t)i * m + j] = V[(size_t)i * m + ord[j]];
  }
  w.swap(w2);
  V.swap(V2);
}
// M = R^{-1} with S = R^T R (upper Cholesky); returns false if S is numerically rank deficient
bool chol_inverse_upper(const std::vector<double>& S, int m, std::vector<double>& M) {
  std::vector<double> R((size_t)m * m, 0.0);
  double dmax = 0.0;
  for (int i = 0; i < m; ++i) dmax = std::max(dmax, S[(size_t)i * m + i]);
  for (int j = 0; j < m; ++j) {
    double d = S[(size_t)j * m + j];
    for (int k = 0; k < j; ++k) d -= R[(size_t)k * m + j] * R[(size_t)k * m + j];
    if (!(d > 1e-11 * dmax)) return false;
    const double rjj = sqrt(d);
    R[(size_t)j * m + j] = rjj;
    for (int i = j + 1; i < m; ++i) {
      double s = S[(size_t)j * m + i];
      for (int k = 0; k < j; ++k) s -= R[(size_t)k * m + j] * R[(size_t)k * m + i];
      R[(size_t)j * m + i] = s / rjj;
    }
  }
  M.assign((size_t)m * m, 0.0);  // upper-triangular inverse by back substitution
  for (int j = 0; j < m; ++j) {
    M[(size_t)j * m + j] = 1.0 / R[(size_t)j * m + j];
    for (int i = j - 1; i >= 0; --i) {
      double s = 0.0;
      for (int k = i + 1; k <= j; ++k) s += R[(size_t)i * m + k] * M[(size_t)k * m + j];
      M[(size_t)i * m + j] = -s / R[(size_t)i * m + i];
    }
  }
  return true;
}

struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ULL + 0xD1B54A32D192ED03ULL) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ULL);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
  }
  double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
  double normal() {
    double u1 = uniform(), u2 = uniform();
    if (u1 < 1e-300) u1 = 1e-300;
    return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
  }
};

// Per-call state of the PCA stages
struct PcaWork {
  sb2_ctx* ctx;
  cudaStream_t st;
  int64_t n_total;  // rows over all ranks
  int g, l;         // feature count padded to at least the block width l
  int g_real;       // un-padded feature count
  // operator (solver 1: dense Gram; solver 0: CSR SpMM passes)
  int solver;
  double* d_mu;     // [g_real] operator mean, all zeros without centring (the Gram operator pads it to g)
  double* d_C;      // [g x g] (solver 1)
  int64_t n;        // (solver 0)
  const int64_t* indptr;
  const int32_t* indices;
  const float* data;
  float* d_Y;       // [n x l]
  float* d_Zc;      // [ZT_COPIES x g x l]
  // scratch
  float* d_Bf;      // [g x l] fp32 copy of a block V (the projection U at the end)
  float* d_shift;   // [l] mu^T V of that block
  double* d_S;      // [l x l]
  double* d_M;      // [l x l]
  double *d_Z, *d_tmp, *d_theta, *d_res;  // [g x l], [g x l], [l], [l]
  Rng* rng;         // refills rank-deficient blocks
  // results
  double* d_V;                // [g x l] Ritz vectors, columns by descending Ritz value
  std::vector<double> theta;  // [l] Ritz values
  double total_var0;          // sum of per-gene variances, ddof 0 (TruncatedSVD's ratio denominator)
  sb2_pca_info stats;         // loop statistics and the ddof-1 total variance
};

int32_t launch_spmm(sb2_ctx* ctx, int64_t n, int l, const int64_t* indptr, const int32_t* indices, const float* data,
                    const float* B, const float* shift, float* Y, int ldy, int ncols_out) {
  const int wpb = 8;
  const unsigned grid = (unsigned)ceil_div64(n, wpb);
  if (n == 0) return SB2_OK;
  if (l == 32) spmm_csr_kernel<1><<<grid, wpb * 32, 0, ctx->stream>>>(n, indptr, indices, data, B, shift, Y, ldy, ncols_out);
  else if (l == 64) spmm_csr_kernel<2><<<grid, wpb * 32, 0, ctx->stream>>>(n, indptr, indices, data, B, shift, Y, ldy, ncols_out);
  else if (l == 128) spmm_csr_kernel<4><<<grid, wpb * 32, 0, ctx->stream>>>(n, indptr, indices, data, B, shift, Y, ldy, ncols_out);
  else { sb2_set_error("spmm: l must be 32, 64 or 128 (got %d)", l); return SB2_E_BADARG; }
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}
int32_t launch_spmm_t(sb2_ctx* ctx, int64_t n, int g, int l, const int64_t* indptr, const int32_t* indices,
                      const float* data, const float* Y, float* Zc, double* Z) {
  const int wpb = 8;
  const unsigned grid = (unsigned)ceil_div64(n, wpb);
  SB2_CUDA(cudaMemsetAsync(Zc, 0, sizeof(float) * (size_t)ZT_COPIES * g * l, ctx->stream));
  if (n > 0) {
    if (l == 32) spmm_csr_t_kernel<32><<<grid, wpb * 32, 0, ctx->stream>>>(n, indptr, indices, data, Y, Zc, g);
    else if (l == 64) spmm_csr_t_kernel<64><<<grid, wpb * 32, 0, ctx->stream>>>(n, indptr, indices, data, Y, Zc, g);
    else if (l == 128) spmm_csr_t_kernel<128><<<grid, wpb * 32, 0, ctx->stream>>>(n, indptr, indices, data, Y, Zc, g);
    else { sb2_set_error("spmm_t: l must be 32, 64 or 128 (got %d)", l); return SB2_E_BADARG; }
    SB2_LAUNCH_CHECK(ctx);
  }
  const int64_t len = (int64_t)g * l;
  reduce_copies_f32_to_f64_kernel<<<(unsigned)ceil_div64(len, 256), 256, 0, ctx->stream>>>(Zc, ZT_COPIES, len, Z);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

// S = A^T B (device, l x l) in w.d_S, and copied to hS unless it is null
int32_t tsmm(PcaWork& w, const double* A, const double* B, std::vector<double>* hS) {
  const int l = w.l;
  SB2_CUDA(cudaMemsetAsync(w.d_S, 0, sizeof(double) * l * l, w.st));
  tsmm_tn_kernel<<<(unsigned)ceil_div64(w.g, 32), 256, sizeof(double) * 2 * 32 * l, w.st>>>(A, B, w.g, l, w.d_S);
  SB2_LAUNCH_CHECK(w.ctx);
  if (!hS) return SB2_OK;
  hS->resize((size_t)l * l);
  SB2_CUDA(cudaMemcpyAsync(hS->data(), w.d_S, sizeof(double) * l * l, cudaMemcpyDeviceToHost, w.st));
  SB2_CUDA(cudaStreamSynchronize(w.st));
  return SB2_OK;
}
// A <- A * M with M on the device (l x l)
int32_t right_mult_device(PcaWork& w, double* A, const double* dM) {
  const int l = w.l;
  right_mult_kernel<<<(unsigned)ceil_div64((int64_t)w.g * l, 256), 256, sizeof(double) * l * l, w.st>>>(A, dM, w.g, l, l, w.d_tmp);
  SB2_LAUNCH_CHECK(w.ctx);
  SB2_CUDA(cudaMemcpyAsync(A, w.d_tmp, sizeof(double) * (size_t)w.g * l, cudaMemcpyDeviceToDevice, w.st));
  return SB2_OK;
}
// A <- A * M (M host l x l)
int32_t right_mult_inplace(PcaWork& w, double* A, const std::vector<double>& hM) {
  SB2_CUDA(cudaMemcpyAsync(w.d_M, hM.data(), sizeof(double) * w.l * w.l, cudaMemcpyHostToDevice, w.st));
  return right_mult_device(w, A, w.d_M);
}
size_t rr_jacobi_smem(int l) { return sizeof(double) * (2 * (size_t)l * (l + 1) + l + RRJ_THREADS) + sizeof(int) * l; }
// Rayleigh-Ritz step: S = V^T Z, its eigenvectors W, V <- V W (Ritz vectors), Z <- Z W (A * Ritz vectors), d_theta <- Ritz
// values (descending).  Blocks up to 64 wide solve S on the device (rr_jacobi_kernel) and nothing travels to the host; the
// 128-wide block's two l x l matrices do not fit one CTA's shared memory, so its S goes through the host Jacobi.
int32_t rayleigh_ritz(PcaWork& w, double* V, double* Z, double* d_theta) {
  const int l = w.l;
  if (l <= 64) {
    SB2_TRY(tsmm(w, V, Z, nullptr));
    rr_jacobi_kernel<<<1, RRJ_THREADS, rr_jacobi_smem(l), w.st>>>(w.d_S, l, w.d_M, d_theta);
    SB2_LAUNCH_CHECK(w.ctx);
    SB2_TRY(right_mult_device(w, V, w.d_M));
    return right_mult_device(w, Z, w.d_M);
  }
  std::vector<double> T, theta, W;
  SB2_TRY(tsmm(w, V, Z, &T));
  for (int i = 0; i < l; ++i)  // symmetrise
    for (int j = i + 1; j < l; ++j) {
      const double a = 0.5 * (T[(size_t)i * l + j] + T[(size_t)j * l + i]);
      T[(size_t)i * l + j] = T[(size_t)j * l + i] = a;
    }
  jacobi_eigh(T, l, theta, W);
  sort_desc(theta, W, l);
  SB2_TRY(right_mult_inplace(w, V, W));
  SB2_TRY(right_mult_inplace(w, Z, W));
  SB2_CUDA(cudaMemcpyAsync(d_theta, theta.data(), sizeof(double) * l, cudaMemcpyHostToDevice, w.st));
  return SB2_OK;
}
// orthonormalise the columns of A (g x l): CholeskyQR, twice; eigen-based fallback if rank deficient
int32_t orthonormalize(PcaWork& w, double* A) {
  const int l = w.l;
  std::vector<double> S, M, dsc(l);
  for (int attempt = 0; attempt < 3; ++attempt) {
    std::vector<int> dropped;
    for (int pass = 0; pass < 2; ++pass) {
      SB2_TRY(tsmm(w, A, A, &S));
      // column scaling first: after a Chebyshev filter the columns differ by many orders of magnitude
      // (each is amplified by p(theta_j)), which would make the Gram matrix numerically singular although the
      // columns are nearly orthogonal.  S' = D^-1/2 S D^-1/2 has a unit diagonal.
      for (int j = 0; j < l; ++j) dsc[j] = S[(size_t)j * l + j] > 0.0 ? 1.0 / sqrt(S[(size_t)j * l + j]) : 0.0;
      for (int i = 0; i < l; ++i)
        for (int j = 0; j < l; ++j) S[(size_t)i * l + j] *= dsc[i] * dsc[j];
      for (int j = 0; j < l; ++j)
        if (dsc[j] == 0.0) S[(size_t)j * l + j] = 1.0;  // all-zero column stays zero
      if (!chol_inverse_upper(S, l, M)) {
        std::vector<double> ev, W;
        jacobi_eigh(S, l, ev, W);
        double emax = 0.0;
        for (double e : ev) emax = std::max(emax, e);
        M.assign((size_t)l * l, 0.0);
        for (int j = 0; j < l; ++j) {
          const double sc = ev[j] > 1e-12 * emax ? 1.0 / sqrt(ev[j]) : 0.0;  // null directions -> zero columns
          for (int i = 0; i < l; ++i) M[(size_t)i * l + j] = W[(size_t)i * l + j] * sc;
        }
      }
      for (int i = 0; i < l; ++i)
        for (int j = 0; j < l; ++j) M[(size_t)i * l + j] *= dsc[i];  // A D^-1/2 M'
      SB2_TRY(right_mult_inplace(w, A, M));
      if (pass == 1) {
        for (int j = 0; j < l; ++j) {
          bool zero = true;
          for (int i = 0; i < l && zero; ++i) zero = M[(size_t)i * l + j] == 0.0;
          if (zero) dropped.push_back(j);
        }
      }
    }
    // directions lost to rank deficiency are replaced by fresh random vectors (only while the feature space
    // can still hold l independent directions) and the block is orthonormalised again
    if (dropped.empty() || w.g_real < l || attempt == 2) break;
    std::vector<double> col((size_t)w.g);
    for (int j : dropped) {
      for (int r = 0; r < w.g; ++r) col[r] = r < w.g_real ? w.rng->normal() : 0.0;
      SB2_CUDA(cudaMemcpy2DAsync(A + j, sizeof(double) * l, col.data(), sizeof(double), sizeof(double), (size_t)w.g,
                                 cudaMemcpyHostToDevice, w.st));
      SB2_CUDA(cudaStreamSynchronize(w.st));
    }
  }
  return SB2_OK;
}
__global__ void mu_dot_kernel(const double* __restrict__ mu, const double* __restrict__ V, int g, int l,
                              float* __restrict__ shift) {
  // one block per column j
  __shared__ double red[256];
  const int j = blockIdx.x;
  double s = 0.0;
  for (int r = threadIdx.x; r < g; r += blockDim.x) s = fma(mu[r], V[(size_t)r * l + j], s);
  red[threadIdx.x] = s;
  __syncthreads();
  for (int k = blockDim.x / 2; k > 0; k >>= 1) {
    if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x == 0) shift[j] = (float)red[0];
}

// Z = A_op * V  (V, Z device g x l fp64); A_op = X_c^T X_c summed over all ranks
int32_t apply_operator(PcaWork& w, const double* V, double* Z) {
  const int g = w.g, l = w.l;
  if (w.solver == 1) {
    // split K so that the grid covers the machine about twice over (fp64 REDs merge the partial tiles)
    const int row_tiles = (int)ceil_div64(g, DSA_T), col_tiles = (int)ceil_div64(l, DSA_T);
    int ksplit = std::max(1, (2 * w.ctx->prop.multiProcessorCount) / (row_tiles * col_tiles));
    ksplit = std::min(ksplit, (int)ceil_div64(g, 4 * DSA_K));
    const int k_per_split = (int)ceil_div64(ceil_div64(g, ksplit), DSA_K) * DSA_K;
    SB2_CUDA(cudaMemsetAsync(Z, 0, sizeof(double) * (size_t)g * l, w.st));
    dense_sym_apply_kernel<<<dim3((unsigned)row_tiles, (unsigned)ceil_div64(g, k_per_split), (unsigned)col_tiles), 256, 0, w.st>>>(
        w.d_C, V, g, l, k_per_split, Z);
    SB2_LAUNCH_CHECK(w.ctx);
    return SB2_OK;
  }
  const int64_t len = (int64_t)g * l;
  f64_to_f32_kernel<<<(unsigned)ceil_div64(len, 256), 256, 0, w.st>>>(V, w.d_Bf, len);
  SB2_LAUNCH_CHECK(w.ctx);
  mu_dot_kernel<<<l, 256, 0, w.st>>>(w.d_mu, V, g, l, w.d_shift);
  SB2_LAUNCH_CHECK(w.ctx);
  SB2_TRY(launch_spmm(w.ctx, w.n, l, w.indptr, w.indices, w.data, w.d_Bf, w.d_shift, w.d_Y, l, l));
  SB2_TRY(launch_spmm_t(w.ctx, w.n, g, l, w.indptr, w.indices, w.data, w.d_Y, w.d_Zc, Z));
  return sb2_comm_allreduce_f64(w.ctx, Z, len);
}

// ---------------------------------------------------------------------------------------------
// host stages of the PCA entries
// Shape checks, block width l (k + oversampling, one of the kernel-supported widths) and route.  g < l genes are padded to
// w.g = l (all-zero genes, eigenvalue 0) and take the dense Gram route.
int32_t init_work(sb2_ctx* ctx, int64_t n, int64_t n_total, int g, int k, int solver, PcaWork& w) {
  SB2_CHECK_ARG(n >= 0 && n_total >= n && n_total >= 2 && g >= 1, "shape");
  SB2_CHECK_ARG(k >= 1 && k < std::min<int64_t>(n_total, g), "n_components must be between 1 and min(n_samples, n_features)-1");
  SB2_CHECK_ARG(k <= 120, "n_components <= 120");
  SB2_CHECK_ARG(solver == 0 || solver == 1, "solver");
  SB2_CUDA(cudaSetDevice(ctx->device));
  const int l = (k + 8 <= 32) ? 32 : (k + 8 <= 64 ? 64 : 128);
  w.ctx = ctx; w.st = ctx->stream; w.n_total = n_total; w.l = l;
  w.g_real = g; w.g = std::max(g, l);
  w.solver = g < l ? 1 : solver;
  return SB2_OK;
}
// The scratch of the iteration, and w.d_mu [g] for the caller to fill.  Allocated after the column statistics and before the
// operator: the order decides where the g x g Gram matrix lands in the memory pool, and csr_gram_kernel's fp64 REDs took
// 84.1 instead of 82.1 ms (1.3M x 2000, H100 80GB HBM3 at 700 W) with this scratch allocated ahead of the statistics.
int32_t alloc_scratch(PcaWork& w, ScratchScope& scr) {
  const size_t l = w.l, blk = (size_t)w.g * l;
  SB2_TRY(scr.alloc(&w.d_mu, (size_t)w.g_real));
  SB2_TRY(scr.alloc(&w.d_S, l * l));
  SB2_TRY(scr.alloc(&w.d_M, l * l));
  SB2_TRY(scr.alloc(&w.d_V, blk));
  SB2_TRY(scr.alloc(&w.d_Z, blk));
  SB2_TRY(scr.alloc(&w.d_tmp, blk));
  SB2_TRY(scr.alloc(&w.d_theta, l));
  SB2_TRY(scr.alloc(&w.d_res, l));
  return scr.alloc(&w.d_Bf, blk);
}

// d_stats [2g]: column sums, then sums of squares, over all n_total rows -> h_mean [g] and the total variances
int32_t gene_moments(PcaWork& w, const double* d_stats, double* h_mean) {
  const int g = w.g_real;
  std::vector<double> hs(2 * (size_t)g);
  SB2_CUDA(cudaMemcpyAsync(hs.data(), d_stats, sizeof(double) * 2 * g, cudaMemcpyDeviceToHost, w.st));
  SB2_CUDA(cudaStreamSynchronize(w.st));
  const double nt = (double)w.n_total;
  for (int j = 0; j < g; ++j) {
    const double mu = hs[j] / nt;
    h_mean[j] = mu;
    w.stats.total_var += (hs[g + j] - nt * mu * mu) / (nt - 1.0);  // per-gene variance, ddof=1 (_pca.py:727-729)
    w.total_var0 += hs[g + j] / nt - mu * mu;
  }
  return SB2_OK;
}
// In-core entries: the gene moments of the CSR rows, column statistics summed over the ranks
int32_t incore_moments(PcaWork& w, ScratchScope& scr, int64_t n, const int64_t* indptr, const int32_t* indices,
                       const float* data, double* h_mean) {
  const int g = w.g_real;
  double* d_stats;
  SB2_TRY(scr.alloc(&d_stats, (size_t)2 * g));
  SB2_TRY(sb2_csr_col_stats(w.ctx, n, g, indptr, indices, data, d_stats, d_stats + g));
  SB2_TRY(sb2_comm_allreduce_f64(w.ctx, d_stats, 2 * (int64_t)g));
  return gene_moments(w, d_stats, h_mean);
}

// Gram operator w.d_C = G - n_total mu mu^T [w.g x w.g], from G = X^T X [g x g] summed over all ranks, zero for padding genes.
// G is centred in place when it needs no padding and the caller hands it over (G_is_scratch); otherwise it is copied.
int32_t gram_operator(PcaWork& w, ScratchScope& scr, const double* G, bool G_is_scratch) {
  const int g = w.g_real, gp = w.g;
  if (gp == g && G_is_scratch) {
    w.d_C = const_cast<double*>(G);
  } else {
    SB2_TRY(scr.alloc(&w.d_C, (size_t)gp * gp));
    SB2_CUDA(cudaMemsetAsync(w.d_C, 0, sizeof(double) * (size_t)gp * gp, w.st));
    SB2_CUDA(cudaMemcpy2DAsync(w.d_C, sizeof(double) * gp, G, sizeof(double) * g, sizeof(double) * g, g,
                               cudaMemcpyDeviceToDevice, w.st));
  }
  if (gp != g) {
    double* mup;
    SB2_TRY(scr.alloc(&mup, (size_t)gp));
    SB2_CUDA(cudaMemsetAsync(mup, 0, sizeof(double) * gp, w.st));
    SB2_CUDA(cudaMemcpyAsync(mup, w.d_mu, sizeof(double) * g, cudaMemcpyDeviceToDevice, w.st));
    w.d_mu = mup;
  }
  center_gram_kernel<<<(unsigned)ceil_div64((int64_t)gp * gp, 256), 256, 0, w.st>>>(w.d_C, w.d_mu, (double)w.n_total, gp);
  SB2_LAUNCH_CHECK(w.ctx);
  return SB2_OK;
}
// In-core entries: the operator of w.solver over the CSR rows, once w.d_mu holds the mean (SpMM: buffers for X_c V, X^T Y)
int32_t incore_operator(PcaWork& w, ScratchScope& scr, int64_t n, const int64_t* indptr, const int32_t* indices,
                        const float* data) {
  const int g = w.g_real, l = w.l;
  if (w.solver == 1) {
    double* G;
    SB2_TRY(scr.alloc(&G, (size_t)g * g));
    SB2_TRY(sb2_csr_gram(w.ctx, n, g, indptr, indices, data, G));
    SB2_TRY(sb2_comm_allreduce_f64(w.ctx, G, (int64_t)g * g));
    return gram_operator(w, scr, G, true);
  }
  w.n = n; w.indptr = indptr; w.indices = indices; w.data = data;
  SB2_TRY(scr.alloc(&w.d_shift, (size_t)l));
  SB2_TRY(scr.alloc(&w.d_Y, (size_t)std::max<int64_t>(n, 1) * l));
  SB2_TRY(scr.alloc(&w.d_Zc, (size_t)ZT_COPIES * g * l));
  return SB2_OK;
}

// Block subspace iteration with Rayleigh-Ritz on the operator w applies, from a start block drawn from `seed` (the same on
// every rank).  Leaves the Ritz vectors in w.d_V (columns by descending Ritz value), the Ritz values in w.theta and the loop
// statistics in w.stats.
int32_t subspace_iteration(PcaWork& w, ScratchScope& scr, int k, int max_iter, double tol, uint64_t seed) {
  sb2_ctx* ctx = w.ctx;
  cudaStream_t st = w.st;
  const int g = w.g_real, gp = w.g, l = w.l;
  if (max_iter <= 0) max_iter = w.solver == 1 ? 4000 : 300;
  // goal: the residual the iteration aims for; tol: the residual that counts as converged.  With the default tolerance the
  // SpMM route (fp32 passes) aims 4x below it: an eigenvector's error is about its residual over its spectral gap, so
  // stopping at the first iterate under 2e-6 leaves the smaller kept components (relative gaps ~1e-2) near 1e-4, while
  // the fp32 rounding floor is lower still.  Iterates that stall at the floor above the goal count as converged once
  // they are under tol.
  double goal = tol;
  if (!(tol > 0.0)) {
    tol = w.solver == 1 ? 1e-10 : 2e-6;
    goal = w.solver == 1 ? tol : tol / 4.0;
  }
  const int64_t blk = (int64_t)gp * l;
  double *d_V = w.d_V, *d_Z = w.d_Z, *d_theta = w.d_theta, *d_res = w.d_res, *P[3];
  SB2_CUDA(cudaFuncSetAttribute(tsmm_tn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * 2 * 32 * l)));
  SB2_CUDA(cudaFuncSetAttribute(right_mult_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * l * l)));
  if (l <= 64) SB2_CUDA(cudaFuncSetAttribute(rr_jacobi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rr_jacobi_smem(l)));

  Rng rng(seed);
  w.rng = &rng;
  {
    std::vector<double> hv((size_t)blk, 0.0);
    for (int r = 0; r < g; ++r)
      for (int j = 0; j < l; ++j) hv[(size_t)r * l + j] = rng.normal();
    SB2_CUDA(cudaMemcpyAsync(d_V, hv.data(), sizeof(double) * (size_t)blk, cudaMemcpyHostToDevice, st));
    SB2_CUDA(cudaStreamSynchronize(st));
  }
  SB2_TRY(orthonormalize(w, d_V));
  for (double*& p : P) SB2_TRY(scr.alloc(&p, (size_t)blk));

  std::vector<double> hres(l);
  std::vector<double>& theta = w.theta;
  theta.resize(l);
  int32_t &it = w.stats.iterations, &converged = w.stats.converged;
  double& max_rel = w.stats.max_rel_residual;
  int stalled = 0;
  double prev_rel = 1e300;
  // Chebyshev-filtered subspace iteration (Zhou & Saad): between two Rayleigh-Ritz steps the block is
  // multiplied by a degree-m Chebyshev polynomial of A that is bounded on the unwanted interval
  // [0, theta_l] (A is PSD; theta_l = smallest Ritz value of the block) and grows fast above it.
  const int cheb_m = 10;
  const unsigned lgrid = (unsigned)ceil_div64(blk, 256);
  for (;;) {
    SB2_TRY(apply_operator(w, d_V, d_Z));
    ++it;
    SB2_TRY(rayleigh_ritz(w, d_V, d_Z, d_theta));
    SB2_CUDA(cudaMemsetAsync(d_res, 0, sizeof(double) * l, st));
    residual_kernel<<<32, (1024 / l) * l, 0, st>>>(d_Z, d_V, d_theta, gp, l, d_res);
    SB2_LAUNCH_CHECK(ctx);
    if (ctx->n_ranks > 1) {
      // one process per GPU: the loop-control scalars must be THE SAME on every rank (the fp64 REDs behind them are
      // order-dependent, and a rank that leaves the loop alone would strand the others in the next all-reduce):
      // rank 0's Ritz values and residuals are broadcast (zero-fill elsewhere + sum all-reduce)
      if (ctx->rank != 0) {
        SB2_CUDA(cudaMemsetAsync(d_theta, 0, sizeof(double) * l, st));
        SB2_CUDA(cudaMemsetAsync(d_res, 0, sizeof(double) * l, st));
      }
      SB2_TRY(sb2_comm_allreduce_f64(ctx, d_theta, l));
      SB2_TRY(sb2_comm_allreduce_f64(ctx, d_res, l));
    }
    // the Ritz values come back together with the residual norms (one sync)
    SB2_CUDA(cudaMemcpyAsync(hres.data(), d_res, sizeof(double) * l, cudaMemcpyDeviceToHost, st));
    SB2_CUDA(cudaMemcpyAsync(theta.data(), d_theta, sizeof(double) * l, cudaMemcpyDeviceToHost, st));
    SB2_CUDA(cudaStreamSynchronize(st));
    max_rel = 0.0;
    const double th1 = std::max(theta[0], 1e-300);
    for (int j = 0; j < k; ++j) max_rel = std::max(max_rel, sqrt(std::max(hres[j], 0.0)) / th1);
    converged = max_rel <= tol && theta[k - 1] > 0.0;
    if (max_rel <= goal && converged) break;
    if (it >= max_iter) break;
    // stagnation at the operator's rounding floor (fp32 SpMM passes): stop; converged iff under tol
    if (it > 3 && max_rel > 0.97 * prev_rel) { if (++stalled >= 3) break; } else stalled = 0;
    prev_rel = max_rel;
    const double cut = theta[l - 1], top = theta[0];
    // degree: the filter amplifies the top of the wanted spectrum by T_m(x0), x0 = (top - c)/e, relative to the
    // cut; beyond ~1e7 the columns next to the cut drown in rounding noise of the dominant directions, so m is
    // capped by acosh(1e7)/acosh(x0) (a wide spectrum gets a low degree, a flat one the full cheb_m)
    int m_use = 0;
    if (it >= 3 && cut > 0.0 && top > 1.0001 * cut) {
      const double x0 = 2.0 * top / cut - 1.0;
      m_use = std::min(cheb_m, (int)floor(acosh(1e7) / acosh(x0)));
    }
    if (m_use >= 2) {
      const double e = 0.5 * cut, c = 0.5 * cut;
      double sigma = e / (top - c);
      const double sigma1 = sigma;
      // Y1 = (sigma1/e) (A V - c V), reusing Z = A V from the Rayleigh-Ritz step
      double *prev = P[0], *cur = P[1], *nxt = P[2];
      SB2_CUDA(cudaMemcpyAsync(prev, d_V, sizeof(double) * (size_t)blk, cudaMemcpyDeviceToDevice, st));
      lincomb3_kernel<<<lgrid, 256, 0, st>>>(blk, sigma1 / e, d_Z, -(sigma1 / e) * c, d_V, 0.0, d_V, cur);
      SB2_LAUNCH_CHECK(ctx);
      for (int i = 2; i <= m_use && it < max_iter; ++i) {
        const double sigma2 = 1.0 / (2.0 / sigma1 - sigma);
        SB2_TRY(apply_operator(w, cur, d_Z));
        ++it;
        lincomb3_kernel<<<lgrid, 256, 0, st>>>(blk, 2.0 * sigma2 / e, d_Z, -(2.0 * sigma2 / e) * c, cur, -(sigma * sigma2), prev, nxt);
        SB2_LAUNCH_CHECK(ctx);
        double* t = prev; prev = cur; cur = nxt; nxt = t;
        sigma = sigma2;
      }
      SB2_CUDA(cudaMemcpyAsync(d_V, cur, sizeof(double) * (size_t)blk, cudaMemcpyDeviceToDevice, st));
    } else {
      SB2_CUDA(cudaMemcpyAsync(d_V, d_Z, sizeof(double) * (size_t)blk, cudaMemcpyDeviceToDevice, st));
    }
    SB2_TRY(orthonormalize(w, d_V));
  }
  return SB2_OK;
}

// Signs of svd_flip(u_based_decision=False) (sklearn/utils/extmath.py:974-981) on the Ritz vectors w.d_V (in place), the
// components d_components [k x g] (rows beyond g in the padded space are all-zero genes and are dropped), and the float32
// projection operator of X_pca = X U - 1 (mu^T U): U [g x l] in w.d_Bf, mu^T U [l] in a fresh w.d_shift.
int32_t projection_operator(PcaWork& w, ScratchScope& scr, int k, float* d_components) {
  const int g = w.g_real, l = w.l;
  double *d_V = w.d_V, *d_am;
  SB2_TRY(scr.alloc(&d_am, (size_t)l));
  col_absmax_kernel<<<l, 256, 0, w.st>>>(d_V, w.g, l, d_am);
  SB2_LAUNCH_CHECK(w.ctx);
  std::vector<double> am(l), hsign(l);
  SB2_CUDA(cudaMemcpyAsync(am.data(), d_am, sizeof(double) * l, cudaMemcpyDeviceToHost, w.st));
  SB2_CUDA(cudaStreamSynchronize(w.st));
  for (int j = 0; j < l; ++j) hsign[j] = am[j] < 0.0 ? -1.0 : 1.0;
  SB2_CUDA(cudaMemcpyAsync(d_am, hsign.data(), sizeof(double) * l, cudaMemcpyHostToDevice, w.st));
  // the first g rows of V (row-major, ld = l) are contiguous already
  components_out_kernel<<<(unsigned)ceil_div64((int64_t)k * g, 256), 256, 0, w.st>>>(d_V, d_am, g, l, k, d_components);
  SB2_LAUNCH_CHECK(w.ctx);
  std::vector<double> Dg((size_t)l * l, 0.0);
  for (int j = 0; j < l; ++j) Dg[(size_t)j * l + j] = hsign[j];
  SB2_TRY(right_mult_inplace(w, d_V, Dg));
  const int64_t len = (int64_t)g * l;
  f64_to_f32_kernel<<<(unsigned)ceil_div64(len, 256), 256, 0, w.st>>>(d_V, w.d_Bf, len);
  SB2_LAUNCH_CHECK(w.ctx);
  SB2_TRY(scr.alloc(&w.d_shift, (size_t)l));
  mu_dot_kernel<<<l, 256, 0, w.st>>>(w.d_mu, d_V, g, l, w.d_shift);
  SB2_LAUNCH_CHECK(w.ctx);
  return SB2_OK;
}

// PCA: explained_variance_ = S^2/(n-1) (_pca.py:760-779), the ratio against the ddof-1 total
void centred_variance(const PcaWork& w, int k, double* h_var, double* h_var_ratio) {
  for (int j = 0; j < k; ++j) {
    const double ev = std::max(w.theta[j], 0.0) / ((double)w.n_total - 1.0);
    h_var[j] = ev;
    h_var_ratio[j] = w.stats.total_var > 0.0 ? ev / w.stats.total_var : 0.0;
  }
}
// TruncatedSVD (sklearn/decomposition/_truncated_svd.py): explained_variance_ = np.var(X_transformed, axis=0) (ddof 0)
// = theta_j / n - (mean of column j)^2, the column mean of X V being mu . v_j; the ratio against sum_g var_g (ddof 0)
int32_t tsvd_variance(const PcaWork& w, int k, const double* h_mean, double* h_var, double* h_var_ratio) {
  const int g = w.g_real, l = w.l;
  std::vector<double> hV((size_t)w.g * l);
  SB2_CUDA(cudaMemcpyAsync(hV.data(), w.d_V, sizeof(double) * hV.size(), cudaMemcpyDeviceToHost, w.st));
  SB2_CUDA(cudaStreamSynchronize(w.st));
  for (int j = 0; j < k; ++j) {
    double m = 0.0;
    for (int r = 0; r < g; ++r) m += h_mean[r] * hV[(size_t)r * l + j];
    const double ev = std::max(w.theta[j], 0.0) / (double)w.n_total - m * m;
    h_var[j] = ev;
    h_var_ratio[j] = w.total_var0 > 0.0 ? ev / w.total_var0 : 0.0;
  }
  return SB2_OK;
}

// waits for the last stage and reports the statistics
int32_t report(const PcaWork& w, sb2_pca_info* info) {
  SB2_CUDA(cudaStreamSynchronize(w.st));
  if (info) *info = w.stats;
  return SB2_OK;
}

}  // namespace

extern "C" {

int32_t sb2_csr_col_stats(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                          const float* d_data, double* d_col_sum, double* d_col_sumsq) {
  SB2_CHECK_ARG(ctx && d_indptr && d_col_sum && d_col_sumsq, "null pointer");
  SB2_CHECK_ARG(n >= 0 && g >= 1, "shape");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  int64_t nnz = 0;
  if (n > 0) {
    SB2_CUDA(cudaMemcpyAsync(&nnz, d_indptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  double* acc;
  SB2_TRY(scr.alloc(&acc, (size_t)STAT_COPIES * 2 * g));
  SB2_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * STAT_COPIES * 2 * g, ctx->stream));
  if (nnz > 0) {
    const int grid = ctx->prop.multiProcessorCount * 8;
    csr_col_stats_kernel<<<grid, 256, 0, ctx->stream>>>(nnz, d_indices, d_data, g, acc);
    SB2_LAUNCH_CHECK(ctx);
  }
  double* both;
  SB2_TRY(scr.alloc(&both, (size_t)2 * g));
  reduce_copies_f64_kernel<<<(unsigned)ceil_div64(2 * g, 256), 256, 0, ctx->stream>>>(acc, STAT_COPIES, 2 * (int64_t)g, both);
  SB2_LAUNCH_CHECK(ctx);
  SB2_CUDA(cudaMemcpyAsync(d_col_sum, both, sizeof(double) * g, cudaMemcpyDeviceToDevice, ctx->stream));
  SB2_CUDA(cudaMemcpyAsync(d_col_sumsq, both + g, sizeof(double) * g, cudaMemcpyDeviceToDevice, ctx->stream));
  return SB2_OK;
}

int32_t sb2_spmm_csr(sb2_ctx* ctx, int64_t n, int32_t g, int32_t l, const int64_t* d_indptr, const int32_t* d_indices,
                     const float* d_data, const float* d_b, const float* d_shift, float* d_y) {
  SB2_CHECK_ARG(ctx && d_indptr && d_b && d_y, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  return launch_spmm(ctx, n, l, d_indptr, d_indices, d_data, d_b, d_shift, d_y, l, l);
}

int32_t sb2_spmm_csr_t(sb2_ctx* ctx, int64_t n, int32_t g, int32_t l, const int64_t* d_indptr,
                       const int32_t* d_indices, const float* d_data, const float* d_y, double* d_z) {
  SB2_CHECK_ARG(ctx && d_indptr && d_y && d_z, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  float* Zc;
  SB2_TRY(scr.alloc(&Zc, (size_t)ZT_COPIES * g * l));
  return launch_spmm_t(ctx, n, g, l, d_indptr, d_indices, d_data, d_y, Zc, d_z);
}

int32_t sb2_csr_gram(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                     const float* d_data, double* d_gram) {
  SB2_CHECK_ARG(ctx && d_indptr && d_gram, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  SB2_CUDA(cudaMemsetAsync(d_gram, 0, sizeof(double) * (size_t)g * g, ctx->stream));
  bool done = false;
  const int NB = (int)ceil_div64(g, GT_W);
  // The tiled kernel is opt-in (SB2_GRAM_TILED=1); the default issues one global fp64 RED per product, which the L2
  // retires, while the tiled kernel's shared-memory fp64 atomicAdd is a CAS loop (ATOMS.CAST.SPIN.64) behind a chain of
  // dependent global loads (block offsets -> indices/data).  Both give the same result up to the fp64 summation order.
  static const bool use_tiled = getenv("SB2_GRAM_TILED") != nullptr;
  if (n >= 2048 && g >= 64 && NB <= 63 && use_tiled) {
    // tiled kernel: needs column-sorted rows (checked while the block-offset table is built)
    ScratchScope scr(ctx);
    uint16_t* boff;
    int* flag;
    int2* pair_tab;
    SB2_TRY(scr.alloc(&boff, (size_t)n * (NB + 1)));
    SB2_TRY(scr.alloc(&flag, 4));
    const int n_pairs = NB * (NB + 1) / 2;
    SB2_TRY(scr.alloc(&pair_tab, (size_t)n_pairs));
    std::vector<int2> hp;
    hp.reserve(n_pairs);
    for (int bi = 0; bi < NB; ++bi)
      for (int bj = bi; bj < NB; ++bj) hp.push_back(make_int2(bi, bj));
    SB2_CUDA(cudaMemcpyAsync(pair_tab, hp.data(), sizeof(int2) * n_pairs, cudaMemcpyHostToDevice, ctx->stream));
    SB2_CUDA(cudaMemsetAsync(flag, 0, 16, ctx->stream));
    gram_block_offsets_kernel<<<(unsigned)ceil_div64(n, 8), 256, 0, ctx->stream>>>(n, d_indptr, d_indices, NB, boff, flag);
    SB2_LAUNCH_CHECK(ctx);
    int hflag = 0;
    SB2_CUDA(cudaMemcpyAsync(&hflag, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    SB2_CUDA(cudaStreamSynchronize(ctx->stream));  // also keeps hp alive until the copy has run
    if (hflag == 0) {
      // row ranges: enough CTAs for ~8 waves, a whole number of waves where possible, ranges of >= 1024 rows
      const int sms = ctx->prop.multiProcessorCount;
      int64_t best_s = 1;
      double best_fill = 0.0;
      const int64_t s_max = std::max<int64_t>(1, n / 1024);
      const int64_t s0 = std::max<int64_t>(1, std::min<int64_t>(s_max, (int64_t)8 * sms / n_pairs));
      for (int64_t sr = s0; sr <= std::min<int64_t>(s_max, s0 + 16); ++sr) {
        const double ctas = (double)n_pairs * (double)sr;
        const double fill = ctas / (ceil(ctas / sms) * sms);
        if (fill > best_fill + 1e-9) { best_fill = fill; best_s = sr; }
      }
      const int64_t rows_per_range = ceil_div64(n, best_s);
      const int64_t n_ranges = ceil_div64(n, rows_per_range);
      const size_t smem = sizeof(double) * GT_W * GT_W;
      SB2_CUDA(cudaFuncSetAttribute(csr_gram_tiles_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      csr_gram_tiles_kernel<<<(unsigned)(n_pairs * n_ranges), GT_THREADS, smem, ctx->stream>>>(
          n, d_indptr, d_indices, d_data, boff, NB, n_pairs, pair_tab, rows_per_range, d_gram, g);
      SB2_LAUNCH_CHECK(ctx);
      done = true;
    }
  }
  if (n > 0 && !done) {
    csr_gram_kernel<<<(unsigned)ceil_div64(n, 8), 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_data, d_gram, g);
    SB2_LAUNCH_CHECK(ctx);
  }
  mirror_upper_kernel<<<(unsigned)ceil_div64((int64_t)g * g, 256), 256, 0, ctx->stream>>>(d_gram, g);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_pca_csr_f32(sb2_ctx* ctx, int64_t n, int64_t n_total, int32_t g, const int64_t* d_indptr,
                        const int32_t* d_indices, const float* d_data, int32_t k, int32_t solver, int32_t max_iter,
                        double tol, uint64_t seed, float* d_x_pca, float* d_components, double* h_var,
                        double* h_var_ratio, double* h_mean, sb2_pca_info* info) {
  SB2_CHECK_ARG(ctx && d_indptr && d_x_pca && d_components && h_var && h_var_ratio && h_mean, "null pointer");
  PcaWork w{};
  SB2_TRY(init_work(ctx, n, n_total, g, k, solver, w));
  ScratchScope scr(ctx);
  SB2_TRY(incore_moments(w, scr, n, d_indptr, d_indices, d_data, h_mean));
  SB2_TRY(alloc_scratch(w, scr));
  SB2_CUDA(cudaMemcpyAsync(w.d_mu, h_mean, sizeof(double) * g, cudaMemcpyHostToDevice, w.st));
  SB2_TRY(incore_operator(w, scr, n, d_indptr, d_indices, d_data));
  SB2_TRY(subspace_iteration(w, scr, k, max_iter, tol, seed));
  SB2_TRY(projection_operator(w, scr, k, d_components));
  SB2_TRY(launch_spmm(ctx, n, w.l, d_indptr, d_indices, d_data, w.d_Bf, w.d_shift, d_x_pca, k, k));
  centred_variance(w, k, h_var, h_var_ratio);
  return report(w, info);
}

// sc.pp.pca(zero_center=False): sklearn TruncatedSVD (src/scanpy/preprocessing/_pca/__init__.py:309-336) - top-k singular
// triplets of X itself; d_x_pca = X V = U Sigma, components sign-fixed like svd_flip(u_based_decision=False)
int32_t sb2_tsvd_csr_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                         const float* d_data, int32_t k, int32_t solver, int32_t max_iter, double tol, uint64_t seed,
                         float* d_x_pca, float* d_components, double* h_var, double* h_var_ratio, sb2_pca_info* info) {
  SB2_CHECK_ARG(ctx && ctx->n_ranks == 1, "sb2_tsvd_csr_f32 is single-rank");
  SB2_CHECK_ARG(d_indptr && d_x_pca && d_components && h_var && h_var_ratio, "null pointer");
  PcaWork w{};
  SB2_TRY(init_work(ctx, n, n, g, k, solver, w));
  ScratchScope scr(ctx);
  std::vector<double> h_mean((size_t)g);
  SB2_TRY(incore_moments(w, scr, n, d_indptr, d_indices, d_data, h_mean.data()));
  SB2_TRY(alloc_scratch(w, scr));
  // the operator is X^T X itself: with an all-zero device mean neither the Gram centring nor the SpMM shift does anything;
  // the true column means stay on the host for the variance formula
  SB2_CUDA(cudaMemsetAsync(w.d_mu, 0, sizeof(double) * g, w.st));
  SB2_TRY(incore_operator(w, scr, n, d_indptr, d_indices, d_data));
  SB2_TRY(subspace_iteration(w, scr, k, max_iter, tol, seed));
  SB2_TRY(projection_operator(w, scr, k, d_components));
  SB2_TRY(launch_spmm(ctx, n, w.l, d_indptr, d_indices, d_data, w.d_Bf, w.d_shift, d_x_pca, k, k));
  SB2_TRY(tsvd_variance(w, k, h_mean.data(), h_var, h_var_ratio));
  return report(w, info);
}

// ---- out-of-core / chunked PCA (sc.pp.pca(chunked=True), src/scanpy/preprocessing/_pca/__init__.py:245-271) ----
// The reference streams row chunks through sklearn's IncrementalPCA and its own test asks the result to equal the full PCA
// (tests/test_pca.py:357-386, rtol 1e-6).  Here the row chunks stream through the EXACT Gram route instead: pass 1
// accumulates column sums and X^T X chunk by chunk (this call), sb2_pca_stream_solve_f32 diagonalises the covariance,
// pass 2 projects each chunk (sb2_pca_stream_project_f32).  Device memory: one chunk + 2 g^2 doubles, whatever n is.
static __global__ void add_f64_kernel(int64_t n, const double* __restrict__ a, double* __restrict__ acc) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) acc[i] += a[i];
}
int32_t sb2_pca_stream_accumulate_f32(sb2_ctx* ctx, int64_t n_chunk, int32_t g, const int64_t* d_indptr,
                                      const int32_t* d_indices, const float* d_data, double* d_stats, double* d_gram) {
  SB2_CHECK_ARG(ctx && d_indptr && d_stats && d_gram && g >= 1 && n_chunk >= 0, "null pointer / shape");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n_chunk == 0) return SB2_OK;
  ScratchScope scr(ctx);
  double *st2, *G;
  SB2_TRY(scr.alloc(&st2, (size_t)2 * g));
  SB2_TRY(scr.alloc(&G, (size_t)g * g));
  SB2_TRY(sb2_csr_col_stats(ctx, n_chunk, g, d_indptr, d_indices, d_data, st2, st2 + g));
  SB2_TRY(sb2_csr_gram(ctx, n_chunk, g, d_indptr, d_indices, d_data, G));
  add_f64_kernel<<<(unsigned)ceil_div64(2 * (int64_t)g, 256), 256, 0, ctx->stream>>>(2 * (int64_t)g, st2, d_stats);
  SB2_LAUNCH_CHECK(ctx);
  add_f64_kernel<<<(unsigned)ceil_div64((int64_t)g * g, 256), 256, 0, ctx->stream>>>((int64_t)g * g, G, d_gram);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}
int32_t sb2_pca_stream_solve_f32(sb2_ctx* ctx, int64_t n_total, int32_t g, const double* d_stats, const double* d_gram,
                                 int32_t k, int32_t max_iter, double tol, uint64_t seed, float* d_components, double* h_var,
                                 double* h_var_ratio, double* h_mean, float* d_proj, float* d_shift, int32_t* h_l,
                                 sb2_pca_info* info) {
  SB2_CHECK_ARG(ctx && d_stats && d_gram && d_components && h_var && h_var_ratio && h_mean && d_proj && d_shift && h_l,
                "null pointer");
  PcaWork w{};
  SB2_TRY(init_work(ctx, 0, n_total, g, k, 1, w));
  ScratchScope scr(ctx);
  SB2_TRY(gene_moments(w, d_stats, h_mean));
  SB2_TRY(alloc_scratch(w, scr));
  SB2_CUDA(cudaMemcpyAsync(w.d_mu, h_mean, sizeof(double) * g, cudaMemcpyHostToDevice, w.st));
  SB2_TRY(gram_operator(w, scr, d_gram, false));
  SB2_TRY(subspace_iteration(w, scr, k, max_iter, tol, seed));
  SB2_TRY(projection_operator(w, scr, k, d_components));
  SB2_CUDA(cudaMemcpyAsync(d_proj, w.d_Bf, sizeof(float) * (size_t)g * w.l, cudaMemcpyDeviceToDevice, w.st));
  SB2_CUDA(cudaMemcpyAsync(d_shift, w.d_shift, sizeof(float) * w.l, cudaMemcpyDeviceToDevice, w.st));
  *h_l = w.l;
  centred_variance(w, k, h_var, h_var_ratio);
  return report(w, info);
}
int32_t sb2_pca_stream_project_f32(sb2_ctx* ctx, int64_t n_chunk, int32_t g, const int64_t* d_indptr,
                                   const int32_t* d_indices, const float* d_data, int32_t k, int32_t l, const float* d_proj,
                                   const float* d_shift, float* d_x_pca) {
  SB2_CHECK_ARG(ctx && d_indptr && d_proj && d_shift && d_x_pca, "null pointer");
  SB2_CHECK_ARG(k >= 1 && k <= l && (l == 32 || l == 64 || l == 128), "k / l");
  SB2_CUDA(cudaSetDevice(ctx->device));
  return launch_spmm(ctx, n_chunk, l, d_indptr, d_indices, d_data, d_proj, d_shift, d_x_pca, k, k);
}

}  // extern "C"

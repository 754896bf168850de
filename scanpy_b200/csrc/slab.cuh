// slab.cuh — the column-slab scheme of the dense per-gene passes (regress.cu, pearson.cu, combat.cu, autocorr.cu,
// aggregate.cu).
//
// One CTA owns a SLAB_THREADS-column slab of a block of rows and each thread one column.  A CSR input is read in place:
// the CTA binary-searches its slab in each of SLAB_ROWS rows (column indices sorted, no duplicates) and scatters the
// slab's stored values into a zeroed shared-memory tile, so implicit zeros are evaluated like stored values.
//
// The passes whose sums must not depend on how the caller splits the rows into blocks work on fixed SLAB_TILE-row
// subtiles and merge them in subtile order; the Pearson residual variance and combat's moments share the merge.
#pragma once
#include <stdint.h>

#include <type_traits>

namespace {

constexpr int SLAB_THREADS = 256;  // one column per thread: 256-column slabs
constexpr int SLAB_ROWS = 16;      // rows staged per step
constexpr int SLAB_TILE = 1024;    // rows per subtile
static_assert(SLAB_TILE == SB2_REGRESS_TILE_ROWS && SLAB_TILE == SB2_PEARSON_TILE_ROWS &&
              SLAB_TILE == SB2_COMBAT_TILE_ROWS && SLAB_TILE == SB2_AUTOCORR_TILE_ROWS &&
              SLAB_TILE == SB2_AGGREGATE_TILE_ROWS && SLAB_TILE % SLAB_ROWS == 0,
              "subtile");

// The slab [c0, c1) of the m rows rid[0..m) of a CSR, scattered into tile[r][col - c0]; tile must be zero on entry.
// Thread r < m has written rid[r] before the call; the caller clears what it reads.
template <typename T>
__device__ __forceinline__ void stage_csr(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                          const T* __restrict__ data, const int64_t* rid, int m, int c0, int c1,
                                          T (*tile)[SLAB_THREADS], int64_t* lo, int64_t* hi) {
  if ((int)threadIdx.x < m) {
    const int64_t r = rid[threadIdx.x];
    const int64_t e1 = indptr[r + 1];
    int64_t a = indptr[r], b = e1;
    while (a < b) {
      const int64_t mid = (a + b) >> 1;
      if (indices[mid] < c0) a = mid + 1; else b = mid;
    }
    lo[threadIdx.x] = a;
    b = e1;
    while (a < b) {
      const int64_t mid = (a + b) >> 1;
      if (indices[mid] < c1) a = mid + 1; else b = mid;
    }
    hi[threadIdx.x] = a;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < m; r += SLAB_THREADS / 32)
    for (int64_t e = lo[r] + lane; e < hi[r]; e += 32) tile[r][indices[e] - c0] = data[e];
  __syncthreads();
}

// acc[i] += part[0][i] + ... in subtile order; the per-gene min / max / NaN likewise (g = 0: sums only, and pmin, pmax,
// pnan, cmin, cmax, cnan may be NULL).  A template only so that the units that do not launch it do not compile it.
template <int = 0>
__global__ void fold_kernel(int64_t nsub, int64_t width, int g, const double* __restrict__ part,
                            const double* __restrict__ pmin, const double* __restrict__ pmax,
                            const int32_t* __restrict__ pnan, double* __restrict__ acc, double* __restrict__ cmin,
                            double* __restrict__ cmax, int32_t* __restrict__ cnan) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < width) {
    double s = acc[i];
    for (int64_t t = 0; t < nsub; ++t) s += part[t * width + i];
    acc[i] = s;
  }
  if (i < g) {
    double a = cmin[i], b = cmax[i];
    int32_t f = cnan[i];
    for (int64_t t = 0; t < nsub; ++t) {
      a = fmin(a, pmin[t * g + i]);
      b = fmax(b, pmax[t * g + i]);
      f |= pnan[t * g + i];
    }
    cmin[i] = a;
    cmax[i] = b;
    cnan[i] = f;
  }
}

// acc[k][j] (k = 0 count, 1 mean, 2 M2, and with SUM_SQ 3 Σx²) merged with the SLAB_TILE-row subtiles' partials
// part[t][k][j] (k = 0 mean, 1 M2, and with SUM_SQ 2 Σx²) in subtile order (Chan et al.)
template <bool SUM_SQ>
__global__ void moments_fold_kernel(int64_t nsub, int64_t rows, int g, const double* __restrict__ part,
                                    double* __restrict__ acc) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g) return;
  double n = acc[j], mean = acc[g + j], m2 = acc[2 * (int64_t)g + j], sq = SUM_SQ ? acc[3 * (int64_t)g + j] : 0.0;
  for (int64_t t = 0; t < nsub; ++t) {
    const double* p = part + t * (SUM_SQ ? 3 : 2) * (int64_t)g;
    const double nb = (double)min((int64_t)SLAB_TILE, rows - t * SLAB_TILE);
    const double mb = p[j], m2b = p[g + j];
    if (n == 0.0) {
      mean = mb;
      m2 = m2b;
    } else {
      const double nn = n + nb, d = mb - mean;
      mean += d * (nb / nn);
      m2 += m2b + d * d * (n * nb / nn);
    }
    n += nb;
    if (SUM_SQ) sq += p[2 * (int64_t)g + j];
  }
  acc[j] = n;
  acc[g + j] = mean;
  acc[2 * (int64_t)g + j] = m2;
  if (SUM_SQ) acc[3 * (int64_t)g + j] = sq;
}

// f(T(), O(), CSR): T the value type of X (double when is_f64), O the output type (double when out_f64; a float64 X
// comes with a float64 output) and CSR a std::bool_constant, true when X comes as CSR arrays (x NULL)
template <typename F>
void with_types(bool is_f64, bool out_f64, const void* x, F&& f) {
  const auto layout = [&](auto t, auto o) {
    if (x) f(t, o, std::false_type());
    else f(t, o, std::true_type());
  };
  if (is_f64) layout(double(), double());
  else if (out_f64) layout(float(), double());
  else layout(float(), float());
}

// f(T(), CSR) for a pass that writes no values of X's type
template <typename F>
void with_types(bool is_f64, const void* x, F&& f) {
  with_types(is_f64, is_f64, x, [&](auto t, auto, auto csr) { f(t, csr); });
}

// f(KMAX) as a std::integral_constant: room for 32 coefficients when wide, 4 otherwise
template <typename F>
void with_kmax(bool wide, F&& f) {
  if (wide) f(std::integral_constant<int, 32>());
  else f(std::integral_constant<int, 4>());
}

}  // namespace

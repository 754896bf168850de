// slab.cuh — the column-slab scheme of the dense per-gene passes (regress.cu, pearson.cu, combat.cu).
//
// One CTA owns a SLAB_THREADS-column slab of a block of rows and each thread one column.  A CSR input is read in place:
// the CTA binary-searches its slab in each of SLAB_ROWS rows (column indices sorted, no duplicates) and scatters the
// slab's stored values into a zeroed shared-memory tile, so implicit zeros are evaluated like stored values.
#pragma once
#include <stdint.h>

namespace {

constexpr int SLAB_THREADS = 256;  // one column per thread: 256-column slabs
constexpr int SLAB_ROWS = 16;      // rows staged per step

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

}  // namespace

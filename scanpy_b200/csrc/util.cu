// util.cu — small utilities shared across files: the device prefix sum of the graph kernels and the host cyclic
// Jacobi eigensolver of PCA's Rayleigh-Ritz step and eigsh's restart problem.
#include <math.h>

#include "common.cuh"

namespace {
constexpr int SCAN_BLOCK = 1024;

__global__ void __launch_bounds__(SCAN_BLOCK)
scan_block_kernel(const int32_t* __restrict__ in, int64_t n, int64_t* __restrict__ out, int64_t* __restrict__ block_sums) {
  __shared__ int64_t warp_sums[32];
  const int64_t i = (int64_t)blockIdx.x * SCAN_BLOCK + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t v = i < n ? (int64_t)in[i] : 0;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int64_t s = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_sums[lane] = s;
  }
  __syncthreads();
  const int64_t incl = x + (warp > 0 ? warp_sums[warp - 1] : 0);
  if (i < n) out[i] = incl - v;  // exclusive within block
  if (threadIdx.x == SCAN_BLOCK - 1) block_sums[blockIdx.x] = incl;
}
__global__ void __launch_bounds__(1024)
scan_sums_kernel(int64_t* __restrict__ block_sums, int64_t nb, int64_t* __restrict__ total) {
  // single block: sequential chunks of 1024 with a running carry
  __shared__ int64_t warp_sums[32];
  __shared__ int64_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t base = 0; base < nb; base += 1024) {
    const int64_t i = base + threadIdx.x;
    const int64_t v = i < nb ? block_sums[i] : 0;
    int64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int64_t s = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
      }
      warp_sums[lane] = s;
    }
    __syncthreads();
    const int64_t incl = x + (warp > 0 ? warp_sums[warp - 1] : 0) + carry;
    if (i < nb) block_sums[i] = incl - v;  // exclusive offset of block i
    __syncthreads();
    if (threadIdx.x == 1023) carry = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}
__global__ void scan_add_kernel(int64_t* __restrict__ out, int64_t n, const int64_t* __restrict__ block_sums,
                                const int64_t* __restrict__ total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] += block_sums[i / SCAN_BLOCK];
  if (i == n) out[n] = *total;
}
}  // namespace

int32_t sb2_scan_i32_to_i64(sb2_ctx* ctx, const int32_t* d_in, int64_t n, int64_t* d_out) {
  ScratchScope scr(ctx);
  const int64_t nb = ceil_div64(n > 0 ? n : 1, SCAN_BLOCK);
  int64_t* sums;
  SB2_TRY(scr.alloc(&sums, (size_t)nb + 1));
  scan_block_kernel<<<(unsigned)nb, SCAN_BLOCK, 0, ctx->stream>>>(d_in, n, d_out, sums);
  SB2_LAUNCH_CHECK(ctx);
  scan_sums_kernel<<<1, 1024, 0, ctx->stream>>>(sums, nb, sums + nb);
  SB2_LAUNCH_CHECK(ctx);
  scan_add_kernel<<<(unsigned)ceil_div64(n + 1, 256), 256, 0, ctx->stream>>>(d_out, n, sums, sums + nb);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

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
        if (fabs(apq) < 1e-300) continue;
        const double app = A[(size_t)p * m + p], aqq = A[(size_t)q * m + q];
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

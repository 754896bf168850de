// autocorr.cu — the per-gene graph sums of
//   sc.metrics.morans_i  (src/scanpy/metrics/_morans_i.py: _morans_i_vec_w)
//   sc.metrics.gearys_c  (src/scanpy/metrics/_gearys_c.py: _gearys_c_vec_w)
//
// For gene c with mean m (from sb2_regress_col_sums) and z = x - m, over the stored arcs i -> j with fp64 weights w:
//   A = Σ_i z_i Σ_j w_ij z_j,   B = Σ_i Σ_j w_ij (x_i - x_j)²,   Q = Σ_i z_i².
// One CTA owns a 256-gene slab of a fixed SLAB_TILE-row subtile of the graph's rows and each thread one gene.  It walks
// the subtile's rows in order; for row i it takes the cells [i, j_0, j_1, ...] (its own value, then its arcs' targets)
// SLAB_ROWS at a time: a CSR X is staged by `stage_csr` with the graph's column indices as the rows, so implicit zeros are
// evaluated like stored values; a dense X is read in place, 256 consecutive genes of a target row per arc.  Everything is
// fp64 on the centred and differenced values: the expanded forms (Σx_i x_j - m Σ...) cancel catastrophically for genes
// whose mean is large against their spread.  Each subtile writes a [3 x g] partial, folded into the accumulators in
// subtile order (slab.cuh: fold_kernel), so the sums do not depend on the launch shape or on how the caller splits the
// graph's rows into blocks of whole subtiles.
//
// The arcs reach arbitrary cells, so every cell's values must be on the device.  The pass is bound by gathering each arc's
// target values, one row walk at a time: on an H100 at 1.3M x 2000 a dense X (no slab searches) takes 0.97 of the time
// of a CSR X (README.md).
#include "common.cuh"
#include "slab.cuh"

namespace {

// grid (subtiles, slabs): part[sub][k][j], k = 0 A, 1 B, 2 Q
template <typename T, bool CSR>
__global__ void __launch_bounds__(SLAB_THREADS)
autocorr_kernel(int64_t row0, int64_t rows, int g, const T* __restrict__ x, const int64_t* __restrict__ xindptr,
                const int32_t* __restrict__ xindices, const T* __restrict__ xdata, const int64_t* __restrict__ gindptr,
                const int32_t* __restrict__ gindices, const double* __restrict__ gw, const double* __restrict__ mean,
                double* __restrict__ part) {
  __shared__ T tile[CSR ? SLAB_ROWS : 1][SLAB_THREADS];
  __shared__ int64_t rid[SLAB_ROWS], lo[SLAB_ROWS], hi[SLAB_ROWS];
  const int64_t sub = blockIdx.x;
  const int c0 = blockIdx.y * SLAB_THREADS, c = c0 + threadIdx.x;
  const int c1 = min(g, c0 + SLAB_THREADS);
  const int cc = min(c, g - 1);  // the threads past the last gene shadow it, without a divergent branch in the walk
  const int64_t s0 = sub * SLAB_TILE, s1 = min(rows, s0 + SLAB_TILE);
  const double m = mean[cc];
  // the gene's running A, B, Q live in its own shared column: in registers ptxas spills them around the staging loop
  __shared__ double sums[3][SLAB_THREADS];
  sums[0][threadIdx.x] = sums[1][threadIdx.x] = sums[2][threadIdx.x] = 0.0;
  if (CSR)
    for (int r = 0; r < SLAB_ROWS; ++r) tile[r][threadIdx.x] = T(0);
  for (int64_t i = s0; i < s1; ++i) {
    const int64_t cell = row0 + i, e0 = gindptr[i], e1 = gindptr[i + 1];
    double xi = 0.0, zi = 0.0, ai = 0.0, bi = 0.0;
    // position e0 - 1 stands for the cell itself, e >= e0 for arc e
    for (int64_t p = e0 - 1; p < e1; p += SLAB_ROWS) {
      const int k = (int)min((int64_t)SLAB_ROWS, e1 - p);
      if (CSR) {
        if ((int)threadIdx.x < k) {
          const int64_t e = p + threadIdx.x;
          rid[threadIdx.x] = e < e0 ? cell : (int64_t)gindices[e];
        }
        stage_csr(xindptr, xindices, xdata, rid, k, c0, c1, tile, lo, hi);
      }
      int r = 0;
      if (p < e0) {
        if (CSR) {
          xi = (double)tile[0][threadIdx.x];
          tile[0][threadIdx.x] = T(0);
        } else {
          xi = (double)x[cell * g + cc];
        }
        zi = xi - m;
        r = 1;
      }
      for (; r < k; ++r) {
        const int64_t e = p + r;
        double v;
        if (CSR) {
          v = (double)tile[r][threadIdx.x];
          tile[r][threadIdx.x] = T(0);
        } else {
          v = (double)x[(int64_t)gindices[e] * g + cc];
        }
        const double w = gw[e], d = xi - v;
        ai += w * (v - m);
        bi += w * (d * d);
      }
      if (CSR) __syncthreads();
    }
    sums[0][threadIdx.x] += ai * zi;
    sums[1][threadIdx.x] += bi;
    sums[2][threadIdx.x] += zi * zi;
  }
  if (c >= g) return;
  double* out = part + sub * 3 * (int64_t)g;
  out[c] = sums[0][threadIdx.x];
  out[g + c] = sums[1][threadIdx.x];
  out[2 * (int64_t)g + c] = sums[2][threadIdx.x];
}

}  // namespace

extern "C" {

int32_t sb2_autocorr_sums(sb2_ctx* ctx, int64_t row0, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                          const int64_t* d_xindptr, const int32_t* d_xindices, const void* d_xdata,
                          const int64_t* d_gindptr, const int32_t* d_gindices, const double* d_gweights,
                          const double* d_mean, double* d_acc) {
  SB2_CHECK_ARG(ctx && d_gindptr && d_gindices && d_gweights && d_mean && d_acc, "null pointer");
  SB2_CHECK_ARG(g >= 1 && rows >= 0 && row0 >= 0, "shape");
  SB2_CHECK_ARG(d_x || (d_xindptr && d_xindices && d_xdata), "X: dense or CSR arrays");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  const int64_t nsub = ceil_div64(rows, SLAB_TILE), slabs = ceil_div64(g, SLAB_THREADS);
  SB2_CHECK_ARG(nsub < INT32_MAX && slabs <= 65535, "shape");
  const int64_t width = 3 * (int64_t)g;
  ScratchScope scr(ctx);
  double* part;
  SB2_TRY(scr.alloc(&part, (size_t)(nsub * width)));
  const dim3 grid((unsigned)nsub, (unsigned)slabs);
  with_types(is_f64, d_x, [&](auto t, auto csr) {
    using T = decltype(t);
    autocorr_kernel<T, decltype(csr)::value><<<grid, SLAB_THREADS, 0, ctx->stream>>>(
        row0, rows, g, static_cast<const T*>(d_x), d_xindptr, d_xindices, static_cast<const T*>(d_xdata), d_gindptr,
        d_gindices, d_gweights, d_mean, part);
  });
  SB2_LAUNCH_CHECK(ctx);
  fold_kernel<><<<(unsigned)ceil_div64(width, 256), 256, 0, ctx->stream>>>(nsub, width, 0, part, nullptr, nullptr,
                                                                           nullptr, d_acc, nullptr, nullptr, nullptr);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

// harmony.cu — the per-cell passes of
//   sc.pp.harmony_integrate  (src/scanpy/preprocessing/_harmony/core.py)
// and of the sklearn KMeans that starts it.  The host (scanpy_b200/_harmony.py) keeps everything sized clusters x
// codes: the penalty schedule, lambda, the ridge solves and the convergence tests.
//
// Storage follows the call's dtype (T = float or double); every sum over cells is fp64 and has no floating-point
// atomics: each CTA writes a partial and fold_kernel adds the partials in CTA order.  The CTA split depends only on the
// shapes, so two runs on equal inputs give equal bits.
#include <math.h>

#include <type_traits>
#include <vector>

#include "common.cuh"

namespace {

constexpr int HM_THREADS = 256;
constexpr int HM_WARPS = HM_THREADS / 32;
constexpr int HM_MAXK = SB2_HARMONY_MAX_K;
constexpr int HM_MAXD = SB2_HARMONY_MAX_D;
constexpr int HM_KPL = HM_MAXK / 32;  // clusters per lane
constexpr int HM_DPL = HM_MAXD / 32;  // columns per lane
constexpr int WS_TILE = 32;           // rows staged per step of wsums
constexpr int WS_NACC = 8;            // outputs per thread of wsums
constexpr int64_t CHUNK_ROWS = 2048;  // rows per CTA of the grouped passes
constexpr int SUM_PARTS = 528;        // CTAs of the plain sums (4 per SM)

template <typename T>
__device__ __forceinline__ T warp_max(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// out[g * width + i] = Σ part[p * width + i] over p in [cb[g], cb[g + 1]) (cb NULL: one group of all `parts`)
__global__ void fold_kernel(int groups, const int64_t* __restrict__ cb, int64_t parts, int64_t width,
                            const double* __restrict__ part, double* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= groups * width) return;
  const int64_t g = e / width, i = e - g * width;
  const int64_t p0 = cb ? cb[g] : 0, p1 = cb ? cb[g + 1] : parts;
  double s = 0.0;
  for (int64_t p = p0; p < p1; ++p) s += part[p * width + i];
  out[e] = s;
}

int32_t fold(sb2_ctx* ctx, int groups, const int64_t* cb, int64_t parts, int64_t width, const double* part,
             double* out) {
  const int64_t total = groups * width;
  fold_kernel<<<(unsigned)ceil_div64(total, 256), 256, 0, ctx->stream>>>(groups, cb, parts, width, part, out);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

// CTA ranges of at most CHUNK_ROWS positions that do not cross a group bound: chunks [lo, hi, group] and, per group,
// its first chunk (cb[groups] = number of chunks)
void make_chunks(int groups, const int64_t* bounds, std::vector<int64_t>& chunks, std::vector<int64_t>& cb) {
  cb.assign(groups + 1, 0);
  for (int g = 0; g < groups; ++g) {
    cb[g] = (int64_t)chunks.size() / 3;
    for (int64_t a = bounds[g]; a < bounds[g + 1]; a += CHUNK_ROWS) {
      chunks.push_back(a);
      chunks.push_back(std::min(bounds[g + 1], a + CHUNK_ROWS));
      chunks.push_back(g);
    }
  }
  cb[groups] = (int64_t)chunks.size() / 3;
}

template <typename T>
int32_t upload(sb2_ctx* ctx, ScratchScope& scr, const std::vector<T>& h, T** d) {
  SB2_TRY(scr.alloc(d, h.size()));
  if (!h.empty()) SB2_CUDA(cudaMemcpyAsync(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  return SB2_OK;
}

template <typename F>
void with_t(bool is_f64, F&& f) {
  if (is_f64) f(double());
  else f(float());
}

// ---------------------------------------------------------------------------------------------------- row norms
template <typename T>
__global__ void __launch_bounds__(HM_THREADS) normalize_kernel(int64_t n, int d, const T* __restrict__ x,
                                                                T* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * HM_WARPS + (threadIdx.x >> 5);
  if (i >= n) return;
  T v[HM_DPL];
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < HM_DPL; ++q) {
    const int j = lane + 32 * q;
    v[q] = j < d ? x[i * d + j] : T(0);
    s += (double)v[q] * (double)v[q];
  }
  s = warp_sum(s);
  const double nrm = fmax(sqrt(s), 1e-12);
#pragma unroll
  for (int q = 0; q < HM_DPL; ++q) {
    const int j = lane + 32 * q;
    if (j < d) out[i * d + j] = (T)((double)v[q] / nrm);
  }
}

// ---------------------------------------------------------------------------------------------------- weighted sums
// grid (chunks, output slices of HM_THREADS * WS_NACC); part[chunk][c * (d + 1) + j]
template <typename ZT, int MODE>
__global__ void __launch_bounds__(HM_THREADS) wsums_kernel(const int64_t* __restrict__ chunks,
                                                            const int64_t* __restrict__ idx, int d, int k,
                                                            const ZT* __restrict__ z, const ZT* __restrict__ r,
                                                            const int32_t* __restrict__ labels,
                                                            double* __restrict__ part) {
  extern __shared__ double ws_sm[];
  double* zt = ws_sm;                   // [WS_TILE][d + 1], column d = 1
  double* rt = ws_sm + WS_TILE * (d + 1);  // [WS_TILE][k] (MODE 0)
  __shared__ int lt[WS_TILE];
  const int64_t lo = chunks[3 * blockIdx.x], hi = chunks[3 * blockIdx.x + 1];
  const int width = k * (d + 1);
  const int o0 = blockIdx.y * HM_THREADS * WS_NACC + threadIdx.x;
  int oc[WS_NACC], oj[WS_NACC];
#pragma unroll
  for (int s = 0; s < WS_NACC; ++s) {
    const int o = min(o0 + s * HM_THREADS, width - 1);
    oc[s] = o / (d + 1);
    oj[s] = o - oc[s] * (d + 1);
  }
  double acc[WS_NACC] = {};
  for (int64_t b = lo; b < hi; b += WS_TILE) {
    const int m = (int)min((int64_t)WS_TILE, hi - b);
    for (int e = threadIdx.x; e < m * (d + 1); e += HM_THREADS) {
      const int t = e / (d + 1), j = e - t * (d + 1);
      const int64_t i = idx ? idx[b + t] : b + t;
      zt[e] = j < d ? (double)z[i * d + j] : 1.0;
    }
    if (MODE == 0)
      for (int e = threadIdx.x; e < m * k; e += HM_THREADS) {
        const int t = e / k, c = e - t * k;
        const int64_t i = idx ? idx[b + t] : b + t;
        rt[e] = (double)r[i * k + c];
      }
    if (MODE == 1 && (int)threadIdx.x < m) lt[threadIdx.x] = labels[idx ? idx[b + threadIdx.x] : b + threadIdx.x];
    __syncthreads();
    for (int t = 0; t < m; ++t) {
#pragma unroll
      for (int s = 0; s < WS_NACC; ++s) {
        const double w = MODE == 0 ? rt[t * k + oc[s]] : MODE == 1 ? (lt[t] == oc[s] ? 1.0 : 0.0) : 1.0;
        acc[s] += w * zt[t * (d + 1) + oj[s]];
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int s = 0; s < WS_NACC; ++s) {
    const int o = o0 + s * HM_THREADS;
    if (o < width) part[(int64_t)blockIdx.x * width + o] = acc[s];
  }
}

// ---------------------------------------------------------------------------------------------------- clustering step
// one warp per listed cell; lane l owns clusters l, l + 32, ...
template <typename T>
__global__ void __launch_bounds__(HM_THREADS) step_kernel(int64_t rows, const int64_t* __restrict__ idx, int d, int k,
                                                           const T* __restrict__ z, const double* __restrict__ y,
                                                           int keys, const int32_t* __restrict__ codes,
                                                           const double* __restrict__ pen, double term,
                                                           T* __restrict__ r, double* __restrict__ ent) {
  extern __shared__ unsigned char st_raw[];
  const int ld = d | 1;  // odd stride: lanes reading one column of different clusters hit different banks
  T* ys = reinterpret_cast<T*>(st_raw);  // [k][ld]
  T* zrow = ys + k * ld + (threadIdx.x >> 5) * d;
  for (int e = threadIdx.x; e < k * d; e += HM_THREADS) ys[(e / d) * ld + e % d] = (T)y[e];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const T* yrow[HM_KPL];
#pragma unroll
  for (int q = 0; q < HM_KPL; ++q) yrow[q] = ys + min(lane + 32 * q, k - 1) * ld;
  for (int64_t p = (int64_t)blockIdx.x * HM_WARPS + (threadIdx.x >> 5); p < rows; p += (int64_t)gridDim.x * HM_WARPS) {
    const int64_t i = idx ? idx[p] : p;
    for (int j = lane; j < d; j += 32) zrow[j] = z[i * d + j];
    __syncwarp();
    T dot[HM_KPL] = {};
    for (int j = 0; j < d; ++j) {
      const T zj = zrow[j];
#pragma unroll
      for (int q = 0; q < HM_KPL; ++q) dot[q] += zj * yrow[q][j];
    }
    T lr[HM_KPL];
    T mx = -INFINITY;
#pragma unroll
    for (int q = 0; q < HM_KPL; ++q) {
      const int c = lane + 32 * q;
      lr[q] = -INFINITY;
      if (c < k) {
        T v = (T)term * (T(1) - dot[q]);
        if (pen) {
          double ps = 0.0;
          for (int u = 0; u < keys; ++u) ps += pen[(int64_t)codes[i * keys + u] * k + c];
          v += (T)ps;
        }
        lr[q] = v;
        mx = max(mx, v);
      }
    }
    mx = warp_max(mx);
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < HM_KPL; ++q) {
      lr[q] = lane + 32 * q < k ? (T)exp((double)(lr[q] - mx)) : T(0);
      s += (double)lr[q];
    }
    s = fmax(warp_sum(s), 1e-12);
    double s2 = 0.0;
#pragma unroll
    for (int q = 0; q < HM_KPL; ++q) {
      lr[q] = (T)((double)lr[q] / s);
      s2 += (double)lr[q];
      if (lane + 32 * q < k) r[i * k + lane + 32 * q] = lr[q];
    }
    s2 = fmax(warp_sum(s2), 1e-12);
    double h = 0.0;
#pragma unroll
    for (int q = 0; q < HM_KPL; ++q)
      if (lane + 32 * q < k) {
        const double rn = (double)lr[q] / s2;
        h += rn * log(rn + 1e-12);
      }
    h = warp_sum(h);
    if (lane == 0) ent[i] = h;
    __syncwarp();
  }
}

// part[cta][(n_codes + 1) * k]; thread c sums column c of its CTA's cells in list order
template <typename T>
__global__ void __launch_bounds__(HM_MAXK) code_sums_kernel(int64_t rows, int64_t per, const int64_t* __restrict__ idx,
                                                             int k, const T* __restrict__ r, int keys,
                                                             const int32_t* __restrict__ codes, int n_codes,
                                                             double* __restrict__ part) {
  extern __shared__ double cs_sm[];
  const int width = (n_codes + 1) * k;
  for (int e = threadIdx.x; e < width; e += blockDim.x) cs_sm[e] = 0.0;
  __syncthreads();
  const int c = threadIdx.x;
  const int64_t p0 = blockIdx.x * per, p1 = min(rows, p0 + per);
  if (c < k)
    for (int64_t p = p0; p < p1; ++p) {
      const int64_t i = idx ? idx[p] : p;
      const double v = (double)r[i * k + c];
      for (int u = 0; u < keys; ++u) cs_sm[codes[i * keys + u] * k + c] += v;
      cs_sm[n_codes * k + c] += v;
    }
  __syncthreads();
  for (int e = threadIdx.x; e < width; e += blockDim.x) part[(int64_t)blockIdx.x * width + e] = cs_sm[e];
}

__global__ void oe_update_kernel(int n_codes, int k, double sign, const double* __restrict__ sums,
                                 const double* __restrict__ pr_b, const double* __restrict__ theta, int stabilized,
                                 double* __restrict__ o, double* __restrict__ e, double* __restrict__ pen) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_codes * k) return;
  const int b = t / k, c = t - b * k;
  const double ov = o[t] + sign * sums[t];
  const double ev = e[t] + sign * (pr_b[b] * sums[n_codes * k + c]);
  o[t] = ov;
  e[t] = ev;
  pen[t] = theta[b] * (log(ev + 1.0) - log((stabilized ? ov + ev : ov) + 1.0));
}

// part[cta] = Σ of the CTA's contiguous share of v, in a fixed order
__global__ void __launch_bounds__(HM_THREADS) sum_kernel(int64_t n, int64_t per, const double* __restrict__ v,
                                                          double* __restrict__ part) {
  __shared__ double red[HM_WARPS];
  const int64_t p0 = blockIdx.x * per, p1 = min(n, p0 + per);
  double s = 0.0;
  for (int64_t i = p0 + threadIdx.x; i < p1; i += HM_THREADS) s += v[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// ---------------------------------------------------------------------------------------------------- k-means start
template <typename T>
__global__ void __launch_bounds__(HM_THREADS) center_kernel(int64_t n, int d, const T* __restrict__ z,
                                                             const double* __restrict__ mean, double* __restrict__ xc,
                                                             double* __restrict__ xx) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * HM_WARPS + (threadIdx.x >> 5);
  if (i >= n) return;
  double s = 0.0;
  for (int j = lane; j < d; j += 32) {
    const double v = (double)z[i * d + j] - mean[j];
    xc[i * d + j] = v;
    s += v * v;
  }
  s = warp_sum(s);
  if (lane == 0) xx[i] = s;
}

// one CTA per uniform: thread t owns a contiguous segment; cumsum(v)[i] is taken as (the sum of the earlier
// segments, serially) + (the running sum within the segment), which is non-decreasing across the segments
__global__ void __launch_bounds__(1024) kpp_search_kernel(int64_t n, const double* __restrict__ v,
                                                          const double* __restrict__ u, int64_t* __restrict__ ids) {
  __shared__ double seg[1024], pre[1024];
  const int t = threadIdx.x;
  const int64_t len = (n + 1023) / 1024, lo = min(n, t * len), hi = min(n, lo + len);
  double s = 0.0;
  for (int64_t i = lo; i < hi; ++i) s += v[i];
  seg[t] = s;
  __syncthreads();
  if (t == 0) {
    double p = 0.0;
    for (int q = 0; q < 1024; ++q) {
      pre[q] = p;
      p += seg[q];
    }
    ids[blockIdx.x] = n - 1;
  }
  __syncthreads();
  const double uu = u[blockIdx.x];
  if ((t == 0 || pre[t] < uu) && uu <= pre[t] + seg[t] && lo < hi) {
    double c = 0.0;
    for (int64_t i = lo; i < hi; ++i) {
      c += v[i];
      if (pre[t] + c >= uu) {
        ids[blockIdx.x] = i;
        break;
      }
    }
  }
}

__global__ void __launch_bounds__(HM_THREADS) kpp_dists_kernel(int64_t n, int d, const double* __restrict__ xc,
                                                                const double* __restrict__ xx, int trials,
                                                                const int64_t* __restrict__ ids,
                                                                const double* __restrict__ closest,
                                                                double* __restrict__ dist, double* __restrict__ part) {
  extern __shared__ double kd_sm[];  // [trials][d], then the candidates' squared norms
  __shared__ double red[HM_WARPS];
  double* cn = kd_sm + trials * d;
  for (int e = threadIdx.x; e < trials * d; e += HM_THREADS) kd_sm[e] = xc[ids[e / d] * d + e % d];
  __syncthreads();
  if ((int)threadIdx.x < trials) {
    double s = 0.0;
    for (int j = 0; j < d; ++j) s += kd_sm[threadIdx.x * d + j] * kd_sm[threadIdx.x * d + j];
    cn[threadIdx.x] = s;
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * HM_THREADS + threadIdx.x;
  double dot[SB2_HARMONY_MAX_TRIALS] = {};
  if (i < n)
    for (int j = 0; j < d; ++j) {
      const double xj = xc[i * d + j];
#pragma unroll
      for (int t = 0; t < SB2_HARMONY_MAX_TRIALS; ++t)
        if (t < trials) dot[t] += xj * kd_sm[t * d + j];
    }
#pragma unroll
  for (int t = 0; t < SB2_HARMONY_MAX_TRIALS; ++t) {
    if (t >= trials) break;
    double v = 0.0;
    if (i < n) {
      v = fmax(-2.0 * dot[t] + cn[t] + xx[i], 0.0);
      if (closest) v = fmin(closest[i], v);
      dist[t * n + i] = v;
    }
    v = block_sum(v, red);
    if (threadIdx.x == 0) part[(int64_t)blockIdx.x * trials + t] = v;
  }
}

__global__ void __launch_bounds__(HM_THREADS) labels_kernel(int64_t n, int d, int k, const double* __restrict__ xc,
                                                             const double* __restrict__ centers,
                                                             const int32_t* __restrict__ old,
                                                             int32_t* __restrict__ labels,
                                                             int32_t* __restrict__ changed) {
  extern __shared__ double lb_sm[];
  const int ld = d | 1;
  double* cs = lb_sm;                   // [k][ld]
  double* cn = lb_sm + k * ld;          // [k]
  double* xr = cn + k + (threadIdx.x >> 5) * d;
  for (int e = threadIdx.x; e < k * d; e += HM_THREADS) cs[(e / d) * ld + e % d] = centers[e];
  __syncthreads();
  for (int c = threadIdx.x; c < k; c += HM_THREADS) {
    double s = 0.0;
    for (int j = 0; j < d; ++j) s += cs[c * ld + j] * cs[c * ld + j];
    cn[c] = s;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * HM_WARPS + (threadIdx.x >> 5);
  if (i >= n) return;
  for (int j = lane; j < d; j += 32) xr[j] = xc[i * d + j];
  __syncwarp();
  double dot[HM_KPL] = {};
  for (int j = 0; j < d; ++j) {
    const double xj = xr[j];
#pragma unroll
    for (int q = 0; q < HM_KPL; ++q) dot[q] += xj * cs[min(lane + 32 * q, k - 1) * ld + j];
  }
  double best = INFINITY;
  int bi = k;
#pragma unroll
  for (int q = 0; q < HM_KPL; ++q) {
    const int c = lane + 32 * q;
    if (c < k) {
      const double v = -2.0 * dot[q] + cn[c];
      if (v < best) best = v, bi = c;  // q ascending: the first of equal values in this lane
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob < best || (ob == best && oi < bi)) best = ob, bi = oi;
  }
  if (lane == 0) {
    labels[i] = bi;
    if (old[i] != bi) *changed = 1;
  }
}

// ---------------------------------------------------------------------------------------------------- correction
// one CTA per chunk of one code tuple: wc[c][j] = Σ_keys w[c][code + 1][j] in shared memory, then one warp per cell
template <typename T>
__global__ void __launch_bounds__(HM_THREADS) apply_kernel(const int64_t* __restrict__ chunks,
                                                            const int64_t* __restrict__ idx, int d, int k, int keys,
                                                            const int32_t* __restrict__ gcodes, int n_codes,
                                                            const double* __restrict__ w, const T* __restrict__ x,
                                                            const T* __restrict__ r, T* __restrict__ zhat,
                                                            T* __restrict__ znorm) {
  extern __shared__ double ap_sm[];
  double* wc = ap_sm;                                  // [k][d]
  double* rr = ap_sm + k * d + (threadIdx.x >> 5) * k;  // this warp's r row
  const int64_t lo = chunks[3 * blockIdx.x], hi = chunks[3 * blockIdx.x + 1], g = chunks[3 * blockIdx.x + 2];
  for (int e = threadIdx.x; e < k * d; e += HM_THREADS) {
    const int c = e / d, j = e - c * d;
    double s = 0.0;
    for (int u = 0; u < keys; ++u) s += w[((int64_t)c * (n_codes + 1) + gcodes[g * keys + u] + 1) * d + j];
    wc[e] = s;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int64_t p = lo + (threadIdx.x >> 5); p < hi; p += HM_WARPS) {
    const int64_t i = idx[p];
    for (int c = lane; c < k; c += 32) rr[c] = (double)r[i * k + c];
    __syncwarp();
    T v[HM_DPL];
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < HM_DPL; ++q) {
      const int j = lane + 32 * q;
      v[q] = T(0);
      if (j < d) {
        double a = 0.0;
        for (int c = 0; c < k; ++c) a += rr[c] * wc[c * d + j];
        v[q] = (T)((double)x[i * d + j] - a);
        zhat[i * d + j] = v[q];
      }
      s += (double)v[q] * (double)v[q];
    }
    const double nrm = fmax(sqrt(warp_sum(s)), 1e-12);
#pragma unroll
    for (int q = 0; q < HM_DPL; ++q) {
      const int j = lane + 32 * q;
      if (j < d) znorm[i * d + j] = (T)((double)v[q] / nrm);
    }
    __syncwarp();
  }
}

int32_t set_smem(const void* fn, size_t bytes) {
  if (bytes > 48 * 1024) SB2_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return SB2_OK;
}

#define HM_SHAPE(d, k)                                                                                 \
  SB2_CHECK_ARG((d) >= 1 && (d) <= SB2_HARMONY_MAX_D && (k) >= 1 && (k) <= SB2_HARMONY_MAX_K, "shape")

}  // namespace

extern "C" {

int32_t sb2_harmony_normalize(sb2_ctx* ctx, int64_t n, int32_t d, int32_t is_f64, const void* d_x, void* d_out) {
  SB2_CHECK_ARG(ctx && d_x && d_out && n >= 0, "null pointer");
  HM_SHAPE(d, 1);
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  with_t(is_f64, [&](auto t) {
    using T = decltype(t);
    normalize_kernel<T><<<(unsigned)ceil_div64(n, HM_WARPS), HM_THREADS, 0, ctx->stream>>>(
        n, d, static_cast<const T*>(d_x), static_cast<T*>(d_out));
  });
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_harmony_wsums(sb2_ctx* ctx, int32_t groups, const int64_t* h_bounds, const int64_t* d_idx, int32_t d,
                          int32_t k, int32_t is_f64, const void* d_z, int32_t mode, const void* d_r,
                          const int32_t* d_labels, double* d_out) {
  SB2_CHECK_ARG(ctx && h_bounds && d_z && d_out && groups >= 1, "null pointer");
  HM_SHAPE(d, k);
  SB2_CHECK_ARG((mode == 0 && d_r) || (mode == 1 && d_labels && is_f64) || (mode == 2 && k == 1), "weights");
  SB2_CUDA(cudaSetDevice(ctx->device));
  std::vector<int64_t> chunks, cb;
  make_chunks(groups, h_bounds, chunks, cb);
  const int64_t nch = cb[groups], width = (int64_t)k * (d + 1);
  ScratchScope scr(ctx);
  if (nch == 0) {
    SB2_CUDA(cudaMemsetAsync(d_out, 0, groups * width * sizeof(double), ctx->stream));
    return SB2_OK;
  }
  int64_t *d_chunks, *d_cb;
  double* part;
  SB2_TRY(upload(ctx, scr, chunks, &d_chunks));
  SB2_TRY(upload(ctx, scr, cb, &d_cb));
  SB2_TRY(scr.alloc(&part, (size_t)(nch * width)));
  SB2_CHECK_ARG(nch < INT32_MAX, "shape");
  const dim3 grid((unsigned)nch, (unsigned)ceil_div64(width, HM_THREADS * WS_NACC));
  const size_t smem = (size_t)WS_TILE * ((d + 1) + (mode == 0 ? k : 0)) * sizeof(double);
  int32_t st = SB2_OK;
  with_t(is_f64, [&](auto t) {
    using T = decltype(t);
    const auto launch = [&](auto kern) {
      st = set_smem((const void*)kern, smem);
      if (st == SB2_OK)
        kern<<<grid, HM_THREADS, smem, ctx->stream>>>(d_chunks, d_idx, d, k, static_cast<const T*>(d_z),
                                                       static_cast<const T*>(d_r), d_labels, part);
    };
    if (mode == 0) launch(wsums_kernel<T, 0>);
    else if (mode == 2) launch(wsums_kernel<T, 2>);
    else if constexpr (std::is_same_v<T, double>) launch(wsums_kernel<double, 1>);
  });
  SB2_TRY(st);
  SB2_LAUNCH_CHECK(ctx);
  return fold(ctx, groups, d_cb, nch, width, part, d_out);
}

int32_t sb2_harmony_step(sb2_ctx* ctx, int64_t rows, const int64_t* d_idx, int32_t d, int32_t k, int32_t is_f64,
                         const void* d_z, const double* d_y, int32_t keys, const int32_t* d_codes, const double* d_pen,
                         double term, void* d_r, double* d_ent) {
  SB2_CHECK_ARG(ctx && d_z && d_y && d_r && d_ent && rows >= 0, "null pointer");
  SB2_CHECK_ARG(!d_pen || (d_codes && keys >= 1), "codes");
  HM_SHAPE(d, k);
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (rows == 0) return SB2_OK;
  int32_t st = SB2_OK;
  with_t(is_f64, [&](auto t) {
    using T = decltype(t);
    const size_t smem = ((size_t)k * (d | 1) + (size_t)HM_WARPS * d) * sizeof(T);
    st = set_smem((const void*)step_kernel<T>, smem);
    if (st != SB2_OK) return;
    const int64_t ctas = std::min<int64_t>(ceil_div64(rows, HM_WARPS * 4), (int64_t)ctx->prop.multiProcessorCount * 8);
    step_kernel<T><<<(unsigned)ctas, HM_THREADS, smem, ctx->stream>>>(
        rows, d_idx, d, k, static_cast<const T*>(d_z), d_y, keys, d_codes, d_pen, term, static_cast<T*>(d_r), d_ent);
  });
  SB2_TRY(st);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_harmony_code_sums(sb2_ctx* ctx, int64_t rows, const int64_t* d_idx, int32_t k, int32_t is_f64,
                              const void* d_r, int32_t keys, const int32_t* d_codes, int32_t n_codes, double* d_out) {
  SB2_CHECK_ARG(ctx && d_r && d_codes && d_out && rows >= 0 && keys >= 1, "null pointer");
  SB2_CHECK_ARG(k >= 1 && k <= SB2_HARMONY_MAX_K && n_codes >= 1 && n_codes <= SB2_HARMONY_MAX_CODES, "shape");
  SB2_CUDA(cudaSetDevice(ctx->device));
  const int64_t width = (int64_t)(n_codes + 1) * k;
  if (rows == 0) {
    SB2_CUDA(cudaMemsetAsync(d_out, 0, width * sizeof(double), ctx->stream));
    return SB2_OK;
  }
  const int64_t parts = std::min<int64_t>(SUM_PARTS, ceil_div64(rows, 256)), per = ceil_div64(rows, parts);
  ScratchScope scr(ctx);
  double* part;
  SB2_TRY(scr.alloc(&part, (size_t)(parts * width)));
  const size_t smem = width * sizeof(double);
  int32_t st = SB2_OK;
  with_t(is_f64, [&](auto t) {
    using T = decltype(t);
    st = set_smem((const void*)code_sums_kernel<T>, smem);
    if (st != SB2_OK) return;
    code_sums_kernel<T><<<(unsigned)ceil_div64(rows, per), HM_MAXK, smem, ctx->stream>>>(
        rows, per, d_idx, k, static_cast<const T*>(d_r), keys, d_codes, n_codes, part);
  });
  SB2_TRY(st);
  SB2_LAUNCH_CHECK(ctx);
  return fold(ctx, 1, nullptr, ceil_div64(rows, per), width, part, d_out);
}

int32_t sb2_harmony_oe_update(sb2_ctx* ctx, int32_t n_codes, int32_t k, double sign, const double* d_sums,
                              const double* d_pr_b, const double* d_theta, int32_t stabilized, double* d_o, double* d_e,
                              double* d_pen) {
  SB2_CHECK_ARG(ctx && d_sums && d_pr_b && d_theta && d_o && d_e && d_pen && n_codes >= 1 && k >= 1, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  oe_update_kernel<<<(unsigned)ceil_div64((int64_t)n_codes * k, 256), 256, 0, ctx->stream>>>(
      n_codes, k, sign, d_sums, d_pr_b, d_theta, stabilized, d_o, d_e, d_pen);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_harmony_sum(sb2_ctx* ctx, int64_t n, const double* d_v, double* d_out) {
  SB2_CHECK_ARG(ctx && d_v && d_out && n >= 1, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  const int64_t parts = std::min<int64_t>(SUM_PARTS, ceil_div64(n, HM_THREADS)), per = ceil_div64(n, parts);
  const int64_t ctas = ceil_div64(n, per);
  ScratchScope scr(ctx);
  double* part;
  SB2_TRY(scr.alloc(&part, (size_t)ctas));
  sum_kernel<<<(unsigned)ctas, HM_THREADS, 0, ctx->stream>>>(n, per, d_v, part);
  SB2_LAUNCH_CHECK(ctx);
  return fold(ctx, 1, nullptr, ctas, 1, part, d_out);
}

int32_t sb2_harmony_center(sb2_ctx* ctx, int64_t n, int32_t d, int32_t is_f64, const void* d_z, const double* d_mean,
                           double* d_xc, double* d_xx) {
  SB2_CHECK_ARG(ctx && d_z && d_mean && d_xc && d_xx && n >= 0, "null pointer");
  HM_SHAPE(d, 1);
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  with_t(is_f64, [&](auto t) {
    using T = decltype(t);
    center_kernel<T><<<(unsigned)ceil_div64(n, HM_WARPS), HM_THREADS, 0, ctx->stream>>>(
        n, d, static_cast<const T*>(d_z), d_mean, d_xc, d_xx);
  });
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_harmony_kpp_search(sb2_ctx* ctx, int64_t n, const double* d_v, int32_t trials, const double* d_u,
                               int64_t* d_ids) {
  SB2_CHECK_ARG(ctx && d_v && d_u && d_ids && n >= 1, "null pointer");
  SB2_CHECK_ARG(trials >= 1 && trials <= SB2_HARMONY_MAX_TRIALS, "trials");
  SB2_CUDA(cudaSetDevice(ctx->device));
  kpp_search_kernel<<<trials, 1024, 0, ctx->stream>>>(n, d_v, d_u, d_ids);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_harmony_kpp_dists(sb2_ctx* ctx, int64_t n, int32_t d, const double* d_xc, const double* d_xx,
                              int32_t trials, const int64_t* d_ids, const double* d_closest, double* d_dist,
                              double* d_pot) {
  SB2_CHECK_ARG(ctx && d_xc && d_xx && d_ids && d_dist && d_pot && n >= 1, "null pointer");
  SB2_CHECK_ARG(trials >= 1 && trials <= SB2_HARMONY_MAX_TRIALS, "trials");
  HM_SHAPE(d, 1);
  SB2_CUDA(cudaSetDevice(ctx->device));
  const int64_t ctas = ceil_div64(n, HM_THREADS);
  ScratchScope scr(ctx);
  double* part;
  SB2_TRY(scr.alloc(&part, (size_t)(ctas * trials)));
  const size_t smem = (size_t)trials * (d + 1) * sizeof(double);
  kpp_dists_kernel<<<(unsigned)ctas, HM_THREADS, smem, ctx->stream>>>(n, d, d_xc, d_xx, trials, d_ids, d_closest,
                                                                      d_dist, part);
  SB2_LAUNCH_CHECK(ctx);
  return fold(ctx, 1, nullptr, ctas, trials, part, d_pot);
}

int32_t sb2_harmony_labels(sb2_ctx* ctx, int64_t n, int32_t d, int32_t k, const double* d_xc, const double* d_centers,
                           const int32_t* d_old, int32_t* d_labels, int32_t* d_changed) {
  SB2_CHECK_ARG(ctx && d_xc && d_centers && d_old && d_labels && d_changed && n >= 0, "null pointer");
  HM_SHAPE(d, k);
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  const size_t smem = ((size_t)k * (d | 1) + k + (size_t)HM_WARPS * d) * sizeof(double);
  SB2_TRY(set_smem((const void*)labels_kernel, smem));
  labels_kernel<<<(unsigned)ceil_div64(n, HM_WARPS), HM_THREADS, smem, ctx->stream>>>(n, d, k, d_xc, d_centers, d_old,
                                                                                        d_labels, d_changed);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

int32_t sb2_harmony_apply(sb2_ctx* ctx, int32_t groups, const int64_t* h_bounds, const int64_t* d_idx, int32_t d,
                          int32_t k, int32_t is_f64, int32_t keys, const int32_t* d_gcodes, int32_t n_codes,
                          const double* d_w, const void* d_x, const void* d_r, void* d_zhat, void* d_znorm) {
  SB2_CHECK_ARG(ctx && h_bounds && d_idx && d_gcodes && d_w && d_x && d_r && d_zhat && d_znorm, "null pointer");
  SB2_CHECK_ARG(groups >= 1 && groups <= SB2_HARMONY_MAX_TUPLES && keys >= 1, "groups");
  SB2_CHECK_ARG(n_codes >= 1 && n_codes <= SB2_HARMONY_MAX_CODES, "codes");
  HM_SHAPE(d, k);
  SB2_CUDA(cudaSetDevice(ctx->device));
  std::vector<int64_t> chunks, cb;
  make_chunks(groups, h_bounds, chunks, cb);
  const int64_t nch = cb[groups];
  if (nch == 0) return SB2_OK;
  SB2_CHECK_ARG(nch < INT32_MAX, "shape");
  ScratchScope scr(ctx);
  int64_t* d_chunks;
  SB2_TRY(upload(ctx, scr, chunks, &d_chunks));
  const size_t smem = ((size_t)k * d + (size_t)HM_WARPS * k) * sizeof(double);
  int32_t st = SB2_OK;
  with_t(is_f64, [&](auto t) {
    using T = decltype(t);
    st = set_smem((const void*)apply_kernel<T>, smem);
    if (st != SB2_OK) return;
    apply_kernel<T><<<(unsigned)nch, HM_THREADS, smem, ctx->stream>>>(
        d_chunks, d_idx, d, k, keys, d_gcodes, n_codes, d_w, static_cast<const T*>(d_x), static_cast<const T*>(d_r),
        static_cast<T*>(d_zhat), static_cast<T*>(d_znorm));
  });
  SB2_TRY(st);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

}  // extern "C"

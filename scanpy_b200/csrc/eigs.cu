// eigs.cu — extreme eigenpairs of a diagonally scaled symmetric CSR operator  M = diag(s) A diag(s)  (A fp32 CSR,
// symmetric; s fp64; all vectors fp64) by thick-restart Lanczos with full (CGS2) re-orthogonalisation.
//
// Replaces the reference's `scipy.sparse.linalg.eigsh(matrix.astype(float64), k, which='LM'|'SM'-style ends, v0=...)` calls:
//   * sc.tl.diffmap / Neighbors.compute_eigen   src/scanpy/neighbors/__init__.py:832-884   (A = connectivities,
//       s = 1/(q z): T_sym = Z^-1 Q^-1 W Q^-1 Z^-1, :791-830)
//   * the spectral initialisation inside umap's simplicial_set_embedding (sc.tl.umap, src/scanpy/tools/_umap.py:196-215):
//       smallest eigenvectors of I - D^-1/2 A D^-1/2  ==  largest of D^-1/2 A D^-1/2
// HBM-bound: one step = 1 SpMV (12 B per stored arc + 16 B per row) + 4 tall-skinny passes over the <= m basis vectors.
// Restart eigenproblem (m x m, m <= 128) is solved on the host by cyclic Jacobi: O(m^3) flops on a 1e4-entry matrix,
// control-plane work like the host-side convergence test.
#include <math.h>

#include <algorithm>
#include <numeric>

#include "common.cuh"

namespace {

constexpr int RB = 1024;  // rows per CTA in the tall-skinny kernels

// y = s .* (A (s .* x)); warp per row
__global__ void __launch_bounds__(256)
eig_spmv_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ w,
                const double* __restrict__ s, const double* __restrict__ x, double* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  double acc = 0.0;
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32) {
    const int32_t c = indices[e];
    acc += (double)w[e] * (s ? s[c] * x[c] : x[c]);
  }
  acc = warp_sum(acc);
  if (lane == 0) y[row] = s ? s[row] * acc : acc;
}

// partial[b][c] = sum over the CTA's rows of V[c][i] * w[i], c < nv  (V column-major: vector c at V + c*ld)
__global__ void __launch_bounds__(256)
eig_dots_kernel(int64_t n, int nv, const double* __restrict__ V, int64_t ld, const double* __restrict__ w,
                double* __restrict__ partial) {
  __shared__ double red[8];
  const int64_t r0 = (int64_t)blockIdx.x * RB;
  double wv[RB / 256];
#pragma unroll
  for (int j = 0; j < RB / 256; ++j) {
    const int64_t i = r0 + threadIdx.x + j * 256;
    wv[j] = i < n ? w[i] : 0.0;
  }
  for (int c = 0; c < nv; ++c) {
    const double* v = V + (size_t)c * ld;
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < RB / 256; ++j) {
      const int64_t i = r0 + threadIdx.x + j * 256;
      if (i < n) acc += v[i] * wv[j];
    }
    const double t = block_sum(acc, red);
    if (threadIdx.x == 0) partial[(size_t)blockIdx.x * nv + c] = t;
  }
}
// h[c] = sum_b partial[b][c]  (fixed order: deterministic); one warp per c
__global__ void eig_reduce_kernel(int nb, int nv, const double* __restrict__ partial, double* __restrict__ h) {
  const int c = blockIdx.x;
  double acc = 0.0;
  for (int b = threadIdx.x; b < nb; b += 32) acc += partial[(size_t)b * nv + c];
  acc = warp_sum(acc);
  if (threadIdx.x == 0) h[c] = acc;
}
// w -= V[:, :nv] h
__global__ void __launch_bounds__(256)
eig_axpy_kernel(int64_t n, int nv, const double* __restrict__ V, int64_t ld, const double* __restrict__ h, double* __restrict__ w) {
  extern __shared__ double sh[];
  for (int c = threadIdx.x; c < nv; c += blockDim.x) sh[c] = h[c];
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = w[i];
  for (int c = 0; c < nv; ++c) acc -= V[(size_t)c * ld + i] * sh[c];
  w[i] = acc;
}
// out = w * (1 / *norm)   (norm on the device: no host round trip inside a Lanczos step)
__global__ void eig_scale_kernel(int64_t n, const double* __restrict__ w, const double* __restrict__ nrm2, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double nr = sqrt(*nrm2);
  out[i] = nr > 0.0 ? w[i] / nr : 0.0;
}
// out[i] = splitmix64(i, salt) mapped to [-1, 1): a start vector unrelated to any Krylov space met so far
__global__ void eig_fresh_kernel(int64_t n, uint64_t salt, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t z = (uint64_t)i + 0x9E3779B97F4A7C15ull * salt;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  out[i] = (double)((z ^ (z >> 31)) >> 11) * (2.0 / 9007199254740992.0) - 1.0;
}
// Vout[:, j0 + t] = V[:, :m] Y[:, t], t < nt <= 8  (Y column-major m x nt in shared memory)
__global__ void __launch_bounds__(256)
eig_rotate_kernel(int64_t n, int m, int nt, const double* __restrict__ V, int64_t ld, const double* __restrict__ Y,
                  double* __restrict__ Vout) {
  extern __shared__ double sy[];
  for (int t = threadIdx.x; t < m * nt; t += blockDim.x) sy[t] = Y[t];
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) acc[t] = 0.0;
  for (int c = 0; c < m; ++c) {
    const double v = V[(size_t)c * ld + i];
#pragma unroll
    for (int t = 0; t < 8; ++t)
      if (t < nt) acc[t] += v * sy[t * m + c];
  }
#pragma unroll
  for (int t = 0; t < 8; ++t)
    if (t < nt) Vout[(size_t)t * ld + i] = acc[t];
}

// transitions of sc.tl.diffmap (Neighbors.compute_transitions): step 0  q = W 1;  step 1  s = 1 / (q z) with
// z = sqrt((Q^-1 W Q^-1) 1) = sqrt(q^-1 .* (W q^-1))   (density_normalize), or s = 1 / sqrt(q) without
__global__ void __launch_bounds__(256)
eig_transition_scale_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                            const float* __restrict__ w, const double* __restrict__ q, int step, int density, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  double acc = 0.0;
  for (int64_t e = indptr[row] + lane; e < indptr[row + 1]; e += 32) acc += (double)w[e] * (step == 0 ? 1.0 : 1.0 / q[indices[e]]);
  acc = warp_sum(acc);
  if (lane != 0) return;
  if (step == 0) out[row] = density ? acc : 1.0 / sqrt(acc);
  else {
    const double qi = 1.0 / q[row];
    out[row] = qi / sqrt(qi * acc);
  }
}

struct Eigs {
  sb2_ctx* ctx;
  cudaStream_t st;
  int64_t n;
  const int64_t* indptr;
  const int32_t* indices;
  const float* w;
  const double* s;
  double *partial, *h;  // [nb * (m+1)], [m + 2]
  int nb;

  int32_t apply(const double* x, double* y) {
    eig_spmv_kernel<<<(unsigned)ceil_div64(n, 8), 256, 0, st>>>(n, indptr, indices, w, s, x, y);
    SB2_LAUNCH_CHECK(ctx);
    return SB2_OK;
  }
  // hdev[0..nv) = V[:, :nv]^T w
  int32_t dots(int nv, const double* V, const double* wv, double* hdev) {
    eig_dots_kernel<<<nb, 256, 0, st>>>(n, nv, V, n, wv, partial);
    SB2_LAUNCH_CHECK(ctx);
    eig_reduce_kernel<<<nv, 32, 0, st>>>(nb, nv, partial, hdev);
    SB2_LAUNCH_CHECK(ctx);
    return SB2_OK;
  }
  int32_t axpy(int nv, const double* V, const double* hdev, double* wv) {
    eig_axpy_kernel<<<(unsigned)ceil_div64(n, 256), 256, sizeof(double) * nv, st>>>(n, nv, V, n, hdev, wv);
    SB2_LAUNCH_CHECK(ctx);
    return SB2_OK;
  }
};

}  // namespace

// d_v0 fp64[n] start vector (any non-zero); which: 0 = largest algebraic, 1 = largest magnitude (scipy 'LM'), 2 = smallest
// algebraic.  Outputs: h_evals[nev] ascending (like eigsh), d_evecs fp64 [nev x n] row e = unit eigenvector of h_evals[e].
extern "C" int32_t sb2_eigsh_csr_scaled(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                        const float* d_weights, const double* d_scale, int32_t nev, int32_t which,
                                        int32_t ncv, double tol, int32_t max_restarts, const double* d_v0,
                                        double* h_evals, double* d_evecs, sb2_eigs_info* info) {
  return eigsh_csr_scaled(ctx, n, d_indptr, d_indices, d_weights, d_scale, nev, which, ncv, tol, max_restarts, d_v0, h_evals,
                          d_evecs, info, true);
}

int32_t eigsh_csr_scaled(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices, const float* d_weights,
                         const double* d_scale, int32_t nev, int32_t which, int32_t ncv, double tol, int32_t max_restarts,
                         const double* d_v0, double* h_evals, double* d_evecs, sb2_eigs_info* info, bool lock_and_search) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_weights && d_v0 && h_evals && d_evecs, "null pointer");
  SB2_CHECK_ARG(n >= 2 && n < INT32_MAX, "n");
  SB2_CHECK_ARG(nev >= 1 && nev < n && nev <= 64, "nev must be in [1, min(n-1, 64)]");
  SB2_CHECK_ARG(which >= 0 && which <= 2, "which");
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  int m = ncv > 0 ? ncv : std::max(2 * nev + 16, 40);
  m = (int)std::min<int64_t>(std::min(m, 128), n - 1);
  SB2_CHECK_ARG(m > nev, "ncv must exceed nev");
  if (tol <= 0.0) tol = 1e-10;
  if (max_restarts <= 0) max_restarts = 400;
  ScratchScope scr(ctx);
  Eigs E{ctx, st, n, d_indptr, d_indices, d_weights, d_scale, nullptr, nullptr, (int)ceil_div64(n, RB)};
  double *V, *V2, *wv;
  SB2_TRY(scr.alloc(&V, (size_t)(m + 1) * n));
  SB2_TRY(scr.alloc(&V2, (size_t)(m + 1) * n));
  SB2_TRY(scr.alloc(&wv, (size_t)n));
  SB2_TRY(scr.alloc(&E.partial, (size_t)E.nb * (m + 2)));
  SB2_TRY(scr.alloc(&E.h, (size_t)2 * (m + 2)));
  double* dY;
  SB2_TRY(scr.alloc(&dY, (size_t)m * 8));
  const unsigned gn = (unsigned)ceil_div64(n, 256);

  // V_0 = v0 / |v0|
  SB2_TRY(E.dots(1, d_v0, d_v0, E.h));
  eig_scale_kernel<<<gn, 256, 0, st>>>(n, d_v0, E.h, V);
  SB2_LAUNCH_CHECK(ctx);

  std::vector<double> T((size_t)m * m, 0.0), Tw, theta, Y, hh(2 * (m + 2));
  std::vector<int> order(m);
  // locked[p]: basis vector p is a converged Ritz vector of an earlier cycle, kept with no coupling to the rest.  A single
  // start vector meets a repeated eigenvalue in one direction only (more copies appear only through rounding), so a set
  // that has converged is locked and searched again from a fresh start vector orthogonal to it; it is final once the
  // best Ritz value of that search has converged without displacing any of the set.  lres[p]: the residual estimate of
  // locked vector p in the cycle that locked it (its estimate in later cycles is exactly 0: it has no coupling).
  std::vector<char> locked(m + 1, 0), locked_next(m + 1, 0);
  std::vector<double> lres(m + 1, 0.0), lres_next(m + 1, 0.0);
  int k = 0, restarts = 0, n_conv = 0, matvecs = 0, nlock = 0;
  for (;;) {
    int me = m;           // effective basis size of this cycle (< m only on an exact invariant subspace)
    double beta_m = 0.0;  // coupling of the residual vector V_me
    for (int j = k; j < m; ++j) {
      SB2_TRY(E.apply(V + (size_t)j * n, wv));
      ++matvecs;
      // CGS2 against V_0..V_j; the summed coefficient of V_j is alpha_j
      SB2_TRY(E.dots(j + 1, V, wv, E.h));
      SB2_TRY(E.axpy(j + 1, V, E.h, wv));
      SB2_TRY(E.dots(j + 1, V, wv, E.h + (m + 2)));
      SB2_TRY(E.axpy(j + 1, V, E.h + (m + 2), wv));
      SB2_TRY(E.dots(1, wv, wv, E.h + 2 * (m + 2) - 1));  // |w|^2 in the last slot
      eig_scale_kernel<<<gn, 256, 0, st>>>(n, wv, E.h + 2 * (m + 2) - 1, V + (size_t)(j + 1) * n);
      SB2_LAUNCH_CHECK(ctx);
      SB2_CUDA(cudaMemcpyAsync(hh.data(), E.h, sizeof(double) * 2 * (m + 2), cudaMemcpyDeviceToHost, st));
      SB2_CUDA(cudaStreamSynchronize(st));
      const double alpha = hh[j] + hh[(m + 2) + j];
      const double beta = sqrt(std::max(0.0, hh[2 * (m + 2) - 1]));
      T[(size_t)j * m + j] = alpha;
      beta_m = beta;
      if (beta <= 1e-13 * std::max(1.0, fabs(alpha))) {  // the Krylov space is invariant: its Ritz pairs are exact
        me = j + 1;
        beta_m = 0.0;
        break;
      }
      if (j + 1 < m) T[(size_t)j * m + j + 1] = T[(size_t)(j + 1) * m + j] = beta;
    }
    if (me < nev) {
      sb2_set_error("eigsh: the Krylov space of the start vector has dimension %d < nev = %d", me, nev);
      return SB2_E_NOTCONV;
    }
    Tw.assign((size_t)me * me, 0.0);
    for (int i = 0; i < me; ++i)
      for (int j = 0; j < me; ++j) Tw[(size_t)i * me + j] = T[(size_t)i * m + j];
    jacobi_eigh(Tw, me, theta, Y);   // Y: me x me, eigenvector i in column i
    order.resize(me);
    std::iota(order.begin(), order.end(), 0);
    auto key = [&](int i) { return which == 1 ? fabs(theta[i]) : which == 0 ? theta[i] : -theta[i]; };
    std::sort(order.begin(), order.end(), [&](int a, int b) { return key(a) > key(b); });
    // Ritz vector i lies in the locked block iff its components outside it are zero (T is block diagonal there); it is
    // then locked vector lock_pos(i) itself (the diagonal block is never rotated)
    auto in_lock = [&](int i) {
      if (nlock == 0) return false;
      for (int r = 0; r < me; ++r)
        if (!locked[r] && Y[(size_t)r * me + i] != 0.0) return false;
      return true;
    };
    auto lock_pos = [&](int i) {
      int p = 0;
      for (int r = 0; r < me; ++r)
        if (Y[(size_t)r * me + i] != 0.0) p = r;
      return p;
    };
    auto res_of = [&](int i) { return in_lock(i) ? lres[lock_pos(i)] : fabs(beta_m * Y[(size_t)(me - 1) * me + i]); };
    n_conv = 0;
    double tnorm = 0.0;
    for (int i = 0; i < me; ++i) tnorm = std::max(tnorm, fabs(theta[i]));
    for (int e = 0; e < nev; ++e)
      if (res_of(order[e]) <= tol * std::max(tnorm, 1e-300)) ++n_conv;
    bool verified = false, relock = false;
    if (n_conv == nev && !lock_and_search) {
      verified = true;
    } else if (n_conv == nev) {
      if (nlock == 0) {
        relock = true;
      } else {
        double kmin = INFINITY;
        int best = -1;
        for (int i = 0; i < me; ++i) {
          if (in_lock(i)) kmin = std::min(kmin, key(i));
          else if (best < 0 || key(i) > key(best)) best = i;
        }
        if (best < 0 || res_of(best) <= tol * std::max(tnorm, 1e-300)) {
          if (best < 0 || key(best) <= kmin + 1e-12 * tnorm) verified = true;
          else relock = true;  // a new Ritz value displaces the locked set: lock the new wanted set and search again
        }
      }
    }
    if (verified && nlock > 0)  // the locked Ritz vectors are the result, ahead of any tie from the last search
      std::stable_partition(order.begin(), order.end(), [&](int i) { return in_lock(i); });
    const bool done = verified || restarts >= max_restarts;
    // Ritz vectors to keep: the wanted nev (final or locked) or nev + a share of the rest (thick restart)
    const int kk = done || relock ? nev : std::min(me - 1, nev + std::max(2, (me - nev) / 2));
    for (int i = 0; i < kk; ++i) {
      locked_next[i] = relock || in_lock(order[i]);
      lres_next[i] = res_of(order[i]);
    }
    std::vector<double> Ycols((size_t)m * 8);
    for (int j0 = 0; j0 < kk; j0 += 8) {
      const int nt = std::min(8, kk - j0);
      for (int t = 0; t < nt; ++t)
        for (int c = 0; c < me; ++c) Ycols[(size_t)t * me + c] = Y[(size_t)c * me + order[j0 + t]];
      SB2_CUDA(cudaMemcpyAsync(dY, Ycols.data(), sizeof(double) * me * nt, cudaMemcpyHostToDevice, st));
      eig_rotate_kernel<<<gn, 256, sizeof(double) * me * 8, st>>>(n, me, nt, V, n, dY, V2 + (size_t)j0 * n);
      SB2_LAUNCH_CHECK(ctx);
      SB2_CUDA(cudaStreamSynchronize(st));  // Ycols is reused by the next group
    }
    if (done) {
      // ascending eigenvalues like eigsh
      std::vector<int> asc(nev);
      std::iota(asc.begin(), asc.end(), 0);
      std::sort(asc.begin(), asc.end(), [&](int a, int b) { return theta[order[a]] < theta[order[b]]; });
      for (int e = 0; e < nev; ++e) {
        h_evals[e] = theta[order[asc[e]]];
        SB2_CUDA(cudaMemcpyAsync(d_evecs + (size_t)e * n, V2 + (size_t)asc[e] * n, sizeof(double) * n,
                                 cudaMemcpyDeviceToDevice, st));
      }
      SB2_CUDA(cudaStreamSynchronize(st));
      if (info) {
        double max_res = 0.0;
        for (int e = 0; e < nev; ++e) max_res = std::max(max_res, res_of(order[e]));
        info->restarts = restarts;
        info->matvecs = matvecs;
        info->n_converged = n_conv;
        info->max_residual = max_res;
      }
      return SB2_OK;
    }
    std::fill(T.begin(), T.end(), 0.0);
    std::fill(locked.begin(), locked.end(), 0);
    std::copy(locked_next.begin(), locked_next.begin() + kk, locked.begin());
    std::copy(lres_next.begin(), lres_next.begin() + kk, lres.begin());
    nlock = (int)std::count(locked.begin(), locked.end(), 1);
    if (relock) {
      // V <- [wanted Ritz vectors (locked), fresh start vector orthogonal to them], T <- diagonal
      eig_fresh_kernel<<<gn, 256, 0, st>>>(n, (uint64_t)(restarts + 1), wv);
      SB2_LAUNCH_CHECK(ctx);
      std::swap(V, V2);
      for (int pass = 0; pass < 2; ++pass) {
        SB2_TRY(E.dots(kk, V, wv, E.h));
        SB2_TRY(E.axpy(kk, V, E.h, wv));
      }
      SB2_TRY(E.dots(1, wv, wv, E.h + 2 * (m + 2) - 1));
      eig_scale_kernel<<<gn, 256, 0, st>>>(n, wv, E.h + 2 * (m + 2) - 1, V + (size_t)kk * n);
      SB2_LAUNCH_CHECK(ctx);
      for (int i = 0; i < kk; ++i) T[(size_t)i * m + i] = theta[order[i]];
    } else {
      // thick restart: V <- [kept Ritz vectors, residual vector], T <- arrowhead (locked rows have no coupling)
      SB2_CUDA(cudaMemcpyAsync(V2 + (size_t)kk * n, V + (size_t)m * n, sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
      std::swap(V, V2);
      for (int i = 0; i < kk; ++i) {
        T[(size_t)i * m + i] = theta[order[i]];
        const double c = beta_m * Y[(size_t)(me - 1) * me + order[i]];
        T[(size_t)i * m + kk] = T[(size_t)kk * m + i] = c;
      }
    }
    k = kk;
    ++restarts;
  }
}

// d_scale fp64[n]: T_sym = diag(d_scale) W diag(d_scale) is the symmetrised transition matrix of
// Neighbors.compute_transitions (src/scanpy/neighbors/__init__.py:791-830)
extern "C" int32_t sb2_transition_scale_f64(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                            const float* d_weights, int32_t density_normalize, double* d_scale) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_weights && d_scale, "null pointer");
  SB2_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return SB2_OK;
  ScratchScope scr(ctx);
  const unsigned grid = (unsigned)ceil_div64(n, 8);
  if (!density_normalize) {
    eig_transition_scale_kernel<<<grid, 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_weights, nullptr, 0, 0, d_scale);
    SB2_LAUNCH_CHECK(ctx);
    return SB2_OK;
  }
  double* q;
  SB2_TRY(scr.alloc(&q, (size_t)n));
  eig_transition_scale_kernel<<<grid, 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_weights, nullptr, 0, 1, q);
  SB2_LAUNCH_CHECK(ctx);
  eig_transition_scale_kernel<<<grid, 256, 0, ctx->stream>>>(n, d_indptr, d_indices, d_weights, q, 1, 1, d_scale);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

"""Exact host restatement of the device UMAP layout (scanpy_b200/csrc/umap.cu).  TEST INFRASTRUCTURE ONLY.

`oracle.graph_tools.simplicial_set_embedding` restates umap-learn's SEQUENTIAL optimiser and is the quality reference.
This module restates what `sb2_umap_layout_f32` itself computes, step for step, so the device layout can be compared
coordinate by coordinate:

* the mode-0 rescale of the initialisation, x = 10 (x - lo) / (hi - lo) per column (0 for a constant column), in fp32;
* wmax = max(w, 0); epochs per sample eps = wmax / w in fp32 for w >= wmax / prune_epochs, else 0 (never sampled), where
  prune_epochs = n_epochs if n_epochs > 10 else (500 if n <= 10000 else 200);
* one epoch = one Jacobi sweep: the owner of vertex j walks its CSR row, keeps its own position `cur` and reads every
  other end point from the previous epoch's snapshot;
* a sampled arc pulls `cur` towards the other end twice, each pull from the updated `cur`; every coordinate of a step is
  clipped to [-4, 4] before it is scaled by alpha = alpha0 (1 - ep / n_epochs) (computed in fp32 like the host loop);
* the closed-form sample test and negative-sample count in float64 exactly as the kernel evaluates them, with the
  count clamped to 64;
* the negative vertices drawn by the kernel's integer hash (integer-exact, so the same vertices are drawn).

`dtype` selects the arithmetic of the epochs: float64 is the truth the device is held to; float32 (IEEE, no FMA, a
correctly rounded pow) measures how far plain fp32 rounding drifts from it, which sets the comparison tolerance.
The keyword mutations (`pulls`, `neg_delta`, `alpha_shift`, `gauss_seidel`, `prune_epochs`, `rate_first`) exist to
show that the tolerance rejects a kernel that is wrong in one of those ways.

`running_counter_schedule` restates the sampling bookkeeping of umap's optimiser (`oracle.graph_tools._optimize`:
epoch_of_next_sample / epoch_of_next_negative_sample) without the forces, to pin the kernel's closed forms to it.
"""
from __future__ import annotations

import math

import numba
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
_S15, _S16, _S32 = np.uint64(15), np.uint64(16), np.uint64(32)
_H1, _H2 = np.uint64(0x7FEB352D), np.uint64(0x846CA68B)
_GOLD, _STEP = np.uint64(0x9E3779B9), np.uint64(0x6D2B79F5)
MAX_NEG = 64  # the kernel's clamp of negative samples per sampled arc (umap has none)

# Tolerance of device-vs-float64 comparisons: TOL_FACTOR times the fp32-vs-fp64 spread of this restatement, and never
# below TOL_FLOOR.  The device's pow is __powf (ex2.approx(b * lg2.approx(d2))), a few ulp from a correctly rounded
# powf, and nvcc contracts the sums into FMAs; both are fp32 roundings of the same size as the ones the fp32
# restatement makes, so a factor of 16 covers them.  The floor is 8 ulp of fp32 at 10, the top of the rescaled box.
TOL_FACTOR = 16.0
TOL_FLOOR = float(8 * np.spacing(np.float32(10.0)))


def seed_mix(seed: int) -> int:
    """sd = (u32)(seed ^ seed >> 32) * 2654435761 + 12345 (mod 2^32), as sb2_umap_layout_f32 derives it."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return (((seed ^ (seed >> 32)) & 0xFFFFFFFF) * 2654435761 + 12345) & 0xFFFFFFFF


def umap_v0(n: int):
    """umap_v0_kernel: the spectral initialisation's Lanczos start vector, 1 + 1e-3 (hash32(i) >> 8) / 2^24."""
    x = np.arange(n, dtype=np.uint64)
    x ^= x >> _S16
    x = (x * _H1) & M32
    x ^= x >> _S15
    x = (x * _H2) & M32
    x ^= x >> _S16
    return 1.0 + 1e-3 * (x >> np.uint64(8)).astype(np.float64) * (1.0 / 16777216.0)


def prune_epochs_for(n: int, n_epochs: int) -> int:
    return n_epochs if n_epochs > 10 else (500 if n <= 10000 else 200)


def epochs_per_sample(w, n: int, n_epochs: int, prune_epochs: int | None = None):
    """umap_wmax_kernel + umap_eps_kernel: fp32 eps per stored arc, 0 = never sampled."""
    w = np.asarray(w, dtype=np.float32)
    if prune_epochs is None:
        prune_epochs = prune_epochs_for(n, n_epochs)
    wmax = np.float32(max(float(w.max()) if w.size else 0.0, 0.0))
    eps = np.zeros(w.shape, np.float32)
    if wmax > 0:
        keep = (w > 0) & (w >= wmax / np.float32(prune_epochs))
        eps[keep] = wmax / w[keep]
    return eps


def rescale(init, dtype=np.float32):
    """umap_rescale_kernel mode 0 in fp32 (min / max over the finite values of each column)."""
    x = np.array(init, dtype=np.float32)
    out = np.zeros_like(x)
    for d in range(x.shape[1]):
        col = x[:, d]
        fin = col[np.isfinite(col)]
        if fin.size == 0:
            continue
        lo, hi = fin.min(), fin.max()
        if hi > lo:
            out[:, d] = np.float32(10.0) * (col - lo) / (hi - lo)
    return out.astype(dtype)


@numba.njit(cache=False, inline="always")
def _hash32(x):
    x ^= x >> _S16
    x = (x * _H1) & M32
    x ^= x >> _S15
    x = (x * _H2) & M32
    x ^= x >> _S16
    return x


@numba.njit(cache=False, inline="always")
def _clip4(v, four):
    if v > four:
        return four
    if v < -four:
        return -four
    return v


@numba.njit(cache=False, inline="always")
def _sampled(nd, epd):
    """Closed form of umap's epoch_of_next_sample: the cnt-th sample of an arc falls in epoch ceil(cnt * eps)."""
    cnt = math.floor(nd / epd)
    return cnt, cnt >= 1 and math.floor((nd - 1.0) / epd) < cnt


@numba.njit(cache=False, inline="always")
def _n_neg(nd, epd, cnt, neg_rate, delta, rate_first=False):
    """Negative samples owed since the previous sample of the arc (epoch_of_next_negative_sample), clamped to 64.
    rate_first: the rounding the kernel once had, floor(epoch * (rate / eps)), which loses a sample when eps divides
    epoch * rate but rate / eps rounds down (eps = 5, rate = 7, epoch 45)."""
    if rate_first:
        r = neg_rate / epd
        c_now = math.floor(nd * r)
        c_prev = 1
        if cnt > 1:
            c_prev = math.floor(math.ceil((cnt - 1) * epd) * r)
        if c_prev < 1:
            c_prev = 1
        return min(MAX_NEG, max(0, c_now - c_prev + delta))
    c_now = math.floor(nd * neg_rate / epd)
    c_prev = 1
    if cnt > 1:
        c_prev = math.floor(math.ceil((cnt - 1) * epd) * neg_rate / epd)
    if c_prev < 1:
        c_prev = 1
    return min(MAX_NEG, max(0, c_now - c_prev + delta))


@numba.njit(cache=False)
def _epoch(indptr, indices, eps, pos_in, pos_out, epoch, alpha, a, b, gamma, neg_rate, sd, K, pulls, neg_delta,
           gauss_seidel, rate_first):
    """One launch of umap_epoch_kernel.  K = [0, 1, 2, 4, 0.001f] in the working dtype."""
    n, dim = pos_in.shape
    zero, one, two, four, c001 = K[0], K[1], K[2], K[3], K[4]
    src = pos_out if gauss_seidel else pos_in
    if gauss_seidel:
        pos_out[:] = pos_in
    nd = float(epoch)
    cur = np.empty(dim, pos_in.dtype)
    oth = np.empty(dim, pos_in.dtype)
    df = np.empty(dim, pos_in.dtype)
    ep_mix = (np.uint64(epoch) * _GOLD) & M32
    nn = np.uint64(n)
    for j in range(n):
        for d in range(dim):
            cur[d] = pos_in[j, d]
        for e in range(indptr[j], indptr[j + 1]):
            ep = eps[e]
            if ep <= 0.0:
                continue
            epd = float(ep)
            cnt, hit = _sampled(nd, epd)
            if not hit:
                continue
            k = indices[e]
            for d in range(dim):
                oth[d] = src[k, d]
            for _rep in range(pulls):
                d2 = zero
                for d in range(dim):
                    t = cur[d] - oth[d]
                    d2 += t * t
                if d2 > zero:
                    pb = d2 ** b
                    gc = -two * a * b * (pb / d2) / (a * pb + one)
                    for d in range(dim):
                        cur[d] += _clip4(gc * (cur[d] - oth[d]), four) * alpha
            n_neg = _n_neg(nd, epd, cnt, neg_rate, neg_delta, rate_first)
            h = _hash32(sd ^ _hash32((ep_mix + (np.uint64(e) & M32)) & M32))
            for p in range(n_neg):
                h = _hash32((h + _STEP * np.uint64(p + 1)) & M32)
                kk = np.int64((h * nn) >> _S32)
                if kk == j:
                    continue
                d2 = zero
                for d in range(dim):
                    df[d] = cur[d] - src[kk, d]
                    d2 += df[d] * df[d]
                if d2 > zero:
                    gc = two * gamma * b / ((c001 + d2) * (a * d2 ** b + one))
                    if gc > zero:
                        for d in range(dim):
                            cur[d] += _clip4(gc * df[d], four) * alpha
        for d in range(dim):
            pos_out[j, d] = cur[d]


def umap_layout(adj, init, *, n_epochs: int, a: float, b: float, gamma: float = 1.0, initial_alpha: float = 1.0,
                negative_sample_rate: int = 5, seed: int = 0, dtype=np.float64, pulls: int = 2, neg_delta: int = 0,
                alpha_shift: int = 0, gauss_seidel: bool = False, prune_epochs: int | None = None,
                rate_first: bool = False):
    """sb2_umap_layout_f32 on a scipy CSR graph (stored arcs in stored order, explicit zeros included) -> [n, dim] dtype."""
    indptr = np.asarray(adj.indptr, dtype=np.int64)
    indices = np.asarray(adj.indices, dtype=np.int64)
    n = adj.shape[0]
    x = rescale(init, dtype)
    if adj.nnz == 0 or n_epochs == 0:
        return x
    eps = epochs_per_sample(adj.data, n, n_epochs, prune_epochs)
    f32 = np.float32
    # the device converts a, b, gamma, alpha0 and 0.001 to fp32; the float64 restatement works on those same values
    a_, b_, g_ = (dtype(f32(v)) for v in (a, b, gamma))
    K = np.array([0.0, 1.0, 2.0, 4.0, f32(0.001)], dtype=dtype)
    sd = np.uint64(seed_mix(seed))
    y = np.empty_like(x)
    for ep in range(n_epochs):
        e_ = ep + alpha_shift
        if dtype == np.float32:
            alpha = f32(initial_alpha) * (f32(1.0) - f32(e_) / f32(n_epochs))
        else:
            alpha = float(f32(initial_alpha)) * (1.0 - e_ / n_epochs)
        _epoch(indptr, indices, eps, x, y, ep, dtype(alpha), a_, b_, g_, float(negative_sample_rate), sd, K, pulls,
               neg_delta, gauss_seidel, rate_first)
        x, y = y, x
    return x


def edge_case_graph(n: int, seed: int = 0, k: int = 10, hub_degree: int = 0):
    """A symmetric fp32 kNN graph (exp(-d / median d) weights, max-symmetrised) on clustered 5-D points, with the rows the
    kernel must get right: vertex 0 isolated (empty row), arcs of weight wmax = 1 and of exact divisors of it (1/2, 1/3,
    1/5, 1/10), arcs below every pruning threshold (wmax / 1000), stored explicit zeros, and, if hub_degree > 0, vertex 1
    joined to hub_degree random vertices (a row much longer than the average)."""
    from scipy import sparse
    from sklearn.neighbors import NearestNeighbors

    rng = np.random.default_rng(seed)
    cent = rng.normal(size=(8, 5)) * 3.0
    x = cent[rng.integers(0, 8, n)] + rng.normal(size=(n, 5))
    dist, idx = NearestNeighbors(n_neighbors=k + 1).fit(x).kneighbors(x)
    d, nb = dist[:, 1:].ravel(), idx[:, 1:].ravel()
    rows = np.repeat(np.arange(n), k)
    g = sparse.csr_matrix((np.exp(-d / np.median(d)), (rows, nb)), shape=(n, n))
    if hub_degree:
        hv = rng.choice(np.arange(2, n), hub_degree, replace=False)
        g = g + sparse.csr_matrix((rng.uniform(0.05, 0.9, hub_degree), (np.ones(hub_degree, int), hv)), shape=(n, n))
    g = g.maximum(g.T).tocsr()
    keep = np.ones(n)
    keep[0] = 0.0
    g = (sparse.diags(keep) @ g @ sparse.diags(keep)).tocsr()
    g.eliminate_zeros()
    g.sort_indices()
    g = g.astype(np.float32)
    g.data *= np.float32(0.9 / g.data.max())
    # overwrite whole symmetric pairs: a random arc (i, j) and its mirror (j, i)
    upper = np.flatnonzero(np.repeat(np.arange(n), np.diff(g.indptr)) < g.indices)
    pick = rng.choice(upper, 5 * 8 * max(1, n // 500), replace=False).reshape(5, -1)
    special = {0: np.float32(1.0), 1: np.float32(0.5), 2: np.float32(1 / 3), 3: np.float32(0.2), 4: np.float32(0.1)}
    vals = np.empty(pick.shape, np.float32)
    for r, v in special.items():
        vals[r] = v
    vals[4, ::2] = np.float32(1e-3)  # below wmax / 500
    vals[3, ::4] = np.float32(0.0)   # explicit zeros
    row_of = np.repeat(np.arange(n), np.diff(g.indptr))
    for arc, v in zip(pick.ravel(), vals.ravel()):
        i, j = row_of[arc], g.indices[arc]
        g.data[arc] = v
        lo, hi = g.indptr[j], g.indptr[j + 1]
        g.data[lo + np.searchsorted(g.indices[lo:hi], i)] = v
    return g


def tolerance(r32, r64) -> float:
    """Max-abs tolerance of a device layout against the float64 restatement (see TOL_FACTOR)."""
    spread = float(np.abs(np.asarray(r32, np.float64) - np.asarray(r64, np.float64)).max(initial=0.0))
    return max(TOL_FACTOR * spread, TOL_FLOOR)


# ------------------------------------------------------------------------------------------ sampling schedules
@numba.njit(cache=False)
def closed_form_schedule(eps, n_epochs, neg_rate):
    """The kernel's schedule -> (sampled bool [arcs, n_epochs], n_neg int64 [arcs, n_epochs])."""
    m = eps.shape[0]
    sampled = np.zeros((m, n_epochs), np.bool_)
    n_neg = np.zeros((m, n_epochs), np.int64)
    for e in range(m):
        if eps[e] <= 0.0:
            continue
        epd = float(eps[e])
        for ep in range(n_epochs):
            cnt, hit = _sampled(float(ep), epd)
            if hit:
                sampled[e, ep] = True
                n_neg[e, ep] = _n_neg(float(ep), epd, cnt, float(neg_rate), 0)
    return sampled, n_neg


def umap_epochs_per_sample(w, n_epochs: int, prune_epochs: int):
    """umap's pruning plus make_epochs_per_sample: n_samples = n_epochs w / wmax in fp32, eps = n_epochs / n_samples in
    float64; -1 = never sampled."""
    w = np.asarray(w, dtype=np.float32)
    wmax = w.max()
    w = np.where(w < wmax / np.float32(prune_epochs), np.float32(0), w)
    n_samples = n_epochs * (w / wmax)
    eps = np.full(w.shape, -1.0)
    pos = n_samples > 0
    eps[pos] = float(n_epochs) / n_samples[pos].astype(np.float64)
    return eps


@numba.njit(cache=False)
def running_counter_schedule(eps, n_epochs, neg_rate):
    """The bookkeeping of oracle.graph_tools._optimize without the forces -> (sampled, n_neg) like closed_form_schedule."""
    m = eps.shape[0]
    sampled = np.zeros((m, n_epochs), np.bool_)
    n_neg = np.zeros((m, n_epochs), np.int64)
    eps_neg = eps / neg_rate
    eonns = eps_neg.copy()
    eons = eps.copy()
    for n in range(n_epochs):
        for i in range(m):
            if eps[i] > 0 and eons[i] <= n:
                sampled[i, n] = True
                eons[i] += eps[i]
                c = int((n - eonns[i]) / eps_neg[i])
                n_neg[i, n] = c
                eonns[i] += c * eps_neg[i]
    return sampled, n_neg

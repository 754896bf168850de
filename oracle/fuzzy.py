"""`fuzzy_simplicial_set` oracle (test infrastructure only; see oracle/__init__.py).

Restates umap-learn (>= 0.5.12, pyproject.toml:76 of the reference; NOT vendored under
/root/reference and not installed here) `umap.umap_.smooth_knn_dist`,
`compute_membership_strengths` and `fuzzy_simplicial_set`, exactly as the reference calls
them from src/scanpy/neighbors/_connectivity.py:124-138:

    fuzzy_simplicial_set(coo((n,1)), n_neighbors, None, None, knn_indices=..., knn_dists=...,
                         set_op_mix_ratio=1.0, local_connectivity=1.0)  ->  .tocsr()

Numerics follow umap's numba code: knn_dists are cast to float32; rho for a fractional
local_connectivity is formed in float64 and rounded once; the sigma bisection runs
in float64 scalars (numba types the Python floats lo/mid/hi as float64) and stores float32;
membership strengths are float32.  The means of the sigma floor are summed in float64 (numba sums
`np.mean` of a float32 array in float32, so a floored sigma can differ from umap's by a few float32
ulps).  The row loop is vectorised over rows with numpy (each row's bisection is independent; rows
that hit the tolerance are frozen, as `break` does).

Pinned against: tests/test_neighbors.py:43-48 (`connectivities_umap`, 4 points) and the in-tree
pbmc68k fixture (obsp/distances -> obsp/connectivities), see tests/test_oracle_goldens.py.
"""
from __future__ import annotations

import numpy as np
from scipy import sparse

SMOOTH_K_TOLERANCE = 1e-5
MIN_K_DIST_SCALE = 1e-3


def smooth_knn_dist(distances: np.ndarray, k: float, *, n_iter: int = 64,
                    local_connectivity: float = 1.0, bandwidth: float = 1.0):
    """-> (sigmas float32[n], rhos float32[n], margin float64[n]).  distances: float32 [n, K], rows in any order.

    margin[i] is the smallest distance of row i's bisection from one of its decisions: the minimum over the
    iterations run of |psum - target| (the `psum > target` branch) and of ||psum - target| - 1e-5| (the stopping
    test).  An implementation whose psum differs by less than that takes every decision the same way, so it ends
    on the same mid, bit for bit."""
    distances = np.asarray(distances, np.float32)
    n, K = distances.shape
    target = np.log2(k) * bandwidth
    rho = np.zeros(n, np.float32)
    mean_distances = float(np.mean(distances.astype(np.float64)))

    # rho: umap_.py smooth_knn_dist, the `non_zero_dists` block.  numba types `interpolation` as float64 and the
    # difference of two float32 distances as float32; the product and sum are float64, rounded once into rho[i]
    index = int(np.floor(local_connectivity))
    interpolation = float(local_connectivity) - index
    nzmask = distances > 0.0
    nnz = nzmask.sum(axis=1)
    # position (within the row) of the m-th non-zero entry, m = 0..: use a stable argsort of ~mask
    order = np.argsort(~nzmask, axis=1, kind="stable")
    nz_sorted = np.take_along_axis(distances, order, axis=1)  # non-zeros first, original order
    enough = nnz >= local_connectivity
    if index > 0:
        r = nz_sorted[:, index - 1].copy()
        if interpolation > SMOOTH_K_TOLERANCE:
            nxt = nz_sorted[:, min(index, K - 1)]
            r = (r.astype(np.float64) + interpolation * (nxt - r).astype(np.float64)).astype(np.float32)
    else:
        r = (interpolation * nz_sorted[:, 0].astype(np.float64)).astype(np.float32)
    rho[enough] = r[enough]
    some = (~enough) & (nnz > 0)
    if some.any():
        rho[some] = np.where(nzmask[some], distances[some], -np.inf).max(axis=1)

    lo = np.zeros(n, np.float64)
    hi = np.full(n, np.inf, np.float64)
    mid = np.ones(n, np.float64)
    active = np.ones(n, bool)
    margin = np.full(n, np.inf)
    d = distances[:, 1:].astype(np.float32) - rho[:, None]  # float32 subtraction as in numba
    d64 = d.astype(np.float64)
    pos = d > 0
    for _ in range(n_iter):
        if not active.any():
            break
        a = active
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            e = np.where(pos[a], np.exp(-(d64[a] / mid[a, None])), 1.0)
        psum = e.sum(axis=1)
        gap = np.abs(psum - target)
        margin[a] = np.minimum(margin[a], np.minimum(gap, np.abs(gap - SMOOTH_K_TOLERANCE)))
        done = gap < SMOOTH_K_TOLERANCE
        ia = np.flatnonzero(a)
        active[ia[done]] = False
        ia, psum = ia[~done], psum[~done]
        gt = psum > target
        # psum > target: hi = mid; mid = (lo+hi)/2
        i_gt = ia[gt]
        hi[i_gt] = mid[i_gt]
        mid[i_gt] = (lo[i_gt] + hi[i_gt]) / 2.0
        # else: lo = mid; mid = mid*2 if hi is inf else (lo+hi)/2
        i_le = ia[~gt]
        lo[i_le] = mid[i_le]
        inf = np.isinf(hi[i_le])
        mid[i_le[inf]] *= 2.0
        fin = i_le[~inf]
        mid[fin] = (lo[fin] + hi[fin]) / 2.0
    result = mid.astype(np.float32)

    mean_ith = distances.astype(np.float64).mean(axis=1)
    floor = np.where(rho > 0.0, MIN_K_DIST_SCALE * mean_ith, MIN_K_DIST_SCALE * mean_distances)
    low = result < floor
    result[low] = floor[low].astype(np.float32)
    return result, rho, margin


def compute_membership_strengths(knn_indices, knn_dists, sigmas, rhos):
    """-> (rows, cols, vals float32) of length n*K (umap_.py compute_membership_strengths)."""
    knn_dists = np.asarray(knn_dists, np.float32)
    n, K = knn_indices.shape
    rows = np.repeat(np.arange(n, dtype=np.int64), K)
    cols = knn_indices.astype(np.int64).ravel()
    diff = knn_dists - rhos[:, None].astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        val = np.exp(-(diff / sigmas[:, None].astype(np.float32))).astype(np.float32)
    val = np.where((diff <= 0.0) | (sigmas[:, None] == 0.0), np.float32(1.0), val)
    val = np.where(knn_indices == np.arange(n)[:, None], np.float32(0.0), val).astype(np.float32)
    keep = cols >= 0  # -1 marks a missing neighbour
    return rows[keep], cols[keep], val.ravel()[keep]


def fuzzy_simplicial_set(knn_indices, knn_dists, n_obs: int, n_neighbors: int, *,
                         set_op_mix_ratio: float = 1.0, local_connectivity: float = 1.0):
    """-> scipy CSR float32, symmetric, zeros eliminated (what `umap()` returns at _connectivity.py:138)."""
    knn_dists = np.asarray(knn_dists).astype(np.float32)
    sigmas, rhos, _ = smooth_knn_dist(knn_dists, float(n_neighbors), local_connectivity=float(local_connectivity))
    rows, cols, vals = compute_membership_strengths(knn_indices, knn_dists, sigmas, rhos)
    result = sparse.coo_matrix((vals, (rows, cols)), shape=(n_obs, n_obs))
    result.eliminate_zeros()
    transpose = result.transpose()
    prod = result.multiply(transpose)
    result = set_op_mix_ratio * (result + transpose - prod) + (1.0 - set_op_mix_ratio) * prod
    result.eliminate_zeros()
    return result.tocsr().astype(np.float32), sigmas, rhos

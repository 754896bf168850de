"""k-lists built directly in numpy for the connectivity tests (tests/test_connectivity_host_cpu.py on the host,
tests/test_gpu_connectivity_exact.py on the device), and the restatements both compare against.

`fuzzy_case` cycles every row through one of the shapes the fuzzy-set kernel must handle; `umap_smooth_knn_dist` and
`umap_membership` transcribe umap-learn's numba loops row by row, with numba's scalar types written out."""
from __future__ import annotations

from functools import lru_cache

import numpy as np
from scipy import sparse

KINDS = ("ascending", "storage order", "leading zeros", "all zero", "all at rho", "ties at rho", "-1 ids",
         "self not first", "self absent")


def _neighbours(rs, n, i, m):
    """m distinct ids other than i, mostly from a window around i so that many edges are mutual."""
    if n - 1 <= m:
        out = np.delete(np.arange(n), i)
        return np.r_[rs.permutation(out), -np.ones(m - len(out), int)]
    w = min(n - 1, 2 * m + 2)
    off = rs.choice(np.r_[np.arange(-(w // 2), 0), np.arange(1, w - w // 2 + 1)], m, replace=False)
    ids = (i + off) % n
    if len(set(ids.tolist())) < m:  # the window wrapped onto itself
        ids = rs.choice(np.delete(np.arange(n), i), m, replace=False)
    return ids


@lru_cache(maxsize=None)
def fuzzy_case(n: int, k: int, seed: int = 0):
    """-> (idx int32 [n, k], dist float64 [n, k]); row i has shape KINDS[i % 9].  Rows never repeat an id; ids run
    out (-1) when n <= k."""
    rs = np.random.RandomState(1000 * k + n + seed)
    idx = np.empty((n, k), np.int64)
    dist = np.empty((n, k))
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        nb = _neighbours(rs, n, i, k - 1)
        d = np.sort(rs.uniform(0.5, 1.5, k - 1)) * rs.uniform(0.2, 5.0)
        row_i, row_d = np.r_[i, nb], np.r_[0.0, d]
        if kind == "storage order":
            p = rs.permutation(k - 1)
            row_i[1:], row_d[1:] = nb[p], d[p]
        elif kind == "leading zeros":
            row_d[1:1 + min(2, k - 1)] = 0.0
        elif kind == "all zero":
            row_d[:] = 0.0
        elif kind == "all at rho":
            row_d[1:] = d[0]
        elif kind == "ties at rho":
            row_d[1:1 + min(3, k - 1)] = d[0]
        elif kind == "-1 ids":
            c = max(1, (k - 1) // 3)
            row_i[k - c:] = -1
        elif kind == "self not first" and k >= 2 and nb[0] >= 0:
            row_i[0], row_i[1] = nb[0], i
            row_d[1] = 0.0
        elif kind == "self absent":
            extra = [j for j in _neighbours(rs, n, i, min(n - 1, k + 2)) if j >= 0 and j not in set(nb.tolist())]
            if extra:
                row_i[0], row_d[0] = extra[0], d[0] * 0.9
        row_i[row_i < 0] = -1
        idx[i], dist[i] = row_i, row_d
    return idx.astype(np.int32), dist


# ------------------------------------------------------------------------------------------ umap-learn, row by row
SMOOTH_K_TOLERANCE, MIN_K_DIST_SCALE = 1e-5, 1e-3


def _numba_mean_f32(a):
    """numba's np.mean of a float32 array: a float32 accumulator, then the float64 quotient."""
    c = np.float32(0.0)
    for v in np.asarray(a, np.float32).ravel():
        c = np.float32(c + v)
    return float(c) / a.size


def umap_smooth_knn_dist(distances, k, *, n_iter=64, local_connectivity=1.0):
    """umap_.py smooth_knn_dist.  Scalar types as numba infers them: distances, rho and result are float32, a float32
    minus a float32 is float32, anything with lo / mid / hi / interpolation is float64."""
    distances = np.asarray(distances, np.float32)
    target = np.log2(k)
    rho = np.zeros(distances.shape[0], np.float32)
    result = np.zeros(distances.shape[0], np.float32)
    mean_distances = _numba_mean_f32(distances)
    for i in range(distances.shape[0]):
        lo, hi, mid = 0.0, np.inf, 1.0
        ith = distances[i]
        nz = ith[ith > 0.0]
        if nz.shape[0] >= local_connectivity:
            index = int(np.floor(local_connectivity))
            interpolation = float(local_connectivity) - index
            if index > 0:
                rho[i] = nz[index - 1]
                if interpolation > SMOOTH_K_TOLERANCE:
                    rho[i] = np.float32(float(rho[i]) + interpolation * float(np.float32(nz[index] - nz[index - 1])))
            else:  # an all-zero row at local_connectivity 0 reads nz[0] out of bounds in numba; kernel and oracle use 0
                rho[i] = np.float32(interpolation * float(nz[0] if nz.shape[0] else 0.0))
        elif nz.shape[0] > 0:
            rho[i] = np.max(nz)
        for _ in range(n_iter):
            psum = 0.0
            for j in range(1, distances.shape[1]):
                d = np.float32(distances[i, j] - rho[i])
                psum += float(np.exp(-(float(d) / mid))) if d > 0 else 1.0
            if abs(psum - target) < SMOOTH_K_TOLERANCE:
                break
            if psum > target:
                hi = mid
                mid = (lo + hi) / 2.0
            else:
                lo = mid
                mid = mid * 2 if hi == np.inf else (lo + hi) / 2.0
        result[i] = mid
        if rho[i] > 0.0:
            mean_ith = _numba_mean_f32(ith)
            if float(result[i]) < MIN_K_DIST_SCALE * mean_ith:
                result[i] = MIN_K_DIST_SCALE * mean_ith
        elif float(result[i]) < MIN_K_DIST_SCALE * mean_distances:
            result[i] = MIN_K_DIST_SCALE * mean_distances
    return result, rho


def umap_membership(knn_indices, knn_dists, sigmas, rhos, n, *, set_op_mix_ratio=1.0):
    """compute_membership_strengths (float32 values; -1 skipped, self 0) and fuzzy_simplicial_set's union."""
    knn_dists = np.asarray(knn_dists, np.float32)
    rows, cols, vals = [], [], []
    for i in range(knn_indices.shape[0]):
        for j in range(knn_indices.shape[1]):
            nb = knn_indices[i, j]
            if nb == -1:
                continue
            diff = np.float32(knn_dists[i, j] - rhos[i])
            if nb == i:
                val = np.float32(0.0)
            elif diff <= 0.0 or sigmas[i] == 0.0:
                val = np.float32(1.0)
            else:
                val = np.exp(-np.float32(diff / sigmas[i]))
            rows.append(i), cols.append(nb), vals.append(val)
    r = sparse.coo_matrix((np.array(vals, np.float32), (rows, cols)), shape=(n, n))
    r.eliminate_zeros()
    t = r.transpose()
    p = r.multiply(t)
    r = set_op_mix_ratio * (r + t - p) + (1.0 - set_op_mix_ratio) * p
    r.eliminate_zeros()
    return r.tocsr()

"""`method='gauss'` / `method='jaccard'` connectivities oracle (test infrastructure only; SURVEY 8f row f3).

numpy restatements of src/scanpy/neighbors/_connectivity.py:17-100 (gauss, the sparse kNN branch that
`sc.pp.neighbors(method='gauss', knn=True)` takes) and :141-186 (jaccard).  Pinned by the reference's 4-point goldens
`connectivities_gauss_knn` / `connectivities_jaccard` (tests/test_neighbors.py:66-72,120-126,195-226).

`gauss_reference` is the whole of the reference's `gauss(distances, n_neighbors, knn=True)`, CSR and dense branch,
with the k-list extraction of src/scanpy/neighbors/_common.py:63-143 it calls; `gauss_knn` is its CSR branch on rows
that store exactly n_neighbors - 1 distances.
"""
from __future__ import annotations

import numpy as np
from scipy import sparse


def gauss_knn(knn_indices, knn_dists):
    """knn_indices/knn_dists [n,k] with self in column 0 -> CSR of gaussian weights, 'copy if missing' symmetrised."""
    n, k = knn_indices.shape
    idx = knn_indices[:, 1:]
    d_sq = np.asarray(knn_dists, np.float64)[:, 1:] ** 2
    sigmas_sq = np.median(d_sq, axis=1)
    sigmas = np.sqrt(sigmas_sq)
    num = 2 * sigmas[:, None] * sigmas[idx]
    den = sigmas_sq[:, None] + sigmas_sq[idx]
    w = np.sqrt(num / den) * np.exp(-d_sq / den)
    m = sparse.lil_matrix((n, n))
    for i in range(n):
        for j, v in zip(idx[i], w[i]):
            m[i, j] = v
    sets = [set(r.tolist()) for r in idx]
    for i in range(n):
        for j, v in zip(idx[i], w[i]):
            if i not in sets[j]:
                m[j, i] = v
    return m.tocsr()


def jaccard(knn_indices):
    n, k = knn_indices.shape
    adjacency = sparse.csr_matrix((np.ones(n * (k - 1)), knn_indices[:, 1:].ravel(), np.arange(0, n * (k - 1) + 1, k - 1)),
                                  shape=(n, n))
    i_idx = np.repeat(np.arange(n), k - 1)
    j_idx = knn_indices[:, 1:].ravel()
    shared = np.asarray(adjacency[i_idx, :].multiply(adjacency[j_idx, :]).sum(axis=1)).ravel()
    jac = shared / (2 * (k - 1) - shared)
    mask = jac != 0
    c = sparse.csr_matrix((jac[mask], (i_idx[mask], j_idx[mask])), shape=(n, n))
    return (c + c.T) / 2


def _ind_dist_from_sparse(d, n_neighbors: int):
    """src/scanpy/neighbors/_common.py:74-143: the constant-nnz shortcut or the slow path, then the self column and
    the truncation to n_neighbors.  The slow path raises ValueError on a row shorter than n_neighbors - 1 (other than
    a one-entry row, which broadcasts), as the reference's does."""
    n = d.shape[0]
    nnzs = d.getnnz(axis=1)
    if (nnzs == nnzs[0]).all():
        indices, distances = d.indices.reshape(n, int(nnzs[0])), d.data.reshape(n, int(nnzs[0]))
    else:
        indices = np.zeros((n, n_neighbors), dtype=int)
        distances = np.zeros((n, n_neighbors), dtype=d.dtype)
        for i in range(n):
            neighbors = d[i].nonzero()
            indices[i, 0] = i
            distances[i, 0] = 0
            if len(neighbors[1]) > n_neighbors - 1:
                sorted_indices = np.argsort(np.asarray(d[i][neighbors]).ravel())[: n_neighbors - 1]
                indices[i, 1:] = neighbors[1][sorted_indices]
                distances[i, 1:] = np.asarray(d[i][neighbors[0][sorted_indices], neighbors[1][sorted_indices]]).ravel()
            else:
                indices[i, 1:] = neighbors[1]
                distances[i, 1:] = np.asarray(d[i][neighbors]).ravel()
    if not (indices[:, 0] == np.arange(n)).any():
        indices = np.hstack([np.arange(n)[:, None], indices])
        distances = np.hstack([np.zeros(n)[:, None], distances])
    if indices.shape[1] > n_neighbors:
        indices, distances = indices[:, :n_neighbors], distances[:, :n_neighbors]
    return indices, distances


def gauss_reference(distances, n_neighbors: int):
    """_connectivity.py:17-100 with knn=True -> CSR (sparse input) or dense ndarray (dense input)."""
    is_csr = sparse.issparse(distances)
    if is_csr:
        distances = sparse.csr_matrix(distances)
        d_sq = distances.power(2)
        indices, distances_sq = _ind_dist_from_sparse(d_sq, n_neighbors)
    else:
        d_sq = np.power(distances, 2)
        rows = np.arange(d_sq.shape[0])[:, None]
        indices = np.argpartition(d_sq, n_neighbors - 1, axis=1)[:, :n_neighbors]
        indices = indices[rows, np.argsort(d_sq[rows, indices])]
        distances_sq = d_sq[rows, indices]
    indices = indices[:, 1:]
    distances_sq = distances_sq[:, 1:]
    sigmas_sq = np.median(distances_sq, axis=1) if is_csr else distances_sq[:, -1] / 4
    sigmas = np.sqrt(sigmas_sq)
    if not is_csr:
        num = 2 * np.multiply.outer(sigmas, sigmas)
        den = np.add.outer(sigmas_sq, sigmas_sq)
        w = np.sqrt(num / den) * np.exp(-d_sq / den)
        mask = np.zeros(d_sq.shape, dtype=bool)
        for i, row in enumerate(indices):
            mask[i, row] = True
            for j in row:
                if i not in set(indices[j]):
                    w[j, i] = w[i, j]
                    mask[j, i] = True
        w[~mask] = 0
        return w
    w = d_sq.copy()
    for i in range(len(d_sq.indptr[:-1])):
        row = d_sq.indices[d_sq.indptr[i]: d_sq.indptr[i + 1]]
        num = 2 * sigmas[i] * sigmas[row]
        den = sigmas_sq[i] + sigmas_sq[row]
        w.data[d_sq.indptr[i]: d_sq.indptr[i + 1]] = np.sqrt(num / den) * np.exp(-d_sq.data[d_sq.indptr[i]: d_sq.indptr[i + 1]] / den)
    w = w.tolil()
    for i, row in enumerate(indices):
        for j in row:
            if i not in set(indices[j]):
                w[j, i] = w[i, j]
    return w.tocsr()

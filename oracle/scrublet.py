"""sc.pp.scrublet oracle (test infrastructure only): an fp64 numpy / scipy / sklearn restatement of the reference path.

  filters, normalize_total, log1p, seurat HVG   oracle.preprocess (src/scanpy/preprocessing/_scrublet/__init__.py:186-227)
  doublets                                      scipy's `x[p0] + x[p1]` (core.py:219-237)
  z-score, PCA(arpack) / TruncatedSVD(arpack)   pipeline.py:18-89, on the dense float64 matrices
  neighbours                                    exact brute force: self, then the k_adj - 1 nearest other points in
                                                (fp64 squared distance, id) order, the squared distance summed over the
                                                columns in order (the order csrc/scrublet.cu defines)
  scores and calls                              core.py:363-474, with scanpy_b200._scrublet's host pieces
"""
from __future__ import annotations

import numpy as np
from scipy import sparse

from oracle import preprocess as opp
from scanpy_b200._scrublet import (doublet_scores, k_adjusted, n_neighbors_default, neighbor_parents, sample_comb,
                                   threshold_minimum)


def filter_genes_cells(x):
    """filter_genes(min_cells=3) then filter_cells(min_genes=3) -> (x, kept cell positions)."""
    x = sparse.csr_matrix(x)
    x = x[:, np.asarray((x > 0).sum(axis=0)).ravel() >= 3]
    keep = np.flatnonzero(np.asarray((x > 0).sum(axis=1)).ravel() >= 3)
    return x[keep], keep


def simulate(x, sim_doublet_ratio, rng):
    x = sparse.csr_matrix(x)
    pairs = sample_comb(x.shape[0], int(x.shape[0] * sim_doublet_ratio), rng)
    return (x[pairs[:, 0]] + x[pairs[:, 1]]).tocsr(), pairs


def preprocess(x_raw, *, sim_doublet_ratio=2.0, log_transform=False, rng):
    """-> (x_obs, x_sim, parents, kept cell positions) ready for `call_doublets`."""
    x, keep = filter_genes_cells(x_raw)
    raw = x.copy()
    xn, _, _ = opp.normalize_total(x)
    hvg = opp.hvg_seurat(opp.log1p(xn))["highly_variable"].to_numpy()
    x_obs = xn[:, hvg]
    x_sim, parents = simulate(raw[:, hvg], sim_doublet_ratio, rng)
    if log_transform:
        x_obs, x_sim = opp.log1p(x_obs), opp.log1p(x_sim)
    x_obs = opp.normalize_total(x_obs, target_sum=1e6)[0]
    x_sim = opp.normalize_total(x_sim, target_sum=1e6)[0]
    return x_obs, x_sim, parents, keep


def embed(x_obs, x_sim, *, mean_center=True, normalize_variance=True, n_prin_comps=30):
    from sklearn.decomposition import PCA, TruncatedSVD

    mean, var = opp.mean_var_cols(sparse.csr_matrix(x_obs))
    sigma = np.sqrt(var) if normalize_variance else np.ones_like(var)
    a = np.asarray(x_obs.toarray(), dtype=np.float64)
    b = np.asarray(x_sim.toarray(), dtype=np.float64)
    if mean_center:
        a, b = (a - mean) * (1 / sigma), (b - mean) * (1 / sigma)
        pca = PCA(n_components=n_prin_comps, svd_solver="arpack", random_state=0).fit(a)
        return np.vstack([pca.transform(a), pca.transform(b)])
    a, b = a * (1 / sigma), b * (1 / sigma)
    svd = TruncatedSVD(n_components=n_prin_comps, algorithm="arpack", random_state=0).fit(a)
    return np.vstack([svd.transform(a), svd.transform(b)])


def sq_dists(x, i):
    """fp64 squared distances of point i to all points, summed over the columns in order, each step rounded."""
    x = np.asarray(x, dtype=np.float64)
    acc = np.zeros(x.shape[0])
    for j in range(x.shape[1]):
        t = x[:, j] - x[i, j]
        acc = acc + t * t
    return acc


def label_count(x, n_first, k, rows=None):
    """-> (count, kth distance, neighbour ids [rows x k] self first then ascending (distance, id), relative gap
    between the (k-1)-th and the k-th other neighbour's squared distance (inf when there is no k-th))."""
    n = x.shape[0]
    rows = np.arange(n) if rows is None else np.asarray(rows)
    count = np.empty(len(rows), np.int64)
    kth = np.empty(len(rows))
    ids = np.empty((len(rows), k), np.int64)
    gap = np.empty(len(rows))
    for r, i in enumerate(rows):
        d = sq_dists(x, i)
        others = np.delete(np.arange(n), i)
        order = others[np.lexsort((others, d[others]))]
        ids[r] = np.concatenate([[i], order[:k - 1]])
        count[r] = int((ids[r] >= n_first).sum())
        kth[r] = np.sqrt(d[order[k - 2]]) if k > 1 else 0.0
        if k > 1 and k - 1 < len(order):
            lo, hi = d[order[k - 2]], d[order[k - 1]]
            gap[r] = (hi - lo) / max(hi, 1e-300)
        else:
            gap[r] = np.inf
    return count, kth, ids, gap


def call_doublets(x_obs, x_sim, parents, *, n_neighbors=None, expected_doublet_rate=0.05, stdev_doublet_rate=0.02,
                  mean_center=True, normalize_variance=True, n_prin_comps=30, threshold=None, embedding=None):
    """-> dict(doublet_score, predicted_doublet, doublet_scores_sim, threshold (None if not found), k, k_adj, count,
    gap, ids, embedding, doublet_neighbor_parents)."""
    n_obs, n_sim = x_obs.shape[0], x_sim.shape[0]
    k = n_neighbors_default(n_obs) if n_neighbors is None else n_neighbors
    k_adj = k_adjusted(k, n_obs, n_sim)
    emb = embed(x_obs, x_sim, mean_center=mean_center, normalize_variance=normalize_variance,
                n_prin_comps=n_prin_comps) if embedding is None else embedding
    count, _, ids, gap = label_count(emb, n_obs, k_adj)
    ld, _ = doublet_scores(count, k_adj=k_adj, n_obs=n_obs, n_sim=n_sim, expected_doublet_rate=expected_doublet_rate,
                           stdev_doublet_rate=stdev_doublet_rate)
    if threshold is None:
        try:
            threshold = threshold_minimum(ld[n_obs:])
        except RuntimeError:
            threshold = None
    pred = np.zeros(n_obs, bool) if threshold is None else ld[:n_obs] > threshold
    return dict(doublet_score=ld[:n_obs], predicted_doublet=pred, doublet_scores_sim=ld[n_obs:], threshold=threshold,
                k=k, k_adj=k_adj, count=count, gap=gap, ids=ids, embedding=emb,
                doublet_neighbor_parents=neighbor_parents(ids[:n_obs], parents, n_obs))

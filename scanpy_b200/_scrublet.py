"""`sc.pp.scrublet` and `sc.pp.scrublet_simulate_doublets` on the device.

References: src/scanpy/preprocessing/_scrublet/__init__.py:25-567 (the wrapper), core.py:188-474 (simulation, classifier,
threshold), pipeline.py:18-89 (z-score, PCA / TruncatedSVD), preprocessing/_utils.py:13-23 (the parent pairs).

Stage by stage: the QC filters, normalize_total, log1p and the seurat HVG statistics are the package's device passes;
the doublets are summed by `sb2_scrublet_pair_sums`; the z-scored PCA runs on the streamed Gram route with the z-score
folded into the statistics and the projection operator, so nothing is densified; the neighbour label counts come from
`sb2_knn_label_count_f32` (exact, (distance, id) order); the O(n) scores, the threshold and the calls stay on the host.
The parent pairs are drawn on the host from the reference's own random stream.
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import ndimage, sparse

from . import _abi, _ops
from ._abi import check, ptr
from ._compat import (LegacyRng, MiniAnnData, accepts_legacy_random_state, as_csr_f32, get_arr, is_anndata_like,
                      log_done, log_start, meta_random_state, warn)
from ._preprocess import _hvg_seurat_frame, log1p, normalize_total
from ._qc import filter_cells, filter_genes


# ------------------------------------------------------------------------------------------ host pieces
def sample_comb(n_obs: int, n_sim: int, rng) -> np.ndarray:
    """Parent pairs [n_sim x 2] drawn without repeating a pair (preprocessing/_utils.py:13-23): sklearn's
    `sample_without_replacement` seeded with the legacy `random_state`, else `rng.choice`."""
    if isinstance(rng, LegacyRng):
        from sklearn.random_projection import sample_without_replacement

        idx = sample_without_replacement(n_obs * n_obs, n_sim, random_state=rng.arg)
    else:
        idx = rng.choice(n_obs * n_obs, size=n_sim, replace=False)
    return np.vstack(np.unravel_index(idx, (n_obs, n_obs))).T


def threshold_minimum(values: np.ndarray, nbins: int = 256, max_num_iter: int = 10000) -> float:
    """`skimage.filters.threshold_minimum`: the minimum between the two modes of the 256-bin histogram, smoothed (in
    float64) by a 3-wide running mean until fewer than three maxima remain.  Raises RuntimeError when it cannot find
    exactly two maxima or runs out of iterations."""
    counts, edges = np.histogram(values, bins=nbins, range=(np.min(values), np.max(values)))
    centers = (edges[:-1] + edges[1:]) / 2
    smooth = counts.astype(np.float64)
    maxima: list[int] = []
    counter = 0
    for counter in range(max_num_iter):
        smooth = ndimage.uniform_filter1d(smooth, 3)
        maxima = _local_maxima(smooth)
        if len(maxima) < 3:
            break
    if len(maxima) != 2:
        raise RuntimeError("Unable to find two maxima in histogram")
    if counter == max_num_iter - 1:
        raise RuntimeError("Maximum iteration reached for histogram smoothing")
    return centers[maxima[0] + int(np.argmin(smooth[maxima[0]:maxima[1] + 1]))]


def _local_maxima(hist: np.ndarray) -> list[int]:
    """The left end of each run that ends a rise (plateaus count once), scanned by direction as skimage does."""
    out, direction = [], 1
    for i in range(hist.shape[0] - 1):
        if direction > 0:
            if hist[i + 1] < hist[i]:
                direction = -1
                out.append(i)
        elif hist[i + 1] > hist[i]:
            direction = 1
    return out


def n_neighbors_default(n_obs: int) -> int:
    return round(0.5 * np.sqrt(n_obs))


def k_adjusted(k: int, n_obs: int, n_sim: int) -> int:
    """core.py:339: the neighbour count scaled by the share of simulated points."""
    return round(k * (1 + n_sim / float(n_obs)))


def doublet_scores(n_sim_neigh: np.ndarray, *, k_adj: int, n_obs: int, n_sim: int, expected_doublet_rate: float,
                   stdev_doublet_rate: float):
    """The Bayesian score and its standard error, in core.py:363-381's float64 expression order."""
    rho = expected_doublet_rate
    r = n_sim / float(n_obs)
    nd = n_sim_neigh.astype(np.float64)
    n = float(k_adj)
    q = (nd + 1) / (n + 2)
    ld = q * rho / r / (1 - rho - q * (1 - rho - rho / r))
    se_q = np.sqrt(q * (1 - q) / (n + 3))
    se_rho = stdev_doublet_rate
    se_ld = (q * rho / r / (1 - rho - q * (1 - rho - rho / r)) ** 2
             * np.sqrt((se_q / q * (1 - rho)) ** 2 + (se_rho / rho * (1 - q)) ** 2))
    return ld, se_ld


def neighbor_parents(ids: np.ndarray, parents: np.ndarray, n_obs: int) -> list:
    """core.py:389-403: per observed cell, the sorted parents of its simulated neighbours."""
    out = []
    for c in range(n_obs):
        row = ids[c] - n_obs
        row = row[row > -1]
        out.append(np.unique(parents[row, :].flatten()) if len(row) else np.array([], dtype=np.intp))
    return out


def _check_options(knn_dist_metric, use_approx_neighbors, synthetic_doublet_umi_subsampling) -> None:
    if knn_dist_metric != "euclidean":
        raise NotImplementedError(f"knn_dist_metric={knn_dist_metric!r}: only 'euclidean' is implemented in "
                                  "scanpy_b200.pp.scrublet")
    if use_approx_neighbors:
        raise NotImplementedError("use_approx_neighbors=True (pynndescent) is not available in scanpy_b200 (exact GPU "
                                  "kNN only); pass None or False")
    if synthetic_doublet_umi_subsampling < 1:
        raise NotImplementedError(f"synthetic_doublet_umi_subsampling={synthetic_doublet_umi_subsampling!r}: UMI "
                                  "subsampling of the simulated doublets is not implemented in scanpy_b200")


# ------------------------------------------------------------------------------------------ device stages
def simulate(x, sim_doublet_ratio: float, rng):
    """core.py:188-238 with subsampling 1: (simulated CSR float32, parent pairs int64 [n_sim x 2], n_counts)."""
    import torch

    ctx = _abi.default_context()
    xc = as_csr_f32(x)
    n_obs = xc.shape[0]
    n_sim = int(n_obs * sim_doublet_ratio)
    pairs = sample_comb(n_obs, n_sim, rng).astype(np.int64)
    nnz_row = np.diff(xc.indptr).astype(np.int64)
    cap = int((nnz_row[pairs[:, 0]] + nnz_row[pairs[:, 1]]).sum()) if n_sim else 0
    d_indptr, d_indices, d_data = _ops.csr_to_device(xc)
    d_pairs = _ops._to_device(np.ascontiguousarray(pairs))
    o_indptr = torch.empty(n_sim + 1, dtype=torch.int64, device="cuda")
    o_indices = torch.empty(max(cap, 1), dtype=torch.int32, device="cuda")
    o_data = torch.empty(max(cap, 1), dtype=torch.float32, device="cuda")
    check(ctx.lib.sb2_scrublet_pair_sums(ctx.handle, n_obs, ptr(d_indptr), ptr(d_indices), ptr(d_data), n_sim,
                                         ptr(d_pairs), ptr(o_indptr), ptr(o_indices), ptr(o_data)))
    indptr = _ops._to_host(o_indptr)
    nnz = int(indptr[-1])
    indices, data = _ops._to_host(o_indices[:nnz], o_data[:nnz])
    sim = sparse.csr_matrix((data, indices, indptr), shape=(n_sim, xc.shape[1]))
    totals = np.asarray(xc.sum(axis=1, dtype=np.float64)).ravel().astype(xc.dtype)
    return sim, pairs, totals[pairs[:, 0]] + totals[pairs[:, 1]]


def _device_csr(x):
    xc = as_csr_f32(x)
    return (xc.shape[0],) + tuple(_ops.csr_to_device(xc))


def manifold(x_obs, x_sim, *, mean_center: bool, normalize_variance: bool, n_prin_comps: int):
    """pipeline.py:18-89 without densifying: the embedding of observed then simulated rows, fp32 [n_obs + n_sim x k]
    on the device.  mean_center: PCA of the z-scored (or centred) observed rows, both sets projected with the observed
    mean and standard deviation; else TruncatedSVD of the (column-scaled) observed rows."""
    import torch

    ctx = _abi.default_context()
    n_obs, *obs = _device_csr(x_obs)
    n_sim, *sim = _device_csr(x_sim)
    g = x_obs.shape[1]
    if not 1 <= n_prin_comps < min(n_obs, g):
        raise ValueError(f"n_components={n_prin_comps!r} must be between 1 and min(n_samples, n_features)="
                         f"{min(n_obs, g)!r} with svd_solver='arpack'")
    if n_prin_comps > 120:  # the block solvers keep n_comps + 8 vectors in a block of at most 128
        raise NotImplementedError(f"scanpy_b200.pp.scrublet computes at most 120 components (n_prin_comps={n_prin_comps!r})")
    stats = torch.zeros(2 * g, dtype=torch.float64, device="cuda")
    gram = torch.zeros((g, g), dtype=torch.float64, device="cuda")
    check(ctx.lib.sb2_pca_stream_accumulate_f32(ctx.handle, n_obs, g, *(ptr(a) for a in obs), ptr(stats), ptr(gram)))
    if normalize_variance:  # mean_var(..., correction=1) of the observed rows (pipeline.py:26, 36)
        mean = stats[:g] / n_obs
        sigma = torch.sqrt((stats[g:] / n_obs - mean * mean) * (n_obs / (n_obs - 1)))
    else:
        sigma = torch.ones(g, dtype=torch.float64, device="cuda")
    out = torch.empty((n_obs + n_sim, n_prin_comps), dtype=torch.float32, device="cuda")
    if mean_center:
        # PCA of X D^-1 (D = diag(sigma)): its statistics are Σx/σ, Σx²/σ², and its Gram D^-1 G D^-1
        stats[:g] /= sigma
        stats[g:] /= sigma * sigma
        gram /= sigma[:, None] * sigma[None, :]
        res, proj, shift, l = _ops._pca_stream_solve(ctx, n_obs, g, stats, gram, n_prin_comps, 0)
        proj[:g * l].view(g, l).mul_((1.0 / sigma).to(torch.float32)[:, None])  # rows of X, not of X D^-1, project
        for r0, (n, csr) in ((0, (n_obs, obs)), (n_obs, (n_sim, sim))):
            if n:
                check(ctx.lib.sb2_pca_stream_project_f32(ctx.handle, n, g, *(ptr(a) for a in csr), n_prin_comps, l,
                                                         ptr(proj), ptr(shift), ptr(out[r0:r0 + n])))
    else:
        if normalize_variance:
            for n, (ip, ix, dx) in ((n_obs, obs), (n_sim, sim)):
                check(ctx.lib.sb2_csr_scale_cols_f32(ctx.handle, n, ptr(ip), ptr(ix), ptr(dx), ptr(sigma), None, 0, 0.0))
        args = (n_obs, g, *(ptr(a) for a in obs), n_prin_comps, 1 if g <= 8192 else 0, 0, 0.0, 0)
        res = _ops._pca_call(ctx.lib.sb2_tsvd_csr_f32, ctx, args, n_obs, g, n_prin_comps, mean=False)
        out[:n_obs] = res["X_pca"]
        if n_sim:  # the SpMM takes 32, 64 or 128 columns: V padded with zero columns
            l = next(w for w in (32, 64, 128) if w >= n_prin_comps)
            v = torch.zeros((g, l), dtype=torch.float32, device="cuda")
            v[:, :n_prin_comps] = res["components"].t()
            y = torch.empty((n_sim, l), dtype=torch.float32, device="cuda")
            check(ctx.lib.sb2_spmm_csr(ctx.handle, n_sim, g, l, *(ptr(a) for a in sim), ptr(v), None, ptr(y)))
            out[n_obs:] = y[:, :n_prin_comps]
    if not res["converged"]:
        warn(f"scanpy_b200 PCA did not reach its residual tolerance (max relative residual "
             f"{res['max_rel_residual']:.3g}); results are approximate", UserWarning)
    return out


def label_count(d_x, n_first: int, k: int, *, with_ids: bool = False):
    """`sb2_knn_label_count_f32` on a device fp32 [n x d] array -> host (count int32 [n], kth float64 [n], ids or None)."""
    import torch

    ctx = _abi.default_context()
    n, d = d_x.shape
    if not 1 <= k <= n:
        raise ValueError(f"Scrublet needs k_adj = {k} neighbours but there are only {n} observed and simulated cells")
    count = torch.empty(n, dtype=torch.int32, device="cuda")
    kth = torch.empty(n, dtype=torch.float64, device="cuda")
    ids = torch.empty((n, k), dtype=torch.int32, device="cuda") if with_ids else None
    check(ctx.lib.sb2_knn_label_count_f32(ctx.handle, n, d, ptr(d_x.contiguous()), n_first, k, ptr(count), ptr(kth),
                                          ptr(ids)))
    if ids is None:
        return (*_ops._to_host(count, kth), None)
    return _ops._to_host(count, kth, ids)


# ------------------------------------------------------------------------------------------ the pipeline
def _call_doublets(x_obs, x_sim, parents, sim_ratio, *, n_neighbors, expected_doublet_rate, stdev_doublet_rate,
                   mean_center, normalize_variance, n_prin_comps, get_doublet_neighbor_parents, threshold, verbose,
                   rng):
    """_scrublet_call_doublets (__init__.py:301-501) -> (doublet_score, predicted_doublet, uns)."""
    n_obs, n_sim = x_obs.shape[0], x_sim.shape[0]
    if n_neighbors is None:
        n_neighbors = n_neighbors_default(n_obs)
    k_adj = k_adjusted(n_neighbors, n_obs, n_sim)
    emb = manifold(x_obs, x_sim, mean_center=mean_center, normalize_variance=normalize_variance,
                   n_prin_comps=n_prin_comps)
    count, _, ids = label_count(emb, n_obs, k_adj, with_ids=get_doublet_neighbor_parents)
    ld, se = doublet_scores(count, k_adj=k_adj, n_obs=n_obs, n_sim=n_sim, expected_doublet_rate=expected_doublet_rate,
                            stdev_doublet_rate=stdev_doublet_rate)
    ld_obs, ld_sim = ld[:n_obs], ld[n_obs:]
    uns = dict(doublet_scores_sim=ld_sim, doublet_parents=parents,
               parameters=dict(expected_doublet_rate=expected_doublet_rate, sim_doublet_ratio=sim_ratio,
                               n_neighbors=n_neighbors, **meta_random_state(rng)))
    if threshold is None:
        try:
            threshold = threshold_minimum(ld_sim)
            if verbose:
                log_start(f"Automatically set threshold at doublet score = {threshold:.2f}")
        except Exception:  # noqa: BLE001  (core.py:435-448)
            if verbose:
                warn("Failed to automatically identify doublet score threshold. Run `call_doublets` with "
                     "user-specified threshold.", UserWarning)
    if threshold is None:
        predicted = np.zeros(n_obs, dtype=bool)
    else:
        uns["threshold"] = threshold
        predicted = ld_obs > threshold
    if get_doublet_neighbor_parents:
        uns["doublet_neighbor_parents"] = neighbor_parents(ids[:n_obs], parents, n_obs)
    return ld_obs, predicted, uns


def _run(x, obs: pd.DataFrame, adata_sim, *, sim_doublet_ratio, log_transform, rng, **kw):
    """_run_scrublet (__init__.py:186-246) on one sample: its obs (positional labels, cells that survive the filter)
    with doublet_score / predicted_doublet, and its `uns['scrublet']`."""
    if adata_sim is not None:
        ld, pred, uns = _call_doublets(as_csr_f32(x), as_csr_f32(adata_sim.X), adata_sim.obsm["doublet_parents"],
                                       adata_sim.uns.get("scrublet", {}).get("parameters", {}).get("sim_doublet_ratio"),
                                       rng=rng, **kw)
    else:
        ad = MiniAnnData(as_csr_f32(x), obs=obs.copy())
        filter_genes(ad, min_cells=3)
        filter_cells(ad, min_genes=3)
        obs = ad.obs
        raw = ad.X.copy()
        normalize_total(ad)
        hvg = _hvg_seurat_frame(log1p(ad.X), None)["highly_variable"].to_numpy()
        x_obs = ad.X[:, hvg]
        x_sim, parents, _ = simulate(raw[:, hvg], sim_doublet_ratio, rng)
        if log_transform:
            x_obs, x_sim = log1p(x_obs), log1p(x_sim)
        x_obs = _normalized(x_obs, 1e6)
        x_sim = _normalized(x_sim, 1e6)
        ld, pred, uns = _call_doublets(x_obs, x_sim, parents, sim_doublet_ratio, rng=rng, **kw)
    obs = obs.copy()
    obs["doublet_score"] = ld
    obs["predicted_doublet"] = pred
    return obs, uns


def _normalized(x, target_sum: float):
    ad = MiniAnnData(x)
    normalize_total(ad, target_sum=target_sum)
    return ad.X


@accepts_legacy_random_state(0)
def scrublet(adata, adata_sim=None, *, batch_key: str | None = None, sim_doublet_ratio: float = 2.0,
             expected_doublet_rate: float = 0.05, stdev_doublet_rate: float = 0.02,
             synthetic_doublet_umi_subsampling: float = 1.0, knn_dist_metric="euclidean", normalize_variance: bool = True,
             log_transform: bool = False, mean_center: bool = True, n_prin_comps: int = 30,
             use_approx_neighbors: bool | None = None, get_doublet_neighbor_parents: bool = False,
             n_neighbors: int | None = None, threshold: float | None = None, verbose: bool = True, copy: bool = False,
             rng=None):
    """Predict doublets using Scrublet (signature of `scanpy.pp.scrublet`).

    Writes `.obs['doublet_score']`, `.obs['predicted_doublet']` and `.uns['scrublet']` as the reference does.  The
    neighbours are exact, in (distance, id) order, at every sample size."""
    _check_options(knn_dist_metric, use_approx_neighbors, synthetic_doublet_umi_subsampling)
    if not isinstance(rng, LegacyRng):
        rng = np.random.default_rng(rng)
    if copy:
        adata = adata.copy()
    start = log_start("Running Scrublet")
    positions = pd.RangeIndex(adata.n_obs).astype(str)
    obs = adata.obs.copy()
    obs.index = positions
    kw = dict(adata_sim=adata_sim, sim_doublet_ratio=sim_doublet_ratio, log_transform=log_transform,
              n_neighbors=n_neighbors, expected_doublet_rate=expected_doublet_rate,
              stdev_doublet_rate=stdev_doublet_rate, mean_center=mean_center, normalize_variance=normalize_variance,
              n_prin_comps=n_prin_comps, get_doublet_neighbor_parents=get_doublet_neighbor_parents,
              threshold=threshold, verbose=verbose)
    x = adata.X
    if batch_key is not None:
        if batch_key not in adata.obs.columns:
            raise ValueError("`batch_key` must be a column of .obs in the input AnnData object,"
                             f"but {batch_key!r} is not in {adata.obs.keys()!r}.")
        batches = np.unique(adata.obs[batch_key])
        sub_rngs = [rng] * len(batches) if isinstance(rng, LegacyRng) else rng.spawn(len(batches))
        xr = x.tocsr() if sparse.issparse(x) else np.asarray(x)
        scrubbed = []
        for batch, sub in zip(batches, sub_rngs, strict=True):
            sel = np.flatnonzero((adata.obs[batch_key] == batch).to_numpy())
            scrubbed.append(_run(xr[sel], obs.iloc[sel], rng=sub, **kw))
        scrubbed_obs = pd.concat([o for o, _ in scrubbed]).astype(adata.obs.dtypes)
        adata.obs = scrubbed_obs.reindex(positions).set_axis(adata.obs.index)
        adata.uns["scrublet"] = dict(batches=dict(zip(batches, [u for _, u in scrubbed], strict=True)),
                                     batched_by=batch_key)
    else:
        o, uns = _run(x, obs, rng=rng, **kw)
        o = o.reindex(positions)
        adata.obs["doublet_score"] = o["doublet_score"].to_numpy()
        adata.obs["predicted_doublet"] = o["predicted_doublet"].to_numpy()
        adata.uns["scrublet"] = uns
    log_done(start)
    return adata if copy else None


@accepts_legacy_random_state(0)
def scrublet_simulate_doublets(adata, *, layer: str | None = None, sim_doublet_ratio: float = 2.0,
                               synthetic_doublet_umi_subsampling: float = 1.0, rng=None):
    """Simulate doublets by adding the counts of random observed transcriptome pairs (signature of
    `scanpy.pp.scrublet_simulate_doublets`): a `MiniAnnData` with the simulated counts in `X` (CSR),
    `obs['n_counts']`, `obsm['doublet_parents']` and `uns['scrublet']['parameters']`."""
    _check_options("euclidean", None, synthetic_doublet_umi_subsampling)
    if not isinstance(rng, LegacyRng):
        rng = np.random.default_rng(rng)
    x = get_arr(adata, layer=layer) if is_anndata_like(adata) else adata
    sim, parents, n_counts = simulate(x, sim_doublet_ratio, rng)
    out = MiniAnnData(sim)
    out.obs["n_counts"] = n_counts
    out.obsm["doublet_parents"] = parents
    out.uns["scrublet"] = {"parameters": {"sim_doublet_ratio": sim_doublet_ratio}}
    return out

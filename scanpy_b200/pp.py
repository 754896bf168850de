"""`sc.pp.pca` and `sc.pp.neighbors` with scanpy's signatures, running on libscanpy_b200 (H100, sm_90a).

Drop-in scope (SURVEY.md 8b): same argument names, same `.obsm/.varm/.obsp/.uns` write-backs, same
exception types/messages where the reference's tests pin them.  Options whose arithmetic is not
implemented on the GPU raise `NotImplementedError` naming the option (never silently different).
References: src/scanpy/preprocessing/_pca/__init__.py:53-384, src/scanpy/neighbors/__init__.py:88-316,
src/scanpy/neighbors/_common.py:17-143, src/scanpy/tools/_utils.py:20-78.
"""
from __future__ import annotations

from types import MappingProxyType
from typing import Any, Mapping

import numpy as np
from scipy import sparse

from . import _ops
from ._preprocess import highly_variable_genes, log1p, normalize_total, scale  # noqa: F401  (SURVEY 8f row f2)
from ._qc import calculate_qc_metrics, filter_cells, filter_genes  # noqa: F401
from ._regress import regress_out  # noqa: F401
from ._compat import (MiniAnnData, accepts_legacy_random_state, as_csr_f32, is_anndata_like, log_done, log_start,
                      meta_random_state, seed_from_rng, settings, warn)

_SPARSE_SOLVERS = ("arpack", "covariance_eigh")  # SvdSolvPCASparseSklearn
_DEFAULT = object()


# ------------------------------------------------------------------------------------------ pca
def _check_mask(adata, mask, dim: str = "var"):
    """src/scanpy/get/get.py:607-660 (boolean masks only)."""
    if mask is None:
        return None
    if isinstance(mask, str):
        frame = adata.var if dim == "var" else adata.obs
        if mask not in frame:
            raise ValueError(f"Did not find `adata.{dim}[{mask!r}]`. ")
        mask_array = np.asarray(frame[mask])
    else:
        if len(mask) != adata.shape[0 if dim == "obs" else 1]:
            raise ValueError("The shape of the mask do not match the data.")
        mask_array = np.asarray(mask)
    if mask_array.dtype != bool:
        raise ValueError("Mask array must be boolean.")
    return mask_array


def _solver_code(svd_solver: str | None, *, n_vars: int) -> int:
    """Map the reference's solver names onto the two CUDA routes (src/.../_pca/__init__.py:425-467).

    'arpack' (the reference default for sparse input) and 'covariance_eigh' are the two exact
    solvers sklearn offers for CSR; both are served by exact block solvers here:
    0 = SpMM-driven subspace iteration, 1 = Gram route.  `None`/'arpack' pick the faster exact
    route for the shape at hand (Gram while the g x g covariance fits comfortably in L2/HBM).
    """
    if svd_solver not in _SPARSE_SOLVERS and svd_solver is not None:
        if svd_solver in ("b200_spmm", "b200_gram"):
            return 0 if svd_solver == "b200_spmm" else 1
        warn(f"Ignoring svd_solver={svd_solver!r} and using arpack, sklearn.decomposition._pca.PCA (with sparse "
             f"input) only supports {set(_SPARSE_SOLVERS)}.", UserWarning)
        svd_solver = "arpack"
    if svd_solver == "covariance_eigh":
        return 1
    return 1 if n_vars <= 8192 else 0


@accepts_legacy_random_state(0)
def pca(data, n_comps: int | None = None, *, layer: str | None = None, obsm: str | None = None,
        zero_center: bool = True, svd_solver: str | None = None, chunked: bool = False,
        chunk_size: int | None = None, rng=None, return_info: bool = False, mask_var=_DEFAULT,
        dtype="float32", key_added: str | None = None, copy: bool = False):
    """Principal component analysis (signature of `scanpy.pp.pca`, _pca/__init__.py:53-71)."""
    start = log_start("computing PCA")
    if (layer is not None or obsm is not None) and chunked:
        raise NotImplementedError("Cannot use `layer`/`obsm` and `chunked` at the same time.")
    return_anndata = is_anndata_like(data)
    if return_anndata:
        adata = data.copy() if copy else data
    else:
        adata = MiniAnnData(data)

    if mask_var is _DEFAULT:
        mask_var = "highly_variable" if "highly_variable" in adata.var else None
    elif mask_var is not None and obsm is not None:
        raise ValueError("Argument `mask_var` is incompatible with `obsm`.")
    mask_var_param, mask_var = mask_var, _check_mask(adata, mask_var, "var")

    if obsm is not None:
        x = adata.obsm[obsm]
    elif layer is not None:
        x = adata.layers[layer]
    else:
        x = adata.X
    if type(x).__module__.startswith("dask"):
        raise NotImplementedError("dask arrays are not supported by scanpy_b200.pp.pca")
    backed = hasattr(x, "row_chunks")  # on-disk CSR (scanpy_b200._io.ZarrCSR)
    if backed and not chunked:
        raise NotImplementedError("an on-disk matrix can only be processed with `chunked=True` in scanpy_b200.pp.pca")
    if mask_var is not None:
        if backed:
            raise NotImplementedError("`mask_var` on an on-disk matrix is not implemented in scanpy_b200.pp.pca")
        x = x[:, mask_var]
    n_obs, n_vars = x.shape
    if n_comps is None:
        min_dim = min(n_vars, n_obs)
        n_comps = min_dim - 1 if min_dim <= settings.N_PCS else settings.N_PCS
    if not (1 <= n_comps < min(n_obs, n_vars)):
        # sklearn's message for svd_solver='arpack' (pinned by tests/test_pca.py:292-296)
        raise ValueError(f"n_components={n_comps!r} must be between 1 and min(n_samples, n_features)="
                         f"{min(n_obs, n_vars)!r} with svd_solver='arpack'")
    xc = x if backed else as_csr_f32(x)
    solver = _solver_code(svd_solver, n_vars=n_vars) if (zero_center and not chunked) else 1
    if not zero_center and not chunked:
        # sklearn TruncatedSVD (_pca/__init__.py:309-336); its solver names are 'arpack' | 'randomized' (default) - both are
        # served by the exact device solver
        if svd_solver not in (None, "arpack", "randomized", "b200_spmm"):
            warn(f"Ignoring {svd_solver=} and using arpack, TruncatedSVD only supports ['arpack', 'randomized'].", UserWarning)
        if backed:
            raise NotImplementedError("`zero_center=False` on an on-disk matrix is not implemented in scanpy_b200.pp.pca")
        out = _ops.tsvd_csr(xc, n_comps, solver=0 if (svd_solver == "b200_spmm" or n_vars > 8192) else 1, seed=seed_from_rng(rng))
    elif chunked:
        # (the reference ignores zero_center / svd_solver here too: "Ignoring zero_center, rng, svd_solver", :246-247)
        # the reference feeds row chunks to IncrementalPCA and expects the full PCA's result (tests/test_pca.py:357-386);
        # here the chunks stream through the exact Gram route (out-of-core: one chunk on the device at a time)
        out = _ops.pca_csr_chunked(xc, n_comps, chunk_size=settings.chunk_size if chunk_size is None else chunk_size,
                                   seed=seed_from_rng(rng))
    else:
        out = _ops.pca_csr(xc, n_comps, solver=solver, seed=seed_from_rng(rng))
    if not out["converged"]:
        # the block iteration stopped on stagnation / its iteration cap before the residual test was met (the SpMM-driven
        # solver works in float32 passes and can sit on its rounding floor): never silently different
        warn(f"scanpy_b200 PCA did not reach its residual tolerance (max relative residual "
             f"{out['max_rel_residual']:.3g} after {out['iterations']} operator applications); results are approximate",
             UserWarning)
    x_pca = out["X_pca"]
    if x_pca.dtype != np.dtype(dtype):
        x_pca = x_pca.astype(dtype)
    components = out["components"]
    variance, variance_ratio = out["variance"], out["variance_ratio"]
    if np.dtype(dtype) == np.float32:
        variance, variance_ratio = variance.astype(np.float32), variance_ratio.astype(np.float32)

    if return_anndata:
        k_obsm, k_varm, k_uns = ("X_pca", "PCs", "pca") if key_added is None else (key_added,) * 3
        adata.obsm[k_obsm] = x_pca
        if obsm:
            pass
        elif mask_var is not None:
            adata.varm[k_varm] = np.zeros(shape=(adata.n_vars, n_comps))
            adata.varm[k_varm][mask_var] = components.T
        else:
            adata.varm[k_varm] = components.T
        adata.uns[k_uns] = dict(
            params=dict(zero_center=zero_center, mask_var=mask_var_param,
                        **(dict(layer=layer) if layer is not None else {}),
                        **(dict(obsm=obsm) if obsm is not None else {})),
            variance=variance, variance_ratio=variance_ratio,
            **(dict(components=components.T) if obsm is not None else {}))
        log_done(start)
        return adata if copy else None
    log_done(start)
    if return_info:
        return x_pca, components, variance_ratio, variance
    return x_pca


# ------------------------------------------------------------------------------------------ neighbors
def _has_self_column(indices, distances) -> bool:
    return bool((indices[:, 0] == np.arange(indices.shape[0])).any())


def _get_sparse_matrix_from_indices_distances(indices, distances, *, keep_self: bool):
    """src/scanpy/neighbors/_common.py:35-61."""
    if not keep_self:
        if not _has_self_column(indices, distances):
            raise AssertionError("The first neighbor should be the cell itself.")
        indices, distances = indices[:, 1:], distances[:, 1:]
    indptr = np.arange(0, np.prod(indices.shape) + 1, indices.shape[1])
    # the reference copies (`distances.copy().ravel()`) so that the matrix never aliases its inputs; after the
    # self column has been sliced off, `np.ascontiguousarray(...).ravel()` already is a fresh buffer (one copy, not two)
    data = np.ascontiguousarray(distances).ravel() if not distances.flags.c_contiguous else distances.copy().ravel()
    cols = np.ascontiguousarray(indices).ravel() if not indices.flags.c_contiguous else indices.copy().ravel()
    return sparse.csr_matrix((data, cols, indptr), shape=(indices.shape[0],) * 2)


def _get_indices_distances_from_sparse_matrix(d, n_neighbors: int):
    """src/scanpy/neighbors/_common.py:74-143 (constant-nnz shortcut + slow path)."""
    nnzs = d.getnnz(axis=1)
    if len(nnzs) and (nnzs == nnzs[0]).all():
        n_obs, k = d.shape[0], int(nnzs[0])
        indices, distances = d.indices.reshape(n_obs, k), d.data.reshape(n_obs, k)
    else:
        warn("Sparse matrix has no constant number of neighbors per row. Cannot efficiently get indices and "
             "distances.", RuntimeWarning)
        n_obs = d.shape[0]
        indices = np.zeros((n_obs, n_neighbors), dtype=int)
        distances = np.zeros((n_obs, n_neighbors), dtype=d.dtype)
        for i in range(n_obs):
            row = d[i]
            cols, vals = row.indices, row.data
            if len(cols) > n_neighbors - 1:
                o = np.argsort(vals)[: n_neighbors - 1]
                cols, vals = cols[o], vals[o]
            indices[i, 0], distances[i, 0] = i, 0
            indices[i, 1:1 + len(cols)] = cols
            distances[i, 1:1 + len(cols)] = vals
    if not _has_self_column(indices, distances):
        indices = np.hstack([np.arange(indices.shape[0])[:, None], indices])
        distances = np.hstack([np.zeros(distances.shape[0])[:, None], distances])
    if indices.shape[1] > n_neighbors:
        indices, distances = indices[:, :n_neighbors], distances[:, :n_neighbors]
    return indices, distances


def _choose_representation(adata, *, use_rep: str | None, n_pcs: int | None):
    """src/scanpy/tools/_utils.py:20-78 (incl. the auto-PCA fallback pinned by tests/test_neighbors_key_added.py)."""
    if use_rep is None and n_pcs == 0:
        use_rep = "X"
    if use_rep is None:
        if adata.n_vars <= settings.N_PCS:
            return adata.X
        if "X_pca" in adata.obsm:
            if n_pcs is not None and n_pcs > adata.obsm["X_pca"].shape[1]:
                raise ValueError("`adata.obsm['X_pca']` does not have enough PCs. Rerun `sc.pp.pca` with adjusted "
                                 "`n_comps`.")
            return adata.obsm["X_pca"][:, :n_pcs]
        warn(f"You’re trying to run this on {adata.n_vars} dimensions of `.X`, if you really want this, set "
             "`use_rep=’X’`.\n         Falling back to preprocessing with `sc.pp.pca` and default params.", UserWarning)
        pca(adata, n_comps=n_pcs if n_pcs is not None else settings.N_PCS)
        return adata.obsm["X_pca"]
    if use_rep in adata.obsm and n_pcs is not None:
        if n_pcs > adata.obsm[use_rep].shape[1]:
            raise ValueError(f"{use_rep} does not have enough Dimensions. Provide a Representation with equal or more "
                             "dimensions than`n_pcs` or lower `n_pcs` ")
        return adata.obsm[use_rep][:, :n_pcs]
    if use_rep in adata.obsm and n_pcs is None:
        return adata.obsm[use_rep]
    if use_rep == "X":
        return adata.X
    raise ValueError(f"Did not find {use_rep} in `.obsm.keys()`. You need to compute it first.")


def _get_indices_distances_from_dense_matrix(d, n_neighbors: int):
    """src/scanpy/neighbors/_common.py:63-71."""
    sample_range = np.arange(d.shape[0])[:, None]
    indices = np.argpartition(d, n_neighbors - 1, axis=1)[:, :n_neighbors]
    indices = indices[sample_range, np.argsort(d[sample_range, indices])]
    return indices, d[sample_range, indices]


def _write_neighbors(adata, key_added, *, dist, conn, params):
    if key_added is None:
        key_added, conns_key, dists_key = "neighbors", "connectivities", "distances"
    else:
        conns_key, dists_key = f"{key_added}_connectivities", f"{key_added}_distances"
    adata.uns[key_added] = dict(connectivities_key=conns_key, distances_key=dists_key, params=params)
    adata.obsp[dists_key] = dist
    adata.obsp[conns_key] = conn
    return key_added, dists_key, conns_key


def _neighbors_from_distances(adata, n_neighbors, *, distances, method, metric, metric_kwds, use_rep, n_pcs, knn,
                              meta_rs, key_added, copy):
    """Precomputed `distances=`: skip PCA and the search, compute connectivities only
    (src/scanpy/neighbors/__init__.py:232-270, :675-701)."""
    ignored = {name for name, val, default in (("use_rep", use_rep, None), ("knn", knn, True), ("n_pcs", n_pcs, None),
                                                 ("metric_kwds", dict(metric_kwds), {})) if val != default}
    if meta_rs.get("random_state") != 0:
        ignored.add("rng/random_state")
        meta_rs = {k: v for k, v in meta_rs.items() if k != "random_state"}
    if ignored:
        warn(f"Parameter(s) ignored if `distances` is given: {ignored}", UserWarning)
    if callable(metric):
        raise TypeError("`metric` must be a string if `distances` is given.")
    start = log_start("computing connectivities")
    adata = adata.copy() if copy else adata
    if sparse.issparse(distances):
        distances = distances.tocsr(copy=True)
        distances.setdiag(0)
        distances.eliminate_zeros()
        knn_indices, knn_distances = _get_indices_distances_from_sparse_matrix(distances, n_neighbors)
    else:
        distances = np.asarray(distances).copy()
        np.fill_diagonal(distances, 0)
        knn_indices, knn_distances = _get_indices_distances_from_dense_matrix(distances, n_neighbors)
    if method == "umap":
        conn, _, _ = _ops.fuzzy_simplicial_set(knn_indices.astype(np.int32), knn_distances.astype(np.float64))
    else:  # 'gauss' | 'jaccard': the reference dispatches on `method` here too (neighbors/__init__.py:672-708)
        conn = _ops.knn_connectivities(knn_indices.astype(np.int32), knn_distances.astype(np.float64), method)
    params = dict(n_neighbors=n_neighbors, method=method, metric=metric, **meta_rs,
                  **({} if not metric_kwds else dict(metric_kwds=metric_kwds)))
    key_added, dists_key, conns_key = _write_neighbors(adata, key_added, dist=distances, conn=conn, params=params)
    log_done(start, f"added to `.uns[{key_added!r}]`, `.obsp[{dists_key!r}]`, `.obsp[{conns_key!r}]`")
    return adata if copy else None


@accepts_legacy_random_state(0)
def neighbors(adata, n_neighbors: int = 15, n_pcs: int | None = None, *, distances=None, use_rep: str | None = None,
              knn: bool = True, method: str = "umap", transformer=None, metric: str | None = None,
              metric_kwds: Mapping[str, Any] = MappingProxyType({}), rng=None, key_added: str | None = None,
              copy: bool = False):
    """kNN graph + UMAP connectivities (signature of `scanpy.pp.neighbors`, neighbors/__init__.py:88-103)."""
    from .transformer import B200KNNTransformer

    meta_rs = meta_random_state(rng)
    if method not in ("umap", "gauss", "jaccard") and method is not None:
        raise ValueError("`method` needs to be one of ('umap', 'gauss', 'jaccard').")
    if distances is not None:
        return _neighbors_from_distances(adata, n_neighbors, distances=distances, method=method, metric=metric,
                                         metric_kwds=metric_kwds, use_rep=use_rep, n_pcs=n_pcs, knn=knn,
                                         meta_rs=meta_rs, key_added=key_added, copy=copy)
    if not knn:
        raise ValueError(f"`method = {method!r} only with `knn = True`.")
    if metric is None:
        metric = "euclidean"
    if callable(metric) or metric not in ("euclidean", "l2"):
        raise NotImplementedError(f"metric={metric!r}: only 'euclidean' is implemented in scanpy_b200.")
    if isinstance(transformer, str) and transformer not in ("sklearn", "b200"):
        if transformer in ("pynndescent", "rapids"):
            raise NotImplementedError(f"transformer={transformer!r} is not available in scanpy_b200 (exact GPU kNN "
                                      "only); pass an instance or None")
        raise ValueError(f"Unknown transformer: {transformer}. Try passing a class or one of "
                         "('pynndescent', 'sklearn', 'rapids')")
    start = log_start("computing neighbors")
    adata = adata.copy() if copy else adata
    if transformer is not None and not isinstance(transformer, str):
        n_neighbors = transformer.get_params()["n_neighbors"]
    elif n_neighbors > adata.shape[0]:
        n_neighbors = 1 + int(0.5 * adata.shape[0])
        warn(f"n_obs too small: adjusting to `n_neighbors = {n_neighbors}`", UserWarning)
    x = _choose_representation(adata, use_rep=use_rep, n_pcs=n_pcs)
    if (transformer is None or isinstance(transformer, str)) and method == "umap":
        # built-in exact kNN: (idx, dist) stay in HBM between the search and the fuzzy-set kernels, so the
        # n x k lists cross PCIe once (device -> host) instead of three times
        xd = x.toarray() if sparse.issparse(x) else np.asarray(x)
        dist_csr, conn = _ops.knn_and_connectivities(np.ascontiguousarray(xd, dtype=np.float32),
                                                     min(n_neighbors, adata.shape[0]))
    else:
        if transformer is None or isinstance(transformer, str):
            transformer = B200KNNTransformer(n_neighbors=n_neighbors, metric=metric)
        d = transformer.fit_transform(x)
        knn_indices, knn_distances = _get_indices_distances_from_sparse_matrix(d, n_neighbors)
        if method == "umap":
            conn, _, _ = _ops.fuzzy_simplicial_set(knn_indices, knn_distances)
        else:  # 'gauss' | 'jaccard' (src/scanpy/neighbors/__init__.py:675-701)
            conn = _ops.knn_connectivities(knn_indices, knn_distances, method)
        dist_csr = _get_sparse_matrix_from_indices_distances(knn_indices, knn_distances, keep_self=False)

    if key_added is None:
        key_added, conns_key, dists_key = "neighbors", "connectivities", "distances"
    else:
        conns_key, dists_key = f"{key_added}_connectivities", f"{key_added}_distances"
    adata.uns[key_added] = dict(
        connectivities_key=conns_key, distances_key=dists_key,
        params=dict(n_neighbors=n_neighbors, method=method, metric=metric, **meta_rs,
                    **({} if not metric_kwds else dict(metric_kwds=metric_kwds)),
                    **({} if use_rep is None else dict(use_rep=use_rep)),
                    **({} if n_pcs is None else dict(n_pcs=n_pcs))))
    adata.obsp[dists_key] = dist_csr
    adata.obsp[conns_key] = conn
    log_done(start, f"added to `.uns[{key_added!r}]`, `.obsp[{dists_key!r}]`, `.obsp[{conns_key!r}]`")
    return adata if copy else None

"""`sc.experimental.pp`: analytic Pearson residuals (Lause et al. 2021) on the device.

References: src/scanpy/experimental/pp/_highly_variable_genes.py:35-395, _normalization.py:36-258, _recipes.py:41-158.
The passes over X run in CUDA: the per-batch gene totals (`sb2_regress_col_sums`, grouped), the cell totals, the
per-gene residual variance and the dense residuals (csrc/pearson.cu).  The g-sized ranking, the median rank and the
final sort are the reference's numpy / pandas code, on the host.

The residual of x[i, j] is clip((x - mu) / sqrt(mu + mu^2 / theta)) with mu = s_i s_j / S, evaluated for every cell and
gene, the zeros of a sparse X included.  Totals and residuals are fp64, each residual rounded once to the output dtype;
the reference sums a float32 X in float32 and computes float32 residuals for it (DESIGN.md §5).

Quirks of the reference that are kept:
* batches are taken in `np.unique` order, and `clip=None` becomes sqrt(n) of the FIRST batch, which every later batch
  reuses (the loop rebinds `clip`);
* a gene whose total is zero in a batch gets residual variance 0 there; `residual_variances` is the mean over batches;
* a zero-total cell (or gene, in `normalize_pearson_residuals`) gives 0 / 0 = NaN, which the clip keeps.

The dense result of `normalize_pearson_residuals` moves to the host `settings.chunk_size` rows at a time, so device
memory does not grow with n x g.  A sparse X is uploaded once as CSR; a dense X streams through by row blocks.
"""
from __future__ import annotations

from types import MappingProxyType

import numpy as np
import pandas as pd
from scipy import sparse

from . import _abi, _ops
from ._abi import check, ptr
from ._compat import accepts_legacy_random_state, get_arr, is_anndata_like, log_done, log_start, logger, settings, warn
from ._regress import _col_sums

PARTIAL_BYTES = 1 << 28  # device scratch for the residual variance's per-subtile partials
_DEFAULT = object()


# ------------------------------------------------------------------------------------------ host helpers
def _check_x(x, fn: str) -> np.dtype:
    """The value dtype X goes to the device in; raises for what the kernels do not take."""
    if hasattr(x, "row_chunks"):  # on-disk CSR (scanpy_b200._io.ZarrCSR)
        raise NotImplementedError(f"{fn} is not implemented for matrices of type {type(x)}")
    if type(x).__module__.startswith("dask"):
        raise NotImplementedError(f"dask arrays are not supported by scanpy_b200's {fn}")
    if sparse.issparse(x) and x.format not in ("csr", "csc"):
        raise NotImplementedError(f"{fn} in scanpy_b200 supports CSR, CSC and dense X, not {x.format}")
    dtype = np.dtype(x.dtype)
    if dtype not in (np.float32, np.float64, np.int32, np.int64):
        raise NotImplementedError(f"{fn} in scanpy_b200 supports float32, float64, int32 and int64 data, not {dtype}")
    return np.dtype(np.float32) if dtype == np.float32 else np.dtype(np.float64)


def check_nonnegative_integers(x) -> bool:
    """src/scanpy/_utils/__init__.py:761-773, on the host."""
    data = x.data if sparse.issparse(x) else np.asarray(x)
    if np.signbit(data).any():
        return False
    if np.issubdtype(data.dtype, np.integer):
        return True
    return not np.any((data % 1) != 0)


def _check_theta_clip(theta, clip) -> None:
    if theta <= 0:
        raise ValueError("Pearson residuals require theta > 0")
    if clip is not None and clip < 0:
        raise ValueError("Pearson residuals require `clip>=0` or `clip=None`.")


def _row_sums(dx: _ops.DeviceX, n: int, g: int):
    """fp64 total of every row, on the device."""
    import torch

    ctx = _abi.default_context()
    out = torch.empty(n, dtype=torch.float64, device="cuda")
    step = n if dx.dense is None else max(1, int(settings.chunk_size))
    for r0 in range(0, n, max(1, step)):
        r1 = min(n, r0 + step)
        d_x, d_indptr, _, d_data = dx.block(r0, r1)
        check(ctx.lib.sb2_pearson_row_sums(ctx.handle, r1 - r0, g, dx.is_f64, ptr(d_x), ptr(d_indptr), ptr(d_data),
                                           ptr(out[r0:r1])))
    return out


def _totals(dx: _ops.DeviceX, n: int, g: int, codes: np.ndarray, n_batches: int):
    """(gene totals per batch [n_batches x g] fp64 on the host, cell totals [n] fp64 on the device)."""
    gene, _ = _col_sums(dx, n, g, group=codes, n_groups=n_batches)
    return gene, _row_sums(dx, n, g)


def _residual_variances(dx: _ops.DeviceX, g: int, rows: np.ndarray, d_rows, d_cells, gene: np.ndarray,
                        total: float, clip: float, theta: float):
    """(population variance of the clipped residuals, Σx²) per gene over the cells `rows` of one batch.  The rows go
    through in blocks of whole subtiles, so the result does not depend on the block size."""
    import torch

    ctx = _abi.default_context()
    acc = torch.zeros(4 * g, dtype=torch.float64, device="cuda")
    d_gene = _ops._to_device(np.ascontiguousarray(gene, dtype=np.float64))
    step = _ops.subtile_block_rows(dx.dense is not None, PARTIAL_BYTES, 3 * g * 8)
    m = len(rows)
    for k0 in range(0, m, step):
        k1 = min(m, k0 + step)
        d_x, d_indptr, d_indices, d_data, d_order = dx.gather(rows, d_rows, k0, k1)
        check(ctx.lib.sb2_pearson_residual_var(ctx.handle, k1 - k0, g, dx.is_f64, ptr(d_x), ptr(d_indptr),
                                               ptr(d_indices), ptr(d_data), ptr(d_order), ptr(d_gene),
                                               ptr(d_cells[k0:k1]), float(total), float(clip), float(theta), ptr(acc)))
    acc = _ops._to_host(acc).reshape(4, g)
    with np.errstate(invalid="ignore", divide="ignore"):
        return acc[2] / acc[0], acc[3]


# ------------------------------------------------------------------------------------------ highly_variable_genes
def _highly_variable_pearson_residuals(adata, *, theta, clip, n_top_genes, batch_key, check_values, layer, subset,
                                       inplace):
    """_highly_variable_genes.py:129-287."""
    x = get_arr(adata, layer=layer)
    computed_on = layer if layer else "adata.X"
    vdtype = _check_x(x, "highly_variable_genes")
    if not sparse.issparse(x):
        x = np.asarray(x)
    if check_values and not check_nonnegative_integers(x):
        warn("`flavor='pearson_residuals'` expects raw count data, but non-integers were found.", UserWarning)
    _check_theta_clip(theta, clip)

    n, g = x.shape
    batch_info = np.zeros(n, dtype=int) if batch_key is None else adata.obs[batch_key].to_numpy()
    batches, codes = np.unique(batch_info, return_inverse=True)
    n_batches = len(batches)
    codes = codes.astype(np.int32).reshape(-1)

    if sparse.issparse(x):
        x = x.tocsr()
    dx = _ops.DeviceX(x, vdtype)
    gene_tot, d_cell = _totals(dx, n, g, codes, n_batches)
    order = np.argsort(codes, kind="stable")  # each batch contiguous, its cells in their original order
    d_order = _ops._to_device(order.astype(np.int64)) if dx.dense is None else None
    d_cells = _ops._to_device(_ops._to_host(d_cell)[order])
    bounds = np.searchsorted(codes[order], np.arange(n_batches + 1))

    residual_gene_vars = []
    sq = np.zeros(g)
    for b in range(n_batches):
        k0, k1 = int(bounds[b]), int(bounds[b + 1])
        nonzero_genes = gene_tot[b] != 0
        if clip is None:
            clip = np.sqrt(k1 - k0)
        sum_total = np.sum(gene_tot[b][nonzero_genes])
        var, sq_b = _residual_variances(dx, g, order[k0:k1], d_order[k0:k1] if d_order is not None else None,
                                        d_cells[k0:k1], gene_tot[b], sum_total, clip, theta)
        sq += sq_b
        residual_gene_vars.append(np.where(nonzero_genes, var, 0.0).reshape(1, -1))
    residual_gene_vars = np.concatenate(residual_gene_vars, axis=0)

    # the reference's host code from here on
    ranks_residual_var = np.argsort(np.argsort(-residual_gene_vars, axis=1), axis=1)
    ranks_residual_var = ranks_residual_var.astype(np.float32)
    highly_variable_nbatches = np.sum((ranks_residual_var < n_top_genes).astype(int), axis=0)
    ranks_residual_var[ranks_residual_var >= n_top_genes] = np.nan
    ranks_masked_array = np.ma.masked_invalid(ranks_residual_var)
    medianrank_residual_var = np.ma.median(ranks_masked_array, axis=0).filled(np.nan)

    # mean_var(x, axis=0, correction=1) from the fp64 totals and Σx²
    means = gene_tot.sum(axis=0) / n
    variances = (sq / n - means**2) * (n / (n - 1))
    df = pd.DataFrame.from_dict(dict(
        means=means,
        variances=variances,
        residual_variances=np.mean(residual_gene_vars, axis=0),
        highly_variable_rank=medianrank_residual_var,
        highly_variable_nbatches=highly_variable_nbatches.astype(np.int64),
        highly_variable_intersection=highly_variable_nbatches == n_batches,
    ))
    df = df.set_index(adata.var.index)
    df = df.sort_values(["highly_variable_nbatches", "highly_variable_rank"], ascending=[False, True],
                        na_position="last")
    high_var = np.zeros(df.shape[0], dtype=bool)
    high_var[:n_top_genes] = True
    df["highly_variable"] = high_var
    df = df.loc[adata.var.index, :]

    if inplace:
        adata.uns["hvg"] = {"flavor": "pearson_residuals", "computed_on": computed_on}
        logger.info("added\n"
                    "    'highly_variable', boolean vector (adata.var)\n"
                    "    'highly_variable_rank', float vector (adata.var)\n"
                    "    'highly_variable_nbatches', int vector (adata.var)\n"
                    "    'highly_variable_intersection', boolean vector (adata.var)\n"
                    "    'means', float vector (adata.var)\n"
                    "    'variances', float vector (adata.var)\n"
                    "    'residual_variances', float vector (adata.var)")
        adata.var["means"] = df["means"].array
        adata.var["variances"] = df["variances"].array
        adata.var["residual_variances"] = df["residual_variances"].array
        adata.var["highly_variable_rank"] = df["highly_variable_rank"].array
        if batch_key is not None:
            adata.var["highly_variable_nbatches"] = df["highly_variable_nbatches"].array
            adata.var["highly_variable_intersection"] = df["highly_variable_intersection"].array
        adata.var["highly_variable"] = df["highly_variable"].array
        if subset:
            adata._inplace_subset_var(df["highly_variable"].to_numpy())
        return None
    if batch_key is None:
        df = df.drop(["highly_variable_nbatches", "highly_variable_intersection"], axis=1)
    if subset:
        df = df.iloc[df["highly_variable"].to_numpy(), :]
    return df


def highly_variable_genes(adata, *, theta: float = 100, clip: float | None = None, n_top_genes: int | None = None,
                          batch_key: str | None = None, chunksize: int = 1000, flavor: str = "pearson_residuals",
                          check_values: bool = True, layer: str | None = None, subset: bool = False,
                          inplace: bool = True):
    """Select highly variable genes using analytic Pearson residuals (signature of
    `scanpy.experimental.pp.highly_variable_genes`).  `chunksize` is accepted and has no effect, as in the reference."""
    logger.info("extracting highly variable genes")
    if not is_anndata_like(adata):
        raise ValueError("`pp.highly_variable_genes` expects an `AnnData` argument, pass `inplace=False` if you want "
                         "to return a `pd.DataFrame`.")
    if flavor != "pearson_residuals":
        raise ValueError("This is an experimental API and only `flavor=pearson_residuals` is available.")
    if n_top_genes is None:
        raise ValueError("`pp.highly_variable_genes` requires the argument `n_top_genes` for "
                         "`flavor='pearson_residuals'`")
    return _highly_variable_pearson_residuals(adata, theta=theta, clip=clip, n_top_genes=n_top_genes,
                                              batch_key=batch_key, check_values=check_values, layer=layer,
                                              subset=subset, inplace=inplace)


# ------------------------------------------------------------------------------------------ normalization
def _pearson_residuals(x, theta, clip, check_values) -> np.ndarray:
    """_normalization.py:36-75: the dense clipped residuals; float32 for float32 X, float64 otherwise."""
    vdtype = _check_x(x, "normalize_pearson_residuals")
    if not sparse.issparse(x):
        x = np.asarray(x)
    _check_theta_clip(theta, clip)
    n, g = x.shape
    if clip is None:
        clip = np.sqrt(n)
    if check_values and not check_nonnegative_integers(x):
        warn("`normalize_pearson_residuals()` expects raw count data, but non-integers were found.", UserWarning)

    ctx = _abi.default_context()
    dx = _ops.DeviceX(x.tocsr() if sparse.issparse(x) else x, vdtype)
    gene_tot, d_cell = _totals(dx, n, g, np.zeros(n, dtype=np.int32), 1)
    sum_total = float(np.sum(gene_tot[0]))
    d_gene = _ops._to_device(np.ascontiguousarray(gene_tot[0]))

    def launch(r0, r1, xargs, d_out):
        d_x, d_indptr, d_indices, d_data = xargs
        check(ctx.lib.sb2_pearson_residuals(ctx.handle, r1 - r0, g, dx.is_f64, ptr(d_x), ptr(d_indptr),
                                            ptr(d_indices), ptr(d_data), ptr(d_gene), ptr(d_cell[r0:r1]), sum_total,
                                            float(clip), float(theta), int(vdtype == np.float64), ptr(d_out)))

    return _ops.write_dense(dx, n, g, vdtype, launch)


def normalize_pearson_residuals(adata, *, theta: float = 100, clip: float | None = None, check_values: bool = True,
                                layer: str | None = None, obsm: str | None = None, inplace: bool = True,
                                copy: bool = False):
    """Apply analytic Pearson residual normalization (signature of
    `scanpy.experimental.pp.normalize_pearson_residuals`)."""
    if copy:
        if not inplace:
            raise ValueError("`copy=True` cannot be used with `inplace=False`.")
        adata = adata.copy()
    x = get_arr(adata, layer=layer, obsm=obsm)
    computed_on = layer or obsm or "adata.X"
    start = log_start(f"computing analytic Pearson residuals on {computed_on}")
    residuals = _pearson_residuals(x, theta, clip, check_values)
    settings_dict = dict(theta=theta, clip=clip, computed_on=computed_on)
    if inplace:
        if layer is not None:
            adata.layers[layer] = residuals
        elif obsm is not None:
            adata.obsm[obsm] = residuals
        else:
            adata.X = residuals
        adata.uns["pearson_residuals_normalization"] = settings_dict
    else:
        results_dict = dict(X=residuals, **settings_dict)
    log_done(start)
    if copy:
        return adata
    if not inplace:
        return results_dict
    return None


# ------------------------------------------------------------------------------------------ PCA and the recipe
def _pca_keys(kwargs_pca):
    key_added = kwargs_pca.get("key_added", None)
    return ("pca", "X_pca", "PCs") if key_added is None else (key_added,) * 3


def _new_like(adata, x, *, obs, var):
    """A fresh object of the input's AnnData type holding only X, the obs / var index."""
    return type(adata)(x, obs=obs, var=var)


def _to_df(ad) -> pd.DataFrame:
    if hasattr(ad, "to_df"):
        return ad.to_df()
    x = ad.X.toarray() if sparse.issparse(ad.X) else ad.X
    return pd.DataFrame(x, index=ad.obs.index, columns=ad.var.index)


def _write_pca(adata, adata_pca, keys, mask_var, n_comps: int) -> None:
    k_uns, k_obsm, k_varm = keys
    norm_settings = adata_pca.uns["pearson_residuals_normalization"]
    norm_dict = dict(**norm_settings, pearson_residuals_df=_to_df(adata_pca))
    if mask_var is not None:
        adata.varm[k_varm] = np.zeros(shape=(adata.n_vars, n_comps))
        adata.varm[k_varm][mask_var] = adata_pca.varm[k_varm]
    else:
        adata.varm[k_varm] = adata_pca.varm[k_varm]
    adata.uns[k_uns] = adata_pca.uns[k_uns]
    adata.uns["pearson_residuals_normalization"] = norm_dict
    adata.obsm[k_obsm] = adata_pca.obsm[k_obsm]


@accepts_legacy_random_state(0)
def normalize_pearson_residuals_pca(adata, *, theta: float = 100, clip: float | None = None, n_comps: int | None = 50,
                                    rng=None, kwargs_pca=MappingProxyType({}), mask_var=_DEFAULT,
                                    check_values: bool = True, layer: str | None = None, inplace: bool = True):
    """Pearson residual normalization and PCA (signature of `scanpy.experimental.pp.normalize_pearson_residuals_pca`).
    `layer` takes the counts from `adata.layers[layer]` instead of `adata.X`."""
    from .pp import _check_mask, pca

    keys = _pca_keys(kwargs_pca)
    if mask_var is _DEFAULT:
        mask_var = "highly_variable" if "highly_variable" in adata.var else None
    mask_var = _check_mask(adata, mask_var, "var")
    _check_theta_clip(theta, clip)
    counts = get_arr(adata, layer=layer)
    _check_x(counts, "normalize_pearson_residuals")
    if mask_var is not None:
        counts = counts[:, mask_var]
        obs, var = adata.obs[[]], adata.var.loc[mask_var][[]]
    else:
        obs, var = adata.obs[[]], adata.var[[]]
    adata_pca = _new_like(adata, counts.copy(), obs=obs.copy(), var=var.copy())
    normalize_pearson_residuals(adata_pca, theta=theta, clip=clip, check_values=check_values)
    pca(adata_pca, n_comps=n_comps, rng=rng, **kwargs_pca)
    n_comps = adata_pca.obsm[keys[1]].shape[1]
    if inplace:
        _write_pca(adata, adata_pca, keys, mask_var, n_comps)
        return None
    return adata_pca


@accepts_legacy_random_state(0)
def recipe_pearson_residuals(adata, *, theta: float = 100, clip: float | None = None, n_top_genes: int = 1000,
                             batch_key: str | None = None, chunksize: int = 1000, n_comps: int | None = 50, rng=None,
                             kwargs_pca=MappingProxyType({}), check_values: bool = True, layer: str | None = None,
                             inplace: bool = True):
    """Gene selection, normalization and PCA by analytic Pearson residuals (signature of
    `scanpy.experimental.pp.recipe_pearson_residuals`).  `layer` takes the counts from `adata.layers[layer]` instead
    of `adata.X`.  Returns `(adata_pca, hvg)` with `inplace=False`."""
    from .pp import pca

    keys = _pca_keys(kwargs_pca)
    if not is_anndata_like(adata):
        raise ValueError("`pp.highly_variable_genes` expects an `AnnData` argument, pass `inplace=False` if you want "
                         "to return a `pd.DataFrame`.")
    _check_theta_clip(theta, clip)
    _check_x(get_arr(adata, layer=layer), "highly_variable_genes")
    hvg_args = dict(flavor="pearson_residuals", n_top_genes=n_top_genes, batch_key=batch_key, theta=theta, clip=clip,
                    chunksize=chunksize, check_values=check_values, layer=layer)
    if inplace:
        highly_variable_genes(adata, **hvg_args, inplace=True)
        mask = np.asarray(adata.var["highly_variable"], dtype=bool)
    else:
        hvg = highly_variable_genes(adata, **hvg_args, inplace=False)
        mask = np.asarray(hvg["highly_variable"], dtype=bool)
    adata_pca = adata[:, mask].copy()
    if layer is not None:
        adata_pca.X = get_arr(adata, layer=layer)[:, mask].copy()
    normalize_pearson_residuals(adata_pca, theta=theta, clip=clip, check_values=check_values)
    pca(adata_pca, n_comps=n_comps, rng=rng, **kwargs_pca)
    if inplace:
        _write_pca(adata, adata_pca, keys, mask, n_comps)
        return None
    return adata_pca, hvg

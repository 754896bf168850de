"""`sc.pp.normalize_total`, `sc.pp.log1p`, `sc.pp.highly_variable_genes(flavor='seurat')` on the device
(SURVEY.md 8f row f2: the CSR passes in front of the hot path).

References: src/scanpy/preprocessing/_normalization.py:127-306, src/scanpy/preprocessing/_simple.py:310-425,
src/scanpy/preprocessing/_highly_variable_genes.py:300-385,452-560,630-844.  The per-non-zero work (row totals,
row scaling, log1p, per-gene sums of expm1) runs in csrc/preprocess.cu; the per-gene binning / z-scoring of
`highly_variable_genes` is g-sized pandas logic and stays on the host exactly as the reference writes it.
Only scipy CSR (or dense, converted) float/int `.X` is supported; other options raise NotImplementedError.
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse

from . import _abi, _ops
from ._abi import check, ptr
from ._compat import is_anndata_like, log_done, log_start, warn


def _as_csr32(x):
    if not sparse.issparse(x):
        x = sparse.csr_matrix(np.asarray(x))
    x = x.tocsr()
    if x.dtype != np.float32:
        x = x.astype(np.float32)
    return x


def normalize_total(adata, *, target_sum: float | None = None, exclude_highly_expressed: bool = False,
                    max_fraction: float = 0.05, key_added: str | None = None, layer: str | None = None,
                    obsm: str | None = None, inplace: bool = True, copy: bool = False):
    """Normalize counts per cell (signature of `scanpy.pp.normalize_total`)."""
    import torch

    if copy:
        if not inplace:
            raise ValueError("`copy=True` cannot be used with `inplace=False`.")
        adata = adata.copy()
    if max_fraction < 0 or max_fraction > 1:
        raise ValueError("Choose max_fraction between 0 and 1.")
    if layer is not None or obsm is not None:
        raise NotImplementedError("`layer`/`obsm` are not implemented in scanpy_b200.pp.normalize_total")
    start = log_start("normalizing counts per cell")
    x = _as_csr32(adata.X)
    n, g = x.shape
    ctx = _abi.default_context()
    d_indptr, d_indices, d_data = _ops.csr_to_device(x)
    counts = torch.empty(n, dtype=torch.float32, device="cuda")
    check(ctx.lib.sb2_csr_row_sums_f32(ctx.handle, n, ptr(d_indptr), ptr(d_indices), ptr(d_data), None, ptr(counts)))
    gene_subset = None
    if exclude_highly_expressed:
        per_col = torch.empty(g, dtype=torch.int32, device="cuda")
        check(ctx.lib.sb2_csr_hiexpr_count_f32(ctx.handle, n, g, ptr(d_indptr), ptr(d_indices), ptr(d_data), ptr(counts),
                                               float(max_fraction), ptr(per_col)))
        check(ctx.lib.sb2_csr_row_sums_f32(ctx.handle, n, ptr(d_indptr), ptr(d_indices), ptr(d_data), ptr(per_col),
                                           ptr(counts)))
        gene_subset = _ops._to_host(per_col) == 0
    counts_per_cell = _ops._to_host(counts).copy()
    if target_sum is None:
        target_sum = np.median(counts_per_cell[counts_per_cell > 0])  # _compute_nnz_median (:20-26)
    counts_per_cell = counts_per_cell / target_sum
    if not np.all(counts_per_cell > 0):
        warn("Some cells have zero counts", UserWarning)
    d_scale = _ops._to_device(counts_per_cell.astype(np.float32))
    check(ctx.lib.sb2_csr_scale_rows_f32(ctx.handle, n, ptr(d_indptr), ptr(d_data), ptr(d_scale)))
    x_new = sparse.csr_matrix((_ops._to_host(d_data), x.indices, x.indptr), shape=x.shape)
    if exclude_highly_expressed:
        names = list(adata.var_names[~gene_subset]) if hasattr(adata, "var_names") else np.flatnonzero(~gene_subset).tolist()
        log_start(f"The following highly-expressed genes are not considered during normalization factor computation:\n{names}")
    dat = dict(X=x_new, norm_factor=counts_per_cell)
    if inplace:
        if key_added is not None:
            adata.obs[key_added] = dat["norm_factor"]
        adata.X = dat["X"]
    log_done(start)
    if copy:
        return adata
    if not inplace:
        return dat
    return None


def log1p(data, *, base=None, copy: bool = False, chunked=None, chunk_size=None, layer=None, obsm=None):
    """Logarithmize the data matrix: X = log(X + 1) (signature of `scanpy.pp.log1p`)."""
    if chunked or layer is not None or obsm is not None:
        raise NotImplementedError("`chunked`/`layer`/`obsm` are not implemented in scanpy_b200.pp.log1p")
    ctx = _abi.default_context()

    def run(x):
        xs = _as_csr32(x)
        d = _ops._to_device(xs.data)
        check(ctx.lib.sb2_log1p_f32(ctx.handle, xs.nnz, ptr(d), 0.0 if base is None else float(base)))
        out = sparse.csr_matrix((_ops._to_host(d), xs.indices, xs.indptr), shape=xs.shape)
        return out if sparse.issparse(x) else out.toarray()

    if is_anndata_like(data):
        adata = data.copy() if copy else data
        if "log1p" in adata.uns:
            warn("adata.X seems to be already log-transformed.", UserWarning)  # _simple.py:404-405
        adata.X = run(adata.X)
        adata.uns["log1p"] = {"base": base}
        return adata if copy else None
    return run(data)


def _col_mean_var_expm1(x_log, log_scale: float):
    """per-gene mean / variance (ddof=1) of expm1(x*log_scale) without materialising it on the host."""
    import torch

    ctx = _abi.default_context()
    xs = _as_csr32(x_log)
    n, g = xs.shape
    d_idx = _ops._to_device(np.asarray(xs.indices, np.int32))
    d_dat = _ops._to_device(xs.data)
    s1 = torch.empty(g, dtype=torch.float64, device="cuda")
    s2 = torch.empty(g, dtype=torch.float64, device="cuda")
    check(ctx.lib.sb2_csr_col_sums_f32(ctx.handle, xs.nnz, g, ptr(d_idx), ptr(d_dat), 1, float(log_scale), ptr(s1), ptr(s2)))
    h1, h2 = _ops._to_host(s1, s2)
    mean = h1 / n
    var = (h2 / n - mean**2) * (n / (n - 1))  # fast_array_utils.stats.mean_var(..., correction=1)
    return mean, var


def _hvg_seurat_frame(x_log, base, *, n_top_genes: int | None = None, min_disp: float = 0.5, max_disp: float = np.inf,
                      min_mean: float = 0.0125, max_mean: float = 3, n_bins: int = 20) -> pd.DataFrame:
    """The seurat flavour's per-gene table of a log1p'd matrix (natural log when `base` is None): means, dispersions,
    dispersions_norm and highly_variable, on a RangeIndex.  Shared by `highly_variable_genes` and `pp.scrublet`, which
    selects genes on a log1p copy of its matrix."""
    mean, var = _col_mean_var_expm1(x_log, 1.0 if base is None else float(np.log(base)))
    # --- per-gene logic, verbatim from _highly_variable_genes.py:347-385,452-560 ---
    mean[mean == 0] = 1e-12
    dispersion = var / mean
    dispersion[dispersion == 0] = np.nan
    with np.errstate(invalid="ignore", divide="ignore"):
        dispersion = np.log(dispersion)
    mean = np.log1p(mean)
    df = pd.DataFrame(dict(means=mean, dispersions=dispersion))
    rv = pd.cut(df["means"], bins=n_bins)
    df["mean_bin"] = rv.cat.set_categories(rv.cat.categories.astype("string"), rename=True)
    stats = df.groupby("mean_bin", observed=True)["dispersions"].agg(avg="mean", dev="std")
    one_gene_per_bin = stats["dev"].isna()
    stats.loc[one_gene_per_bin, "dev"] = stats.loc[one_gene_per_bin, "avg"]
    stats.loc[one_gene_per_bin, "avg"] = 0
    per_gene = stats.loc[df["mean_bin"]].set_index(df.index)
    df["dispersions_norm"] = (df["dispersions"] - per_gene["avg"]) / per_gene["dev"]
    dn = df["dispersions_norm"].to_numpy()
    if n_top_genes is None:
        dnz = np.nan_to_num(dn)
        hv = (mean > min_mean) & (mean < max_mean) & (dnz > min_disp) & (dnz < max_disp)
    else:
        v = dn[~np.isnan(dn)]
        n = n_top_genes
        if n > v.size:
            warn(f"`n_top_genes` (={n}) > number of normalized dispersions (={v.size}), returning all genes with "
                 "normalized dispersions.", UserWarning)
            n = v.size
        v = np.sort(v)[::-1]
        hv = np.nan_to_num(dn, nan=-np.inf) >= v[n - 1]
    df["highly_variable"] = hv
    return df.drop(columns=["mean_bin"])


def highly_variable_genes(adata, *, layer=None, n_top_genes: int | None = None, min_disp: float = 0.5,
                          max_disp: float = np.inf, min_mean: float = 0.0125, max_mean: float = 3, span: float = 0.3,
                          n_bins: int = 20, flavor: str = "seurat", subset: bool = False, inplace: bool = True,
                          batch_key=None, filter_unexpressed_genes=None, check_values: bool = True):
    """Annotate highly variable genes (signature of `scanpy.pp.highly_variable_genes`; flavor='seurat' only)."""
    if flavor != "seurat":
        raise NotImplementedError(f"flavor={flavor!r}: only 'seurat' is implemented in scanpy_b200")
    if batch_key is not None or layer is not None:
        raise NotImplementedError("`batch_key`/`layer` are not implemented in scanpy_b200.pp.highly_variable_genes")
    start = log_start("extracting highly variable genes")
    if n_top_genes is not None and (min_disp, max_disp, min_mean, max_mean) != (0.5, np.inf, 0.0125, 3):
        warn("If you pass `n_top_genes`, all cutoffs are ignored.", UserWarning)
    base = adata.uns.get("log1p", {}).get("base")
    df = _hvg_seurat_frame(adata.X, base, n_top_genes=n_top_genes, min_disp=min_disp, max_disp=max_disp,
                           min_mean=min_mean, max_mean=max_mean, n_bins=n_bins)
    df.index = adata.var.index
    log_done(start)
    if inplace:
        adata.uns["hvg"] = {"flavor": flavor}
        adata.var["highly_variable"] = df["highly_variable"].to_numpy()
        adata.var["means"] = df["means"].to_numpy()
        adata.var["dispersions"] = df["dispersions"].to_numpy()
        adata.var["dispersions_norm"] = df["dispersions_norm"].to_numpy().astype("float32", copy=False)
        if subset:
            raise NotImplementedError("`subset=True` needs AnnData._inplace_subset_var; subset with adata[:, mask] instead")
        return None
    if subset:
        df = df.iloc[df["highly_variable"].to_numpy(), :]
    return df


def _scale_array(x, *, zero_center: bool, max_value, mask_obs):
    """`scale_array` / `scale_array_masked` (src/scanpy/preprocessing/_scale.py:150-264) on the device.
    -> (scaled x, mean float64[g], std float64[g])."""
    import torch

    ctx = _abi.default_context()
    n, g = x.shape
    has_max = 0 if max_value is None else 1
    mx = 0.0 if max_value is None else float(max_value)
    d_mask = None if mask_obs is None else _ops._to_device(np.ascontiguousarray(mask_obs, dtype=np.uint8))
    n_sel = n if mask_obs is None else int(np.count_nonzero(mask_obs))
    s1 = torch.empty(g, dtype=torch.float64, device="cuda")
    s2 = torch.empty(g, dtype=torch.float64, device="cuda")
    is_sparse = sparse.issparse(x)
    if is_sparse:
        xs = _as_csr32(x)
        # the reference's statistics (`x.multiply(x)`) and densification sum duplicate entries first; the kernels see one
        # value per (row, column).  The uncentred output below keeps x's own entries, each divided and clipped.
        xc = xs
        if not xs.has_canonical_format:
            xc = xs.copy()
            xc.sum_duplicates()
        d_indptr, d_indices, d_data = _ops.csr_to_device(xc)
        check(ctx.lib.sb2_csr_col_stats_rows_f32(ctx.handle, n, g, ptr(d_indptr), ptr(d_indices), ptr(d_data),
                                                 ptr(d_mask) if d_mask is not None else None, ptr(s1), ptr(s2)))
    else:
        xd = np.ascontiguousarray(x)
        if np.issubdtype(xd.dtype, np.integer):
            xd = xd.astype(np.float64)  # "integer input is cast to float" (_scale.py:181-186)
        if xd.dtype not in (np.float32, np.float64):
            xd = xd.astype(np.float32)
        is64 = int(xd.dtype == np.float64)
        d_x = _ops._to_device(xd)
        check(ctx.lib.sb2_dense_col_stats(ctx.handle, n, g, ptr(d_x), is64, ptr(d_mask) if d_mask is not None else None,
                                          ptr(s1), ptr(s2)))
    # mean_var(..., correction=1) (fast_array_utils.stats): var = (E[x^2] - E[x]^2) * n / (n - 1); g-sized, on the device
    mean = s1 / n_sel
    var = (s2 / n_sel - mean * mean) * (n_sel / (n_sel - 1)) if n_sel > 1 else torch.full_like(mean, float("nan"))
    std = torch.sqrt(var)
    std[std == 0] = 1
    if is_sparse and not zero_center:
        if xc is not xs:
            d_indptr, d_indices, d_data = _ops.csr_to_device(xs)
        check(ctx.lib.sb2_csr_scale_cols_f32(ctx.handle, n, ptr(d_indptr), ptr(d_indices), ptr(d_data), ptr(std),
                                             ptr(d_mask) if d_mask is not None else None, has_max, mx))
        out = sparse.csr_matrix((_ops._to_host(d_data), xs.indices, xs.indptr), shape=xs.shape)
    elif is_sparse:
        warn("zero-centering a sparse array/matrix densifies it.", UserWarning)
        d_out = torch.empty((n, g), dtype=torch.float64, device="cuda")
        check(ctx.lib.sb2_csr_scale_dense_f64(ctx.handle, n, g, ptr(d_indptr), ptr(d_indices), ptr(d_data), ptr(mean),
                                              ptr(std), ptr(d_mask) if d_mask is not None else None, has_max, mx,
                                              ptr(d_out)))
        out = _ops._to_host(d_out)
        if mask_obs is not None:  # the reference assigns the dense block back into the sparse matrix (_scale.py:251-256)
            out = sparse.csr_matrix(out)
    else:
        check(ctx.lib.sb2_dense_scale(ctx.handle, n, g, ptr(d_x), is64, ptr(mean) if zero_center else None, ptr(std),
                                      ptr(d_mask) if d_mask is not None else None, has_max, mx))
        out = _ops._to_host(d_x)
    h_mean, h_std = _ops._to_host(mean, std)
    return out, h_mean.copy(), h_std.copy()


def scale(data, *, zero_center: bool = True, max_value: float | None = None, copy: bool = False, layer: str | None = None,
          obsm: str | None = None, mask_obs=None):
    """Scale data to unit variance and zero mean (signature of `scanpy.pp.scale`, _scale.py:72-147,286-327; the V1
    preset's `zero_center=True` default)."""
    if layer is not None or obsm is not None:
        raise NotImplementedError("`layer`/`obsm` are not implemented in scanpy_b200.pp.scale")
    if not zero_center and max_value is not None:
        log_start("... be careful when using `max_value` without `zero_center`.")
    if is_anndata_like(data):
        adata = data.copy() if copy else data
        names = ("mean", "std")
        if mask_obs is not None:
            names = (f"mean of {mask_obs}", f"std of {mask_obs}") if isinstance(mask_obs, str) else ("mean with mask", "std with mask")
            from .pp import _check_mask

            mask_obs = _check_mask(adata, mask_obs, "obs")
        x, mean, std = _scale_array(adata.X, zero_center=zero_center, max_value=max_value, mask_obs=mask_obs)
        adata.var[names[0]] = mean
        adata.var[names[1]] = std
        adata.X = x
        return adata if copy else None
    x = data
    if isinstance(mask_obs, str):
        raise ValueError("Cannot use refererence for mask without providing anndata object as argument")
    if sparse.issparse(x) and x.format == "csc":
        x = x.tocsr()
    if mask_obs is not None:
        mask_obs = np.asarray(mask_obs)
        if mask_obs.dtype != bool:
            raise ValueError("Mask array must be boolean.")
        if len(mask_obs) != x.shape[0]:
            raise ValueError("The shape of the mask do not match the data.")
    out, _, _ = _scale_array(x, zero_center=zero_center, max_value=max_value, mask_obs=mask_obs)
    return out

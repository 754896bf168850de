"""normalize_total / log1p / highly_variable_genes(flavor='seurat') oracle (test infrastructure only).

numpy/pandas restatements of the reference's own code (scanpy itself cannot be imported here: anndata,
fast_array_utils, ... are missing):
  normalize_total  src/scanpy/preprocessing/_normalization.py:20-125 (incl. the numba `_normalize_csr`)
  log1p            src/scanpy/preprocessing/_simple.py:359-380
  HVG seurat       src/scanpy/preprocessing/_highly_variable_genes.py:300-385,452-560
Pinned by: the docstring example of normalize_total (_normalization.py:205-241), tests/test_normalization.py:30-71
and the Seurat-produced golden tests/_scripts/seurat_hvg.csv on pbmc68k_reduced (tests/test_highly_variable_genes.py:379-421).
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse


def normalize_total(x, *, target_sum=None, exclude_highly_expressed=False, max_fraction=0.05):
    """-> (x_normalised CSR float32, counts_per_cell / target_sum, gene_subset or None)."""
    x = sparse.csr_matrix(x).astype(np.float32) if not np.issubdtype(x.dtype, np.floating) else sparse.csr_matrix(x).copy()
    n, g = x.shape
    rowid = np.repeat(np.arange(n), np.diff(x.indptr))
    counts_per_cell = np.zeros(n, np.float64)
    np.add.at(counts_per_cell, rowid, x.data.astype(np.float64))
    counts_per_cell = counts_per_cell.astype(x.dtype)
    gene_subset = None
    if exclude_highly_expressed:
        hi = x.data.astype(np.float64) > max_fraction * counts_per_cell[rowid].astype(np.float64)
        counts_per_cols = np.bincount(x.indices[hi], minlength=g).astype(np.int32)
        keep = counts_per_cols[x.indices] == 0
        c2 = np.zeros(n, np.float64)
        np.add.at(c2, rowid[keep], x.data[keep].astype(np.float64))
        counts_per_cell = c2.astype(x.dtype)
        gene_subset = counts_per_cols == 0
    if target_sum is None:
        target_sum = np.median(counts_per_cell[counts_per_cell > 0])
    counts_per_cell = counts_per_cell / target_sum
    scaling = counts_per_cell.copy() + (counts_per_cell == 0)
    x.data = np.true_divide(x.data, np.repeat(scaling, np.diff(x.indptr))).astype(x.dtype)
    return x, counts_per_cell, gene_subset


def log1p(x, *, base=None):
    x = x.copy()
    np.log1p(x.data, out=x.data)
    if base is not None:
        np.divide(x.data, np.log(base), out=x.data)
    return x


def mean_var_cols(x, *, correction=1):
    """fast_array_utils.stats.mean_var(axis=0, correction=1): float64 mean and mean of squares."""
    n = x.shape[0]
    xd = x.astype(np.float64)
    mean = np.asarray(xd.mean(axis=0)).ravel()
    mean_sq = np.asarray(xd.multiply(xd).mean(axis=0)).ravel()
    var = mean_sq - mean**2
    if correction:
        var *= n / (n - correction)
    return mean, var


def hvg_seurat(x_log, *, n_top_genes=None, min_disp=0.5, max_disp=np.inf, min_mean=0.0125, max_mean=3.0, n_bins=20,
               log_base=None):
    """highly_variable_genes(flavor='seurat') on log1p data -> DataFrame(means, dispersions, dispersions_norm, highly_variable)."""
    x = x_log.copy()
    if log_base is not None:
        x.data *= np.log(log_base)
    x.data = np.expm1(x.data)
    mean, var = mean_var_cols(x)
    return hvg_seurat_from_stats(mean, var, n_top_genes=n_top_genes, min_disp=min_disp, max_disp=max_disp,
                                 min_mean=min_mean, max_mean=max_mean, n_bins=n_bins)


def hvg_seurat_from_stats(mean, var, *, n_top_genes=None, min_disp=0.5, max_disp=np.inf, min_mean=0.0125,
                          max_mean=3.0, n_bins=20):
    mean = mean.copy()
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
    one = stats["dev"].isna()
    stats.loc[one, "dev"] = stats.loc[one, "avg"]
    stats.loc[one, "avg"] = 0
    per_gene = stats.loc[df["mean_bin"]].set_index(df.index)
    df["dispersions_norm"] = (df["dispersions"] - per_gene["avg"]) / per_gene["dev"]
    dn = df["dispersions_norm"].to_numpy()
    if n_top_genes is None:
        dnz = np.nan_to_num(dn)
        hv = (mean > min_mean) & (mean < max_mean) & (dnz > min_disp) & (dnz < max_disp)
    else:
        v = dn[~np.isnan(dn)]
        n = min(n_top_genes, v.size)
        v = np.sort(v)[::-1]
        hv = np.nan_to_num(dn, nan=-np.inf) >= v[n - 1]
    df["highly_variable"] = hv
    return df.drop(columns=["mean_bin"])


def scale(x, *, zero_center=True, max_value=None, mask_obs=None, stats=None):
    """`scale_array` / `scale_array_masked` / `clip_array` / `scale_and_clip_csr`
    (src/scanpy/preprocessing/_scale.py:52-69,150-283) restated in numpy -> (x_scaled, mean, std).
    Pinned by the reference's goldens in tests/test_scaling.py:15-53 (X_original / X_scaled_original /
    X_centered_original and their clipped / masked variants, reproduced in tests/golden/).
    `stats=(mean, std)` skips the statistics and applies the arithmetic with the given float64 mean and std (a zero std
    is used as given), so the scaling step can be compared on its own."""
    sp = sparse.issparse(x)
    if sp:
        x = sparse.csr_matrix(x).copy()
    else:
        x = np.array(x, copy=True)
    if np.issubdtype(x.dtype, np.integer):
        x = x.astype(np.float64)
    sel = slice(None) if mask_obs is None else np.asarray(mask_obs, bool)
    sub = x[sel, :]
    n = sub.shape[0]
    if stats is not None:
        mean, std = (np.asarray(s, np.float64) for s in stats)
    else:
        if sp:
            d64 = sub.astype(np.float64)
            mean = np.asarray(d64.mean(axis=0)).ravel()
            mean_sq = np.asarray(d64.multiply(d64).mean(axis=0)).ravel()
        else:
            mean = sub.mean(axis=0, dtype=np.float64)
            mean_sq = np.multiply(sub, sub, dtype=np.float64).mean(axis=0, dtype=np.float64)
        var = (mean_sq - mean**2) * (n / (n - 1))
        std = np.sqrt(var)
        std[std == 0] = 1
    if sp and not zero_center:
        rows = np.repeat(np.arange(x.shape[0]), np.diff(x.indptr))
        on = np.ones(x.nnz, bool) if mask_obs is None else np.asarray(mask_obs, bool)[rows]
        v = x.data.astype(np.float64) / std[x.indices]
        if max_value is not None:
            v = np.minimum(max_value, v)
        x.data[on] = v[on].astype(x.dtype)
        return x, mean, std
    if sp:
        assert mask_obs is None
        out = np.asarray(x.todense()) - mean  # `x -= mean` on a sparse matrix: todense (in x.dtype), then float64
        out = out / std
    else:
        out = sub.copy()
        if zero_center:
            out -= mean  # in place: rounded to x.dtype
        out /= std
    if max_value is not None:
        out[out > max_value] = max_value
        if zero_center:
            out[out < -max_value] = -max_value
    if not sp and mask_obs is not None:
        full = x.copy()
        full[sel, :] = out
        out = full
    return out, mean, std

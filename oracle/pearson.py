"""Analytic Pearson residuals oracle (test infrastructure only): numpy restatements, in fp64 and vectorised over gene
blocks, of
  _pearson_residuals                   src/scanpy/experimental/pp/_normalization.py:36-75
  _highly_variable_pearson_residuals   src/scanpy/experimental/pp/_highly_variable_genes.py:129-287
with the reference's quirks: batches in `np.unique` order; `clip=None` becomes sqrt(n) of the first batch and every
later batch reuses it; genes with zero total in a batch are left out of it and get residual variance 0; NaN residuals
(0 / 0 for a zero-total cell or gene) survive the clip.  The residual variance is the reference's two-pass population
variance.  Totals are fp64 (the reference sums a float32 X in float32; for integer counts below 2^24 both agree).
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse

GENE_BLOCK = 256


def _dense64(x):
    return x.toarray().astype(np.float64) if sparse.issparse(x) else np.asarray(x, dtype=np.float64)


def _clip(r, clip):
    """np.clip / numba's min(max(r, -clip), clip): NaN stays NaN."""
    r = np.where(r < -clip, -clip, r)
    return np.where(r > clip, clip, r)


def _residual_block(xb, sums_genes, sums_cells, sum_total, clip, theta):
    mu = np.outer(sums_cells, sums_genes) / sum_total
    with np.errstate(invalid="ignore", divide="ignore"):
        r = (xb - mu) / np.sqrt(mu + mu * mu / theta)
    return _clip(r, clip)


def pearson_residuals(x, *, theta=100.0, clip=None):
    """The reference's normalised matrix, in fp64 (round to float32 for a float32 X to compare)."""
    xd = _dense64(x)
    n, g = xd.shape
    if clip is None:
        clip = np.sqrt(n)
    sums_genes = xd.sum(axis=0)
    sums_cells = xd.sum(axis=1)
    sum_total = np.sum(sums_genes)
    out = np.empty((n, g))
    for j0 in range(0, g, GENE_BLOCK):
        j1 = min(g, j0 + GENE_BLOCK)
        out[:, j0:j1] = _residual_block(xd[:, j0:j1], sums_genes[j0:j1], sums_cells, sum_total, clip, theta)
    return out


def residual_variances(xb, *, theta, clip):
    """_calculate_res_dense on one batch (zero genes already removed): two-pass population variance per gene."""
    n, g = xb.shape
    sums_genes = xb.sum(axis=0)
    sums_cells = xb.sum(axis=1)
    sum_total = np.sum(sums_genes)
    out = np.empty(g)
    for j0 in range(0, g, GENE_BLOCK):
        j1 = min(g, j0 + GENE_BLOCK)
        r = _residual_block(xb[:, j0:j1], sums_genes[j0:j1], sums_cells, sum_total, clip, theta)
        mean = r.sum(axis=0) / n
        out[j0:j1] = ((r - mean) ** 2).sum(axis=0) / n
    return out


def batch_residual_variances(x, *, theta=100.0, clip=None, batch=None):
    """[n_batches x g] residual variances and the clip of the first batch, with the reference's per-batch loop."""
    xd = _dense64(x)
    n, g = xd.shape
    batch_info = np.zeros(n, dtype=int) if batch is None else np.asarray(batch)
    out = []
    for b in np.unique(batch_info):
        xb = xd[batch_info == b]
        nonzero_genes = xb.sum(axis=0) != 0
        if clip is None:
            clip = np.sqrt(xb.shape[0])
        v = np.zeros(g)
        v[nonzero_genes] = residual_variances(xb[:, nonzero_genes], theta=theta, clip=clip)
        out.append(v)
    return np.stack(out), clip


def mean_var(x):
    """mean_var(x, axis=0, correction=1) from fp64 sums: mean = Σx / n, var = (Σx² / n - mean²) n / (n - 1)."""
    xd = _dense64(x)
    n = xd.shape[0]
    means = xd.sum(axis=0) / n
    return means, ((xd * xd).sum(axis=0) / n - means**2) * (n / (n - 1))


def highly_variable_pearson_residuals(x, *, theta=100.0, clip=None, n_top_genes=1000, batch=None, var_names=None):
    """The reference's DataFrame for `inplace=False, subset=False` (all columns kept, genes in var order)."""
    residual_gene_vars, _ = batch_residual_variances(x, theta=theta, clip=clip, batch=batch)
    n_batches = residual_gene_vars.shape[0]
    ranks_residual_var = np.argsort(np.argsort(-residual_gene_vars, axis=1), axis=1).astype(np.float32)
    highly_variable_nbatches = np.sum((ranks_residual_var < n_top_genes).astype(int), axis=0)
    ranks_residual_var[ranks_residual_var >= n_top_genes] = np.nan
    medianrank = np.ma.median(np.ma.masked_invalid(ranks_residual_var), axis=0).filled(np.nan)
    means, variances = mean_var(x)
    index = pd.Index(var_names if var_names is not None else [str(i) for i in range(x.shape[1])])
    df = pd.DataFrame.from_dict(dict(
        means=means, variances=variances, residual_variances=np.mean(residual_gene_vars, axis=0),
        highly_variable_rank=medianrank, highly_variable_nbatches=highly_variable_nbatches.astype(np.int64),
        highly_variable_intersection=highly_variable_nbatches == n_batches)).set_index(index)
    df = df.sort_values(["highly_variable_nbatches", "highly_variable_rank"], ascending=[False, True],
                        na_position="last")
    high_var = np.zeros(df.shape[0], dtype=bool)
    high_var[:n_top_genes] = True
    df["highly_variable"] = high_var
    return df.loc[index, :], residual_gene_vars

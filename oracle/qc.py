"""calculate_qc_metrics / filter_cells / filter_genes oracle (test infrastructure only).

numpy/pandas restatements of the reference's own code (scanpy cannot be imported here: anndata, numba,
fast_array_utils are missing):
  describe_obs / describe_var            src/scanpy/preprocessing/_qc.py:41-196
  top_proportions(_dense/_sparse_csr)    src/scanpy/preprocessing/_qc.py:310-360
  top_segment_proportions (dense, CSR)   src/scanpy/preprocessing/_qc.py:376-457 (the numba CSR kernel, line by line)
  filter_cells / filter_genes            src/scanpy/preprocessing/_simple.py:53-306
Sums accumulate in fp64 (the reference accumulates in X's dtype; for integer-valued data both agree) and are then cast
to the dtype the reference returns for X's dtype.  Pinned by the reference's tests/test_qc_metrics.py, the
filter_cells docstring on krumsiek11 (_simple.py:104-133) and tests/test_preprocessing.py:611-676.
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse


def sum_dtype(dtype) -> np.dtype:
    dtype = np.dtype(dtype)
    if dtype.kind in "biu":
        return np.dtype(np.int64)
    return np.dtype(np.float64) if dtype == np.float64 else np.dtype(np.float32)


def _row_sums64(x) -> np.ndarray:
    if sparse.issparse(x):
        return np.asarray(x.astype(np.float64).sum(axis=1)).ravel()
    return np.asarray(x, dtype=np.float64).sum(axis=1)


def _col_sums64(x) -> np.ndarray:
    if sparse.issparse(x):
        return np.asarray(x.astype(np.float64).sum(axis=0)).ravel()
    return np.asarray(x, dtype=np.float64).sum(axis=0)


# ------------------------------------------------------------------------------------------ top-n proportions
def top_proportions(mtx, n: int) -> np.ndarray:
    """_qc.py:310-360: cumulative proportions of the 1..n largest values per row."""
    if sparse.issparse(mtx):
        mtx = sparse.csr_matrix(mtx)
        values = np.zeros((mtx.shape[0], n), dtype=np.float64)
        for i in range(mtx.shape[0]):
            start, end = mtx.indptr[i], mtx.indptr[i + 1]
            vec = np.zeros(n, dtype=np.float64)
            if end - start <= n:
                vec[: end - start] = mtx.data[start:end]
                total = vec.sum()
            else:
                vec[:] = -(np.partition(-mtx.data[start:end], n - 1)[:n])
                total = mtx.data[start:end].sum()
            vec[::-1].sort()
            values[i, :] = vec.cumsum() / total
        return values
    mtx = np.asarray(mtx)
    sums = mtx.sum(axis=1)
    partitioned = np.apply_along_axis(np.argpartition, 1, -mtx, n - 1)[:, :n]
    values = np.zeros_like(partitioned, dtype=np.float64)
    for i in range(partitioned.shape[0]):
        vec = mtx[i, partitioned[i, :]]
        vec[::-1].sort()
        values[i, :] = np.cumsum(vec) / sums[i]
    return values


def check_ns(mtx, ns) -> None:
    """_qc.py:363-373."""
    if not (max(ns) <= mtx.shape[1] and min(ns) > 0):
        raise IndexError("Positions outside range of features.")


def top_segment_sums_csr(data, indptr, ns) -> np.ndarray:
    """The numba `top_segment_proportions_sparse_csr` (_qc.py:430-457) without the final division, in fp64: per row,
    the m = max(ns) largest stored values (a row with at most m stored values: all of them, zero-padded to m), and the
    sum of the n largest of that vector for every n in sorted(ns)."""
    ns = np.sort(np.asarray(ns, dtype=np.int64))
    maxidx = int(ns[-1])
    n_rows = indptr.size - 1
    out = np.zeros((n_rows, ns.size), dtype=np.float64)
    for i in range(n_rows):
        start, end = int(indptr[i]), int(indptr[i + 1])
        vec = np.zeros(maxidx, dtype=np.float64)
        if end - start <= maxidx:
            vec[: end - start] = data[start:end]
        else:
            vec[:] = -(np.partition(-data[start:end].astype(np.float64), maxidx))[:maxidx]
        vec = -np.sort(-vec)
        out[i] = np.cumsum(vec)[ns - 1]
    return out


def top_segment_proportions(mtx, ns) -> np.ndarray:
    """_qc.py:376-427: dense rows partition the full row, sparse rows follow the CSR kernel."""
    check_ns(mtx, ns)
    if sparse.issparse(mtx):
        mtx = sparse.csr_matrix(mtx)
        sums = _row_sums64(mtx)
        return top_segment_sums_csr(mtx.data, mtx.indptr, ns) / sums[:, None]
    mtx = np.asarray(mtx)
    ns = np.sort(ns)
    sums = mtx.sum(axis=1)
    partitioned = np.apply_along_axis(np.partition, 1, mtx, mtx.shape[1] - ns)[:, ::-1][:, : ns[-1]]
    values = np.zeros((mtx.shape[0], len(ns)))
    acc = np.zeros(mtx.shape[0])
    prev = 0
    for j, n in enumerate(ns):
        acc += partitioned[:, prev:n].sum(axis=1)
        values[:, j] = acc
        prev = n
    return values / sums[:, None]


# ------------------------------------------------------------------------------------------ describe_obs / describe_var
def _count_nonzero(x, axis: int) -> np.ndarray:
    if sparse.issparse(x):
        return np.asarray((x != 0).sum(axis=axis), dtype=np.int64).ravel()
    return np.count_nonzero(np.asarray(x), axis=axis).astype(np.int64)


def describe_obs(x, *, obs_names, var, expr_type="counts", var_type="genes", qc_vars=(), percent_top=(50, 100, 200, 500),
                 log1p=True) -> pd.DataFrame:
    """_qc.py:84-129 on X (explicit zeros already eliminated, as calculate_qc_metrics does); the top-n shares follow
    the CSR kernel for every input type, as the device does."""
    sd = sum_dtype(x.dtype)
    obs = pd.DataFrame(index=obs_names)
    obs[f"n_{var_type}_by_{expr_type}"] = _count_nonzero(x, 1)
    if log1p:
        obs[f"log1p_n_{var_type}_by_{expr_type}"] = np.log1p(obs[f"n_{var_type}_by_{expr_type}"])
    total = _row_sums64(x).astype(sd)
    obs[f"total_{expr_type}"] = total
    if log1p:
        obs[f"log1p_total_{expr_type}"] = np.log1p(obs[f"total_{expr_type}"])
    if percent_top:
        ns = sorted(percent_top)
        check_ns(x, ns)
        csr = sparse.csr_matrix(x)
        csr.eliminate_zeros()
        with np.errstate(invalid="ignore", divide="ignore"):
            proportions = top_segment_sums_csr(csr.data, csr.indptr, ns) / total.astype(np.float64)[:, None]
        for i, n in enumerate(ns):
            obs[f"pct_{expr_type}_in_top_{n}_{var_type}"] = proportions[:, i] * 100
    for qc_var in qc_vars:
        mask = var[qc_var].to_numpy()
        sub = x[:, mask]
        obs[f"total_{expr_type}_{qc_var}"] = _row_sums64(sub).astype(sd)
        if log1p:
            obs[f"log1p_total_{expr_type}_{qc_var}"] = np.log1p(obs[f"total_{expr_type}_{qc_var}"])
        with np.errstate(invalid="ignore", divide="ignore"):
            obs[f"pct_{expr_type}_{qc_var}"] = obs[f"total_{expr_type}_{qc_var}"] / obs[f"total_{expr_type}"] * 100
    return obs


def describe_var(x, *, var_names, expr_type="counts", log1p=True) -> pd.DataFrame:
    """_qc.py:172-196."""
    sd = sum_dtype(x.dtype)
    var = pd.DataFrame(index=var_names)
    total = _col_sums64(x).astype(sd)
    var[f"n_cells_by_{expr_type}"] = _count_nonzero(x, 0)
    var[f"mean_{expr_type}"] = total / x.shape[0]
    if log1p:
        var[f"log1p_mean_{expr_type}"] = np.log1p(var[f"mean_{expr_type}"])
    var[f"pct_dropout_by_{expr_type}"] = (1 - var[f"n_cells_by_{expr_type}"] / x.shape[0]) * 100
    var[f"total_{expr_type}"] = total
    if log1p:
        var[f"log1p_total_{expr_type}"] = np.log1p(var[f"total_{expr_type}"])
    return var


def calculate_qc_metrics(x, *, obs_names, var, qc_vars=(), percent_top=(50, 100, 200, 500), log1p=True, **kw):
    """_qc.py:275-307 -> (obs_metrics, var_metrics)."""
    if sparse.issparse(x):
        x = x.copy()
        x.eliminate_zeros()
    if isinstance(qc_vars, str):
        qc_vars = [qc_vars]
    return (describe_obs(x, obs_names=obs_names, var=var, qc_vars=qc_vars, percent_top=percent_top, log1p=log1p, **kw),
            describe_var(x, var_names=var.index, log1p=log1p, **{k: v for k, v in kw.items() if k == "expr_type"}))


# ------------------------------------------------------------------------------------------ filters
def _filter_number(x, axis: int, by_count: bool) -> np.ndarray:
    if by_count:  # stats.sum(data > 0, axis)
        if sparse.issparse(x):
            return np.asarray((x > 0).sum(axis=axis), dtype=np.int64).ravel()
        return np.asarray(np.asarray(x) > 0).sum(axis=axis).astype(np.int64)
    sums = _row_sums64(x) if axis == 1 else _col_sums64(x)
    return sums.astype(sum_dtype(x.dtype))


def filter_cells(x, *, min_counts=None, min_genes=None, max_counts=None, max_genes=None):
    """_simple.py:168-196 -> (cells_subset, number_per_cell)."""
    min_number = min_counts if min_genes is None else min_genes
    max_number = max_counts if max_genes is None else max_genes
    number = _filter_number(x, 1, not (min_genes is None and max_genes is None))
    subset = number >= min_number if min_number is not None else number <= max_number
    return subset, number


def filter_genes(x, *, min_counts=None, min_cells=None, max_counts=None, max_cells=None):
    """_simple.py:282-306 -> (gene_subset, number_per_gene)."""
    min_number = min_counts if min_cells is None else min_cells
    max_number = max_counts if max_cells is None else max_cells
    number = _filter_number(x, 0, not (min_cells is None and max_cells is None))
    subset = number >= min_number if min_number is not None else number <= max_number
    return subset, number

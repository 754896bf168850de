"""`sc.pp.calculate_qc_metrics`, `sc.pp.filter_cells`, `sc.pp.filter_genes` on the device.

References: src/scanpy/preprocessing/_qc.py:41-307,363-373,430-457 and src/scanpy/preprocessing/_simple.py:53-306.  The
per-non-zero work (per-cell counts, totals, gene-mask totals and top-n sums; per-gene counts and totals) runs in
csrc/qc.cu and the existing `sb2_csr_col_sums_f32`; the n- and g-sized arithmetic (log1p, the divisions) stays in numpy.

Accumulation is fp64 on the device.  The reference sums in X's dtype (float32 for float32 X): for integer-valued counts
below 2^24 per row both are identical, otherwise these results are the more exact ones (DESIGN.md §5).  The output
dtypes follow the reference for X's dtype: counts are int64; totals are float32 for float32 X, float64 for float64 X and
int64 for integer X; the top-n shares are float64.
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse

from . import _abi, _ops
from ._abi import check, ptr
from ._compat import is_anndata_like, log_done, log_start, logger, settings, warn
from ._preprocess import _as_csr32

MAX_QC_VARS = 32  # one uint32 bit-set per gene


def _sum_dtype(dtype) -> np.dtype:
    """dtype of `stats.sum(x, axis=...)` for X of this dtype."""
    dtype = np.dtype(dtype)
    if dtype.kind in "biu":
        return np.dtype(np.int64)
    return np.dtype(np.float64) if dtype == np.float64 else np.dtype(np.float32)


def _is_backed(x) -> bool:
    return hasattr(x, "row_chunks")  # on-disk CSR (scanpy_b200._io.ZarrCSR)


def _row_chunks(x, chunk_size: int | None):
    """(r0, r1, d_indptr, d_indices, d_data) CUDA tensors over the rows: the whole matrix for an in-memory CSR,
    `chunk_size` rows at a time from disk."""
    if _is_backed(x):
        for r0, r1, indptr, indices, data in x.row_chunks(settings.chunk_size if chunk_size is None else chunk_size):
            yield r0, r1, _ops._to_device(indptr), _ops._to_device(indices), _ops._to_device(data)
        return
    yield (0, x.shape[0], *_ops.csr_to_device(x))


def _device_pass(x, *, positive_only: bool, qc_bits=None, n_qc: int = 0, ns=(), rows: bool = True, cols: bool = True,
                 chunk_size: int | None = None):
    """Per-row (count, total, qc totals [n x n_qc], top sums [n x len(ns)]) and per-column (count, total) of a CSR with
    float32 data, fp64 / int64 on the host.  An on-disk X streams through one chunk at a time; the per-column results
    accumulate on the device."""
    import torch

    ctx = _abi.default_context()
    n, g = x.shape
    h_ns = np.ascontiguousarray(ns, dtype=np.int32)
    d_bits = _ops._to_device(np.ascontiguousarray(qc_bits, dtype=np.uint32)) if n_qc else None
    out = dict(count=np.empty(n, np.int64), total=np.empty(n, np.float64), qc=np.empty((n, n_qc), np.float64),
               top=np.empty((n, h_ns.size), np.float64))
    col_count = torch.zeros(g, dtype=torch.int64, device="cuda")
    col_total = torch.zeros(g, dtype=torch.float64, device="cuda")
    for r0, r1, d_indptr, d_indices, d_data in _row_chunks(x, chunk_size):
        m = r1 - r0
        nnz = int(d_data.numel())
        if rows:
            cnt = torch.empty(m, dtype=torch.int64, device="cuda")
            tot = torch.empty(m, dtype=torch.float64, device="cuda")
            qc = torch.empty((m, n_qc), dtype=torch.float64, device="cuda")
            top = torch.empty((m, h_ns.size), dtype=torch.float64, device="cuda")
            check(ctx.lib.sb2_csr_qc_rows_f32(ctx.handle, m, g, ptr(d_indptr), ptr(d_indices), ptr(d_data),
                                              int(positive_only), ptr(d_bits), n_qc, ptr(h_ns) if h_ns.size else None,
                                              int(h_ns.size), ptr(cnt), ptr(tot), ptr(qc) if n_qc else None,
                                              ptr(top) if h_ns.size else None))
            h = _ops._to_host(cnt, tot, qc, top)
            for key, val in zip(("count", "total", "qc", "top"), h):
                out[key][r0:r1] = val
        if cols:
            c = torch.empty(g, dtype=torch.int64, device="cuda")
            s1 = torch.empty(g, dtype=torch.float64, device="cuda")
            s2 = torch.empty(g, dtype=torch.float64, device="cuda")
            check(ctx.lib.sb2_csr_col_counts_f32(ctx.handle, nnz, g, ptr(d_indices), ptr(d_data), int(positive_only), ptr(c)))
            check(ctx.lib.sb2_csr_col_sums_f32(ctx.handle, nnz, g, ptr(d_indices), ptr(d_data), 0, 1.0, ptr(s1), ptr(s2)))
            col_count += c
            col_total += s1
    if cols:
        out["col_count"], out["col_total"] = _ops._to_host(col_count, col_total)
    return out


def _get_x(adata, *, layer, use_raw):
    """src/scanpy/get/get.py `_get_arr(adata, layer=..., use_raw=...)`."""
    if use_raw and layer is not None:
        raise ValueError(f"Cannot use expression from both layer and raw. You provided: `use_raw={use_raw}` and "
                         f"`layer={layer}`")
    if layer is not None:
        return adata.layers[layer]
    if use_raw:
        return adata.raw.X
    return adata.X


def _check_ns(ns, n_vars: int) -> None:
    """`check_ns` (_qc.py:363-373)."""
    if not (max(ns) <= n_vars and min(ns) > 0):
        raise IndexError("Positions outside range of features.")


def calculate_qc_metrics(adata, *, expr_type: str = "counts", var_type: str = "genes", qc_vars=(),
                         percent_top=(50, 100, 200, 500), layer: str | None = None, use_raw: bool = False,
                         inplace: bool = False, log1p: bool = True, parallel: bool | None = None):
    """Calculate quality control metrics (signature of `scanpy.pp.calculate_qc_metrics`).

    Returns `(obs_metrics, var_metrics)` DataFrames, or writes them into `adata.obs` / `adata.var` with `inplace=True`.
    `adata.X` may be an on-disk CSR (`read_zarr_backed`): its rows then stream through the device
    `settings.chunk_size` at a time and it is not modified."""
    if parallel is not None:
        warn("Argument `parallel` is deprecated, and currently has no effect.", FutureWarning)
    x = _get_x(adata, layer=layer, use_raw=use_raw)
    if type(x).__module__.startswith("dask"):
        raise NotImplementedError("dask arrays are not supported by scanpy_b200.pp.calculate_qc_metrics")
    if isinstance(qc_vars, str):
        qc_vars = [qc_vars]
    qc_vars = list(qc_vars)
    n, g = x.shape
    ns = sorted(percent_top) if percent_top else []
    if ns:
        _check_ns(ns, g)
    if len(qc_vars) > MAX_QC_VARS:
        raise NotImplementedError(f"at most {MAX_QC_VARS} qc_vars per call are implemented in scanpy_b200")
    bits = np.zeros(g, np.uint32)
    for b, qc_var in enumerate(qc_vars):
        mask = np.asarray(adata.var[qc_var].to_numpy(), dtype=bool)
        bits[mask] |= np.uint32(1 << b)
    start = log_start("calculating QC metrics")
    if _is_backed(x):
        xc, sd = x, _sum_dtype(x.dtype)
    else:
        if sparse.issparse(x):
            x.eliminate_zeros()  # the reference's host bookkeeping; the device counts do not depend on it
        sd = _sum_dtype(x.dtype)
        xc = _as_csr32(x)
    r = _device_pass(xc, positive_only=False, qc_bits=bits, n_qc=len(qc_vars), ns=ns)

    # describe_obs (_qc.py:92-124)
    obs = pd.DataFrame(index=adata.obs.index)
    obs[f"n_{var_type}_by_{expr_type}"] = r["count"]
    if log1p:
        obs[f"log1p_n_{var_type}_by_{expr_type}"] = np.log1p(obs[f"n_{var_type}_by_{expr_type}"])
    total = r["total"].astype(sd)
    obs[f"total_{expr_type}"] = total
    if log1p:
        obs[f"log1p_total_{expr_type}"] = np.log1p(obs[f"total_{expr_type}"])
    if ns:
        with np.errstate(invalid="ignore", divide="ignore"):
            proportions = r["top"] / total.astype(np.float64)[:, None]
        for i, k in enumerate(ns):
            obs[f"pct_{expr_type}_in_top_{k}_{var_type}"] = proportions[:, i] * 100
    for b, qc_var in enumerate(qc_vars):
        obs[f"total_{expr_type}_{qc_var}"] = r["qc"][:, b].astype(sd)
        if log1p:
            obs[f"log1p_total_{expr_type}_{qc_var}"] = np.log1p(obs[f"total_{expr_type}_{qc_var}"])
        with np.errstate(invalid="ignore", divide="ignore"):
            obs[f"pct_{expr_type}_{qc_var}"] = obs[f"total_{expr_type}_{qc_var}"] / obs[f"total_{expr_type}"] * 100

    # describe_var (_qc.py:177-192)
    var = pd.DataFrame(index=adata.var.index)
    var_total = r["col_total"].astype(sd)
    var[f"n_cells_by_{expr_type}"] = r["col_count"]
    var[f"mean_{expr_type}"] = var_total / n
    if log1p:
        var[f"log1p_mean_{expr_type}"] = np.log1p(var[f"mean_{expr_type}"])
    var[f"pct_dropout_by_{expr_type}"] = (1 - var[f"n_cells_by_{expr_type}"] / n) * 100
    var[f"total_{expr_type}"] = var_total
    if log1p:
        var[f"log1p_total_{expr_type}"] = np.log1p(var[f"total_{expr_type}"])
    log_done(start)
    if inplace:
        for col in obs.columns:
            adata.obs[col] = obs[col].to_numpy()
        for col in var.columns:
            adata.var[col] = var[col].to_numpy()
        return None
    return obs, var


def _one_option(options: dict) -> None:
    if sum(v is not None for v in options.values()) != 1:
        names = "`, `".join(options)
        raise ValueError(f"Provide exactly one of the optional parameters `{names}` per call.")


def _filter_number(x, *, axis: int, by_count: bool):
    """The number per cell (axis=1) or gene (axis=0) the filters threshold: `stats.sum(data > 0, axis)` (int64) or
    `stats.sum(data, axis)` (X's sum dtype)."""
    sd = _sum_dtype(x.dtype)
    r = _device_pass(_as_csr32(x), positive_only=True, rows=axis == 1, cols=axis == 0)
    if axis == 1:
        return r["count"] if by_count else r["total"].astype(sd)
    return r["col_count"] if by_count else r["col_total"].astype(sd)


def filter_cells(data, *, min_counts: int | None = None, min_genes: int | None = None, max_counts: int | None = None,
                 max_genes: int | None = None, inplace: bool = True, copy: bool = False):
    """Filter cell outliers based on counts and numbers of genes expressed (signature of `scanpy.pp.filter_cells`).

    AnnData input: writes `obs['n_genes' | 'n_counts']` and subsets the cells in place; array input or `inplace=False`:
    returns `(cells_subset, number_per_cell)`."""
    if copy:
        logger.warning("`copy` is deprecated, use `inplace` instead.")
    _one_option(dict(min_counts=min_counts, min_genes=min_genes, max_counts=max_counts, max_genes=max_genes))
    if is_anndata_like(data):
        if _is_backed(data.X):
            raise NotImplementedError(f"filter_cells is not implemented for matrices of type {type(data.X)}")
        adata = data.copy() if copy else data
        cell_subset, number = filter_cells(adata.X, min_counts=min_counts, min_genes=min_genes, max_counts=max_counts,
                                           max_genes=max_genes)
        if not inplace:
            return cell_subset, number
        adata.obs["n_counts" if min_genes is None and max_genes is None else "n_genes"] = number
        adata._inplace_subset_obs(cell_subset)
        return adata if copy else None
    if _is_backed(data):
        raise NotImplementedError(f"filter_cells is not implemented for matrices of type {type(data)}")
    min_number = min_counts if min_genes is None else min_genes
    max_number = max_counts if max_genes is None else max_genes
    number_per_cell = _filter_number(data, axis=1, by_count=not (min_genes is None and max_genes is None))
    cell_subset = number_per_cell >= min_number if min_number is not None else number_per_cell <= max_number
    s = int(np.sum(~cell_subset))
    if s > 0:
        msg = f"filtered out {s} cells that have "
        if min_genes is not None or min_counts is not None:
            msg += "less than " + (f"{min_genes} genes expressed" if min_counts is None else f"{min_counts} counts")
        if max_genes is not None or max_counts is not None:
            msg += "more than " + (f"{max_genes} genes expressed" if max_counts is None else f"{max_counts} counts")
        logger.info(msg)
    return cell_subset, number_per_cell


def filter_genes(data, *, min_counts: int | None = None, min_cells: int | None = None, max_counts: int | None = None,
                 max_cells: int | None = None, inplace: bool = True, copy: bool = False):
    """Filter genes based on number of cells or counts (signature of `scanpy.pp.filter_genes`).

    AnnData input: writes `var['n_cells' | 'n_counts']` and subsets the genes in place; array input or `inplace=False`:
    returns `(gene_subset, number_per_gene)`."""
    if copy:
        logger.warning("`copy` is deprecated, use `inplace` instead.")
    _one_option(dict(min_counts=min_counts, min_cells=min_cells, max_counts=max_counts, max_cells=max_cells))
    if is_anndata_like(data):
        if _is_backed(data.X):
            raise NotImplementedError(f"filter_genes is not implemented for matrices of type {type(data.X)}")
        adata = data.copy() if copy else data
        gene_subset, number = filter_genes(adata.X, min_cells=min_cells, min_counts=min_counts, max_cells=max_cells,
                                           max_counts=max_counts)
        if not inplace:
            return gene_subset, number
        adata.var["n_counts" if min_cells is None and max_cells is None else "n_cells"] = number
        adata._inplace_subset_var(gene_subset)
        return adata if copy else None
    if _is_backed(data):
        raise NotImplementedError(f"filter_genes is not implemented for matrices of type {type(data)}")
    min_number = min_counts if min_cells is None else min_cells
    max_number = max_counts if max_cells is None else max_cells
    number_per_gene = _filter_number(data, axis=0, by_count=not (min_cells is None and max_cells is None))
    gene_subset = number_per_gene >= min_number if min_number is not None else number_per_gene <= max_number
    s = int(np.sum(~gene_subset))
    if s > 0:
        msg = f"filtered out {s} genes that are detected "
        if min_cells is not None or min_counts is not None:
            msg += "in less than " + (f"{min_cells} cells" if min_counts is None else f"{min_counts} counts")
        if max_cells is not None or max_counts is not None:
            msg += "in more than " + (f"{max_cells} cells" if max_counts is None else f"{max_counts} counts")
        logger.info(msg)
    return gene_subset, number_per_gene

"""`sc.pp.regress_out` on the device.

Reference: src/scanpy/preprocessing/_simple.py:468-681.  The two passes over X (the column sums `WᵀX` or the
per-category sums, and the dense residual) run in csrc/regress.cu; the n- and g-sized arithmetic stays in numpy: the
Gram matrix and its determinant (the reference's own expression, so the branch taken is the same), its inverse, the SVD
of the regressors, the category means and the 2 x 2 solves.

Branches and output dtypes follow the reference:
* categorical key: residual of each gene on [1, r] with r(cell) = the gene's mean over the cell's category (0 for a
  missing category); float64 output.  The means are exact fp64 means (the reference uses float32 means and a GLM; the
  results differ by about 1e-7, DESIGN.md §5).
* numeric keys with det(AᵀA) != 0: X - A inv(AᵀA) AᵀX in X's float dtype (integer X becomes float32 up to 4 bytes per
  value, float64 above), each value computed in fp64 and rounded once.
* numeric keys with det(AᵀA) == 0 (the reference's GLM fallback): the least-squares residual X - Q QᵀX, Q an orthonormal
  basis of range(A); float64 output.
In both GLM paths genes whose values are all equal are returned unchanged.

The dense result moves through the device `settings.chunk_size` rows at a time, each block copied into the host array
before the next, so device memory does not grow with n x g.  A dense X is streamed the same way; a sparse X stays on
the device as CSR.
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse

from . import _abi, _ops
from ._abi import check, ptr
from ._compat import log_done, log_start, logger, settings

MAX_REGRESSORS = 32  # the intercept included
TILE = 1024  # SB2_REGRESS_TILE_ROWS: the column sums' fixed row subtile
PARTIAL_BYTES = 1 << 28  # device scratch for the column sums' per-subtile partials


def _float_dtype(dtype, *, integer_to) -> np.dtype:
    dtype = np.dtype(dtype)
    if dtype.kind in "biu":
        return np.dtype(integer_to if integer_to is not None else (np.float32 if dtype.itemsize <= 4 else np.float64))
    if dtype not in (np.float32, np.float64):
        raise NotImplementedError(f"regress_out in scanpy_b200 supports float32 and float64 data, not {dtype}")
    return dtype


def _is_categorical(col: pd.Series) -> bool:
    # string and object columns are categoricals once the reference's sanitize_anndata has run
    return isinstance(col.dtype, pd.CategoricalDtype) or col.dtype == object or pd.api.types.is_string_dtype(col.dtype)


_DeviceX = _ops.DeviceX


def _col_sums(dx: _DeviceX, n: int, g: int, *, w=None, group=None, n_groups: int = 0):
    """Weighted (`w`, n x p fp64): WᵀX [p x g]; grouped (`group`, int32 [n] in [0, n_groups)): the per-group column sums
    [n_groups x g].  Also the per-gene min, max and NaN flag."""
    import torch

    ctx = _abi.default_context()
    width = w.shape[1] if w is not None else n_groups
    acc = torch.zeros(width * g, dtype=torch.float64, device="cuda")
    cmin = torch.full((g,), np.inf, dtype=torch.float64, device="cuda")
    cmax = torch.full((g,), -np.inf, dtype=torch.float64, device="cuda")
    cnan = torch.zeros(g, dtype=torch.int32, device="cuda")
    d_w = _ops._to_device(np.ascontiguousarray(w, dtype=np.float64)) if w is not None else None
    # blocks are whole subtiles (so the sums do not depend on the block size), bounded by the partials' scratch and,
    # for a dense X, by settings.chunk_size
    subtiles = max(1, PARTIAL_BYTES // ((width + 3) * g * 8))
    if dx.dense is not None:
        subtiles = min(subtiles, max(1, settings.chunk_size // TILE))
    step = subtiles * TILE
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        d_x, d_indptr, d_indices, d_data = dx.block(r0, r1)
        d_group = d_order = None
        if group is not None:
            grp = group[r0:r1]
            order = np.lexsort((grp, np.arange(r1 - r0) // TILE)).astype(np.int32)  # by (subtile, group, row)
            d_group, d_order = _ops._to_device(grp), _ops._to_device(order)
        check(ctx.lib.sb2_regress_col_sums(ctx.handle, r1 - r0, g, dx.is_f64, ptr(d_x), ptr(d_indptr), ptr(d_indices),
                                           ptr(d_data), ptr(d_w[r0:] if d_w is not None else None),
                                           width if w is not None else 0, ptr(d_group), ptr(d_order), n_groups,
                                           ptr(acc), ptr(cmin), ptr(cmax), ptr(cnan)))
    acc, cmin, cmax, cnan = _ops._to_host(acc, cmin, cmax, cnan)
    constant = (cnan == 0) & (cmin == cmax)
    return acc.reshape(width, g), constant


def _residual(dx: _DeviceX, n: int, g: int, out_dtype: np.dtype, *, w=None, coef=None, codes=None, means=None, b0=None,
              b1=None, passthrough=None) -> np.ndarray:
    """The dense result, `settings.chunk_size` rows at a time, each block copied to the host before the next."""
    import torch

    ctx = _abi.default_context()
    out = np.empty((n, g), dtype=out_dtype)
    up = lambda a, dt: None if a is None else _ops._to_device(np.ascontiguousarray(a, dtype=dt))  # noqa: E731
    d_w, d_coef, d_codes, d_means = up(w, np.float64), up(coef, np.float64), up(codes, np.int32), up(means, np.float64)
    d_b0, d_b1, d_pass = up(b0, np.float64), up(b1, np.float64), up(passthrough, np.uint8)
    tdt = torch.float64 if out_dtype == np.float64 else torch.float32
    step = max(1, int(settings.chunk_size))
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        d_x, d_indptr, d_indices, d_data = dx.block(r0, r1)
        d_out = torch.empty((r1 - r0, g), dtype=tdt, device="cuda")
        check(ctx.lib.sb2_regress_residual(
            ctx.handle, r1 - r0, g, dx.is_f64, ptr(d_x), ptr(d_indptr), ptr(d_indices), ptr(d_data),
            ptr(d_w[r0:] if d_w is not None else None), coef.shape[0] if coef is not None else 0, ptr(d_coef),
            ptr(d_codes[r0:] if d_codes is not None else None), ptr(d_means), ptr(d_b0), ptr(d_b1), ptr(d_pass),
            int(out_dtype == np.float64), ptr(d_out)))
        out[r0:r1] = _ops._to_host(d_out)
    return out


def _categorical_fit(sums: np.ndarray, counts: np.ndarray, n: int, has_missing: bool):
    """Per-gene means [C x g] and the least-squares coefficients (b0, b1) of x on [1, r].  `sums` holds one row per
    category and a last row for the cells with a missing category.  Σr = Σ_k S_k and Σr² = Σr·x = Σ_k S_k² / n_k."""
    s, s_missing = sums[:-1], sums[-1]
    with np.errstate(invalid="ignore", divide="ignore"):
        means = np.where(counts[:, None] > 0, s / counts[:, None], 0.0)
    g = sums.shape[1]
    if not has_missing:
        return means, np.zeros(g), np.ones(g)
    used = counts > 0
    sr = s.sum(axis=0)
    sx = sr + s_missing
    srr = (s[used] ** 2 / counts[used, None]).sum(axis=0)
    det = n * srr - sr * sr
    with np.errstate(invalid="ignore", divide="ignore"):
        b1 = np.where(det != 0, (n * srr - sr * sx) / det, 0.0)
    b0 = (sx - b1 * sr) / n
    return means, b0, b1


def regress_out(adata, keys, *, layer: str | None = None, n_jobs: int | None = None, copy: bool = False):
    """Regress out (mostly) unwanted sources of variation (signature of `scanpy.pp.regress_out`).

    Writes the corrected dense matrix to `adata.X` (or `adata.layers[layer]`); returns the copy with `copy=True`.
    `n_jobs` is accepted for compatibility and has no effect on the result."""
    start = log_start(f"regressing out {keys}")
    adata = adata.copy() if copy else adata
    if isinstance(keys, str):
        keys = [keys]
    keys = list(keys)
    x = adata.layers[layer] if layer is not None else adata.X
    if hasattr(x, "row_chunks"):  # on-disk CSR (scanpy_b200._io.ZarrCSR)
        raise NotImplementedError(f"regress_out is not implemented for matrices of type {type(x)}")
    if sparse.issparse(x):
        logger.info("    sparse input is densified and may lead to high memory use")
    else:
        x = np.asarray(x)
    n, g = x.shape
    obs = adata.obs

    if keys and keys[0] in obs and _is_categorical(obs[keys[0]]):
        if len(keys) > 1:
            raise ValueError("If providing categorical variable, only a single one is allowed. For this one we regress "
                             "on the mean for each category.")
        logger.debug("... regressing on per-gene means within categories")
        col = obs[keys[0]]
        cat = col.cat if isinstance(col.dtype, pd.CategoricalDtype) else pd.Categorical(col)
        codes = np.asarray(cat.codes, dtype=np.int32)
        n_cat = len(cat.categories)
        vdtype = _float_dtype(x.dtype, integer_to=None)
        dx = _DeviceX(x, vdtype)
        group = np.where(codes < 0, n_cat, codes).astype(np.int32)
        sums, constant = _col_sums(dx, n, g, group=group, n_groups=n_cat + 1)
        counts = np.bincount(codes[codes >= 0], minlength=n_cat)
        means, b0, b1 = _categorical_fit(sums, counts, n, bool((codes < 0).any()))
        res = _residual(dx, n, g, np.dtype(np.float64), codes=codes, means=means, b0=b0, b1=b1, passthrough=constant)
    else:
        regressors = obs[keys] if keys else obs.copy()
        regressors.insert(0, "ones", 1.0)
        a = regressors.to_numpy()
        if a.shape[1] > MAX_REGRESSORS:
            raise NotImplementedError(f"regress_out in scanpy_b200 supports at most {MAX_REGRESSORS} regressors, the "
                                      f"intercept included; got {a.shape[1]}")
        if np.linalg.det(a.T @ a) != 0:  # the reference's test for its numpy shortcut
            a = np.asarray(a, dtype=np.float64)
            vdtype = _float_dtype(x.dtype, integer_to=None)
            dx = _DeviceX(x, vdtype)
            atx, _ = _col_sums(dx, n, g, w=a)
            coef = np.linalg.inv(a.T @ a) @ atx
            res = _residual(dx, n, g, vdtype, w=a, coef=coef)
        else:  # the GLM fallback: the least-squares residual, through an orthonormal basis of range(A)
            a = np.asarray(a, dtype=np.float64)
            u, s, _ = np.linalg.svd(a, full_matrices=False)
            rank = int((s > s.max() * max(a.shape) * np.finfo(np.float64).eps).sum())
            q = np.ascontiguousarray(u[:, :rank])
            vdtype = _float_dtype(x.dtype, integer_to=np.float64)  # statsmodels reads integer data as float64
            dx = _DeviceX(x, vdtype)
            qtx, constant = _col_sums(dx, n, g, w=q)
            res = _residual(dx, n, g, np.dtype(np.float64), w=q, coef=qtx, passthrough=constant)

    if layer is not None:
        adata.layers[layer] = res
    else:
        adata.X = res
    log_done(start)
    return adata if copy else None

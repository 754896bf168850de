"""regress_out oracle (test infrastructure only): a numpy restatement of src/scanpy/preprocessing/_simple.py:468-681.

* numeric keys, det(AᵀA) != 0: `numpy_regress_out` — coeff = inv(AᵀA) @ (AᵀX), `data[i] -= A[i] @ coeff` in X's float
  dtype (integer X cast to float32 up to 4 bytes per value, float64 above).
* numeric keys, det(AᵀA) == 0, and a categorical key: `_regress_out_chunk`.  statsmodels is not installed, so its
  Gaussian / identity GLM is restated as the per-gene least-squares residual (`np.linalg.lstsq`), which is what
  `result.resid_response` is.  Columns whose values are all equal are returned unchanged; float64 output.
* the categorical regressor is `_create_regressor_categorical`: the gene's float32 mean over the cell's category, 0 for
  a missing category.  `exact_means=True` uses fp64 means instead (what scanpy_b200 computes).
Pinned by the reference's tests/_data/regress_test_small.npy and regress_test_small_cat.npy (tests/golden/
pbmc68k_regress.npz).
"""
from __future__ import annotations

import numpy as np
from scipy import sparse


def _dense(x, dtype=None):
    x = x.toarray() if sparse.issparse(x) else np.array(x)
    return x if dtype is None else x.astype(dtype)


def _int_target(dtype):
    return np.float32 if np.dtype(dtype).itemsize <= 4 else np.float64


def design(obs, keys):
    """The reference's regressor matrix for numeric keys: obs[keys] (all of obs for no keys) after a column of ones."""
    regressors = obs[keys] if keys else obs.copy()
    regressors.insert(0, "ones", 1.0)
    return regressors.to_numpy()


def categorical_regressor(x, codes, n_categories, *, exact_means=False):
    """`_create_regressor_categorical`: r[i, j] = mean of x[:, j] over the cells of category codes[i] (0 if codes[i] < 0)."""
    reg = np.zeros(x.shape, dtype=np.float64 if exact_means else np.float32)
    for c in range(n_categories):
        mask = codes == c
        if mask.any():
            reg[mask] = x[mask].mean(axis=0, dtype=np.float64 if exact_means else None)
    return reg


def glm_residuals(x, regressors, *, per_gene=False):
    """`_regress_out_chunk`: per gene, the least-squares residual on `regressors` (n x p, or n x g per gene with
    per_gene=True: then the design is [1, regressors[:, j]]); constant genes unchanged.  float64."""
    x = np.asarray(x)
    out = np.empty(x.shape, dtype=np.float64)
    for j in range(x.shape[1]):
        col = x[:, j]
        if not (col != col[0]).any():
            out[:, j] = col
            continue
        a = np.c_[np.ones(x.shape[0]), regressors[:, j]] if per_gene else regressors
        a = np.asarray(a, dtype=np.float64)
        y = col.astype(np.float64)
        coef = np.linalg.lstsq(a, y, rcond=None)[0]
        out[:, j] = y - a @ coef
    return out


def regress_out(x, *, regressors=None, codes=None, n_categories=None, exact_means=False):
    """The reference's result for X (dense or sparse) with either the numeric design `regressors` (see `design`) or the
    categorical `codes` (int, -1 = missing) of `n_categories` categories."""
    if codes is not None:
        xd = _dense(x)
        if np.issubdtype(xd.dtype, np.integer):
            xd = xd.astype(_int_target(xd.dtype))
        reg = categorical_regressor(xd, np.asarray(codes), n_categories, exact_means=exact_means)
        return glm_residuals(xd, reg, per_gene=True)
    a = np.asarray(regressors)
    if np.linalg.det(a.T @ a) != 0:
        xd = _dense(x)
        if np.issubdtype(xd.dtype, np.integer):
            xd = xd.astype(_int_target(xd.dtype))
        coeff = np.linalg.inv(a.T @ a) @ (a.T @ xd)
        for i in range(xd.shape[0]):
            xd[i] -= a[i] @ coeff
        return xd
    return glm_residuals(_dense(x), a)

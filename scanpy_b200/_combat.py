"""`sc.pp.combat` on the device.

Reference: src/scanpy/preprocessing/_combat.py.  The passes over X run in CUDA: the design-matrix product DᵀX
(`sb2_regress_col_sums`, grouped for the batch columns and weighted for the covariate columns), the per-batch moments
of r = x - stand_mean and the dense corrected matrix (csrc/combat.cu).  Everything sized batches x genes stays in numpy:
inv(DᵀD), b_hat, the pooled variance, gamma_hat / delta_hat, the priors and the empirical-Bayes iteration.

From the per-batch count n_b, mean m_b and sum of squared deviations M2_b of r (zeros of a sparse X included):
* var_pooled = Σ_b (M2_b + n_b (m_b - (b_hat[b] - grand_mean))²) / n, the mean of (x - D b_hat)² without cancellation;
* the standardised data s = r / sqrt(vp) (0 where vp == 0) has batch mean m_b / sqrt(vp) = gamma_hat and sum of squared
  deviations M2_b / vp, so delta_hat = M2_b / (vp (n_b - 1)) and every sum of squares `_it_sol` forms is
  Σ (s - γ)² = M2_b / vp + n_b (m_b / sqrt(vp) - γ)²: the iteration needs no further pass over X.

Reference details kept:
* batches in `groupby(key, observed=True)` order (category order, unused categories dropped; sorted values otherwise);
* the design without patsy: the batch one-hot columns, then the non-numeric covariates coded as `~ 0 + Q(a) + Q(b)` (the
  first factor full rank, later ones without their first level; bool is categorical), then the numeric covariates;
* delta_hat and the priors use ddof = 1, t2 ddof = 0; `_it_sol` is restated literally, Python `max` and all;
* zero-variance genes are reported with the reference's `print` and get what its expression gives (stand_mean).
Deviation: NaN or inf in X raises ValueError (the reference turns every output NaN; DESIGN.md §5).

The corrected float64 matrix moves to the host `settings.chunk_size` rows at a time, so device memory does not grow with
n x g.  A sparse X is uploaded once as CSR; a dense X streams through by row blocks.
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from numpy import linalg as la
from scipy import sparse

from . import _abi, _ops
from ._abi import check, ptr
from ._compat import logger
from ._regress import _col_sums_stats

MAX_COVARIATES = 32  # design columns besides the batch columns (sb2_regress_col_sums' weighted mode)
TILE = _ops.SUBTILE_ROWS  # SB2_COMBAT_TILE_ROWS
PARTIAL_BYTES = 1 << 28  # device scratch for the moments' per-subtile partials


# ------------------------------------------------------------------------------------------ host helpers
def check_args(adata, key: str, covariates) -> None:
    """The reference's argument checks, in its order and with its messages."""
    if key not in adata.obs:
        raise ValueError(f"Could not find the key {key!r} in adata.obs")
    if covariates is not None:
        cov_exist = np.isin(covariates, adata.obs.columns)
        if np.any(~cov_exist):
            missing_cov = np.array(covariates)[~cov_exist].tolist()
            raise ValueError(f"Could not find the covariate(s) {missing_cov!r} in adata.obs")
        if key in covariates:
            raise ValueError("Batch key and covariates cannot overlap")
        if len(covariates) != len(set(covariates)):
            raise ValueError("Covariates must be unique")


def value_dtype(x) -> np.dtype:
    """The dtype X goes to the device in; raises for what the kernels do not take."""
    if hasattr(x, "row_chunks"):  # on-disk CSR (scanpy_b200._io.ZarrCSR)
        raise NotImplementedError(f"combat is not implemented for matrices of type {type(x)}")
    if sparse.issparse(x) and x.format not in ("csr", "csc"):
        raise NotImplementedError(f"combat in scanpy_b200 supports CSR, CSC and dense X, not {x.format}")
    dtype = np.dtype(x.dtype)
    if dtype.kind in "iu":
        return np.dtype(np.float64)
    if dtype not in (np.float32, np.float64):
        raise NotImplementedError(f"combat in scanpy_b200 supports float32, float64 and integer data, not {dtype}")
    return dtype


def batch_groups(model: pd.DataFrame, key: str):
    """(levels, code of every cell in [0, n_batch), cells per batch) in the reference's `groupby(key, observed=True)`
    order.  Cells whose batch is missing belong to no group there; they are rejected here."""
    indices = model.groupby(key, observed=True).indices
    levels = list(indices)
    codes = np.full(len(model), -1, dtype=np.int32)
    for b, idx in enumerate(indices.values()):
        codes[idx] = b
    if (codes < 0).any():
        raise ValueError(f"adata.obs[{key!r}] has missing values; ComBat needs a batch for every cell")
    return levels, codes, np.array([len(v) for v in indices.values()])


def _factor_levels(col: pd.Series) -> list:
    """patsy's levels of a categorical factor: the categories of a pandas Categorical, (False, True) for bool, the sorted
    distinct values otherwise."""
    if isinstance(col.dtype, pd.CategoricalDtype):
        return list(col.cat.categories)
    if pd.api.types.is_bool_dtype(col.dtype):
        return [False, True]
    return sorted(pd.unique(col.dropna()))


def design_matrix(model: pd.DataFrame, key: str, levels) -> pd.DataFrame:
    """`_design_matrix` without patsy: the batch one-hot columns, then `~ 0 + Q(a) + Q(b) + ...` over the non-numeric
    covariates (the first factor gets a column for every level, each later one drops its first level), then the numeric
    covariates as they are.  float64 columns named as patsy names them."""
    cols: dict[str, np.ndarray] = {}
    batch = model[key].to_numpy()
    for lv in levels:
        cols[f"C(Q('{key}'), levels=batch_levels)[{lv}]"] = (batch == lv).astype(np.float64)
    rest = model.drop([key], axis=1)
    numerical = list(rest.select_dtypes("number").columns)
    logger.info(f"Found {len(levels)} batches\n")
    other = [c for c in rest.columns if c not in numerical]
    for i, c in enumerate(other):
        values = rest[c].to_numpy()
        for j, lv in enumerate(_factor_levels(rest[c])):
            if i > 0 and j == 0:
                continue
            cols[f"Q('{c}')[{lv}]" if i == 0 else f"Q('{c}')[T.{lv}]"] = (values == lv).astype(np.float64)
    if other:
        logger.info(f"Found {len(other)} categorical variables:")
        logger.info(f"\t{', '.join(other)}\n")
    logger.info(f"Found {len(numerical)} numerical variables:")
    logger.info(f"\t{', '.join(numerical)}\n")
    for c in numerical:
        cols[c] = rest[c].to_numpy(dtype=np.float64)
    return pd.DataFrame(cols, index=model.index)


def _aprior(delta_hat: np.ndarray) -> float:
    m, s2 = pd.Series(delta_hat).mean(), pd.Series(delta_hat).var()
    return (2 * s2 + m**2) / s2


def _bprior(delta_hat: np.ndarray) -> float:
    m, s2 = pd.Series(delta_hat).mean(), pd.Series(delta_hat).var()
    return (m * s2 + m**3) / s2


def it_sol(mean_s, m2_s, n: int, g_hat, d_hat, *, g_bar: float, t2: float, a: float, b: float, conv: float = 0.0001):
    """`_it_sol` for one batch, with the sum of squares of the standardised data about g_new taken in closed form from
    that data's mean `mean_s` and sum of squared deviations `m2_s`.  -> (gamma, delta, iterations)."""
    g_old, d_old = g_hat.copy(), d_hat.copy()
    change, count = 1, 0
    g_new, d_new = g_old, d_old
    with np.errstate(divide="ignore", invalid="ignore"):
        while change > conv:
            g_new = (t2 * n * g_hat + d_old * g_bar) / (t2 * n + d_old)
            sum2 = m2_s + n * (mean_s - g_new) ** 2
            d_new = (0.5 * sum2 + b) / (n / 2.0 + a - 1.0)
            change = max((abs(g_new - g_old) / g_old).max(), (abs(d_new - d_old) / d_old).max())
            g_old, d_old = g_new, d_new
            count += 1
    return g_new, d_new, count


def eb_fit(counts, means, m2, b_hat_batch, grand_mean):
    """Everything between the moments pass and the writer, on the host.  `means` / `m2` [n_batch x g]: the mean and sum of
    squared deviations of r = x - stand_mean per batch.  -> dict(var_pooled, gamma_hat, delta_hat, gamma_star,
    delta_star, iterations)."""
    counts = np.asarray(counts)
    n_array = float(counts.sum())
    dev = means - (b_hat_batch - grand_mean)
    var_pooled = (m2 + counts[:, None] * dev * dev).sum(axis=0) / n_array
    zero = var_pooled == 0
    if np.sum(zero) > 0:
        print(f"Found {np.sum(zero)} genes with zero variance.")
    sv = np.sqrt(var_pooled)
    with np.errstate(divide="ignore", invalid="ignore"):
        mean_s = np.where(zero, 0.0, means / sv)
        m2_s = np.where(zero, 0.0, m2 / var_pooled)
    logger.info("Fitting L/S model and finding priors\n")
    gamma_hat = mean_s
    delta_hat = m2_s / (counts[:, None] - 1)
    gamma_bar = gamma_hat.mean(axis=1)
    t2 = gamma_hat.var(axis=1)
    a_prior = [_aprior(d) for d in delta_hat]
    b_prior = [_bprior(d) for d in delta_hat]
    logger.info("Finding parametric adjustments\n")
    gamma_star, delta_star, iterations = [], [], []
    for i in range(len(counts)):
        gamma, delta, count = it_sol(mean_s[i], m2_s[i], int(counts[i]), gamma_hat[i], delta_hat[i], g_bar=gamma_bar[i],
                                     t2=t2[i], a=a_prior[i], b=b_prior[i])
        gamma_star.append(gamma)
        delta_star.append(delta)
        iterations.append(count)
    return dict(var_pooled=var_pooled, gamma_hat=gamma_hat, delta_hat=delta_hat, gamma_star=np.array(gamma_star),
                delta_star=np.array(delta_star), iterations=iterations)


# ------------------------------------------------------------------------------------------ device passes
def _moments(dx: _ops.DeviceX, g: int, codes: np.ndarray, n_batch: int, cov: np.ndarray, grand, beta):
    """(mean, M2) of r per batch [n_batch x g] each.  Each batch's rows go through in blocks of whole subtiles, so the
    result does not depend on the block size."""
    import torch

    ctx = _abi.default_context()
    order = np.argsort(codes, kind="stable")  # each batch contiguous, its cells in their original order
    bounds = np.searchsorted(codes[order], np.arange(n_batch + 1))
    p = cov.shape[1]
    d_order = _ops._to_device(order.astype(np.int64)) if dx.dense is None else None
    d_cov = _ops._to_device(np.ascontiguousarray(cov[order])) if p else None
    d_grand = _ops._to_device(np.ascontiguousarray(grand, dtype=np.float64))
    d_beta = _ops._to_device(np.ascontiguousarray(beta, dtype=np.float64)) if p else None
    step = _ops.subtile_block_rows(dx.dense is not None, PARTIAL_BYTES, 2 * g * 8)
    accs = torch.zeros((n_batch, 3, g), dtype=torch.float64, device="cuda")
    for b in range(n_batch):
        for k0 in range(int(bounds[b]), int(bounds[b + 1]), step):
            k1 = min(int(bounds[b + 1]), k0 + step)
            d_x, d_indptr, d_indices, d_data, d_ord = dx.gather(order, d_order, k0, k1)
            check(ctx.lib.sb2_combat_moments(ctx.handle, k1 - k0, g, dx.is_f64, ptr(d_x), ptr(d_indptr),
                                             ptr(d_indices), ptr(d_data), ptr(d_ord),
                                             ptr(d_cov[k0:] if p else None), p, ptr(d_grand), ptr(d_beta),
                                             ptr(accs[b])))
    accs = _ops._to_host(accs)
    return accs[:, 1], accs[:, 2]


def _adjust(dx: _ops.DeviceX, n: int, g: int, codes, cov, grand, beta, sqrt_vp, gamma_star, dsq) -> np.ndarray:
    """The corrected float64 matrix (`_ops.write_dense`)."""
    ctx = _abi.default_context()
    p = cov.shape[1]
    up = lambda a, dt: _ops._to_device(np.ascontiguousarray(a, dtype=dt))  # noqa: E731
    d_codes, d_grand, d_sv = up(codes, np.int32), up(grand, np.float64), up(sqrt_vp, np.float64)
    d_gamma, d_dsq = up(gamma_star, np.float64), up(dsq, np.float64)
    d_cov, d_beta = (up(cov, np.float64), up(beta, np.float64)) if p else (None, None)

    def launch(r0, r1, xargs, d_out):
        d_x, d_indptr, d_indices, d_data = xargs
        check(ctx.lib.sb2_combat_adjust(ctx.handle, r1 - r0, g, dx.is_f64, ptr(d_x), ptr(d_indptr), ptr(d_indices),
                                        ptr(d_data), ptr(d_codes[r0:]), ptr(d_cov[r0:] if p else None), p,
                                        ptr(d_grand), ptr(d_beta), ptr(d_sv), ptr(d_gamma), ptr(d_dsq), ptr(d_out)))

    return _ops.write_dense(dx, n, g, np.dtype(np.float64), launch)


# ------------------------------------------------------------------------------------------ combat
def combat(adata, key: str = "batch", *, covariates=None, inplace: bool = True):
    """ComBat batch-effect correction (signature of `scanpy.pp.combat`).

    Writes the corrected dense float64 matrix to `adata.X`, or returns it with `inplace=False`."""
    check_args(adata, key, covariates)
    x = adata.X
    vdtype = value_dtype(x)
    if not sparse.issparse(x):
        x = np.asarray(x)
    n, g = x.shape

    model = adata.obs[[key, *(covariates if covariates else [])]]
    levels, codes, counts = batch_groups(model, key)
    small_batches = [batch for batch, size in zip(levels, counts, strict=True) if size < 2]
    if small_batches:
        raise ValueError(f"Batches {small_batches!r} have fewer than 2 cells. ComBat requires at least 2 cells per "
                         "batch to estimate within-batch variance. Filter these batches before running combat.")
    logger.info("Standardizing Data across genes.\n")
    design = design_matrix(model, key, levels)
    n_batch = len(levels)
    if design.shape[1] - n_batch > MAX_COVARIATES:
        raise NotImplementedError(f"combat in scanpy_b200 supports at most {MAX_COVARIATES} covariate columns in the "
                                  f"design; got {design.shape[1] - n_batch}")
    d = design.to_numpy()
    inv = la.inv(np.dot(d.T, d))  # the reference's own expression: a singular design raises as there
    cov = np.ascontiguousarray(d[:, n_batch:])

    dx = _ops.DeviceX(x.tocsr() if sparse.issparse(x) else x, vdtype)
    btx, cmin, cmax, cnan = _col_sums_stats(dx, n, g, group=codes, n_groups=n_batch)
    if cnan.any() or not (np.isfinite(cmin).all() and np.isfinite(cmax).all()):
        raise ValueError("combat in scanpy_b200 requires finite values in X; it holds NaN or infinity")
    dtx = np.vstack([btx, _col_sums_stats(dx, n, g, w=cov)[0]]) if cov.shape[1] else btx
    b_hat = inv @ dtx
    grand_mean = np.dot((counts / float(counts.sum())).T, b_hat[:n_batch, :])
    beta = b_hat[n_batch:]

    means, m2 = _moments(dx, g, codes, n_batch, cov, grand_mean, beta)
    fit = eb_fit(counts, means, m2, b_hat[:n_batch], grand_mean)
    logger.info("Adjusting data\n")
    res = _adjust(dx, n, g, codes, cov, grand_mean, beta, np.sqrt(fit["var_pooled"]), fit["gamma_star"],
                  np.sqrt(fit["delta_star"]))
    if inplace:
        adata.X = res
        return None
    return res

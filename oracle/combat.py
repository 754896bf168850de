"""combat oracle (test infrastructure only): a numpy fp64 restatement of src/scanpy/preprocessing/_combat.py in the
reference's own expression order.

It takes the design matrix as numbers (n x (n_batch + covariate columns), batch columns first) and the cells of each
batch, and works directly on the dense data: b_hat = (inv(DᵀD) Dᵀ) dataᵀ, the pooled variance as the mean of the
squared residual, gamma_hat as inv(BᵀB) Bᵀ sᵀ, and every `_it_sol` sum of squares over the standardised data itself.
None of the device path's closed forms (per-batch moments, Chan merges, sums of squares from a mean and an M2) is used,
so it cross-checks them.  Arrays are n x g (the reference holds data transposed, g x n).
"""
from __future__ import annotations

import numpy as np
from numpy import linalg as la
from scipy import sparse


def _dense(x) -> np.ndarray:
    return np.asarray(x.toarray() if sparse.issparse(x) else x, dtype=np.float64)


def standardize(x, design: np.ndarray, batch_idx: list[np.ndarray]):
    """`_standardize_data` -> (s_data, var_pooled [g], stand_mean [n x g], b_hat, grand_mean)."""
    data = _dense(x)
    n_batch = len(batch_idx)
    n_batches = np.array([len(v) for v in batch_idx])
    n_array = float(sum(n_batches))
    b_hat = np.dot(np.dot(la.inv(np.dot(design.T, design)), design.T), data)
    grand_mean = np.dot((n_batches / n_array).T, b_hat[:n_batch, :])
    var_pooled = ((data - np.dot(design, b_hat)) ** 2).mean(axis=0)
    tmp = design.copy()
    tmp[:, :n_batch] = 0
    stand_mean = grand_mean[np.newaxis, :] + np.dot(tmp, b_hat)
    with np.errstate(divide="ignore", invalid="ignore"):
        s_data = np.where(var_pooled == 0, 0, (data - stand_mean) / np.sqrt(var_pooled))
    return s_data, var_pooled, stand_mean, b_hat, grand_mean


def it_sol(s_data, g_hat, d_hat, *, g_bar, t2, a, b, conv=0.0001):
    """`_it_sol` on the standardised data of one batch (cells x genes) -> (gamma, delta, iterations)."""
    n = (1 - np.isnan(s_data)).sum(axis=0)
    g_old, d_old = g_hat.copy(), d_hat.copy()
    change, count = 1, 0
    g_new, d_new = g_old, d_old
    with np.errstate(divide="ignore", invalid="ignore"):
        while change > conv:
            g_new = (t2 * n * g_hat + d_old * g_bar) / (t2 * n + d_old)
            sum2 = ((s_data - g_new[np.newaxis, :]) ** 2).sum(axis=0)
            d_new = (0.5 * sum2 + b) / (n / 2.0 + a - 1.0)
            change = max((abs(g_new - g_old) / g_old).max(), (abs(d_new - d_old) / d_old).max())
            g_old, d_old = g_new, d_new
            count += 1
    return g_new, d_new, count


def _aprior(d):
    m, s2 = d.mean(), d.var(ddof=1)
    return (2 * s2 + m**2) / s2


def _bprior(d):
    m, s2 = d.mean(), d.var(ddof=1)
    return (m * s2 + m**3) / s2


def combat(x, design: np.ndarray, batch_idx: list[np.ndarray]):
    """The corrected matrix [n x g] float64 and the intermediates (dict)."""
    design = np.asarray(design, dtype=np.float64)
    n_batch = len(batch_idx)
    s_data, var_pooled, stand_mean, b_hat, grand_mean = standardize(x, design, batch_idx)
    batch_design = design[:, :n_batch]
    gamma_hat = la.inv(batch_design.T @ batch_design) @ batch_design.T @ s_data
    delta_hat = [s_data[idx].var(axis=0, ddof=1) for idx in batch_idx]
    gamma_bar = gamma_hat.mean(axis=1)
    t2 = gamma_hat.var(axis=1)
    a_prior = [_aprior(d) for d in delta_hat]
    b_prior = [_bprior(d) for d in delta_hat]
    gamma_star, delta_star, iterations = [], [], []
    for i, idx in enumerate(batch_idx):
        gamma, delta, count = it_sol(s_data[idx], gamma_hat[i], delta_hat[i], g_bar=gamma_bar[i], t2=t2[i],
                                     a=a_prior[i], b=b_prior[i])
        gamma_star.append(gamma)
        delta_star.append(delta)
        iterations.append(count)
    gamma_star, delta_star = np.array(gamma_star), np.array(delta_star)
    bayesdata = s_data
    for j, idx in enumerate(batch_idx):
        dsq = np.sqrt(delta_star[j, :])
        numer = bayesdata[idx] - np.dot(batch_design[idx], gamma_star)
        bayesdata[idx] = numer / dsq[np.newaxis, :]
    out = bayesdata * np.sqrt(var_pooled)[np.newaxis, :] + stand_mean
    return out, dict(var_pooled=var_pooled, stand_mean=stand_mean, b_hat=b_hat, grand_mean=grand_mean,
                     gamma_hat=gamma_hat, delta_hat=np.array(delta_hat), gamma_star=gamma_star,
                     delta_star=delta_star, iterations=iterations)

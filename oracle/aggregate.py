"""sc.get.aggregate oracle (test infrastructure only): a numpy / pandas restatement in float64 of
src/scanpy/get/_aggregated.py's grouping and statistics.

Groups come from pandas' own `groupby(keys, observed=True)` on the label columns (missing labels get no group; level
combinations no row has are absent), named "_".join of their levels; masked-out rows count in no group, but their
group stays.  The statistics per group are np.sum, the mean as Σx / n, the two-pass variance (mean first, then the
squared deviations), (x != 0).sum() and np.median, all in float64 on the dense rows.  For a large CSR, `sparse_moments`
gives the same sums from the stored entries (the zeros' share of the squared deviations is (n - nnz) mean²), and
`median_columns` the medians of chosen columns.  None of the device path's Welford or Chan steps is used."""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse


def group_codes(obs: pd.DataFrame, keys, mask=None):
    """-> (names pd.Index, codes int64 [n] with -1 for no group or masked out, counts int64 [G])."""
    keys = [keys] if isinstance(keys, str) else list(keys)
    grouped = obs[keys].groupby(keys, observed=True, sort=True, dropna=True)
    codes = grouped.ngroup().fillna(-1).to_numpy().astype(np.int64)
    names = pd.Index(["_".join(map(str, k if isinstance(k, tuple) else (k,))) for k in grouped.size().index])
    if mask is not None:
        codes = np.where(np.asarray(mask, dtype=bool), codes, -1)
    return names, codes, np.bincount(codes[codes >= 0], minlength=len(names))


def dense_stats(x, codes, n_groups: int, *, median: bool = True) -> dict:
    """float64 per-group sum, mean (Σx / n), m2 (two-pass), nnz and median of the rows of x (dense or sparse)."""
    x = x.toarray() if sparse.issparse(x) else np.asarray(x)
    x = x.astype(np.float64)
    g = x.shape[1]
    out = {k: np.zeros((n_groups, g)) for k in ("sum", "m2", "nnz")}
    out["mean"] = np.full((n_groups, g), np.nan)
    out["median"] = np.full((n_groups, g), np.nan)
    for k in range(n_groups):
        xs = x[codes == k]
        if xs.shape[0] == 0:
            continue
        out["sum"][k] = xs.sum(axis=0)
        mu = xs.sum(axis=0) / xs.shape[0]
        out["mean"][k] = mu
        out["m2"][k] = ((xs - mu) ** 2).sum(axis=0)
        out["nnz"][k] = (xs != 0).sum(axis=0)
        if median:
            out["median"][k] = np.median(xs, axis=0)
    return out


def sparse_moments(x, codes, n_groups: int) -> dict:
    """float64 sum, mean, m2 (two-pass) and nnz per group of a CSR's rows, from the stored entries."""
    x = sparse.csr_matrix(x, dtype=np.float64, copy=True)  # a copy: eliminate_zeros rewrites indptr / indices in place
    x.eliminate_zeros()
    n = x.shape[0]
    keep = codes >= 0
    ind = sparse.csr_matrix((np.ones(keep.sum()), (codes[keep], np.flatnonzero(keep))), shape=(n_groups, n))
    counts = np.asarray(ind.sum(axis=1)).ravel()
    s = np.asarray((ind @ x).todense())
    nnz = np.asarray((ind @ (x != 0).astype(np.float64)).todense())
    with np.errstate(invalid="ignore", divide="ignore"):
        mu = s / counts[:, None]
    coo = x.tocoo()
    rc = codes[coo.row]
    ok = rc >= 0
    dev = np.zeros_like(coo.data)
    dev[ok] = (coo.data[ok] - mu[rc[ok], coo.col[ok]]) ** 2
    d = sparse.csr_matrix((dev, (coo.row, coo.col)), shape=x.shape)
    m2 = np.asarray((ind @ d).todense()) + (counts[:, None] - nnz) * np.nan_to_num(mu) ** 2
    return dict(sum=s, mean=mu, m2=m2, nnz=nnz, counts=counts)


def median_columns(x, codes, n_groups: int, cols) -> np.ndarray:
    """np.median per group of the columns `cols` of x -> float64 [G x len(cols)] (NaN for empty groups)."""
    sub = x[:, cols]
    sub = sub.toarray() if sparse.issparse(sub) else np.asarray(sub)
    sub = sub.astype(np.float64)
    out = np.full((n_groups, len(cols)), np.nan)
    order = np.argsort(codes, kind="stable")
    bounds = np.searchsorted(codes[order], np.arange(n_groups + 1))
    for k in range(n_groups):
        if bounds[k + 1] > bounds[k]:
            out[k] = np.median(sub[order[bounds[k]:bounds[k + 1]]], axis=0)
    return out


def variance(m2, counts, dof: int):
    """The reference's var from M2: M2 / n (0 for an empty group), times n / (n - dof) (NaN where n <= dof)."""
    n = np.asarray(counts, dtype=np.float64)[:, None]
    var = np.divide(m2, n, out=np.zeros_like(m2), where=n > 0)
    if dof != 0:
        denom = np.where(counts > dof, counts - dof, np.nan)
        var = var * (counts / denom)[:, None]
    return var

"""Moran's I / Geary's C oracle (test infrastructure only): an fp64 numpy restatement of src/scanpy/metrics/_morans_i.py
(`_morans_i_vec_w`), _gearys_c.py (`_gearys_c_vec_w`) and the constant handling of _common.py, vectorised over genes.

For x over the n cells, z = x - mean(x) and the stored arcs i -> j with weights w (duplicates, explicit zeros and
self-loops count as stored):
  A = Σ_i z_i Σ_j w_ij z_j = Σ Z ⊙ (W Z),   B = Σ_(i->j) w_ij (x_i - x_j)²,   Q = Σ_i z_i²
Moran's I = n / S0 * A / Q, Geary's C = (n - 1) * B / (2 * S0 * Q), S0 = Σ w.  Features whose values are all equal
(none NaN) are NaN.  A CPU test pins these against a literal transcription of the reference's per-arc loops.
"""
from __future__ import annotations

import numpy as np
from scipy import sparse

ARC_BLOCK = 1 << 25  # arcs x genes per block of the B sum


def _dense(x) -> np.ndarray:
    x = x.toarray() if sparse.issparse(x) else np.asarray(x)
    return x.astype(np.float64)


def sums(graph, x):
    """`graph` scipy sparse [n x n], `x` [n x g] (cells along the rows) -> (A, B, Q) fp64 [g] each, and the constant
    flag [g]."""
    w = sparse.csr_matrix(graph).astype(np.float64)
    x = _dense(x)
    n, g = x.shape
    z = x - x.mean(axis=0)
    a = (z * (w @ z)).sum(axis=0)
    q = (z * z).sum(axis=0)
    rows = np.repeat(np.arange(n), np.diff(w.indptr))
    cols, wt = w.indices, w.data
    b = np.empty(g)
    step = max(1, ARC_BLOCK // max(1, len(cols)))
    for c0 in range(0, g, step):
        d = x[rows, c0:c0 + step] - x[cols, c0:c0 + step]
        b[c0:c0 + step] = (wt[:, None] * (d * d)).sum(axis=0)
    with np.errstate(invalid="ignore"):
        constant = ~np.isnan(x).any(axis=0) & (x == x[:1]).all(axis=0) if n else np.ones(g, dtype=bool)
    return a, b, q, constant


def _finish(stat, graph, x):
    a, b, q, constant = sums(graph, x)
    n = graph.shape[0]
    s0 = np.asarray(graph.data, dtype=np.float64).sum()
    with np.errstate(divide="ignore", invalid="ignore"):
        out = stat(n, s0, a, b, q)
    out[constant] = np.nan
    return out


def morans_i(graph, x) -> np.ndarray:
    """Moran's I of every column of `x` [n x g] on `graph`."""
    return _finish(lambda n, s0, a, b, q: n / s0 * a / q, graph, x)


def gearys_c(graph, x) -> np.ndarray:
    """Geary's C of every column of `x` [n x g] on `graph`."""
    return _finish(lambda n, s0, a, b, q: (n - 1) * b / (2 * s0 * q), graph, x)

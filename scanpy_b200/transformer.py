"""sklearn-shaped plug-ins: the reference's own operator API for this path.

`B200KNNTransformer` satisfies `KnnTransformerLike` (src/scanpy/neighbors/_types.py:53-64): pass it as
`sc.pp.neighbors(adata, transformer=B200KNNTransformer(n_neighbors=15))` into UNMODIFIED scanpy
(precedent: src/scanpy/neighbors/_backends/rapids.py:39-101).  `transform` returns a CSR distance
matrix with exactly `n_neighbors` stored entries per row, self included in column 0 (pynndescent
style), ascending by distance — the layout `_ind_dist_shortcut` (src/scanpy/neighbors/_common.py:126-143)
expects.  `B200PCA` exposes the attribute set `pca()` reads from a fitted sklearn PCA
(src/scanpy/preprocessing/_pca/__init__.py:349-362).
"""
from __future__ import annotations

import numpy as np
from scipy import sparse

from . import _ops
from ._compat import as_csr_f32


class B200KNNTransformer:
    """Exact euclidean kNN on one H100 (hand-written sm_90a kernels, see csrc/knn.cu)."""

    def __init__(self, n_neighbors: int = 15, *, metric: str = "euclidean", **_ignored):
        if metric not in ("euclidean", "l2"):
            raise NotImplementedError(f"metric={metric!r}: only 'euclidean' is implemented")
        self.n_neighbors = int(n_neighbors)
        self.metric = metric
        self._fit_x = None
        self.last_info_ = None

    def get_params(self, deep: bool = True) -> dict:
        return dict(n_neighbors=self.n_neighbors, metric=self.metric)

    def set_params(self, **params):
        for k, v in params.items():
            if k not in ("n_neighbors", "metric"):
                raise ValueError(f"Invalid parameter {k!r} for B200KNNTransformer")
            setattr(self, k, v)
        return self

    def fit(self, x, y=None):
        if sparse.issparse(x):
            x = x.toarray()
        self._fit_x = np.ascontiguousarray(x, dtype=np.float32)
        return self

    def transform(self, x=None):
        if self._fit_x is None:
            raise RuntimeError("B200KNNTransformer is not fitted")
        if x is not None:
            xq = x.toarray() if sparse.issparse(x) else np.asarray(x)
            if xq.shape != self._fit_x.shape or not np.array_equal(np.asarray(xq, np.float32), self._fit_x):
                raise NotImplementedError("B200KNNTransformer.transform only answers queries for the fitted points "
                                          "(the only use scanpy makes of it)")
        n = self._fit_x.shape[0]
        k = min(self.n_neighbors, n)
        idx, dist, info = _ops.knn(self._fit_x, k)
        self.last_info_ = info
        indptr = np.arange(0, n * k + 1, k, dtype=np.int64 if n * k >= 2**31 else np.int32)
        return sparse.csr_matrix((dist.ravel(), idx.ravel(), indptr), shape=(n, n))

    def fit_transform(self, x, y=None):
        return self.fit(x).transform()


class B200PCA:
    """sklearn.decomposition.PCA-shaped front-end of `sb2_pca_csr_f32` (zero-centred, CSR or dense input)."""

    def __init__(self, n_components: int, *, svd_solver: str = "arpack", random_state: int = 0):
        self.n_components = n_components
        self.svd_solver = svd_solver
        self.random_state = random_state

    def fit_transform(self, x, y=None):
        from .pp import _solver_code

        xc = as_csr_f32(x)
        out = _ops.pca_csr(xc, self.n_components, solver=_solver_code(self.svd_solver, n_vars=xc.shape[1]),
                           seed=int(self.random_state or 0))
        if not out["converged"]:
            import warnings

            warnings.warn(f"B200PCA did not reach its residual tolerance (max relative residual {out['max_rel_residual']:.3g})",
                          UserWarning, stacklevel=2)
        self.components_ = out["components"]
        self.explained_variance_ = out["variance"]
        self.explained_variance_ratio_ = out["variance_ratio"]
        self.mean_ = out["mean"]
        self.singular_values_ = np.sqrt(out["variance"] * (xc.shape[0] - 1))
        self.n_iter_ = out["iterations"]
        return out["X_pca"]

    def fit(self, x, y=None):
        self.fit_transform(x)
        return self

"""`sc.metrics.modularity` on the device (SURVEY.md 8f row f3; src/scanpy/metrics/_metrics.py:125-223).

The reference builds an igraph from the adjacency and calls `Graph.modularity(codes, "weight")` (resolution 1); here the
CSR graph goes to sb2_modularity_csr_f32 (fixed-point community totals, csrc/leiden.cu) and never leaves the device.
"""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import sparse

from . import _ops
from ._compat import is_anndata_like
from .tl import _choose_graph


def _codes(labels):
    """_metrics.py:216-223."""
    if isinstance(labels, pd.Series):
        labels = labels.astype("category").array
    if not isinstance(labels, pd.Categorical):
        labels = pd.Categorical(labels)
    return labels.codes


def modularity(adata_or_connectivities, /, labels="leiden", *, neighbors_key: str | None = None,
               is_directed: bool | None = None, mode: str = "calculate") -> float:
    """Modularity of a clustering on a connectivities graph (signature of `scanpy.metrics.modularity`)."""
    if is_anndata_like(adata_or_connectivities):
        adata = adata_or_connectivities
        if is_directed:
            raise ValueError(f"Connectivities stored in `AnnData` are undirected, can’t specify `{is_directed=!r}`")
        if mode in {"retrieve", "update"} and not isinstance(labels, str):
            raise ValueError("`labels` must be a string when `mode` is `'retrieve'` or `'update'`")
        if mode == "retrieve":
            return adata.uns[labels]["modularity"]
        labels_vec = adata.obs[labels] if isinstance(labels, str) else labels
        m = modularity(_choose_graph(adata, None, neighbors_key), labels_vec, is_directed=False)
        if mode == "update":
            adata.uns[labels]["modularity"] = m
        return m
    if isinstance(labels, str):
        raise TypeError("`labels` must be provided as array when passing a connectivities array")
    if is_directed is None:
        raise TypeError("`is_directed` must be provided when passing a connectivities array")
    adj = adata_or_connectivities
    adj = adj.tocsr() if sparse.issparse(adj) else sparse.csr_matrix(np.asarray(adj))
    if is_directed:
        # igraph's directed modularity uses out-/in-strength products; only the symmetric objective runs on the device
        if (abs(adj - adj.T) > 1e-12 * max(1.0, abs(adj).max())).nnz:
            raise NotImplementedError("directed modularity of a non-symmetric adjacency is not implemented in scanpy_b200")
    if adj.dtype != np.float32:
        adj = adj.astype(np.float32)
    # a missing label has code -1, which _ops.modularity rejects (igraph rejects a negative membership too)
    return float(_ops.modularity(adj, np.asarray(_codes(labels)), resolution=1.0))

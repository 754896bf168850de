"""`sc.metrics` on the device.

* `modularity` (SURVEY.md 8f row f3; src/scanpy/metrics/_metrics.py:125-223): the reference builds an igraph from the
  adjacency and calls `Graph.modularity(codes, "weight")` (resolution 1); here the CSR graph goes to
  sb2_modularity_csr_f32 (fixed-point community totals, csrc/leiden.cu) and never leaves the device.
* `morans_i` and `gearys_c` (src/scanpy/metrics/_morans_i.py, _gearys_c.py, _common.py): the per-feature graph sums
  A, B and Q run in CUDA (`_autocorr`, csrc/autocorr.cu); the final formulas are the reference's, in fp64 on the host:
  Moran's I = n / S0 * A / Q and Geary's C = (n - 1) * B / (2 * S0 * Q), S0 the sum of the graph's weights.
"""
from __future__ import annotations

import warnings

import numpy as np
import pandas as pd
from scipy import sparse

from . import _ops
from ._autocorr import graph_sums
from ._compat import get_arr, is_anndata_like
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


# ------------------------------------------------------------------------------------------ Moran's I, Geary's C
def _get_graph(adata, *, use_graph: str | None, neighbors_key: str | None):
    """_common.py `_get_graph`, with `NeighborsView` (src/scanpy/_utils/__init__.py:857-965) restated."""
    if use_graph is not None:
        if neighbors_key is not None:
            raise TypeError("Cannot specify both `use_graph` and `neighbors_key`.")
        return adata.obsp[use_graph]
    if neighbors_key is None or neighbors_key == "neighbors":
        if "neighbors" not in adata.uns:
            raise KeyError('No "neighbors" in .uns')
        neighbors, conns_key = adata.uns["neighbors"], "connectivities"
    else:
        if neighbors_key not in adata.uns:
            raise KeyError(f"No {neighbors_key!r} in .uns")
        neighbors = adata.uns[neighbors_key]
        conns_key = neighbors["connectivities_key"]
    conns = adata.obsp[conns_key] if conns_key in adata.obsp else neighbors.get(conns_key)
    if conns is None:
        raise ValueError("Must run neighbors first.")
    return conns


def _resolve_vals(val):
    """_common.py `_resolve_vals`: an ndarray, or a CSR for any scipy sparse format."""
    if type(val).__module__.startswith("dask"):
        raise NotImplementedError("dask arrays are not supported by scanpy_b200's morans_i and gearys_c")
    if isinstance(val, (pd.DataFrame, pd.Series)):
        return val.to_numpy()
    if isinstance(val, np.ndarray):
        return np.asarray(val)
    if sparse.issparse(val):
        return val.tocsr()
    raise TypeError(f"Unsupported type {type(val)}")


def _autocorrelation(name: str, graph, vals, *, cells_along_rows: bool):
    """(n, S0, [A, B, Q] [3 x g], constant [g], one_dim) of the features of `vals`: (n_features, n_cells) or (n_cells,),
    or (n_cells, n_features) with `cells_along_rows` (what `_get_arr` returns: it goes to the device untransposed)."""
    if not (sparse.issparse(graph) and graph.format == "csr"):
        raise TypeError(f"{name}: the graph must be a scipy CSR matrix, not {type(graph)}")
    # the reference's asserts (_common.py), raised explicitly so that they hold under `python -O` too
    if graph.shape[0] != graph.shape[1]:
        raise AssertionError("`g` should be a square adjacency matrix")
    x = _resolve_vals(vals)
    n = graph.shape[0]
    one_dim = x.ndim == 1
    if one_dim:
        x = x.reshape(-1, 1)
    elif x.ndim != 2:
        raise NotImplementedError(f"{name} metric not implemented for vals of type {type(x).__module__}."
                                  f"{type(x).__qualname__} and ndim {x.ndim}.")
    elif not cells_along_rows:
        x = x.T  # an ndarray view, or a CSR's CSC twin: the device reads it as CSR
    if x.shape[0] != n:
        raise AssertionError(f"{name}: the graph has {n} cells, the values {x.shape[0]}")
    if x.dtype not in (np.float32, np.float64):
        x = x.astype(np.float64)
    s0 = graph.data.astype(np.float64).sum()
    if x.shape[1] == 0:
        return n, s0, np.zeros((3, 0)), np.zeros(0, dtype=bool), one_dim
    sums, constant = graph_sums(graph, x)
    return n, s0, sums, constant, one_dim


def _finish(stat, n, s0, sums, constant, one_dim):
    """The reference's constant handling around `stat(n, s0, A, B, Q)`: a constant 1-D vector divides 0 / 0 in its numba
    kernel (ZeroDivisionError); constant rows of a matrix get NaN, with the reference's warning."""
    if one_dim:
        if constant[0]:
            raise ZeroDivisionError("division by zero")
        return np.float64(stat(float(n), float(s0), *(float(v) for v in sums[:, 0])))
    with np.errstate(divide="ignore", invalid="ignore"):
        out = stat(n, s0, *sums)
    if constant.any():
        # stacklevel: the caller of morans_i / gearys_c
        warnings.warn(f"{int(constant.sum())} variables were constant, will return nan for these.", UserWarning,
                      stacklevel=4)
        out[constant] = np.nan
    return out


def _metric(stat, name: str, adata_or_graph, vals, *, use_graph, neighbors_key, layer, obsm, obsp, use_raw):
    """`stat(n, S0, A, B, Q)` of every feature: `morans_i` / `gearys_c` for an AnnData (the graph and, without `vals`,
    the cells x features matrix chosen from it) or a CSR graph."""
    rows = False
    graph = adata_or_graph
    if is_anndata_like(adata_or_graph):
        graph = _get_graph(adata_or_graph, use_graph=use_graph, neighbors_key=neighbors_key)
        if vals is None:
            vals, rows = get_arr(adata_or_graph, use_raw=use_raw, layer=layer, obsm=obsm, obsp=obsp), True
    return _finish(stat, *_autocorrelation(name, graph, vals, cells_along_rows=rows))


def _morans_i(n, s0, a, b, q):
    return n / s0 * a / q


def _gearys_c(n, s0, a, b, q):
    return (n - 1) * b / (2 * s0 * q)


def morans_i(adata_or_graph, /, vals=None, *, use_graph: str | None = None, neighbors_key: str | None = None,
             layer: str | None = None, obsm: str | None = None, obsp: str | None = None, use_raw: bool = False):
    """Moran's I global autocorrelation of each feature on a graph (signature of `scanpy.metrics.morans_i`).

    `vals` (n_features, n_cells) or (n_cells,), or chosen from the AnnData with `layer` / `obsm` / `obsp` / `use_raw`;
    the graph is `.obsp[use_graph]` or the neighbors connectivities.  Returns a float64 array, or a scalar for 1-D
    `vals`; constant features get NaN."""
    return _metric(_morans_i, "Moran’s I", adata_or_graph, vals, use_graph=use_graph, neighbors_key=neighbors_key,
                   layer=layer, obsm=obsm, obsp=obsp, use_raw=use_raw)


def gearys_c(adata_or_graph, /, vals=None, *, use_graph: str | None = None, neighbors_key: str | None = None,
             layer: str | None = None, obsm: str | None = None, obsp: str | None = None, use_raw: bool = False):
    """Geary's C autocorrelation of each feature on a graph (signature of `scanpy.metrics.gearys_c`); arguments and
    results as `morans_i`."""
    return _metric(_gearys_c, "Geary’s C", adata_or_graph, vals, use_graph=use_graph, neighbors_key=neighbors_key,
                   layer=layer, obsm=obsm, obsp=obsp, use_raw=use_raw)

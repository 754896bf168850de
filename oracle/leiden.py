"""ctypes wrapper around oracle/leiden_ref.c (test infrastructure only; see oracle/__init__.py).

Mirrors what scanpy's `leiden()` extracts from the back-end: `.membership` and `.modularity`
(src/scanpy/tools/_leiden.py:198,219).  Label level: the reference's tests hold no Leiden golden, but its in-tree fixture
pbmc68k_reduced stores `obs/louvain` (scanpy's own sc.tl.louvain output on the stored connectivities); on the unweighted
graph this oracle reproduces it at ARI 0.94-0.98 (tests/test_oracle_leiden_guarantees.py).
"""
from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path

import numpy as np
from scipy import sparse

_HERE = Path(__file__).resolve().parent
_lib = None


def build() -> Path:
    so = _HERE / "libleiden_ref.so"
    src = _HERE / "leiden_ref.c"
    if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        subprocess.run(["make", "-C", str(_HERE), "libleiden_ref.so"], check=True, capture_output=True)
    return so


def _load():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(str(build()))
        P = ctypes.c_void_p
        lib.leiden_ref.restype = ctypes.c_int
        lib.leiden_ref.argtypes = [ctypes.c_int32, P, P, P, ctypes.c_double, ctypes.c_int32, ctypes.c_uint64,
                                   P, P, P, P]
        lib.leiden_ref2.restype = ctypes.c_int
        lib.leiden_ref2.argtypes = [ctypes.c_int32, P, P, P, ctypes.c_double, ctypes.c_int32, ctypes.c_uint64, ctypes.c_double,
                                    P, P, P, P]
        lib.modularity_ref.restype = ctypes.c_double
        lib.modularity_ref.argtypes = [ctypes.c_int32, P, P, P, ctypes.c_double, P]
        _lib = lib
    return _lib


def _csr_args(adj):
    adj = adj.tocsr()
    indptr = np.ascontiguousarray(adj.indptr, np.int64)
    indices = np.ascontiguousarray(adj.indices, np.int32)
    w = np.ascontiguousarray(adj.data, np.float64)
    return adj.shape[0], indptr, indices, w


def leiden(adj, *, resolution: float = 1.0, n_iterations: int = -1, seed: int = 0, beta: float = 0.0):
    """-> (membership int32[n] renumbered by decreasing size, modularity at `resolution`, n_passes).

    beta = 0: greedy refinement, what leidenalg's optimiser does for scanpy's flavor='leidenalg';
    beta > 0: the paper's randomised refinement over well-connected vertices/communities, what igraph's
    community_leiden does for flavor='igraph' (scanpy passes igraph's default beta = 0.01)."""
    lib = _load()
    n, indptr, indices, w = _csr_args(adj)
    member = np.empty(n, np.int32)
    q = ctypes.c_double()
    nc = ctypes.c_int32()
    passes = ctypes.c_int32()
    rc = lib.leiden_ref2(n, indptr.ctypes.data, indices.ctypes.data, w.ctypes.data, float(resolution),
                         int(n_iterations), int(seed), float(beta), member.ctypes.data, ctypes.addressof(q),
                         ctypes.addressof(nc), ctypes.addressof(passes))
    assert rc == 0
    return member, q.value, passes.value


def modularity(adj, membership, *, resolution: float = 1.0) -> float:
    lib = _load()
    n, indptr, indices, w = _csr_args(adj)
    m = np.ascontiguousarray(membership, np.int32)
    return lib.modularity_ref(n, indptr.ctypes.data, indices.ctypes.data, w.ctypes.data, float(resolution),
                              m.ctypes.data)


# ------------------------------------------------------------------------------------------ plain fp64 checks
def _graph64(adj):
    """float64 CSR copy without stored zeros (a stored zero is not an edge, like the reference's `adjacency.nonzero()`)."""
    g = sparse.csr_matrix(adj, dtype=np.float64, copy=True)
    g.eliminate_zeros()
    return g


def modularity_fp64(adj, labels, *, resolution: float = 1.0) -> float:
    """Q = (sum of the stored arcs (i, j) with c_i == c_j  -  gamma sum_c K_c^2 / W) / W in plain numpy float64, with
    W = the sum of all stored arcs and K_c = the sum of the row sums of c's members.  A self-loop is one stored arc and
    counts once: this is Q of the reference's igraph graph, where every stored entry becomes one edge.  (networkx counts a
    loop twice in a degree, so it is no reference on graphs with self-loops.)  Labels may have gaps; 0 for an empty graph."""
    g = _graph64(adj)
    m = np.asarray(labels).ravel().astype(np.int64)
    total = g.data.sum()
    if total == 0.0:
        return 0.0
    rows = np.repeat(np.arange(g.shape[0]), np.diff(g.indptr))
    internal = g.data[m[rows] == m[g.indices]].sum()
    kc = np.bincount(m, weights=np.asarray(g.sum(axis=1)).ravel())
    return float((internal - resolution * (kc @ kc) / total) / total)


def community_tables(g, m):
    """-> (k, W, ind, e, kc) of a float64 CSR graph and labels m: vertex strengths (row sums, a self-loop once), the total
    W, the n x nc community indicator, e[c, d] = the weight of the arcs from c to d (sparse) and the community strengths."""
    n = g.shape[0]
    k = np.asarray(g.sum(axis=1)).ravel()
    nc = int(m.max()) + 1 if n else 0
    ind = sparse.csr_matrix((np.ones(n), (np.arange(n), m)), shape=(n, nc))
    e = (ind.T @ g @ ind).tocoo()
    kc = np.asarray(ind.T @ k).ravel()
    return k, k.sum(), ind, e, kc


def check_guarantees(adj, labels, gamma: float = 1.0, *, connected: bool = True, separated: bool = True,
                     node_optimal: bool = True, rtol: float = 1e-9) -> None:
    """Assert the guarantees Traag, Waltman & van Eck (2019) prove for a converged Leiden run, for the RB objective at
    resolution `gamma` (gains in weight units, tolerance rtol x the largest arc weight, so scaled graphs check alike):
      connected     every community induces a connected subgraph (Leiden, after any number of iterations)
      separated     gamma-separation: merging two communities never gains,  e_cd - gamma K_c K_d / W <= tol
      node_optimal  no vertex gains by moving to another existing community:  w(v, c) - gamma k_v K_c / W  is not above
                    staying,  w(v, own \\ v) - gamma k_v (K_own - k_v) / W  (a vertex's own self-loop is left out of its
                    weight to its own community; moves to an empty community are not checked)."""
    from scipy.sparse.csgraph import connected_components

    g = _graph64(adj)
    m = np.asarray(labels).ravel().astype(np.int64)
    n = g.shape[0]
    assert m.shape == (n,) and (m >= 0).all()
    tol = rtol * (g.data.max() if g.nnz else 0.0)
    k, two_m, ind, e, kc = community_tables(g, m)
    nc = kc.size
    rows = np.repeat(np.arange(n), np.diff(g.indptr))
    cols = g.indices
    same = m[rows] == m[cols]
    if connected:
        # the arcs inside communities split every community into components: connected iff exactly one per community
        intra = sparse.csr_matrix((np.ones(int(same.sum())), (rows[same], cols[same])), shape=(n, n))
        _, comp = connected_components(intra, directed=False)
        pairs = np.unique(np.stack([m, comp]), axis=1)
        per = np.bincount(pairs[0], minlength=nc)
        bad = np.flatnonzero(per > 1)
        assert bad.size == 0, f"community {bad[0]} has {per[bad[0]]} components ({bad.size} disconnected communities)"
    if two_m == 0.0:
        return
    if separated:
        off = e.row != e.col
        gain = e.data[off] - gamma * kc[e.row[off]] * kc[e.col[off]] / two_m
        if gain.size:
            assert gain.max() <= tol, f"two communities could be merged with gain {gain.max():.6g} (tolerance {tol:.3g})"
    if node_optimal:
        loop = rows == cols
        own_w = np.bincount(rows[same & ~loop], weights=g.data[same & ~loop], minlength=n)
        stay = own_w - gamma * k * (kc[m] - k) / two_m
        # the best move to an adjacent community ...
        wv = (g @ ind).tocoo()
        other = wv.col != m[wv.row]
        best = np.full(n, -np.inf)
        np.maximum.at(best, wv.row[other], wv.data[other] - gamma * k[wv.row[other]] * kc[wv.col[other]] / two_m)
        # ... or to the weakest non-empty community other than its own (no weight towards it: gain -gamma k_v K_c / W)
        alive = np.flatnonzero(np.bincount(m, minlength=nc) > 0)
        if alive.size > 1:
            order = alive[np.argsort(kc[alive], kind="stable")]
            weakest = np.where(m == order[0], kc[order[1]], kc[order[0]])
            best = np.maximum(best, -gamma * k * weakest / two_m)
        excess = best - stay
        v = int(np.argmax(excess))
        assert excess[v] <= tol, f"vertex {v} could still be moved with a gain of {excess[v]:.6g} (tolerance {tol:.3g})"

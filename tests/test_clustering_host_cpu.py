"""Host-side parts of the clustering path, no GPU: label checks of metrics.modularity, the graph tl.leiden / tl.louvain
hand to the device, and the fp64 references (oracle.leiden.modularity_fp64 / check_guarantees) the device tests use."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import leiden as old
from scanpy_b200 import _abi, _ops, tl


@pytest.fixture
def no_device(monkeypatch):
    """Any device call fails the test: the checks under test must come first."""
    def boom(*a, **k):
        raise AssertionError("the device was reached")
    monkeypatch.setattr(_abi, "default_context", boom)
    monkeypatch.setattr(_ops, "csr_to_device", boom)


def _two_triangles():
    i = np.array([0, 0, 1, 3, 3, 4, 2])
    j = np.array([1, 2, 2, 4, 5, 5, 3])
    g = sparse.csr_matrix((np.ones(7), (i, j)), shape=(6, 6))
    return (g + g.T).tocsr().astype(np.float32)


def test_modularity_rejects_missing_labels_before_any_device_call(no_device):
    g = _two_triangles()
    with pytest.raises(ValueError, match="missing"):
        sb.metrics.modularity(g, ["a", "a", None, "b", "b", "b"], is_directed=False)
    with pytest.raises(ValueError, match="missing"):
        sb.metrics.modularity(g, pd.Series(["a", "a", "a", np.nan, "b", "b"]), is_directed=False)
    with pytest.raises(ValueError, match="non-negative"):
        _ops.modularity(g, np.array([0, 0, 0, -1, 1, 1]))
    with pytest.raises(ValueError, match="6 vertices"):
        _ops.modularity(g, np.zeros(5, int))


def test_clustering_graph_drops_explicit_zeros():
    g = _two_triangles()
    assert tl._clustering_graph(g, use_weights=True) is g          # nothing to drop: no copy
    z = g.copy()
    z.data[z.indices == 5] = 0.0                                    # stored zeros in column 5 only (not symmetric: fine here)
    out = tl._clustering_graph(z, use_weights=True)
    assert out is not z and (z.data == 0).sum() == 2                # the caller's matrix is left alone
    assert out.nnz == g.nnz - 2 and (out.data != 0).all() and out.dtype == np.float32
    ones = tl._clustering_graph(z * 3.5, use_weights=False)
    assert ones.nnz == g.nnz - 2 and (ones.data == 1.0).all()
    f64 = tl._clustering_graph(g.astype(np.float64), use_weights=True)
    assert f64.dtype == np.float32 and (f64 != g).nnz == 0


def test_modularity_fp64_counts_a_self_loop_once():
    # arcs 0-1 (weight 1 each way) and a loop of weight 2 on vertex 2: W = 4, k = (1, 1, 2)
    g = sparse.csr_matrix((np.array([1.0, 1.0, 2.0]), (np.array([0, 1, 2]), np.array([1, 0, 2]))), shape=(3, 3))
    assert old.modularity_fp64(g, [0, 0, 1]) == pytest.approx((4 - (2 * 2 + 2 * 2) / 4) / 4, abs=1e-15)
    assert old.modularity_fp64(g, [5, 5, 9], resolution=0.5) == pytest.approx((4 - 0.5 * 8 / 4) / 4, abs=1e-15)
    assert old.modularity_fp64(g, [0, 1, 2]) == pytest.approx((2 - 6 / 4) / 4, abs=1e-15)
    assert old.modularity_fp64(sparse.csr_matrix((3, 3)), [0, 1, 2]) == 0.0


def test_modularity_fp64_matches_the_oracle_and_networkx_without_loops(pbmc68k_graph):
    import networkx as nx

    f = pbmc68k_graph
    g = sparse.csr_matrix((f["conn_data"].astype(np.float64), f["conn_indices"], f["conn_indptr"]), shape=(700, 700))
    lab = f["louvain_codes"].astype(int)
    G = nx.from_scipy_sparse_array(g)
    comms = [set(np.flatnonzero(lab == c).tolist()) for c in range(lab.max() + 1)]
    for gamma in (0.3, 1.0, 2.5):
        q = old.modularity_fp64(g, lab, resolution=gamma)
        assert abs(q - old.modularity(g, lab, resolution=gamma)) < 1e-12
        assert abs(q - nx.community.modularity(G, comms, weight="weight", resolution=gamma)) < 1e-12
        assert old.modularity_fp64(g * 2.0**-40, lab, resolution=gamma) == pytest.approx(q, abs=1e-14)


def _ring(r=6, s=5, eps=0.5, loops=0.0):
    g = sparse.lil_matrix((r * s, r * s))
    for c in range(r):
        for a in range(s):
            for b in range(a + 1, s):
                g[c * s + a, c * s + b] = g[c * s + b, c * s + a] = 1.0
        u, v = c * s, ((c + 1) % r) * s + 1
        g[u, v] = g[v, u] = eps
    g.setdiag(loops)
    return g.tocsr()


@pytest.mark.parametrize("scale", [1.0, 2.0**-50, 1e12])
@pytest.mark.parametrize("loops", [0.0, 3.0])
def test_check_guarantees_accepts_the_optimum_and_rejects_each_violation(scale, loops):
    """The checker must pass the clique partition of a ring of cliques (the optimum: eps < s(s-1)/r) at any weight scale,
    with or without self-loops, and fail on a disconnected community, a mergeable pair and a misplaced vertex."""
    g = _ring(loops=loops) * scale
    r, s = 6, 5
    good = np.repeat(np.arange(r), s)
    old.check_guarantees(g, good)
    split = good.copy()
    split[[0, 1, 7, 8]] = r                     # {0, 1} of clique 0 and {7, 8} of clique 1: one community, two pieces
    with pytest.raises(AssertionError, match="components"):
        old.check_guarantees(g, split, separated=False, node_optimal=False)
    with pytest.raises(AssertionError, match="merged"):
        old.check_guarantees(g, good, 0.0, connected=False, node_optimal=False)   # at gamma = 0 every adjacent pair merges
    moved = good.copy()
    moved[2] = 1                                 # vertex 2 (all its arcs inside clique 0) placed in clique 1
    with pytest.raises(AssertionError, match="moved"):
        old.check_guarantees(g, moved, connected=False, separated=False)
    # the self-loop of a vertex is not weight towards its own community: with a huge loop on vertex 2, staying in
    # clique 0 is still worth only its 4 clique arcs
    h = g.tolil()
    h[2, 2] = 1e6 * scale
    with pytest.raises(AssertionError, match="moved"):
        old.check_guarantees(h.tocsr(), moved, 1e-9, connected=False, separated=False)

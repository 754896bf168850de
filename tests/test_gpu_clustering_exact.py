"""Leiden, Louvain and modularity (csrc/leiden.cu) against answers that are exact, not just good.

Every case has one right answer: connected components at resolution 0, singletons at a huge resolution, the clique
partition of a ring of cliques, the guarantees Traag, Waltman & van Eck (2019) prove for a converged Leiden run
(oracle.leiden.check_guarantees), the plain fp64 modularity formula (oracle.leiden.modularity_fp64), identical results
under a power-of-two rescaling of the weights, and identical results with explicitly stored zeros.

The kernels work on fixed-point weights: one unit is 2^-e of the input, e = 32 - ceil(log2(max arc weight)), so an arc
moves by at most half a unit (<= 2^-33 x the largest weight).  The guarantees and the fp64 formula are evaluated on that
fixed-point graph (`_device_graph`), where they must hold to 1e-9; Q is also compared with the float32 input graph.
Labels and Q are in the form the device returns: communities ordered by decreasing size, ties by the smaller first member.
"""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse
from scipy.sparse.csgraph import connected_components
from sklearn.metrics import adjusted_rand_score

import scanpy_b200 as sb
from oracle import leiden as old
from scanpy_b200 import _ops
from scanpy_b200._abi import B200Error
from scanpy_b200._synth import synth_scipy

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------ graphs and helpers
def _renumber(lab):
    """Labels in the device's order: decreasing community size, ties -> smaller first member."""
    _, first, inv, cnt = np.unique(lab, return_index=True, return_inverse=True, return_counts=True)
    order = np.lexsort((first, -cnt))
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    return rank[inv.ravel()]


def _device_graph(g):
    """The graph the kernels optimise: the float32 weights rounded to the fixed-point grid 2^-e (ties to even, like llrint)."""
    g = sparse.csr_matrix(g, dtype=np.float32).astype(np.float64)
    if g.nnz == 0 or g.data.max() == 0.0:
        return g
    f, ex = np.frexp(g.data.max())
    e = 32 - (int(ex) - 1 if f == 0.5 else int(ex))
    g.data = np.ldexp(np.rint(np.ldexp(g.data, e)), -e)
    return g


def _close(q, ref, tol=1e-9):
    return abs(q - ref) <= tol * max(1.0, abs(ref))


def _sym(n, i, j, w, loops=None):
    """Symmetric float32 CSR from undirected edges (i, j, w) with i != j, plus self-loops {v: w} stored once."""
    i, j, w = np.asarray(i, np.int64), np.asarray(j, np.int64), np.asarray(w, np.float64)
    v = np.array(list((loops or {}).keys()), np.int64)
    wv = np.array(list((loops or {}).values()), np.float64)
    g = sparse.csr_matrix((np.r_[w, w, wv], (np.r_[i, j, v], np.r_[j, i, v])), shape=(n, n), dtype=np.float64)
    g.sort_indices()
    return g.astype(np.float32)


def _components_graph(seed=0):
    """Components of distinct sizes (random trees + extra edges, weights in [0.5, 2]), 5 isolated vertices and one vertex
    whose only arc is a self-loop, in shuffled vertex order.  -> (graph, component of every vertex)."""
    rs = np.random.RandomState(seed)
    sizes = [60, 33, 17, 9, 4, 2]
    n = sum(sizes) + 5 + 1
    perm = rs.permutation(n)
    pairs, comp, start = set(), np.arange(n), 0
    for s in sizes:
        vs = np.arange(start, start + s)
        comp[vs] = start
        edges = [(vs[t], vs[rs.randint(t)]) for t in range(1, s)]                  # random spanning tree ...
        edges += [tuple(rs.choice(vs, 2, replace=False)) for _ in range(s)]          # ... plus random chords
        pairs |= {(min(a, b), max(a, b)) for a, b in edges}
        start += s
    i, j = np.array(sorted(pairs)).T
    g = _sym(n, perm[i], perm[j], rs.uniform(0.5, 2.0, len(i)), loops={perm[n - 1]: 1.5})   # vertex n-1: loop only
    lab = np.empty(n, np.int64)
    lab[perm] = comp
    return g, lab


def _ring_of_cliques(r, s, eps):
    """r cliques K_s with unit weights; clique t is joined to clique t+1 (mod r) by one edge of weight eps."""
    iu, ju = np.triu_indices(s, 1)
    base = (np.arange(r) * s)[:, None]
    i = np.concatenate([(base + iu).ravel(), np.arange(r) * s])
    j = np.concatenate([(base + ju).ravel(), (np.arange(r) * s + s + 1) % (r * s)])
    w = np.concatenate([np.ones(r * len(iu)), np.full(r, eps)])
    return _sym(r * s, i, j, w)


_KNN = {}


def _knn_graph(seed=0, n=3000):
    """UMAP connectivities of a synthetic count matrix (_synth) through the CUDA pca -> neighbors path."""
    if (seed, n) not in _KNN:
        x, _ = synth_scipy(n, 400, n_clusters=10, r=24, seed=seed)
        ad = sb.MiniAnnData(x)
        sb.pp.pca(ad, n_comps=20)
        sb.pp.neighbors(ad, n_neighbors=15)
        _KNN[seed, n] = ad.obsp["connectivities"].astype(np.float32)
    return _KNN[seed, n].copy()


def _with_hubs(g, seed, n_hubs=16, degree=2000):
    """g plus n_hubs new vertices, each joined to `degree`+ random vertices (weights in (0, 1]): rows far above 32
    arcs, the hash-slice branch of the level-0 decisions."""
    rs = np.random.RandomState(seed)
    n = g.shape[0]
    i, j = [], []
    for h in range(n_hubs):
        nb = rs.choice(n, degree + rs.randint(0, 200), replace=False)
        i.append(np.full(nb.size, n + h)), j.append(nb)
    i, j = np.concatenate(i), np.concatenate(j)
    extra = _sym(n + n_hubs, i, j, rs.uniform(1e-3, 1.0, i.size))
    big = sparse.block_diag([g, sparse.csr_matrix((n_hubs, n_hubs))], format="csr", dtype=np.float32)
    return (big + extra).tocsr()


def _with_loops(g, seed, frac=0.2):
    rs = np.random.RandomState(seed)
    v = rs.choice(g.shape[0], int(frac * g.shape[0]), replace=False)
    loops = sparse.csr_matrix((rs.uniform(0.05, 1.0, v.size), (v, v)), shape=g.shape)
    return (g.astype(np.float64) + loops).astype(np.float32).tocsr()


def _wide_weights(g, seed, lo=1e-6, hi=1e3):
    """Same arcs (self-loops included), symmetric weights log-uniform in [lo, hi]."""
    rs = np.random.RandomState(seed)
    u = sparse.triu(g, 0, format="csr").astype(np.float64)
    u.data = 10.0 ** rs.uniform(np.log10(lo), np.log10(hi), u.nnz)
    return (u + sparse.triu(u, 1).T).astype(np.float32).tocsr()


def _adata(n):
    return sb.MiniAnnData(sparse.csr_matrix((n, 1), dtype=np.float32))


def _general_graph(kind, seed):
    g = _knn_graph(seed)
    if kind == "hubs":
        g = _with_hubs(g, seed)
    elif kind == "loops":
        g = _with_loops(g, seed)
    elif kind == "wide":
        g = _wide_weights(g, seed)
    return g


# ------------------------------------------------------------------------------------------ resolution extremes
def test_resolution_zero_gives_connected_components():
    """At gamma = 0 every arc is a gain: the optimum is the connected components, isolated and self-loop-only vertices
    stay alone.  Leiden and Louvain must return exactly the (renumbered) components."""
    for seed in range(3):
        g, _ = _components_graph(seed)
        _, cc = connected_components(g, directed=False)
        want = _renumber(cc)
        m, q, _ = _ops.leiden(g, resolution=0.0, seed=seed)
        np.testing.assert_array_equal(m, want)
        assert _close(q, old.modularity_fp64(_device_graph(g), m, resolution=0.0)) and _close(q, 1.0)
        ml, ql, _ = _ops.louvain(g, resolution=0.0, seed=seed)
        np.testing.assert_array_equal(ml, want)
        assert _close(ql, 1.0)


def test_huge_resolution_gives_singletons():
    """At gamma = 1e6 every merge loses (weights >= 0.5, total weight ~ 500): every vertex stays alone, labels are
    arange(n) and Q = (self-loops - gamma sum_v k_v^2 / W) / W."""
    for seed in range(3):
        g, _ = _components_graph(seed)
        n = g.shape[0]
        for fn in (_ops.leiden, _ops.louvain):
            m, q, _ = fn(g, resolution=1e6, seed=seed)
            np.testing.assert_array_equal(m, np.arange(n))
            assert _close(q, old.modularity_fp64(_device_graph(g), m, resolution=1e6)), fn.__name__
            assert _close(q, old.modularity_fp64(g, m, resolution=1e6), 1e-6)


# ------------------------------------------------------------------------------------------ ring of cliques
# Merging two adjacent cliques gains iff eps > gamma K_c^2 / W = gamma (s(s-1) + 2 eps) / r, so the clique partition is
# gamma-separated whenever eps < gamma s(s-1) / r; splitting a clique always loses.
@pytest.mark.parametrize("r,s,eps", [
    (30, 8, 1.0),         # 240 vertices: four starts, 8 vertex classes (s(s-1)/r = 1.87, margin 1.87x)
    (12000, 10, 1e-3),    # 120,000 vertices: one start, first-pass and refinement cut-offs active (7.5e-3, margin 7.5x)
])
def test_ring_of_cliques_is_found_exactly(r, s, eps):
    assert eps < s * (s - 1) / r / 1.8
    g = _ring_of_cliques(r, s, eps)
    want = np.repeat(np.arange(r), s)
    m, q, _ = _ops.leiden(g, seed=0)
    np.testing.assert_array_equal(m, want)
    assert _close(q, old.modularity_fp64(_device_graph(g), want))
    assert _close(q, old.modularity_fp64(g, want))


# ------------------------------------------------------------------------------------------ guarantees on general graphs
@pytest.mark.parametrize("kind", ["knn", "hubs", "loops", "wide"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_guarantees_on_general_graphs(kind, seed):
    """Converged Leiden (n_iterations=-1): connected, gamma-separated, node-optimal.  Louvain: gamma-separated (it may leave
    communities disconnected and is not node-optimal at level 0).  Two Leiden iterations: connected.  Q = the fp64 formula."""
    gamma = (1.0, 0.5, 2.0)[seed]
    g = _general_graph(kind, seed)
    if kind == "hubs":
        assert (np.diff(g.indptr)[-16:] >= 2000).all()
    gd = _device_graph(g)
    m, q, _ = _ops.leiden(g, resolution=gamma, seed=seed)
    old.check_guarantees(gd, m, gamma)
    assert _close(q, old.modularity_fp64(gd, m, resolution=gamma))
    assert _close(q, old.modularity_fp64(g, m, resolution=gamma), 1e-6)
    ml, ql, _ = _ops.louvain(g, resolution=gamma, seed=seed)
    old.check_guarantees(gd, ml, gamma, connected=False, node_optimal=False)
    assert _close(ql, old.modularity_fp64(gd, ml, resolution=gamma))
    m2, q2, info = _ops.leiden(g, resolution=gamma, n_iterations=2, seed=seed)
    assert info["passes"] == 2
    old.check_guarantees(gd, m2, gamma, separated=False, node_optimal=False)
    assert _close(q2, old.modularity_fp64(gd, m2, resolution=gamma))


# ------------------------------------------------------------------------------------------ modularity kernel
@pytest.mark.parametrize("gamma", [0.3, 1.0, 2.5])
def test_modularity_kernel_matches_fp64(gamma):
    """sb2_modularity_csr_f32 on graphs with self-loops, isolated vertices and weights over 1e-6 .. 1e3, for random labels
    with gaps in the ids."""
    rs = np.random.RandomState(int(gamma * 10))
    for g in (_with_loops(_knn_graph(0), 1), _wide_weights(_with_loops(_knn_graph(1), 2), 3)):
        n = g.shape[0]
        keep = rs.rand(n) > 0.02                       # ~2 % isolated vertices
        g = (sparse.diags(keep.astype(np.float32)) @ g @ sparse.diags(keep.astype(np.float32))).tocsr()
        g.eliminate_zeros()
        assert (np.diff(g.indptr) == 0).any() and g.diagonal().any()
        gd = _device_graph(g)
        for n_lab in (2, 17, 400):
            lab = rs.choice(rs.choice(n, n_lab, replace=False), n)   # n_lab ids anywhere in [0, n)
            q = _ops.modularity(g, lab, resolution=gamma)
            assert _close(q, old.modularity_fp64(gd, lab, resolution=gamma)), (n_lab, q)
            assert _close(q, old.modularity_fp64(g, lab, resolution=gamma), 1e-6)


# ------------------------------------------------------------------------------------------ scale invariance
def _scaled(g, f):
    h = g.copy()
    h.data = (h.data.astype(np.float64) * f).astype(np.float32)
    return h


@pytest.mark.parametrize("k", [-60, -30, 30, 60])
def test_power_of_two_scale_gives_identical_results(k):
    """Q and the RB objective do not depend on the units of the weights; with a power-of-two fixed-point scale the device
    sees bit-identical integers, so labels and Q must be identical."""
    for g in (_ring_of_cliques(30, 8, 1.0), _knn_graph(0)):
        h = _scaled(g, 2.0 ** k)
        assert (h.data.astype(np.float64) == g.data.astype(np.float64) * 2.0 ** k).all()   # exact in float32
        m, q, _ = _ops.leiden(g, seed=0)
        mh, qh, _ = _ops.leiden(h, seed=0)
        np.testing.assert_array_equal(mh, m)
        assert qh == q
        ml, ql, _ = _ops.louvain(g, seed=0)
        mlh, qlh, _ = _ops.louvain(h, seed=0)
        np.testing.assert_array_equal(mlh, ml)
        assert qlh == ql
        assert sb.metrics.modularity(h, m, is_directed=False) == sb.metrics.modularity(g, m, is_directed=False)


@pytest.mark.parametrize("f", [1e-7, 3e5])
def test_other_scales_give_the_same_clustering(f):
    r, s = 30, 8
    m, _, _ = _ops.leiden(_scaled(_ring_of_cliques(r, s, 1.0), f), seed=0)
    np.testing.assert_array_equal(m, np.repeat(np.arange(r), s))
    g = _knn_graph(0)
    m0, q0, _ = _ops.leiden(g, seed=0)
    m1, q1, _ = _ops.leiden(_scaled(g, f), seed=0)
    assert adjusted_rand_score(m0, m1) >= 0.99
    assert abs(q1 - q0) <= 1e-6


# ------------------------------------------------------------------------------------------ explicit zeros
def test_explicit_zeros_are_not_edges():
    """The reference's graph holds the stored NONZERO entries only.  Symmetric stored zeros between communities must
    change nothing: tl.leiden with and without weights, tl.louvain with its defaults (unweighted), metrics.modularity."""
    g = _knn_graph(0)
    n = g.shape[0]
    m, _, _ = _ops.leiden(g, seed=0)
    rs = np.random.RandomState(0)
    i, j = rs.randint(0, n, 20000), rs.randint(0, n, 20000)
    ok = (m[i] != m[j]) & (np.asarray(g[i, j]).ravel() == 0)
    a, b = np.unique(np.stack([np.minimum(i, j), np.maximum(i, j)])[:, ok], axis=1)
    coo = g.tocoo()   # (sparse + sparse would drop the zeros: build the union of the stored entries directly)
    g0 = sparse.csr_matrix((np.r_[coo.data, np.zeros(2 * a.size, np.float32)],
                            (np.r_[coo.row, a, b], np.r_[coo.col, b, a])), shape=g.shape)
    g0.sort_indices()
    pairs = np.stack([a, b])
    assert g0.nnz == g.nnz + 2 * pairs.shape[1] and pairs.shape[1] > 1000 and (g0 != g).nnz == 0
    outs = []
    for adj in (g, g0):
        ad = _adata(n)
        sb.tl.leiden(ad, adjacency=adj, flavor="igraph", key_added="w")
        sb.tl.leiden(ad, adjacency=adj, flavor="igraph", use_weights=False, key_added="u")
        sb.tl.louvain(ad, adjacency=adj)
        lab = ad.obs["w"].cat.codes.to_numpy()
        outs.append(dict(w=lab, qw=ad.uns["w"]["modularity"], u=ad.obs["u"].cat.codes.to_numpy(), qu=ad.uns["u"]["modularity"],
                         lv=ad.obs["louvain"].cat.codes.to_numpy(), q=sb.metrics.modularity(adj, lab, is_directed=False)))
    a, b = outs
    for key in ("w", "u", "lv"):
        np.testing.assert_array_equal(b[key], a[key], err_msg=key)
    assert b["qw"] == a["qw"] and b["qu"] == a["qu"] and b["q"] == a["q"]


# ------------------------------------------------------------------------------------------ bad input
@pytest.mark.parametrize("bad", [np.nan, np.inf, -0.25])
def test_bad_weights_are_rejected(bad):
    g = _knn_graph(0)
    n = g.shape[0]
    h = g.copy()
    v = h.indices[h.indptr[5]]
    h[5, v] = bad
    h[v, 5] = bad
    lab = np.zeros(n, np.int64)
    with pytest.raises(B200Error, match="non-negative"):
        sb.tl.leiden(_adata(n), adjacency=h, flavor="igraph")
    with pytest.raises(B200Error, match="non-negative"):
        sb.tl.louvain(_adata(n), adjacency=h, use_weights=True)
    with pytest.raises(B200Error, match="non-negative"):
        sb.metrics.modularity(h, lab, is_directed=False)
    m, q, _ = _ops.leiden(g, seed=0)   # the context is still usable
    assert _close(q, old.modularity_fp64(_device_graph(g), m))


def test_unused_categories_do_not_change_modularity():
    """A categorical with more categories than cells (as on a subset of a larger object), most of them unused."""
    g = _knn_graph(0)
    n = g.shape[0]
    m, q, _ = _ops.leiden(g, seed=0)
    cats = [f"c{i}" for i in range(n + 500)]
    ids = np.linspace(3, len(cats) - 1, m.max() + 1).astype(np.int64)   # the communities' codes, far apart, some >= n
    spread = ids[m]
    assert spread.max() >= n and len(np.unique(ids)) == m.max() + 1
    labels = pd.Categorical.from_codes(spread, categories=cats)
    q_cat = sb.metrics.modularity(g, labels, is_directed=False)
    assert q_cat == sb.metrics.modularity(g, m, is_directed=False)
    assert _close(q_cat, q)
    assert sb.metrics.modularity(g, pd.Series(labels), is_directed=False) == q_cat

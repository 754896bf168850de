"""The thick-restart Lanczos solver (sb2_eigsh_csr_scaled, csrc/eigs.cu) against dense float64 `numpy.linalg.eigh` of the
same operator diag(s) A diag(s), on the spectra where single-vector Lanczos goes wrong: repeated extreme eigenvalues
(one copy of eigenvalue 1 per connected component), exact pairs (a cycle), an eigenvalue -1 under `LM` (an even cycle),
and nev close to n, where the basis size m = min(max(2 nev + 16, 40), 128, n - 1) is clipped.  Then tl.diffmap on a
disconnected graph, and the UMAP spectral initialisation (sb2_umap_spectral_init_f32) on a connected one.
Each case prints its eigenvalue and residual errors."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse.csgraph import connected_components

from oracle import umap_schedule as us

pytestmark = pytest.mark.gpu


def _knn_graph(n, n_comp, seed=0, k=10, dim=6):
    """Symmetric fp32 kNN graph of n_comp far-apart Gaussian blobs: exactly n_comp connected components."""
    from sklearn.neighbors import NearestNeighbors

    rng = np.random.default_rng(seed)
    lab = np.arange(n) % n_comp
    x = rng.normal(size=(n, dim)) + 1000.0 * np.eye(n_comp, dim)[lab] if n_comp > 1 else rng.normal(size=(n, dim))
    dist, idx = NearestNeighbors(n_neighbors=k + 1).fit(x).kneighbors(x)
    g = sparse.csr_matrix((np.exp(-dist[:, 1:].ravel() / np.median(dist[:, 1:])), (np.repeat(np.arange(n), k),
                                                                                      idx[:, 1:].ravel())), shape=(n, n))
    g = g.maximum(g.T).tocsr().astype(np.float32)
    g.sort_indices()
    assert connected_components(g)[0] == n_comp
    return g


def _cycle(n):
    i = np.arange(n)
    g = sparse.csr_matrix((np.ones(2 * n, np.float32), (np.r_[i, i], np.r_[(i + 1) % n, (i - 1) % n])), shape=(n, n))
    g.sort_indices()
    return g


GRAPHS = {
    "knn connected": lambda: _knn_graph(1500, 1),
    "knn 2 components": lambda: _knn_graph(1500, 2),
    "knn 3 components": lambda: _knn_graph(1500, 3),
    "knn 5 components": lambda: _knn_graph(2000, 5),
    "cycle 200": lambda: _cycle(200),
    "cycle 30": lambda: _cycle(30),
    "knn 70": lambda: _knn_graph(70, 1, k=8),
    "knn + even cycle": lambda: sparse.block_diag([_knn_graph(1000, 1), _cycle(40)], format="csr").astype(np.float32),
}


@pytest.fixture(scope="module")
def graphs():
    return {}


def _graph(graphs, name):
    if name not in graphs:
        graphs[name] = GRAPHS[name]()
    return graphs[name]


def _scale(ctx, g, dev, kind):
    from scanpy_b200 import _graph_tools, _ops

    if kind == "unscaled":
        return None, np.ones(g.shape[0])
    if kind == "transition":  # diffmap's T_sym, scale from the device like tl.diffmap
        d_s = _graph_tools._transition_scale_device(ctx, *dev, g.shape[0])
        return d_s, _ops._to_host(d_s)
    deg = np.asarray(g.astype(np.float64).sum(axis=1)).ravel()  # D^-1/2 A D^-1/2
    s = 1.0 / np.sqrt(deg)
    return _ops._to_device(s), s


def _wanted(w, nev, which):
    """Indices (into the ascending spectrum w) of the nev extreme eigenvalues; the boundary must not split a tie."""
    key = {"LA": w, "SA": -w, "LM": np.abs(w)}[which]
    order = np.argsort(-key, kind="stable")
    if nev < len(w):
        assert key[order[nev - 1]] - key[order[nev]] > 1e-9, "ambiguous wanted set"
    return order[:nev]


def _clusters(w, tol=1e-6):
    """Groups of the ascending spectrum closer than tol, as (lo, hi) index ranges, with each group's gap to the rest."""
    cuts = np.flatnonzero(np.diff(w) > tol) + 1
    edges = np.r_[0, cuts, len(w)]
    out = []
    for lo, hi in zip(edges[:-1], edges[1:]):
        gap = min(w[lo] - w[lo - 1] if lo > 0 else np.inf, w[hi] - w[hi - 1] if hi < len(w) else np.inf)
        out.append((lo, hi, gap))
    return out


def check_eigsh(name, g, kind, nev, which, **kw):
    from scanpy_b200 import _abi, _ops

    ctx = _abi.default_context()
    dev = _ops.csr_to_device(g)
    d_s, s = _scale(ctx, g, dev, kind)
    n = g.shape[0]
    ev, vecs, info = _ops.eigsh_scaled_device(ctx, *dev, n, nev, d_scale=d_s, which=which, **kw)
    V = _ops._to_host(vecs).T  # n x nev
    M = (sparse.diags(s) @ g.astype(np.float64) @ sparse.diags(s)).toarray()
    w, Q = np.linalg.eigh(M)
    want = np.sort(_wanted(w, nev, which))
    if which == "LM":
        ev_err = np.abs(np.sort(np.abs(ev)) - np.sort(np.abs(w[want]))).max()
    else:
        ev_err = np.abs(ev - w[want]).max()
    R = M @ V - V * ev
    res = np.linalg.norm(R, axis=0)
    orth = np.abs(V.T @ V - np.eye(nev)).max()
    # span: returned vectors of each eigenvalue cluster lie in its true eigenspace, with the cluster's multiplicity when
    # the whole cluster is wanted (Davis-Kahan: sin theta <= |R|_F / gap)
    span_err = 0.0
    for lo, hi, gap in _clusters(w):
        got = np.flatnonzero((ev >= w[lo] - 1e-7) & (ev <= w[hi - 1] + 1e-7))
        if np.isin(np.arange(lo, hi), want).all():
            assert len(got) == hi - lo, (name, "multiplicity", w[lo], hi - lo, len(got))
        if len(got) == 0 or gap <= 1e-6:
            continue
        Vg = V[:, got]
        sin = np.linalg.norm(Vg - Q[:, lo:hi] @ (Q[:, lo:hi].T @ Vg), 2)
        span_err = max(span_err, sin)
        assert sin <= 2 * np.linalg.norm(R[:, got]) / gap + 1e-10, (name, w[lo], sin, gap)
    mult = np.diff(np.r_[0, np.flatnonzero(np.diff(w[want]) > 1e-6) + 1, nev])
    print(f"{name} [{kind}, {which}, nev={nev}, n={n}]: |eval err| {ev_err:.2e}, max residual {res.max():.2e}, "
          f"orthonormality {orth:.2e}, span {span_err:.2e}, wanted multiplicities {mult.max()}, "
          f"reported residual {info['max_residual']:.2e}, n_converged {info['n_converged']}, restarts {info['restarts']}, matvecs {info['matvecs']}")
    assert ev_err <= 1e-9, (name, ev, w[want])
    assert res.max() <= 1e-8
    assert orth <= 1e-10
    # the reported residual is the returned pairs' own (their estimate in the cycle that locked them), not 0
    assert res.max() <= 10 * info["max_residual"] + 1e-12, (res.max(), info["max_residual"])
    # a report of convergence is a promise about the wanted set, not only about residuals
    assert info["n_converged"] == nev
    return ev, V, info


CASES = [
    ("knn connected", "transition", "LM", 1),
    ("knn connected", "transition", "LM", 3),
    ("knn connected", "transition", "LM", 15),
    ("knn connected", "transition", "LM", 64),
    ("knn connected", "unscaled", "LA", 3),
    ("knn connected", "unscaled", "SA", 15),
    ("knn connected", "invsqrt", "LA", 15),
    ("knn 2 components", "transition", "LM", 15),
    ("knn 3 components", "transition", "LM", 3),
    ("knn 3 components", "transition", "LM", 15),
    ("knn 3 components", "invsqrt", "LA", 3),
    ("knn 5 components", "transition", "LM", 15),
    ("knn 5 components", "transition", "LA", 64),
    ("cycle 200", "unscaled", "LA", 3),
    ("cycle 200", "unscaled", "LA", 15),
    ("cycle 200", "unscaled", "SA", 3),
    ("cycle 200", "transition", "LM", 14),  # 15 would split the four of +-cos(2 pi k / 200)
    ("cycle 30", "unscaled", "LA", 15),
    ("knn 70", "transition", "LM", 64),
    ("knn + even cycle", "transition", "LM", 3),
    ("knn + even cycle", "transition", "LM", 7),
    ("knn + even cycle", "invsqrt", "SA", 3),
]


@pytest.mark.parametrize("graph, kind, which, nev", CASES, ids=lambda v: str(v).replace(" ", "_"))
def test_eigsh_against_dense_truth(graphs, graph, kind, which, nev):
    check_eigsh(graph, _graph(graphs, graph), kind, nev, which)


def test_diffmap_on_a_disconnected_graph():
    """tl.diffmap on a 3-component neighbours graph: eigenvalue 1 three times, as dense eigh and scipy's eigsh find."""
    import scanpy_b200 as sb
    from oracle import graph_tools as og

    rng = np.random.default_rng(5)
    x = np.concatenate([rng.normal(size=(500, 8)) + 1000.0 * c for c in range(3)]).astype(np.float32)
    ad = sb.MiniAnnData(x)
    sb.pp.neighbors(ad, n_neighbors=15, use_rep="X")
    conn = ad.obsp["connectivities"]
    assert connected_components(conn)[0] == 3
    sb.tl.diffmap(ad, n_comps=15)
    evals, basis = ad.uns["diffmap_evals"], ad.obsm["X_diffmap"]
    truth = np.linalg.eigh(og.transitions_sym(conn.astype(np.float64)).toarray())[0]
    top = truth[np.argsort(-np.abs(truth))[:15]]
    top = top[np.argsort(-top)]
    np.testing.assert_array_equal(evals[:3], np.float32(1.0))
    np.testing.assert_allclose(evals, top, atol=2e-6)
    ref_evals, _ = og.diffmap_eigen(conn, 15, seed=0)
    np.testing.assert_allclose(evals, ref_evals, atol=2e-6)
    np.testing.assert_allclose(np.linalg.norm(basis.astype(np.float64), axis=0), 1.0, atol=1e-5)
    # the three eigenvectors of eigenvalue 1 span the component indicators scaled by z, T_sym = Z^-1 (Q^-1 W Q^-1) Z^-1
    # with z^2 the row sums of the density-normalised Q^-1 W Q^-1 (transitions_sym)
    w = conn.astype(np.float64).tocsr()
    q = np.asarray(w.sum(axis=0)).ravel()
    z = np.sqrt(np.asarray(w.multiply(1 / q[:, None]).multiply(1 / q[None, :]).sum(axis=0)).ravel())
    lab = connected_components(conn)[1]
    ind = np.stack([z * (lab == c) for c in range(3)], axis=1)
    ind /= np.linalg.norm(ind, axis=0)
    top3 = basis[:, :3].astype(np.float64)
    sin = np.linalg.norm(top3 - ind @ (ind.T @ top3), 2)
    assert sin < 1e-5, sin  # float32 storage of the basis: about 1e-7 per entry
    print(f"diffmap 3 components: evals {evals[:5]}, max |eval - dense| {np.abs(evals - top).max():.2e}, "
          f"eigenspace of 1 vs density-scaled indicators: sin {sin:.2e}")


@pytest.mark.parametrize("dim", [1, 2, 3, 8, 16])
def test_umap_spectral_init(graphs, dim):
    """sb2_umap_spectral_init_f32: eigenvectors 2..dim+1 of D^-1/2 A D^-1/2, expanded to max|x| = 10, plus N(0, 1e-4)."""
    import torch

    from scanpy_b200 import _abi, _ops
    from scanpy_b200._ops import check, ptr

    g = _graph(graphs, "knn connected")
    n = g.shape[0]
    ctx = _abi.default_context()
    dp, di, dw = _ops.csr_to_device(g)
    x = torch.empty((n, dim), dtype=torch.float32, device="cuda")
    check(ctx.lib.sb2_umap_spectral_init_f32(ctx.handle, n, ptr(dp), ptr(di), ptr(dw), dim, 11, ptr(x)))
    x = _ops._to_host(x).astype(np.float64)
    # the same solve as the initialisation's (nev = dim + 1, largest, ncv = max(2 nev + 16, 40), tol 1e-5, 60 restarts,
    # its start vector): the unjittered columns, so the jitter can be isolated exactly
    nev = dim + 1
    deg = np.asarray(g.astype(np.float64).sum(axis=1)).ravel()
    s = 1.0 / np.sqrt(deg)
    ev, vecs, _ = _ops.eigsh_scaled_device(ctx, dp, di, dw, n, nev, d_scale=_ops._to_device(s), which="LA",
                                          v0=us.umap_v0(n), ncv=max(2 * nev + 16, 40), tol=1e-5, max_restarts=60)
    pick = _ops._to_host(vecs)[::-1][1:].T.astype(np.float32)  # column c = eigenvector nev-2-c
    expand = np.float32(10.0) / np.abs(pick).max()
    jitter = x - pick.astype(np.float64) * expand
    assert abs(np.abs(x).max() - 10.0) <= 6e-4
    assert 0.9e-4 < jitter.std() < 1.1e-4 and abs(jitter.mean()) < 1e-5, (jitter.std(), jitter.mean())
    # against dense truth: the columns, expansion undone, lie in the span of eigenvectors 2..dim+1
    w, Q = np.linalg.eigh((sparse.diags(s) @ g.astype(np.float64) @ sparse.diags(s)).toarray())
    S = Q[:, n - 1 - dim:n - 1]
    y = x / float(expand)
    jit = 2e-4 * np.sqrt(n) / float(expand)  # the jitter's share, expansion undone (2 x its expected norm)
    gap = min(w[n - 1] - w[n - 2], w[n - 1 - dim] - w[n - 2 - dim])
    sin_span = np.linalg.norm(y - S @ (S.T @ y), axis=0) / np.linalg.norm(y, axis=0)
    # tol 1e-5 alone would allow 1e-5 / gap (about 3e-3 here); the solve converges well past it, to about 1e-4
    bound = min(2 * 1e-5 / gap + jit, 2e-4)
    print(f"spectral init dim={dim}: max|x| {np.abs(x).max():.6f}, jitter std {jitter.std():.3e}, span sin "
          f"{sin_span.max():.2e} (bound {bound:.2e}, gap {gap:.2e})")
    assert sin_span.max() <= bound
    # each column is its eigenvector up to sign where the eigenvalue is isolated
    for c in range(dim):
        i = n - 2 - c
        gap_c = min(w[i + 1] - w[i], w[i] - w[i - 1])
        if gap_c < 1e-3:
            continue
        cos = abs(y[:, c] @ Q[:, i]) / np.linalg.norm(y[:, c])
        assert np.sqrt(max(0.0, 1 - cos**2)) <= 2 * 1e-5 / gap_c + jit, (dim, c, cos, gap_c)

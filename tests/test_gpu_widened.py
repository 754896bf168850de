"""GPU tests of the widened rows (SURVEY.md 8f): pp.scale, tl.louvain, metrics.modularity, tl.umap, tl.diffmap, tl.paga,
chunked PCA.  Same rule as test_gpu_parity.py: every product call goes through the C ABI, the oracle is the checker."""
import warnings

import numpy as np
import pandas as pd
import pytest
from scipy import sparse
from sklearn.metrics import adjusted_rand_score

import scanpy_b200 as sb
from oracle import leiden as old, preprocess as opre
from scanpy_b200._synth import synth_scipy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scaling_literals():
    from conftest import GOLDEN

    return np.load(GOLDEN / "reference_scaling_literals.npz")


@pytest.fixture(scope="module")
def graph_small():
    x, lab = synth_scipy(5000, 600, n_clusters=10, r=40)
    ad = sb.MiniAnnData(x)
    sb.pp.pca(ad, n_comps=30)
    sb.pp.neighbors(ad, n_neighbors=15)
    return ad, lab


# ------------------------------------------------------------------------------------------ pp.scale
@pytest.mark.parametrize("typ", [np.array, sparse.csr_matrix, sparse.csc_matrix], ids=lambda t: t.__name__)
@pytest.mark.parametrize("container", ["anndata", "array"])
@pytest.mark.parametrize("dtype", [np.float32, np.int64])
@pytest.mark.parametrize("zero_center", [True, False], ids=["center", "no_center"])
@pytest.mark.parametrize("masked", [False, True], ids=["no_mask", "mask"])
def test_scale_reference_goldens(scaling_literals, typ, container, dtype, zero_center, masked):
    # the reference's own matrix: tests/test_scaling.py:72-116
    L = scaling_literals
    x0 = L["X_for_mask"] if masked else L["X_original"]
    mask = np.array((0, 0, 1, 1, 1, 0, 0), dtype=bool) if masked else None
    expected = (L["X_centered_for_mask"] if zero_center else L["X_scaled_for_mask"]) if masked else (
        L["X_centered_original"] if zero_center else L["X_scaled_original"])
    x = typ(x0.astype(dtype))
    data = sb.MiniAnnData(x) if container == "anndata" else x
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = sb.pp.scale(data, zero_center=zero_center, copy=container == "array", mask_obs=mask)
    got = data.X if out is None else out
    got = got.toarray() if sparse.issparse(got) else np.asarray(got)
    assert np.allclose(got, expected)


def test_scale_clip_goldens_and_mask_string(scaling_literals):
    L = scaling_literals
    # tests/test_scaling.py:146-175 (clipped goldens) and :119-126 (string mask)
    out = sb.pp.scale(sparse.csr_matrix(L["X_original"].astype(np.float32)), zero_center=False, max_value=1)
    assert np.allclose(out.toarray(), L["X_scaled_original_clipped"])
    out = sb.pp.scale(L["X_for_mask"].astype(np.float32), zero_center=False, max_value=1,
                      mask_obs=np.array((0, 0, 1, 1, 1, 0, 0), dtype=bool))
    assert np.allclose(out, L["X_scaled_for_mask_clipped"])
    with pytest.raises(ValueError, match=r"Cannot.*refer.*mask.*without.*anndata"):
        sb.pp.scale(L["X_original"], mask_obs="mask")
    ad = sb.MiniAnnData(L["X_for_mask"].astype(np.float32))
    ad.obs["some cells"] = np.array((0, 0, 1, 1, 1, 0, 0), dtype=bool)
    sb.pp.scale(ad, mask_obs="some cells")
    assert np.array_equal(ad.X, L["X_centered_for_mask"])
    assert "mean of some cells" in ad.var.columns


@pytest.mark.parametrize("zero_center", [True, False])
@pytest.mark.parametrize("max_value", [None, 2.5])
def test_scale_matches_oracle_on_synthetic(zero_center, max_value):
    x, _ = synth_scipy(3000, 500, n_clusters=6, r=32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = sb.pp.scale(x, zero_center=zero_center, max_value=max_value, copy=True)
    ref, mean, std = opre.scale(x, zero_center=zero_center, max_value=max_value)
    if zero_center:
        assert got.dtype == np.float64 and not sparse.issparse(got)
        np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9)
        if max_value is not None:
            assert got.min() >= -max_value and got.max() <= max_value
    else:
        assert sparse.issparse(got) and got.dtype == np.float32
        assert (got.indices == x.indices).all()
        np.testing.assert_allclose(got.data, ref.data, rtol=2e-7)
    # dense float32 input: in-place float32 semantics
    xd = x[:500].toarray()
    got_d = sb.pp.scale(xd, zero_center=zero_center, max_value=max_value, copy=True)
    ref_d, _, _ = opre.scale(xd, zero_center=zero_center, max_value=max_value)
    assert got_d.dtype == np.float32
    np.testing.assert_allclose(got_d, ref_d, rtol=2e-6, atol=2e-6)
    ad = sb.MiniAnnData(x.copy())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sb.pp.scale(ad, zero_center=zero_center, max_value=max_value)
    np.testing.assert_allclose(ad.var["mean"], mean, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(ad.var["std"], std, rtol=1e-9)


# ------------------------------------------------------------------------------------------ louvain / modularity
def test_louvain_vs_networkx_and_planted(graph_small):
    import networkx as nx

    ad, lab = graph_small
    ad = ad.copy()
    sb.tl.louvain(ad, use_weights=True)
    got = ad.obs["louvain"].to_numpy().astype(int)
    assert ad.uns["louvain"]["params"] == dict(resolution=None, random_state=0)
    conn = ad.obsp["connectivities"]
    q_got = sb.metrics.modularity(conn, got, is_directed=False)
    g = nx.from_scipy_sparse_array(conn)
    parts = nx.community.louvain_communities(g, weight="weight", resolution=1.0, seed=0)
    q_nx = nx.community.modularity(g, parts, weight="weight")
    ref = np.empty(conn.shape[0], int)
    for i, p in enumerate(parts):
        ref[list(p)] = i
    # quality floor: an independent Louvain implementation, and our own modularity kernel against networkx's
    assert abs(sb.metrics.modularity(conn, ref, is_directed=False) - q_nx) < 1e-6
    assert q_got > q_nx - 5e-3, (q_got, q_nx)
    assert adjusted_rand_score(lab, got) > 0.95
    # labels ordered by decreasing size like every scanpy clustering
    sizes = np.bincount(got)
    assert (np.diff(sizes) <= 0).all()
    # same seed -> same labels; restrict_to only relabels the chosen cluster (tests/test_clustering.py:177-213 pattern)
    ad2 = ad.copy()
    sb.tl.louvain(ad2, use_weights=True)
    assert (ad2.obs["louvain"].to_numpy() == ad.obs["louvain"].to_numpy()).all()
    sb.tl.louvain(ad, use_weights=True, restrict_to=("louvain", ["0"]), resolution=2.0)
    r = ad.obs["louvain_R"].astype(str).to_numpy()
    base = ad.obs["louvain"].astype(str).to_numpy()
    assert (r[base != "0"] == base[base != "0"]).all()
    assert all(v.startswith("0,") for v in r[base == "0"])
    with pytest.raises(ValueError, match="flavor"):
        sb.tl.louvain(ad, flavor="nope")


def test_louvain_unweighted_default_and_igraph_flavor(graph_small):
    ad, lab = graph_small
    ad = ad.copy()
    sb.tl.louvain(ad)  # use_weights=False default: every arc weighs 1
    a = ad.obs["louvain"].to_numpy().astype(int)
    assert adjusted_rand_score(lab, a) > 0.9
    with pytest.warns(UserWarning, match="no effect"):
        sb.tl.louvain(ad, flavor="igraph", resolution=3.0, key_added="lv_ig")
    b = ad.obs["lv_ig"].to_numpy().astype(int)
    assert adjusted_rand_score(a, b) > 0.9


def test_metrics_modularity_api(graph_small):
    # tests/test_metrics.py:311-344: in [0, 1] on a clustering, retrieve == calculate == update
    ad, _ = graph_small
    ad = ad.copy()
    sb.tl.leiden(ad, flavor="igraph")
    m_ret = sb.metrics.modularity(ad, mode="retrieve")
    m_calc = sb.metrics.modularity(ad, mode="calculate")
    assert 0 <= m_calc <= 1
    assert abs(m_ret - m_calc) < 1e-9
    ad.uns["leiden"]["modularity"] = -1.0
    assert sb.metrics.modularity(ad, mode="update") == pytest.approx(m_calc)
    assert ad.uns["leiden"]["modularity"] == pytest.approx(m_calc)
    conn = ad.obsp["connectivities"]
    labels = ad.obs["leiden"]
    m_arr = sb.metrics.modularity(conn, labels, is_directed=False)
    assert m_arr == pytest.approx(m_calc)
    assert m_arr == pytest.approx(old.modularity(conn, labels.cat.codes.to_numpy()), abs=1e-7)
    assert sb.metrics.modularity(conn.toarray(), pd.Series(labels.astype(str)), is_directed=False) == pytest.approx(m_calc)
    with pytest.raises(TypeError, match="labels"):
        sb.metrics.modularity(conn, "leiden", is_directed=False)
    with pytest.raises(TypeError, match="is_directed"):
        sb.metrics.modularity(conn, labels)
    with pytest.raises(ValueError, match="undirected"):
        sb.metrics.modularity(ad, is_directed=True)


# ------------------------------------------------------------------------------------------ tl.umap
@pytest.fixture(scope="module")
def overlap_graph():
    """Six overlapping Gaussian clusters in 10-D (connected kNN graph), UMAP connectivities from the device."""
    rng = np.random.default_rng(0)
    cent = rng.normal(size=(6, 10)) * 2.0
    x = np.concatenate([rng.normal(size=(400, 10)) + cent[c] for c in range(6)]).astype(np.float32)
    lab = np.repeat(np.arange(6), 400)
    ad = sb.MiniAnnData(x)
    sb.pp.neighbors(ad, n_neighbors=15, use_rep="X")
    return ad, x, lab


def test_umap_quality_matches_sequential_oracle(overlap_graph):
    from sklearn.manifold import trustworthiness
    from sklearn.metrics import silhouette_score

    from oracle import graph_tools as og

    ad, x, lab = overlap_graph
    ad = ad.copy()
    conn_before = ad.obsp["connectivities"].copy()
    sb.tl.umap(ad)
    emb = ad.obsm["X_umap"]
    assert emb.shape == (len(x), 2) and emb.dtype == np.float32 and np.isfinite(emb).all()
    # parameters recorded like the reference (a, b of find_ab_params(1.0, 0.5); random_state 0)
    p = ad.uns["umap"]["params"]
    assert p["a"] == pytest.approx(0.5830300, rel=1e-5) and p["b"] == pytest.approx(1.3341669, rel=1e-5)
    assert p["random_state"] == 0
    # tests/test_embedding.py:83-96: the graph is not touched, no explicit zeros
    conn = ad.obsp["connectivities"]
    assert (conn.data == conn_before.data).all() and conn.nnz == conn_before.nnz and (conn.data == 0).sum() == 0
    ref = og.simplicial_set_embedding(conn_before, a=p["a"], b=p["b"])
    t_got, t_ref = trustworthiness(x, emb, n_neighbors=15), trustworthiness(x, ref, n_neighbors=15)
    s_got, s_ref = silhouette_score(emb, lab), silhouette_score(ref, lab)
    assert t_got > t_ref - 0.02, (t_got, t_ref)
    assert s_got > s_ref - 0.1, (s_got, s_ref)
    # layout scale comparable with the sequential optimiser's (same forces, same schedule)
    assert 0.3 < emb.std() / ref.std() < 3.0


def test_umap_init_dtype_keys_and_seeds(overlap_graph):
    ad, x, _ = overlap_graph
    # tests/test_embedding.py:48-66: float32 / float64 initial positions give the same embedding; params recorded per key
    a1, a2 = ad.copy(), ad.copy()
    init = x[:, :2]
    sb.tl.umap(a1, init_pos=init.astype(np.float32), maxiter=100)
    sb.tl.umap(a2, init_pos=init.astype(np.float64), maxiter=100, key_added="custom_key")
    np.testing.assert_array_almost_equal(a1.obsm["X_umap"], a2.obsm["custom_key"])
    assert a1.uns["umap"]["params"]["a"] == a2.uns["custom_key"]["params"]["a"]
    assert a1.uns["umap"]["params"]["b"] == a2.uns["custom_key"]["params"]["b"]
    # an .obsm key as init_pos, 3 components, random init; same seed -> same layout, other seed -> another
    a1.obsm["my_init"] = np.ascontiguousarray(x[:, :3])
    sb.tl.umap(a1, init_pos="my_init", n_components=3, maxiter=50, key_added="u3")
    assert a1.obsm["u3"].shape == (len(x), 3)
    b1, b2, b3 = ad.copy(), ad.copy(), ad.copy()
    sb.tl.umap(b1, init_pos="random", maxiter=50, random_state=3)
    sb.tl.umap(b2, init_pos="random", maxiter=50, random_state=3)
    sb.tl.umap(b3, init_pos="random", maxiter=50, random_state=4)
    assert (b1.obsm["X_umap"] == b2.obsm["X_umap"]).all()
    assert not (b1.obsm["X_umap"] == b3.obsm["X_umap"]).all()
    with pytest.raises(ValueError, match="Run `sc.pp.neighbors` first"):
        sb.tl.umap(sb.MiniAnnData(x))
    with pytest.raises(ValueError, match="Unknown method"):
        sb.tl.umap(ad.copy(), method="nope")


# ------------------------------------------------------------------------------------------ tl.diffmap
def test_diffmap_matches_reference_eigsh(overlap_graph):
    from oracle import graph_tools as og

    ad, _, _ = overlap_graph
    ad = ad.copy()
    sb.tl.diffmap(ad, n_comps=15)
    evals = ad.uns["diffmap_evals"]
    basis = ad.obsm["X_diffmap"]
    ref_evals, ref_basis = og.diffmap_eigen(ad.obsp["connectivities"], 15, seed=0)
    assert evals.dtype == np.float32 and basis.dtype == np.float32 and basis.shape == (ad.n_obs, 15)
    assert (np.diff(evals) <= 1e-7).all()  # sort='decrease'
    np.testing.assert_allclose(evals, ref_evals, atol=2e-6)
    # eigenvectors up to sign where the eigenvalue is isolated; the spanned subspace everywhere
    gaps = np.minimum(np.abs(np.diff(ref_evals, prepend=np.inf)), np.abs(np.diff(ref_evals, append=-np.inf)))
    for c in np.flatnonzero(gaps > 1e-3):
        dot = abs(float(basis[:, c].astype(np.float64) @ ref_basis[:, c].astype(np.float64)))
        assert dot > 1 - 1e-4, (c, dot, gaps[c])
    q, _ = np.linalg.qr(ref_basis.astype(np.float64))
    resid = basis.astype(np.float64) - q @ (q.T @ basis.astype(np.float64))
    assert np.abs(resid).max() < 1e-3
    np.testing.assert_allclose(np.linalg.norm(basis.astype(np.float64), axis=0), 1.0, atol=1e-5)


def test_diffmap_seeds_and_keys(overlap_graph):
    # tests/test_embedding.py:99-139: same seed reproducible, other seed differs (bitwise), key_added layouts
    ad, _, _ = overlap_graph
    d1, d2, d3 = (sb.tl.diffmap(ad, copy=True, random_state=s).obsm["X_diffmap"].copy() for s in (0, 0, 1234))
    np.testing.assert_array_equal(d1, d2)
    assert not np.array_equal(d1, d3)
    a = sb.tl.diffmap(ad, key_added="custom_key", copy=True, n_comps=5)
    assert "custom_key" in a.obsm and isinstance(a.uns["custom_key"], dict) and len(a.uns["custom_key"]["evals"]) == 5
    with pytest.raises(ValueError, match="greater than 2"):
        sb.tl.diffmap(ad.copy(), n_comps=2)
    with pytest.raises(ValueError, match="pp.neighbors"):
        sb.tl.diffmap(sb.MiniAnnData(np.zeros((5, 3), np.float32)))


def test_eigsh_ends_of_the_spectrum(overlap_graph):
    """sb2_eigsh_csr_scaled against scipy's eigsh on the same operator: largest / smallest algebraic, unscaled."""
    from scipy.sparse.linalg import eigsh

    from scanpy_b200 import _abi, _ops

    ad, _, _ = overlap_graph
    conn = ad.obsp["connectivities"].tocsr().astype(np.float32)
    ctx = _abi.default_context()
    dp, di, dw = _ops.csr_to_device(conn)
    for which in ("LA", "SA"):
        ev, vecs, info = _ops.eigsh_scaled_device(ctx, dp, di, dw, conn.shape[0], 4, which=which)
        ref = eigsh(conn.astype(np.float64), k=4, which=which)[0]
        np.testing.assert_allclose(ev, np.sort(ref), rtol=1e-8, atol=1e-8)
        v = _ops._to_host(vecs)
        # residual |A v - lambda v| of every returned pair
        r = conn.astype(np.float64) @ v.T - v.T * ev
        assert np.abs(r).max() < 1e-6 and info["n_converged"] == 4


# ------------------------------------------------------------------------------------------ tl.paga
def test_paga_matches_oracle(graph_small):
    from oracle import graph_tools as og

    ad, _ = graph_small
    ad = ad.copy()
    sb.tl.leiden(ad, flavor="igraph")
    sb.tl.paga(ad)
    assert ad.uns["paga"]["groups"] == "leiden"
    codes = ad.obs["leiden"].cat.codes.to_numpy()
    conn, tree, ns = og.paga_v1_2(ad.obsp["distances"], codes)
    np.testing.assert_array_equal(ad.uns["leiden_sizes"], ns)
    np.testing.assert_allclose(ad.uns["paga"]["connectivities"].toarray(), conn.toarray(), rtol=1e-12)
    np.testing.assert_allclose(ad.uns["paga"]["connectivities_tree"].toarray(), tree.toarray(), rtol=1e-12)
    c = ad.uns["paga"]["connectivities"]
    assert abs(c - c.T).max() < 1e-12 and c.max() <= 1.0
    with pytest.raises(KeyError, match="not found"):
        sb.tl.paga(ad, groups="nope")
    with pytest.raises(ValueError, match="tl.leiden"):
        sb.tl.paga(graph_small[0].copy())


# ------------------------------------------------------------------------------------------ chunked / out-of-core PCA
def test_pca_chunked_equals_full():
    """tests/test_pca.py:357-386: chunked PCA == default PCA (rtol 1e-6 there on |X_pca|, |PCs|, variance, variance_ratio);
    plus the fp64 truth bar of the hot path (1e-4 relative per component)."""
    from oracle import pca as opca

    x, _ = synth_scipy(7000, 700, n_clusters=8, r=40)
    full, chunked = sb.MiniAnnData(x), sb.MiniAnnData(x)
    sb.pp.pca(full, n_comps=30, svd_solver="covariance_eigh")
    sb.pp.pca(chunked, n_comps=30, chunked=True, chunk_size=1111)  # 7 ragged chunks
    a, b = np.abs(full.obsm["X_pca"]), np.abs(chunked.obsm["X_pca"])
    scale = np.abs(full.obsm["X_pca"]).max(axis=0)
    assert (np.abs(a - b) / scale).max() < 2e-6
    np.testing.assert_allclose(np.abs(chunked.varm["PCs"]), np.abs(full.varm["PCs"]), atol=2e-6)
    np.testing.assert_allclose(chunked.uns["pca"]["variance"], full.uns["pca"]["variance"], rtol=1e-6)
    np.testing.assert_allclose(chunked.uns["pca"]["variance_ratio"], full.uns["pca"]["variance_ratio"], rtol=1e-6)
    ref = opca.pca_arpack(x.astype(np.float64), 30, dtype="float64")
    xp = opca.align_signs(chunked.obsm["X_pca"].astype(np.float64), ref["X_pca"])
    rel = np.linalg.norm(xp - ref["X_pca"], axis=0) / np.linalg.norm(ref["X_pca"], axis=0)
    assert rel.max() < 1e-4
    # one chunk larger than the matrix, and the plain-array entry point
    xp1 = sb.pp.pca(x, n_comps=10, chunked=True, chunk_size=10**6)
    np.testing.assert_allclose(np.abs(xp1), np.abs(full.obsm["X_pca"][:, :10]), atol=5e-5 * scale[:10].max())


def test_pca_chunked_from_an_on_disk_zarr_store(tmp_path):
    """f4: rows stream from a zarr-v3 CSR store (sharded + zstd, as anndata writes it) through the device; X never exists in
    host memory as a whole on the product side.  Result == the in-core PCA of the same matrix."""
    import zarr_writer

    x, _ = synth_scipy(5000, 600, n_clusters=6, r=40)
    zarr_writer.write_csr_store(tmp_path / "x.zarr", x, mode="sharded", chunk=65536, inner=8192)
    backed = sb.read_zarr_backed(tmp_path / "x.zarr")
    sb.pp.pca(backed, n_comps=20, chunked=True, chunk_size=777)
    full = sb.MiniAnnData(x)
    sb.pp.pca(full, n_comps=20, svd_solver="covariance_eigh")
    scale = np.abs(full.obsm["X_pca"]).max(axis=0)
    assert (np.abs(np.abs(backed.obsm["X_pca"]) - np.abs(full.obsm["X_pca"])) / scale).max() < 2e-6
    np.testing.assert_allclose(backed.uns["pca"]["variance"], full.uns["pca"]["variance"], rtol=1e-6)
    with pytest.raises(NotImplementedError, match="chunked=True"):
        sb.pp.pca(sb.read_zarr_backed(tmp_path / "x.zarr"), n_comps=5)


@pytest.mark.parametrize("solver", [None, "b200_spmm"])
def test_pca_zero_center_false_matches_truncated_svd(solver):
    """`zero_center=False` = sklearn TruncatedSVD (src/scanpy/preprocessing/_pca/__init__.py:309-336): X V, V^T with
    svd_flip signs, np.var-based explained variance; checked against the exact arpack solver in float64."""
    from oracle import pca as opca

    x, _ = synth_scipy(5000, 700, n_clusters=8, r=40)
    k = 20
    ref = opca.truncated_svd_arpack(x, k)
    ad = sb.MiniAnnData(x)
    sb.pp.pca(ad, n_comps=k, zero_center=False, svd_solver=solver)
    xp = opca.align_signs(ad.obsm["X_pca"].astype(np.float64), ref["X_pca"])
    rel = np.linalg.norm(xp - ref["X_pca"], axis=0) / np.linalg.norm(ref["X_pca"], axis=0)
    tol = 1e-4 if solver is None else 2e-3   # the SpMM route runs float32 passes (its noise floor / the spectral gap)
    assert rel.max() < tol, rel.max()
    assert ad.uns["pca"]["params"]["zero_center"] is False
    np.testing.assert_allclose(ad.uns["pca"]["variance"], ref["variance"], rtol=2e-4 if solver is None else 5e-3)
    np.testing.assert_allclose(ad.uns["pca"]["variance_ratio"], ref["variance_ratio"], rtol=2e-4 if solver is None else 5e-3)
    pcs = ad.varm["PCs"].T
    np.testing.assert_allclose(np.abs(pcs), np.abs(ref["components"]), atol=2e-4 if solver is None else 5e-3)
    # svd_flip(u_based_decision=False): the largest-|.| loading of every component is positive, as in the reference's output
    assert (pcs[np.arange(k), np.abs(pcs).argmax(axis=1)] > 0).all()
    # the first component is the mean direction: far from the centred PCA's
    sb.pp.pca(ad, n_comps=k, key_added="centred")
    assert abs(ad.obsm["centred"][:, 0].mean()) < 1e-3 < abs(ad.obsm["X_pca"][:, 0].mean())


def test_clustering_reproduces_the_reference_fixtures_stored_louvain(pbmc68k_graph):
    """The reference's own label-level golden (see tests/test_oracle_leiden_guarantees.py): `obs/louvain` of the in-tree
    pbmc68k_reduced fixture = scanpy's `sc.tl.louvain` defaults on the stored connectivities.  `sb.tl.louvain` with the same
    defaults (vtraag, unweighted), and `sb.tl.leiden(use_weights=False)`, must land on that partition as closely as
    independent CPU optimisers do (networkx Louvain 0.94-0.97, sequential oracle 0.94-0.98)."""
    f = pbmc68k_graph
    n = len(f["conn_indptr"]) - 1
    conn = sparse.csr_matrix((f["conn_data"].astype(np.float32), f["conn_indices"], f["conn_indptr"]), shape=(n, n))
    stored = f["louvain_codes"].astype(int)
    ad = sb.MiniAnnData(sparse.csr_matrix((n, 3), dtype=np.float32))
    ad.obsp["connectivities"] = conn
    ad.uns["neighbors"] = dict(connectivities_key="connectivities", distances_key="distances", params=dict(method="umap"))
    sb.tl.louvain(ad)
    lv = ad.obs["louvain"].to_numpy().astype(int)
    sb.tl.leiden(ad, use_weights=False, flavor="igraph")
    ld = ad.obs["leiden"].to_numpy().astype(int)
    a_lv, a_ld = adjusted_rand_score(stored, lv), adjusted_rand_score(stored, ld)
    print(f"\n[pbmc68k stored louvain] ARI device louvain {a_lv:.3f} ({lv.max() + 1} clusters), device leiden {a_ld:.3f} ({ld.max() + 1})")
    assert a_lv > 0.9 and a_ld > 0.9, (a_lv, a_ld)
    assert 10 <= lv.max() + 1 <= 12 and 10 <= ld.max() + 1 <= 12


def test_umap_quality_matches_the_reference_fixtures_stored_embedding(pbmc68k_graph):
    """Device `tl.umap` on the fixture's stored connectivities vs the embedding the reference itself stored there
    (`obsm/X_umap`; see tests/test_oracle_goldens.py for what can and cannot be compared)."""
    from sklearn.manifold import trustworthiness
    from sklearn.metrics import silhouette_score
    from sklearn.neighbors import NearestNeighbors

    f = pbmc68k_graph
    n = 700
    conn = sparse.csr_matrix((f["conn_data"].astype(np.float32), f["conn_indices"], f["conn_indptr"]), shape=(n, n))
    stored, lab, x30 = f["X_umap"], f["louvain_codes"].astype(int), f["X_pca"][:, :30]
    ad = sb.MiniAnnData(sparse.csr_matrix((n, 3), dtype=np.float32))
    ad.obsp["connectivities"] = conn
    ad.uns["neighbors"] = dict(connectivities_key="connectivities", distances_key="distances", params=dict(method="umap"))
    sb.tl.umap(ad)
    emb = ad.obsm["X_umap"]

    def nbrs(a, k=15):
        return NearestNeighbors(n_neighbors=k + 1).fit(a).kneighbors(a, return_distance=False)[:, 1:]

    ov = float(np.mean([len(set(p) & set(q)) / 15 for p, q in zip(nbrs(emb), nbrs(stored))]))
    t_got, t_ref = trustworthiness(x30, emb, n_neighbors=10), trustworthiness(x30, stored, n_neighbors=10)
    s_got, s_ref = silhouette_score(emb, lab), silhouette_score(stored, lab)
    print(f"\n[pbmc68k stored X_umap] trustworthiness {t_got:.4f} (stored {t_ref:.4f}), silhouette {s_got:.3f} ({s_ref:.3f}), "
          f"15-NN overlap with the stored embedding {ov:.3f} (sequential oracle: 0.64-0.65, oracle seed-vs-seed 0.675)")
    assert t_got > t_ref - 0.015 and s_got > s_ref - 0.08 and ov > 0.55

"""GPU parity tests (need an H100: `pytest -m gpu`).  Every product call goes through the C ABI
(ctypes -> libscanpy_b200.so); the oracle (tests-only) is the checker.

Bars (BASELINE.json north_star): X_pca within 1e-4 relative up to sign, identical kNN index sets,
Leiden ARI >= 0.99 (on unambiguous, planted partitions).
"""
import numpy as np
import pytest
from scipy import sparse
from sklearn.metrics import adjusted_rand_score

import scanpy_b200 as sb
from oracle import fuzzy as ofz, knn as oknn, leiden as old, pca as opca
from scanpy_b200 import _ops
from scanpy_b200._synth import synth_scipy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def synth_small():
    x, lab = synth_scipy(6000, 800, n_clusters=12, r=48)
    return x, lab


def _rel_err(a, b):
    a = opca.align_signs(np.asarray(a, np.float64), b)
    return np.linalg.norm(a - b, axis=0) / np.linalg.norm(b, axis=0)


# ------------------------------------------------------------------------------------------ PCA
@pytest.mark.parametrize("solver", ["arpack", "covariance_eigh", "b200_spmm"])
def test_pca_golden_A_pca(literals, solver):
    # reference golden: tests/test_pca.py:34-59,225-233 (norm(|A_pca[:, :4]| - |X_pca|) < 2e-5)
    a = sparse.csr_matrix(literals["A_list"].astype(np.float32))
    x_pca = sb.pp.pca(a, n_comps=4, svd_solver=solver)
    assert x_pca.dtype == np.float32
    assert np.linalg.norm(np.abs(literals["A_pca"][:, :4]) - np.abs(x_pca)) < 2e-5
    # dense input gives the same (tests/test_pca.py:62-80 array-type matrix)
    x_dense = sb.pp.pca(literals["A_list"].astype(np.float32), n_comps=4, svd_solver=solver)
    np.testing.assert_allclose(np.abs(x_dense), np.abs(x_pca), atol=2e-5)


@pytest.mark.parametrize("solver,tol", [(1, 1e-4), (0, 1e-4)])
def test_pca_matches_reference(synth_small, solver, tol):
    x, _ = synth_small
    k = 30
    out = _ops.pca_csr(x, k, solver=solver)
    ref32 = opca.pca_arpack(x, k)                                       # the reference call, float32 ARPACK
    ref64 = opca.pca_arpack(x.astype(np.float64), k, dtype="float64")   # same call in double = ground truth
    s = ref64["singular_values"]
    gap = np.r_[s[:-1] - s[1:], s[-1] * 1e-3] / s
    e64 = _rel_err(out["X_pca"], ref64["X_pca"])
    noise = _rel_err(ref32["X_pca"], ref64["X_pca"])  # the reference's own float32 noise per component
    # 1e-4 relative (up to sign) on every component against ground truth ...
    assert e64.max() < tol, (e64.max(), gap.min())
    # ... and against the float32 reference within its own noise
    e32 = _rel_err(out["X_pca"], ref32["X_pca"].astype(np.float64))
    assert (e32 < np.maximum(1e-4, 2.0 * noise + 1e-5)).all(), (e32.max(), noise.max())
    np.testing.assert_allclose(out["variance"], ref64["variance"], rtol=1e-5)
    np.testing.assert_allclose(out["variance_ratio"], ref64["variance_ratio"], rtol=1e-5)
    np.testing.assert_allclose(out["mean"], ref64["mean"], rtol=1e-6, atol=1e-9)
    # sign convention svd_flip(u_based_decision=False): max-|.| entry of each component positive
    comp = out["components"]
    assert (comp[np.arange(k), np.abs(comp).argmax(axis=1)] > 0).all()
    np.testing.assert_allclose(np.abs(comp), np.abs(ref64["components"]), atol=2e-4)
    # components orthonormal, X_pca columns uncorrelated (tests/test_pca.py style invariants)
    np.testing.assert_allclose(comp @ comp.T, np.eye(k), atol=1e-5)


@pytest.mark.parametrize("solver", [1, 0])
def test_pca_wide_block_matches_fp64(solver):
    # n_comps between 57 and 120 iterates a 128-wide block, whose Rayleigh-Ritz step is solved on the host; a latent
    # dimension well above n_comps keeps the spectrum gapped past the cut
    x, _ = synth_scipy(6000, 800, n_clusters=12, r=160)
    k = 80
    out = _ops.pca_csr(x, k, solver=solver)
    truth = opca.pca_gram_f64(x, k)
    assert out["converged"]
    e64 = _rel_err(out["X_pca"], truth["X_pca"])
    assert e64.max() < 1e-4, (e64.max(), truth["gaps"].min())
    np.testing.assert_allclose(out["variance"], truth["variance"], rtol=1e-5)
    np.testing.assert_allclose(out["variance_ratio"], truth["variance_ratio"], rtol=1e-5)
    # svd_flip(u_based_decision=False) signs: the components match the fp64 truth as they are, not only up to sign
    comp = out["components"]
    assert (comp[np.arange(k), np.abs(comp).argmax(axis=1)] > 0).all()
    np.testing.assert_allclose(comp, truth["components"], atol=2e-4)


def test_pca_anndata_writeback_and_mask(synth_small):
    x, _ = synth_small
    x = x[:1500]
    ad = sb.MiniAnnData(x)
    rs = np.random.RandomState(1)
    mask = rs.rand(x.shape[1]) < 0.6
    ad.var["highly_variable"] = mask
    sb.pp.pca(ad, n_comps=10)  # mask_var defaults to var['highly_variable'] (_pca/__init__.py:221-232)
    assert ad.obsm["X_pca"].shape == (1500, 10) and ad.obsm["X_pca"].dtype == np.float32
    assert ad.varm["PCs"].shape == (x.shape[1], 10)
    assert (ad.varm["PCs"][~mask] == 0).all() and np.abs(ad.varm["PCs"][mask]).sum() > 0
    assert ad.uns["pca"]["params"] == dict(zero_center=True, mask_var="highly_variable")
    assert ad.uns["pca"]["variance"].shape == (10,) and ad.uns["pca"]["variance_ratio"].shape == (10,)
    # mask == explicit subset (tests/test_pca.py:461-506)
    sub = sb.pp.pca(x[:, mask], n_comps=10)
    np.testing.assert_allclose(np.abs(sub), np.abs(ad.obsm["X_pca"]), atol=2e-4)
    # same seed -> identical, copy=True leaves the input untouched (tests/test_pca.py:333-354)
    ad2 = sb.pp.pca(sb.MiniAnnData(x), n_comps=10, copy=True)
    ad3 = sb.pp.pca(sb.MiniAnnData(x), n_comps=10, copy=True, random_state=0)
    np.testing.assert_array_equal(ad2.obsm["X_pca"], ad3.obsm["X_pca"])
    # n_comps default = min(50, min(shape)-1) (tests/test_pca.py:277-290)
    tiny = sb.pp.pca(x[:20, :30], return_info=True)
    assert tiny[0].shape == (20, 19) and tiny[1].shape == (19, 30)


def test_pca_building_blocks_linear_algebra(synth_small):
    # size-independent properties: SpMM linearity, X^T(XB) == G B, column stats == numpy
    import torch

    x, _ = synth_small
    n, g = x.shape
    ctx = sb._abi.default_context()
    dp, di, dd = _ops.csr_to_device(x)
    rs = np.random.RandomState(0)
    b = rs.standard_normal((g, 64)).astype(np.float32)
    d_b = torch.from_numpy(b).cuda()
    y = torch.empty((n, 64), dtype=torch.float32, device="cuda")
    sb._abi.check(ctx.lib.sb2_spmm_csr(ctx.handle, n, g, 64, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(d_b), None, _ops.ptr(y)))
    y_ref = x.astype(np.float64) @ b.astype(np.float64)
    np.testing.assert_allclose(y.cpu().numpy(), y_ref, rtol=2e-5, atol=2e-5)
    z = torch.empty((g, 64), dtype=torch.float64, device="cuda")
    sb._abi.check(ctx.lib.sb2_spmm_csr_t(ctx.handle, n, g, 64, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(y), _ops.ptr(z)))
    z_ref = x.astype(np.float64).T @ y.cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(z.cpu().numpy(), z_ref, rtol=2e-4, atol=2e-3 * np.abs(z_ref).max() * 1e-2)
    gram = torch.empty((g, g), dtype=torch.float64, device="cuda")
    sb._abi.check(ctx.lib.sb2_csr_gram(ctx.handle, n, g, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(gram)))
    g_ref = (x.astype(np.float64).T @ x.astype(np.float64)).toarray()
    np.testing.assert_allclose(gram.cpu().numpy(), g_ref, rtol=1e-12, atol=1e-9)
    s1 = torch.empty(g, dtype=torch.float64, device="cuda"); s2 = torch.empty(g, dtype=torch.float64, device="cuda")
    sb._abi.check(ctx.lib.sb2_csr_col_stats(ctx.handle, n, g, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(s1), _ops.ptr(s2)))
    xd = x.astype(np.float64)
    np.testing.assert_allclose(s1.cpu().numpy(), np.asarray(xd.sum(axis=0)).ravel(), rtol=1e-12)
    np.testing.assert_allclose(s2.cpu().numpy(), np.asarray(xd.multiply(xd).sum(axis=0)).ravel(), rtol=1e-12)


# ------------------------------------------------------------------------------------------ kNN
def test_knn_golden_4points(literals):
    # tests/test_neighbors.py:23-39,151-192
    x, k = literals["X4"].astype(np.float32), int(literals["n_neighbors4"])
    idx, dist, _ = _ops.knn(x, k)
    assert (idx[:, 0] == np.arange(4)).all()
    d = sb.pp._get_sparse_matrix_from_indices_distances(idx, dist, keep_self=False).toarray()
    np.testing.assert_allclose(d, literals["distances_euclidean"], rtol=1e-6)


def test_knn_golden_pbmc68k(pbmc68k_graph):
    f = pbmc68k_graph
    k = int(f["n_neighbors"][0])
    idx, dist, _ = _ops.knn(np.ascontiguousarray(f["X_pca"][:, :30]), k)
    for i in range(700):
        assert set(f["dist_indices"][f["dist_indptr"][i]:f["dist_indptr"][i + 1]].tolist()) == set(idx[i, 1:].tolist())
    np.testing.assert_allclose(dist[:, 1:], np.sort(f["dist_data"].reshape(700, k - 1), axis=1), rtol=1e-5)


@pytest.mark.parametrize("n,d,k", [(1, 3, 1), (5, 2, 5), (127, 7, 15), (129, 50, 15), (1000, 50, 30), (4097, 33, 10),
                                   (12345, 50, 15), (3000, 100, 30), (2000, 150, 8), (6000, 50, 30), (5000, 40, 45), (100, 8, 56),
                                   # tile-shape boundaries of the tensor-core pass (knn_tc2.cu: the split-precision K axis is
                                   # staged in 1 / 2 / 4 slices, switching at d = 74 and d = 117 with 227 KB of shared memory)
                                   (3000, 57, 15), (3000, 58, 15), (2500, 73, 40), (2500, 74, 15), (2500, 116, 15),
                                   (2500, 117, 30), (3000, 150, 56)])
def test_knn_identical_index_sets(n, d, k):
    rs = np.random.RandomState(n + d)
    x = rs.standard_normal((n, d)).astype(np.float32)
    x[: n // 3] += 2.5  # two blobs
    idx, dist, info = _ops.knn(x, k)
    oi, od = oknn.knn_brute(x, k) if n > 1 else (np.zeros((1, 1), int), np.zeros((1, 1)))
    assert idx.shape == (n, k) and idx.dtype == np.int32 and dist.dtype == np.float64
    assert (idx[:, 0] == np.arange(n)).all() and (dist[:, 0] == 0).all()
    assert (np.diff(dist, axis=1) >= 0).all()  # ascending rows
    assert oknn.same_neighbor_sets(idx, dist, oi, od).all()   # vs the reference's own call (sklearn brute, float32 in)
    np.testing.assert_allclose(dist[:, 1:], od[:, 1:], rtol=1e-6, atol=1e-7)  # (sklearn's self distance is ~5e-7, not 0)
    if n > 1:   # and literally identical sets against float64 brute force
        ei, ed2 = oknn.knn_exact_f64(x, np.arange(n), k)
        assert oknn.exact_set_mismatches(idx, ei, ed2, k).sum() == 0


def test_knn_threshold_estimate_and_tiers_agree_with_oracle(monkeypatch):
    # large enough (>= 1024 candidate tiles) for the sampled starting threshold of the tensor sweep; every
    # configuration of the tiers must return the same exact result, and that result must match the oracle
    rs = np.random.RandomState(5)
    n, d, k = 140_000, 12, 15
    c = rs.standard_normal((20, d)).astype(np.float32) * 4
    x = (c[rs.randint(0, 20, n)] + rs.standard_normal((n, d))).astype(np.float32)
    idx, dist, info = _ops.knn(x, k)
    assert info["pass1_tensor"] == 2   # tensor-core sweep
    rows = rs.choice(n, 1500, replace=False)
    oi, od2 = oknn.knn_exact_f64(x, rows, k)          # float64 brute force: "identical" means identical
    assert oknn.exact_set_mismatches(idx[rows], oi, od2, k).sum() == 0
    np.testing.assert_allclose(dist[rows][:, 1:], np.sqrt(od2[:, 1:k]), rtol=1e-6, atol=1e-7)
    for env in (dict(SB2_KNN_EST="0"), dict(SB2_KNN_TIERS="3"), dict(SB2_KNN_TIERS="3", SB2_KNN_EST="0"), dict(SB2_KNN_LIST="64"),
                dict(SB2_KNN_SCAN_SLOTS="0"), dict(SB2_KNN_PASS1="ffma")):
        for key in ("SB2_KNN_EST", "SB2_KNN_TIERS", "SB2_KNN_LIST", "SB2_KNN_SCAN_SLOTS", "SB2_KNN_PASS1"):
            monkeypatch.delenv(key, raising=False)
        for key, val in env.items():
            monkeypatch.setenv(key, val)
        idx2, dist2, _ = _ops.knn(x, k)
        assert (idx2 == idx).all() and (dist2 == dist).all(), env


def test_knn_resweep_tier_far_from_origin(monkeypatch):
    # data far from the origin: the fp16 tier's rounding bound (|dq| R + |q| max|dc|) swamps the neighbour gaps, so
    # rows fall through to the gathered split-precision re-sweep (forced here even for few rows) and stay exact
    monkeypatch.setenv("SB2_KNN_SCAN_SLOTS", "0")
    rs = np.random.RandomState(9)
    y = (rs.standard_normal((6000, 24)) * 0.05 + 40.0).astype(np.float32)
    idx, dist, info = _ops.knn(y, 15)
    assert info["n_resweep"] > 0
    oi, od = oknn.knn_brute(y, 15)
    assert oknn.same_neighbor_sets(idx, dist, oi, od).all()
    np.testing.assert_allclose(dist[:, 1:], od[:, 1:], rtol=1e-6, atol=1e-7)


def test_knn_duplicates_zero_rows_and_scale():
    rs = np.random.RandomState(3)
    x = np.zeros((600, 12), np.float32)          # 200 all-zero cells (legal: empty CSR rows) -> exact ties
    x[200:] = rs.standard_normal((400, 12))
    x[300:340] = x[299]                          # a block of exact duplicates
    idx, dist, info = _ops.knn(x, 15)
    oi, od = oknn.knn_brute(x, 15)
    np.testing.assert_allclose(dist, od, atol=1e-6)          # distances identical even where ids tie
    assert (idx[:, 0] == np.arange(600)).all()               # self forced into column 0
    assert info["n_uncertified"] >= 240                      # tie rows went through the exact fallback
    assert oknn.same_neighbor_sets(idx, dist, oi, od).all()  # ties at the k-th distance may resolve to other ids
    # far-from-origin data: rounding bound grows, certificate must still give exact sets
    y = rs.standard_normal((3000, 20)).astype(np.float32) * 0.01 + 1000.0
    idx, dist, info = _ops.knn(y, 10)
    oi, od = oknn.knn_brute(y, 10)
    assert oknn.same_neighbor_sets(idx, dist, oi, od).all()


def test_knn_rejects_unsupported_shapes():
    x = np.zeros((300, 151), np.float32)
    with pytest.raises(sb._abi.B200Error, match="d must be in"):
        _ops.knn(x, 5)
    with pytest.raises(sb._abi.B200Error, match="k must be in"):
        _ops.knn(x[:, :10], 57)


def test_knn_ffma_pass_still_exact(monkeypatch):
    # the CUDA-core first pass stays selectable (SB2_KNN_PASS1=ffma, read per call by sb2_knn_l2_f32); same exact result
    monkeypatch.setenv("SB2_KNN_PASS1", "ffma")
    rs = np.random.RandomState(11)
    x = rs.standard_normal((3000, 100)).astype(np.float32)
    idx, dist, info = _ops.knn(x, 30)
    assert info["pass1_tensor"] == 0
    oi, od = oknn.knn_brute(x, 30)
    assert oknn.same_neighbor_sets(idx, dist, oi, od).all()
    with pytest.raises(sb._abi.B200Error, match="k > 30 needs the tensor-core pass"):
        _ops.knn(x, 31)


def test_knn_transformer_in_reference_pipeline_shape():
    # KnnTransformerLike contract (src/scanpy/neighbors/_types.py:53-64, _common.py:126-143)
    rs = np.random.RandomState(0)
    x = rs.standard_normal((500, 20)).astype(np.float32)
    t = sb.B200KNNTransformer(n_neighbors=15)
    d = t.fit_transform(x)
    assert sparse.issparse(d) and d.shape == (500, 500) and (d.getnnz(axis=1) == 15).all()
    i, dist = oknn.indices_distances_from_sparse(d, 15)  # the reference's own post-processing
    oi, od = oknn.knn_brute(x, 15)
    assert oknn.same_neighbor_sets(i, dist, oi, od).all()


def test_knn_tensor_score_error_within_bound():
    """MEASURES the tensor-core scores against float64 on the hardware and checks the rounding-error bound the exactness
    certificate rests on (knn_tc2_error_coefs + the measured fp16 residual norms): for every proposal (q, c) of a
    cold-start sweep  |s_tensor / s^2 - (q.c - |c|^2/2)| <= eps(q).  Adversarial magnitudes: data far from the origin
    (huge common offset), wide dynamic range across coordinates, every K-slice count (d 20 -> K 32, d 50 -> 64, d 100 ->
    terms 3: K 320 in two slices), both operand formats."""
    import torch

    ctx = sb._abi.default_context()
    rs = np.random.RandomState(0)
    worst = {}
    for d, terms, kind in [(20, 1, "offset"), (50, 1, "plain"), (50, 3, "offset"), (50, 1, "range"), (100, 3, "range"), (7, 3, "plain"),
                           (100, 1, "offset")]:
        n = 3000
        x = rs.standard_normal((n, d))
        if kind == "offset":
            x = x * 0.3 + 25.0                      # far from the origin: |x| >> neighbour distances
        elif kind == "range":
            x = x * np.logspace(-3, 1.5, d)[None]   # coordinates spanning 4.5 orders of magnitude
        x = np.ascontiguousarray(x, np.float32)
        d_x = torch.from_numpy(x).cuda()
        sc = torch.empty((n, 64), dtype=torch.float32, device="cuda")
        ix = torch.empty((n, 64), dtype=torch.int32, device="cuda")
        dn = torch.zeros(n, dtype=torch.float32, device="cuda")
        meta = np.zeros(6, np.float64)
        sb._abi.check(ctx.lib.sb2_knn_debug_proposals_f32(ctx.handle, n, d, _ops.ptr(d_x), terms, _ops.ptr(sc), _ops.ptr(ix), _ops.ptr(dn),
                                                          meta.ctypes.data))
        torch.cuda.synchronize()
        inv_s2, r2, dmax, cq, cn, _ = meta
        sc, ix, dn = sc.cpu().numpy().astype(np.float64), ix.cpu().numpy(), dn.cpu().numpy().astype(np.float64)
        x64 = x.astype(np.float64)
        qn = np.sqrt((x64 ** 2).sum(1))
        R = np.sqrt(r2)
        eps = cn * 0.5 * R * R + cq * qn * R
        if terms == 1:
            eps = eps + (dn * R + (qn + dn) * dmax) * (1 + 1e-6)
        used = ix >= 0
        c = x64[np.where(used, ix, 0)]                                        # [n, 64, d]
        s_exact = np.einsum("nd,nmd->nm", x64, c) - 0.5 * (c ** 2).sum(-1)
        err = np.abs(sc * inv_s2 - s_exact)
        ratio = (err / eps[:, None])[used]
        worst[(d, terms, kind)] = float(ratio.max())
        assert used.sum() > n * 32
        assert ratio.max() <= 1.0, (d, terms, kind, ratio.max())
    print("\n[tensor score error / certified bound] " + ", ".join(f"d={k[0]} terms={k[1]} {k[2]}: {v:.3f}" for k, v in worst.items()))


@pytest.mark.parametrize("k", [40, 56])
def test_connectivities_large_k(k):
    # k-lists longer than 32 (the reference has no limit: src/scanpy/neighbors/_connectivity.py:103-138)
    from oracle import connectivity as oconn

    rs = np.random.RandomState(k)
    x = rs.standard_normal((1500, 10)).astype(np.float32)
    x[:400] += 2.0
    idx, dist, _ = _ops.knn(x, k)
    c, sig, rho = _ops.fuzzy_simplicial_set(idx, dist)
    oc, osig, orho = ofz.fuzzy_simplicial_set(idx, dist, 1500, k)
    oc.sort_indices()
    assert c.nnz == oc.nnz and (c.indices == oc.indices).all() and abs(c - c.T).max() == 0
    np.testing.assert_allclose(c.data, oc.data, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(sig, osig, rtol=1e-6)
    for method, ofun in (("gauss", lambda: oconn.gauss_knn(idx, dist)), ("jaccard", lambda: oconn.jaccard(idx))):
        g = _ops.knn_connectivities(idx, dist, method)
        o = ofun().tocsr()
        o.sort_indices(); o.eliminate_zeros()
        assert g.nnz == o.nnz and (g.indices == o.indices).all()
        np.testing.assert_allclose(g.data, o.data, rtol=1e-12, atol=1e-300)


def test_neighbors_precomputed_distances_honours_method(synth_small):
    # ADVICE r1: `distances=` + method='gauss' / 'jaccard' must dispatch like the reference (neighbors/__init__.py:672-708)
    x, _ = synth_small
    ad = sb.MiniAnnData(x[:900])
    sb.pp.pca(ad, n_comps=12)
    sb.pp.neighbors(ad, n_neighbors=10)
    for method in ("gauss", "jaccard"):
        ref = sb.MiniAnnData(x[:900], obsm={"X_pca": ad.obsm["X_pca"].copy()})
        sb.pp.neighbors(ref, n_neighbors=10, method=method)
        got = sb.MiniAnnData(x[:900])
        sb.pp.neighbors(got, n_neighbors=10, method=method, distances=ad.obsp["distances"])
        assert got.uns["neighbors"]["params"]["method"] == method
        np.testing.assert_allclose(got.obsp["connectivities"].toarray(), ref.obsp["connectivities"].toarray(), rtol=1e-9, atol=1e-12)
        assert abs(got.obsp["connectivities"] - ad.obsp["connectivities"]).max() > 1e-3   # and it is NOT the umap graph


# ------------------------------------------------------------------------------------------ connectivities
def test_fuzzy_goldens(literals, pbmc68k_graph):
    x, k = literals["X4"].astype(np.float32), int(literals["n_neighbors4"])
    idx, dist, _ = _ops.knn(x, k)
    c, _, _ = _ops.fuzzy_simplicial_set(idx, dist)
    np.testing.assert_allclose(c.toarray(), literals["connectivities_umap"], atol=5e-8)  # tests/test_neighbors.py:43-48
    f = pbmc68k_graph
    n, k = 700, int(f["n_neighbors"][0])
    di, dd = f["dist_indices"].reshape(n, k - 1), f["dist_data"].reshape(n, k - 1)
    o = np.argsort(dd, axis=1, kind="stable")
    idx = np.hstack([np.arange(n)[:, None], np.take_along_axis(di, o, 1)]).astype(np.int32)
    dist = np.hstack([np.zeros((n, 1)), np.take_along_axis(dd, o, 1)])
    c, _, _ = _ops.fuzzy_simplicial_set(idx, dist)
    g = sparse.csr_matrix((f["conn_data"], f["conn_indices"], f["conn_indptr"]), shape=(n, n))
    g.sort_indices()
    assert c.nnz == 9992 and (c.indices == g.indices).all() and (c.indptr == g.indptr).all()
    np.testing.assert_allclose(c.data, g.data, atol=5e-7)


@pytest.mark.parametrize("n,k", [(50, 5), (3000, 15), (20000, 30)])
def test_fuzzy_matches_oracle(n, k):
    rs = np.random.RandomState(n)
    x = rs.standard_normal((n, 10)).astype(np.float32)
    x[: n // 10] = x[0]  # duplicates -> zero distances -> rho / sigma-floor branches
    idx, dist, _ = _ops.knn(x, k)
    c, sig, rho = _ops.fuzzy_simplicial_set(idx, dist)
    oc, osig, orho = ofz.fuzzy_simplicial_set(idx, dist, n, k)
    assert c.dtype == np.float32 and c.has_sorted_indices and (c.data != 0).all() and c.diagonal().sum() == 0
    assert abs(c - c.T).max() == 0  # exactly symmetric
    oc.sort_indices()
    assert c.nnz == oc.nnz and (c.indices == oc.indices).all()
    np.testing.assert_allclose(c.data, oc.data, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(rho, orho, rtol=0, atol=0)
    np.testing.assert_allclose(sig, osig, rtol=1e-6)


# ------------------------------------------------------------------------------------------ Leiden
def test_leiden_properties_and_quality(pbmc68k_graph):
    f = pbmc68k_graph
    n = 700
    g = sparse.csr_matrix((f["conn_data"].astype(np.float32), f["conn_indices"], f["conn_indptr"]), shape=(n, n))
    m0, q0, info = _ops.leiden(g, seed=0)
    m0b, q0b, _ = _ops.leiden(g, seed=0)
    assert (m0 == m0b).all() and q0 == q0b                 # same seed -> identical (tests/test_clustering.py:67-102)
    m1, _, _ = _ops.leiden(g, seed=1)
    assert 0.0 <= q0 <= 1.0                                # tests/test_metrics.py:311-344
    assert (np.diff(np.bincount(m0)) <= 0).all()           # '0' is the largest cluster
    assert abs(old.modularity(g, m0) - q0) < 1e-7          # our Q == independent restatement
    assert abs(_ops.modularity(g, m0) - q0) < 1e-12
    mo, qo, _ = old.leiden(g, seed=0)
    assert q0 >= qo - 1.5e-3                               # quality guard vs the sequential oracle
    assert adjusted_rand_score(m1, m0) > 0.9               # other seed: same structure (label-level gate: next test)
    lo, _, _ = _ops.leiden(g, resolution=0.2, seed=0)
    hi, _, _ = _ops.leiden(g, resolution=3.0, seed=0)
    assert lo.max() < m0.max() < hi.max()
    two, _, i2 = _ops.leiden(g, n_iterations=2, seed=0)
    assert i2["passes"] == 2


def _overlapping_knn_graph(n, k=15, seed=0, sep=1.6):
    """UMAP connectivities of overlapping gaussian clusters (NOT separable blobs) through the CUDA kNN + fuzzy set."""
    rs = np.random.RandomState(seed)
    centers = rs.standard_normal((12, 10)) * sep
    lab = rs.randint(0, 12, n)
    x = (centers[lab] + rs.standard_normal((n, 10))).astype(np.float32)
    idx, dist, _ = _ops.knn(x, k)
    c, _, _ = _ops.fuzzy_simplicial_set(idx, dist)
    return c, lab


def test_leiden_real_graph_within_oracle_spread(pbmc68k_graph):
    """Label-level gate on the reference's own real-data graph.  ARI >= 0.99 against ONE oracle run is not a property
    the sequential algorithm itself has there (tests/test_oracle_leiden_guarantees.py: seed-to-seed ARI 0.95-1.0, for
    both back-end flavours), so the gate is: for >= 5 seeds, quality at least the oracle's median and agreement with the
    oracle runs no worse than the oracle runs agree among themselves; plus the reference's own NMI > 0.9 bar
    (tests/test_clustering.py:130-163)."""
    from sklearn.metrics import normalized_mutual_info_score

    f = pbmc68k_graph
    g = sparse.csr_matrix((f["conn_data"].astype(np.float32), f["conn_indices"], f["conn_indptr"]), shape=(700, 700))
    oracle = [old.leiden(g, seed=s, beta=b) for b in (0.0, 0.01) for s in range(6)]       # both flavours
    o_ari = [adjusted_rand_score(oracle[i][0], oracle[j][0]) for i in range(len(oracle)) for j in range(i)]
    q_med = float(np.median([r[1] for r in oracle]))
    worst = []
    for seed in range(6):
        m, q, _ = _ops.leiden(g, seed=seed)
        a = [adjusted_rand_score(r[0], m) for r in oracle]
        nmi = [normalized_mutual_info_score(r[0], m) for r in oracle]
        worst.append(min(a))
        assert q >= q_med - 1.5e-3, (seed, q, q_med)                     # quality: not below the oracle's median
        assert np.median(a) >= np.median(o_ari) - 0.02, (seed, np.median(a), np.median(o_ari))
        assert min(a) >= min(o_ari) - 0.02, (seed, min(a), min(o_ari))   # inside the oracle's own spread
        assert min(nmi) > 0.9
        assert m.max() == oracle[0][0].max()                             # same number of communities (12)
    print(f"\n[pbmc68k] oracle-vs-oracle ARI min {min(o_ari):.3f} median {np.median(o_ari):.3f}; CUDA-vs-oracle worst {min(worst):.3f}")


def test_leiden_cutoffs_and_empty_moves_do_not_cost_quality(monkeypatch):
    """The two performance cut-offs (first-pass local moving stops below 0.5 % movers, refinement stops below 0.1 %
    merges) against SB2_LEIDEN_EXACT=1, which runs every phase to its fixed point - on overlapping clusters."""
    g, lab = _overlapping_knn_graph(60_000)
    m_fast, q_fast, _ = _ops.leiden(g, seed=0)
    monkeypatch.setenv("SB2_LEIDEN_EXACT", "1")
    m_exact, q_exact, _ = _ops.leiden(g, seed=0)
    monkeypatch.delenv("SB2_LEIDEN_EXACT")
    mo, qo, _ = old.leiden(g, seed=0)
    mo2, qo2, _ = old.leiden(g, seed=1)
    spread = adjusted_rand_score(mo, mo2)
    print(f"\n[overlap 60k] Q cut-offs {q_fast:.5f} exact {q_exact:.5f} oracle {qo:.5f}/{qo2:.5f}; ARI fast-vs-exact "
          f"{adjusted_rand_score(m_fast, m_exact):.3f}, fast-vs-oracle {adjusted_rand_score(m_fast, mo):.3f}, oracle seed-vs-seed {spread:.3f}")
    assert q_fast >= q_exact - 1e-3 and q_fast >= min(qo, qo2) - 1e-3
    assert adjusted_rand_score(m_fast, mo) >= spread - 0.03
    assert adjusted_rand_score(m_exact, mo) >= spread - 0.03


def test_leiden_overlapping_100k_vs_oracle():
    g, lab = _overlapping_knn_graph(100_000, sep=1.3)
    m, q, info = _ops.leiden(g, seed=0)
    runs = [old.leiden(g, seed=s) for s in range(3)]
    o_ari = [adjusted_rand_score(runs[i][0], runs[j][0]) for i in range(3) for j in range(i)]
    a = [adjusted_rand_score(r[0], m) for r in runs]
    print(f"\n[overlap 100k] Q {q:.5f} oracle {[round(r[1], 5) for r in runs]}; ARI vs oracle {np.round(a, 3)}, oracle seed-vs-seed {np.round(o_ari, 3)}; "
          f"ARI vs planted {adjusted_rand_score(lab, m):.3f} (oracle {adjusted_rand_score(lab, runs[0][0]):.3f})")
    assert q >= min(r[1] for r in runs) - 1e-3
    assert min(a) >= min(o_ari) - 0.03
    # every community connected (the Leiden guarantee), checked on the CUDA result
    from scipy.sparse.csgraph import connected_components
    for c in range(m.max() + 1):
        mem = np.flatnonzero(m == c)
        assert connected_components(g[mem][:, mem], directed=False)[0] == 1


def test_leiden_planted_ari(synth_small):
    x, lab = synth_small
    ad = sb.MiniAnnData(x)
    sb.pp.pca(ad, n_comps=30)
    sb.pp.neighbors(ad, n_neighbors=15)
    sb.tl.leiden(ad, flavor="igraph", n_iterations=-1)
    got = ad.obs["leiden"].to_numpy().astype(int)
    mo, qo, _ = old.leiden(ad.obsp["connectivities"], seed=0)
    assert adjusted_rand_score(mo, got) >= 0.99
    assert adjusted_rand_score(lab, got) >= 0.99
    assert ad.uns["leiden"]["modularity"] >= qo - 1e-3


def test_pipeline_writebacks_match_contract(synth_small):
    # SURVEY.md Appendix B, key by key
    x, _ = synth_small
    ad = sb.MiniAnnData(x[:2500])
    with pytest.warns(UserWarning, match="Falling back to preprocessing with `sc.pp.pca`"):
        sb.pp.neighbors(ad, n_neighbors=10, n_pcs=20)      # auto-PCA (tests/test_neighbors_key_added.py:53-61)
    assert ad.obsm["X_pca"].shape == (2500, 20)
    assert ad.uns["neighbors"] == dict(connectivities_key="connectivities", distances_key="distances",
                                       params=dict(n_neighbors=10, method="umap", metric="euclidean", random_state=0, n_pcs=20))
    d, c = ad.obsp["distances"], ad.obsp["connectivities"]
    assert (np.diff(d.indptr) == 9).all() and (d.indptr == np.arange(0, 2500 * 9 + 1, 9)).all()
    assert c.dtype == np.float32 and abs(c - c.T).max() == 0 and (c.data != 0).all()
    sb.pp.neighbors(ad, n_neighbors=10, n_pcs=20, key_added="nb2", rng=5)
    assert "random_state" not in ad.uns["nb2"]["params"] and ad.uns["nb2"]["distances_key"] == "nb2_distances"
    assert (ad.obsp["nb2_connectivities"] != c).nnz == 0   # key_added equivalence (tests/test_neighbors_key_added.py:35-50)
    sb.tl.leiden(ad, resolution=0.8, flavor="igraph", n_iterations=2, random_state=3, key_added="cl")
    assert ad.uns["cl"]["params"] == dict(resolution=0.8, n_iterations=2, random_state=3)
    assert str(ad.obs["cl"].dtype) == "category" and list(ad.obs["cl"].cat.categories) == [str(i) for i in range(len(ad.obs["cl"].cat.categories))]
    sb.tl.leiden(ad, flavor="igraph", neighbors_key="nb2", restrict_to=("cl", ["0"]))
    r = ad.obs["leiden_R"].astype(str)
    assert (r[ad.obs["cl"] != "0"] == ad.obs["cl"].astype(str)[ad.obs["cl"] != "0"]).all()
    assert r[ad.obs["cl"] == "0"].str.startswith("0,").all()  # tests/test_clustering.py:177-213


def test_neighbors_precomputed_distances_and_use_rep(synth_small):
    # recompute-from-stored-distances equivalence (tests/test_neighbors.py:275-296) and use_rep (:251-261)
    x, _ = synth_small
    ad = sb.MiniAnnData(x[:1200])
    sb.pp.pca(ad, n_comps=15)
    sb.pp.neighbors(ad, n_neighbors=12)
    ad2 = sb.MiniAnnData(x[:1200])
    with pytest.warns(UserWarning, match="ignored if `distances` is given"):
        sb.pp.neighbors(ad2, n_neighbors=12, distances=ad.obsp["distances"], n_pcs=5)
    np.testing.assert_allclose(ad2.obsp["connectivities"].toarray(), ad.obsp["connectivities"].toarray(), rtol=1e-5)
    assert ad2.uns["neighbors"]["params"]["method"] == "umap"
    np.testing.assert_allclose(ad2.obsp["distances"].toarray(), ad.obsp["distances"].toarray(), rtol=1e-5)
    p, p_d = (dict(a.uns["neighbors"]["params"]) for a in (ad, ad2))
    assert p.pop("metric") == "euclidean" and p_d.pop("metric") is None and p == p_d
    # a dense precomputed matrix means ALL pairwise distances (src/scanpy/neighbors/_common.py:63-71)
    from sklearn.metrics import pairwise_distances
    full = pairwise_distances(ad.obsm["X_pca"].astype(np.float64))
    ad3 = sb.MiniAnnData(x[:1200])
    sb.pp.neighbors(ad3, n_neighbors=12, distances=full)
    np.testing.assert_allclose(ad3.obsp["connectivities"].toarray(), ad.obsp["connectivities"].toarray(), rtol=1e-4, atol=1e-6)
    ad4 = sb.MiniAnnData(x[:1200], obsm={"X_rep": ad.obsm["X_pca"].copy()})
    sb.pp.neighbors(ad4, n_neighbors=12, use_rep="X_rep")
    assert (ad4.obsp["distances"] != ad.obsp["distances"]).nnz == 0
    assert ad4.uns["neighbors"]["params"]["use_rep"] == "X_rep"
    # n_pcs slicing == PCA with fewer components (tests/test_pca.py:389-400)
    sb.pp.neighbors(ad, n_neighbors=12, n_pcs=8, key_added="p8")
    ad5 = sb.MiniAnnData(x[:1200], obsm={"X_pca": ad.obsm["X_pca"][:, :8].copy()})
    sb.pp.neighbors(ad5, n_neighbors=12)
    assert (ad5.obsp["distances"] != ad.obsp["p8_distances"]).nnz == 0


# ------------------------------------------------------------------------------------------ preprocessing (8f, f2)
def _raw_pbmc():
    from pathlib import Path

    f = np.load(Path(__file__).parent / "golden" / "pbmc68k_raw_seurat_hvg.npz")
    return sparse.csr_matrix((f["raw_data"], f["raw_indices"], f["raw_indptr"]), shape=(700, 765)), f


def test_preprocess_chain_matches_seurat_golden():
    # the reference's own golden: tests/test_highly_variable_genes.py:379-421 (rtol = atol = 2e-5 there)
    x, f = _raw_pbmc()
    ad = sb.MiniAnnData(x.copy())
    sb.pp.normalize_total(ad, target_sum=1e4)
    sb.pp.log1p(ad)
    assert ad.uns["log1p"] == {"base": None}
    sb.pp.highly_variable_genes(ad, flavor="seurat", min_mean=0.0125, max_mean=3, min_disp=0.5)
    np.testing.assert_array_equal(ad.var["highly_variable"].to_numpy(), f["highly_variable"])
    for k in ("means", "dispersions", "dispersions_norm"):
        np.testing.assert_allclose(ad.var[k].to_numpy(), f[k], rtol=2e-5, atol=2e-5)
    # and the whole chain feeds the hot path: mask_var picks var['highly_variable'] up
    sb.pp.pca(ad, n_comps=10)
    assert (ad.varm["PCs"][~f["highly_variable"]] == 0).all()


def test_normalize_total_and_log1p_match_oracle():
    from oracle import preprocess as op

    a = np.array([[3, 3, 3, 6, 6], [1, 1, 1, 2, 2], [1, 22, 1, 2, 2]], dtype=np.float32)
    out = sb.pp.normalize_total(sb.MiniAnnData(sparse.csr_matrix(a)), target_sum=1, inplace=False)
    np.testing.assert_allclose(out["X"].toarray(), op.normalize_total(a, target_sum=1)[0].toarray(), rtol=1e-7)
    out = sb.pp.normalize_total(sb.MiniAnnData(sparse.csr_matrix(a)), target_sum=1, exclude_highly_expressed=True,
                                max_fraction=0.2, inplace=False)
    np.testing.assert_allclose(out["X"].toarray(), [[0.5, 0.5, 0.5, 1, 1], [0.5, 0.5, 0.5, 1, 1], [0.5, 11, 0.5, 1, 1]], rtol=1e-6)
    rs = np.random.RandomState(0)
    x = sparse.random(5000, 300, density=0.1, format="csr", random_state=rs, data_rvs=lambda s: rs.poisson(3, s) + 1).astype(np.float32)
    x[17] = 0  # an empty cell
    x.eliminate_zeros()
    ad = sb.MiniAnnData(x.copy())
    with pytest.warns(UserWarning, match="Some cells have zero counts"):
        sb.pp.normalize_total(ad, key_added="nf")
    ox, oc, _ = op.normalize_total(x)
    np.testing.assert_allclose(ad.X.data, ox.data, rtol=1e-6)
    np.testing.assert_allclose(ad.obs["nf"].to_numpy(), oc, rtol=1e-6)
    sb.pp.log1p(ad, base=2)
    np.testing.assert_allclose(ad.X.data, op.log1p(ox, base=2).data, rtol=2e-6)
    with pytest.raises(ValueError, match="max_fraction between 0 and 1"):
        sb.pp.normalize_total(ad, max_fraction=2)


# ------------------------------------------------------------------------------------------ gauss / jaccard (8f, f3)
def test_gauss_jaccard_goldens_and_oracle(literals):
    from oracle import connectivity as oconn

    # reference 4-point goldens: tests/test_neighbors.py:66-72,120-126,195-226
    ad = sb.MiniAnnData(literals["X4"].astype(np.float32))
    for method, key in (("gauss", "connectivities_gauss_knn"), ("jaccard", "connectivities_jaccard")):
        sb.pp.neighbors(ad, n_neighbors=int(literals["n_neighbors4"]), method=method, key_added=method)
        c = ad.obsp[f"{method}_connectivities"]
        assert c.dtype == np.float64 and ad.uns[method]["params"]["method"] == method
        np.testing.assert_allclose(c.toarray(), literals[key], rtol=1e-6, atol=1e-7)
    rs = np.random.RandomState(1)
    x = rs.standard_normal((3000, 12)).astype(np.float32)
    x[:1000] += 3
    idx, dist, _ = _ops.knn(x, 15)
    for method, ofun in (("gauss", lambda: oconn.gauss_knn(idx, dist)), ("jaccard", lambda: oconn.jaccard(idx))):
        c = _ops.knn_connectivities(idx, dist, method)
        o = ofun().tocsr()
        o.sort_indices(); o.eliminate_zeros()
        assert c.has_sorted_indices and c.nnz == o.nnz and (c.indices == o.indices).all()
        np.testing.assert_allclose(c.data, o.data, rtol=1e-12, atol=1e-300)
        assert abs(c - c.T).max() < 1e-15

"""PCA against float64 truth where the solver branches (need an H100: `pytest -m gpu`).

csrc/pca.cu iterates a block of l = 32 / 64 / 128 columns (l picked from n_comps + 8), pads g < l genes with zero genes
(which forces the Gram route), refills directions lost to rank deficiency with random vectors, and has two operators
(dense Gram, CSR SpMM passes) and two Rayleigh-Ritz solvers (device Jacobi for l <= 64, host Jacobi for l = 128).  Every
case here runs such a branch on both operators where the route allows and compares with a float64 truth through
`oracle.pca.compare_pca`: per component where the truth's relative eigengap is >= 1e-3 (X_pca 1e-4 up to sign, loadings
2e-4 with svd_flip signs), as a subspace inside closer clusters (principal-angle sine 1e-4), and |X_pca| <= 1e-5 of the
first column with variance <= 1e-9 of the largest on null components; variance and variance_ratio to 1e-5.  A result that
reports `converged` must meet that bar.  Each case prints its measured errors next to the bars.
"""
import warnings

import numpy as np
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import pca as opca
from scanpy_b200 import _ops
from scanpy_b200._synth import synth_scipy

pytestmark = pytest.mark.gpu

CAP = {1: 4000, 0: 300}   # default iteration caps of the Gram and SpMM routes


def _check(label, out, truth, k, *, require=True, **bars):
    rep = opca.compare_pca(out, truth, k, **bars)
    print(f"\n[{label}] converged={out['converged']} iterations={out['iterations']} "
          f"residual={out['max_rel_residual']:.1e} min gap {rep['min_gap']:.1e}: {rep['summary']}")
    # a result that says it converged meets the bar; one that does not must say so
    assert rep["ok"] or not out["converged"], (label, rep["failures"])
    if require:
        assert rep["ok"], (label, rep["failures"])
        assert out["converged"], label
    return rep


def _csr(a):
    x = sparse.csr_matrix(np.asarray(a, np.float32))
    x.eliminate_zeros()
    return x


# ------------------------------------------------------------------------------------------ block widths
@pytest.mark.parametrize("k", [1, 24, 25, 56, 57, 120])
def test_block_width_boundaries(k):
    # l = 32 up to k = 24, 64 up to k = 56, 128 up to k = 120 (8 guard vectors); the latent rank ~2k keeps the spectrum
    # gapped past the cut
    x, _ = synth_scipy(4000, 600, n_clusters=12, r=max(8, 2 * k), seed=k)
    truth = opca.pca_full_f64(x, dense=False)
    for solver in (1, 0):
        _check(f"k={k} solver={solver}", _ops.pca_csr(x, k, solver=solver), truth, k)


def test_more_than_120_components_is_refused():
    x, _ = synth_scipy(600, 300, n_clusters=6, r=16)
    with pytest.raises(sb._abi.B200Error, match=r"n_components <= 120"):
        _ops.pca_csr(x, 121, solver=1)
    with pytest.raises(NotImplementedError, match=r"at most 120 components \(n_comps=121\)"):
        sb.pp.pca(x, n_comps=121)
    with pytest.raises(NotImplementedError, match=r"at most 120 components \(n_comps=121\)"):
        sb.pp.pca(x, n_comps=121, chunked=True, chunk_size=100)


# ------------------------------------------------------------------------------------------ padding (g < l)
@pytest.mark.parametrize("g", [20, 31, 33, 63, 100])
def test_padding_fewer_genes_than_the_block(g):
    k = g - 1
    x, _ = synth_scipy(400, g, n_clusters=6, r=min(g, 24), density=0.3, seed=g)
    truth = opca.pca_full_f64(x)
    outs = {}
    for solver in (1, 0):   # g < l forces the Gram route whatever was asked for
        outs[solver] = _ops.pca_csr(x, k, solver=solver)
        _check(f"g={g} k={k} solver={solver}", outs[solver], truth, k)
    a, b = outs[1], outs[0]
    keep = truth["spectrum"][:k] > 1e-12 * truth["spectrum"][0]   # null components are any orthonormal completion
    scale = np.abs(a["X_pca"][:, keep]).max(axis=0)
    assert (np.abs(a["X_pca"] - b["X_pca"])[:, keep] / scale).max() < 1e-6
    np.testing.assert_allclose(a["components"][keep], b["components"][keep], atol=1e-6)
    np.testing.assert_allclose(a["variance"], b["variance"], rtol=1e-10, atol=0.0)


def test_padding_default_n_comps_values():
    # the default n_comps on a 20 x 30 slice: min(shape) - 1 = 19 components from a 32-wide block over 30 + 2 padding genes
    x, _ = synth_scipy(6000, 800, n_clusters=12, r=48)
    x = x[:20, :30]
    x_pca, comps, ratio, var = sb.pp.pca(x, return_info=True)
    assert x_pca.shape == (20, 19) and comps.shape == (19, 30)
    truth = opca.pca_full_f64(x)
    got = dict(X_pca=x_pca, components=comps, variance=var, variance_ratio=ratio, converged=True, iterations=0,
               max_rel_residual=0.0)
    _check("20x30 default n_comps", got, truth, 19)


# ------------------------------------------------------------------------------------------ rank deficiency
def _profiles(n_profiles=12, repeats=5, g=300, seed=3):
    p, _ = synth_scipy(n_profiles, g, n_clusters=4, r=12, density=0.2, seed=seed)
    rows = np.random.RandomState(seed).permutation(np.repeat(np.arange(n_profiles), repeats))
    return p[rows]


def _low_rank_product(n=300, g=120, r=6, seed=4):
    rs = np.random.RandomState(seed)
    return _csr(rs.randint(-2, 3, (n, r)) @ rs.randint(0, 4, (r, g)))   # integers: exactly rank r in float32


RANK_CASES = {
    "40 cells x 500 genes, k=30": (lambda: synth_scipy(40, 500, n_clusters=4, r=24, density=0.1, seed=5)[0], 30),
    "31 cells, k=30": (lambda: synth_scipy(31, 400, n_clusters=4, r=24, density=0.1, seed=6)[0], 30),
    "12 profiles x 5, k=10 (rank 11)": (lambda: _profiles(), 10),
    "12 profiles x 5, k=15 (rank 11)": (lambda: _profiles(), 15),
    "rank-6 product, k=12": (lambda: _low_rank_product(), 12),
}


@pytest.mark.parametrize("case", list(RANK_CASES))
def test_rank_deficient(case):
    make, k = RANK_CASES[case]
    x = make()
    truth = opca.pca_full_f64(x)
    for solver in (1, 0):
        out = _ops.pca_csr(x, k, solver=solver)
        _check(f"{case} solver={solver}", out, truth, k)
        assert out["iterations"] <= CAP[solver] // 4, (case, solver, out["iterations"])


@pytest.mark.parametrize("svd_solver", ["covariance_eigh", "b200_spmm"])
def test_rank_below_k_does_not_warn(svd_solver):
    # 11 distinct centred directions, 15 components asked for: components 11..14 are exactly null, which is an answer,
    # not a failure to converge
    x = _profiles()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        x_pca, comps, ratio, var = sb.pp.pca(x, n_comps=15, svd_solver=svd_solver, return_info=True)
    msgs = [str(w.message) for w in rec if "residual tolerance" in str(w.message)]
    truth = opca.pca_full_f64(x)
    got = dict(X_pca=x_pca, components=comps, variance=var, variance_ratio=ratio, converged=not msgs, iterations=-1,
               max_rel_residual=float("nan"))
    _check(f"pp.pca rank 11 < k=15 {svd_solver}", got, truth, 15)
    assert not msgs, msgs


# ------------------------------------------------------------------------------------------ degenerate columns
def test_degenerate_columns_and_empty_rows():
    x, _ = synth_scipy(2000, 200, n_clusters=8, r=16, density=0.2, seed=7)
    d = x.toarray()
    d[:, 3] = 0.0                     # an all-zero gene
    d[:, 6] = d[:, 5] = 30.0 * d[:, 5]  # a duplicated dominant pair: the top loading is a tie of equal sign
    d[100:160] = 0.0                  # empty rows
    a = _csr(d)
    d2 = d.copy()
    d2[:, 4], d2[:, 9] = 2.5, 7.0     # constant non-zero genes (and no empty rows left)
    b = _csr(d2)
    for name, x, k in (("zero gene, duplicated pair, empty rows", a, 10), ("constant genes", b, 10)):
        truth = opca.pca_full_f64(x)
        for solver in (1, 0):
            out = _ops.pca_csr(x, k, solver=solver)
            _check(f"{name} solver={solver}", out, truth, k)
            assert out["mean"][3] == 0.0
            if x is b:
                np.testing.assert_allclose(out["mean"][[4, 9]], [2.5, 7.0], rtol=1e-12)
            np.testing.assert_allclose(out["total_var"], truth["total_var"], rtol=1e-10)
    # the first component is the duplicated pair; svd_flip's tie (equal |.|, equal sign) leaves it positive
    comp = _ops.pca_csr(a, 3, solver=1)["components"][0]
    assert abs(comp[5] - comp[6]) < 1e-6 and comp[5] > 0.5


def test_one_gene_carries_all_variance():
    rs = np.random.RandomState(8)
    d = np.zeros((500, 50))
    d[:, 17] = rs.standard_normal(500) * 10 * (rs.rand(500) < 0.5)
    d[:, 30] = 4.0
    x = _csr(d)
    truth = opca.pca_full_f64(x)
    for solver in (1, 0):
        out = _ops.pca_csr(x, 3, solver=solver)
        _check(f"one gene solver={solver}", out, truth, 3)
        np.testing.assert_allclose(out["variance_ratio"][0], 1.0, rtol=1e-6)
        assert out["components"][0, 17] > 0.999999


# ------------------------------------------------------------------------------------------ large gene means
def test_large_gene_means():
    # genes with means 100..1000 and spread ~1: X_pca = X U - 1 (mu^T U) cancels in float32, as does the reference's
    # float32 ARPACK run.  The Gram route projects in fp64 and meets the fp64 bar; the SpMM route centres every pass in
    # fp32 and must say that it cannot (converged=False, and pp.pca warns)
    rs = np.random.RandomState(9)
    n, g, k = 3000, 300, 20
    mu = rs.uniform(100.0, 1000.0, g)
    z = rs.standard_normal((n, 12)) * np.linspace(2.0, 0.5, 12)
    d = mu + z @ (rs.standard_normal((12, g)) / np.sqrt(12)) + 0.3 * rs.standard_normal((n, g))
    x = _csr(d)
    truth = opca.pca_full_f64(x)
    ref32 = opca.pca_arpack(x, k)
    cols = np.arange(k)
    t = opca.project(truth, cols)
    noise = np.linalg.norm(opca.align_signs(ref32["X_pca"].astype(np.float64), t) - t, axis=0) / np.linalg.norm(t, axis=0)
    out = _ops.pca_csr(x, k, solver=1)
    e32 = np.linalg.norm(opca.align_signs(out["X_pca"].astype(np.float64), ref32["X_pca"]) - ref32["X_pca"], axis=0) \
        / np.linalg.norm(ref32["X_pca"], axis=0)
    print(f"\n[large means solver=1] vs the live float32 ARPACK call: max {e32.max():.2e} (bar: max(1e-4, 2x the "
          f"reference's own error vs fp64, max {noise.max():.2e}))")
    assert (e32 < np.maximum(1e-4, 2.0 * noise + 1e-5)).all(), (e32.max(), noise.max())
    _check("large means solver=1 vs fp64", out, truth, k)
    out = _ops.pca_csr(x, k, solver=0)
    _check("large means solver=0 vs fp64", out, truth, k, require=False)
    assert not out["converged"]
    with pytest.warns(UserWarning, match="did not reach its residual tolerance"):
        sb.pp.pca(x, n_comps=k, svd_solver="b200_spmm")


# ------------------------------------------------------------------------------------------ zero_center=False
@pytest.mark.parametrize("k", [24, 100])
def test_zero_center_false_block_widths(k):
    x, _ = synth_scipy(3000, 400, n_clusters=8, r=2 * k, seed=10 + k)
    truth = opca.pca_full_f64(x, zero_center=False)
    ref = opca.truncated_svd_arpack(x, k)
    np.testing.assert_allclose(truth["variance"][:k], ref["variance"], rtol=1e-8)   # the truth restates the reference
    for solver in (1, 0):
        _check(f"zero_center=False k={k} solver={solver}", _ops.tsvd_csr(x, k, solver=solver), truth, k)


# ------------------------------------------------------------------------------------------ chunked
@pytest.mark.parametrize("k", [20, 100])
def test_chunked_ragged_chunks_over_empty_rows(k):
    x, _ = synth_scipy(5000, 600, n_clusters=8, r=2 * k, seed=20 + k)
    x = x.tolil()
    x[1500:1900] = 0                  # chunk boundaries 1665 and 1998 (chunk_size 333) fall inside / at the end of this run
    x = x.tocsr().astype(np.float32)
    x.eliminate_zeros()
    full = _ops.pca_csr(x, k, solver=1)
    ch = _ops.pca_csr_chunked(x, k, chunk_size=333)
    scale = np.abs(full["X_pca"]).max(axis=0)
    diff = (np.abs(full["X_pca"] - ch["X_pca"]) / scale).max()
    print(f"\n[chunked k={k}] vs in-core Gram route: {diff:.2e} (bar 2e-6)")
    assert diff < 2e-6
    np.testing.assert_allclose(ch["components"], full["components"], atol=2e-6)
    np.testing.assert_allclose(ch["variance"], full["variance"], rtol=1e-9)
    np.testing.assert_allclose(ch["variance_ratio"], full["variance_ratio"], rtol=1e-9)
    truth = opca.pca_full_f64(x, dense=False)
    _check(f"chunked k={k}", ch, truth, k)


# ------------------------------------------------------------------------------------------ building blocks
def _awkward_csr(n=3000, g=300, seed=11):
    """Random CSR with one fully dense row (g > 32 entries per row), a run of empty rows and rows whose column indices
    are not sorted."""
    rs = np.random.RandomState(seed)
    d = (rs.rand(n, g) < 0.04) * rs.uniform(0.1, 2.0, (n, g))
    d[7] = rs.uniform(0.1, 2.0, g)
    d[100:140] = 0.0
    x = _csr(d)
    x.sort_indices()
    for r in range(200, 260):
        lo, hi = x.indptr[r], x.indptr[r + 1]
        p = rs.permutation(hi - lo)
        x.indices[lo:hi] = x.indices[lo:hi][p]
        x.data[lo:hi] = x.data[lo:hi][p]
    x.has_sorted_indices = False
    return x


@pytest.mark.parametrize("l", [32, 64, 128])
def test_building_blocks_awkward_rows(l):
    import torch

    x = _awkward_csr()
    assert not x.has_sorted_indices
    n, g = x.shape
    ctx = sb._abi.default_context()
    dp, di, dd = _ops.csr_to_device(x)
    xd = x.astype(np.float64)
    rs = np.random.RandomState(l)
    b = rs.standard_normal((g, l)).astype(np.float32)
    shift = rs.standard_normal(l).astype(np.float32)
    y = torch.empty((n, l), dtype=torch.float32, device="cuda")
    ys = torch.empty((n, l), dtype=torch.float32, device="cuda")
    d_b, d_shift = torch.from_numpy(b).cuda(), torch.from_numpy(shift).cuda()
    sb._abi.check(ctx.lib.sb2_spmm_csr(ctx.handle, n, g, l, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(d_b), None,
                                       _ops.ptr(y)))
    sb._abi.check(ctx.lib.sb2_spmm_csr(ctx.handle, n, g, l, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(d_b),
                                       _ops.ptr(d_shift), _ops.ptr(ys)))
    y_ref = np.asarray(xd @ b.astype(np.float64))
    np.testing.assert_allclose(y.cpu().numpy(), y_ref, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(ys.cpu().numpy(), y_ref - shift, rtol=2e-5, atol=2e-5)
    z = torch.empty((g, l), dtype=torch.float64, device="cuda")
    sb._abi.check(ctx.lib.sb2_spmm_csr_t(ctx.handle, n, g, l, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(y),
                                         _ops.ptr(z)))
    z_ref = np.asarray(xd.T @ y.cpu().numpy().astype(np.float64))
    np.testing.assert_allclose(z.cpu().numpy(), z_ref, rtol=2e-4, atol=2e-3 * np.abs(z_ref).max() * 1e-2)
    gram = torch.empty((g, g), dtype=torch.float64, device="cuda")
    sb._abi.check(ctx.lib.sb2_csr_gram(ctx.handle, n, g, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(gram)))
    np.testing.assert_allclose(gram.cpu().numpy(), (xd.T @ xd).toarray(), rtol=1e-12, atol=1e-9)
    s1 = torch.empty(g, dtype=torch.float64, device="cuda")
    s2 = torch.empty(g, dtype=torch.float64, device="cuda")
    sb._abi.check(ctx.lib.sb2_csr_col_stats(ctx.handle, n, g, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(s1),
                                            _ops.ptr(s2)))
    np.testing.assert_allclose(s1.cpu().numpy(), np.asarray(xd.sum(axis=0)).ravel(), rtol=1e-12)
    np.testing.assert_allclose(s2.cpu().numpy(), np.asarray(xd.multiply(xd).sum(axis=0)).ravel(), rtol=1e-12)
    print(f"\n[building blocks l={l}] X B {np.abs(y.cpu().numpy() - y_ref).max():.2e}, "
          f"X^T Y {np.abs(z.cpu().numpy() - z_ref).max() / np.abs(z_ref).max():.2e} (relative to max)")

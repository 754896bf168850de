"""metrics.morans_i / metrics.gearys_c on the H100: the reference's own tests (tests/test_metrics.py:40-171) on the in-tree
pbmc68k fixtures, the oracle (oracle/autocorr.py) across formats, dtypes and awkward graphs, bit-identity across layouts
and block sizes, and a 200k-cell neighbors graph."""
import warnings
from functools import partial

import numpy as np
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import autocorr as oac
from scanpy_b200 import _autocorr
from scanpy_b200._compat import MiniAnnData

from test_autocorr_cpu import METRICS, pbmc68k_reduced

pytestmark = pytest.mark.gpu

ORACLE = {"gearys_c": oac.gearys_c, "morans_i": oac.morans_i}


@pytest.fixture(params=list(METRICS), ids=list(METRICS))
def name(request):
    return request.param


# ------------------------------------------------------------------------------------------ the reference's tests
def test_consistency(name):
    metric = METRICS[name]
    pbmc = pbmc68k_reduced()
    g = pbmc.obsp["connectivities"]
    eq = partial(np.testing.assert_allclose, atol=1e-11)
    mito = pbmc.obs["percent_mito"]
    eq(metric(g, mito), metric(g, mito))
    eq(metric(g, mito), metric(pbmc, vals=mito))
    eq(metric(g, mito), metric(g, mito.values))
    assert isinstance(metric(g, mito), np.float64)
    eq(metric(pbmc, obsm="X_pca"), metric(g, pbmc.obsm["X_pca"].T))
    all_genes = metric(pbmc, layer="raw")
    first_gene = metric(pbmc, vals=pbmc.layers["raw"][:, 0].toarray().ravel())
    np.testing.assert_allclose(all_genes[0], first_gene, rtol=1e-9)
    eq(metric(pbmc, layer="raw"), metric(pbmc, vals=pbmc.layers["raw"].T.toarray()))
    # and against the oracle
    eq(all_genes, ORACLE[name](g, pbmc.layers["raw"]))


@pytest.mark.parametrize(("name", "size", "expected"), [("gearys_c", 30, 0.0), ("morans_i", 50, 1.0)])
def test_correctness(name, size, expected):
    metric = METRICS[name]
    rng = np.random.default_rng()
    connected = np.zeros(100)
    connected[rng.choice(100, size=size, replace=False)] = 1
    m = connected.astype(bool)
    graph = np.zeros((100, 100))
    graph[np.ix_(m, m)] = 1
    graph[np.ix_(~m, ~m)] = 1
    graph = sparse.csr_matrix(graph)
    np.testing.assert_equal(metric(graph, connected), expected)
    np.testing.assert_equal(metric(graph, connected), metric(graph, sparse.csr_matrix(connected)))


@pytest.mark.parametrize("array_type", [np.asarray, sparse.csr_matrix, sparse.csr_array, sparse.csc_matrix,
                                        sparse.coo_matrix], ids=["numpy", "csr_matrix", "csr_array", "csc", "coo"])
def test_graph_metrics_w_constant_values(name, array_type):
    metric = METRICS[name]
    rng = np.random.default_rng()
    pbmc = pbmc68k_reduced()
    x_t = pbmc.layers["raw"].T.tocsr()
    g = pbmc.obsp["connectivities"].copy()
    eq = partial(np.testing.assert_allclose, atol=1e-11)
    const_inds = rng.choice(x_t.shape[0], 10, replace=False)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", sparse.SparseEfficiencyWarning)
        x_t_zero_vals = x_t.copy()
        x_t_zero_vals[const_inds, :] = 0
        x_t_zero_vals = array_type(x_t_zero_vals.toarray() if array_type is np.asarray else x_t_zero_vals)
        x_t_const_vals = x_t.copy()
        x_t_const_vals[const_inds, :] = 42
        x_t_const_vals = array_type(x_t_const_vals.toarray() if array_type is np.asarray else x_t_const_vals)
    results_full = metric(g, array_type(x_t.toarray() if array_type is np.asarray else x_t))
    with pytest.warns(UserWarning, match=r"10 variables were constant, will return nan for these"):
        results_const_zeros = metric(g, x_t_zero_vals)
    with pytest.warns(UserWarning, match=r"10 variables were constant, will return nan for these"):
        results_const_vals = metric(g, x_t_const_vals)
    assert not np.isnan(results_full).any()
    eq(results_const_zeros, results_const_vals)
    np.testing.assert_array_equal(np.nan, results_const_zeros[const_inds])
    np.testing.assert_array_equal(np.nan, results_const_vals[const_inds])
    non_const = ~np.isin(np.arange(x_t.shape[0]), const_inds)
    eq(results_full[non_const], results_const_zeros[non_const])


@pytest.mark.parametrize(("neigh_params", "metric_params"), [
    pytest.param(dict(key_added="foo"), dict(use_graph="foo_connectivities"), id="use_graph"),
    pytest.param(dict(key_added="bar"), dict(neighbors_key="bar"), id="neighbors_key"),
])
def test_metrics_graph_params(name, neigh_params, metric_params):
    rng = np.random.default_rng()
    adata = MiniAnnData(rng.normal(size=(10, 20)))
    sb.pp.neighbors(adata, **neigh_params)
    if "use_graph" in metric_params:  # make sure no extra stuff is there
        adata = MiniAnnData(adata.X, obsp=adata.obsp)
    r = METRICS[name](adata, **metric_params)
    assert r.shape == (20,)


def test_constant_vector_divides_by_zero(name):
    g = sparse.identity(6, format="csr") + sparse.eye(6, k=1, format="csr")
    with pytest.raises(ZeroDivisionError):
        METRICS[name](g, np.full(6, 3.0))
    assert np.isnan(METRICS[name](g, np.r_[np.nan, np.arange(5.0)]))


# ------------------------------------------------------------------------------------------ the oracle
N, G = 2500, 300  # not multiples of 16, 256 or 1024


def knn_graph(rng):
    idx = rng.integers(0, N, size=(N, 15))
    g = sparse.csr_matrix((rng.uniform(0.05, 1.0, idx.size), idx.ravel(), np.arange(0, idx.size + 1, 15)), shape=(N, N))
    g.sum_duplicates()
    return ((g + g.T) / 2).tocsr()


def directed_graph(rng):
    """Explicit zeros, self-loops, empty rows and one hub row with an arc to every cell."""
    g = sparse.random(N, N, density=6 / N, format="lil", random_state=rng)
    g.setdiag(np.where(np.arange(N) % 5 == 0, 0.7, 0.0))
    g[17, :] = rng.uniform(0.1, 2.0, N)
    g[np.arange(40, 60)] = 0
    g = g.tocsr()
    g.data[::9] = 0.0
    assert (np.diff(g.indptr) == 0).any() and (g.data == 0).any() and np.diff(g.indptr).max() == N
    return g


def negative_graph(rng):
    g = knn_graph(rng)
    g.data = g.data - 0.4
    return g


GRAPHS = {"knn": knn_graph, "directed": directed_graph, "negative": negative_graph}


def values(rng, dtype):
    """N x G with a gene of mean / sd ~ 1e3, a NaN gene (float dtypes) and an all-zero gene."""
    counts = rng.poisson(rng.gamma(0.4, 2.0, G), size=(N, G)) * (rng.random((N, G)) < 0.3)
    counts[:2] += np.array([[1], [2]])  # no gene is constant by chance
    x = counts.astype(np.float64)
    x[:, 5] = 20000 + rng.poisson(400, N) - 400 if np.dtype(dtype).kind in "iu" else 1e3 + rng.standard_normal(N)
    x[:, 9] = 0
    if np.dtype(dtype).kind == "f":
        x[:, 11] = rng.standard_normal(N)
        x[123, 11] = np.nan
        x[:, 13] = rng.standard_normal(N) * 3.7  # non-integer values
    return x.astype(dtype)


FMTS = {"csr": sparse.csr_matrix, "csc": sparse.csc_matrix, "dense": np.asarray}


@pytest.mark.parametrize("graph", list(GRAPHS))
@pytest.mark.parametrize("fmt", list(FMTS))
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64], ids=lambda d: np.dtype(d).name)
def test_oracle_parity(graph, fmt, dtype):
    rng = np.random.default_rng(7)
    g = GRAPHS[graph](rng)
    x = values(rng, dtype)
    vals = FMTS[fmt](x.T)
    for name, metric in METRICS.items():
        with pytest.warns(UserWarning, match="1 variables were constant"):
            got = metric(g, vals)
        want = ORACLE[name](g, x)
        assert np.isnan(got[9]) and (np.isnan(got[11]) if np.dtype(dtype).kind == "f" else np.isfinite(got[11]))
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-11, err_msg=f"{name} {graph} {fmt}")


def test_bit_identical_across_layouts_calls_and_blocks():
    rng = np.random.default_rng(11)
    g = directed_graph(rng)
    x = values(rng, np.float64)
    ref, const = _autocorr.graph_sums(g, sparse.csr_matrix(x))
    for other in (sparse.csc_matrix(x), x, sparse.csr_matrix(x)):
        got, c = _autocorr.graph_sums(g, other)
        assert got.tobytes() == ref.tobytes() and (c == const).all()
    # dense column blocks of 256 genes, graph row blocks of one subtile
    got, c = _autocorr.graph_sums(g, x, dense_bytes=N * 8 * 256, partial_bytes=3 * G * 8)
    assert got.tobytes() == ref.tobytes() and (c == const).all()
    got, c = _autocorr.graph_sums(g, sparse.csr_matrix(x), partial_bytes=3 * G * 8)
    assert got.tobytes() == ref.tobytes()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        for metric in METRICS.values():
            a, b = metric(g, x.T), metric(g, sparse.csr_matrix(x.T))
            assert a.tobytes() == b.tobytes()


def test_neighbors_graph_200k():
    from scanpy_b200._synth import synth_scipy

    x, _ = synth_scipy(200_000, 2000, n_clusters=12, r=32, device="cuda")
    adata = MiniAnnData(x)
    sb.pp.pca(adata, n_comps=30)
    sb.pp.neighbors(adata, n_neighbors=15)
    g = adata.obsp["connectivities"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        got = {name: metric(adata) for name, metric in METRICS.items()}
    genes = np.random.default_rng(0).choice(2000, 64, replace=False)
    xs = x[:, genes]
    for name in METRICS:
        want = ORACLE[name](g, xs)
        np.testing.assert_allclose(got[name][genes], want, rtol=0, atol=1e-11, err_msg=name)

"""CPU tests for metrics.morans_i / metrics.gearys_c: the oracle (oracle/autocorr.py) against a literal transcription of
the reference's per-arc loops (src/scanpy/metrics/_morans_i.py `_morans_i_vec_w`, _gearys_c.py `_gearys_c_vec_w`) and
against exact cases, and the graph and `vals` resolution the public functions do before touching a device."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import autocorr as oac
from scanpy_b200._compat import MiniAnnData, get_arr

from conftest import GOLDEN

METRICS = {"gearys_c": sb.metrics.gearys_c, "morans_i": sb.metrics.morans_i}


def pbmc68k_reduced():
    """The reference's pbmc68k_reduced as far as its metrics tests read it: obsp connectivities, obsm X_pca, the raw
    counts as layer "raw" and obs percent_mito."""
    gr = np.load(GOLDEN / "pbmc68k_reduced_graph.npz")
    h = np.load(GOLDEN / "pbmc68k_raw_seurat_hvg.npz")
    d = np.load(GOLDEN / "pbmc68k_regress.npz")
    conn = sparse.csr_matrix((gr["conn_data"], gr["conn_indices"], gr["conn_indptr"]), shape=(700, 700))
    raw = sparse.csr_matrix((h["raw_data"], h["raw_indices"], h["raw_indptr"]), shape=(700, 765))
    ad = MiniAnnData(raw, obs=pd.DataFrame({"percent_mito": d["percent_mito"]}, index=[f"c{i}" for i in range(700)]),
                     obsm={"X_pca": gr["X_pca"]}, obsp={"connectivities": conn},
                     uns={"neighbors": dict(connectivities_key="connectivities", distances_key="distances")})
    ad.layers["raw"] = raw.copy()
    return ad


def loop_morans_i(g, x):
    """`_morans_i_vec_w`, statement by statement."""
    z = (x - x.mean()).astype(np.float64)
    z2ss = (z * z).sum()
    inum = 0.0
    for i in range(len(x)):
        s = slice(g.indptr[i], g.indptr[i + 1])
        inum += (g.data[s] * z[g.indices[s]]).sum() * z[i]
    return len(x) / g.data.sum() * inum / z2ss


def loop_gearys_c(g, x):
    """`_gearys_c_vec_w`, statement by statement."""
    n = len(g.indptr) - 1
    x = x.astype(np.float64)
    x_bar = x.mean()
    total = 0.0
    for i in range(n):
        s = slice(g.indptr[i], g.indptr[i + 1])
        total += np.sum(g.data[s] * ((x[i] - x[g.indices[s]]) ** 2))
    return (n - 1) * total / (2 * g.data.sum() * ((x - x_bar) ** 2).sum())


def odd_graph(n, rng):
    """Directed, with explicit zeros, self-loops, empty rows, negative weights and a hub row."""
    g = sparse.random(n, n, density=0.05, format="lil", random_state=rng)
    g[np.arange(0, n, 7), np.arange(0, n, 7)] = 0.5
    g[3, :] = rng.standard_normal(n)
    g[5, :] = 0
    g = g.tocsr()
    g.data[::11] = 0.0
    g.data[::13] *= -1
    assert (np.diff(g.indptr) == 0).any() and (g.data == 0).any()
    return g


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_matches_the_per_arc_loops(seed):
    rng = np.random.default_rng(seed)
    n, g = 90, 7
    graph = odd_graph(n, rng)
    x = rng.standard_normal((n, g)) * rng.uniform(0.1, 10, g) + rng.uniform(-5, 5, g)
    x[:, 2] = np.where(rng.random(n) < 0.7, 0.0, x[:, 2])
    x[:, 3] = 1e3 + rng.standard_normal(n)
    want_i = [loop_morans_i(graph, x[:, j]) for j in range(g)]
    want_c = [loop_gearys_c(graph, x[:, j]) for j in range(g)]
    np.testing.assert_allclose(oac.morans_i(graph, x), want_i, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(oac.gearys_c(graph, x), want_c, rtol=1e-10, atol=1e-12)


def test_oracle_constant_and_nan_features():
    rng = np.random.default_rng(2)
    graph = odd_graph(40, rng)
    x = rng.standard_normal((40, 4))
    x[:, 1] = 42.0
    x[:, 2] = 0.0
    x[5, 3] = np.nan
    for fn in (oac.morans_i, oac.gearys_c):
        r = fn(graph, x)
        assert np.isnan(r[1:]).all() and np.isfinite(r[0])
    _, _, _, constant = oac.sums(graph, x)
    assert constant.tolist() == [False, True, True, False]


@pytest.mark.parametrize(("fn", "size", "expected"), [(oac.gearys_c, 30, 0.0), (oac.morans_i, 50, 1.0)])
def test_oracle_perfectly_separated_groups(fn, size, expected):
    """The reference's test_correctness: two cliques, the indicator of one of them."""
    rng = np.random.default_rng(3)
    connected = np.zeros(100)
    connected[rng.choice(100, size=size, replace=False)] = 1
    m = connected.astype(bool)
    graph = np.zeros((100, 100))
    graph[np.ix_(m, m)] = 1
    graph[np.ix_(~m, ~m)] = 1
    np.testing.assert_equal(fn(sparse.csr_matrix(graph), connected[:, None])[0], expected)


# ------------------------------------------------------------------------------------------ resolution, before the device
@pytest.mark.parametrize("metric", METRICS.values(), ids=METRICS.keys())
@pytest.mark.parametrize(("params", "err_cls", "pattern"), [
    pytest.param(dict(use_graph="foo", neighbors_key="bar"), TypeError, r"both", id="both"),
    pytest.param(dict(use_graph="foo"), KeyError, r"foo", id="no_graph"),
    pytest.param(dict(neighbors_key="bar"), KeyError, r"bar", id="no_key"),
    pytest.param({}, KeyError, r"neighbors.*uns", id="nothing"),
])
def test_metrics_graph_params_errors(metric, params, err_cls, pattern):
    """The reference's test_metrics_graph_params_errors, on a MiniAnnData."""
    adata = MiniAnnData(np.zeros((10, 20)))
    with pytest.raises(err_cls, match=pattern):
        metric(adata, **params)


@pytest.mark.parametrize("metric", METRICS.values(), ids=METRICS.keys())
def test_graph_resolution(metric):
    adata = MiniAnnData(np.zeros((10, 20)), uns={"neighbors": {"params": {}}})
    with pytest.raises(ValueError, match="Must run neighbors first."):
        metric(adata)
    adata.uns["bar"] = dict(connectivities_key="bar_connectivities")
    with pytest.raises(ValueError, match="Must run neighbors first."):
        metric(adata, neighbors_key="bar")
    with pytest.raises(TypeError, match="Cannot specify both `use_graph` and `neighbors_key`."):
        metric(adata, use_graph="x", neighbors_key="bar")


def test_graph_connectivities_fall_back_to_uns():
    from scanpy_b200.metrics import _get_graph

    g = sparse.identity(10, format="csr")
    adata = MiniAnnData(np.zeros((10, 20)), uns={"neighbors": {"connectivities": g}})
    assert _get_graph(adata, use_graph=None, neighbors_key=None) is g
    adata.obsp["connectivities"] = h = sparse.identity(10, format="csr")
    assert _get_graph(adata, use_graph=None, neighbors_key="neighbors") is h
    adata.uns["k"] = dict(connectivities_key="kc")
    adata.obsp["kc"] = g
    assert _get_graph(adata, use_graph=None, neighbors_key="k") is g
    assert _get_graph(adata, use_graph="kc", neighbors_key=None) is g


def test_get_arr_choices_and_messages():
    adata = MiniAnnData(np.zeros((4, 3)), obsm={"m": np.ones((4, 2))}, obsp={"p": np.eye(4)})
    adata.layers["l"] = np.full((4, 3), 2.0)
    assert get_arr(adata) is adata.X
    assert get_arr(adata, layer="l") is adata.layers["l"]
    assert get_arr(adata, obsm="m") is adata.obsm["m"]
    assert get_arr(adata, obsp="p") is adata.obsp["p"]
    with pytest.raises(ValueError, match=r"^Only one of `layer`, or `obsm` can be specified\.$"):
        get_arr(adata, layer="l", obsm="m")
    with pytest.raises(ValueError, match=r"^Only one of `use_raw`, `layer`, or `obsp` can be specified\.$"):
        get_arr(adata, use_raw=True, layer="l", obsp="p")
    with pytest.raises(TypeError, match="use_raw expected to be bool"):
        get_arr(adata, use_raw=1)


@pytest.mark.parametrize("metric", METRICS.values(), ids=METRICS.keys())
def test_vals_and_graph_rejections(metric):
    g = sparse.identity(6, format="csr")
    with pytest.raises(TypeError, match="Unsupported type"):
        metric(g, [1.0, 2.0, 3.0, 4.0, 5.0, 6.0])
    with pytest.raises(NotImplementedError, match="ndim 3"):
        metric(g, np.zeros((2, 3, 6)))
    with pytest.raises(TypeError, match="CSR"):
        metric(g.tocsc(), np.arange(6.0))
    with pytest.raises(AssertionError, match="square"):
        metric(sparse.csr_matrix((6, 5)), np.arange(6.0))
    with pytest.raises(AssertionError):
        metric(g, np.arange(5.0))
    with pytest.raises(AssertionError):
        metric(g, np.zeros((2, 5)))
    with pytest.raises(ValueError, match="Only one of `layer`, or `obsm` can be specified."):
        metric(MiniAnnData(np.zeros((6, 2)), obsp={"connectivities": g},
                           uns={"neighbors": dict(connectivities_key="connectivities")}), layer="a", obsm="b")


def test_pbmc_fixture_shapes():
    ad = pbmc68k_reduced()
    assert ad.obsp["connectivities"].shape == (700, 700) and ad.layers["raw"].shape == (700, 765)
    assert ad.obs["percent_mito"].shape == (700,)

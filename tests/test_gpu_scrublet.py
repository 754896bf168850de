"""sc.pp.scrublet on the H100: the doublet sums bit-identical to scipy, the exact label count against the fp64 oracle
(oracle/scrublet.py) across data kinds and shapes, and the whole call on the pbmc68k counts against the oracle's
restatement of the reference path, batched and with each option."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import scrublet as osc
from scanpy_b200 import _ops, _scrublet
from scanpy_b200._compat import LegacyRng, MiniAnnData
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


def counts():
    return ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts").tocsr().astype(np.float32)


def pbmc(x=None, obs=None):
    x = counts() if x is None else x
    return MiniAnnData(x, obs=obs if obs is not None else pd.DataFrame(index=[f"c{i}" for i in range(x.shape[0])]))


def assert_csr_bits(got, ref):
    ref = ref.tocsr()
    np.testing.assert_array_equal(got.indptr, ref.indptr)
    np.testing.assert_array_equal(got.indices, ref.indices)
    np.testing.assert_array_equal(got.data.view(np.uint32), ref.data.astype(np.float32).view(np.uint32))


# ------------------------------------------------------------------------------------------ pair sums
@pytest.mark.parametrize("rng", [LegacyRng(0), np.random.default_rng(11)], ids=["legacy", "rng"])
def test_pair_sums_pbmc_bit_identical(rng):
    x = counts()
    sim, pairs, n_counts = _scrublet.simulate(x, 2.0, rng)
    assert pairs.shape == (1400, 2)
    assert_csr_bits(sim, x[pairs[:, 0]] + x[pairs[:, 1]])
    np.testing.assert_array_equal(n_counts, np.asarray(x.sum(1)).ravel()[pairs[:, 0]] + np.asarray(x.sum(1)).ravel()[pairs[:, 1]])


def test_pair_sums_adversarial_rows():
    rs = np.random.default_rng(0)
    g = 30_000
    rows = [
        sparse.csr_matrix((1, g), dtype=np.float32),                                         # empty
        sparse.csr_matrix((rs.random(20_000).astype(np.float32) + 1, (np.zeros(20_000, int),
                                                                       np.sort(rs.choice(g, 20_000, replace=False)))),
                          shape=(1, g)),                                                     # 20k stored values
        sparse.csr_matrix((np.array([0, 2, 0, -3], np.float32), ([0, 0, 0, 0], [1, 5, 9, 12])), shape=(1, g)),  # stored 0
        sparse.csr_matrix((np.array([1, 3, np.nan], np.float32), ([0, 0, 0], [5, 12, 40])), shape=(1, g)),  # cancels
        sparse.csr_matrix((rs.random(20_000).astype(np.float32), (np.zeros(20_000, int),
                                                                   np.sort(rs.choice(g, 20_000, replace=False)))),
                          shape=(1, g)),
    ]
    x = sparse.vstack(rows).tocsr()
    x.has_canonical_format = True
    pairs = np.array([[0, 0], [0, 1], [1, 0], [1, 1], [2, 3], [3, 2], [2, 2], [1, 4], [4, 1], [3, 0], [0, 2]])

    class Fixed:  # a generator whose choice returns the flat indices of the pairs above
        def choice(self, n, size, replace):
            return pairs[:, 0] * x.shape[0] + pairs[:, 1]

    sim, got_pairs, _ = _scrublet.simulate(x, len(pairs) / x.shape[0], Fixed())
    np.testing.assert_array_equal(got_pairs, pairs)
    ref = x[pairs[:, 0]] + x[pairs[:, 1]]
    assert_csr_bits(sim, ref)
    assert sim[4].nnz == 2  # rows 2 + 3: 2 + 1 and 0 + nan stay; the stored zeros and -3 + 3 drop
    assert sim[0].nnz == 0


# ------------------------------------------------------------------------------------------ label count
def points(kind, n, d, seed=0):
    rs = np.random.default_rng(seed)
    if kind == "uniform":
        return rs.random((n, d), dtype=np.float32)
    if kind == "clustered":
        centres = rs.normal(0, 10, (8, d))
        return (centres[rs.integers(0, 8, n)] + rs.normal(0, 0.3, (n, d))).astype(np.float32)
    if kind == "grid":  # integer lattice: mass ties of the distances
        return rs.integers(-3, 4, (n, d)).astype(np.float32)
    if kind == "duplicates":  # every point twice, as the doublets (i, j) and (j, i) are
        half = rs.normal(0, 1, ((n + 1) // 2, d)).astype(np.float32)
        return np.repeat(half, 2, axis=0)[:n][rs.permutation(n)]
    raise ValueError(kind)


def check_label_count(x, n_first, k):
    import torch

    count, kth, ids = _scrublet.label_count(torch.from_numpy(x).cuda(), n_first, k, with_ids=True)
    ocount, okth, oids, _ = osc.label_count(x, n_first, k)
    np.testing.assert_array_equal(count, ocount)
    np.testing.assert_array_equal(kth, okth)
    np.testing.assert_array_equal(ids[:, 0], np.arange(x.shape[0]))
    np.testing.assert_array_equal(np.sort(ids, axis=1), np.sort(oids, axis=1))


@pytest.mark.parametrize("kind", ["uniform", "clustered", "grid", "duplicates"])
@pytest.mark.parametrize("k", [1, 2, 57, 150])
def test_label_count_kinds(kind, k):
    check_label_count(points(kind, 1111, 30, seed=k), 400, k)


@pytest.mark.parametrize("d", [1, 30, 150])
def test_label_count_dims(d):
    check_label_count(points("clustered", 1283, d, seed=d), 500, 40)


@pytest.mark.parametrize("k", [1024, 1100])
def test_label_count_large_k(k):
    check_label_count(points("uniform", 1100, 8, seed=3), 300, k)


def test_label_count_band_overflow():
    # 2000 points on 9 lattice sites: hundreds of equal distances at every threshold, far more than the band holds
    x = np.random.default_rng(5).integers(0, 3, (2000, 2)).astype(np.float32)
    check_label_count(x, 700, 150)


def test_label_count_refuses_out_of_range():
    import torch

    from scanpy_b200._abi import B200Error

    x = points("uniform", 100, 4)
    x[3, 1] = np.inf
    with pytest.raises(B200Error, match="finite"):
        _scrublet.label_count(torch.from_numpy(x).cuda(), 50, 5)


# ------------------------------------------------------------------------------------------ end to end
def oracle_run(x, *, rng, sim_doublet_ratio=2.0, log_transform=False, **kw):
    x_obs, x_sim, parents, keep = osc.preprocess(x, sim_doublet_ratio=sim_doublet_ratio, log_transform=log_transform,
                                                 rng=rng)
    return osc.call_doublets(x_obs, x_sim, parents, **kw), parents, keep


def assert_scores_match(got_scores, res, what=""):
    """Scores equal to the oracle's; a row may differ only where the oracle's (k-1)-th and k-th neighbours are within
    1e-5 of each other (relative), and such rows are reported."""
    n_obs = len(res["doublet_score"])
    diff = np.flatnonzero(got_scores != res["doublet_score"])
    near = res["gap"][:n_obs] < 1e-5
    assert np.all(near[diff]), f"{what}: rows {diff[~near[diff]][:10]} differ without a near-tie"
    if len(diff):
        print(f"{what}: {len(diff)} rows differ at near-ties (gap < 1e-5)")
    return diff


def test_pbmc_end_to_end():
    adata = pbmc()
    sb.pp.scrublet(adata)
    res, parents, keep = oracle_run(counts(), rng=LegacyRng(0))
    assert len(keep) == adata.n_obs and res["k_adj"] == 39
    uns = adata.uns["scrublet"]
    np.testing.assert_array_equal(uns["doublet_parents"], parents)
    diff = assert_scores_match(adata.obs["doublet_score"].to_numpy(), res, "pbmc")
    if len(diff) == 0:
        np.testing.assert_array_equal(uns["doublet_scores_sim"], res["doublet_scores_sim"])
        np.testing.assert_array_equal(adata.obs["predicted_doublet"].to_numpy(), res["predicted_doublet"])
        assert uns.get("threshold") == res["threshold"]
    assert uns["parameters"] == dict(expected_doublet_rate=0.05, sim_doublet_ratio=2.0, n_neighbors=13, random_state=0)
    assert adata.obs["predicted_doublet"].dtype == bool


def test_bit_identical_across_calls():
    a, b = pbmc(), pbmc()
    sb.pp.scrublet(a, get_doublet_neighbor_parents=True)
    sb.pp.scrublet(b, get_doublet_neighbor_parents=True)
    np.testing.assert_array_equal(a.obs["doublet_score"].to_numpy(), b.obs["doublet_score"].to_numpy())
    np.testing.assert_array_equal(a.uns["scrublet"]["doublet_scores_sim"], b.uns["scrublet"]["doublet_scores_sim"])
    for u, v in zip(a.uns["scrublet"]["doublet_neighbor_parents"], b.uns["scrublet"]["doublet_neighbor_parents"]):
        np.testing.assert_array_equal(u, v)


@pytest.mark.parametrize("kw", [
    dict(mean_center=False), dict(normalize_variance=False), dict(mean_center=False, normalize_variance=False),
    dict(log_transform=True), dict(n_prin_comps=10), dict(threshold=0.2), dict(get_doublet_neighbor_parents=True),
    dict(n_neighbors=20, expected_doublet_rate=0.1),
], ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()))
def test_options_against_oracle(kw):
    adata = pbmc()
    sb.pp.scrublet(adata, rng=5, **kw)
    okw = {k: v for k, v in kw.items() if k != "get_doublet_neighbor_parents"}
    res, parents, _ = oracle_run(counts(), rng=np.random.default_rng(5), **okw)
    uns = adata.uns["scrublet"]
    np.testing.assert_array_equal(uns["doublet_parents"], parents)
    assert "random_state" not in uns["parameters"]
    diff = assert_scores_match(adata.obs["doublet_score"].to_numpy(), res, str(kw))
    if "threshold" in kw:
        assert uns["threshold"] == kw["threshold"]
        np.testing.assert_array_equal(adata.obs["predicted_doublet"].to_numpy(),
                                      adata.obs["doublet_score"].to_numpy() > kw["threshold"])
    if kw.get("get_doublet_neighbor_parents") and len(diff) == 0:
        for u, v in zip(uns["doublet_neighbor_parents"], res["doublet_neighbor_parents"]):
            np.testing.assert_array_equal(u, v)


def test_batched_each_batch_equals_its_own_run():
    x = counts()
    rs = np.random.default_rng(0)
    # three rows of fewer than three genes: dropped by the internal filter_cells, NaN in the result
    low = sparse.csr_matrix((np.ones(3, np.float32), ([0, 1, 1], [0, 5, 6])), shape=(3, x.shape[1]))
    x = sparse.vstack([x, low]).tocsr()
    batch = pd.Categorical(rs.choice(["s1", "s2", "s3"], x.shape[0]), categories=["s3", "s1", "s2"])
    names = [f"c{i % 500}" for i in range(x.shape[0])]  # duplicate obs_names
    obs = pd.DataFrame({"sample": batch}, index=names)
    adata = pbmc(x, obs)
    sb.pp.scrublet(adata, batch_key="sample")
    assert list(adata.obs_names if hasattr(adata, "obs_names") else adata.obs.index) == names
    assert isinstance(adata.obs["sample"].dtype, pd.CategoricalDtype)
    assert adata.uns["scrublet"]["batched_by"] == "sample"
    assert set(adata.uns["scrublet"]["batches"]) == {"s1", "s2", "s3"}
    score = adata.obs["doublet_score"].to_numpy()
    assert np.isnan(score[-3:]).all() and not np.isnan(score[:-3]).any()
    for b in ["s1", "s2", "s3"]:
        sel = np.flatnonzero(batch == b)
        one = pbmc(x[sel], pd.DataFrame(index=[names[i] for i in sel]))
        sb.pp.scrublet(one)
        np.testing.assert_array_equal(score[sel], one.obs["doublet_score"].to_numpy())
        np.testing.assert_array_equal(adata.uns["scrublet"]["batches"][b]["doublet_scores_sim"],
                                      one.uns["scrublet"]["doublet_scores_sim"])


def test_batched_rng_streams_are_spawned():
    x = counts()
    batch = np.repeat(["a", "b"], [350, 350])
    adata = pbmc(x, pd.DataFrame({"batch": batch}, index=[f"c{i}" for i in range(700)]))
    sb.pp.scrublet(adata, batch_key="batch", rng=9)
    subs = np.random.default_rng(9).spawn(2)
    for b, sub in zip(["a", "b"], subs):
        res, parents, _ = oracle_run(x[np.flatnonzero(batch == b)], rng=sub)
        np.testing.assert_array_equal(adata.uns["scrublet"]["batches"][b]["doublet_parents"], parents)


def test_simulate_then_call_equals_one_call():
    # tests/test_scrublet.py's test_scrublet_data, restated with this package's preprocessing
    x = counts()
    one = pbmc()
    sb.pp.scrublet(one)
    ad = pbmc()
    sb.pp.filter_genes(ad, min_cells=3)
    sb.pp.filter_cells(ad, min_genes=3)
    raw = ad.X.copy()
    sb.pp.normalize_total(ad)
    logged = MiniAnnData(ad.X.copy())
    sb.pp.log1p(logged)
    sb.pp.highly_variable_genes(logged)
    hvg = logged.var["highly_variable"].to_numpy()
    obs = MiniAnnData(ad.X[:, hvg], layers={"raw": raw[:, hvg]})
    sim = sb.pp.scrublet_simulate_doublets(obs, layer="raw")
    assert sim.X.shape == (2 * x.shape[0], int(hvg.sum()))
    assert sim.uns["scrublet"]["parameters"] == {"sim_doublet_ratio": 2.0}
    sb.pp.normalize_total(obs, target_sum=1e6)
    sb.pp.normalize_total(sim, target_sum=1e6)
    sb.pp.scrublet(obs, adata_sim=sim)
    np.testing.assert_allclose(obs.obs["doublet_score"].to_numpy(), one.obs["doublet_score"].to_numpy(), atol=1e-15)
    np.testing.assert_array_equal(obs.uns["scrublet"]["doublet_parents"], one.uns["scrublet"]["doublet_parents"])


def test_copy_leaves_input():
    adata = pbmc()
    out = sb.pp.scrublet(adata, copy=True)
    assert "doublet_score" not in adata.obs and "scrublet" not in adata.uns
    assert "doublet_score" in out.obs


def test_large_sample_against_exact_knn():
    """One seeded 12k-cell negative-binomial sample (36k points, past the reference's 8192-point switch to approximate
    neighbours): the device's label counts on its embedding equal the exact fp64 count on sampled rows."""
    rs = np.random.default_rng(12)
    n, g = 12_000, 2000
    mu = np.exp(rs.normal(-1.0, 1.2, g)) * rs.choice([0.5, 1.0, 2.0], (6, 1))[rs.integers(0, 6, n)][:, 0:1]
    xd = rs.negative_binomial(2, 2 / (2 + mu)).astype(np.float32)
    x = sparse.csr_matrix(xd)
    x_obs, x_sim, parents, _ = osc.preprocess(x, rng=LegacyRng(0))
    n_obs, n_sim = x_obs.shape[0], x_sim.shape[0]
    k_adj = _scrublet.k_adjusted(_scrublet.n_neighbors_default(n_obs), n_obs, n_sim)
    emb = _scrublet.manifold(x_obs, x_sim, mean_center=True, normalize_variance=True, n_prin_comps=30)
    count, kth, _ = _scrublet.label_count(emb, n_obs, k_adj)
    host = _ops._to_host(emb)
    rows = np.random.default_rng(1).choice(n_obs + n_sim, 64, replace=False)
    ocount, okth, _, _ = osc.label_count(host, n_obs, k_adj, rows=rows)
    np.testing.assert_array_equal(count[rows], ocount)
    np.testing.assert_array_equal(kth[rows], okth)

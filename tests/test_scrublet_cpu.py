"""sc.pp.scrublet host logic without a device: the parent-pair streams, the restated threshold_minimum, the score formula
against the reference's literals, the neighbour-count rounding, option refusals and the oracle's own pieces."""
import numpy as np
import pytest
from scipy import sparse

from oracle import scrublet as osc
from scanpy_b200 import _scrublet
from scanpy_b200._compat import LegacyRng, MiniAnnData


def test_parent_pairs_legacy_literal():
    # tests/test_scrublet.py:267-286 of the reference: n_obs = 200, sim_doublet_ratio = 0.02, default random_state 0
    pairs = _scrublet.sample_comb(200, int(200 * 0.02), LegacyRng(0))
    np.testing.assert_array_equal(pairs, [[13, 132], [106, 43], [152, 3], [160, 103]])


def test_parent_pairs_rng_stream():
    got = _scrublet.sample_comb(300, 600, np.random.default_rng(7))
    idx = np.random.default_rng(7).choice(300 * 300, size=600, replace=False)
    np.testing.assert_array_equal(got, np.stack([idx // 300, idx % 300], axis=1))
    assert len({tuple(p) for p in got}) == 600


def test_parent_pairs_spawned_per_batch():
    subs = np.random.default_rng(3).spawn(3)
    ref = np.random.default_rng(3).spawn(3)
    for n, a, b in zip((50, 70, 90), subs, ref):
        idx = b.choice(n * n, size=2 * n, replace=False)
        np.testing.assert_array_equal(_scrublet.sample_comb(n, 2 * n, a), np.stack([idx // n, idx % n], axis=1))


def _values_with_hist(counts):
    """Values on [0, 255] whose 256-bin histogram is `counts` (bin i holds value i)."""
    return np.repeat(np.arange(256, dtype=np.float64), counts)


def test_threshold_minimum_two_modes():
    # two triangles peaking at bins 64 and 192 with the valley at bin 128 (one added everywhere keeps the range [0, 255]);
    # one smoothing step leaves the two peaks and makes bin 128 the unique minimum between them
    i = np.arange(256)
    counts = np.where(i < 128, 64 - np.abs(i - 64), 64 - np.abs(i - 192)) + 1
    t = _scrublet.threshold_minimum(_values_with_hist(counts))
    assert t == (128 + 0.5) * 255 / 256


def test_threshold_minimum_plateau_counts_once():
    # the triangles of the test above with flat tops 47 bins wide: each plateau is one maximum, the valley stays at 128
    i = np.arange(256)
    counts = np.minimum(np.where(i < 128, 64 - np.abs(i - 64), 64 - np.abs(i - 192)), 40) + 1
    assert _scrublet.threshold_minimum(_values_with_hist(counts)) == (128 + 0.5) * 255 / 256
    assert _scrublet._local_maxima(np.array([0, 5, 5, 5, 0, 3, 0], float)) == [3, 5]


def test_threshold_minimum_one_mode_fails():
    x = np.arange(256)
    counts = (100 * np.exp(-((x - 128) / 30.0) ** 2)).astype(int) + 1
    with pytest.raises(RuntimeError, match="two maxima"):
        _scrublet.threshold_minimum(_values_with_hist(counts))


def test_threshold_minimum_iteration_limit():
    # the two-triangle histogram needs one smoothing step; stopping on the last allowed step is a failure, as in skimage
    i = np.arange(256)
    counts = np.where(i < 128, 64 - np.abs(i - 64), 64 - np.abs(i - 192)) + 1
    with pytest.raises(RuntimeError, match="Maximum iteration"):
        _scrublet.threshold_minimum(_values_with_hist(counts), max_num_iter=1)
    assert _scrublet.threshold_minimum(_values_with_hist(counts), max_num_iter=2) == (128 + 0.5) * 255 / 256
    # many modes that one step cannot merge: the maxima test fails first
    wavy = (100 * (1 + np.sin(i / 4.0))).astype(int) + 1
    with pytest.raises(RuntimeError, match="two maxima"):
        _scrublet.threshold_minimum(_values_with_hist(wavy), max_num_iter=1)


def test_score_formula_reference_literals():
    # tests/test_scrublet.py:40 (pbmc200: n_obs 200, k 7, k_adj 21) and :79 (batches of 100: k 5, k_adj 15)
    ld, _ = _scrublet.doublet_scores(np.array([19]), k_adj=21, n_obs=200, n_sim=400, expected_doublet_rate=0.05,
                                     stdev_doublet_rate=0.02)
    np.testing.assert_allclose(ld, [0.149254], atol=1e-6)
    ld, se = _scrublet.doublet_scores(np.array([13, 14]), k_adj=15, n_obs=100, n_sim=200, expected_doublet_rate=0.05,
                                      stdev_doublet_rate=0.02)
    np.testing.assert_allclose(ld, [0.109375, 0.164835], atol=1e-6)
    assert (se > 0).all()


def test_neighbour_count_rounding():
    assert _scrublet.n_neighbors_default(200) == 7
    assert _scrublet.n_neighbors_default(100) == 5
    assert _scrublet.k_adjusted(7, 200, 400) == 21
    assert _scrublet.n_neighbors_default(10_000) == 50 and _scrublet.k_adjusted(50, 10_000, 20_000) == 150
    assert _scrublet.n_neighbors_default(100_000) == 158 and _scrublet.k_adjusted(158, 100_000, 200_000) == 474
    assert _scrublet.n_neighbors_default(700) == 13 and _scrublet.k_adjusted(13, 700, 1400) == 39


def test_neighbor_parents():
    parents = np.array([[0, 1], [2, 1], [3, 3], [0, 0]])
    ids = np.array([[0, 4, 1, 5], [1, 0, 2, 3], [0, 1, 0, 1]])   # n_obs = 2: id 2 + j is doublet j
    got = _scrublet.neighbor_parents(ids, parents, 2)
    assert len(got) == 2
    np.testing.assert_array_equal(got[0], [0, 3])
    np.testing.assert_array_equal(got[1], [0, 1, 2])
    assert _scrublet.neighbor_parents(np.array([[0, 1], [1, 0]]), parents, 2)[0].size == 0


@pytest.mark.parametrize("kw, text", [
    (dict(knn_dist_metric="cosine"), "knn_dist_metric='cosine'"),
    (dict(use_approx_neighbors=True), "use_approx_neighbors=True"),
    (dict(synthetic_doublet_umi_subsampling=0.5), "synthetic_doublet_umi_subsampling=0.5"),
])
def test_refused_options(kw, text):
    adata = MiniAnnData(sparse.random(20, 30, density=0.3, format="csr", random_state=0))
    with pytest.raises(NotImplementedError, match=text.replace("(", r"\(")):
        _scrublet.scrublet(adata, **kw)
    assert "doublet_score" not in adata.obs


def test_batch_key_missing():
    adata = MiniAnnData(sparse.random(20, 30, density=0.3, format="csr", random_state=0))
    with pytest.raises(ValueError, match="`batch_key` must be a column of .obs"):
        _scrublet.scrublet(adata, batch_key="sample")


def test_rng_and_random_state_exclusive():
    with pytest.raises(TypeError, match="at most one"):
        _scrublet.scrublet(MiniAnnData(sparse.eye(5, format="csr")), random_state=0, rng=1)


def test_oracle_label_count_order_and_gap():
    x = np.array([[0.0], [1.0], [1.0], [3.0], [-1.0]])
    count, kth, ids, gap = osc.label_count(x, 3, 3)
    # point 0: others at squared distances 1 (ids 1, 2, 4) and 9; the two nearest by (distance, id) are 1, 2
    np.testing.assert_array_equal(ids[0], [0, 1, 2])
    assert count[0] == 0 and kth[0] == 1.0 and gap[0] == 0.0
    # point 3: nearest others 1, 2 (squared 4), then 0 (9)
    np.testing.assert_array_equal(ids[3], [3, 1, 2])
    assert count[3] == 1 and np.isclose(gap[3], 5 / 9)


def test_oracle_simulate_matches_scipy_sum():
    x = sparse.random(40, 25, density=0.3, format="csr", random_state=1, dtype=np.float32)
    sim, pairs = osc.simulate(x, 2.0, np.random.default_rng(0))
    ref = x[pairs[:, 0]] + x[pairs[:, 1]]
    assert (abs(sim - ref)).nnz == 0 and sim.shape == (80, 25)

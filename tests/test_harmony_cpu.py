"""Host-side contracts of `pp.harmony_integrate` (no GPU): the oracle pinned to the reference's own outputs, the
oracle's k-means start against live sklearn, and the reference's host-only cases (batch codes, theta, lambda, the
multi-key correction, validation and warnings) restated against scanpy_b200/_harmony.py."""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import pandas as pd
import pytest

from oracle import harmony as oh
from scanpy_b200 import _harmony as hm
from scanpy_b200._compat import MiniAnnData

GOLDEN = Path(__file__).resolve().parent / "golden"
SENT = hm.SUPPRESS_PENALTY


def pbmc68k():
    """X_pca (700 x 50) and obs with bulk_labels and the reference test's batch2."""
    g = np.load(GOLDEN / "harmony_pbmc68k.npz")
    x = np.load(GOLDEN / "pbmc68k_reduced_graph.npz")["X_pca"]
    bulk = np.load(GOLDEN / "pbmc68k_regress.npz")["bulk_labels_codes"].astype(np.int64)
    obs = pd.DataFrame({"bulk_labels": pd.Categorical.from_codes(bulk, [f"b{i}" for i in range(bulk.max() + 1)]),
                        "batch2": np.array(["A", "B", "C"])[g["batch2_codes"]]})
    return x, obs, g


def golden_cases():
    x, obs, g = pbmc68k()
    return {case: p for case, p in json.loads(str(g["params"])).items()}


def case_args(p: dict) -> dict:
    p = dict(p)
    p.pop("keys")
    flavor = p.pop("flavor")
    return dict(p, stabilized_penalty=flavor == "harmony2", dynamic_lambda=flavor == "harmony2")


@pytest.mark.parametrize("case", list(golden_cases()))
def test_oracle_reproduces_reference(case):
    x, obs, g = pbmc68k()
    p = golden_cases()[case]
    codes, n_levels = hm.get_batch_codes(obs, p["keys"])
    z, its = oh.harmony(x.astype(np.float64), codes, n_levels, centers=g[f"{case}/centers"], **case_args(p))
    assert its == g[f"{case}/iters"].tolist()
    assert np.abs(z[g["rows"]] - g[f"{case}/out"]).max() <= 1e-10 * np.abs(x).max()


@pytest.mark.parametrize("n_clusters", [2, 23, 50])
def test_oracle_kmeans_start_matches_sklearn(n_clusters):
    from sklearn.cluster import KMeans

    x, _, _ = pbmc68k()
    z = x.astype(np.float64)
    z /= np.linalg.norm(z, axis=1, keepdims=True)
    gen = np.random.default_rng(0)
    want = KMeans(n_clusters, random_state=hm.spawn_random_state(gen), max_iter=25).fit(z).cluster_centers_
    got, _ = oh.kmeans_start(z, n_clusters, hm.spawn_random_state(np.random.default_rng(0)))
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def repeated_points(n=5000, d=64, distinct=40, seed=0):
    """`distinct` points repeated to n rows: ± pairs of sign vectors / 8, so the rows have norm 1, the mean is 0 and
    every squared distance is exact in float64 whatever the order of its sums.  k-means++ then reaches a potential of
    exactly 0, and Lloyd sees clusters without points."""
    rng = np.random.default_rng(seed)
    s = rng.choice([-0.125, 0.125], size=(distinct // 2, d))
    pts = np.vstack([s, -s])
    return pts[rng.permutation(np.resize(np.arange(distinct), n))]


def test_oracle_kmeans_start_with_fewer_distinct_points_than_clusters():
    """Zero potential in k-means++ and clusters that Lloyd leaves empty, where sklearn skips the relocation and warns."""
    from sklearn.cluster import KMeans
    from sklearn.exceptions import ConvergenceWarning

    x = repeated_points()
    with pytest.warns(ConvergenceWarning, match="distinct clusters"):
        want = KMeans(64, random_state=hm.spawn_random_state(np.random.default_rng(2)), max_iter=25).fit(x)
    got, _ = oh.kmeans_start(x, 64, hm.spawn_random_state(np.random.default_rng(2)))
    np.testing.assert_array_equal(got, want.cluster_centers_)


def test_golden_kmeans_centres_are_sklearns():
    """The recorded centres are sklearn's from the spawned stream of rng=0 on the normalised X_pca."""
    x, _, g = pbmc68k()
    z = x.astype(np.float64)
    z /= np.maximum(np.linalg.norm(z, axis=1, keepdims=True), 1e-12)
    got, _ = oh.kmeans_start(z, 23, hm.spawn_random_state(np.random.default_rng(0)))
    np.testing.assert_allclose(got, g["harmony2/centers"], rtol=0, atol=1e-12)


def test_spawn_does_not_advance_parent():
    a, b = np.random.default_rng(5), np.random.default_rng(5)
    hm.spawn_random_state(a)
    np.testing.assert_array_equal(a.permutation(100), b.permutation(100))


@pytest.mark.parametrize(("prop", "want"), [(0.05, 19), (0.1, 9), (1.0, 1), (0.3, 3)])
def test_block_count_is_float_floor_division(prop, want):
    assert hm.n_blocks_of(10_000, prop) == want
    assert hm.n_blocks_of(5, 0.05) == 5


@pytest.mark.parametrize(("n", "blocks"), [(103, 19), (700, 19), (19, 19), (50, 9)])
def test_block_bounds_follow_array_split(n, blocks):
    want = np.cumsum([0] + [len(a) for a in np.array_split(np.arange(n), blocks)])
    np.testing.assert_array_equal(hm.block_bounds(n, blocks), want)


def test_batch_codes_and_theta():
    obs = pd.DataFrame({"batch": pd.Categorical(["b0", "b1", "b2", "b3", "b4", "b0"],
                                                categories=["b0", "b1", "b2", "b3", "b4"]),
                        "sex": pd.Categorical(["f", "m", "f", "m", "f", "m"], categories=["f", "m"])})
    codes, n_levels = hm.get_batch_codes(obs, ["batch", "sex"])
    np.testing.assert_array_equal(n_levels, [5, 2])
    np.testing.assert_array_equal(codes[:, 0], [0, 1, 2, 3, 4, 0])
    np.testing.assert_array_equal(codes[:, 1], [5, 6, 5, 6, 5, 6])
    np.testing.assert_array_equal(hm.get_theta_array([2.0, 0.1], n_levels, np.dtype(np.float32)),
                                  np.array([[2, 2, 2, 2, 2, 0.1, 0.1]], dtype=np.float32))
    np.testing.assert_array_equal(hm.get_theta_array(2.0, n_levels, np.dtype(np.float32)),
                                  np.full((1, 7), 2.0, dtype=np.float32))
    per_level = np.arange(7.0)
    np.testing.assert_array_equal(hm.get_theta_array(per_level, n_levels, np.float64), per_level[None])


def test_unused_category_is_a_level():
    obs = pd.DataFrame({"b": pd.Categorical(["x", "z", "x"], categories=["x", "y", "z"])})
    codes, n_levels = hm.get_batch_codes(obs, "b")
    np.testing.assert_array_equal(codes[:, 0], [0, 2, 0])
    assert n_levels.tolist() == [3]


@pytest.mark.parametrize("size", [1, 6])
def test_theta_rejects_invalid_length(size):
    with pytest.raises(ValueError, match=r"batch variables \(2\) or categorical levels \(7\)"):
        hm.get_theta_array([2.0] * size, np.array([5, 2]), np.dtype(np.float32))


def test_theta_rejects_unsupported_type():
    with pytest.raises(ValueError, match="theta must be a scalar or an array-like"):
        hm.get_theta_array({"batch": 2.0}, np.array([5, 2]), np.dtype(np.float32))


def test_batch_keys_are_nonempty_and_complete():
    obs = pd.DataFrame({"batch": ["a", None]})
    with pytest.raises(ValueError, match="contains missing values"):
        hm.get_batch_codes(obs, "batch")
    with pytest.raises(ValueError, match="at least one column"):
        hm.get_batch_codes(obs, [])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_lambda_pruning(dtype):
    n_b = np.array([0, 100, 1, 50], dtype=dtype)
    o = np.array([[0, 0, 0], [30, 40, 30], [0, 0, 1], [20, 15, 15]], dtype=dtype)
    e = np.ones((4, 3), dtype=dtype) * 10
    got = hm.compute_lambda_kb(e, o=o, n_b=n_b, alpha=0.2, threshold=1e-5, ridge_lambda=1.0, dynamic_lambda=True)
    sentinel = dtype(SENT)
    assert np.all(got[0] == sentinel)
    np.testing.assert_allclose(got[1], np.full(3, 2.0, dtype=dtype))
    assert got[2, 0] == sentinel and got[2, 1] == sentinel
    np.testing.assert_allclose(got[2, 2], dtype(2.0))
    np.testing.assert_allclose(got[3], np.full(3, 2.0, dtype=dtype))
    np.testing.assert_array_equal(got, oh.lambda_kb(e.astype(np.float64), o.astype(np.float64),
                                                     n_b.astype(np.float64), alpha=0.2, threshold=1e-5,
                                                     ridge_lambda=1.0, dynamic_lambda=True).astype(dtype))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_lambda_fixed_and_zero_denominator(dtype):
    e = np.ones((3, 5), dtype=dtype)
    got = hm.compute_lambda_kb(e, o=e, n_b=np.ones(3, dtype=dtype), alpha=0.5, threshold=1e-5, ridge_lambda=1.0,
                               dynamic_lambda=False)
    np.testing.assert_array_equal(got, np.ones_like(e))
    got = hm.compute_lambda_kb(np.array([[0.0, 5.0]], dtype=dtype), o=np.array([[0.0, 10.0]], dtype=dtype),
                               n_b=np.array([100.0], dtype=dtype), alpha=0.2, threshold=None, ridge_lambda=1.0,
                               dynamic_lambda=True)
    assert got[0, 0] == dtype(SENT)
    np.testing.assert_allclose(got[0, 1], dtype(1.0))


def _group_sums(x, codes, r):
    gcodes, gid = np.unique(codes, axis=0, return_inverse=True)
    gid = gid.ravel()
    s = np.stack([r[gid == c].sum(axis=0) for c in range(len(gcodes))])
    t = np.stack([r[gid == c].T @ x[gid == c] for c in range(len(gcodes))])
    return gcodes, gid, s, t


def test_multi_key_correction_matches_dense_design():
    """The grouped-sum gram and right-hand sides against the dense one-hot design solved by lstsq, with a suppressed
    pair; the correction z = x - Σ_k r_k (design @ w_k)."""
    rng = np.random.default_rng(734)
    levels = np.array([2, 3])
    codes = np.column_stack([rng.integers(0, lv, size=31) for lv in levels]) + np.array([0, 2])
    x = rng.normal(size=(31, 5))
    r = rng.random(size=(31, 3))
    r /= r.sum(axis=1, keepdims=True)
    lam = rng.uniform(0.2, 1.0, size=(5, 3))
    lam[1, 1] = SENT
    gcodes, gid, s, t = _group_sums(x, codes, r)
    w = hm.multi_weights(s, t, gcodes, lam)
    design = np.zeros((31, 6))
    design[:, 0] = 1
    for j in range(2):
        design[np.arange(31), codes[:, j] + 1] = 1
    expected = x.copy()
    got = x.copy()
    for k in range(3):
        active = lam[:, k] < SENT
        keep = np.concatenate(([True], active))
        sq = np.sqrt(r[:, k])
        pen = np.zeros((active.sum(), keep.sum()))
        pen[:, 1:] = np.diag(np.sqrt(lam[active, k]))
        a = np.vstack((sq[:, None] * design[:, keep], pen))
        b = np.vstack((sq[:, None] * x, np.zeros((active.sum(), 5))))
        wk = np.zeros((6, 5))
        wk[keep] = np.linalg.lstsq(a, b, rcond=None)[0]
        wk[0] = 0
        expected -= r[:, k, None] * (design @ wk)
        got -= r[:, k, None] * (design @ w[k])
    np.testing.assert_allclose(got, expected, atol=1e-11, rtol=1e-11)
    np.testing.assert_allclose(got, oh._correct_multi(x, codes, 5, r, lam), atol=1e-11, rtol=1e-11)


def test_multi_key_singular_fallback(monkeypatch):
    rng = np.random.default_rng(734)
    x = rng.normal(size=(12, 3))
    codes = np.column_stack((np.resize([0, 1], 12), np.resize([2, 3, 4], 12)))
    r = rng.random(size=(12, 2))
    r /= r.sum(axis=1, keepdims=True)
    gcodes, _, s, t = _group_sums(x, codes, r)
    expected = hm.multi_weights(s, t, gcodes, np.ones((5, 2)))
    monkeypatch.setattr(np.linalg, "matrix_rank", lambda _: 0)
    np.testing.assert_allclose(hm.multi_weights(s, t, gcodes, np.ones((5, 2))), expected, atol=1e-12, rtol=1e-12)


def test_fast_path_matches_oracle():
    rng = np.random.default_rng(1)
    codes = rng.integers(0, 4, size=40)
    x = rng.normal(size=(40, 6))
    r = rng.random(size=(40, 3))
    r /= r.sum(axis=1, keepdims=True)
    o = np.stack([r[codes == b].sum(axis=0) for b in range(4)])
    lam = 0.2 * rng.uniform(1, 3, size=(4, 3))
    lam[2, 0] = SENT
    gcodes, gid, s, t = _group_sums(x, codes[:, None], r)
    phi = np.zeros((3, 5, 6))
    phi[:, 0] = t.sum(axis=0)
    phi[:, gcodes[:, 0] + 1] = t.transpose(1, 0, 2)
    w = hm.fast_weights(phi, o, lam)
    got = x - sum(r[:, k, None] * w[k][codes + 1] for k in range(3))
    np.testing.assert_allclose(got, oh._correct_fast(x, codes, 4, r, o, lam), atol=1e-12, rtol=1e-12)


# ------------------------------------------------------------------------------------------ public validation
@pytest.fixture
def adata():
    x, obs, _ = pbmc68k()
    return MiniAnnData(np.zeros((len(x), 1), dtype=np.float32), obs=obs.copy(), obsm={"X_pca": x.copy()})


@pytest.fixture
def no_device(monkeypatch):
    """Replaces the device run: returns its input, so only the host-side checks run."""
    calls = []

    def fake_fit(x, codes, n_levels, **kw):
        hm.get_theta_array(kw["theta"], n_levels, x.dtype)
        calls.append((x, codes, n_levels, kw))
        return x

    monkeypatch.setattr(hm, "fit", fake_fit)
    return calls


def run(adata, *args, **kw):
    from scanpy_b200 import pp

    pp.harmony_integrate(adata, *args, **kw)


def test_public_writes_dtype(adata, no_device):
    run(adata, "bulk_labels", dtype=np.float32)
    assert adata.obsm["X_pca_harmony"].dtype == np.float32
    run(adata, ["bulk_labels", "batch2"], adjusted_basis="two", theta=[2.0, 0.1])
    assert adata.obsm["two"].dtype == np.float64
    x, codes, n_levels, kw = no_device[-1]
    assert codes.shape == (700, 2) and n_levels.tolist() == [10, 3]
    assert kw["stabilized_penalty"] and kw["dynamic_lambda"]


def test_public_rejections(adata, no_device):
    with pytest.raises(ValueError, match="flavor must be"):
        run(adata, "bulk_labels", flavor="harmony3")
    with pytest.raises(ValueError, match="correction_method must be 'fast'"):
        run(adata, "bulk_labels", correction_method="original")
    with pytest.raises(ValueError, match="not available"):
        run(adata, "bulk_labels", basis="nonexistent")
    with pytest.raises(KeyError):
        run(adata, "nonexistent_key")
    with pytest.raises(ValueError, match="max_iter_harmony must be >= 1"):
        run(adata, "bulk_labels", max_iter_harmony=0)
    with pytest.raises(ValueError, match="at least one column"):
        run(adata, [])
    with pytest.raises(ValueError, match=r"batch variables \(2\) or categorical levels \(13\)"):
        run(adata, ["bulk_labels", "batch2"], theta=[1.0, 2.0, 3.0])
    bad = adata.copy()
    bad.obsm["X_pca"][3, 2] = np.nan
    with pytest.raises(ValueError, match="contains NaN values"):
        run(bad, "bulk_labels")
    bad = adata.copy()
    bad.obs["m"] = pd.Series(["a"] * 699 + [None], index=bad.obs.index)
    with pytest.raises(ValueError, match="contains missing values"):
        run(bad, "m")
    assert not no_device


@pytest.mark.parametrize("bad_alpha", [-0.1, 0.0, float("inf"), float("nan")])
def test_public_bad_alpha(adata, no_device, bad_alpha):
    with pytest.raises(ValueError, match="alpha must be a finite positive"):
        run(adata, "bulk_labels", alpha=bad_alpha)


@pytest.mark.parametrize("bad", [-0.1, 1.5, 2.0])
def test_public_bad_prune_threshold(adata, no_device, bad):
    with pytest.raises(ValueError, match="batch_prune_threshold must be in"):
        run(adata, "bulk_labels", batch_prune_threshold=bad)


@pytest.mark.parametrize("ridge_lambda", [0.0, -0.1, float("inf"), float("nan")])
@pytest.mark.parametrize("multikey", [False, True])
def test_public_harmony1_bad_ridge_lambda(adata, no_device, ridge_lambda, multikey):
    adata.obs["dup"] = adata.obs["bulk_labels"]
    with pytest.raises(ValueError, match="ridge_lambda must be a finite positive"):
        run(adata, ["bulk_labels", "dup"] if multikey else "bulk_labels", flavor="harmony1",
            ridge_lambda=ridge_lambda)


def test_public_flavor_warnings(adata, no_device):
    with pytest.warns(UserWarning, match="ridge_lambda is ignored"):
        run(adata, "bulk_labels", flavor="harmony2", ridge_lambda=2.0)
    with pytest.warns(UserWarning, match="alpha is ignored"):
        run(adata, "bulk_labels", flavor="harmony1", alpha=0.5)
    with pytest.warns(UserWarning, match="batch_prune_threshold is ignored"):
        run(adata, "bulk_labels", flavor="harmony1", batch_prune_threshold=0.01)
    assert len(no_device) == 3
    assert not no_device[1][3]["stabilized_penalty"]


def test_caps_raise_not_implemented():
    with pytest.raises(NotImplementedError, match="n_clusters up to 128"):
        hm.check_caps(50, 129, 8, 8)
    with pytest.raises(NotImplementedError, match="basis width up to 128"):
        hm.check_caps(129, 100, 8, 8)
    with pytest.raises(NotImplementedError, match="batch levels over all keys up to 128"):
        hm.check_caps(50, 100, 129, 8)
    hm.check_caps(50, 100, 64 + 3, 192)

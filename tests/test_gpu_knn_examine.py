"""How the tensor-core kNN sweep examines its scores (knn_tc2.cu: a max-tree fast path per row, a warp-wide rare path that
walks a hit mask): the final (idx, dist) must not depend on where the sub-lists start (the sampled threshold at its
default rank, at another rank, a cold start) nor on which consumer loop runs.  The adversarial inputs drive many
insertions, and the SB2_KNN_STAMPS=1 counters show the rare path ran.  Needs an H100 (`pytest -m gpu`)."""
import re

import numpy as np
import pytest

from scanpy_b200 import _ops

pytestmark = pytest.mark.gpu

SWITCHES = ("SB2_KNN_PIPE", "SB2_KNN_TIERS", "SB2_KNN_EST", "SB2_KNN_EST_RANK", "SB2_KNN_STAMPS")
# >= 512 candidate tiles of 128, so the default run samples a starting threshold
N = 70_000
SETTINGS = ({}, {"SB2_KNN_EST": "0"}, {"SB2_KNN_EST_RANK": "3"}, {"SB2_KNN_EST_RANK": "1"}, {"SB2_KNN_PIPE": "0"})


def _blobs(n, d, seed):
    rs = np.random.RandomState(seed)
    x = rs.standard_normal((n, d)).astype(np.float32)
    x[: n // 3] += 2.5
    return x


def _near_duplicates(n, d, seed):
    # 4000 points within 1e-3 of one centre: their rows see thousands of almost equal top scores
    x = _blobs(n, d, seed)
    rs = np.random.RandomState(seed + 1)
    x[1000:5000] = x[0] + 1e-3 * rs.standard_normal((4000, d)).astype(np.float32)
    return x


def _one_tile_clusters(n, d, seed):
    # tight clusters of 128 consecutive points: every row's neighbours arrive in the same candidate tile
    rs = np.random.RandomState(seed)
    centres = 4.0 * rs.standard_normal((n // 128 + 1, d)).astype(np.float32)
    return centres[np.arange(n) // 128] + 0.05 * rs.standard_normal((n, d)).astype(np.float32)


def _run(monkeypatch, capfd, x, k, env):
    for key in SWITCHES:
        monkeypatch.delenv(key, raising=False)
    for key, val in env.items():
        monkeypatch.setenv(key, val)
    capfd.readouterr()
    return _ops.knn(x, k)


def _check_exact(x, k, idx, dist, rows):
    # fp64 brute force on a sample of rows: the distances must be the exact k smallest
    xd = x.astype(np.float64)
    for r in rows:
        d2 = ((xd - xd[r]) ** 2).sum(axis=1)
        kth = np.partition(d2, k - 1)[k - 1]
        assert np.all(d2[idx[r]] <= kth * (1 + 1e-12) + 1e-12)
        np.testing.assert_allclose(np.sort(dist[r] ** 2), np.sort(d2[idx[r]]), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("d", [50, 150])
@pytest.mark.parametrize("k", [15, 40])
def test_examine_independent_of_seed_and_loop(monkeypatch, capfd, d, k):
    x = _blobs(N, d, d + k)
    ref_i, ref_d, ref_f = _run(monkeypatch, capfd, x, k, {})
    for env in SETTINGS[1:]:
        i, dd, _ = _run(monkeypatch, capfd, x, k, env)
        assert np.array_equal(i, ref_i) and np.array_equal(dd, ref_d), env
    _check_exact(x, k, ref_i, ref_d, range(0, N, N // 25))


def _counters(err):
    lines = [ln for ln in err.splitlines() if ln.startswith("[sb2 knn stamps]")]
    assert lines
    m = re.search(r"rare-path tiles ([0-9.]+)%, insertions/row ([0-9.]+)", lines[0])
    assert m, lines[0]
    return float(m.group(1)), float(m.group(2))


@pytest.mark.parametrize("make", [_near_duplicates, _one_tile_clusters])
def test_examine_adversarial_insertions(monkeypatch, capfd, make):
    d, k = 50, 15
    x = make(N, d, 5)
    ref_i, ref_d, _ = _run(monkeypatch, capfd, x, k, {})
    out = {}
    for env in SETTINGS[1:]:
        i, dd, _ = _run(monkeypatch, capfd, x, k, env)
        assert np.array_equal(i, ref_i) and np.array_equal(dd, ref_d), env
    for name, env in (("seeded", {}), ("cold", {"SB2_KNN_EST": "0"})):
        i, dd, _ = _run(monkeypatch, capfd, x, k, dict(env, SB2_KNN_STAMPS="1"))
        assert np.array_equal(i, ref_i) and np.array_equal(dd, ref_d)
        out[name] = _counters(capfd.readouterr().err)
    # the rare path ran, and a cold start (every list starts at -inf) inserts at least the 64 proposals of every row
    assert out["seeded"][0] > 0 and out["seeded"][1] > 0
    assert out["cold"][1] >= 64 and out["cold"][1] > out["seeded"][1]
    _check_exact(x, k, ref_i, ref_d, list(range(1000, 1010)) + list(range(0, N, N // 20)))

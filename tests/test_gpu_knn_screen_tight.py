"""The width of the tile screen's short sweep (knn.cu screen_prep, SB2_KNN_NEAR consecutive tiles of the kd order per
query block, 64 by default): the bound u(q) >= d_k(q) it gives decides which tiles the screen keeps.  With the default,
with 5, 8 and 32 near tiles and with the screen off, (idx, dist) must be bit-identical; against float64 brute force the
wider sweep's u is at most the narrower one's and still at least d_k for every row, and the screen with the tighter u
keeps a subset of the tiles.  Needs an H100 (`pytest -m gpu`)."""
import numpy as np
import pytest

import scanpy_b200 as sb
from oracle import knn as oknn
from scanpy_b200 import _ops

pytestmark = pytest.mark.gpu

SWITCHES = ("SB2_KNN_SCREEN", "SB2_KNN_PIPE", "SB2_KNN_TIERS", "SB2_KNN_EST", "SB2_KNN_STAMPS", "SB2_KNN_LIST", "SB2_KNN_SCAN_SLOTS",
            "SB2_KNN_NEAR")
# 5: one cold pass of 5 tiles; 8: one cold pass; 32 and the default 64: a cold pass of 8, then a seeded pass of all
VARIANTS = ({"SB2_KNN_SCREEN": "1"}, {"SB2_KNN_SCREEN": "1", "SB2_KNN_NEAR": "5"}, {"SB2_KNN_SCREEN": "1", "SB2_KNN_NEAR": "8"},
            {"SB2_KNN_SCREEN": "1", "SB2_KNN_NEAR": "32"}, {"SB2_KNN_SCREEN": "0"})


def _planted(n, d, seed, n_clusters=24, spread=4.0):
    rs = np.random.RandomState(seed)
    centres = spread * rs.standard_normal((n_clusters, d))
    lab = rs.randint(0, n_clusters, n)
    return (centres[lab] + rs.standard_normal((n, d))).astype(np.float32)


def _set_env(monkeypatch, env):
    for key in SWITCHES:
        monkeypatch.delenv(key, raising=False)
    for key, val in env.items():
        monkeypatch.setenv(key, val)


def _all_same(monkeypatch, run, env=None):
    out = []
    for v in VARIANTS:
        _set_env(monkeypatch, dict(env or {}, **v))
        out.append(run())
    i0, d0 = out[-1][0], out[-1][1]
    for r in out[:-1]:
        if isinstance(i0, np.ndarray):
            assert np.array_equal(r[0], i0) and np.array_equal(r[1], d0)
        else:
            assert r[0].equal(i0) and r[1].equal(d0)


@pytest.mark.parametrize("n,d,k", [
    (70_001, 50, 15),
    (9_001, 20, 15),
    (9_001, 50, 1),
    (9_001, 50, 40),      # 128-proposal lists
    (5_000, 150, 15),     # K = 160
    (4_100, 50, 15),      # 33 tiles: the default's 64 near tiles are all of them, 32 leave one out
    (129, 50, 15),        # the last block holds one row
])
def test_near_widths_match_full_sweep_planted(monkeypatch, n, d, k):
    x = _planted(n, d, n + d + k)
    _all_same(monkeypatch, lambda: _ops.knn(x, k))


def test_near_widths_uniform_duplicates_far_from_origin(monkeypatch):
    rs = np.random.RandomState(5)
    u = rs.uniform(-1, 1, (12_345, 50)).astype(np.float32)
    _all_same(monkeypatch, lambda: _ops.knn(u, 15))
    x = _planted(6_000, 24, 11)
    x[:300] = 0.0
    x[1000:1400] = x[999]
    _all_same(monkeypatch, lambda: _ops.knn(x, 15))
    y = (rs.standard_normal((5_000, 24)) * 0.05 + 40.0).astype(np.float32)
    _all_same(monkeypatch, lambda: _ops.knn(y, 15))
    _all_same(monkeypatch, lambda: _ops.knn(y, 15), {"SB2_KNN_SCAN_SLOTS": "16"})   # few open rows: the exact scan


@pytest.mark.parametrize("q0,n_query", [(0, 100), (1280, 5000), (25_984, 4_016)])
def test_near_widths_query_subranges(monkeypatch, q0, n_query):
    import torch

    ctx = sb._abi.default_context()
    d_x = torch.from_numpy(_planted(30_000, 50, 7)).cuda()
    _all_same(monkeypatch, lambda: _ops.knn_device(ctx, d_x, 15, q0=q0, n_query=n_query)[:2])


def _debug_screen(x, k):
    import torch

    ctx = sb._abi.default_context()
    n, d = x.shape
    nb = (n + 127) // 128
    d_x = torch.from_numpy(x).cuda()
    perm = torch.empty(n, dtype=torch.int32, device="cuda")
    lists = torch.empty(nb * nb, dtype=torch.int32, device="cuda")
    lens = torch.empty(nb, dtype=torch.int32, device="cuda")
    ub = torch.empty(n, dtype=torch.float32, device="cuda")
    _ops.check(ctx.lib.sb2_knn_debug_screen_f32(ctx.handle, n, d, _ops.ptr(d_x), k, _ops.ptr(perm), _ops.ptr(lists),
                                                _ops.ptr(lens), _ops.ptr(ub)))
    return perm.cpu().numpy(), lists.cpu().numpy().reshape(nb, nb), lens.cpu().numpy(), ub.cpu().numpy()


@pytest.mark.parametrize("n,d,k", [(24_000, 50, 15), (12_000, 20, 40)])
def test_wider_near_sweep_bound_is_tighter_and_still_a_bound(monkeypatch, n, d, k):
    # the 64 near tiles contain the 8 (also where the list is clamped at either end of the order), so every sub-list
    # ends at least as high and u can only shrink
    x = _planted(n, d, 21)
    _set_env(monkeypatch, {"SB2_KNN_NEAR": "8"})
    p1, l1, n1, u1 = _debug_screen(x, k)
    _set_env(monkeypatch, {})
    p2, l2, n2, u2 = _debug_screen(x, k)
    assert np.array_equal(p1, p2)
    assert np.all(u2 <= u1)
    assert np.any(u2 < u1)
    assert n2.sum() <= n1.sum()
    for b in range(len(n1)):                           # a smaller u keeps a subset of the tiles
        assert np.isin(l2[b, :n2[b]], l1[b, :n1[b]]).all()
    _, kd2 = oknn.knn_exact_f64(x, p2, k)              # exact squared k-th distances of every row, float64
    assert np.all(kd2[:, k - 1] <= u2.astype(np.float64) ** 2)


def test_lists_are_deterministic_with_the_wide_near_sweep(monkeypatch):
    _set_env(monkeypatch, {})
    x = _planted(70_001, 50, 3)
    a, b = _debug_screen(x, 15), _debug_screen(x, 15)
    assert np.array_equal(np.sort(a[0]), np.arange(len(x)))
    for u, v in zip(a, b):
        assert np.array_equal(u, v)


@pytest.mark.parametrize("value", ["0", "65", "128", "abc", "8x"])
def test_bad_near_width_is_rejected(monkeypatch, value):
    # an A/B run must not silently measure the default width instead of the one it asked for
    x = _planted(3_000, 20, 2)
    _set_env(monkeypatch, {"SB2_KNN_SCREEN": "1", "SB2_KNN_NEAR": value})
    with pytest.raises(sb._abi.B200Error, match="SB2_KNN_NEAR"):
        _ops.knn(x, 15)
    _set_env(monkeypatch, {"SB2_KNN_SCREEN": "0", "SB2_KNN_NEAR": value})   # no screen: the width is never used
    _ops.knn(x, 15)

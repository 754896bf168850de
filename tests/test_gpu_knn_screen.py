"""The tile screen of the tensor-core kNN (knn_tc2.cu: kd order, per-block candidate tile lists): the sweep skips tiles
that a bound certifies are too far from every row of a query block, so with the screen (SB2_KNN_SCREEN=1, at every
size) and without it (SB2_KNN_SCREEN=0) the final (idx, dist) must be bit-identical.  The skipped tiles are checked
against float64 brute force, and the kd order for being a deterministic permutation.  Needs an H100 (`pytest -m gpu`)."""
import numpy as np
import pytest

import scanpy_b200 as sb
from oracle import knn as oknn
from scanpy_b200 import _ops

pytestmark = pytest.mark.gpu

SWITCHES = ("SB2_KNN_SCREEN", "SB2_KNN_PIPE", "SB2_KNN_TIERS", "SB2_KNN_EST", "SB2_KNN_STAMPS", "SB2_KNN_LIST", "SB2_KNN_SCAN_SLOTS")


def _planted(n, d, seed, n_clusters=24, spread=4.0):
    rs = np.random.RandomState(seed)
    centres = spread * rs.standard_normal((n_clusters, d))
    lab = rs.randint(0, n_clusters, n)   # storage order mixes the clusters, as the benchmark's data does
    return (centres[lab] + rs.standard_normal((n, d))).astype(np.float32)


def _uniform(n, d, seed):
    return np.random.RandomState(seed).uniform(-1.0, 1.0, (n, d)).astype(np.float32)


def _set_env(monkeypatch, env):
    for key in SWITCHES:
        monkeypatch.delenv(key, raising=False)
    for key, val in env.items():
        monkeypatch.setenv(key, val)


def _on_off(monkeypatch, run, env=None):
    out = []
    for screen in ("1", "0"):
        _set_env(monkeypatch, dict(env or {}, SB2_KNN_SCREEN=screen))
        out.append(run())
    return out


def _assert_same(a, b):
    (i1, d1, _), (i0, d0, _) = a, b
    assert np.array_equal(i1, i0)
    assert np.array_equal(d1, d0)


@pytest.mark.parametrize("n,d,k", [
    (70_001, 50, 15),     # planted clusters at the default's size: the screen skips most tiles
    (9_001, 20, 15),
    (9_001, 50, 1),
    (9_001, 50, 40),      # 128-proposal lists
    (5_000, 150, 15),     # K = 160
    (129, 50, 15),        # two blocks, the second holds one row; fewer tiles than the short sweep's eight
])
def test_screen_matches_full_sweep_planted(monkeypatch, n, d, k):
    x = _planted(n, d, n + d + k)
    _assert_same(*_on_off(monkeypatch, lambda: _ops.knn(x, k)))


@pytest.mark.parametrize("n,d,k", [(20_000, 20, 15), (12_345, 50, 15)])
def test_screen_matches_full_sweep_uniform(monkeypatch, n, d, k):
    # no structure: the screen keeps most tiles, and must still agree
    x = _uniform(n, d, n + d)
    _assert_same(*_on_off(monkeypatch, lambda: _ops.knn(x, k)))


def test_screen_default_switches_on_at_512_tiles(monkeypatch):
    # unset: the screen runs from 512 candidate tiles on; same neighbours as with it off and on
    x = _planted(66_000, 50, 3)
    _set_env(monkeypatch, {})
    auto = _ops.knn(x, 15)
    off, on = _on_off(monkeypatch, lambda: _ops.knn(x, 15))[::-1]
    _assert_same(auto, off)
    _assert_same(on, off)
    assert auto[2]["pass1_issued_flops"] < off[2]["pass1_issued_flops"]   # only visited tiles are counted


def test_screen_duplicates_zero_rows_far_from_origin(monkeypatch):
    rs = np.random.RandomState(11)
    x = _planted(6_000, 24, 11)
    x[:300] = 0.0                       # all-zero rows: exact ties
    x[1000:1400] = x[999]               # a flood of exact duplicates
    _assert_same(*_on_off(monkeypatch, lambda: _ops.knn(x, 15)))
    y = (rs.standard_normal((5_000, 24)) * 0.05 + 40.0).astype(np.float32)   # the fp16 bound swamps the gaps
    _assert_same(*_on_off(monkeypatch, lambda: _ops.knn(y, 15)))
    _assert_same(*_on_off(monkeypatch, lambda: _ops.knn(y, 15), {"SB2_KNN_SCAN_SLOTS": "16"}))   # few open rows: exact scan


@pytest.mark.parametrize("env", [{}, {"SB2_KNN_PIPE": "0"}, {"SB2_KNN_EST": "0"}, {"SB2_KNN_LIST": "128"}])
def test_screen_other_switches(monkeypatch, env):
    x = _planted(30_000, 50, 5)
    _assert_same(*_on_off(monkeypatch, lambda: _ops.knn(x, 15), env))


@pytest.mark.parametrize("q0,n_query", [(0, 100), (1280, 5000), (8960, 21_040), (25_984, 4_016)])
def test_screen_query_subranges(monkeypatch, q0, n_query):
    import torch

    ctx = sb._abi.default_context()
    x = _planted(30_000, 50, 7)
    d_x = torch.from_numpy(x).cuda()
    (i1, d1, _), (i0, d0, _) = _on_off(monkeypatch, lambda: _ops.knn_device(ctx, d_x, 15, q0=q0, n_query=n_query))
    assert torch.equal(i1, i0) and torch.equal(d1, d0)
    full = _ops.knn(x, 15)
    assert np.array_equal(i1.cpu().numpy(), full[0][q0:q0 + n_query])


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


def test_kd_order_is_a_deterministic_permutation(monkeypatch):
    _set_env(monkeypatch, {})
    for n in (129, 5_000, 70_001):
        x = _planted(n, 50, n)
        p1, l1, n1, u1 = _debug_screen(x, 15)
        p2, l2, n2, u2 = _debug_screen(x, 15)
        assert np.array_equal(np.sort(p1), np.arange(n))
        assert np.array_equal(p1, p2) and np.array_equal(n1, n2) and np.array_equal(u1, u2)
        for b in range(len(n1)):
            assert np.array_equal(l1[b, :n1[b]], l2[b, :n2[b]])
            assert np.all(np.diff(l1[b, :n1[b]]) > 0)


@pytest.mark.parametrize("n,d,k", [(40_000, 50, 15), (20_000, 20, 40)])
def test_skipped_tiles_are_farther_than_every_kth_neighbour(monkeypatch, n, d, k):
    _set_env(monkeypatch, {})
    x = _planted(n, d, 21)
    perm, lists, lens, ub = _debug_screen(x, k)
    nb = len(lens)
    assert lens.sum() < 0.9 * nb * nb       # the planted clusters let the screen skip tiles
    xd = x.astype(np.float64)
    xp = xd[perm]
    rs = np.random.RandomState(1)
    for b in sorted(rs.choice(nb, 6, replace=False)):
        rows = np.arange(128 * b, min(128 * b + 128, n))
        _, kd2 = oknn.knn_exact_f64(x, perm[rows], k)        # exact squared k-th distances, float64
        kth = kd2[:, k - 1]
        assert np.all(kth <= ub[rows].astype(np.float64) ** 2)
        keep = np.zeros(nb, bool)
        keep[lists[b, :lens[b]]] = True
        skipped = np.flatnonzero(~keep)
        pts = np.concatenate([np.arange(128 * t, min(128 * t + 128, n)) for t in skipped]) if len(skipped) else np.zeros(0, int)
        for lo in range(0, len(pts), 8192):
            c = xp[pts[lo:lo + 8192]]
            d2 = ((xp[rows][:, None, :] - c[None, :, :]) ** 2).sum(-1)
            assert np.all(d2.min(axis=1) > kth)


def test_unstructured_data_falls_back_to_the_full_sweep(monkeypatch, capfd):
    # uniform data above 512 tiles: the lists would keep nearly every tile, so the default drops them and sweeps every
    # tile of the kd-ordered images from the sampled estimate; SB2_KNN_SCREEN=1 keeps them; all agree with the screen off
    x = _uniform(70_000, 20, 4)
    _set_env(monkeypatch, {"SB2_KNN_STAMPS": "1"})
    capfd.readouterr()
    auto = _ops.knn(x, 15)
    err = capfd.readouterr().err
    line = [ln for ln in err.splitlines() if ln.startswith("[sb2 knn screen]")]
    assert line and "full sweep" in line[0], line
    on, off = _on_off(monkeypatch, lambda: _ops.knn(x, 15))
    _assert_same(auto, off)
    _assert_same(on, off)

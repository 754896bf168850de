"""The kd order's split rules (knn_tc2.cu): by default each segment is split along its sampled principal direction,
with SB2_KNN_SPLIT=coord on its coordinate of largest sampled variance.  The order must be a deterministic permutation,
the same whether a level's segments are split by one CTA each or by many (SB2_KNN_KD_WIDE), each split must put the
smallest projections on a float64 restatement of the direction on the left, and the kNN's (idx, dist) must be
bit-identical under both rules.  Needs an H100 (`pytest -m gpu`)."""
import numpy as np
import pytest

import scanpy_b200 as sb
from oracle import knn as oknn
from scanpy_b200 import _ops

pytestmark = pytest.mark.gpu

SWITCHES = ("SB2_KNN_SCREEN", "SB2_KNN_SPLIT", "SB2_KNN_KD_WIDE", "SB2_KNN_STAMPS", "SB2_KNN_NEAR")
CN = 128
SAMPLES = 512
POWER_ITERS = 12


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


def _debug_screen(x, k=15):
    import torch

    ctx = sb._abi.default_context()
    n, d = x.shape
    nb = (n + CN - 1) // CN
    d_x = torch.from_numpy(x).cuda()
    perm = torch.empty(n, dtype=torch.int32, device="cuda")
    lists = torch.empty(nb * nb, dtype=torch.int32, device="cuda")
    lens = torch.empty(nb, dtype=torch.int32, device="cuda")
    ub = torch.empty(n, dtype=torch.float32, device="cuda")
    _ops.check(ctx.lib.sb2_knn_debug_screen_f32(ctx.handle, n, d, _ops.ptr(d_x), k, _ops.ptr(perm), _ops.ptr(lists),
                                                _ops.ptr(lens), _ops.ptr(ub)))
    return perm.cpu().numpy().astype(np.int64), lists.cpu().numpy().reshape(nb, nb), lens.cpu().numpy(), ub.cpu().numpy()


@pytest.mark.parametrize("split", ["principal", "coord"])
@pytest.mark.parametrize("n", [129, 5_000, 70_001])
def test_order_is_the_same_with_one_or_many_ctas_per_segment(monkeypatch, split, n):
    x = _planted(n, 50, n)
    x[: n // 10] = x[0]                     # a flood of equal keys at every level
    perms = []
    for wide in ("1", "1000", str(10 ** 9), None):      # every level wide, some, none, the default threshold
        _set_env(monkeypatch, {"SB2_KNN_SPLIT": split, **({"SB2_KNN_KD_WIDE": wide} if wide else {})})
        perms.append(_debug_screen(x)[0])
    assert np.array_equal(np.sort(perms[0]), np.arange(n))
    for p in perms[1:]:
        assert np.array_equal(p, perms[0])
    _set_env(monkeypatch, {"SB2_KNN_SPLIT": split})
    assert np.array_equal(_debug_screen(x)[0], perms[0])     # deterministic


def _direction(s):
    """float64 restatement of kd_dir_kernel's target: the sample's top principal direction, largest |v_j| positive"""
    c = s - s.mean(0)
    w, V = np.linalg.eigh(c.T @ c)
    v = V[:, -1]
    v = v if v[np.argmax(np.abs(v))] > 0 else -v
    return v, w


def test_each_split_puts_the_smallest_projections_left(monkeypatch):
    # anisotropic data with a clear eigengap, so the direction is well defined; the levels 0 and 1 are checked
    rs = np.random.RandomState(5)
    n, d = 70_001, 50
    scales = np.concatenate([[12.0, 3.0, 1.5], np.ones(d - 3)])
    q, _ = np.linalg.qr(rs.standard_normal((d, d)))
    x = ((rs.standard_normal((n, d)) * scales) @ q.T).astype(np.float32)
    _set_env(monkeypatch, {"SB2_KNN_KD_WIDE": "1000"})
    perm = _debug_screen(x)[0]
    xd = x.astype(np.float64)
    segs = [(0, n, np.arange(n))]         # (a, b, the segment's points in position order before its split)
    for _level in range(2):
        nxt = []
        for a, b, pts in segs:
            ln = b - a
            m = a + CN * (((ln + CN - 1) // CN) // 2)
            ns = min(ln, SAMPLES)
            v, w = _direction(xd[pts[(np.arange(ns) * ln) // ns]])
            assert w[-1] > 1.5 * w[-2]
            proj = xd[pts] @ v
            left = np.zeros(n, bool)
            left[perm[a:m]] = True
            assert np.array_equal(np.sort(perm[a:b]), np.sort(pts))
            pl, pr = proj[left[pts]], proj[~left[pts]]
            assert pl.max() <= pr.min() + 1e-4 * (proj.max() - proj.min())
            # the next level sees each half in position order
            nxt += [(a, m, pts[left[pts]]), (m, b, pts[~left[pts]])]
        segs = nxt


CASES = [
    (70_001, 50, 15),
    (9_001, 20, 15),
    (9_001, 50, 40),
    (5_000, 150, 15),
    (129, 50, 15),
]


@pytest.mark.parametrize("n,d,k", CASES)
def test_knn_identical_under_both_rules(monkeypatch, n, d, k):
    x = _planted(n, d, n + d + k)
    out = []
    for split in ("coord", "principal"):
        _set_env(monkeypatch, {"SB2_KNN_SCREEN": "1", "SB2_KNN_SPLIT": split})
        out.append(_ops.knn(x, k))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


def test_knn_identical_under_both_rules_duplicates_zero_rows_uniform(monkeypatch):
    x = _planted(6_000, 24, 11)
    x[:300] = 0.0
    x[1000:1400] = x[999]
    y = np.random.RandomState(3).uniform(-1.0, 1.0, (12_345, 50)).astype(np.float32)
    for data in (x, y):
        out = []
        for split in ("coord", "principal"):
            _set_env(monkeypatch, {"SB2_KNN_SCREEN": "1", "SB2_KNN_SPLIT": split})
            out.append(_ops.knn(data, 15))
        assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


@pytest.mark.parametrize("split", ["principal", "coord"])
def test_skipped_tiles_are_farther_than_every_kth_neighbour(monkeypatch, split):
    # the radii bound their tiles under either order: no skipped tile holds a point within a row's k-th distance
    _set_env(monkeypatch, {"SB2_KNN_SPLIT": split})
    n, k = 30_000, 15
    x = _planted(n, 50, 23)
    perm, lists, lens, ub = _debug_screen(x, k)
    nb = len(lens)
    assert lens.sum() < 0.9 * nb * nb
    xp = x.astype(np.float64)[perm]
    rs = np.random.RandomState(2)
    for b in sorted(rs.choice(nb, 5, replace=False)):
        rows = np.arange(CN * b, min(CN * b + CN, n))
        _, kd2 = oknn.knn_exact_f64(x, perm[rows], k)
        kth = kd2[:, k - 1]
        assert np.all(kth <= ub[rows].astype(np.float64) ** 2)
        keep = np.zeros(nb, bool)
        keep[lists[b, :lens[b]]] = True
        pts = np.concatenate([np.arange(CN * t, min(CN * t + CN, n)) for t in np.flatnonzero(~keep)])
        for lo in range(0, len(pts), 8192):
            c = xp[pts[lo:lo + 8192]]
            d2 = ((xp[rows][:, None, :] - c[None, :, :]) ** 2).sum(-1)
            assert np.all(d2.min(axis=1) > kth)


@pytest.mark.parametrize("env", [{"SB2_KNN_SPLIT": "pca"}, {"SB2_KNN_KD_WIDE": "0"}, {"SB2_KNN_KD_WIDE": "12x"}])
def test_unknown_switch_values_fail_the_screened_call(monkeypatch, env):
    _set_env(monkeypatch, {"SB2_KNN_SCREEN": "1", **env})
    with pytest.raises(sb._abi.B200Error):
        _ops.knn(_planted(2_000, 20, 1), 15)

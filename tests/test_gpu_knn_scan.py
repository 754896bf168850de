"""The two fast paths of the tensor-core kNN sweep's examination (knn_tc2.cu): the integer maximum of the scores' bit
patterns (default) against the float max tree (SB2_KNN_SCAN=float).  The integer test is only exact while a row's
threshold tau has a clear sign bit, and the kernel falls back to the float test otherwise, so the raw proposals and the
final (idx, dist) must be bit-identical on every input: seeded and cold starts, both consumer loops, both list sizes,
and data whose rows keep a negative tau (points around the origin: the score q.c - |c|^2/2 of every neighbour of a point
closer to the origin than to its neighbours is negative) next to the same points far from it.  Needs an H100
(`pytest -m gpu`)."""
import numpy as np
import pytest

import scanpy_b200 as sb
from scanpy_b200 import _ops

pytestmark = pytest.mark.gpu

SWITCHES = ("SB2_KNN_SCAN", "SB2_KNN_PIPE", "SB2_KNN_TIERS", "SB2_KNN_EST", "SB2_KNN_EST_RANK", "SB2_KNN_STAMPS")


def _blobs(n, d, seed):
    rs = np.random.RandomState(seed)
    x = rs.standard_normal((n, d)).astype(np.float32)
    x[: n // 3] += 2.5
    return x


def _around_origin(n, d, seed):
    # one Gaussian centred on the origin: a point's k-th neighbour is farther away than the origin for most rows
    return np.random.RandomState(seed).standard_normal((n, d)).astype(np.float32)


def _far_away(n, d, seed):
    # the same points translated: every score a list keeps is positive
    return _around_origin(n, d, seed) + np.float32(8.0)


def _both(monkeypatch, run, env):
    """run() with the float and with the integer fast path, the other switches equal"""
    out = []
    for scan in ("float", None):
        for key in SWITCHES:
            monkeypatch.delenv(key, raising=False)
        for key, val in env.items():
            monkeypatch.setenv(key, val)
        if scan:
            monkeypatch.setenv("SB2_KNN_SCAN", scan)
        out.append(run())
    return out


@pytest.mark.parametrize("make", [_blobs, _around_origin, _far_away])
@pytest.mark.parametrize("n,d,k,env", [
    (3001, 50, 15, {}),                          # ragged n, cold start, pipelined loop at K = 64
    (3001, 50, 15, {"SB2_KNN_PIPE": "0"}),       # single-buffer loop
    (3001, 50, 15, {"SB2_KNN_TIERS": "3"}),      # split tier, K = 160
    (2500, 150, 15, {}),                         # d = 150
    (2500, 150, 40, {}),                         # d = 150, 128-proposal lists (NG = 4)
    (3001, 50, 40, {}),
    (70_001, 50, 15, {}),                        # >= 512 candidate tiles: sampled starting threshold, ragged n
    (70_001, 50, 15, {"SB2_KNN_EST": "0"}),      # same size, cold start
])
def test_integer_scan_matches_float_scan(monkeypatch, make, n, d, k, env):
    x = make(n, d, n + d + k)
    (i0, d0, f0), (i1, d1, f1) = _both(monkeypatch, lambda: _ops.knn(x, k), env)
    assert np.array_equal(i0, i1) and np.array_equal(d0, d1)
    assert f0["n_uncertified"] == f1["n_uncertified"] and f0["n_resweep"] == f1["n_resweep"]


@pytest.mark.parametrize("make", [_blobs, _around_origin, _far_away])
@pytest.mark.parametrize("d,terms", [(50, 1), (50, 3), (150, 1), (150, 3), (20, 1)])
def test_integer_scan_raw_proposals_identical(monkeypatch, make, d, terms):
    # the proposals themselves (scores in the kernel's units and their ids) of one cold-start sweep
    import torch

    ctx = sb._abi.default_context()
    n = 3001
    x = make(n, d, d * terms)
    d_x = torch.from_numpy(x).cuda()

    def run():
        sc = torch.empty((n, 64), dtype=torch.float32, device="cuda")
        ix = torch.empty((n, 64), dtype=torch.int32, device="cuda")
        meta = np.zeros(6, np.float64)
        sb._abi.check(ctx.lib.sb2_knn_debug_proposals_f32(ctx.handle, n, d, _ops.ptr(d_x), terms, _ops.ptr(sc), _ops.ptr(ix), None,
                                                          meta.ctypes.data))
        torch.cuda.synchronize()
        return sc.cpu().numpy(), ix.cpu().numpy(), meta

    (s0, x0, m0), (s1, x1, m1) = _both(monkeypatch, run, {})
    assert np.array_equal(s0.view(np.uint32), s1.view(np.uint32)) and np.array_equal(x0, x1) and np.array_equal(m0, m1)
    # the inputs do what their names say: the thresholds the lists end with (their minima) are negative for most rows
    # of the Gaussian around the origin and positive for every row of the translated one
    tau = s0.reshape(n, 4, 16).min(axis=2)
    if make is _around_origin:
        assert (tau < 0).mean() > 0.4
    if make is _far_away:
        assert (tau > 0).all()

"""The pipelined consumer loop of the tensor-core kNN sweep (knn_tc2.cu, two accumulator sets per warpgroup) against the
single-buffer loop it replaces (SB2_KNN_PIPE=0): same candidate tiles in the same order, same scores, so the proposals
and the final (idx, dist) must be bit-identical.  Needs an H100 (`pytest -m gpu`)."""
import numpy as np
import pytest

import scanpy_b200 as sb
from scanpy_b200 import _ops

pytestmark = pytest.mark.gpu

SWITCHES = ("SB2_KNN_PIPE", "SB2_KNN_TIERS", "SB2_KNN_EST", "SB2_KNN_STAMPS")


def _data(n, d, seed):
    rs = np.random.RandomState(seed)
    x = rs.standard_normal((n, d)).astype(np.float32)
    x[: n // 3] += 2.5  # two blobs
    return x


def _both(monkeypatch, run, env):
    """run() under SB2_KNN_PIPE=0 and =1 with the same other switches"""
    out = []
    for pipe in ("0", "1"):
        for key in SWITCHES:
            monkeypatch.delenv(key, raising=False)
        for key, val in env.items():
            monkeypatch.setenv(key, val)
        monkeypatch.setenv("SB2_KNN_PIPE", pipe)
        out.append(run())
    return out


@pytest.mark.parametrize("n,d,k,env", [
    (3001, 50, 15, {}),                          # ragged n, fp16 tier (K = 64)
    (3001, 50, 15, {"SB2_KNN_TIERS": "3"}),      # split tier (K = 160)
    (2500, 150, 15, {}),                         # fp16 tier at K = 160
    (2500, 150, 15, {"SB2_KNN_TIERS": "3"}),     # split tier at K = 512 in four slices: single-buffer loop either way
    (3001, 50, 40, {}),                          # 128-proposal lists (NG = 4)
    (70_000, 50, 15, {}),                        # >= 512 candidate tiles: sampled starting threshold
    (70_000, 50, 15, {"SB2_KNN_EST": "0"}),      # same size, cold start
    (129, 50, 15, {}),                           # two query CTAs, the second one holds a single row
])
def test_pipelined_sweep_matches_single_buffer(monkeypatch, n, d, k, env):
    x = _data(n, d, n + d + k)
    (i0, d0, f0), (i1, d1, f1) = _both(monkeypatch, lambda: _ops.knn(x, k), env)
    assert np.array_equal(i0, i1) and np.array_equal(d0, d1)
    assert f0["n_uncertified"] == f1["n_uncertified"] and f0["n_resweep"] == f1["n_resweep"]
    assert f0["pass1_issued_flops"] == f1["pass1_issued_flops"]


def test_pipelined_sweep_query_below_one_tile(monkeypatch):
    import torch

    ctx = sb._abi.default_context()
    x = _data(5000, 50, 7)
    d_x = torch.from_numpy(x).cuda()
    (i0, d0, _), (i1, d1, _) = _both(monkeypatch, lambda: _ops.knn_device(ctx, d_x, 15, q0=0, n_query=100), {})
    assert torch.equal(i0, i1) and torch.equal(d0, d1)


@pytest.mark.parametrize("d,terms", [(50, 1), (50, 3), (150, 1), (150, 3), (20, 1)])
def test_pipelined_sweep_raw_proposals_identical(monkeypatch, d, terms):
    # the proposals themselves (scores in the kernel's units and their ids) of one cold-start sweep
    import torch

    ctx = sb._abi.default_context()
    n = 3001
    d_x = torch.from_numpy(_data(n, d, d * terms)).cuda()

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


@pytest.mark.parametrize("d,tiers,loop", [(50, None, "pipelined"), (50, "3", "pipelined"), (150, None, "pipelined"),
                                          (150, "3", "single-buffer"), (20, None, "single-buffer")])
def test_sweep_loop_choice_and_stamps(monkeypatch, capfd, d, tiers, loop):
    # which loop a shape gets (SB2_KNN_STAMPS=1 reports it with the phase split on stderr), and SB2_KNN_PIPE=0 always
    # takes the single-buffer one
    x = _data(3001, d, 3)
    env = {"SB2_KNN_STAMPS": "1"}
    if tiers:
        env["SB2_KNN_TIERS"] = tiers
    _both(monkeypatch, lambda: _ops.knn(x, 15), env)
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[sb2 knn stamps]")]
    assert len(lines) >= 2
    assert all("single-buffer loop" in ln for ln in lines[: len(lines) // 2])
    assert all(f"{loop} loop" in ln for ln in lines[len(lines) // 2:])
    assert all("wait full" in ln and "insert" in ln for ln in lines)

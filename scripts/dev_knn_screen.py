"""A/B of the kNN tile screen on the bench workload's own X_pca (1.3M x 50, k = 15): SB2_KNN_SCREEN=0 (every query
block sweeps every candidate tile) against the default (kd order, per-block tile lists).

PCA runs once; then the two settings alternate over --rounds rounds of _ops.knn_device.  Per setting: pass1_ms (CUDA
events around the sweep launches, which with the screen include the kd order, the short sweep and the screen), issued
tensor TFLOP/s, uncertified and re-swept rows; from one extra run with SB2_KNN_STAMPS=1 the split of the consumer
warpgroups' cycles and the screen's line: the surviving fraction of (block, tile) pairs, the list-length distribution and
the ms of the kd order and of the screen.  Asserts that (idx, dist) are bit-identical between the two settings.  Prints
the card name and its power limit: the numbers mean nothing without them.

    python scripts/dev_knn_screen.py [--n 1300000] [--rounds 5]
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from scanpy_b200 import _abi, _ops  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception as exc:  # the numbers are still printed, flagged
        return f"unknown ({exc!r})"


def setting(var, s):
    if s == "auto":
        os.environ.pop(var, None)
    else:
        os.environ[var] = s


def stamped(ctx, xp, k):
    """one knn_device call with SB2_KNN_STAMPS=1; the library prints one line per sweep launch on fd 2"""
    os.environ["SB2_KNN_STAMPS"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            _ops.knn_device(ctx, xp, k)
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["SB2_KNN_STAMPS"]
        f.seek(0)
        return [ln for ln in f.read().splitlines() if ln.startswith(("[sb2 knn stamps]", "[sb2 knn screen]"))]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_300_000)
    p.add_argument("--genes", type=int, default=2000)
    p.add_argument("--k", type=int, default=15)
    p.add_argument("--rounds", type=int, default=5)
    a = p.parse_args()
    print("card:", card(), flush=True)
    x, _ = synth_scipy(a.n, a.genes, device="cuda")
    ctx = _abi.default_context()
    ip, ix, dat = _ops.csr_to_device(x)
    xp = _ops.pca_csr_device(ctx, ip, ix, dat, a.n, a.genes, 50, solver=1)["X_pca"].contiguous()
    print(f"X_pca {tuple(xp.shape)}", flush=True)
    var, settings = "SB2_KNN_SCREEN", ("0", "auto")
    old, new = settings
    ms = {s: [] for s in settings}
    ref = {}
    for r in range(a.rounds + 1):            # round 0 warms both settings up
        for s in settings:
            setting(var, s)
            idx, dist, info = _ops.knn_device(ctx, xp, a.k)
            torch.cuda.synchronize()
            if r == 0:
                ref[s] = (idx.clone(), dist.clone(), info)
                continue
            ms[s].append(info["pass1_ms"])
            issued = info["pass1_issued_flops"] / (info["pass1_ms"] * 1e-3) / 1e12
            print(f"round {r} {var}={s}: pass1 {info['pass1_ms']:.1f} ms, issued {issued:.0f} TFLOP/s, "
                  f"uncertified {info['n_uncertified']}, resweep {info['n_resweep']}", flush=True)
    (i0, d0, f0), (i1, d1, f1) = ref[old], ref[new]
    same = bool(torch.equal(i0, i1) and torch.equal(d0, d1))
    print(f"(idx, dist) bit-identical between {var}={old} and {var}={new}: {same}; uncertified {f0['n_uncertified']} / "
          f"{f1['n_uncertified']}, resweep {f0['n_resweep']} / {f1['n_resweep']}", flush=True)
    for s in settings:
        v = np.array(ms[s])
        print(f"{var}={s}: pass1_ms median {np.median(v):.1f} min {v.min():.1f} max {v.max():.1f} over {len(v)} rounds", flush=True)
    print(f"pass1 median ratio new/old {np.median(ms[new]) / np.median(ms[old]):.3f}; slowest new {max(ms[new]):.1f} ms vs "
          f"fastest old {min(ms[old]):.1f} ms", flush=True)
    for s in settings:
        setting(var, s)
        for ln in stamped(ctx, xp, a.k):
            print(f"{var}={s} {ln}", flush=True)
    os.environ.pop(var, None)
    print("card:", card(), flush=True)
    assert same, f"{var}={old} and {var}={new} disagree"


if __name__ == "__main__":
    main()

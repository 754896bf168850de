"""The kNN tile screen under the kd order's two split rules, on the bench workload's own X_pca (1.3M x 50, k = 15):
SB2_KNN_SPLIT=coord (each segment split on its coordinate of largest sampled variance) against the default (its
sampled principal direction).

Per rule, from sb2_knn_debug_screen_f32: the kept fraction of (block, tile) pairs, the list lengths and the median tile
radius r_t (float64, from the order itself); from one SB2_KNN_STAMPS=1 run: the screen's line (kd order ms, images +
short sweep + screen ms) and each sweep's (cycles per visited tile, insertions per row).  The kd order is also timed with
SB2_KNN_KD_WIDE set above n, so that every level takes the one-CTA-per-segment split.  Then pass1_ms (CUDA events around
the whole kNN first pass, screen included) over --rounds alternated rounds, median and min-max, and whether (idx, dist)
are bit-identical between the rules.  Last, the same rounds on unclustered 1.3M x 50 data (uniform and Gaussian), where
the screen drops its lists: there the new rule can only cost.  Prints the card name and power limit.

    python scripts/dev_knn_split.py [--n 1300000] [--rounds 5]
"""
import argparse
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from dev_knn_screen import card, stamped  # noqa: E402
from dev_knn_screen_tight import debug_screen  # noqa: E402
from scanpy_b200 import _abi, _ops  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402

RULES = {"coord": {"SB2_KNN_SPLIT": "coord"}, "principal": {}}


def use(env):
    for key in ("SB2_KNN_SPLIT", "SB2_KNN_KD_WIDE", "SB2_KNN_STAMPS"):
        os.environ.pop(key, None)
    os.environ.update(env)


def median_radius(xp, perm):
    n, d = xp.shape
    r = []
    for t0 in range(0, n, 128 * 4096):
        x = xp.double()[perm[t0:t0 + 128 * 4096]]
        full = x.shape[0] // 128
        xt = x[:full * 128].view(full, 128, d)
        r.append(((xt - xt.mean(1, keepdim=True)) ** 2).sum(-1).sqrt().amax(1))
    return float(torch.cat(r).median())


def report_lines(tag, lines):
    for ln in lines:
        m = re.search(r"(\d+) cycles/tile.*insertions/row ([\d.]+)", ln)
        o = re.search(r"kd order ([\d.]+) ms", ln)
        extra = f"  => cycles/tile {m.group(1)}, insertions/row {m.group(2)}" if m else (f"  => kd order {o.group(1)} ms" if o else "")
        print(f"{tag} {ln}{extra}", flush=True)


def kd_kernels(ctx, xp, k):
    """device time of the kd order's kernels in one profiled call (a run of its own: tracing slows the host)"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _ops.knn_device(ctx, xp, k)
        torch.cuda.synchronize()
    rows = [(e.key, e.device_time_total / 1e3, e.count) for e in prof.key_averages() if "kd_" in e.key]
    return ", ".join(f"{re.sub(r'.*(kd_[a-z_]+).*', r'\1', n)} {ms:.2f} ms / {c}" for n, ms, c in sorted(rows, key=lambda r: -r[1]))


def timed_rounds(ctx, xp, k, rounds):
    ms = {s: [] for s in RULES}
    ref = {}
    for r in range(rounds + 1):        # round 0 warms both rules up
        for s, env in RULES.items():
            use(env)
            idx, dist, info = _ops.knn_device(ctx, xp, k)
            torch.cuda.synchronize()
            if r == 0:
                ref[s] = (idx.clone(), dist.clone())
            else:
                ms[s].append(info["pass1_ms"])
    (i0, d0), (i1, d1) = ref["coord"], ref["principal"]
    return ms, torch.equal(i0, i1) and torch.equal(d0, d1)


def summary(v):
    v = np.array(v)
    return f"median {np.median(v):.1f} (min {v.min():.1f}, max {v.max():.1f}) over {len(v)}"


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
    for s, env in RULES.items():
        use(env)
        perm, lens, _ = debug_screen(ctx, xp, a.k)
        nb = lens.numel()
        ln = lens.sort().values
        print(f"{s}: kept (block, tile) pairs {float(lens.double().sum()) / nb / nb:.4f}, list length min {int(ln[0])} "
              f"median {int(ln[nb // 2])} max {int(ln[-1])}, median tile radius {median_radius(xp, perm):.4f}", flush=True)
        report_lines(s, stamped(ctx, xp, a.k))
        use(dict(env, SB2_KNN_KD_WIDE=str(2 * a.n)))
        report_lines(f"{s} (one CTA per segment)", [ln for ln in stamped(ctx, xp, a.k) if ln.startswith("[sb2 knn screen]")])
        use(env)
        print(f"{s} kd order kernels (device ms / launches): {kd_kernels(ctx, xp, a.k)}", flush=True)
    ms, same = timed_rounds(ctx, xp, a.k, a.rounds)
    for s in RULES:
        print(f"{s}: pass1_ms {summary(ms[s])}", flush=True)
    print(f"(idx, dist) bit-identical between the rules: {same}", flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for kind in ("uniform", "gauss"):
        shape = (a.n, 50)
        y = ((torch.rand(shape, generator=g, device="cuda") * 2 - 1) if kind == "uniform"
             else torch.randn(shape, generator=g, device="cuda")).contiguous()
        yms, ysame = timed_rounds(ctx, y, a.k, a.rounds)
        for s, env in RULES.items():
            use(env)
            line = [ln for ln in stamped(ctx, y, a.k) if ln.startswith("[sb2 knn screen]")]
            print(f"{kind} {a.n} x 50, {s}: pass1_ms {summary(yms[s])}; {line[0] if line else ''}", flush=True)
        print(f"{kind}: (idx, dist) bit-identical between the rules: {ysame}", flush=True)
        same = same and ysame
    use({})
    print("card:", card(), flush=True)
    assert same


if __name__ == "__main__":
    main()

"""Measurement of sb2_leiden_csr_f32 on the benchmark graph on an H100 (not a test; bench.py does not run it).

Builds the benchmark's connectivities once (scanpy_b200._synth at 1.3M x 2000 -> device PCA, 50 components -> exact
kNN, k=15 -> fuzzy simplicial set), then times the Leiden call alone (resolution 1, n_iterations=-1, seed 0) with CUDA
events over --reps calls after a warm-up.  It prints the GPU name and power limit, then per path:
* Leiden ms per call (median, min-max);
* one extra call with SB2_TIMING=1: the phase split (local_move / refine / aggregate / finalize; these timings
  synchronise after every phase, so their sum is above the untimed call), the local-moving sweeps and refinement
  rounds per (pass, level, vertices) with each level's synchronised ms, the refinement work-list per round, and the
  host synchronisations of the sweep loops and the aggregation;
* the labels' SHA-1, the modularity and the passes / levels / moves;
* what a sweep loop kept on the device could save at most: the local-moving + refinement ms of the levels that fit
  one co-resident grid of one warp per vertex (at most 64 warps per SM), and the level-0 sweeps and rounds times the
  time of their fixed bookkeeping, timed here as a stand-in (a memset of n int32 flags, an int64 prefix sum over them
  and one scalar read back to the host).

Usage: python scripts/dev_leiden.py [--n 1300000] [--reps 5]
"""
import argparse
import hashlib
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from scanpy_b200 import _abi, _ops  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable ({e})"


def connectivities(n, g):
    ctx = _abi.default_context()
    x, _ = synth_scipy(n, g, device="cuda")
    d_indptr, d_indices, d_data = _ops.csr_to_device(x)
    d_x = _ops.pca_csr_device(ctx, d_indptr, d_indices, d_data, n, g, 50)["X_pca"]
    idx, dist, _ = _ops.knn_device(ctx, d_x, 15)
    indptr, indices, data, _, _ = _ops.fuzzy_simplicial_set_device(ctx, idx, dist, n, 15)
    torch.cuda.synchronize()
    return ctx, indptr, indices, data


def call(ctx, graph, n):
    member, q, nc, info = _ops.leiden_device(ctx, *graph, n, resolution=1.0, n_iterations=-1, seed=0)
    return member, q, nc, info


def timed(ctx, graph, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = call(ctx, graph, n)
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def traced(ctx, graph, n):
    """One call with SB2_TIMING=1; the library's stderr goes to a file that is parsed afterwards."""
    os.environ["SB2_TIMING"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            out = call(ctx, graph, n)
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["SB2_TIMING"]
        f.seek(0)
        text = f.read()
    return out, parse(text, n)


def parse(text, n0):
    """-> dict(phases, syncs, sweeps / rounds / lm_ms / rf_ms, each {(pass, level, n): value})."""
    sweeps, rounds, lm_ms, rf_ms = {}, defaultdict(list), {}, {}
    p, lev = -1, 0
    phases, syncs = None, None
    for line in text.splitlines():
        if m := re.search(r"local_move n=(\d+) sweeps=(\d+)", line):
            nl = int(m[1])
            if nl == n0:
                p, lev = p + 1, 0
            else:
                lev += 1
            sweeps[(p, lev, nl)] = int(m[2])
        elif m := re.search(r"refine n=(\d+) round=(\d+) singletons=(\d+)", line):
            rounds[(p, lev, int(m[1]))].append(int(m[3]))
        elif m := re.search(r"level n=(\d+) (local_move|refine) ([\d.]+) ms", line):
            (lm_ms if m[2] == "local_move" else rf_ms)[(p, lev, int(m[1]))] = float(m[3])
        elif m := re.search(r"local_move ([\d.]+) ms \((\d+) calls\) refine ([\d.]+) ms aggregate ([\d.]+) ms "
                            r"finalize ([\d.]+) ms syncs=(\d+)", line):
            phases = dict(local_move=float(m[1]), refine=float(m[3]), aggregate=float(m[4]), finalize=float(m[5]))
            syncs = int(m[6])
    return dict(phases=phases, syncs=syncs, sweeps=sweeps, rounds=dict(rounds), lm_ms=lm_ms, rf_ms=rf_ms)


def fingerprint(out):
    member, q, nc, info = out
    h = hashlib.sha1(member.cpu().numpy().astype(np.int32).tobytes()).hexdigest()
    return dict(sha1=h, modularity=q, n_communities=nc, **info)


def report(tag, times, fp, tr):
    t = np.array(times)
    print(f"\n== {tag}: Leiden {np.median(t):.1f} ms median, {t.min():.1f}-{t.max():.1f} ms over {t.size} calls")
    print(f"   labels sha1 {fp['sha1']}  modularity {fp['modularity']!r}  communities {fp['n_communities']}  "
          f"passes {fp['passes']} levels {fp['levels']} moves {fp['moves']}")
    ph = tr["phases"] or {}
    print("   SB2_TIMING phases (synchronised): " + ", ".join(f"{k} {v:.1f} ms" for k, v in ph.items())
          + f"; host syncs of the sweeps, rounds and aggregation {tr['syncs']}")
    tot_sw = sum(tr["sweeps"].values())
    tot_rd = sum(len(r) for r in tr["rounds"].values())
    print(f"   sweeps {tot_sw}, refinement rounds {tot_rd}")
    print("   pass level        n  sweeps  lm ms  us/sweep  rounds  rf ms  refinement work-list per round")
    for key, s in tr["sweeps"].items():
        lm, rf = tr["lm_ms"].get(key, 0.0), tr["rf_ms"].get(key, 0.0)
        rl = tr["rounds"].get(key, [])
        print(f"   {key[0]:4d} {key[1]:5d} {key[2]:8d} {s:7d} {lm:6.2f} {1e3 * lm / max(s, 1):9.1f} "
              f"{len(rl):7d} {rf:6.2f}  {rl}")


def ceilings(tr, n0, stage_ms):
    """Upper bounds on what keeping the sweep loop on the device could save, from the traced call."""
    torch.cuda.synchronize()
    limit = 64 * torch.cuda.get_device_properties(0).multi_processor_count
    small = sum(v for k, v in tr["lm_ms"].items() if k[2] <= limit) + sum(v for k, v in tr["rf_ms"].items() if k[2] <= limit)
    print(f"\n   levels of at most {limit} vertices (64 warps per SM): local_move + refine {small:.1f} ms, "
          f"{100 * small / stage_ms:.1f} % of the {stage_ms:.1f} ms stage")
    flags = torch.zeros(n0, dtype=torch.int32, device="cuda")

    def bookkeeping():
        flags.zero_()
        return int(torch.cumsum(flags, 0, dtype=torch.int64)[-1])

    for _ in range(5):
        bookkeeping()
    reps = 200
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        bookkeeping()
    b.record()
    b.synchronize()
    per = a.elapsed_time(b) / reps
    l0 = sum(s for k, s in tr["sweeps"].items() if k[2] == n0) + sum(len(r) for k, r in tr["rounds"].items() if k[2] == n0)
    print(f"   level 0: {l0} sweeps and rounds x {1e3 * per:.1f} us of stand-in bookkeeping at n = {n0} "
          f"= {l0 * per:.2f} ms, {100 * l0 * per / stage_ms:.1f} % of the stage")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_300_000)
    ap.add_argument("--g", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dev_leiden.py needs a CUDA device")
    print("GPU:", gpu_line())
    ctx, *graph = connectivities(a.n, a.g)
    print(f"graph: {a.n} vertices, {graph[1].numel()} arcs")
    call(ctx, graph, a.n)   # warm-up
    times, fps = [], []
    for _ in range(a.reps):
        ms, out = timed(ctx, graph, a.n)
        times.append(ms)
        fps.append(fingerprint(out))
    fp = fps[0]
    assert all(f == fp for f in fps), "repeated calls gave different results"
    out, tr = traced(ctx, graph, a.n)
    assert fingerprint(out) == fp, "the traced call gave a different result"
    report("sb2_leiden_csr_f32", times, fp, tr)
    ceilings(tr, a.n, float(np.median(times)))


if __name__ == "__main__":
    main()

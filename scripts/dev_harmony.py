"""Measurement of sb.pp.harmony_integrate on an H100 (not a test; bench.py does not run it).

1.3M cells x 50 components, K = 100, 8 and 64 batches, one key and two keys (the second with 3 levels), float64 and
float32.  The schedule is pinned (negative tolerances, 2 outer x 10 clustering iterations) so every configuration does
the same work.  For each it prints the GPU name and power limit, the call time of `_harmony.fit` split into the k-means
start and the rest, the time per clustering iteration, the device time of each kernel from torch.profiler over one
clustering iteration, the bytes each pass must move (counted from the shapes, not measured), the host cost of the
permutation draws, and the oracle timed on the host CPU on a subsample and extrapolated linearly to all cells.

Usage: python scripts/dev_harmony.py [--n 1300000] [--out results.json]   (--out: also write the results as JSON)
"""
import argparse
import json
import re
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pandas as pd

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from oracle import harmony as oh  # noqa: E402
from scanpy_b200 import _harmony as hm  # noqa: E402

SUBSAMPLE = 20_000
D, K = 50, 100
OUTER, INNER = 2, 10


def data(n, n_batches, keys, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, D)) + rng.normal(scale=3.0, size=(30, D))[rng.integers(0, 30, size=n)]
    cols = {}
    for j, nb in enumerate([n_batches, 3][:keys]):
        b = rng.integers(0, nb, size=n)
        x += rng.normal(scale=1.0, size=(nb, D))[b]
        cols[f"k{j}"] = pd.Categorical.from_codes(b, [str(i) for i in range(nb)])
    return x, pd.DataFrame(cols)


def args(**kw):
    a = dict(theta=2.0, sigma=0.1, n_clusters=K, max_iter_harmony=OUTER, max_iter_clustering=INNER, tol_harmony=-1.0,
             tol_clustering=-1.0, ridge_lambda=1.0, block_proportion=0.05, tau=0, alpha=0.2,
             batch_prune_threshold=1e-5, stabilized_penalty=True, dynamic_lambda=True)
    a.update(kw)
    return a


def bytes_per_pass(n, dtype, keys):
    s = np.dtype(dtype).itemsize
    z, r = n * D * s, n * K * s
    return {"centroids RᵀZ (read R, Z)": z + r, "block steps (read Z, write R, per-cell entropy)": z + r + 8 * n,
            "code sums old + new (read R twice)": 2 * r + 2 * 4 * keys * n,
            "clustering iteration total": (z + r) + (z + r + 8 * n) + 2 * r,
            "correction sums RᵀX per tuple (read R, X)": z + r, "apply (read X, R; write z_hat, z_norm)": 3 * z + r}


def profile_kernels(x, codes, n_levels, centers):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        hm.fit(x, codes, n_levels, gen=np.random.default_rng(0), centers=centers,
               **args(max_iter_harmony=1, max_iter_clustering=1))
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" and ev.count:
            t = getattr(ev, "device_time_total", None) or ev.cuda_time_total
            m = re.search(r"(\w+_kernel)", ev.key)
            name = m.group(1) if m else ev.key.strip()[:40]
            prev = out.get(name, {"calls": 0, "ms": 0.0})
            out[name] = {"calls": prev["calls"] + ev.count, "ms": round(prev["ms"] + t / 1e3, 3)}
    return dict(sorted(out.items(), key=lambda kv: -kv[1]["ms"])[:14])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_300_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("GPU:", gpu)
    res = {"gpu": gpu, "n": a.n, "d": D, "k": K, "schedule": f"{OUTER} outer x {INNER} clustering iterations",
           "runs": []}
    gen = np.random.default_rng(0)
    t0 = time.perf_counter()
    for _ in range(5):
        gen.permutation(a.n)
    res["host_permutation_ms"] = (time.perf_counter() - t0) / 5 * 1e3
    print(f"host rng.permutation({a.n}): {res['host_permutation_ms']:.1f} ms per draw")
    for n_batches, keys, dtype in [(8, 1, np.float64), (64, 1, np.float64), (8, 2, np.float64), (64, 2, np.float64),
                                   (8, 1, np.float32), (64, 2, np.float32)]:
        x, obs = data(a.n, n_batches, keys)
        x = x.astype(dtype)
        codes, n_levels = hm.get_batch_codes(obs, list(obs.columns))
        hm.fit(x[:20000], codes[:20000], n_levels, gen=np.random.default_rng(0), **args(max_iter_harmony=1,
                                                                                           max_iter_clustering=2))
        torch.cuda.synchronize()
        # k-means start alone
        dev = hm._Dev(x, codes, int(n_levels.sum()))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        centers = hm.kmeans_start(dev, K, hm.spawn_random_state(np.random.default_rng(0)), x.dtype)
        torch.cuda.synchronize()
        t_km = time.perf_counter() - t0
        del dev
        # the schedule from those centres, twice
        ts = []
        for _ in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            hm.fit(x, codes, n_levels, gen=np.random.default_rng(0), centers=centers, **args())
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        # one outer iteration of one clustering iteration: setup + correction, to split the per-iteration cost
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hm.fit(x, codes, n_levels, gen=np.random.default_rng(0), centers=centers,
               **args(max_iter_harmony=1, max_iter_clustering=1))
        torch.cuda.synchronize()
        t_one = time.perf_counter() - t0
        per_clust = (min(ts) - t_one) / (OUTER * INNER - 1)  # 19 clustering iterations and one correction
        run = {"batches": n_batches, "keys": keys, "dtype": np.dtype(dtype).name, "kmeans_start_s": round(t_km, 3),
               "fit_from_centres_s": [round(t, 3) for t in ts], "one_iteration_fit_s": round(t_one, 3),
               "per_clustering_iteration_ms_est": round(per_clust * 1e3, 2),
               "bytes_counted_GB": {k: round(v / 1e9, 3) for k, v in bytes_per_pass(a.n, dtype, keys).items()},
               "kernels_one_iteration": profile_kernels(x, codes, n_levels, centers)}
        print(json.dumps(run, indent=1, ensure_ascii=False))
        res["runs"].append(run)
    # the oracle on the host CPU, on a subsample, extrapolated linearly in n
    x, obs = data(SUBSAMPLE, 8, 1)
    codes, n_levels = hm.get_batch_codes(obs, list(obs.columns))
    z = x / np.linalg.norm(x, axis=1, keepdims=True)
    centers, _ = oh.kmeans_start(z, K, hm.spawn_random_state(np.random.default_rng(0)))
    t0 = time.perf_counter()
    oa = args()
    oh.harmony(x, codes, n_levels, centers=centers, rng=0, **oa)
    t_or = time.perf_counter() - t0
    res["oracle_host_s_subsample"] = round(t_or, 2)
    res["oracle_host_s_extrapolated_to_n"] = round(t_or * a.n / SUBSAMPLE, 1)
    print(f"oracle (numpy, host CPU): {t_or:.2f} s at {SUBSAMPLE} cells, extrapolated {t_or * a.n / SUBSAMPLE:.0f} s "
          f"at {a.n} (an extrapolation, not a measurement)")
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1, ensure_ascii=False))


if __name__ == "__main__":
    main()

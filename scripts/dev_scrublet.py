"""Measurement of sb.pp.scrublet on an H100 (not a test; bench.py does not run it).

Seeded negative-binomial integer counts as float32 CSR (NB(2) per gene around log-normal means, three cell sizes), two
cases:
* A: 1.3M x 2000 in 128 samples, `batch_key="sample"` (about 10k cells, 30k points and k_adj = 150 per sample);
* B: one 100k-cell sample x 2000 (300k points, k_adj = 474).
It prints the GPU name and power limit, then per case the call time and the time per stage (doublet synthesis, PCA,
label count, rest), each a host clock around the stage ending in a device synchronise.  For B it also times the label
count kernel alone with CUDA events on the call's own embedding and reports its distance FLOP rate, counting
LC_PASSES passes over all n^2 pairs with a subtraction and an FMA (3 FLOP) per coordinate, against the data sheet's FP32
rate.  The CPU comparison is the fp64 oracle (oracle/scrublet.py) on one 10k-cell sample: preprocessing and PCA timed
whole, its brute-force neighbour count timed on 300 rows and scaled to all rows.

Usage: python scripts/dev_scrublet.py [--cases A,B] [--reps 3] [--no-oracle]
"""
import argparse
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pandas as pd
from scipy import sparse

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import scanpy_b200 as sb  # noqa: E402
from oracle import scrublet as osc  # noqa: E402
from scanpy_b200 import _scrublet  # noqa: E402
from scanpy_b200._compat import LegacyRng, MiniAnnData  # noqa: E402

FP32_PEAK = 67e12  # H100 SXM5 data-sheet FP32 (non-tensor) FLOP/s
LC_PASSES = 5      # four radix passes and the band pass of sb2_knn_label_count_f32
CASES = {"A": (1_300_000, 2000, 128), "B": (100_000, 2000, 1)}


def nb_counts(n, g, seed=0):
    """CSR float32: NB(2) counts around per-gene log-normal means times a cell size of 0.5, 1 or 2 (about 530 stored
    values per row at 2000 genes)."""
    rng = np.random.default_rng(seed)
    w = np.exp(rng.normal(-1.5, 1.3, g)).astype(np.float32)
    size = rng.choice(np.array([0.5, 1.0, 2.0], np.float32), n)
    rows = []
    for r0 in range(0, n, 50_000):
        mu = size[r0:r0 + 50_000, None] * w[None, :]
        rows.append(sparse.csr_matrix(rng.negative_binomial(2, 2 / (2 + mu)).astype(np.float32)))
    return sparse.vstack(rows).tocsr()


STAGES = {}


def timed(name, fn):
    def wrapped(*a, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*a, **kw)
        torch.cuda.synchronize()
        STAGES[name] = STAGES.get(name, 0.0) + time.perf_counter() - t0
        return out
    return wrapped


_scrublet.simulate = timed("synthesis", _scrublet.simulate)
_scrublet.manifold = timed("pca", _scrublet.manifold)
_lc = _scrublet.label_count
_scrublet.label_count = timed("label count", _lc)
EMB = {}
_manifold = _scrublet.manifold


def keep_embedding(*a, **kw):
    EMB["last"] = _manifold(*a, **kw)
    return EMB["last"]


_scrublet.manifold = keep_embedding


def run_case(key, reps):
    n, g, n_samples = CASES[key]
    x = nb_counts(n, g)
    obs = pd.DataFrame({"sample": np.random.default_rng(1).integers(0, n_samples, n).astype(str)})
    print(f"\n== {key}: {n} x {g}, nnz {x.nnz} ({x.nnz / n:.0f} per row), {n_samples} sample(s)")
    for rep in range(reps + 1):
        STAGES.clear()
        adata = MiniAnnData(x, obs=obs.copy())
        t0 = time.perf_counter()
        sb.pp.scrublet(adata, batch_key="sample" if n_samples > 1 else None, verbose=False)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        rest = total - sum(STAGES.values())
        tag = "warm-up" if rep == 0 else f"rep {rep}"
        print(f"{tag}: call {total:.2f} s; " + ", ".join(f"{k} {v:.3f} s" for k, v in STAGES.items())
              + f", rest {rest:.2f} s; predicted doublets {int(np.nansum(adata.obs['predicted_doublet'].astype(float)))}")
    if n_samples == 1:
        emb = EMB["last"]
        m, d = emb.shape
        n_obs = int(adata.obs["doublet_score"].notna().sum())
        k_adj = _scrublet.k_adjusted(_scrublet.n_neighbors_default(n_obs), n_obs, m - n_obs)
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            _lc(emb, n_obs, k_adj)
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b) / 1e3)
        t = float(np.median(ts))
        flops = LC_PASSES * float(m) ** 2 * d * 3
        print(f"label count alone: n = {m} points, d = {d}, k_adj = {k_adj}: {t:.3f} s (median of {reps}); "
              f"{flops:.3g} distance FLOP -> {flops / t / 1e12:.1f} TFLOP/s = {100 * flops / t / FP32_PEAK:.0f} % of "
              "the 67 TFLOP/s FP32 data-sheet rate")


def oracle_10k():
    x = nb_counts(10_000, 2000, seed=2)
    t0 = time.perf_counter()
    x_obs, x_sim, parents, _ = osc.preprocess(x, rng=LegacyRng(0))
    emb = osc.embed(x_obs, x_sim)
    t_pre = time.perf_counter() - t0
    n_obs = x_obs.shape[0]
    k_adj = _scrublet.k_adjusted(_scrublet.n_neighbors_default(n_obs), n_obs, x_sim.shape[0])
    rows = np.arange(300)
    t0 = time.perf_counter()
    osc.label_count(emb, n_obs, k_adj, rows=rows)
    t_knn = (time.perf_counter() - t0) * emb.shape[0] / len(rows)
    print(f"\n== oracle (host, fp64) on one 10k-cell sample: preprocessing + PCA {t_pre:.1f} s, exact neighbour count "
          f"{t_knn:.0f} s (300 rows timed, scaled to {emb.shape[0]})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="A,B")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"GPU: {torch.cuda.get_device_name(0)}; nvidia-smi name, power limit, max SM clock: {q}")
    for key in args.cases.split(","):
        run_case(key, args.reps)
    if not args.no_oracle:
        oracle_10k()


if __name__ == "__main__":
    main()

"""Measurement of sb.metrics.morans_i / sb.metrics.gearys_c on an H100 (not a test; bench.py does not run it).

Two workloads, each a log-normalised float32 CSR from scanpy_b200._synth with its `sb.pp.neighbors` connectivities
(PCA 50, 15 neighbours): 1.3M cells x 2000 genes and 300k cells x 20,000 genes.  For each it prints the GPU name and
power limit, the call time of both metrics through the AnnData path (host CSR in), the device time of pass 1 (Σx and
the constancy flag, sb2_regress_col_sums) and of pass 2 (the graph sums, sb2_autocorr_sums) from CUDA events on the
resident inputs, the arc x gene terms per second of pass 2, and the oracle (oracle/autocorr.py, numpy on the host CPU)
timed on a sample of genes and extrapolated to all of them.  On the first workload pass 2 is also timed with X dense on
the device, which reads the same values without the per-arc slab searches of a CSR X.

Usage: python scripts/dev_autocorr.py [--reps 5] [--sample 16]
"""
import argparse
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import scanpy_b200 as sb  # noqa: E402
from oracle import autocorr as oac  # noqa: E402
from scanpy_b200 import _autocorr, _ops  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402


def event_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def run(n, g, reps, sample, dense_check):
    t0 = time.perf_counter()
    x, _ = synth_scipy(n, g, n_clusters=16, r=32, device="cuda")
    adata = sb.MiniAnnData(x)
    sb.pp.pca(adata, n_comps=50)
    sb.pp.neighbors(adata, n_neighbors=15)
    graph = adata.obsp["connectivities"]
    print(f"\n== {n} x {g}: X nnz {x.nnz} ({x.nnz / n / g:.1%}), graph arcs {graph.nnz} ({graph.nnz / n:.1f} per cell); "
          f"inputs made in {time.perf_counter() - t0:.0f} s")

    for name, metric in (("morans_i", sb.metrics.morans_i), ("gearys_c", sb.metrics.gearys_c)):
        ts = []
        for _ in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = metric(adata)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        print(f"{name} call (host CSR in, {out.shape[0]} values out): min {min(ts) * 1e3:.0f} ms over 2 calls")

    dgraph = _ops.DeviceX(graph, np.float64)
    dx = _ops.DeviceX(x, np.dtype(np.float32))
    mean, _ = _autocorr._means(dx, n, g)
    p1, _ = event_ms(lambda: _autocorr._means(dx, n, g), reps)
    p2, p2min = event_ms(lambda: _autocorr._sums(dgraph, dx, n, g, mean), reps)
    terms = float(graph.nnz + n) * g
    print(f"pass 1 (Σx, constancy): median {p1:.1f} ms; pass 2 (A, B, Q): median {p2:.1f} ms, min {p2min:.1f} ms over "
          f"{reps}; {terms:.3g} (arc + own value) x gene terms -> {terms / (p2 * 1e-3):.3g} terms/s")
    if dense_check:
        dd = _ops.DeviceX(torch.from_numpy(x.toarray()).cuda(), np.dtype(np.float32))
        pd_, _ = event_ms(lambda: _autocorr._sums(dgraph, dd, n, g, mean), reps)
        print(f"pass 2 with X dense on the device (no slab searches, {4 * g * (graph.nnz + n) / 1e9:.0f} GB of target "
              f"rows read through the caches): median {pd_:.1f} ms = {pd_ / p2:.2f} of the CSR pass")
        del dd
        torch.cuda.empty_cache()

    genes = np.random.default_rng(0).choice(g, sample, replace=False)
    xs = x[:, genes]
    t0 = time.perf_counter()
    oac.morans_i(graph, xs)
    oac.gearys_c(graph, xs)
    t_or = time.perf_counter() - t0
    print(f"oracle (numpy, host CPU, both metrics) on {sample} genes: {t_or:.1f} s -> EXTRAPOLATED to {g} genes: "
          f"{t_or * g / sample:.0f} s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=16)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {smi}")
    run(1_300_000, 2000, args.reps, args.sample, dense_check=True)
    run(300_000, 20_000, args.reps, args.sample, dense_check=False)


if __name__ == "__main__":
    main()

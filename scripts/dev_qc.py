"""Measurement of sb.pp.calculate_qc_metrics on an H100 (not a test; bench.py does not run it).

Two shapes: config C (1.3M cells x 2000 genes, integer counts derived from scanpy_b200._synth, ~100 stored values per
row) and a 10x-like wide shape (300k x 20,000 at 5 %, ~1000 stored values per row, where the top-500 selection does the
most work).  For each it prints the GPU name and power limit, the end-to-end call time (host CSR in, DataFrames out), the
device time of the row pass (sb2_csr_qc_rows_f32) and of the column pass (sb2_csr_col_counts_f32 + sb2_csr_col_sums_f32)
from CUDA events on a device-resident CSR, the bytes model 8 nnz + 8 (n+1) + outputs against 3.35 TB/s, a spot check
of sampled rows against the CPU oracle and the oracle's own time on a row slab.

Usage: python scripts/dev_qc.py [--shape C|wide|both] [--reps 20]
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
from oracle import qc as oqc  # noqa: E402
from scanpy_b200 import _abi, _ops  # noqa: E402
from scanpy_b200._abi import check, ptr  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM5 80GB data-sheet HBM3 bandwidth
PERCENT_TOP = (50, 100, 200, 500)


def config_c():
    x, _ = synth_scipy(1_300_000, 2000, device="cuda")
    x.data = np.rint(np.expm1(x.data)).astype(np.float32)  # log1p(CP10k) back to integer counts
    x.eliminate_zeros()
    return x


def wide(n=300_000, g=20_000, per_row=1000, seed=0):
    rng = np.random.default_rng(seed)
    stride = g // per_row  # one column per stride-wide band: sorted, unique, 5 % dense
    indices = (np.arange(per_row, dtype=np.int32) * stride + rng.integers(0, stride, (n, per_row), dtype=np.int32)).ravel()
    data = rng.geometric(0.3, n * per_row).astype(np.float32)
    indptr = np.arange(0, n * per_row + 1, per_row, dtype=np.int64)
    return sparse.csr_matrix((data, indices, indptr), shape=(n, g))


def device_times(x, qc_bits, reps):
    ctx = _abi.default_context()
    n, g = x.shape
    d_indptr, d_indices, d_data = _ops.csr_to_device(x)
    d_bits = _ops._to_device(qc_bits)
    ns = np.array(PERCENT_TOP, np.int32)
    cnt = torch.empty(n, dtype=torch.int64, device="cuda")
    tot = torch.empty(n, dtype=torch.float64, device="cuda")
    qc = torch.empty(n, dtype=torch.float64, device="cuda")
    top = torch.empty((n, ns.size), dtype=torch.float64, device="cuda")
    c = torch.empty(g, dtype=torch.int64, device="cuda")
    s1 = torch.empty(g, dtype=torch.float64, device="cuda")
    s2 = torch.empty(g, dtype=torch.float64, device="cuda")

    def rows():
        check(ctx.lib.sb2_csr_qc_rows_f32(ctx.handle, n, g, ptr(d_indptr), ptr(d_indices), ptr(d_data), 0, ptr(d_bits), 1,
                                          ptr(ns), ns.size, ptr(cnt), ptr(tot), ptr(qc), ptr(top)))

    def cols():
        check(ctx.lib.sb2_csr_col_counts_f32(ctx.handle, x.nnz, g, ptr(d_indices), ptr(d_data), 0, ptr(c)))
        check(ctx.lib.sb2_csr_col_sums_f32(ctx.handle, x.nnz, g, ptr(d_indices), ptr(d_data), 0, 1.0, ptr(s1), ptr(s2)))

    out = {}
    for name, fn in (("rows", rows), ("cols", cols)):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        out[name] = (float(np.median(ts)), float(np.min(ts)))
    return out


def run(name, x, reps):
    n, g = x.shape
    nnz = x.nnz
    print(f"\n== {name}: {n} x {g}, nnz {nnz} ({nnz / n:.0f} per row)")
    var = pd.DataFrame(index=[f"g{i}" for i in range(g)])
    var["mt"] = np.arange(g) % 50 == 0
    bits = var["mt"].to_numpy().astype(np.uint32)
    ad = sb.MiniAnnData(x, var=var)
    ts = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        obs, _ = sb.pp.calculate_qc_metrics(ad, qc_vars=["mt"])
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    print(f"end to end (host CSR in, DataFrames out): min {min(ts) * 1e3:.1f} ms over 3 calls")
    dt = device_times(x, bits, reps)
    row_bytes = 8 * nnz + 4 * nnz + 8 * (n + 1) + n * (8 + 8 + 8 + 8 * len(PERCENT_TOP))  # + indices for the mt mask
    col_bytes = 2 * 8 * nnz + 2 * 8 * g
    for key, nbytes in (("rows", row_bytes), ("cols", col_bytes)):
        med, best = dt[key]
        print(f"device {key} pass: median {med:.3f} ms, min {best:.3f} ms over {reps}; bytes model {nbytes / 1e9:.3f} GB "
              f"-> {nbytes / (med * 1e-3) / 1e12:.2f} TB/s = {nbytes / (med * 1e-3) / HBM_BPS:.0%} of 3.35 TB/s")
    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(n, 512, replace=False))
    sub = x[rows]
    ref, _ = oqc.calculate_qc_metrics(sub, obs_names=obs.index[rows], var=var, qc_vars=["mt"])
    got = obs.iloc[rows]
    worst = max(float(np.nanmax(np.abs(got[c].to_numpy(float) - ref[c].to_numpy(float)) /
                                np.maximum(np.abs(ref[c].to_numpy(float)), 1e-300))) for c in ref.columns)
    print(f"spot check, 512 sampled rows vs the CPU oracle: max relative difference {worst:.2e}")
    slab = x[:20_000]
    t0 = time.perf_counter()
    oqc.calculate_qc_metrics(slab, obs_names=obs.index[:20_000], var=var, qc_vars=["mt"])
    t = time.perf_counter() - t0
    print(f"CPU oracle (numpy restatement, single thread; not the reference) on 20,000 rows: {t:.2f} s "
          f"({t / 20_000 * n:.0f} s extrapolated to {n} rows)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="both", choices=("C", "wide", "both"))
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name())
    if a.shape in ("C", "both"):
        run("config C", config_c(), a.reps)
    if a.shape in ("wide", "both"):
        run("wide (10x-like)", wide(), a.reps)


if __name__ == "__main__":
    main()

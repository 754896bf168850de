"""Measurement of sb.get.aggregate on an H100 (not a test; bench.py does not run it).

Config C (1.3M cells x 2000 genes, log-normalised float32 CSR from scanpy_b200._synth) grouped two ways: about 250
groups (the 32 planted clusters x 8 samples) and 20,000 groups.  For each it prints the GPU name and power limit, then
from CUDA events:
* the whole call from a host CSR (upload, group order, device passes, download), for sum / mean / var / count_nonzero
  together and for median alone;
* the moments pass (sb2_aggregate_moments) and the median pass (sb2_aggregate_median) on the resident CSR, with the
  moments pass's bytes (the CSR's indices and values, the indptr twice, the order) over its time against 3.35 TB/s;
* the host-side scipy conversion a CSC X or `axis="var"` needs before the call (tocsr of the CSC, and of X.T);
and the fp64 oracle's time on the host CPU on a row subsample, extrapolated linearly to all rows.

Usage: python scripts/dev_aggregate.py [--reps 3] [--n 1300000]
"""
import argparse
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pandas as pd

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import scanpy_b200 as sb  # noqa: E402
from oracle import aggregate as oag  # noqa: E402
from scanpy_b200 import _abi, _aggregate, _ops  # noqa: E402
from scanpy_b200._abi import check, ptr  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM5 80GB data-sheet HBM3 bandwidth
SUBSAMPLE = 50_000


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


def host_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def run(x, codes, label, reps):
    n, g = x.shape
    n_groups = int(codes.max()) + 1
    print(f"\n== {n} x {g}, nnz {x.nnz}, {label}: {n_groups} groups "
          f"(rows per group {np.bincount(codes).min()}..{np.bincount(codes).max()})")
    obs = pd.DataFrame({"k": pd.Categorical.from_codes(codes, [f"k{i}" for i in range(n_groups)])})
    ad = sb.MiniAnnData(x, obs=obs)
    for funcs in (["sum", "mean", "var", "count_nonzero"], ["median"]):
        med, best = event_ms(lambda f=funcs: sb.get.aggregate(ad, "k", f), reps)
        print(f"call from host CSR, {'/'.join(funcs)}: median {med:.1f} ms, best {best:.1f} ms")

    ctx = _abi.default_context()
    dx = _ops.DeviceX(x, np.dtype(np.float32))
    d_order, offsets = _aggregate.group_order(codes.astype(np.int32), n_groups)
    groups = np.flatnonzero(np.diff(offsets))
    seg_row = np.append(offsets[groups], offsets[-1]).astype(np.int64)
    seg_group = groups.astype(np.int32)
    seg_n0 = np.zeros(groups.size, np.int64)
    acc = [torch.zeros((n_groups, g), dtype=torch.float64, device="cuda") for _ in range(3)]
    nnz = torch.zeros((n_groups, g), dtype=torch.int64, device="cuda")
    med_out = torch.empty((n_groups, g), dtype=torch.float32, device="cuda")
    xa = (None, dx.indptr, dx.indices, dx.data, d_order)

    def order():
        _aggregate.group_order(codes.astype(np.int32), n_groups)

    def moments():
        check(ctx.lib.sb2_aggregate_moments(ctx.handle, groups.size, seg_row.ctypes.data, seg_group.ctypes.data,
                                            seg_n0.ctypes.data, g, 0, *map(ptr, xa), *map(ptr, acc), ptr(nnz)))

    def median():
        check(ctx.lib.sb2_aggregate_median(ctx.handle, groups.size, seg_row.ctypes.data, seg_group.ctypes.data, g, 0,
                                           *map(ptr, xa), ptr(med_out)))

    o_ms, _ = event_ms(order, reps)
    m_ms, m_best = event_ms(moments, reps)
    d_ms, d_best = event_ms(median, max(1, reps // 2))
    nbytes = x.nnz * (4 + 4) + 2 * (n + 1) * 8 + n * 8 + 4 * n_groups * g * 8
    print(f"group order (incl. codes upload and offsets download): {o_ms:.2f} ms")
    print(f"moments pass: median {m_ms:.2f} ms, best {m_best:.2f} ms; {nbytes / 1e9:.2f} GB -> "
          f"{nbytes / (m_best * 1e-3) / 1e12:.2f} TB/s = {nbytes / (m_best * 1e-3) / HBM_BPS:.1%} of 3.35 TB/s")
    print(f"median pass: median {d_ms:.1f} ms, best {d_best:.1f} ms")

    sub = np.random.default_rng(0).choice(n, SUBSAMPLE, replace=False)
    xs, cs = x[sub], codes[sub]
    t0 = time.perf_counter()
    oag.sparse_moments(xs, cs, n_groups)
    t_or = time.perf_counter() - t0
    print(f"fp64 oracle moments (scipy, host CPU) on {SUBSAMPLE} rows: {t_or * 1e3:.0f} ms -> extrapolated to {n} "
          f"rows: {t_or * n / SUBSAMPLE:.1f} s (extrapolation, not measured)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_300_000)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"GPU: {q.stdout.strip()}  (torch: {torch.cuda.get_device_name(0)})")
    x, labels = synth_scipy(args.n, 2000, n_clusters=32, r=64, seed=0, device="cuda")
    x = x.tocsr()
    rng = np.random.default_rng(1)
    sample = rng.integers(0, 8, args.n)
    run(x, (np.asarray(labels) * 8 + sample).astype(np.int64), "32 clusters x 8 samples", args.reps)
    run(x, rng.integers(0, 20_000, args.n), "random", args.reps)

    csc = x.tocsc()
    print(f"\nhost conversion for a CSC X (scipy tocsr): {host_ms(lambda: csc.tocsr(), 2):.0f} ms")
    print(f"host conversion for axis='var' (X.T -> CSR): {host_ms(lambda: x.T.tocsr(), 2):.0f} ms")


if __name__ == "__main__":
    main()

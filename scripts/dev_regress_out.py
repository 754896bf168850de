"""Measurement of sb.pp.regress_out on an H100 (not a test; bench.py does not run it).

Config C (1.3M cells x 2000 genes, log-normalised CSR from scanpy_b200._synth, float32) with two numeric keys (the numpy
shortcut) and, separately, one 32-category key.  For each it prints the GPU name and power limit, the end-to-end call time
(host CSR in, host float32 / float64 ndarray out), the device time of the column-sum pass (sb2_regress_col_sums) and of
the residual pass (sb2_regress_residual) from CUDA events on the resident CSR, the bytes each pass must move against
3.35 TB/s, the share of the call spent copying the result to the host, a spot check of sampled rows against the oracle
and the reference's numpy shortcut timed on the host CPU on a row slab.

Usage: python scripts/dev_regress_out.py [--reps 10]
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
from oracle import regress as orr  # noqa: E402
from scanpy_b200 import _abi, _ops, _regress  # noqa: E402
from scanpy_b200._abi import check, ptr  # noqa: E402
from scanpy_b200._compat import settings  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM5 80GB data-sheet HBM3 bandwidth


def event_ms(fn, reps):
    for _ in range(2):
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


def run(name, x, obs, keys, reps):
    n, g = x.shape
    print(f"\n== {name}: {n} x {g}, nnz {x.nnz}, keys {keys}")
    ad = sb.MiniAnnData(x, obs=obs)
    ts, d2h = [], []
    for _ in range(3):
        ad.X = x
        _ops.TRANSFER["d2h"] = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sb.pp.regress_out(ad, keys)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
        d2h.append(_ops.TRANSFER["d2h"])
    out = ad.X
    print(f"end to end (host CSR in, host {out.dtype} ndarray out): min {min(ts) * 1e3:.0f} ms, "
          f"median {np.median(ts) * 1e3:.0f} ms over 3 calls; {d2h[-1] / 1e9:.2f} GB copied to the host")

    # device passes on the resident CSR, with the call's own host-side inputs
    ctx = _abi.default_context()
    dx = _regress._DeviceX(x, np.dtype(np.float32))
    categorical = keys == ["cat"]
    if categorical:
        codes = obs["cat"].cat.codes.to_numpy().astype(np.int32)
        n_groups = int(codes.max()) + 2
        order = np.lexsort((codes, np.arange(n) // _regress.TILE)).astype(np.int32)
        d_group, d_order = _ops._to_device(codes), _ops._to_device(order)
        width, d_w, p = n_groups, None, 0
        d_means = torch.zeros((n_groups - 1) * g, dtype=torch.float64, device="cuda")
        d_b0 = torch.zeros(g, dtype=torch.float64, device="cuda")
        d_b1 = torch.ones(g, dtype=torch.float64, device="cuda")
        out_f64, out_bytes = 1, 8
    else:
        a = orr.design(obs, keys).astype(np.float64)
        d_w, p, width = _ops._to_device(a), a.shape[1], a.shape[1]
        d_group = d_order = None
        d_coef = torch.zeros(p * g, dtype=torch.float64, device="cuda")
        out_f64, out_bytes = 0, 4
    acc = torch.zeros(width * g, dtype=torch.float64, device="cuda")
    mn, mx = torch.zeros(g, dtype=torch.float64, device="cuda"), torch.zeros(g, dtype=torch.float64, device="cuda")
    fl = torch.zeros(g, dtype=torch.int32, device="cuda")
    step = settings.chunk_size
    d_out = torch.empty((step, g), dtype=torch.float64 if out_f64 else torch.float32, device="cuda")

    def pass1():
        check(ctx.lib.sb2_regress_col_sums(ctx.handle, n, g, 0, None, ptr(dx.indptr), ptr(dx.indices), ptr(dx.data),
                                           ptr(d_w), p, ptr(d_group), ptr(d_order), width if categorical else 0,
                                           ptr(acc), ptr(mn), ptr(mx), ptr(fl)))

    def pass2():
        for r0 in range(0, n, step):
            r1 = min(n, r0 + step)
            if categorical:
                check(ctx.lib.sb2_regress_residual(ctx.handle, r1 - r0, g, 0, None, ptr(dx.indptr[r0:]), ptr(dx.indices),
                                                   ptr(dx.data), None, 0, None, ptr(d_group[r0:]), ptr(d_means),
                                                   ptr(d_b0), ptr(d_b1), None, out_f64, ptr(d_out)))
            else:
                check(ctx.lib.sb2_regress_residual(ctx.handle, r1 - r0, g, 0, None, ptr(dx.indptr[r0:]), ptr(dx.indices),
                                                   ptr(dx.data), ptr(d_w[r0:]), p, ptr(d_coef), None, None, None, None,
                                                   None, out_f64, ptr(d_out)))

    csr_bytes = 8 * x.nnz + 8 * (n + 1)
    b1 = csr_bytes + (8 * p * n if not categorical else 8 * n)
    b2 = csr_bytes + out_bytes * n * g + (8 * p * n if not categorical else 4 * n)
    t_pass = {}
    for label, fn, nbytes in (("column sums", pass1, b1), ("residual", pass2, b2)):
        med, best = event_ms(fn, reps)
        t_pass[label] = med
        print(f"device {label} pass: median {med:.2f} ms, min {best:.2f} ms over {reps}; bytes {nbytes / 1e9:.2f} GB -> "
              f"{nbytes / (med * 1e-3) / 1e12:.2f} TB/s = {nbytes / (med * 1e-3) / HBM_BPS:.0%} of 3.35 TB/s")
    dev = sum(t_pass.values()) * 1e-3
    print(f"device passes {dev * 1e3:.0f} ms = {dev / min(ts):.0%} of the call; the rest (copying {d2h[-1] / 1e9:.1f} GB "
          f"to the host, uploads, host algebra) {(min(ts) - dev) * 1e3:.0f} ms = {(min(ts) - dev) / min(ts):.0%}")
    # d2h alone: one block copy timed the way the call does it
    t0 = time.perf_counter()
    for r0 in range(0, n, step):
        _ops._to_host(d_out[: min(step, n - r0)])
    t_copy = time.perf_counter() - t0
    print(f"device->host copies of the result alone: {t_copy * 1e3:.0f} ms = {t_copy / min(ts):.0%} of the call "
          f"({n * g * out_bytes / t_copy / 1e9:.1f} GB/s)")

    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(n, 256, replace=False))
    if not categorical:  # the shortcut's residual of a row depends on all rows only through coeff
        coeff = np.linalg.inv(a.T @ a) @ np.asarray(x.T @ a).T
        ref = (x[rows].toarray() - a[rows] @ coeff).astype(np.float32)
        worst = float(np.max(np.abs(out[rows] - ref) / np.maximum(np.abs(ref), 1e-6)))
        print(f"spot check, 256 sampled rows vs a host restatement: max relative difference {worst:.2e}")
        slab = x[:100_000].toarray()
        t0 = time.perf_counter()
        orr.regress_out(slab, regressors=a[:100_000])
        t = time.perf_counter() - t0
        print(f"reference numpy shortcut (oracle restatement, host CPU) on 100,000 dense rows: {t:.2f} s "
              f"({t * n / 100_000:.0f} s extrapolated to {n} rows)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name())
    x, _ = synth_scipy(1_300_000, 2000, device="cuda")
    n = x.shape[0]
    rng = np.random.default_rng(0)
    obs = pd.DataFrame({"total_counts": np.ravel(x.sum(axis=1)), "pct_counts_mt": rng.random(n) * 10,
                        "cat": pd.Categorical.from_codes(rng.integers(0, 32, n), [f"b{i}" for i in range(32)])})
    run("two numeric keys (numpy shortcut)", x, obs, ["total_counts", "pct_counts_mt"], a.reps)
    run("one 32-category key", x, obs, ["cat"], a.reps)


if __name__ == "__main__":
    main()

"""Measurement of sb.pp.combat on an H100 (not a test; bench.py does not run it).

Config C (1.3M cells x 2000 genes, log-normalised CSR from scanpy_b200._synth, float32) with 8 and 64 batches, each
without covariates and with two numeric covariates.  For each it prints the GPU name and power limit, the end-to-end call
time (host CSR in, host float64 ndarray out), the device time of each pass from CUDA events on the resident CSR (DᵀX by
sb2_regress_col_sums grouped and weighted, the per-batch moments by sb2_combat_moments, the corrected matrix by
sb2_combat_adjust), the bytes each pass must move against 3.35 TB/s, the time of the device->host copies of the result,
and the oracle (the reference's dense numpy algorithm) timed on the host CPU on a 50,000-row subsample and extrapolated
linearly to all rows.

Usage: python scripts/dev_combat.py [--reps 5]
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
from oracle import combat as oc  # noqa: E402
from scanpy_b200 import _abi, _combat, _ops  # noqa: E402
from scanpy_b200._abi import check, ptr  # noqa: E402
from scanpy_b200._compat import settings  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM5 80GB data-sheet HBM3 bandwidth
SUBSAMPLE = 50_000


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


def run(x, obs, covariates, reps):
    n, g = x.shape
    nb = obs["batch"].nunique()
    print(f"\n== {n} x {g}, nnz {x.nnz}, {nb} batches, covariates {covariates or 'none'}")
    ad = sb.MiniAnnData(x, obs=obs)
    ts = []
    for _ in range(3):
        ad.X = x
        _ops.TRANSFER["d2h"] = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sb.pp.combat(ad, "batch", covariates=covariates or None)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    print(f"end to end (host CSR in, host float64 ndarray out): min {min(ts) * 1e3:.0f} ms, median "
          f"{np.median(ts) * 1e3:.0f} ms over 3 calls; {_ops.TRANSFER['d2h'] / 1e9:.2f} GB copied to the host")

    # the device passes on the resident CSR, with the call's own host-side inputs
    ctx = _abi.default_context()
    model = obs[["batch", *covariates]]
    levels, codes, counts = _combat.batch_groups(model, "batch")
    design = _combat.design_matrix(model, "batch", levels).to_numpy()
    cov = np.ascontiguousarray(design[:, nb:])
    p = cov.shape[1]
    dx = _ops.DeviceX(x, np.dtype(np.float32))
    order_g = np.lexsort((codes, np.arange(n) // _combat.TILE)).astype(np.int32)
    d_group, d_order_g = _ops._to_device(codes), _ops._to_device(order_g)
    order = np.argsort(codes, kind="stable")
    bounds = np.searchsorted(codes[order], np.arange(nb + 1))
    d_order = _ops._to_device(order.astype(np.int64))
    d_cov_sorted = _ops._to_device(np.ascontiguousarray(cov[order])) if p else None
    d_cov = _ops._to_device(cov) if p else None
    f64 = dict(dtype=torch.float64, device="cuda")
    acc_b, acc_w = torch.zeros(nb * g, **f64), torch.zeros(max(p, 1) * g, **f64)
    mn, mx, fl = torch.zeros(g, **f64), torch.zeros(g, **f64), torch.zeros(g, dtype=torch.int32, device="cuda")
    grand, beta = torch.zeros(g, **f64), torch.zeros(max(p, 1) * g, **f64)
    accs = torch.zeros((nb, 3, g), **f64)
    sv, dsq, gam = torch.ones(g, **f64), torch.ones(nb * g, **f64), torch.zeros(nb * g, **f64)
    step = settings.chunk_size
    d_out = torch.empty((step, g), **f64)

    def dtx_batch():
        check(ctx.lib.sb2_regress_col_sums(ctx.handle, n, g, 0, None, ptr(dx.indptr), ptr(dx.indices), ptr(dx.data),
                                           None, 0, ptr(d_group), ptr(d_order_g), nb, ptr(acc_b), ptr(mn), ptr(mx),
                                           ptr(fl)))

    def dtx_cov():
        check(ctx.lib.sb2_regress_col_sums(ctx.handle, n, g, 0, None, ptr(dx.indptr), ptr(dx.indices), ptr(dx.data),
                                           ptr(d_cov), p, None, None, 0, ptr(acc_w), ptr(mn), ptr(mx), ptr(fl)))

    def moments():
        for b in range(nb):
            k0, k1 = int(bounds[b]), int(bounds[b + 1])
            check(ctx.lib.sb2_combat_moments(ctx.handle, k1 - k0, g, 0, None, ptr(dx.indptr), ptr(dx.indices),
                                             ptr(dx.data), ptr(d_order[k0:k1]), ptr(d_cov_sorted[k0:] if p else None),
                                             p, ptr(grand), ptr(beta) if p else None, ptr(accs[b])))

    def adjust():
        for r0 in range(0, n, step):
            r1 = min(n, r0 + step)
            check(ctx.lib.sb2_combat_adjust(ctx.handle, r1 - r0, g, 0, None, ptr(dx.indptr[r0:]), ptr(dx.indices),
                                            ptr(dx.data), ptr(d_group[r0:]), ptr(d_cov[r0:] if p else None), p,
                                            ptr(grand), ptr(beta) if p else None, ptr(sv), ptr(gam), ptr(dsq),
                                            ptr(d_out)))

    csr = 8 * x.nnz + 8 * (n + 1)
    passes = [("DᵀX, batch columns (grouped)", dtx_batch, csr + 8 * n)]
    if p:
        passes.append((f"DᵀX, {p} covariate columns (weighted)", dtx_cov, csr + 8 * p * n))
    passes += [("per-batch moments", moments, csr + 8 * n + 8 * p * n),
               ("corrected matrix", adjust, csr + 8 * n * g + 4 * n + 8 * p * n)]
    dev = 0.0
    for label, fn, nbytes in passes:
        med, best = event_ms(fn, reps)
        dev += med
        print(f"device pass {label}: median {med:.2f} ms, min {best:.2f} ms over {reps}; bytes {nbytes / 1e9:.2f} GB -> "
              f"{nbytes / (med * 1e-3) / 1e12:.2f} TB/s = {nbytes / (med * 1e-3) / HBM_BPS:.0%} of 3.35 TB/s")
    print(f"device passes {dev:.0f} ms = {dev * 1e-3 / min(ts):.0%} of the call")
    t0 = time.perf_counter()
    for r0 in range(0, n, step):
        _ops._to_host(d_out[: min(step, n - r0)])
    t_copy = time.perf_counter() - t0
    print(f"device->host copies of the result alone: {t_copy * 1e3:.0f} ms = {t_copy / min(ts):.0%} of the call "
          f"({n * g * 8 / t_copy / 1e9:.1f} GB/s)")

    sub = x[:SUBSAMPLE]
    sub_design = design[:SUBSAMPLE]
    sub_idx = [np.flatnonzero(codes[:SUBSAMPLE] == b) for b in range(nb)]
    t0 = time.perf_counter()
    oc.combat(sub, sub_design, sub_idx)
    t = time.perf_counter() - t0
    print(f"oracle (the reference's dense numpy algorithm, host CPU) on the first {SUBSAMPLE} rows: {t:.2f} s; "
          f"EXTRAPOLATED linearly to {n} rows: {t * n / SUBSAMPLE:.0f} s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name())
    x, _ = synth_scipy(1_300_000, 2000, device="cuda")
    n = x.shape[0]
    rng = np.random.default_rng(0)
    for nb in (8, 64):
        obs = pd.DataFrame({"batch": pd.Categorical.from_codes(rng.integers(0, nb, n), [f"b{i}" for i in range(nb)]),
                            "total_counts": np.ravel(x.sum(axis=1)), "pct_counts_mt": rng.random(n) * 10})
        run(x, obs, [], a.reps)
        run(x, obs, ["total_counts", "pct_counts_mt"], a.reps)


if __name__ == "__main__":
    main()

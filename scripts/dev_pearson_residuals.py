"""Measurement of sb.experimental.pp (analytic Pearson residuals) on an H100 (not a test; bench.py does not run it).

Seeded negative-binomial integer counts as float32 CSR at two shapes: 1.3M x 2000 (the config C shape) and 300k x 20,000
with about 1000 stored values per row (selection runs on all genes), each with 1 and 8 batches.  It prints the GPU name
and power limit, then for each case:
* the device time of the residual-variance sweep (all batches) and of the residual writer (one settings.chunk_size
  block), from warmed-up CUDA events on the resident CSR;
* the sweep's fp64 rate from OPS_PER_RESIDUAL against the data sheet's FP64 (non-tensor) peak, and the writer's bytes/s
  against 3.35 TB/s;
* the end-to-end time of highly_variable_genes and normalize_pearson_residuals, with the share spent in device-to-host
  copies and in the host `check_values` test;
* the oracle's residual variance on a row slab, timed on the host and extrapolated to all rows;
* a spot check of sampled genes (variance) and rows (residuals) against fp64 numpy.

Usage: python scripts/dev_pearson_residuals.py [--reps 5] [--shapes A,B]
"""
import argparse
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
from scipy import sparse

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import scanpy_b200 as sb  # noqa: E402
from oracle import pearson as opr  # noqa: E402
from scanpy_b200 import _abi, _ops, _pearson  # noqa: E402
from scanpy_b200._abi import check, ptr  # noqa: E402
from scanpy_b200._compat import settings  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM5 80GB data-sheet HBM3 bandwidth
FP64_PEAK = 34e12  # H100 SXM5 data-sheet FP64 (non-tensor) FLOP/s
# per residual: mu = sg*sc/S (2), mu*mu/theta + mu (3), sqrt (1), (x - mu)/sqrt (2), clip (2 compares),
# shifted sums d, d*d (3), x*x + sq (2); a division or square root counts as one operation
OPS_PER_RESIDUAL = 15
SHAPES = {"A": (1_300_000, 2000, 200), "B": (300_000, 20_000, 1000)}


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
    return float(np.median(ts))


def nb_counts(n, g, per_row, seed=0):
    """CSR float32 with `per_row` stored values per row on average: NB(2) counts >= 1 at random positions."""
    rng = np.random.default_rng(seed)
    w = rng.lognormal(0, 1.5, g)
    w /= w.sum()
    nnz_row = rng.poisson(per_row, n).clip(1, g)
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(nnz_row, out=indptr[1:])
    cols = rng.choice(g, size=int(indptr[-1]), p=w).astype(np.int32)
    vals = (1 + rng.negative_binomial(2, 0.5, cols.size)).astype(np.float32)
    x = sparse.csr_matrix((vals, cols, indptr), shape=(n, g))
    x.sum_duplicates()
    return x


def timed_to_host(acc):
    inner = _ops._to_host

    def wrapped(*t):
        t0 = time.perf_counter()
        out = inner(*t)
        acc[0] += time.perf_counter() - t0
        return out

    return wrapped


def run(name, x, n_batches, reps):
    n, g = x.shape
    batch = np.random.default_rng(1).integers(0, n_batches, n) if n_batches > 1 else None
    print(f"\n== {name}: {n} x {g}, nnz {x.nnz} ({x.nnz / n:.0f} per row), {n_batches} batch(es)")
    # device time of the sweep over all batches on the resident CSR
    ctx = _abi.default_context()
    dx = _ops.DeviceX(x, np.dtype(np.float32))
    codes = np.zeros(n, np.int32) if batch is None else batch.astype(np.int32)
    gene_tot, d_cell = _pearson._totals(dx, n, g, codes, n_batches)
    order = np.argsort(codes, kind="stable")
    d_order = _ops._to_device(order.astype(np.int64))
    d_cells = _ops._to_device(_ops._to_host(d_cell)[order])
    bounds = np.searchsorted(codes[order], np.arange(n_batches + 1))
    d_genes = [_ops._to_device(gene_tot[b]) for b in range(n_batches)]
    acc = torch.zeros(4 * g, dtype=torch.float64, device="cuda")
    clip = float(np.sqrt(bounds[1] - bounds[0]))

    def sweep():
        acc.zero_()
        for b in range(n_batches):
            k0, k1 = int(bounds[b]), int(bounds[b + 1])
            check(ctx.lib.sb2_pearson_residual_var(ctx.handle, k1 - k0, g, 0, None, ptr(dx.indptr), ptr(dx.indices),
                                                   ptr(dx.data), ptr(d_order[k0:k1]), ptr(d_genes[b]),
                                                   ptr(d_cells[k0:k1]), float(gene_tot[b].sum()), clip, 100.0,
                                                   ptr(acc)))

    t_sweep = event_ms(sweep, reps)
    ops = float(n) * g * OPS_PER_RESIDUAL
    print(f"  sweep (sb2_pearson_residual_var): {t_sweep:.2f} ms, {ops / t_sweep / 1e9:.2f} TFLOP/s fp64 "
          f"({100 * ops / t_sweep / 1e-3 / FP64_PEAK:.1f} % of {FP64_PEAK / 1e12:.0f} TFLOP/s)")

    # device time of the writer on one chunk_size block
    rows = min(n, settings.chunk_size)
    d_out = torch.empty((rows, g), dtype=torch.float32, device="cuda")
    d_gene_all = _ops._to_device(gene_tot.sum(axis=0))
    total = float(gene_tot.sum())

    def writer():
        check(ctx.lib.sb2_pearson_residuals(ctx.handle, rows, g, 0, None, ptr(dx.indptr), ptr(dx.indices),
                                            ptr(dx.data), ptr(d_gene_all), ptr(d_cell), total, float(np.sqrt(n)), 100.0,
                                            0, ptr(d_out)))

    t_w = event_ms(writer, reps)
    nnz_rows = int(x.indptr[rows])
    moved = rows * g * 4 + nnz_rows * 8 + rows * 16
    print(f"  writer (sb2_pearson_residuals, {rows} rows): {t_w:.2f} ms, {moved / t_w / 1e9:.3f} TB/s "
          f"({100 * moved / t_w / 1e-3 / HBM_BPS:.1f} % of 3.35 TB/s)")
    del dx, d_out

    # end to end
    ad = sb.MiniAnnData(x)
    if batch is not None:
        ad.obs["batch"] = batch
    t0 = time.perf_counter()
    ok = _pearson.check_nonnegative_integers(x)
    t_check = time.perf_counter() - t0
    d2h = [0.0]
    orig = _ops._to_host
    _ops._to_host = timed_to_host(d2h)
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        df = sb.experimental.pp.highly_variable_genes(ad, n_top_genes=2000 if g > 2000 else 500,
                                                      batch_key="batch" if batch is not None else None,
                                                      inplace=False)
        t_hvg = time.perf_counter() - t0
        print(f"  highly_variable_genes end to end: {t_hvg:.3f} s; D2H {100 * d2h[0] / t_hvg:.1f} %, check_values "
              f"{100 * t_check / t_hvg:.1f} % (counts: {ok})")
        if n_batches == 1 and n * g <= 3e9:
            d2h[0] = 0.0
            t0 = time.perf_counter()
            res = sb.experimental.pp.normalize_pearson_residuals(ad, inplace=False)["X"]
            t_norm = time.perf_counter() - t0
            print(f"  normalize_pearson_residuals end to end: {t_norm:.3f} s ({res.nbytes / 1e9:.1f} GB float32); "
                  f"D2H {100 * d2h[0] / t_norm:.1f} %, check_values {100 * t_check / t_norm:.1f} %")
        else:
            res = None
    finally:
        _ops._to_host = orig

    # the oracle on a row slab, extrapolated (one batch of the slab's rows)
    slab = 2000
    xs = x[:slab].toarray().astype(np.float64)
    nz = xs.sum(axis=0) != 0
    t0 = time.perf_counter()
    opr.residual_variances(xs[:, nz], theta=100.0, clip=np.sqrt(slab))
    t_or = (time.perf_counter() - t0) * (n / slab) * (g / max(1, nz.sum()))
    print(f"  oracle (numpy fp64, two passes) extrapolated to all rows: {t_or:.1f} s")

    # spot check: sampled genes' residual variance (first batch) and sampled rows' residuals, against fp64 numpy
    rng = np.random.default_rng(5)
    rows_b = order[bounds[0]:bounds[1]]
    xb = x[rows_b]
    sg = gene_tot[0]
    sc = np.asarray(xb.sum(axis=1), dtype=np.float64).ravel()
    genes = rng.choice(np.flatnonzero(sg > 0), 8, replace=False)
    col = xb[:, genes].toarray().astype(np.float64)
    mu = np.outer(sc, sg[genes]) / np.sum(sg[sg != 0])
    r = opr._clip((col - mu) / np.sqrt(mu + mu * mu / 100.0), clip)
    got = df["residual_variances"].to_numpy()[genes] if n_batches == 1 else None
    if got is not None:
        rel = np.abs(got - r.var(axis=0)) / r.var(axis=0)
        print(f"  spot check, 8 genes: max relative difference of the residual variance {rel.max():.2e}")
    if res is not None:
        pick = rng.choice(n, 4, replace=False)
        allsc = np.asarray(x.sum(axis=1), dtype=np.float64).ravel()
        sg_all = gene_tot.sum(axis=0)
        mu = np.outer(allsc[pick], sg_all) / sg_all.sum()
        ref = opr._clip((x[pick].toarray() - mu) / np.sqrt(mu + mu * mu / 100.0), np.sqrt(n))
        ulp = np.abs(res[pick].astype(np.float64) - ref) / np.spacing(np.abs(ref).astype(np.float32))
        print(f"  spot check, 4 rows: max difference {ulp.max():.2f} float32 ulp")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default="A,B")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print(f"GPU: {torch.cuda.get_device_name(0)}; nvidia-smi name, power limit: {q}")
    for key in args.shapes.split(","):
        n, g, per_row = SHAPES[key]
        x = nb_counts(n, g, per_row, seed=0)
        for nb in (1, 8):
            run(f"shape {key}", x, nb, args.reps)
        del x


if __name__ == "__main__":
    main()

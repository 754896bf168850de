"""Measurement of sb2_csr_gram (G = X^T X in float64, the PCA's Gram operator) on an H100 (not a test; bench.py does not
run it).

Builds the benchmark's synthetic CSR (scanpy_b200._synth, 1.3M cells x 2000 genes by default) on the device and times
sb2_csr_gram with CUDA events over --reps calls after two warm-up calls.  It prints the GPU name, power limit and SM
clock read in the same run, the call time, and the bytes the row-by-row Gram design must move, computed from the shapes:
  index   the column index of the CSR: the count and scatter passes read the column indices three times and indptr
          twice, the scatter writes one 8-byte word per stored value, the accumulate kernel reads it back with x_ri;
  tails   the row tails the accumulate kernel reads, 8 bytes (column + value) per product x_ri x_rj (i <= j), from L2
          while the row chunk is resident;
  flush   one fp64 RED per G cell of the upper triangle per row chunk (at most).
HBM bytes are index + one read of the CSR + the flush; the tails are L2 traffic.

Usage: python scripts/dev_gram.py [--n-cells 1300000] [--n-genes 2000] [--reps 10]
"""
import argparse
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import scanpy_b200 as sb  # noqa: E402
from scanpy_b200 import _ops  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet
CHUNK_BYTES = 16 * 2**20  # GR_CHUNK_BYTES in csrc/pca.cu


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n-cells", type=int, default=1_300_000)
    p.add_argument("--n-genes", type=int, default=2000)
    p.add_argument("--reps", type=int, default=10)
    a = p.parse_args()
    n, g = a.n_cells, a.n_genes
    x, _ = synth_scipy(n, g, device="cuda")
    ctx = sb._abi.default_context()
    dp, di, dd = _ops.csr_to_device(x)
    gram = torch.empty((g, g), dtype=torch.float64, device="cuda")

    def call():
        sb._abi.check(ctx.lib.sb2_csr_gram(ctx.handle, n, g, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(gram)))

    for _ in range(2):
        call()
    ts = []
    for _ in range(a.reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        call()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e))
    state = gpu_state()
    ms = float(np.median(ts))

    nnz_r = np.diff(x.indptr).astype(np.float64)
    nnz = float(nnz_r.sum())
    products = float((nnz_r * (nnz_r + 1) / 2).sum())
    chunk_rows = 1024 * max(1, CHUNK_BYTES // max(1, int(8 * nnz) // n) // 1024)
    n_chunks = -(-n // chunk_rows)
    index = 3 * 4 * nnz + 2 * 8 * (n + 1) + 8 * nnz + 8 * nnz + 4 * nnz
    csr = 8 * nnz + 8 * (n + 1)
    flush = 8 * n_chunks * g * (g + 1) / 2
    tails = 8 * products
    hbm = index + csr + flush
    print(f"GPU: {state}")
    print(f"{n} x {g}, nnz {nnz:.4g} ({nnz / n:.1f} per row), {products:.4g} products, {n_chunks} row chunks of "
          f"{chunk_rows} rows")
    print(f"sb2_csr_gram: median {ms:.2f} ms, min {min(ts):.2f}, max {max(ts):.2f} over {a.reps} calls")
    print(f"bytes: index {index / 1e9:.2f} GB, CSR once {csr / 1e9:.2f} GB, flush <= {flush / 1e9:.2f} GB, "
          f"tails {tails / 1e9:.1f} GB (L2)")
    print(f"HBM side {hbm / 1e9:.2f} GB in {ms:.2f} ms = {hbm / (ms * 1e-3) / 1e12:.3f} TB/s "
          f"({hbm / (ms * 1e-3) / HBM_PEAK:.1%} of 3.35 TB/s); tails {tails / (ms * 1e-3) / 1e12:.2f} TB/s from L2")


if __name__ == "__main__":
    main()

"""The per-gene graph sums of `sc.metrics.morans_i` and `sc.metrics.gearys_c` on the device.

Reference: src/scanpy/metrics/_morans_i.py, _gearys_c.py.  For a feature x over the n cells (implicit zeros counted),
m = mean(x), z = x - m and the stored arcs i -> j of the graph with fp64 weights w:
  A = Σ_i z_i Σ_j w_ij z_j (the reference's `inum`),  B = Σ_i Σ_j w_ij (x_i - x_j)² (its `total`),  Q = Σ_i z_i².
Pass 1 is sb2_regress_col_sums with one weight column of ones (Σx, and the flag of the features whose values are all
equal); pass 2 is sb2_autocorr_sums (csrc/autocorr.cu).  Both read X with the cells along the rows.

The arcs reach arbitrary cells, so all of X's cells are on the device during pass 2.  A sparse X is uploaded once as
CSR.  A dense X goes up in column blocks: all n rows of a range of genes, a multiple of 256 wide and at most
`dense_bytes`, so device memory does not grow with n x g; each block is a complete X for both passes.  The graph goes up
once with float64 weights, and its rows go through pass 2 in blocks of whole subtiles (`partial_bytes` of partials).
The sums are bit-identical across runs, block sizes, and CSR, CSC or dense X of the same values.
"""
from __future__ import annotations

import numpy as np
from scipy import sparse

from . import _abi, _ops, _regress
from ._abi import check, ptr

DENSE_BYTES = 1 << 30    # device budget of one dense column block of X
PARTIAL_BYTES = 1 << 28  # device scratch for pass 2's per-subtile partials
SLAB = 256               # genes per CTA in both passes: dense column blocks are multiples of it


def _means(dx: _ops.DeviceX, n: int, g: int):
    """(fp64 mean of every gene, flag of the genes whose values are all equal and none NaN)."""
    sums, constant = _regress._col_sums(dx, n, g, w=np.ones((n, 1)))
    return sums[0] / n, constant


def _sums(dgraph: _ops.DeviceX, dx: _ops.DeviceX, n: int, g: int, mean: np.ndarray, *,
          partial_bytes: int = PARTIAL_BYTES) -> np.ndarray:
    """[A, B, Q] fp64 [3 x g] of the genes of `dx` (all n cells) over the graph `dgraph` (n x n, fp64 weights)."""
    import torch

    ctx = _abi.default_context()
    acc = torch.zeros(3 * g, dtype=torch.float64, device="cuda")
    d_mean = _ops._to_device(np.ascontiguousarray(mean, dtype=np.float64))
    d_x, d_xindptr, d_xindices, d_xdata = dx.block(0, n)
    step = _ops.subtile_block_rows(False, partial_bytes, 3 * g * 8)
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        check(ctx.lib.sb2_autocorr_sums(ctx.handle, r0, r1 - r0, g, dx.is_f64, ptr(d_x), ptr(d_xindptr),
                                        ptr(d_xindices), ptr(d_xdata), ptr(dgraph.indptr[r0:]), ptr(dgraph.indices),
                                        ptr(dgraph.data), ptr(d_mean), ptr(acc)))
    return _ops._to_host(acc).reshape(3, g)


def graph_sums(graph, x, *, dense_bytes: int = DENSE_BYTES, partial_bytes: int = PARTIAL_BYTES):
    """`graph` scipy CSR [n x n]; `x` [n x g] (cells along the rows) a float32 / float64 ndarray or scipy sparse matrix.
    -> ([A, B, Q] fp64 [3 x g], constant bool [g])."""
    n, g = x.shape
    vdtype = np.dtype(x.dtype)
    dgraph = _ops.DeviceX(graph, np.float64)
    if sparse.issparse(x):
        dx = _ops.DeviceX(x, vdtype)
        mean, constant = _means(dx, n, g)
        return _sums(dgraph, dx, n, g, mean, partial_bytes=partial_bytes), constant
    out = np.empty((3, g), dtype=np.float64)
    constant = np.empty(g, dtype=bool)
    width = max(SLAB, dense_bytes // max(1, n * vdtype.itemsize) // SLAB * SLAB)
    for c0 in range(0, g, width):
        c1 = min(g, c0 + width)
        dx = _ops.DeviceX(_ops._to_device(np.ascontiguousarray(x[:, c0:c1], dtype=vdtype)), vdtype)
        mean, constant[c0:c1] = _means(dx, n, c1 - c0)
        out[:, c0:c1] = _sums(dgraph, dx, n, c1 - c0, mean, partial_bytes=partial_bytes)
    return out, constant

"""The per-group statistics of `sc.get.aggregate` on the device (csrc/aggregate.cu).

Reference: src/scanpy/get/_aggregated.py (`Aggregate`).  The statistics are taken over the rows of X: a CSC X, or the
transposed X of `axis="var"`, is converted to CSR on the host with scipy first.  Then, on the device:
* `sb2_aggregate_group_order` sorts the kept rows by group (stable), giving each group's rows and count;
* `sb2_aggregate_moments` gives Σx, the mean, M2 and the count of x != 0 of every group in one pass over X;
* `sb2_aggregate_median` gives np.median per (group, gene) by radix selection.
A CSR X is uploaded once and read through the group order.  A dense X goes up in row blocks gathered in group order:
for the moments at most `settings.chunk_size` rows (rounded to whole subtiles, so a group longer than a block is cut
at subtile bounds and the result does not depend on the block size), for the median whole groups.

Integer X is sent as float64.  Its sums are exact integers when every group's Σ|x| stays below 2**53; that bound is
checked (max|x| times the largest group) before the pass, and integer input beyond it raises.
"""
from __future__ import annotations

import numpy as np
from scipy import sparse

from . import _abi, _ops
from ._abi import check, ptr

TILE = _ops.SUBTILE_ROWS  # SB2_AGGREGATE_TILE_ROWS
EXACT = 2.0**53


def value_dtype(x) -> np.dtype:
    """The dtype X goes to the device in; raises for what the kernels do not take."""
    dtype = np.dtype(x.dtype)
    if dtype.kind in "iu":
        return np.dtype(np.float64)
    if dtype not in (np.float32, np.float64):
        raise NotImplementedError(f"aggregate in scanpy_b200 supports float32, float64 and integer data, not {dtype}")
    return dtype


def _check_integer_bound(x, largest_group: int) -> None:
    vals = x.data if sparse.issparse(x) else np.asarray(x)
    if vals.size == 0 or largest_group == 0:
        return
    top = float(np.abs(vals.astype(np.float64, copy=False)).max())
    if top * largest_group >= EXACT:
        raise NotImplementedError(f"aggregate in scanpy_b200 sums integers exactly in float64 only while max|x| x the "
                                  f"largest group ({top:.0f} x {largest_group}) stays below 2**53")


def _dense_blocks(offsets: np.ndarray, groups: np.ndarray, step: int, *, whole: bool):
    """Row blocks of the group order for a dense X: lists of segments (group, first position, end position, rows of
    the group before the segment), at most `step` rows a block; a longer group is cut at multiples of TILE rows, or,
    with `whole`, gets a block of its own."""
    block, rows = [], 0
    for grp in groups:
        a, e = int(offsets[grp]), int(offsets[grp + 1])
        pieces = [(a, e)] if whole or e - a <= step else [(p, min(e, p + step)) for p in range(a, e, step)]
        for p0, p1 in pieces:
            if block and rows + (p1 - p0) > step:
                yield block
                block, rows = [], 0
            block.append((int(grp), p0, p1, p0 - a))
            rows += p1 - p0
    if block:
        yield block


def _segments(block, k0: int):
    seg_row = np.array([s[1] - k0 for s in block] + [block[-1][2] - k0], dtype=np.int64)
    seg_group = np.array([s[0] for s in block], dtype=np.int32)
    seg_n0 = np.array([s[3] for s in block], dtype=np.int64)
    return seg_row, seg_group, seg_n0


def group_order(codes: np.ndarray, n_groups: int):
    """-> (d_order int64 CUDA tensor, offsets int64 [n_groups + 1] host array): the kept rows by group, stable."""
    import torch

    ctx = _abi.default_context()
    n = codes.shape[0]
    d_codes = _ops._to_device(np.ascontiguousarray(codes, dtype=np.int32))
    d_order = torch.empty(max(n, 1), dtype=torch.int64, device="cuda")
    d_offsets = torch.empty(n_groups + 1, dtype=torch.int64, device="cuda")
    check(ctx.lib.sb2_aggregate_group_order(ctx.handle, n, ptr(d_codes), n_groups, ptr(d_order), ptr(d_offsets)))
    return d_order, _ops._to_host(d_offsets)


def group_stats(x, codes: np.ndarray, n_groups: int, *, moments: bool = True, median: bool = False) -> dict:
    """Per-group statistics of the rows of `x` (dense ndarray or scipy sparse; codes int [n_rows], -1: no group).

    -> dict(counts int64 [G], and with `moments` sum, mean, m2 fp64 [G x g] and nnz int64 [G x g], and with `median`
    median [G x g] in the value dtype of the device pass (float32 for float32 X, float64 otherwise)).  Groups without
    rows get zeros, and a NaN median."""
    import torch

    from ._compat import settings

    ctx = _abi.default_context()
    vdtype = value_dtype(x)
    if sparse.issparse(x):
        x = x.tocsr()
    n, g = x.shape
    d_order, offsets = group_order(codes, n_groups)
    counts = np.diff(offsets)
    if np.dtype(x.dtype).kind in "iu":
        _check_integer_bound(x, int(counts.max(initial=0)))
    groups = np.flatnonzero(counts)
    out = dict(counts=counts)
    if g == 0:
        return dict(out, sum=np.zeros((n_groups, 0)), mean=np.zeros((n_groups, 0)), m2=np.zeros((n_groups, 0)),
                    nnz=np.zeros((n_groups, 0), np.int64), median=np.zeros((n_groups, 0), vdtype))
    dx = _ops.DeviceX(x, vdtype)
    if moments:
        acc = [torch.zeros((n_groups, g), dtype=torch.float64, device="cuda") for _ in range(3)]
        nnz = torch.zeros((n_groups, g), dtype=torch.int64, device="cuda")
        if dx.dense is None:
            blocks = [[(int(grp), int(offsets[grp]), int(offsets[grp + 1]), 0) for grp in groups]] if groups.size else []
        else:
            step = max(1, int(settings.chunk_size) // TILE) * TILE
            blocks = list(_dense_blocks(offsets, groups, step, whole=False))
        for block in blocks:
            k0, k1 = (0, 0) if dx.dense is None else (block[0][1], block[-1][2])
            seg_row, seg_group, seg_n0 = _segments(block, k0)
            xa = _block_args(dx, d_order, offsets[-1], k0, k1)
            check(ctx.lib.sb2_aggregate_moments(ctx.handle, len(block), seg_row.ctypes.data, seg_group.ctypes.data,
                                                seg_n0.ctypes.data, g, dx.is_f64, *map(ptr, xa), *map(ptr, acc),
                                                ptr(nnz)))
        out.update(zip(("sum", "mean", "m2", "nnz"), _ops._to_host(*acc, nnz)))
    if median:
        mdt = torch.float64 if dx.is_f64 else torch.float32
        med = torch.full((n_groups, g), float("nan"), dtype=mdt, device="cuda")
        if dx.dense is None:
            blocks = [[(int(grp), int(offsets[grp]), int(offsets[grp + 1]), 0) for grp in groups]] if groups.size else []
        else:
            blocks = list(_dense_blocks(offsets, groups, max(1, int(settings.chunk_size)), whole=True))
        for block in blocks:
            k0, k1 = (0, 0) if dx.dense is None else (block[0][1], block[-1][2])
            seg_row, seg_group, _ = _segments(block, k0)
            xa = _block_args(dx, d_order, offsets[-1], k0, k1)
            check(ctx.lib.sb2_aggregate_median(ctx.handle, len(block), seg_row.ctypes.data, seg_group.ctypes.data, g,
                                               dx.is_f64, *map(ptr, xa), ptr(med)))
        out["median"] = _ops._to_host(med)
    return out


def _block_args(dx: _ops.DeviceX, d_order, kept: int, k0: int, k1: int):
    """(d_x, d_indptr, d_indices, d_data, d_order) of a call: the CSR read through the whole group order, or the dense
    rows at positions [k0, k1) of the order gathered on the host."""
    if dx.dense is None:
        return None, dx.indptr, dx.indices, dx.data, d_order[:max(int(kept), 1)]
    rows = _ops._to_host(d_order[k0:k1]) if k1 > k0 else np.zeros(0, np.int64)
    return _ops._to_device(np.ascontiguousarray(dx.dense[rows], dtype=dx.dtype)), None, None, None, None

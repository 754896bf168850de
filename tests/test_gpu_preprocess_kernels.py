"""The kernels of csrc/preprocess.cu (normalize_total, log1p, the seurat-HVG column sums, scale) called directly on CSR
and dense arrays built in numpy, against float64 restatements, at the shapes where they can go wrong: warp-per-row
kernels with a 32-lane stride and 8 rows per CTA, a grid-stride nnz loop with fp64 REDs into MV_COPIES = 32 copies,
64-row dense CTAs with a 256-column thread stride, one CTA per row for the CSR -> dense scale, and masks that switch
whole CTAs off.  Rows outside a mask hold 1e30, so any leak shows.

Tolerances come from the arithmetic.  u = 2^-24 is float32's unit round-off, 2^-53 float64's; an ulp of a value t is
2^-23·|t| (never less than the float32 spacing at t), with 2^-149 below the normal range.
* Row sums accumulate in fp64 in some order and round once to float32.  m terms summed in any order are within
  (m - 1)·2^-53·Σ|x| of the exact sum (math.fsum), so the device value is that sum rounded to float32 unless the sum
  lies that close to a float32 rounding midpoint; then either neighbour is accepted.
* hiexpr counts compare (double)x > max_fraction·(double)row_sum, as numba does: integer counts, equal.  Exact ties
  are built in and are not counted.
* Row scaling is one float32 division per entry (no fast-math in the Makefile): bit-exact with numpy.
* log1p: CUDA's log1pf is within 1 ulp, the fp64 division by ln b keeps that relative error and the final rounding adds
  half an ulp: 2 ulp of log1p(x)/ln b in float64.  0, -0, -1, x < -1, inf and NaN are exact (signs included, except a
  NaN's).
* expm1 column sums with one stored value per column: s1 is expm1f of the float32 argument (double)x·ln b rounded once,
  as numpy's `x *= np.log(base)` on float32 data does; expm1f is within 1 ulp of expm1 of that argument in float64, and
  s2 = s1·s1 is exact in fp64.  Arguments past 88.72 overflow to inf on both sides.
* Column sums in fp64: any order of the m terms of a column, then the 32 copies, is within (m + 32)·2^-53·Σ|v| of the
  exact sum.  The truth is summed in 80-bit long double (error m·2^-64·Σ|v|, 1/2048 of that bar), or with math.fsum
  where long double is no wider than double.
* Scale kernels do a double op, the cast, then the clip, exactly as oracle.preprocess.scale does when it is fed the
  same mean and std: bit-exact, with the rows outside the mask untouched.
"""
from __future__ import annotations

import math
import warnings

import numpy as np
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import preprocess as op
from scanpy_b200 import _abi, _ops
from scanpy_b200._abi import check, ptr

pytestmark = pytest.mark.gpu

E53 = 2.0**-53
OFF = np.float32(1e30)  # the value rows outside a mask hold
ROW_LENGTHS = [0, 1, 31, 32, 33, 63, 64, 65, 1000]
HUB = 200_003
# (n, length of row 0): n = 1 runs each row length alone; longer n cycle through them, with empty rows on both sides
# of the 8-row CTA edges and, at n = 4099, one hub row
ROW_CASES = [(1, m) for m in ROW_LENGTHS] + [(n, 0) for n in (7, 8, 9, 4099)]
ROW_IDS = [f"n1-len{m}" if n == 1 else f"n{n}" for n, m in ROW_CASES]
G_ROWS = 3001
MASKS = ["none", "on", "off", "alt", "cta64", "last"]


def _dev(a):
    return _ops._to_device(np.ascontiguousarray(a if a.size else np.zeros(1, a.dtype)))


def _call(name, *args):
    """Run entry point `name`: numpy arrays are uploaded (an empty one as one element, so its pointer is not NULL) and
    held until the call returns, torch tensors and None pass as pointers, everything else as it is."""
    ctx = _abi.default_context()
    held = [_dev(a) if isinstance(a, np.ndarray) else a for a in args]
    check(getattr(ctx.lib, name)(ctx.handle, *[ptr(a) if a is None or hasattr(a, "data_ptr") else a for a in held]))


def _host(t):
    return np.array(_ops._to_host(t))


def _empty(n, dtype):
    import torch

    return torch.empty(n, dtype=dtype, device="cuda")


def _values(rs, k):
    """float32 values over twelve decades, a fifth of them negative."""
    return (np.where(rs.rand(k) < 0.2, -1.0, 1.0) * 10.0 ** rs.uniform(-6, 6, k)).astype(np.float32)


def _row_lengths(n, first):
    if n == 1:
        return np.array([first], np.int64)
    lengths = np.resize(np.array(ROW_LENGTHS, np.int64), n)
    if n > 16:
        lengths[[7, 8, 15, 16, n - 2]] = 0
        lengths[2050 % n] = HUB
    return lengths


def _csr_arrays(n, first, rs, g=G_ROWS):
    lengths = _row_lengths(n, first)
    indptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    indices = rs.randint(0, g, int(indptr[-1])).astype(np.int32)
    return indptr, indices, _values(rs, indices.size)


def _mask(kind, n):
    r = np.arange(n)
    m = {"none": None, "on": np.ones(n, bool), "off": np.zeros(n, bool), "alt": r % 2 == 0,
         "cta64": ~((r >= 64) & (r < 128)), "last": r == n - 1}[kind]
    return m


def _ulp(t):
    return np.maximum(np.abs(t) * 2.0**-23, 2.0**-149)


def _float32_bracket(s, err):
    """The float32 values an fp64 result within err of s can round to: [f32(s - err), f32(s + err)]."""
    err = np.asarray(err) * (1 + 1e-6) + np.abs(s) * E53
    return (s - err).astype(np.float32), (s + err).astype(np.float32)


def _col_truth(cols, v, g):
    """-> (Σv, Σv², Σ|v|, count) per column, summed in long double (math.fsum if it is no wider than double)."""
    order = np.argsort(cols, kind="stable")
    cols, v = cols[order], v.astype(np.float64)[order]
    count = np.bincount(cols, minlength=g)
    starts = np.concatenate([[0], np.cumsum(count)[:-1]])
    out = np.zeros((3, g))
    hit = count > 0
    if np.finfo(np.longdouble).nmant >= 63:
        vl = v.astype(np.longdouble)
        for k, arr in enumerate((vl, vl * vl, np.abs(vl))):
            if v.size:
                out[k, hit] = np.add.reduceat(arr, starts[hit]).astype(np.float64)
    else:
        for c in np.flatnonzero(hit):
            seg = v[starts[c]:starts[c] + count[c]]
            out[:, c] = math.fsum(seg), math.fsum(seg * seg), math.fsum(np.abs(seg))
    return out[0], out[1], out[2], count


def _check_col_sums(s1, s2, cols, v, g):
    t1, t2, a1, m = _col_truth(cols, v, g)
    bar = (m + 32) * E53
    np.testing.assert_array_less(np.abs(s1 - t1), bar * a1 * (1 + 1e-9) + 1e-300)
    np.testing.assert_array_less(np.abs(s2 - t2), bar * t2 * (1 + 1e-9) + 1e-300)


# ---------------------------------------------------------------------------------------------- normalize_total rows
@pytest.mark.parametrize("skip", [False, True], ids=["all", "skip_cols"])
@pytest.mark.parametrize("n,first", ROW_CASES, ids=ROW_IDS)
def test_row_sums(n, first, skip):
    rs = np.random.RandomState(n * 131 + first)
    indptr, indices, data = _csr_arrays(n, first, rs)
    skip_cols = (rs.rand(G_ROWS) < 0.3).astype(np.int32) if skip else None
    out = _empty(n, _torch().float32)
    _call("sb2_csr_row_sums_f32", n, indptr, indices, data, skip_cols, out)
    got = _host(out)
    keep = np.ones(indices.size, bool) if not skip else skip_cols[indices] == 0
    s, err = np.zeros(n), np.zeros(n)
    for r in range(n):
        seg = data[indptr[r]:indptr[r + 1]][keep[indptr[r]:indptr[r + 1]]].astype(np.float64)
        s[r] = math.fsum(seg)
        err[r] = max(seg.size - 1, 0) * E53 * math.fsum(np.abs(seg))
    lo, hi = _float32_bracket(s, err)
    bad = np.flatnonzero((got < lo) | (got > hi))
    assert bad.size == 0, (bad[:5], got[bad[:5]], s[bad[:5]])


@pytest.mark.parametrize("max_fraction", [0.05, 0.25])
@pytest.mark.parametrize("n,first", ROW_CASES, ids=ROW_IDS)
def test_hiexpr_count_with_exact_ties(n, first, max_fraction):
    rs = np.random.RandomState(n * 17 + first)
    indptr, indices, _ = _csr_arrays(n, first, rs)
    data = rs.randint(1, 60, indices.size).astype(np.float32)
    rows = np.repeat(np.arange(n), np.diff(indptr))
    # row sums are an input: 1/max_fraction times an integer t, so t·(1/max_fraction)·max_fraction == t in fp64;
    # every third stored entry is set to its row's t, an exact tie
    t = rs.randint(1, 60, n).astype(np.float64)
    row_sums = (t * round(1 / max_fraction)).astype(np.float32)
    tie = np.arange(indices.size) % 3 == 0
    data[tie] = t[rows[tie]]
    thr = max_fraction * row_sums.astype(np.float64)
    assert (data[tie].astype(np.float64) == thr[rows[tie]]).all()
    ref = np.bincount(indices[data.astype(np.float64) > thr[rows]], minlength=G_ROWS).astype(np.int32)
    out = _empty(G_ROWS, _torch().int32)
    _call("sb2_csr_hiexpr_count_f32", n, G_ROWS, indptr, indices, data, row_sums, max_fraction, out)
    np.testing.assert_array_equal(_host(out), ref)


@pytest.mark.parametrize("n,first", ROW_CASES, ids=ROW_IDS)
def test_scale_rows_divides_by_one_for_a_zero_scale(n, first):
    rs = np.random.RandomState(n * 29 + first)
    indptr, _, data = _csr_arrays(n, first, rs)
    scale = (10.0 ** rs.uniform(-4, 4, n)).astype(np.float32)
    scale[np.arange(n) % 3 == 0] = 0  # row 0 of every case, and rows with entries at n > 1
    ref = data / np.repeat(np.where(scale == 0, np.float32(1), scale), np.diff(indptr))
    d_data = _dev(data)
    _call("sb2_csr_scale_rows_f32", n, indptr, d_data, scale)
    np.testing.assert_array_equal(_host(d_data)[:data.size], ref)


# ---------------------------------------------------------------------------------------------------------- log1p
def _log_inputs(rs):
    special = np.array([0.0, -0.0, -1.0, -1.5, -7.0, -np.inf, np.inf, np.nan, 1e-45, -1e-45, 1e-38, 3.4e38],
                       np.float32)
    parts = [special, rs.uniform(-1, 0, 30_000), 10.0 ** rs.uniform(-45, 38.5, 300_000), rs.uniform(0, 20, 300_000),
             -(10.0 ** rs.uniform(-45, 0, 30_000))]
    return np.concatenate([p.astype(np.float32) for p in parts])  # 660,012 values: not a multiple of 256


@pytest.mark.parametrize("base", [None, 2, np.e, 10, 0.5], ids=["none", "2", "e", "10", "0.5"])
def test_log1p_within_two_ulp(base):
    x = _log_inputs(np.random.RandomState(11))
    d = _dev(x)
    _call("sb2_log1p_f32", x.size, d, 0.0 if base is None else float(base))
    got = _host(d)
    with np.errstate(divide="ignore", invalid="ignore"):
        truth = np.log1p(x.astype(np.float64))
        if base is not None:
            truth = truth / np.log(base)
    t32 = truth.astype(np.float32)
    exact = (x == 0) | (x <= -1) | ~np.isfinite(x)
    np.testing.assert_array_equal(got[exact], t32[exact])
    num = exact & ~np.isnan(t32)
    np.testing.assert_array_equal(np.signbit(got[num]), np.signbit(t32[num]))
    rest = ~exact
    ulp = _ulp(truth[rest])
    err = np.abs(got[rest].astype(np.float64) - truth[rest])
    bad = np.flatnonzero(err > 2 * ulp)
    assert bad.size == 0, (x[rest][bad[:5]], got[rest][bad[:5]], truth[rest][bad[:5]])


def test_log1p_rejects_bad_bases():
    for b in (1.0, -2.0):
        with pytest.raises(_abi.B200Error, match="base"):
            _call("sb2_log1p_f32", 4, np.ones(4, np.float32), b)


# ------------------------------------------------------------------------------------------- HVG / PCA column sums
def _col_sums(cols, data, g, *, expm1=False, log_scale=1.0):
    torch = _torch()
    s1, s2 = _empty(g, torch.float64), _empty(g, torch.float64)
    _call("sb2_csr_col_sums_f32", data.size, g, cols, data, int(expm1), log_scale, s1, s2)
    return _host(s1), _host(s2)


@pytest.mark.parametrize("base", [None, 2, np.e, 10, 0.5], ids=["none", "2", "e", "10", "0.5"])
def test_col_sums_expm1_one_value_per_column(base):
    """s1 is the one expm1 value itself, so it shows the argument's rounding: a float32 multiply by (float)ln b would
    be up to ~x·ln b ulp off here."""
    ls = 1.0 if base is None else float(np.log(base))
    rs = np.random.RandomState(13)
    edge = np.float32(88.72283 / abs(ls))
    x = np.concatenate([rs.uniform(0, 13, 100_000), np.linspace(80, 95, 2001) / abs(ls),
                        edge + np.arange(-40, 41) * np.spacing(edge), [0.0, 1e-30, 200.0]]).astype(np.float32)
    g = x.size
    cols = rs.permutation(g).astype(np.int32)
    s1, s2 = _col_sums(cols, x, g, expm1=True, log_scale=ls)
    arg = x if base is None else (x.astype(np.float64) * ls).astype(np.float32)
    with np.errstate(over="ignore"):
        truth = np.expm1(arg.astype(np.float64))
        t32 = truth.astype(np.float32)
    got1, got2 = s1[cols], s2[cols]
    fmax = np.float64(np.finfo(np.float32).max)
    over = truth >= fmax * (1 - 2.0**-23)  # within one float32 ulp of the top: either side of the overflow
    assert over.any() == (ls > 0)
    ulp = _ulp(truth)
    ok = (got1 == t32) | (np.abs(got1 - truth) <= ulp) | (over & (got1 == np.inf))
    assert (got1[truth > 2 * fmax] == np.inf).all()  # well past the range: inf on both sides
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, (bad.size, x[bad[:5]], got1[bad[:5]], truth[bad[:5]])
    assert (got1.astype(np.float32) == got1).all()
    np.testing.assert_array_equal(got2, got1 * got1)


NNZ_CASES = ["0", "1", "255", "256", "257", "grid*256-1", "grid*256+1"]  # grid = SMs·8, the column-sum launch


def _nnz(name):
    if name.startswith("grid"):
        grid = _abi.default_context().device_info().sm_count * 8
        return grid * 256 + (1 if name.endswith("+1") else -1)
    return int(name)


@pytest.mark.parametrize("g", [1, 2, 257, 40_000])
@pytest.mark.parametrize("nnz_name", NNZ_CASES)
def test_col_sums_by_nnz(nnz_name, g):
    nnz = _nnz(nnz_name)
    rs = np.random.RandomState(nnz % 1000 + g)
    cols = rs.randint(0, g, nnz).astype(np.int32)
    v = _values(rs, nnz)
    s1, s2 = _col_sums(cols, v, g)
    _check_col_sums(s1, s2, cols, v, g)


@pytest.mark.parametrize("g", [1, 40_000])
def test_col_sums_thirty_million(g):
    """~3·10^7 values, all in one column at g = 1.  Multiples of 2^-6 below 16: every partial sum of v (< 2^29) and of
    v² (multiples of 2^-12 below 2^33) is exact in fp64, so the device sums must equal the exact ones."""
    nnz = 30_000_001
    rs = np.random.RandomState(g)
    cols = rs.randint(0, g, nnz).astype(np.int32)
    v = (rs.randint(-1023, 1024, nnz) / 64.0).astype(np.float32)
    s1, s2 = _col_sums(cols, v, g)
    v64 = v.astype(np.float64)
    np.testing.assert_array_equal(s1, np.bincount(cols, v64, minlength=g))
    np.testing.assert_array_equal(s2, np.bincount(cols, v64 * v64, minlength=g))


# ----------------------------------------------------------------------------------------------------- scale stats
def _u8(mask):
    return None if mask is None else mask.astype(np.uint8)


@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("n,first", ROW_CASES, ids=ROW_IDS)
def test_csr_col_stats_rows_masked(n, first, mask_kind):
    torch = _torch()
    rs = np.random.RandomState(n * 7 + first)
    indptr, indices, data = _csr_arrays(n, first, rs)
    mask = _mask(mask_kind, n)
    rows = np.repeat(np.arange(n), np.diff(indptr))
    on = np.ones(indices.size, bool) if mask is None else mask[rows]
    data[~on] = OFF
    s1, s2 = _empty(G_ROWS, torch.float64), _empty(G_ROWS, torch.float64)
    _call("sb2_csr_col_stats_rows_f32", n, G_ROWS, indptr, indices, data, _u8(mask), s1, s2)
    _check_col_sums(_host(s1), _host(s2), indices[on], data[on], G_ROWS)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("g", [1, 255, 256, 257, 513])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 2049, 5000])
def test_dense_col_stats(n, g, mask_kind, dtype):
    torch = _torch()
    rs = np.random.RandomState(n + g)
    x = _values(rs, n * g).reshape(n, g).astype(dtype)
    mask = _mask(mask_kind, n)
    if mask is not None:
        x[~mask] = OFF
    s1, s2 = _empty(g, torch.float64), _empty(g, torch.float64)
    _call("sb2_dense_col_stats", n, g, x, int(dtype == np.float64), _u8(mask), s1, s2)
    sel = x if mask is None else x[mask]
    cols = np.tile(np.arange(g, dtype=np.int32), sel.shape[0])
    _check_col_sums(_host(s1), _host(s2), cols, sel.ravel(), g)


# ------------------------------------------------------------------------------------------------------- scaling
def _stats(rs, g):
    mean = rs.uniform(-2, 2, g)
    std = 10.0 ** rs.uniform(-1, 1, g)
    std[::5] = 1.0
    return mean, std


@pytest.mark.parametrize("max_value", [None, 0.7])
@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("n,first", ROW_CASES, ids=ROW_IDS)
def test_csr_scale_cols(n, first, mask_kind, max_value):
    rs = np.random.RandomState(n * 3 + first)
    indptr, indices, data = _csr_arrays(n, first, rs)
    data = (data / np.float32(1e5)).astype(np.float32)  # within a few decades of the clip
    mask = _mask(mask_kind, n)
    rows = np.repeat(np.arange(n), np.diff(indptr))
    if mask is not None:
        data[~mask[rows]] = OFF
    mean, std = _stats(rs, G_ROWS)
    x = sparse.csr_matrix((data, indices, indptr), shape=(n, G_ROWS))
    ref, _, _ = op.scale(x, zero_center=False, max_value=max_value, mask_obs=mask, stats=(mean, std))
    d_data = _dev(data)
    _call("sb2_csr_scale_cols_f32", n, indptr, indices, d_data, std, _u8(mask), int(max_value is not None),
          max_value or 0.0)
    got = _host(d_data)[:data.size]
    np.testing.assert_array_equal(got, ref.data)
    if mask is not None:
        assert (got[~mask[rows]] == OFF).all()


def _full_rows_csr(rs, n, g):
    """Rows of 0 entries, of all g, and of a random unique subset in random order; values over a few decades."""
    lens = np.array([[0, g, rs.randint(0, g + 1)][r % 3] for r in range(n)])
    idx = [rs.permutation(g)[:k] for k in lens]
    indices = np.concatenate(idx).astype(np.int32) if lens.sum() else np.zeros(0, np.int32)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    data = (rs.standard_normal(indices.size) * 3).astype(np.float32)
    return indptr, indices, data


@pytest.mark.parametrize("max_value", [None, 0.7])
@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("g", [1, 255, 256, 257, 4097])
def test_csr_scale_to_dense(g, mask_kind, max_value):
    torch = _torch()
    n = 130
    rs = np.random.RandomState(g)
    indptr, indices, data = _full_rows_csr(rs, n, g)
    mask = _mask(mask_kind, n)
    mean, std = _stats(rs, g)
    x = sparse.csr_matrix((data, indices, indptr), shape=(n, g))
    out = _empty((n, g), torch.float64)
    _call("sb2_csr_scale_dense_f64", n, g, indptr, indices, data, mean, std, _u8(mask), int(max_value is not None),
          max_value or 0.0, out)
    got = _host(out)
    on = np.ones(n, bool) if mask is None else mask
    if on.any():
        ref, _, _ = op.scale(x[on], zero_center=True, max_value=max_value, stats=(mean, std))
        np.testing.assert_array_equal(got[on], ref)
    np.testing.assert_array_equal(got[~on], x[~on].toarray().astype(np.float64))


@pytest.mark.parametrize("max_value", [None, 0.7])
@pytest.mark.parametrize("zero_center", [True, False], ids=["centred", "uncentred"])
@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,g", [(1, 1), (63, 255), (130, 257), (2049, 513)])
def test_dense_scale(n, g, dtype, mask_kind, zero_center, max_value):
    assert (n * g) % 256 != 0
    rs = np.random.RandomState(n + g)
    x = (rs.standard_normal((n, g)) * 3).astype(dtype)
    mask = _mask(mask_kind, n)
    if mask is not None:
        x[~mask] = OFF
    mean, std = _stats(rs, g)
    ref, _, _ = op.scale(x, zero_center=zero_center, max_value=max_value, mask_obs=mask, stats=(mean, std))
    d_x = _dev(x)
    _call("sb2_dense_scale", n, g, d_x, int(dtype == np.float64), mean if zero_center else None, std, _u8(mask),
          int(max_value is not None), max_value or 0.0)
    got = _host(d_x)
    np.testing.assert_array_equal(got, ref)
    if mask is not None:
        assert (got[~mask] == OFF).all()


# -------------------------------------------------------------------------------------------------- public level
def _dup_counts_csr(rs, n, g, per_row):
    """Integer counts with duplicate (row, column) entries and unsorted columns in every row."""
    lens = rs.poisson(per_row, n)
    lens[::17] = 0
    indptr = np.concatenate([[0], np.cumsum(lens)])
    cols = rs.randint(0, g, indptr[-1])
    dup = rs.rand(cols.size) < 0.2
    cols[1:][dup[1:]] = cols[:-1][dup[1:]]  # repeat the previous entry's column (within a row, mostly)
    data = rs.randint(1, 30, cols.size).astype(np.float32)
    x = sparse.csr_matrix((data, cols.astype(np.int32), indptr), shape=(n, g))
    assert not x.has_canonical_format and not x.has_sorted_indices
    return x


@pytest.mark.parametrize("exclude", [False, True])
def test_normalize_total_and_log1p_on_duplicated_unsorted_csr(exclude):
    rs = np.random.RandomState(21)
    x = _dup_counts_csr(rs, 3000, 200, 40)
    x.data[x.indptr[5]:x.indptr[6]] = 0
    x.data[x.indptr[5]] = 1000  # one entry well above max_fraction of its row
    ad = sb.MiniAnnData(x.copy())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sb.pp.normalize_total(ad, exclude_highly_expressed=exclude, max_fraction=0.1, key_added="nf")
    ox, oc, subset = op.normalize_total(x, exclude_highly_expressed=exclude, max_fraction=0.1)
    if exclude:
        assert subset.any() and not subset.all()
    np.testing.assert_array_equal(ad.X.indices, x.indices)
    np.testing.assert_array_equal(ad.X.data, ox.data)
    np.testing.assert_array_equal(ad.obs["nf"].to_numpy(), oc)
    for base in (None, 2, 10):
        b = sb.pp.log1p(ad.X, base=base)
        o = op.log1p(ox, base=base)
        np.testing.assert_array_equal(b.indices, x.indices)
        # each side within 1.5 float32 ulp of log1p(x)/ln b
        assert (np.abs(b.data.astype(np.float64) - o.data) <= 3 * np.spacing(np.abs(o.data))).all()


def _dyadic_dup_csr(rs, n, g):
    """Duplicated, unsorted CSR of quarters below 16: the float32 sums of duplicates are exact."""
    x = _dup_counts_csr(rs, n, g, 30)
    x.data = (rs.randint(1, 64, x.nnz) / 4.0).astype(np.float32)
    return x


@pytest.mark.parametrize("max_value", [None, 2.5])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("zero_center", [True, False], ids=["centred", "uncentred"])
def test_scale_on_duplicated_unsorted_csr(zero_center, masked, max_value):
    rs = np.random.RandomState(23)
    n, g = 2000, 150
    x = _dyadic_dup_csr(rs, n, g)
    mask = (np.arange(n) % 5 != 3) if masked else None
    ad = sb.MiniAnnData(x.copy())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sb.pp.scale(ad, zero_center=zero_center, max_value=max_value, mask_obs=mask)
    names = ("mean with mask", "std with mask") if masked else ("mean", "std")
    got = ad.X
    if zero_center and masked:  # the masked rows are scaled by the dense branch, the others stay as they were
        ref_on, mean, std = op.scale(x[mask], zero_center=True, max_value=max_value)
        dense = got.toarray()
        np.testing.assert_allclose(dense[mask], ref_on, rtol=1e-12, atol=1e-12)
        np.testing.assert_array_equal(dense[~mask], x[~mask].toarray())
    else:
        ref, mean, std = op.scale(x, zero_center=zero_center, max_value=max_value, mask_obs=mask)
        if zero_center:
            np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
        else:  # per stored entry, as the reference's loop; its std may differ from the oracle's in the last bits
            np.testing.assert_array_equal(got.indices, x.indices)
            assert (np.abs(got.data.astype(np.float64) - ref.data) <= np.spacing(np.abs(ref.data))).all()
    np.testing.assert_allclose(ad.var[names[0]].to_numpy(), mean, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(ad.var[names[1]].to_numpy(), std, rtol=1e-12)


@pytest.mark.parametrize("base", [2, 10])
def test_hvg_on_log_base_data(base):
    rs = np.random.RandomState(base)
    counts = sparse.random(2000, 400, density=0.1, format="csr", random_state=rs,
                           data_rvs=lambda k: rs.poisson(4, k) + 1).astype(np.float32)
    counts = counts.multiply(rs.gamma(2.0, 1.0, (1, 400))).tocsr().astype(np.float32)  # gene-wise spread
    xn, _, _ = op.normalize_total(counts, target_sum=1e4)
    xl = op.log1p(xn, base=base)
    ad = sb.MiniAnnData(xl.copy())
    ad.uns["log1p"] = {"base": base}
    sb.pp.highly_variable_genes(ad, flavor="seurat")
    ref = op.hvg_seurat(xl, log_base=base)
    # Neither CUDA's expm1f nor numpy's float32 expm1 is correctly rounded (each within 1 ulp), so per value the two
    # differ by at most 2^-22·e, and e² by 2^-21·e²; the per-gene sums carry that into the mean, the variance and
    # log(var / mean).  2e-14 of the terms more covers the fp64 sums and the cancellation in E[x²] - E[x]².
    n, g = xl.shape
    e = np.expm1((xl.data.astype(np.float64) * np.log(base)).astype(np.float32).astype(np.float64))
    m = np.bincount(xl.indices, e, minlength=g) / n
    q = np.bincount(xl.indices, e * e, minlength=g) / n
    b1 = np.bincount(xl.indices, 2.0**-22 * e, minlength=g) / n
    b2 = np.bincount(xl.indices, 2.0**-21 * e * e, minlength=g) / n * (1 + 2.0**-20)
    var = (q - m * m) * n / (n - 1)
    bvar = (b2 + 2 * m * b1 + b1 * b1 + 2e-14 * q) * n / (n - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        bound_means = b1 / (1 + m) + 1e-15
        bound_disp = 1.01 * (bvar / var + b1 / m) + 1e-14
    for key, bound in (("means", bound_means), ("dispersions", bound_disp)):
        got_k, ref_k = ad.var[key].to_numpy(), ref[key].to_numpy()
        np.testing.assert_array_equal(np.isnan(got_k), np.isnan(ref_k))
        fin = ~np.isnan(ref_k)
        assert (np.abs(got_k - ref_k)[fin] <= bound[fin]).all(), (key, np.max(np.abs(got_k - ref_k)[fin] / bound[fin]))
    np.testing.assert_array_equal(ad.var["highly_variable"].to_numpy(), ref["highly_variable"].to_numpy())
    assert 0 < ad.var["highly_variable"].sum() < 400


def _torch():
    import torch

    return torch

"""oracle.preprocess pinned before the device tests lean on it (no GPU needed).

* normalize_total: the reference's numba `_normalize_csr` and `axis_mul_or_truediv` (_normalization.py:29-125,
  _utils/__init__.py:603-660) transcribed row by row, per stored entry, against the vectorised oracle: bit-identical.
* scale: the numba `scale_and_clip_csr` loop (_scale.py:267-283) transcribed row by row against the oracle's uncentred
  CSR branch, and the oracle's `stats=` shortcut against its own statistics: bit-identical.
* A CSR holding duplicate (row, column) entries: scipy's `multiply` / `mean` / `todense` sum duplicates before they
  square or subtract, so the oracle's scale statistics and its centred output are those of the `sum_duplicates()` form.
  pp.scale relies on this to canonicalise its input first.
"""
from __future__ import annotations

import numpy as np
import pytest
from scipy import sparse

from oracle import preprocess as op


def _dup_csr(rs, n, g, nnz, *, dyadic=True):
    """A float32 CSR with duplicate (row, column) entries and unsorted column indices."""
    rows = np.sort(rs.randint(0, n, nnz))
    cols = rs.randint(0, g, nnz)
    cols[: nnz // 4] = cols[nnz // 4: 2 * (nnz // 4)]  # force repeats within a row where the rows coincide
    rows[: nnz // 4] = rows[nnz // 4: 2 * (nnz // 4)]
    order = np.argsort(rows, kind="stable")
    rows, cols = rows[order], cols[order]
    vals = (rs.randint(1, 64, nnz) / 4.0 if dyadic else rs.lognormal(0, 1, nnz)).astype(np.float32)
    indptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))])
    x = sparse.csr_matrix((vals, cols.astype(np.int32), indptr), shape=(n, g))
    assert not x.has_canonical_format
    return x


def _normalize_loops(x, *, target_sum=None, exclude_highly_expressed=False, max_fraction=0.05):
    """`_normalize_csr` + `_normalize_total_helper` for a CSR, one stored entry at a time."""
    n, g = x.shape
    indptr, indices, data = x.indptr, x.indices, x.data
    counts = np.zeros(n, dtype=data.dtype)
    for i in range(n):
        count = 0.0
        for j in range(indptr[i], indptr[i + 1]):
            count += float(data[j])
        counts[i] = count
    per_col = np.zeros(g, np.int32)
    if exclude_highly_expressed:
        for r in range(n):
            for j in range(indptr[r], indptr[r + 1]):
                if float(data[j]) > max_fraction * float(counts[r]):
                    per_col[indices[j]] += 1
        for i in range(n):
            count = 0.0
            for j in range(indptr[i], indptr[i + 1]):
                if per_col[indices[j]] == 0:
                    count += float(data[j])
            counts[i] = count
    if target_sum is None:
        target_sum = np.median(counts[counts > 0])
    counts = counts / target_sum
    scaling = counts.copy() + (counts == 0)
    out = data.copy()
    for i in range(n):
        for j in range(indptr[i], indptr[i + 1]):
            out[j] = data[j] / scaling[i]
    return out, counts, (per_col == 0) if exclude_highly_expressed else None


@pytest.mark.parametrize("exclude", [False, True])
@pytest.mark.parametrize("target_sum", [None, 1e4])
def test_normalize_total_oracle_matches_the_row_loops(exclude, target_sum):
    rs = np.random.RandomState(3)
    x = sparse.random(300, 40, density=0.5, format="csr", random_state=rs,
                      data_rvs=lambda s: rs.uniform(1, 2, s)).astype(np.float32)
    x[5] = 0
    x.eliminate_zeros()
    x.data[x.indptr[9]] = 4 * x.data[x.indptr[9] + 1:x.indptr[10]].sum()  # one gene well above max_fraction
    xd = _dup_csr(rs, 300, 40, 3000, dyadic=False)
    for m, frac in ((x, 0.2), (xd, 0.6)):
        got, counts, subset = op.normalize_total(m, target_sum=target_sum, exclude_highly_expressed=exclude,
                                                 max_fraction=frac)
        data, ref_counts, ref_subset = _normalize_loops(m, target_sum=target_sum, exclude_highly_expressed=exclude,
                                                        max_fraction=frac)
        assert got.dtype == np.float32 and counts.dtype == np.float32
        np.testing.assert_array_equal(got.data, data)
        np.testing.assert_array_equal(got.indices, m.indices)
        np.testing.assert_array_equal(counts, ref_counts)
        if exclude:
            np.testing.assert_array_equal(subset, ref_subset)
            assert subset.any() and not subset.all()


def test_normalize_total_oracle_counts_duplicates_per_entry():
    """The exclusion test compares each stored entry, not the (row, column) sum: two entries of 3 in a row of total 10
    stay under max_fraction 0.5 although together they exceed it."""
    x = sparse.csr_matrix((np.array([3, 3, 4], np.float32), np.array([0, 0, 1]), np.array([0, 3])), shape=(1, 2))
    _, counts, subset = op.normalize_total(x, target_sum=1, exclude_highly_expressed=True, max_fraction=0.5)
    assert subset.tolist() == [True, True] and counts.tolist() == [10.0]


def _scale_and_clip_loops(x, std, mask, max_value):
    data = x.data.copy()
    for i in range(x.shape[0]):
        if mask[i]:
            for j in range(x.indptr[i], x.indptr[i + 1]):
                v = float(data[j]) / std[x.indices[j]]
                data[j] = min(max_value, v) if max_value is not None else v
    return data


@pytest.mark.parametrize("max_value", [None, 0.7, 2.5])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dup", [False, True])
def test_scale_and_clip_csr_oracle_matches_the_row_loop(max_value, masked, dup):
    rs = np.random.RandomState(5)
    if dup:
        x = _dup_csr(rs, 200, 30, 2000, dyadic=False)
    else:
        x = sparse.random(200, 30, density=0.3, format="csr", random_state=rs).astype(np.float32)
        x.data -= 0.3  # negative entries: the uncentred clip has no lower bound
    mask = (np.arange(200) % 3 != 1) if masked else np.ones(200, bool)
    got, mean, std = op.scale(x, zero_center=False, max_value=max_value, mask_obs=mask if masked else None)
    np.testing.assert_array_equal(got.data, _scale_and_clip_loops(x, std, mask, max_value))
    assert got.dtype == np.float32 and (got.indices == x.indices).all()
    again, m2, s2 = op.scale(x, zero_center=False, max_value=max_value, mask_obs=mask if masked else None,
                             stats=(mean, std))
    np.testing.assert_array_equal(again.data, got.data)
    assert (m2 == mean).all() and (s2 == std).all()


def test_scale_oracle_sums_duplicates_before_squaring():
    """A row holding (0: 1, 0: 2, 1: 3) is the row (3, 3): Σx² of column 0 is 9, not 1 + 4."""
    x = sparse.csr_matrix((np.array([1, 2, 3, 5], np.float32), np.array([0, 0, 1, 1]), np.array([0, 3, 4])),
                          shape=(2, 2))
    _, mean, std = op.scale(x, zero_center=False)
    np.testing.assert_array_equal(mean, [1.5, 4.0])
    # column 0 holds (3, 0): mean 1.5, Σx² = 9 -> var = (9/2 - 2.25) * 2 = 4.5
    np.testing.assert_array_equal(std, np.sqrt([4.5, 2.0]))


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("zero_center", [False, True])
def test_scale_oracle_treats_duplicates_as_their_sum(masked, zero_center):
    """Statistics (and the centred output) of a duplicated CSR equal those of its sum_duplicates() form.  The values
    are quarters below 16, so the float32 sums of duplicates are exact."""
    rs = np.random.RandomState(7)
    x = _dup_csr(rs, 400, 25, 5000)
    xc = x.copy()
    xc.sum_duplicates()
    assert xc.nnz < x.nnz
    mask = (np.arange(400) % 4 != 0) if masked else None
    if masked and zero_center:  # the oracle densifies the masked rows only through the dense branch
        sel = mask
        a, ma, sa = op.scale(x[sel], zero_center=True)
        b, mb, sb = op.scale(xc[sel], zero_center=True)
    else:
        a, ma, sa = op.scale(x, zero_center=zero_center, mask_obs=mask)
        b, mb, sb = op.scale(xc, zero_center=zero_center, mask_obs=mask)
    np.testing.assert_array_equal(ma, mb)
    np.testing.assert_array_equal(sa, sb)
    if zero_center:
        np.testing.assert_array_equal(a, b)
    else:  # the output keeps every stored entry, each divided on its own
        assert a.nnz == x.nnz and (a.indices == x.indices).all()

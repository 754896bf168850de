"""Connectivity oracles and host guards, without a device.

The fuzzy-set oracle (`oracle/fuzzy.py`, vectorised over rows) is pinned to a row-by-row transcription of umap-learn's
numba loops (tests/connectivity_cases.py) on k-lists that hold every row shape the kernel meets.  `gauss_reference` is
pinned to `gauss_knn`.  The guards of `pp.neighbors` and of the host k-list entry points all raise before any device
call, so they are checked here too.
"""
from __future__ import annotations

import numpy as np
import pytest
from scipy import sparse

import connectivity_cases as cc
import scanpy_b200 as sb
from oracle import connectivity as oconn, fuzzy as ofz
from scanpy_b200 import _ops, pp

U32 = 2.0**-24


@pytest.mark.parametrize("n,k", [(60, 8), (40, 33), (5, 9)])
@pytest.mark.parametrize("lc", [0.0, 0.5, 1.0, 1.5, 2.0])
def test_fuzzy_oracle_matches_umap_loops(n, k, lc):
    idx, dist = cc.fuzzy_case(n, k)
    d32 = dist.astype(np.float32)
    sig, rho, margin = ofz.smooth_knn_dist(d32, float(k), local_connectivity=lc)
    usig, urho = cc.umap_smooth_knn_dist(d32, float(k), local_connectivity=lc)
    np.testing.assert_array_equal(rho, urho)
    assert (margin > 0).all()
    # numba accumulates np.mean of float32 in float32; the oracle (like the kernel) sums in float64.  The two only
    # meet where the sigma floor 1e-3 * mean applies, and there a float32 sum of m non-negative terms is within
    # (m - 1) * 2^-24 of the exact one, plus one float32 rounding of the floor.
    mean_all = float(np.mean(d32.astype(np.float64)))
    floored = np.where(rho > 0, sig == np.float32(1e-3 * d32.astype(np.float64).mean(axis=1)), sig == np.float32(1e-3 * mean_all))
    np.testing.assert_array_equal(sig[~floored], usig[~floored])
    m = np.where(rho > 0, k, n * k)[floored]
    assert (np.abs(sig[floored] - usig[floored]) <= (m - 1) * U32 * sig[floored] + np.spacing(sig[floored])).all()
    for mix in (0.0, 0.25, 1.0):
        c, _, _ = ofz.fuzzy_simplicial_set(idx, dist, n, k, set_op_mix_ratio=mix, local_connectivity=lc)
        u = cc.umap_membership(idx, d32, sig, rho, n, set_op_mix_ratio=mix)
        c.sort_indices(), u.sort_indices()
        assert (c.indptr == u.indptr).all() and (c.indices == u.indices).all()
        # numpy's vectorised and scalar float32 exp may differ by an ulp; the union adds three float32 roundings
        np.testing.assert_allclose(c.data, u.data, rtol=8 * U32, atol=0)


def test_fuzzy_oracle_rounds_fractional_rho_once():
    # local_connectivity 0.3: rho = 0.3 * nz[0] in float64, rounded once; a float32 product rounds float32(0.3) instead
    x = np.float32(1.4236548)
    d = np.array([[0.0, x, 2.0, 3.0]], np.float32)
    _, rho, _ = ofz.smooth_knn_dist(d, 4.0, local_connectivity=0.3)
    _, urho = cc.umap_smooth_knn_dist(d, 4.0, local_connectivity=0.3)
    assert rho[0] == urho[0] == np.float32(0.3 * float(x)) != np.float32(0.3) * x


def test_fuzzy_oracle_margin_is_the_closest_decision():
    # every distance at rho: psum = k - 1 at each step, so the margin is |k - 1 - log2 k| - 0 or ... - 1e-5
    d = np.array([[0.0, 1.0, 1.0, 1.0, 1.0]], np.float32)
    _, _, margin = ofz.smooth_knn_dist(d, 5.0)
    gap = 4 - np.log2(5.0)
    assert margin[0] == min(gap, gap - 1e-5)


def test_gauss_reference_matches_gauss_knn():
    rs = np.random.RandomState(3)
    for n, k in ((50, 2), (60, 6), (70, 7), (80, 33)):
        idx = np.stack([np.r_[i, rs.choice(np.delete(np.arange(n), i), k - 1, replace=False)] for i in range(n)])
        dist = np.c_[np.zeros(n), rs.uniform(0.2, 2.0, (n, k - 1))]  # storage order: not sorted
        csr = sparse.csr_matrix((dist[:, 1:].ravel(), idx[:, 1:].ravel(), np.arange(0, n * (k - 1) + 1, k - 1)), shape=(n, n))
        ref = oconn.gauss_reference(csr, k)
        # the reference reads the CSR in column order; gauss_knn takes the same lists in that order
        srt = csr.copy(); srt.sort_indices()
        li = np.c_[np.arange(n), srt.indices.reshape(n, k - 1)]
        ld = np.c_[np.zeros(n), srt.data.reshape(n, k - 1)]
        g = oconn.gauss_knn(li, ld)
        assert abs(ref - g).max() == 0 and ref.nnz == g.nnz


def test_gauss_reference_dense_branch_is_not_the_sparse_rule():
    # the reason dense `distances` with method='gauss' is refused: sigma_i^2 = (largest k-list d^2) / 4, dense output
    rs = np.random.RandomState(4)
    x = rs.standard_normal((40, 3))
    full = np.sqrt(((x[:, None] - x[None]) ** 2).sum(-1))
    w = oconn.gauss_reference(full, 6)
    assert isinstance(w, np.ndarray) and w.shape == (40, 40)
    srt = np.sort(full, axis=1)[:, 1:6] ** 2
    i, j = 0, int(np.argsort(full[0])[1])
    s2 = srt[:, -1] / 4
    expect = np.sqrt(2 * np.sqrt(s2[i] * s2[j]) / (s2[i] + s2[j])) * np.exp(-full[i, j] ** 2 / (s2[i] + s2[j]))
    assert w[i, j] == pytest.approx(expect, rel=1e-14)
    o = np.argsort(full, axis=1)[:, :6]
    sp = oconn.gauss_knn(o, np.take_along_axis(full, o, 1)).toarray()
    assert abs(sp - w).max() > 1e-3


def test_gauss_reference_refuses_short_rows_like_the_reference():
    m = sparse.csr_matrix(np.array([[0, 1.0, 2.0, 0], [1.0, 0, 1.5, 2.5], [2.0, 1.5, 0, 1.0], [0, 2.5, 1.0, 0]]))
    with pytest.raises(ValueError):
        oconn.gauss_reference(m, 4)


# ------------------------------------------------------------------------------------------ host guards
def _ragged(n=300, seed=0, radius=1.2):
    from sklearn.neighbors import radius_neighbors_graph

    x = np.random.RandomState(seed).standard_normal((n, 5))
    return radius_neighbors_graph(x, radius, mode="distance")


def test_short_precomputed_rows_raise():
    d = _ragged()
    nnz = d.getnnz(axis=1)
    first = int(np.flatnonzero(nnz < 14)[0])
    with pytest.warns(RuntimeWarning, match="no constant number"), \
            pytest.raises(ValueError, match=rf"row {first} of the distance matrix stores {nnz[first]} "):
        pp._get_indices_distances_from_sparse_matrix(d, 15)
    with pytest.warns(RuntimeWarning), pytest.raises(ValueError, match=f"row {first} "):
        sb.pp.neighbors(sb.MiniAnnData(np.zeros((300, 2), np.float32)), n_neighbors=15, distances=d)
    # a one-entry row is refused too (the reference repeats that entry)
    one = sparse.csr_matrix(([1.0, 1.0, 2.0, 1.0, 2.0], ([0, 1, 1, 2, 2], [1, 0, 2, 0, 1])), shape=(3, 3))
    with pytest.warns(RuntimeWarning), pytest.raises(ValueError, match="row 0 .* stores 1 "):
        pp._get_indices_distances_from_sparse_matrix(one, 3)
    # constant rows shorter than n_neighbors - 1: the lists would be narrower than n_neighbors
    with pytest.raises(ValueError, match="stores 1 neighbour distances"):
        pp._get_indices_distances_from_sparse_matrix(sparse.csr_matrix(np.array([[0, 1.0], [1.0, 0]])), 3)


def test_long_precomputed_rows_keep_the_nearest():
    d = _ragged(seed=1, radius=3.0)
    nnz = d.getnnz(axis=1)
    k = int(nnz.min()) + 1  # every row long enough, most longer
    assert k >= 2 and (nnz > k - 1).mean() > 0.5
    with pytest.warns(RuntimeWarning):
        idx, dist = pp._get_indices_distances_from_sparse_matrix(d, k)
    assert idx.shape == (d.shape[0], k) and (idx[:, 0] == np.arange(d.shape[0])).all()
    for i in range(d.shape[0]):
        row = d[i]
        o = np.argsort(row.data)[: k - 1]
        np.testing.assert_array_equal(idx[i, 1:], row.indices[o])
        np.testing.assert_array_equal(dist[i, 1:], row.data[o])


@pytest.mark.parametrize("entry", ["fuzzy", "gauss", "jaccard"])
def test_repeated_ids_are_refused(entry):
    idx, dist = cc.fuzzy_case(20, 5)
    idx = idx.copy()
    idx[7, 3] = idx[7, 1]
    call = (lambda: _ops.fuzzy_simplicial_set(idx, dist)) if entry == "fuzzy" else \
        (lambda: _ops.knn_connectivities(idx, dist, entry))
    with pytest.raises(NotImplementedError, match=f"row 7 names neighbour {idx[7, 1]} more than once"):
        call()


def test_repeated_minus_one_ids_are_not_repeats():
    idx = np.array([[0, 1, -1, -1], [1, 0, -1, -1]])
    _ops._refuse_repeated_ids(idx)  # no raise


def test_precomputed_gauss_guards():
    ad = sb.MiniAnnData(np.zeros((6, 2), np.float32))
    full = np.abs(np.subtract.outer(np.arange(6.0), np.arange(6.0)))
    with pytest.raises(NotImplementedError, match="method='gauss' with dense `distances`"):
        sb.pp.neighbors(ad, n_neighbors=3, distances=full, method="gauss")
    wide = sparse.csr_matrix(full)  # 5 stored distances per row, n_neighbors - 1 = 2
    with pytest.raises(NotImplementedError, match="more than n_neighbors - 1"):
        sb.pp.neighbors(ad, n_neighbors=3, distances=wide, method="gauss")


@pytest.mark.parametrize("n_neighbors", [0, 1, 65, 100])
def test_precomputed_n_neighbors_out_of_range(n_neighbors):
    ad = sb.MiniAnnData(np.zeros((200, 2), np.float32))
    d = sparse.random(200, 200, density=0.6, format="csr", random_state=0)
    with pytest.raises(NotImplementedError, match=f"n_neighbors={n_neighbors} with `distances`"):
        sb.pp.neighbors(ad, n_neighbors=n_neighbors, distances=d)

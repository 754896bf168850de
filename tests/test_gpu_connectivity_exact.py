"""The connectivity kernels of csrc/graph.cu against exact restatements, on k-lists built in numpy (no kNN), so that
every row shape can be made: k = 2, the MK = 32 / 64 register lists at k = 32 / 33 and 64, rows in storage order,
duplicates, -1 ids, self not first or absent, hub rows past the 32-entry bitonic sort.

Tolerances come from the arithmetic.  u = 2^-24 is float32's unit round-off.
* rho takes the same float32 comparisons and copies as umap, so it is bit-exact at an integer local_connectivity.  At a
  fractional one umap rounds nz[i-1] + t * (nz[i] - nz[i-1]) once from float64 and the kernel forms it in float32: at
  most one float32 ulp apart (at t = 0.5, used here, the product is exact and both agree).
* sigma: the bisection runs in float64 on both sides and sums in the same order.  The device's exp and numpy's are
  each within 1 float64 ulp, so psum differs by at most ~k * 2^-52 < 1e-12.  A row whose oracle margin (its closest
  decision, `oracle.fuzzy.smooth_knn_dist`) exceeds 1e-12 takes every decision the same way and ends on the same mid:
  sigma is bit-exact there.  Any other row is held to the stopping rule itself: |psum(sigma) - log2 k| <= 1e-5 plus
  the change of psum over one float32 ulp of sigma.
* Membership: the kernel computes v = expf(-(d - rho) / sigma) with d - rho as in the restatement, one float32
  division (u relative in the argument x, so u·|x| relative in v) and CUDA's expf (2 ulp = 4u relative).  So the
  directed value is within e(v) = (|x| + 4)·u·v of the float64 exp(-x), recomputed from the device's own sigma and
  rho.  The union mix (a + b - ab) + (1 - mix) ab takes at most six float32 roundings of terms no larger than 2c,
  so C is within e(a) + e(b) + 6u·c; 2^-126 more covers float32 underflow.
* jaccard values are ratios of small integers in float64 and their average: bit-identical to the oracle.
* gauss: sqrt(num / den) * exp(-d^2 / den) with the same operation order as numpy; the two exps differ by at most
  2 ulp, the product adds 1: 4 float64 ulp.
"""
from __future__ import annotations

import numpy as np
import pytest
from scipy import sparse

import connectivity_cases as cc
import scanpy_b200 as sb
from oracle import connectivity as oconn, fuzzy as ofz
from scanpy_b200 import _abi, _ops
from scanpy_b200._abi import check, ptr

pytestmark = pytest.mark.gpu

U = 2.0**-24
TINY = 2.0**-126
KS = [2, 3, 31, 32, 33, 63, 64]
NS = [1, 2, 127, 128, 129, 4099]
LCS = [0.0, 0.5, 1.0, 1.5, 2.0]
MIXES = [0.0, 0.25, 1.0]


def _csr_ok(c):
    """Sorted, unique columns in every row and no explicit zeros."""
    assert c.has_sorted_indices and (c.data != 0).all()
    up = np.diff(c.indices) > 0
    ends = c.indptr[1:-1]
    up[ends[(ends > 0) & (ends < c.nnz)] - 1] = True  # a row may start below the previous row's end
    assert up.all()


def _directed_f64(idx, d32, sig, rho):
    """-> (rows, cols, v, e): the float64 membership of every list entry from the device's sigma / rho, and its bound."""
    n, k = idx.shape
    dd = d32 - rho[:, None]  # float32, as in the kernel
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        x = dd.astype(np.float64) / sig.astype(np.float64)[:, None]
        v = np.where((dd <= 0) | (sig[:, None] == 0), 1.0, np.exp(-x))
    e = np.where((dd <= 0) | (sig[:, None] == 0), 0.0, (np.abs(x) + 4) * U * v)
    selfc = idx == np.arange(n)[:, None]
    v[selfc], e[selfc] = 0.0, 0.0
    keep = idx >= 0
    rows = np.repeat(np.arange(n), k).reshape(n, k)
    return rows[keep], idx[keep], v[keep], e[keep]


def _union_ref(idx, d32, sig, rho, mix):
    n = idx.shape[0]
    r, c, v, e = _directed_f64(idx, d32, sig, rho)
    a = sparse.csr_matrix((v, (r, c)), shape=(n, n))
    ea = sparse.csr_matrix((e, (r, c)), shape=(n, n))
    p = a.multiply(a.T)
    ref = mix * (a + a.T - p) + (1.0 - mix) * p
    bound = ea + ea.T + 6 * U * abs(ref)
    return ref.tocsr(), bound.tocsr(), a


def _psum(d32, rho, sig, k):
    dd = (d32[:, 1:] - rho[:, None]).astype(np.float64)
    with np.errstate(over="ignore", divide="ignore"):
        return np.where(dd > 0, np.exp(-(dd / np.asarray(sig, np.float64)[:, None])), 1.0).sum(axis=1)


# ------------------------------------------------------------------------------------------ fuzzy_rows_kernel + union
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("k", KS)
def test_fuzzy_rows_and_union(n, k):
    idx, dist = cc.fuzzy_case(n, k)
    d32 = dist.astype(np.float32)
    kinds_seen = {cc.KINDS[i % 9] for i in range(n)}
    for lc in [x for x in LCS if x < k]:
        osig, orho, margin = ofz.smooth_knn_dist(d32, float(k), local_connectivity=lc)
        for mix in MIXES:
            c, sig, rho = _ops.fuzzy_simplicial_set(idx, dist, set_op_mix_ratio=mix, local_connectivity=lc)
            if lc == int(lc):
                np.testing.assert_array_equal(rho, orho)
            else:
                assert (np.abs(rho - orho) <= np.spacing(orho)).all()
            exact = (margin > 1e-12) & (rho == orho)
            np.testing.assert_array_equal(sig[exact], osig[exact])
            rest = np.flatnonzero(~exact)
            if len(rest):
                floor = np.where(rho > 0, 1e-3 * d32.astype(np.float64).mean(axis=1),
                                 1e-3 * d32.astype(np.float64).mean())[rest]
                ps = _psum(d32[rest], rho[rest], sig[rest], k)
                ps_up = _psum(d32[rest], rho[rest], sig[rest] + np.spacing(sig[rest]), k)
                ok = (np.abs(ps - np.log2(k)) <= 1e-5 + np.abs(ps_up - ps)) | (sig[rest] == np.float32(floor))
                assert ok.all(), rest[~ok]
            _csr_ok(c)
            assert abs(c - c.T).max() == 0 and c.dtype == np.float32
            ref, bound, a = _union_ref(idx, d32, sig, rho, mix)
            dev = c.astype(np.float64)
            extra = dev.copy(); extra.data[:] = 1
            extra = extra - extra.multiply(ref != 0)
            assert extra.count_nonzero() == 0  # no device entry where the restatement has none
            big = ref.copy(); big.data = (big.data > 2**-120).astype(float); big.eliminate_zeros()
            missing = big - big.multiply(dev != 0)
            assert missing.count_nonzero() == 0
            over = abs(dev - ref) - bound
            assert over.max() <= TINY if over.nnz else True
    if n >= 9:  # every row shape, and both mutual and non-mutual edges (at mix = 1 the latter store a itself)
        assert kinds_seen == set(cc.KINDS)
        mutual = a.multiply(a.T != 0)
        assert mutual.count_nonzero() > 0 and (a - mutual).count_nonzero() > 0


def test_fuzzy_capacity_without_self_and_without_mutual_edges():
    # lists of k real neighbours (no self column), none mutual: the union has 2 n k entries
    n, k = 1000, 5
    idx = ((np.arange(n)[:, None] + 1 + np.arange(k)[None] * 7) % n).astype(np.int32)
    assert not any(i in set(idx[j].tolist()) for i in range(n) for j in idx[i])
    dist = np.sort(np.random.RandomState(0).uniform(0.5, 1.5, (n, k)), axis=1)
    c, sig, rho = _ops.fuzzy_simplicial_set(idx, dist)
    assert c.nnz == 2 * n * k and abs(c - c.T).max() == 0
    ref, bound, _ = _union_ref(idx, dist.astype(np.float32), sig, rho, 1.0)
    assert (abs(c.astype(np.float64) - ref) - bound).max() <= TINY


# ------------------------------------------------------------------------------------------ symmetrize through jaccard
def _star_graph(lengths=(31, 32, 33, 64, 5000)):
    """k = 3 lists.  Hub h lists (a, b), a lists (h, b), b lists (h, a), and L leaves list (h, a): rows h and a get
    L + 2 entries, a leaf row 2.  One more cell links to a leaf only (a 1-entry row) and one has no shared neighbour
    with its list (an empty row)."""
    lists = []
    for length in lengths:
        h = len(lists)
        a, b = h + 1, h + 2
        lists += [[h, a, b], [a, h, b], [b, h, a]]
        for _ in range(length - 2):
            lists.append([len(lists), h, a])
    leaf = 3
    one = len(lists)
    lists.append([one, leaf, 1])  # J[one, leaf] = |{leaf, 1} & {0, 1}| = 1; J[one, 1] = |{leaf, 1} & {0, 2}| = 0
    empty = len(lists)
    lists.append([empty, 4, 5])  # leaves 4, 5 list (0, 1): nothing shared with {4, 5}
    return np.array(lists, np.int32), one, empty


def _jaccard_bitwise(idx):
    c = _ops.knn_connectivities(idx, np.zeros(idx.shape), "jaccard")
    c2 = _ops.knn_connectivities(idx, np.zeros(idx.shape), "jaccard")
    o = oconn.jaccard(idx).tocsr()
    o.sort_indices(); o.eliminate_zeros()
    _csr_ok(c)
    assert (c.indptr == o.indptr).all() and (c.indices == o.indices).all() and (c.data == o.data).all()
    assert (c.indptr == c2.indptr).all() and (c.indices == c2.indices).all() and (c.data == c2.data).all()
    assert (c != c.T).nnz == 0
    return c


def test_symmetrize_row_lengths_and_hub():
    idx, one, empty = _star_graph()
    c = _jaccard_bitwise(idx)
    lens = np.diff(c.indptr)
    assert {0, 1, 31, 32, 33, 64, 5000} <= set(lens.tolist())
    assert lens[one] == 1 and lens[empty] == 0


@pytest.mark.parametrize("k", [3, 31, 32, 33, 64])
def test_symmetrize_random_lists(k):
    n = 3000
    rs = np.random.RandomState(k)
    idx = np.stack([np.r_[i, cc._neighbours(rs, n, i, k - 1)] for i in range(n)]).astype(np.int32)
    # self not first in every 7th row: the reference keeps its diagonal J[i, i] = 1
    sn = np.arange(0, n, 7)
    idx[sn, 0], idx[sn, 1] = idx[sn, 1], sn
    c = _jaccard_bitwise(idx)
    np.testing.assert_array_equal(c.diagonal()[sn], 1.0)
    assert (np.delete(c.diagonal(), sn) == 0).all()


def test_symmetrize_fully_non_mutual_and_empty():
    n, k = 500, 4
    idx = np.c_[np.arange(n), (np.arange(n)[:, None] + np.arange(1, k)[None]) % n].astype(np.int32)
    c = _jaccard_bitwise(idx)  # i -> i+1, i+2, i+3: none mutual; i+1 shares 2, i+2 shares 1, i+3 shares none
    assert c.nnz == 2 * n * (k - 2)
    idx2 = np.c_[np.arange(n), (np.arange(n) + 1) % n].astype(np.int32)
    c2 = _jaccard_bitwise(idx2)  # k = 2: no two single-neighbour sets share
    assert c2.nnz == 0


# ------------------------------------------------------------------------------------------ gauss
@pytest.mark.parametrize("k", [2, 3, 4, 7, 8, 32, 33, 64])
@pytest.mark.parametrize("order", ["ascending", "storage"])
def test_gauss_within_4_ulp(k, order):
    n = 2000
    rs = np.random.RandomState(k)
    idx = np.stack([np.r_[i, cc._neighbours(rs, n, i, k - 1)] for i in range(n)]).astype(np.int32)
    dist = np.c_[np.zeros(n), np.sort(rs.uniform(0.3, 2.0, (n, k - 1)), axis=1) * rs.uniform(0.5, 2, (n, 1))]
    if order == "storage":
        p = np.argsort(rs.rand(n, k - 1), axis=1) + 1
        idx[:, 1:] = np.take_along_axis(idx, p, 1)
        dist[:, 1:] = np.take_along_axis(dist, p, 1)
    # self not first, a duplicate at distance 0 first (at k = 2 self would be the only entry and its sigma 0)
    sn = np.arange(5, n, 11) if k > 2 else np.arange(0)
    idx[sn, 0], idx[sn, 1] = idx[sn, 1], sn
    dist[sn, 1] = 0.0
    c = _ops.knn_connectivities(idx, dist, "gauss")
    o = oconn.gauss_knn(idx, dist).tocsr()
    o.sort_indices(); o.eliminate_zeros()
    _csr_ok(c)
    assert (c.indptr == o.indptr).all() and (c.indices == o.indices).all()
    assert (np.abs(c.data - o.data) <= 4 * np.spacing(np.abs(o.data))).all()
    assert (c.diagonal()[sn] == o.diagonal()[sn]).all() and (c.diagonal()[sn] > 0).all()


def test_gauss_duplicate_flood_gives_the_oracles_nans():
    n, k = 300, 6
    rs = np.random.RandomState(0)
    idx = np.stack([np.r_[i, cc._neighbours(rs, n, i, k - 1)] for i in range(n)]).astype(np.int32)
    dist = np.c_[np.zeros(n), np.sort(rs.uniform(0.3, 2.0, (n, k - 1)), axis=1)]
    for i in range(k + 1):  # k + 1 identical cells that list each other: sigma = 0, 0 / 0 between them
        others = [j for j in range(k + 1) if j != i][: k - 1]
        idx[i] = [i] + others
        dist[i] = 0.0
    c = _ops.knn_connectivities(idx, dist, "gauss")
    o = oconn.gauss_knn(idx, dist).tocsr()
    o.sort_indices(); o.eliminate_zeros()
    assert (c.indptr == o.indptr).all() and (c.indices == o.indices).all()
    nan = np.isnan(o.data)
    assert nan.sum() >= k * (k - 1) and (np.isnan(c.data) == nan).all()
    assert (np.abs(c.data[~nan] - o.data[~nan]) <= 4 * np.spacing(np.abs(o.data[~nan]))).all()


# ------------------------------------------------------------------------------------------ sb2_group_arc_counts
@pytest.mark.parametrize("G", [1, 300])
def test_group_arc_counts_exact(G):
    import torch

    rs = np.random.RandomState(G)
    lens = np.r_[0, 1, 31, 32, 33, 5000, rs.randint(0, 70, 2000)]
    n = len(lens)
    indptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    indices = rs.randint(0, n, indptr[-1]).astype(np.int32)
    codes = rs.randint(0, G, n).astype(np.int32)
    codes[rs.rand(n) < 0.05] = -1
    codes[rs.rand(n) < 0.05] = G + rs.randint(0, 3)
    if G == 1:  # one group, mostly: row 5's 5,000 arcs all land in one MATCH.ANY class
        codes[:] = 0
        codes[rs.rand(n) < 0.05] = -1
    ctx = _abi.default_context()
    d_counts = torch.empty((G, G), dtype=torch.int64, device="cuda")
    d_ip, d_ix, d_cd = (_ops._to_device(a) for a in (indptr, indices, codes))
    check(ctx.lib.sb2_group_arc_counts(ctx.handle, n, ptr(d_ip), ptr(d_ix), ptr(d_cd), G, ptr(d_counts)))
    got = _ops._to_host(d_counts)
    rows = np.repeat(np.arange(n), lens)
    gi, gj = codes[rows], codes[indices]
    ok = (gi >= 0) & (gi < G) & (gj >= 0) & (gj < G)
    ref = np.zeros((G, G), np.int64)
    np.add.at(ref, (gi[ok], gj[ok]), 1)
    np.testing.assert_array_equal(got, ref)


# ------------------------------------------------------------------------------------------ public paths
def _knn_csr(n, k, rs, width=None):
    """Constant-width CSR without self, columns sorted (scipy order), width stored distances per row."""
    width = width or k - 1
    idx = np.stack([np.sort(cc._neighbours(rs, n, i, width)) for i in range(n)])
    d = rs.uniform(0.3, 2.0, (n, width))
    return sparse.csr_matrix((d.ravel(), idx.ravel(), np.arange(0, n * width + 1, width)), shape=(n, n))


@pytest.mark.parametrize("method", ["umap", "jaccard", "gauss"])
@pytest.mark.parametrize("wide", [False, True])
def test_precomputed_distances_match_the_reference(method, wide):
    from oracle import knn as oknn

    if method == "gauss" and wide:
        pytest.skip("refused: tests/test_connectivity_host_cpu.py::test_precomputed_gauss_guards")
    n, k = 1500, 12
    rs = np.random.RandomState(7)
    d = _knn_csr(n, k, rs, width=k + 8 if wide else None)
    ad = sb.MiniAnnData(np.zeros((n, 2), np.float32))
    sb.pp.neighbors(ad, n_neighbors=k, distances=d, method=method)
    got = ad.obsp["connectivities"]
    li, ld = oknn.indices_distances_from_sparse(d, k)  # shortcut: storage (column) order, truncated
    if method == "umap":
        o, _, _ = ofz.fuzzy_simplicial_set(li, ld, n, k)
        o = o.tocsr(); o.sort_indices()
        assert (got.indices == o.indices).all() and (got.indptr == o.indptr).all()
        np.testing.assert_allclose(got.data, o.data, rtol=2e-6, atol=1e-7)
    elif method == "jaccard":
        o = oconn.jaccard(li).tocsr(); o.sort_indices(); o.eliminate_zeros()
        assert (got.indices == o.indices).all() and (got.data == o.data).all()
    else:
        o = oconn.gauss_reference(d, k).tocsr(); o.sort_indices(); o.eliminate_zeros()
        assert (got.indices == o.indices).all() and (got.indptr == o.indptr).all()
        assert (np.abs(got.data - o.data) <= 4 * np.spacing(np.abs(o.data))).all()


def test_transformer_with_duplicate_cells_keeps_jaccards_diagonal():
    from sklearn.neighbors import KNeighborsTransformer

    from scanpy_b200 import pp

    rs = np.random.RandomState(3)
    x = rs.standard_normal((600, 8)).astype(np.float32)
    x[300:400] = x[:100]  # duplicated cells
    k = 10
    ad = sb.MiniAnnData(x)
    tr = KNeighborsTransformer(n_neighbors=k, mode="distance")
    sb.pp.neighbors(ad, transformer=tr, method="jaccard", use_rep="X")
    got = ad.obsp["connectivities"]
    li, _ = pp._get_indices_distances_from_sparse_matrix(tr.fit_transform(x), k)
    assert (li[:, 0] != np.arange(600)).any()  # some row starts with its duplicate
    o = oconn.jaccard(li).tocsr(); o.sort_indices(); o.eliminate_zeros()
    assert (got.indices == o.indices).all() and (got.data == o.data).all()
    np.testing.assert_array_equal(got.diagonal(), o.diagonal())
    assert (o.diagonal() == 1).sum() > 0

"""sc.get.aggregate on the H100: the reference's tests (tests/test_aggregated.py) restated on the pbmc68k counts, every
func against the fp64 oracle (oracle/aggregate.py) across formats, dtypes, masks and NA labels, the variance's
cancellation case, median edge cases, and scale and determinism."""
import warnings

import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import aggregate as oag
from scanpy_b200 import _abi, _aggregate
from scanpy_b200._compat import MiniAnnData, settings
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

FUNCS = ["count_nonzero", "sum", "median", "mean", "var"]
FMTS = {"csr": sparse.csr_matrix, "csc": sparse.csc_matrix, "dense": np.asarray}


def pbmc(fmt="csr", dtype=np.float32, *, with_na=False, unused=False):
    """The 700 x 765 pbmc68k counts, grouped by bulk_labels x louvain."""
    x = ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts").tocsr().astype(np.float32)
    x = FMTS[fmt](x if fmt != "dense" else x.toarray()).astype(dtype)
    bulk = np.load(GOLDEN / "pbmc68k_regress.npz")["bulk_labels_codes"]
    louv = np.load(GOLDEN / "pbmc68k_reduced_graph.npz")["louvain_codes"]
    obs = pd.DataFrame({"bulk": pd.Categorical([f"b{c}" for c in bulk]),
                        "louvain": pd.Categorical(louv.astype(str))}, index=[f"c{i}" for i in range(x.shape[0])])
    if unused:
        obs["louvain"] = obs["louvain"].cat.add_categories(["unused"])
    if with_na:
        obs.iloc[list(range(0, x.shape[0], 5)), obs.columns.get_loc("louvain")] = np.nan
    return MiniAnnData(x, obs=obs, var=pd.DataFrame(index=[f"g{i}" for i in range(x.shape[1])]))


def ref_median(x, codes, n_groups):
    """np.median per group in X's own dtype (the reference's arithmetic: float32 stays float32)."""
    dense = x.toarray() if sparse.issparse(x) else np.asarray(x)
    out = np.full((n_groups, dense.shape[1]), np.nan)
    for k in range(n_groups):
        rows = dense[codes == k]
        if rows.shape[0]:
            out[k] = np.median(rows, axis=0)
    return out


def expected(x, obs, keys, func, *, mask=None, dof=1):
    names, codes, counts = oag.group_codes(obs, keys, mask)
    st = oag.dense_stats(x, codes, len(names), median=False)
    return names, counts, dict(sum=st["sum"], count_nonzero=st["nnz"], mean=st["mean"],
                               var=oag.variance(st["m2"], counts, dof), median=ref_median(x, codes, len(names)))


def assert_matches(got, ref, func, *, exact):
    assert got.shape == ref.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    if exact or func in ("count_nonzero", "median"):
        np.testing.assert_array_equal(got, ref)
    else:
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-300)


# ------------------------------------------------------------------------------------------ vs the oracle
@pytest.mark.parametrize("func", FUNCS)
@pytest.mark.parametrize("fmt", list(FMTS))
@pytest.mark.parametrize("use_mask", [True, False], ids=["masked", "unmasked"])
@pytest.mark.parametrize("with_na", [True, False], ids=["na", "no_na"])
@pytest.mark.parametrize("unused", [True, False], ids=["unused_kept", "no_unused"])
def test_aggregate_vs_oracle(func, fmt, use_mask, with_na, unused):
    ad = pbmc(fmt, with_na=with_na, unused=unused)
    kw = {}
    if use_mask:
        mask = np.ones(ad.shape[0], dtype=bool)
        mask[::4] = False
        kw["mask"] = mask
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        res = sb.get.aggregate(ad, ["bulk", "louvain"], func, **kw)
        names, counts, exp = expected(ad.X, ad.obs, ["bulk", "louvain"], func, mask=kw.get("mask"))
    assert res.obs.index.tolist() == names.tolist()
    assert res.obs["n_obs_aggregated"].tolist() == counts.tolist()
    assert_matches(res.layers[func], exp[func], func, exact=False)


@pytest.mark.parametrize("fmt", list(FMTS))
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int64])
def test_formats_and_dtypes(fmt, dtype):
    ad = pbmc(fmt, dtype)
    res = sb.get.aggregate(ad, ["bulk", "louvain"], FUNCS)
    names, counts, exp = expected(ad.X, ad.obs, ["bulk", "louvain"], None)
    integer = np.dtype(dtype).kind == "i"
    for f in FUNCS:
        assert_matches(res.layers[f], exp[f], f, exact=f == "sum" and integer)
    sp = fmt != "dense"
    assert res.layers["sum"].dtype == (np.int64 if sp and integer else np.float64)
    assert res.layers["count_nonzero"].dtype == (np.int64 if sp else np.float64)
    assert res.layers["median"].dtype == (np.float32 if not sp and dtype == np.float32 else np.float64)


@pytest.mark.parametrize("fmt", list(FMTS))
@pytest.mark.parametrize("func", FUNCS)
def test_aggregate_axis(fmt, func):
    ad = pbmc(fmt)
    ex = sb.get.aggregate(ad, ["louvain"], func)
    t = MiniAnnData(ad.X.T, obs=ad.var, var=ad.obs)
    got = sb.get.aggregate(t, ["louvain"], func, axis=1).T
    assert got.obs.index.tolist() == ex.obs.index.tolist()
    assert got.obs["n_obs_aggregated"].tolist() == ex.obs["n_obs_aggregated"].tolist()
    np.testing.assert_array_equal(got.layers[func], ex.layers[func])


@pytest.mark.parametrize("axis", [0, 1])
def test_mask(axis):
    ad = pbmc("csr")
    mask = (ad.obs["louvain"] == "0").to_numpy()
    ad.obs["mask_col"] = mask
    if axis == 1:
        ad = MiniAnnData(ad.X.T.tocsr(), obs=ad.var, var=ad.obs)
    by_ref = sb.get.aggregate(ad, "louvain", "sum", axis=axis, mask="mask_col")
    by_value = sb.get.aggregate(ad, "louvain", "sum", axis=axis, mask=mask)
    np.testing.assert_array_equal(by_ref.layers["sum"], by_value.layers["sum"])
    s = by_ref.layers["sum"] if axis == 0 else by_ref.layers["sum"].T
    names = (by_ref.obs if axis == 0 else by_ref.var).index.tolist()
    assert (s[names.index("0")] > 0).any()
    assert (np.delete(s, names.index("0"), axis=0) == 0).all()


@pytest.mark.parametrize("fmt", ["dense", "csr"])
def test_var_no_catastrophic_cancellation(fmt):
    rng = np.random.default_rng(0)
    x = np.vstack([1e8 + 1e-3 * rng.standard_normal((1000, 4)) for _ in range(2)])
    obs = pd.DataFrame({"group": pd.Categorical(np.repeat(["a", "b"], 1000))}, index=[f"c{i}" for i in range(2000)])
    ad = MiniAnnData(FMTS[fmt](x), obs=obs, var=pd.DataFrame(index=[f"g{i}" for i in range(4)]))
    want = np.vstack([np.var(x[:1000], axis=0), np.var(x[1000:], axis=0)])
    np.testing.assert_allclose(sb.get.aggregate(ad, "group", "var", dof=0).layers["var"], want, rtol=1e-4)


# ------------------------------------------------------------------------------------------ median edge cases
def median_case(x, codes):
    n_groups = int(codes.max()) + 1
    obs = pd.DataFrame({"k": pd.Categorical(codes.astype(str), categories=[str(i) for i in range(n_groups)])},
                       index=[f"c{i}" for i in range(x.shape[0])])
    return MiniAnnData(x, obs=obs, var=pd.DataFrame(index=[f"g{i}" for i in range(x.shape[1])]))


@pytest.mark.parametrize("fmt", ["dense", "csr"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_median_edges(fmt, dtype):
    rng = np.random.default_rng(3)
    sizes = [1, 2, 3, 4, 7, 10, 1025, 2048, 333]
    codes = np.repeat(np.arange(len(sizes)), sizes)
    rng.shuffle(codes)
    n, g = codes.size, 70
    x = rng.choice([-3.5, -1.0, 0.0, 0.0, 0.0, 1.0, 2.0, 2.0, 7.25], size=(n, g)).astype(dtype)
    x[:, 0] = 0.0                                             # all zeros
    x[:, 1] = 0.0
    x[rng.integers(0, n), 1] = 5.0                            # one stored value
    x[:, 2] = rng.standard_normal(n) * 1e-3 - 2.0             # all negative
    x[:, 3] = np.where(rng.random(n) < 0.5, 1.0, -1.0)        # ties across the middle
    if dtype == np.float64:                                   # values one ulp apart
        x[:, 4] = 1.0 + rng.integers(0, 4, n) * np.spacing(1.0)
        x[:, 5] = -(1.0 + rng.integers(0, 4, n) * np.spacing(1.0))
    xs = FMTS[fmt](x)
    if fmt == "csr":  # explicit stored zeros in every row
        xs = sparse.csr_matrix(x)
        coo = xs.tocoo()
        extra = (np.arange(n), np.full(n, 6))
        xs = sparse.csr_matrix((np.r_[coo.data, np.zeros(n, dtype)], (np.r_[coo.row, extra[0]], np.r_[coo.col, extra[1]])),
                               shape=(n, g))
        xs.sum_duplicates()
        assert xs.nnz > sparse.csr_matrix(x).nnz - 1
    ad = median_case(xs, codes)
    got = sb.get.aggregate(ad, "k", "median").layers["median"]
    want = ref_median(x, codes, len(sizes))
    np.testing.assert_array_equal(got, want)


def test_median_nan_semantics():
    x = np.array([[1.0, 0.0], [np.nan, 2.0], [3.0, np.nan], [4.0, 5.0]])
    codes = np.zeros(4, int)
    dense = sb.get.aggregate(median_case(x, codes), "k", "median").layers["median"]
    assert np.isnan(dense).all()  # np.median: any NaN gives NaN
    csr = sb.get.aggregate(median_case(sparse.csr_matrix(x), codes), "k", "median").layers["median"]
    np.testing.assert_array_equal(csr, [[3.5, 3.5]])  # sklearn's csc_median_axis_0: NaN sorts last


def test_nan_propagates_in_moments():
    x = np.array([[1.0, 0.0], [np.nan, 2.0], [3.0, 1.0]])
    codes = np.array([0, 0, 1])
    res = sb.get.aggregate(median_case(sparse.csr_matrix(x), codes), "k", ["sum", "mean", "var", "count_nonzero"],
                           dof=0).layers
    assert np.isnan(res["sum"][0, 0]) and np.isnan(res["mean"][0, 0]) and np.isnan(res["var"][0, 0])
    assert res["count_nonzero"][0].tolist() == [2, 1]
    assert res["sum"][1].tolist() == [3.0, 1.0]


# ------------------------------------------------------------------------------------------ scale and determinism
def test_many_tiny_groups_and_one_large():
    rng = np.random.default_rng(5)
    n_small, n_big, g = 20_000 * 5, 200_000, 64
    codes = np.r_[np.repeat(np.arange(20_000), 5), np.full(n_big, 20_000)]
    rng.shuffle(codes)
    x = sparse.random(n_small + n_big, g, density=0.1, random_state=6, format="csr", dtype=np.float32)
    x.data = np.round(x.data * 20).astype(np.float32)
    ad = median_case(x, codes)
    ctx = _abi.default_context()
    before = ctx.launches
    res = sb.get.aggregate(ad, "k", ["sum", "mean", "var", "count_nonzero"], dof=1)
    launches = ctx.launches - before
    assert launches <= 10, launches  # the group order's few kernels, then one moments launch and one fold
    st = oag.sparse_moments(x, codes, 20_001)
    np.testing.assert_allclose(res.layers["sum"], st["sum"], rtol=1e-12)
    np.testing.assert_array_equal(res.layers["count_nonzero"], st["nnz"])
    np.testing.assert_allclose(res.layers["var"], oag.variance(st["m2"], st["counts"], 1), rtol=1e-11, atol=1e-300)
    med = sb.get.aggregate(ad, "k", "median").layers["median"]
    cols = [0, 17, 63]
    np.testing.assert_array_equal(med[:, cols], oag.median_columns(x, codes, 20_001, cols))


@pytest.mark.parametrize("fmt", ["csr", "dense"])
def test_bit_identical_across_calls_and_blocks(fmt):
    rng = np.random.default_rng(7)
    n, g = 30_000, 300
    codes = rng.integers(0, 12, n)
    codes[:9000] = 3  # one group of several subtiles
    x = sparse.random(n, g, density=0.2, random_state=8, format="csr", dtype=np.float64)
    x.data = rng.lognormal(size=x.nnz)
    ad = median_case(FMTS[fmt](x if fmt == "csr" else x.toarray()), codes)
    old = settings.chunk_size
    try:
        outs = []
        for chunk in (50_000, 50_000, 2048, 5000):
            settings.chunk_size = chunk
            outs.append(sb.get.aggregate(ad, "k", FUNCS).layers)
    finally:
        settings.chunk_size = old
    for o in outs[1:]:
        for f in FUNCS:
            assert o[f].tobytes() == outs[0][f].tobytes(), f


def test_group_order_is_stable():
    rng = np.random.default_rng(9)
    codes = rng.integers(-1, 50, 300_001).astype(np.int32)
    d_order, offsets = _aggregate.group_order(codes, 50)
    order = _ops_host(d_order)[:offsets[-1]]
    keep = np.flatnonzero(codes >= 0)
    want = keep[np.argsort(codes[keep], kind="stable")]
    np.testing.assert_array_equal(order, want)
    np.testing.assert_array_equal(np.diff(offsets), np.bincount(codes[codes >= 0], minlength=50))


def _ops_host(t):
    from scanpy_b200 import _ops

    return _ops._to_host(t)


def test_large_csr_against_oracle():
    rng = np.random.default_rng(11)
    n, g, k = 200_000, 2000, 1000
    x = sparse.random(n, g, density=0.05, random_state=12, format="csr", dtype=np.float32)
    x.data = np.log1p(rng.poisson(3.0, x.nnz) + 1).astype(np.float32)
    codes = rng.integers(0, k, n)
    ad = median_case(x, codes)
    res = sb.get.aggregate(ad, "k", FUNCS)
    st = oag.sparse_moments(x, codes, k)
    np.testing.assert_allclose(res.layers["sum"], st["sum"], rtol=1e-12)
    np.testing.assert_allclose(res.layers["mean"], st["mean"], rtol=1e-12)
    np.testing.assert_allclose(res.layers["var"], oag.variance(st["m2"], st["counts"], 1), rtol=1e-11)
    np.testing.assert_array_equal(res.layers["count_nonzero"], st["nnz"])
    cols = list(range(0, g, 97))
    dense = x[:, cols].toarray()
    want = ref_median(dense, codes, k)
    np.testing.assert_array_equal(res.layers["median"][:, cols], want)

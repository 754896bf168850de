"""sc.get.aggregate without a GPU: the oracle (oracle/aggregate.py) against the reference's literal tests
(tests/test_aggregated.py), and the host side of `scanpy_b200.get.aggregate` (argument errors, axis, mask, the
result's layout and dtypes) with the oracle's statistics standing in for the device pass."""
import warnings
from itertools import product

import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import aggregate as oag
from scanpy_b200 import _aggregate, get
from scanpy_b200._compat import MiniAnnData


def fake_group_stats(x, codes, n_groups, *, moments=True, median=False):
    """`_aggregate.group_stats` computed by the oracle, with the device pass's dtypes."""
    st = oag.dense_stats(x, codes, n_groups)
    counts = np.bincount(codes[codes >= 0], minlength=n_groups).astype(np.int64)
    vdt = _aggregate.value_dtype(x)
    mean = np.where(counts[:, None] > 0, st["mean"], 0.0)
    return dict(counts=counts, sum=st["sum"], mean=mean, m2=st["m2"], nnz=st["nnz"].astype(np.int64),
                median=st["median"].astype(vdt))


@pytest.fixture(autouse=True)
def oracle_stats(monkeypatch):
    monkeypatch.setattr(_aggregate, "group_stats", fake_group_stats)


def adata_of(x, obs, var=None):
    var = var if var is not None else pd.DataFrame(index=[f"gene_{i}" for i in range(x.shape[1])])
    return MiniAnnData(x, obs=obs, var=var)


BLOCK = np.block([[np.ones((2, 2)), np.zeros((2, 2))], [np.zeros((2, 2)), np.ones((2, 2))]])
BLOCK_OBS = pd.DataFrame({"a": ["a", "a", "b", "b"], "b": ["c", "d", "d", "d"]}, index=["a_c", "a_d", "b_d1", "b_d2"])
BLOCK_LAYERS = {"count_nonzero": np.array([[1, 1, 0, 0], [1, 1, 0, 0], [0, 0, 2, 2]]),
                "sum": np.array([[1, 1, 0, 0], [1, 1, 0, 0], [0, 0, 2, 2]]),
                "mean": np.array([[1, 1, 0, 0], [1, 1, 0, 0], [0, 0, 1, 1]])}


# ------------------------------------------------------------------------------------------ the reference's literals
@pytest.mark.parametrize("metrics", [["count_nonzero"], ["sum", "mean", "count_nonzero"], ["mean"]])
def test_aggregate_examples(metrics):
    res = sb.get.aggregate(adata_of(BLOCK, BLOCK_OBS.copy()), by=["a", "b"], func=metrics)
    assert list(res.obs_names if hasattr(res, "obs_names") else res.obs.index) == ["a_c", "a_d", "b_d"]
    assert res.obs["a"].tolist() == ["a", "a", "b"] and res.obs["b"].tolist() == ["c", "d", "d"]
    assert isinstance(res.obs["a"].dtype, pd.CategoricalDtype)
    assert res.obs["n_obs_aggregated"].tolist() == [1, 1, 2]
    assert list(res.var.index) == [f"gene_{i}" for i in range(4)]
    assert set(res.layers) == set(metrics)
    for m in metrics:
        np.testing.assert_array_equal(res.layers[m], BLOCK_LAYERS[m])
    assert res.shape == (3, 4) and res.X is None


def test_nan():
    x = np.arange(6) + np.arange(6)[:, None]
    obs = pd.DataFrame(dict(cell_type=[np.nan, np.nan, "B", "C", "B", "B"], sample_id=["s1", "s1", "s1", "s2", "s2", "s2"],
                            patient_type=[*(["responder"] * 3), *(["control"] * 3)]),
                       index=[f"cell{i}" for i in range(6)])
    res = sb.get.aggregate(adata_of(x, obs), by=["sample_id", "patient_type", "cell_type"], func="sum", layer=None)
    assert res.obs.index.tolist() == ["s1_responder_B", "s2_control_B", "s2_control_C"]
    assert res.obs["n_obs_aggregated"].tolist() == [1, 2, 1]
    names, codes, counts = oag.group_codes(obs, ["sample_id", "patient_type", "cell_type"])
    assert names.tolist() == res.obs.index.tolist() and counts.tolist() == [1, 2, 1]


def test_factors():
    obs = pd.DataFrame(product(range(5), repeat=4), columns=list("abcd"))
    obs.index = [f"cell_{i:04d}" for i in range(obs.shape[0])]
    x = np.arange(obs.shape[0]).reshape(-1, 1)
    res = sb.get.aggregate(adata_of(x, obs), by=["a", "b", "c", "d"], func="sum")
    np.testing.assert_equal(res.layers["sum"], x)


@pytest.mark.parametrize(("label_cols", "expected"), [
    (dict(a=["a", "b", "c"], b=["d", "d", "f"], c=["g", "h", "h"]), ["a_d_g", "b_d_h", "c_f_h"]),
    (dict(a=["a", "b", "c"], b=["d", "d", "f"]), ["a_d", "b_d", "c_f"]),
    (dict(a=["a", "b", "c"], c=["g", "h", "h"]), ["a_g", "b_h", "c_h"]),
    (dict(b=["d", "d", "f"], c=["g", "h", "h"]), ["d_g", "d_h", "f_h"]),
], ids=["three", "two-1", "two-2", "two-3"])
def test_combine_categories(label_cols, expected):
    label_df = pd.DataFrame({k: pd.Categorical(v) for k, v in label_cols.items()})
    result, result_label_df = get.combine_categories(label_df)
    assert isinstance(result, pd.Categorical)
    pd.testing.assert_extension_array_equal(result, pd.Categorical(expected))
    pd.testing.assert_index_equal(pd.Index(result), result_label_df.index.astype("category"))
    reconstructed = pd.DataFrame([x.split("_") for x in result], columns=list(label_cols),
                                 index=result.astype(str)).astype("category")
    pd.testing.assert_frame_equal(reconstructed, result_label_df)


@pytest.mark.parametrize("dof", [0, 1, 4])
def test_aggregate_var_group_matches_dof(dof):
    run = max(1, dof)
    x = np.array([1.0] * run + [2.0] * run + [3.0] * run).reshape(3 * run, 1)
    obs = pd.DataFrame({"group": pd.Categorical(["a"] * run + ["b"] * run + ["a"] * run)},
                       index=[f"cell_{i}" for i in range(3 * run)])
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        var = sb.get.aggregate(adata_of(x, obs), "group", "var", dof=dof).layers["var"]
    msgs = [str(w.message) for w in rec if issubclass(w.category, RuntimeWarning)]
    assert any("groups ['b'] will be nan" in m for m in msgs) == (dof > 0)
    a = np.array([1.0] * run + [3.0] * run)
    np.testing.assert_allclose(var[0, 0], np.var(a, ddof=dof))
    if dof > 0:
        assert np.isnan(var[1, 0])
    else:
        assert var[1, 0] == 0.0
    names, codes, counts = oag.group_codes(obs, "group")
    st = oag.dense_stats(x, codes, len(names))
    np.testing.assert_allclose(oag.variance(st["m2"], counts, dof), var, equal_nan=True)


def test_var_no_catastrophic_cancellation_oracle():
    rng = np.random.default_rng(0)
    x = 1e8 + 1e-3 * rng.standard_normal((2000, 4))
    codes = np.repeat([0, 1], 1000)
    st = oag.dense_stats(x, codes, 2, median=False)
    expected = np.vstack([np.var(x[:1000], axis=0), np.var(x[1000:], axis=0)])
    np.testing.assert_allclose(oag.variance(st["m2"], np.array([1000, 1000]), 0), expected, rtol=1e-4)
    sp = oag.sparse_moments(sparse.csr_matrix(x), codes, 2)
    np.testing.assert_allclose(oag.variance(sp["m2"], sp["counts"], 0), expected, rtol=1e-4)


def test_oracle_sparse_matches_dense():
    rng = np.random.default_rng(1)
    x = sparse.random(300, 40, density=0.2, random_state=2, format="csr") * 10 - sparse.random(300, 40, density=0.05,
                                                                                               random_state=3)
    codes = rng.integers(-1, 7, 300)
    d = oag.dense_stats(x, codes, 7)
    s = oag.sparse_moments(x, codes, 7)
    for k in ("sum", "m2", "nnz"):
        np.testing.assert_allclose(s[k], d[k], rtol=1e-12, atol=1e-12)
    cols = [0, 5, 39]
    np.testing.assert_array_equal(oag.median_columns(x, codes, 7, cols), d["median"][:, cols])


# ------------------------------------------------------------------------------------------ host logic
def blobs(n=60, g=5, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.poisson(2.0, (n, g)).astype(np.float32)
    obs = pd.DataFrame({"blobs": pd.Categorical(rng.integers(0, 3, n).astype(str)),
                        "extra": rng.choice(["u", "v"], n)}, index=[f"c{i}" for i in range(n)])
    var = pd.DataFrame({"mask_col": np.arange(g) % 2 == 0}, index=[f"g{i}" for i in range(g)])
    return adata_of(x, obs, var)


def test_func_errors():
    ad = blobs()
    with pytest.raises(ValueError, match=r"func \{'foo'\} is not one of dict_keys\(\['count_nonzero', 'sum', "
                                         r"'median', 'mean', 'var'\]\)"):
        sb.get.aggregate(ad, "blobs", ["sum", "foo"])
    with pytest.raises(TypeError, match="not iterable"):
        sb.get.aggregate(ad, 123, "sum")


@pytest.mark.parametrize(("kwargs", "match"), [
    (dict(layer="test", obsm="test"), r"Only one of `layer`, or `obsm` can be specified"),
    (dict(obsm="test", axis=1), r"`obsm` cannot be used when `dim` is `var`"),
    (dict(varm="test", axis=0), r"`varm` cannot be used when `dim` is `obs`"),
    (dict(axis="foo"), r"was 'foo'"),
])
def test_old_api_errors(kwargs, match):
    ad = blobs()
    ad.layers["test"] = ad.X.copy()
    ad.obsm["test"] = ad.X.copy()
    ad.varm["test"] = np.column_stack([ad.X[0], ad.X[1]])
    with pytest.raises((TypeError, ValueError), match=match):
        sb.get.aggregate(ad, by="blobs", func="sum", **kwargs)


def test_not_implemented():
    ad = blobs()
    with pytest.raises(NotImplementedError, match="AnnData input"):
        sb.get.aggregate(ad.X, "blobs", "sum")
    with pytest.raises(NotImplementedError, match="acc="):
        sb.get.aggregate(ad, "blobs", "sum", acc="X")
    ad.layers["coo"] = sparse.coo_matrix(ad.X)
    with pytest.raises(NotImplementedError, match="not supported for aggregation"):
        sb.get.aggregate(ad, "blobs", "sum", layer="coo")
    fake_dask = type("Array", (), dict(__module__="dask.array.core", shape=(60, 5), dtype=np.float32, T=None))()
    ad.layers["dask"] = fake_dask
    with pytest.raises(NotImplementedError, match="dask"):
        sb.get.aggregate(ad, "blobs", "sum", layer="dask")
    ref = type("AdRef", (), dict(__module__="anndata.acc"))()
    with pytest.raises(NotImplementedError, match="anndata.acc"):
        sb.get.aggregate(ad, [ref], "sum")
    with pytest.raises(NotImplementedError, match="anndata.acc"):
        sb.get.aggregate(ad, "blobs", "sum", mask=ref)


@pytest.mark.parametrize("axis", [0, 1, "obs", "var"])
def test_mask_by_name_and_array(axis):
    ad = blobs()
    mask = (ad.obs["blobs"] == "0").to_numpy()
    ad.obs["mask_col"] = mask
    if axis in (1, "var"):
        ad = ad.T
        ad.var["mask_col"] = mask
    by_ref = sb.get.aggregate(ad, "blobs", "sum", axis=axis, mask="mask_col")
    by_value = sb.get.aggregate(ad, "blobs", "sum", axis=axis, mask=mask)
    s_ref, s_val = by_ref.layers["sum"], by_value.layers["sum"]
    np.testing.assert_array_equal(s_ref, s_val)
    if axis in (1, "var"):
        assert list(by_ref.var.index) == ["0", "1", "2"]
        assert (s_ref[:, 1:] == 0).all() and (s_ref[:, 0] > 0).any()
    else:
        assert list(by_ref.obs.index) == ["0", "1", "2"]
        assert (s_ref[1:] == 0).all()
        assert by_ref.obs["n_obs_aggregated"].tolist() == [mask.sum(), 0, 0]


def test_mask_errors():
    ad = blobs()
    with pytest.raises(ValueError, match=r"Did not find `adata.obs\['nope'\]`"):
        sb.get.aggregate(ad, "blobs", "sum", mask="nope")
    with pytest.raises(ValueError, match="The shape of the mask do not match the data."):
        sb.get.aggregate(ad, "blobs", "sum", mask=np.ones(3, bool))
    with pytest.raises(ValueError, match="Mask array must be boolean."):
        sb.get.aggregate(ad, "blobs", "sum", mask=np.ones(60))


@pytest.mark.parametrize(("fmt", "dtype", "expected"), [
    ("dense", np.float32, dict(sum=np.float64, count_nonzero=np.float64, mean=np.float64, var=np.float64,
                               median=np.float32)),
    ("dense", np.int64, dict(sum=np.float64, count_nonzero=np.float64, mean=np.float64, var=np.float64,
                             median=np.float64)),
    ("dense", np.float64, dict(sum=np.float64, count_nonzero=np.float64, median=np.float64)),
    ("csr", np.float32, dict(sum=np.float64, count_nonzero=np.int64, mean=np.float64, var=np.float64,
                             median=np.float64)),
    ("csc", np.int32, dict(sum=np.int64, count_nonzero=np.int64, mean=np.float64, var=np.float64,
                           median=np.float64)),
])
def test_result_dtypes_and_layout(fmt, dtype, expected):
    ad = blobs()
    x = ad.X.astype(dtype)
    ad.X = {"dense": x, "csr": sparse.csr_matrix(x), "csc": sparse.csc_array(x)}[fmt]
    res = sb.get.aggregate(ad, ["blobs", "extra"], list(AGG := get.AGG_FUNCS))
    assert set(res.layers) == set(AGG)
    for k, dt in expected.items():
        assert res.layers[k].dtype == dt, k
    assert res.shape == (len(res.obs), 5)
    assert list(res.obs.columns) == ["blobs", "extra", "n_obs_aggregated"]
    assert res.var is ad.var


def test_obsm_varm_layout():
    ad = blobs()
    ad.obsm["test"] = ad.X[:, ::2].copy()
    ad.obsm["df"] = pd.DataFrame(ad.X[:, :2], index=ad.obs.index, columns=["pc_a", "pc_b"])
    r = sb.get.aggregate(ad, "blobs", ["sum", "mean"], obsm="test")
    assert list(r.var.index) == ["0", "1", "2"]
    expected = pd.DataFrame(ad.obsm["test"]).groupby(ad.obs["blobs"].to_numpy()).sum().to_numpy()
    np.testing.assert_allclose(r.layers["sum"], expected)
    rd = sb.get.aggregate(ad, "blobs", "sum", obsm="df")
    assert list(rd.var.index) == ["pc_a", "pc_b"]
    t = ad.T
    rv = sb.get.aggregate(t, "blobs", ["sum", "mean"], varm="test")
    assert rv.shape == (3, 3)[::-1] or rv.shape == (3, 3)
    np.testing.assert_allclose(rv.T.layers["sum"], r.layers["sum"])
    np.testing.assert_allclose(rv.layers["sum"], r.layers["sum"].T)


def test_mean_alone_vs_with_var_on_masked_out_group():
    ad = blobs()
    mask = (ad.obs["blobs"] != "2").to_numpy()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        alone = sb.get.aggregate(ad, "blobs", "mean", mask=mask).layers["mean"]
        both = sb.get.aggregate(ad, "blobs", ["mean", "var"], mask=mask).layers
    assert np.isnan(alone[2]).all() and (both["mean"][2] == 0).all() and np.isnan(both["var"][2]).all()
    np.testing.assert_allclose(alone[:2], both["mean"][:2])


def test_mini_anndata_layers_only():
    layers = {"a": np.arange(6.0).reshape(2, 3)}
    obs = pd.DataFrame(index=["r0", "r1"])
    var = pd.DataFrame(index=["c0", "c1", "c2"])
    m = MiniAnnData(None, obs=obs, var=var, layers=layers)
    assert m.X is None and m.shape == (2, 3) and m.n_obs == 2 and m.n_vars == 3
    t = m.T
    assert t.shape == (3, 2) and list(t.obs.index) == ["c0", "c1", "c2"] and list(t.var.index) == ["r0", "r1"]
    np.testing.assert_array_equal(t.layers["a"], layers["a"].T)
    assert m.copy().shape == (2, 3)
    assert MiniAnnData(None, obs=obs, var=var).shape == (2, 3)
    x = MiniAnnData(np.zeros((4, 2)))
    assert x.shape == (4, 2) and list(x.obs.index) == ["0", "1", "2", "3"] and x.layers == {}

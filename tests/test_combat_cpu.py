"""CPU tests for combat: the oracle (oracle/combat.py) against the reference's own properties
(tests/test_combat.py), the design matrix without patsy, the host empirical-Bayes solver fed closed-form sums against
the oracle's direct `_it_sol`, and the argument errors the public function raises before touching a device."""
import numpy as np
import pandas as pd
import pytest
from sklearn.datasets import make_blobs

import scanpy_b200 as sb
from oracle import combat as oc
from scanpy_b200 import _combat, _ops
from scanpy_b200._compat import MiniAnnData
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN


def blobs():
    """The reference's `sc.datasets.blobs()`: 640 cells, 11 genes, 5 centres, the centre as a categorical obs column."""
    x, y = make_blobs(n_samples=640, n_features=11, centers=5, cluster_std=1.0, random_state=0)
    return MiniAnnData(x.astype(np.float32), obs=pd.DataFrame({"blobs": pd.Categorical(y.astype(str))},
                                                               index=[str(i) for i in range(640)]))


def oracle_inputs(obs, key, covariates=()):
    """(design as numbers, the cells of each batch) the way combat builds them."""
    model = obs[[key, *covariates]]
    levels, codes, _ = _combat.batch_groups(model, key)
    design = _combat.design_matrix(model, key, levels).to_numpy()
    return design, [np.flatnonzero(codes == b) for b in range(len(levels))]


# ------------------------------------------------------------------------------------------ the reference's properties
def test_standardized_data_has_zero_gene_means():
    ad = blobs()
    design, idx = oracle_inputs(ad.obs, "blobs")
    s_data, *_ = oc.standardize(ad.X, design, idx)
    assert np.allclose(s_data.mean(axis=0), 0)


def test_design_with_numeric_covariates():
    rng = np.random.default_rng(0)
    ad = blobs()
    ad.obs["cat1"] = rng.binomial(3, 0.5, size=ad.n_obs)
    ad.obs["cat2"] = rng.binomial(2, 0.1, size=ad.n_obs)
    ad.obs["num1"] = rng.standard_normal(ad.n_obs)
    model = ad.obs[["cat1", "cat2", "num1", "blobs"]]
    cats = ad.obs["blobs"].cat.categories
    design = _combat.design_matrix(model, "blobs", cats)
    assert len(design.columns) == 4 + len(cats) - 1


def test_design_columns_by_hand():
    obs = pd.DataFrame({
        "batch": pd.Categorical(["b", "a", "b", "c", "a", "b"], categories=["c", "b", "a", "unused"]),
        "s": np.array(["v", "u", "w", "u", "v", "v"], dtype=object),
        "flag": [True, True, False, True, True, False],
        "k": np.array([3, 1, 4, 1, 5, 9], dtype=np.int64),
        "z": [0.5, -1.0, 2.0, 0.0, 1.5, 3.0],
    })
    model = obs[["batch", "k", "s", "flag", "z"]]
    levels, codes, counts = _combat.batch_groups(model, "batch")
    assert levels == ["c", "b", "a"] and codes.tolist() == [1, 2, 1, 0, 2, 1] and counts.tolist() == [1, 3, 2]
    d = _combat.design_matrix(model, "batch", levels)
    expect = pd.DataFrame({
        "C(Q('batch'), levels=batch_levels)[c]": [0, 0, 0, 1, 0, 0],
        "C(Q('batch'), levels=batch_levels)[b]": [1, 0, 1, 0, 0, 1],
        "C(Q('batch'), levels=batch_levels)[a]": [0, 1, 0, 0, 1, 0],
        "Q('s')[u]": [0, 1, 0, 1, 0, 0],
        "Q('s')[v]": [1, 0, 0, 0, 1, 1],
        "Q('s')[w]": [0, 0, 1, 0, 0, 0],
        "Q('flag')[T.True]": [1, 1, 0, 1, 1, 0],
        "k": [3, 1, 4, 1, 5, 9],
        "z": [0.5, -1.0, 2.0, 0.0, 1.5, 3.0],
    }, dtype=np.float64)
    pd.testing.assert_frame_equal(d.reset_index(drop=True), expect)


def test_batch_order_of_a_non_categorical_key():
    model = pd.DataFrame({"batch": [3, 1, 2, 3, 1, 2, 2]})
    levels, codes, counts = _combat.batch_groups(model, "batch")
    assert levels == [1, 2, 3] and codes.tolist() == [2, 0, 1, 2, 0, 1, 1] and counts.tolist() == [2, 3, 2]


def test_bool_covariate_first_gets_both_levels():
    obs = pd.DataFrame({"batch": ["x", "y"] * 4, "flag": [True] * 8})
    levels, _, _ = _combat.batch_groups(obs, "batch")
    d = _combat.design_matrix(obs, "batch", levels)
    assert list(d.columns[2:]) == ["Q('flag')[False]", "Q('flag')[True]"]
    assert (d["Q('flag')[False]"] == 0).all()


# ------------------------------------------------------------------------------------------ the host EB solver
N, G = 600, 40


def eb_case(case, seed=0):
    """(x [N x G], obs, covariates) for the solver checks."""
    rng = np.random.default_rng(seed)
    n_batch = 1 if case == "one_batch" else 4
    b = rng.integers(0, n_batch, N)
    x = np.log1p(rng.gamma(1.5, 2.0, (N, G)) * (rng.random((N, G)) > 0.3)) + 0.4 * b[:, None] * rng.random(G)
    obs = pd.DataFrame({"batch": pd.Categorical(b)})
    covariates = []
    if case == "zero_var":
        x[:, [3, 17]] = 0.0
    if case == "absent":
        x[b == 1, 5] = 0.0
        x[b == 2, 9] = 0.0
    if case == "negative":
        x -= 2.0 * (b[:, None] == 0)  # batch 0 well below the rest: gamma_hat < 0 there
    if case == "covariates":
        obs["num"] = rng.normal(size=N)
        obs["k"] = rng.integers(0, 3, N)
        x += 0.3 * obs["num"].to_numpy()[:, None]
        covariates = ["num", "k"]
    return x, obs, covariates


@pytest.mark.parametrize("case", ["plain", "zero_var", "absent", "negative", "one_batch", "covariates"])
def test_eb_from_closed_form_sums_matches_the_direct_iteration(case, capsys):
    x, obs, covariates = eb_case(case)
    design, idx = oracle_inputs(obs, "batch", covariates)
    ref, inter = oc.combat(x, design, idx)
    # the moments of r = x - stand_mean per batch, as the device pass returns them
    r = x - inter["stand_mean"]
    counts = np.array([len(i) for i in idx])
    means = np.stack([r[i].mean(axis=0) for i in idx])
    m2 = np.stack([((r[i] - r[i].mean(axis=0)) ** 2).sum(axis=0) for i in idx])
    fit = _combat.eb_fit(counts, means, m2, inter["b_hat"][:len(idx)], inter["grand_mean"])
    assert fit["iterations"] == inter["iterations"]
    if case == "zero_var":
        assert "Found 2 genes with zero variance." in capsys.readouterr().out
        assert fit["iterations"] == [1] * len(idx)  # g_old == 0 makes Python's max() return nan
    if case == "negative":
        assert (fit["gamma_hat"][0] < 0).all()
    np.testing.assert_allclose(fit["var_pooled"], inter["var_pooled"], rtol=1e-12, atol=1e-15)
    for k in ("gamma_hat", "delta_hat", "gamma_star", "delta_star"):
        np.testing.assert_allclose(fit[k], inter[k], rtol=1e-9, atol=1e-12, err_msg=k)
    # the writer's expression from these fits gives the oracle's result
    sv = np.sqrt(fit["var_pooled"])
    codes = np.zeros(N, dtype=int)
    for b, i in enumerate(idx):
        codes[i] = b
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(sv == 0, 0.0, r / sv)
    got = ((s - fit["gamma_star"][codes]) / np.sqrt(fit["delta_star"])[codes]) * sv + inter["stand_mean"]
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-10 * np.abs(x).max())


def test_it_sol_max_quirk():
    """Python's max(a, b): a NaN first argument ends the loop, a NaN second argument does not."""
    assert np.isnan(max(np.nan, 1.0)) and max(1.0, np.nan) == 1.0
    # a zero-variance gene (g_hat = d_hat = 0): g_new = 0, the gamma ratio is 0 / 0 = nan -> one iteration
    g, d, count = _combat.it_sol(np.array([0.0, 0.5]), np.array([0.0, 3.0]), 10, np.array([0.0, 0.5]),
                                 np.array([0.0, 0.3]), g_bar=0.2, t2=0.1, a=2.0, b=1.0)
    assert count == 1
    # only d_old == 0 with g_old != 0: d ratio inf, the loop goes on
    g, d, count = _combat.it_sol(np.array([0.4, 0.5]), np.array([0.0, 3.0]), 10, np.array([0.4, 0.5]),
                                 np.array([0.0, 0.3]), g_bar=0.2, t2=0.1, a=2.0, b=1.0)
    assert count > 1


# ------------------------------------------------------------------------------------------ argument errors
def _adata(n=20):
    rng = np.random.default_rng(0)
    obs = pd.DataFrame({"batch": pd.Categorical(["a", "b"] * (n // 2)), "num": rng.random(n),
                        "s": np.array(["u", "v", "w", "v"] * (n // 4), dtype=object)},
                       index=[f"c{i}" for i in range(n)])
    return MiniAnnData(rng.random((n, 5)), obs=obs)


def test_errors_before_the_device(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("the device was touched")

    monkeypatch.setattr(_ops, "DeviceX", no_device)
    with pytest.raises(ValueError, match=r"Could not find the key 'nope' in adata.obs"):
        sb.pp.combat(_adata(), "nope")
    with pytest.raises(ValueError, match=r"Could not find the covariate\(s\) \['x', 'y'\] in adata.obs"):
        sb.pp.combat(_adata(), "batch", covariates=["num", "x", "y"])
    with pytest.raises(ValueError, match="Batch key and covariates cannot overlap"):
        sb.pp.combat(_adata(), "batch", covariates=["num", "batch"])
    with pytest.raises(ValueError, match="Covariates must be unique"):
        sb.pp.combat(_adata(), "batch", covariates=["num", "num"])
    ad = _adata()
    ad.obs["batch"] = pd.Categorical(["single"] + ["other"] * (ad.n_obs - 1))
    with pytest.raises(ValueError, match=r"Batches \['single'\] have fewer than 2 cells"):
        sb.pp.combat(ad, "batch")
    ad = _adata()
    ad.obs["batch"] = pd.Categorical([None] + ["a", "b"] * 9 + ["a"])
    with pytest.raises(ValueError, match="has missing values"):
        sb.pp.combat(ad, "batch")
    ad = _adata(40)
    for i in range(33):
        ad.obs[f"k{i}"] = np.random.default_rng(i).random(40)
    with pytest.raises(NotImplementedError, match="at most 32 covariate columns"):
        sb.pp.combat(ad, "batch", covariates=[f"k{i}" for i in range(33)])
    with pytest.raises(AssertionError, match="device was touched"):  # 32 is within the limit
        sb.pp.combat(ad, "batch", covariates=[f"k{i}" for i in range(32)])
    ad = _adata()
    ad.obs["twice"] = ad.obs["num"]
    with pytest.raises(np.linalg.LinAlgError):  # an exactly singular design fails in inv(DᵀD) as in the reference
        sb.pp.combat(ad, "batch", covariates=["num", "twice"])
    with pytest.raises(NotImplementedError, match="float16"):
        sb.pp.combat(MiniAnnData(_adata().X.astype(np.float16), obs=_adata().obs), "batch")
    backed = MiniAnnData(ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts"))
    backed.obs = pd.DataFrame({"batch": pd.Categorical(np.arange(backed.n_obs) % 2)})
    with pytest.raises(NotImplementedError, match="combat is not implemented for matrices of type"):
        sb.pp.combat(backed, "batch")

"""CPU tests for regress_out: the oracle (oracle/regress.py) against the reference's goldens
(tests/test_preprocessing.py:472-488) and a per-gene lstsq, the host-side least-squares algebra, and the argument errors
the public function raises before touching a device."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import regress as orr
from scanpy_b200 import _regress
from scanpy_b200._compat import MiniAnnData
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN


def pbmc68k_small():
    """The reference's `pbmc68k_reduced().raw.to_adata()[:200, :200]` and its obs columns."""
    h = np.load(GOLDEN / "pbmc68k_raw_seurat_hvg.npz")
    d = np.load(GOLDEN / "pbmc68k_regress.npz")
    raw = sparse.csr_matrix((h["raw_data"], h["raw_indices"], h["raw_indptr"]), shape=(700, 765))
    obs = pd.DataFrame({"n_counts": d["n_counts"][:200], "percent_mito": d["percent_mito"][:200],
                        "bulk_labels": pd.Categorical.from_codes(d["bulk_labels_codes"][:200].astype(int),
                                                                 [f"l{i}" for i in range(10)])},
                       index=[f"c{i}" for i in range(200)])
    return raw[:200, :200].tocsr(), obs, d


def test_oracle_reproduces_the_numeric_golden():
    x, obs, d = pbmc68k_small()
    r = orr.regress_out(x, regressors=orr.design(obs, ["n_counts", "percent_mito"]))
    np.testing.assert_allclose(r, d["regress_test_small"], atol=0)


def test_oracle_reproduces_the_categorical_golden():
    x, obs, d = pbmc68k_small()
    codes = obs["bulk_labels"].cat.codes.to_numpy()
    r = orr.regress_out(x, codes=codes, n_categories=10)
    np.testing.assert_allclose(r, d["regress_test_small_cat"], atol=1e-6)
    # fp64 category means (what the device computes) stay inside the same tolerance
    r64 = orr.regress_out(x, codes=codes, n_categories=10, exact_means=True)
    np.testing.assert_allclose(r64, d["regress_test_small_cat"], atol=1e-6)


def test_oracle_glm_fallback_is_the_per_gene_lstsq():
    rng = np.random.default_rng(0)
    x = rng.normal(size=(300, 12))
    x[:, 3] = 2.5  # constant: unchanged
    k = rng.normal(size=300)
    a = np.c_[np.ones(300), k, k]  # singular
    assert np.linalg.det(a.T @ a) == 0 or abs(np.linalg.det(a.T @ a)) < 1e-6
    r = orr.glm_residuals(x, a)
    for j in range(12):
        if j == 3:
            assert (r[:, j] == 2.5).all()
            continue
        coef = np.linalg.lstsq(a, x[:, j], rcond=None)[0]
        np.testing.assert_allclose(r[:, j], x[:, j] - a @ coef, rtol=0, atol=1e-12)


@pytest.mark.parametrize("missing", [False, True])
def test_categorical_normal_equations_match_lstsq(missing):
    """The per-gene 2 x 2 solve from the per-category sums equals the lstsq residual on [1, r] with fp64 means."""
    rng = np.random.default_rng(1)
    n, g, c = 500, 30, 7
    x = rng.gamma(2.0, 1.0, size=(n, g))
    codes = rng.integers(0, c, n)
    if missing:
        codes[rng.random(n) < 0.2] = -1
    codes[codes == 5] = 6  # an unused category
    grp = np.where(codes < 0, c, codes)
    sums = np.stack([x[grp == k].sum(0) for k in range(c + 1)])
    counts = np.bincount(codes[codes >= 0], minlength=c)
    means, b0, b1 = _regress._categorical_fit(sums, counts, n, missing)
    r = np.where(codes[:, None] >= 0, means[np.maximum(codes, 0)], 0.0)
    got = x - (b0 + b1 * r)
    ref = orr.glm_residuals(x, orr.categorical_regressor(x, codes, c, exact_means=True), per_gene=True)
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12 * np.abs(x).max())


def _adata(x=None):
    rng = np.random.default_rng(0)
    x = rng.random((20, 5)) if x is None else x
    obs = pd.DataFrame({"a": rng.random(20), "b": rng.random(20), "cat": pd.Categorical(rng.integers(0, 3, 20)),
                        "s": np.array(["u", "v"] * 10, dtype=object)}, index=[f"c{i}" for i in range(20)])
    return MiniAnnData(x, obs=obs)


def test_errors_before_the_device(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("the device was touched")

    monkeypatch.setattr(_regress, "_DeviceX", no_device)
    with pytest.raises(ValueError, match="If providing categorical variable, only a single one is allowed"):
        sb.pp.regress_out(_adata(), ["cat", "a"])
    with pytest.raises(ValueError, match="only a single one is allowed"):
        sb.pp.regress_out(_adata(), ["s", "a"])  # a string column counts as categorical
    with pytest.raises(KeyError):
        sb.pp.regress_out(_adata(), ["a", "missing"])
    with pytest.raises(TypeError):
        sb.pp.regress_out(_adata(), ["a", "s"])  # a string column after a numeric key: numpy cannot take det()
    ad = _adata()
    for i in range(32):
        ad.obs[f"k{i}"] = np.random.default_rng(i).random(20)
    with pytest.raises(NotImplementedError, match="at most 32 regressors"):
        sb.pp.regress_out(ad, [f"k{i}" for i in range(32)])
    # 31 keys and the intercept are within the limit
    with pytest.raises(AssertionError, match="device was touched"):
        sb.pp.regress_out(ad, [f"k{i}" for i in range(31)])
    backed = _adata(ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts"))
    backed.obs = pd.DataFrame({"a": np.arange(backed.n_obs, dtype=float)})
    with pytest.raises(NotImplementedError, match="regress_out is not implemented for matrices of type"):
        sb.pp.regress_out(backed, ["a"])


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64, np.uint16])
@pytest.mark.parametrize("path", ["shortcut", "fallback", "categorical"])
def test_output_dtypes(dtype, path):
    rng = np.random.default_rng(2)
    x = rng.integers(0, 9, (60, 8)).astype(dtype)
    obs = pd.DataFrame({"a": rng.random(60), "cat": pd.Categorical(rng.integers(0, 3, 60))})
    if path == "categorical":
        r = orr.regress_out(x, codes=obs["cat"].cat.codes.to_numpy(), n_categories=3)
        expect = np.float64
    else:
        keys = ["a"] if path == "shortcut" else ["a", "a"]
        r = orr.regress_out(x, regressors=orr.design(obs, keys))
        expect = np.float64 if path == "fallback" else (
            dtype if np.dtype(dtype).kind == "f" else (np.float32 if np.dtype(dtype).itemsize <= 4 else np.float64))
    assert r.dtype == expect
    # the host picks the same value dtype for the device
    if path == "shortcut":
        assert _regress._float_dtype(dtype, integer_to=None) == expect

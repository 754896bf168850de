"""CPU tests for the analytic Pearson residuals: the oracle (oracle/pearson.py) against the reference's own relations
and a literal transcription of its numba loop, the batch quirks, and the argument errors and warnings the public
functions raise before touching a device."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import pearson as opr
from scanpy_b200 import _abi, _ops
from scanpy_b200._compat import MiniAnnData
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN

TOY = np.array([[3, 6], [2, 4], [1, 0]])


def numba_loop_variance(x, *, theta, clip):
    """_calculate_res_dense (_highly_variable_genes.py:90-126), one cell and one gene at a time."""
    n, g = x.shape
    sums_genes, sums_cells = x.sum(axis=0), x.sum(axis=1)
    sum_total = np.sum(sums_genes)
    out = np.zeros(g)

    def res(gene, cell):
        mu = sums_genes[gene] * sums_cells[cell] / sum_total
        pre = (x[cell, gene] - mu) / np.sqrt(mu + mu * mu / theta)
        return min(max(pre, -clip), clip)

    for gene in range(g):
        mean = sum(res(gene, c) for c in range(n)) / n
        out[gene] = sum((res(gene, c) - mean) ** 2 for c in range(n)) / n
    return out


@pytest.mark.parametrize("theta", [0.01, 1, 100, np.inf])
@pytest.mark.parametrize("clip", [None, 1, np.inf])
def test_oracle_toy_matrix(theta, clip):
    """tests/test_normalization.py:139-191 of the reference, on the oracle."""
    ns, ps = TOY.sum(axis=1), TOY.sum(axis=0) / TOY.sum()
    mu = np.outer(ns, ps)
    expect = (TOY - mu) / np.sqrt(mu) if np.isinf(theta) else (TOY - mu) / np.sqrt(mu + mu**2 / theta)
    out = opr.pearson_residuals(TOY, theta=theta, clip=clip)
    if clip is None:
        threshold = np.sqrt(TOY.shape[0]).astype(np.float32)
        assert out.max() <= threshold and out.min() >= -threshold
    elif np.isinf(clip):
        np.testing.assert_allclose(out, expect)
    else:
        assert out.max() <= clip and out.min() >= -clip


@pytest.mark.parametrize("theta", [1, 100, np.inf])
@pytest.mark.parametrize("clip", [None, 0.5, np.inf])
def test_oracle_variances_are_np_var_of_its_residuals(theta, clip):
    x = np.random.default_rng(0).negative_binomial(2, 0.3, (300, 40)).astype(np.float64)
    x[:, 5] = 0
    var, _ = opr.batch_residual_variances(x, theta=theta, clip=clip)
    ref = np.var(opr.pearson_residuals(x, theta=theta, clip=clip), axis=0)
    ref[5] = 0.0  # a zero gene is left out and gets 0
    np.testing.assert_allclose(var[0], ref, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("theta", [0.5, 100, np.inf])
def test_oracle_matches_the_numba_loop(theta):
    x = np.random.default_rng(1).negative_binomial(1, 0.4, (40, 7)).astype(np.float64)
    x[0, :] += 1  # no zero gene
    for clip in (np.sqrt(40), 1.0):
        np.testing.assert_allclose(opr.residual_variances(x, theta=theta, clip=clip),
                                   numba_loop_variance(x, theta=theta, clip=clip), rtol=1e-12)


def test_oracle_clip_of_the_first_batch_binds():
    """clip=None becomes sqrt(n) of the first batch in np.unique order, reused by every later batch."""
    rng = np.random.default_rng(2)
    sizes = {"b": 60, "a": 9, "c": 200}  # "a" is first in np.unique order and the smallest
    batch = np.concatenate([[k] * v for k, v in sizes.items()])
    x = rng.negative_binomial(2, 0.2, (len(batch), 30)).astype(np.float64)
    x[batch == "c", 3] = 400  # residuals far beyond sqrt(9) in batch c
    x[batch == "c", 4] = 0
    x[rng.random(len(batch)) < 0.5, 4] = 0
    var, clip = opr.batch_residual_variances(x, batch=batch)
    assert clip == np.sqrt(9)
    xc = x[batch == "c"]
    nz = xc.sum(axis=0) != 0
    np.testing.assert_array_equal(var[2][nz], opr.residual_variances(xc[:, nz], theta=100, clip=3.0))
    own = opr.residual_variances(xc[:, nz], theta=100, clip=np.sqrt(200))
    assert not np.allclose(var[2][nz], own)


def test_oracle_gene_zero_in_one_batch_only():
    rng = np.random.default_rng(3)
    batch = np.array([0] * 100 + [1] * 150 + [2] * 80)
    x = rng.negative_binomial(3, 0.3, (330, 20)).astype(np.float64)
    x[batch == 1, 7] = 0
    assert x[:, 7].sum() > 0
    df, var = opr.highly_variable_pearson_residuals(x, batch=batch, n_top_genes=5)
    assert var[1, 7] == 0 and var[0, 7] > 0 and var[2, 7] > 0
    assert df["residual_variances"].iloc[7] == var[:, 7].mean()


# ------------------------------------------------------------------------------------------ errors and warnings
@pytest.fixture
def no_device(monkeypatch):
    def touched(*a, **k):
        raise AssertionError("the device was touched")

    monkeypatch.setattr(_ops, "DeviceX", touched)
    monkeypatch.setattr(_abi, "default_context", touched)


def _counts(dtype=np.float32, fmt=sparse.csr_matrix):
    x = np.random.default_rng(0).negative_binomial(2, 0.3, (30, 12)).astype(dtype)
    return MiniAnnData(fmt(x))


PP = sb.experimental.pp


@pytest.mark.parametrize("call", ["hvg", "norm", "pca", "recipe"])
def test_theta_and_clip_errors(no_device, call):
    fn = dict(hvg=lambda ad, **k: PP.highly_variable_genes(ad, n_top_genes=5, **k),
              norm=PP.normalize_pearson_residuals, pca=PP.normalize_pearson_residuals_pca,
              recipe=lambda ad, **k: PP.recipe_pearson_residuals(ad, n_top_genes=5, **k))[call]
    for theta in (0, -1):
        with pytest.raises(ValueError, match="Pearson residuals require theta > 0"):
            fn(_counts(), theta=theta)
    with pytest.raises(ValueError, match=r"Pearson residuals require `clip>=0` or `clip=None`\."):
        fn(_counts(), clip=-1)


def test_hvg_argument_errors(no_device):
    with pytest.raises(ValueError, match="requires the argument `n_top_genes`"):
        PP.highly_variable_genes(_counts())
    with pytest.raises(ValueError, match="only `flavor=pearson_residuals` is available"):
        PP.highly_variable_genes(_counts(), n_top_genes=5, flavor="seurat_v3")
    with pytest.raises(ValueError, match="expects an `AnnData` argument"):
        PP.highly_variable_genes(np.ones((4, 4)), n_top_genes=2)


@pytest.mark.parametrize("call", ["hvg", "norm"])
def test_unsupported_input(no_device, call):
    fn = (lambda ad: PP.highly_variable_genes(ad, n_top_genes=5)) if call == "hvg" else PP.normalize_pearson_residuals
    backed = MiniAnnData(ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts"))
    with pytest.raises(NotImplementedError, match="is not implemented for matrices of type"):
        fn(backed)
    with pytest.raises(NotImplementedError, match="supports float32, float64, int32 and int64 data, not uint16"):
        fn(_counts(np.uint16))
    with pytest.raises(NotImplementedError, match="supports CSR, CSC and dense X, not coo"):
        fn(_counts(fmt=sparse.coo_matrix))


def test_normalize_argument_errors(no_device):
    with pytest.raises(ValueError, match="`copy=True` cannot be used with `inplace=False`."):
        PP.normalize_pearson_residuals(_counts(), copy=True, inplace=False)
    ad = _counts()
    ad.layers["c"] = ad.X.copy()
    ad.obsm["c"] = ad.X.toarray()
    with pytest.raises(ValueError, match="Only one of `layer`, or `obsm` can be specified."):
        PP.normalize_pearson_residuals(ad, layer="c", obsm="c")


@pytest.mark.parametrize("fmt", [sparse.csr_matrix, np.asarray])
def test_check_values_warnings(no_device, fmt):
    ad = _counts(np.float32, fmt)
    x = ad.X.toarray() if sparse.issparse(ad.X) else ad.X
    i, j = np.nonzero(x)
    x[i[0], j[0]] = 0.5
    ad.X = fmt(x)
    with pytest.warns(UserWarning, match=r"`flavor='pearson_residuals'` expects raw count data, but non-integers"):
        with pytest.raises(AssertionError, match="device was touched"):
            PP.highly_variable_genes(ad, n_top_genes=5)
    with pytest.warns(UserWarning, match=r"`normalize_pearson_residuals\(\)` expects raw count data, but non-integers"):
        with pytest.raises(AssertionError, match="device was touched"):
            PP.normalize_pearson_residuals(ad)
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("error")
        with pytest.raises(AssertionError, match="device was touched"):
            PP.highly_variable_genes(ad, n_top_genes=5, check_values=False)
        with pytest.raises(AssertionError, match="device was touched"):
            PP.normalize_pearson_residuals(ad, check_values=False)
        with pytest.raises(AssertionError, match="device was touched"):
            PP.normalize_pearson_residuals(_counts())  # integer-valued float32: no warning


def test_check_nonnegative_integers():
    from scanpy_b200._pearson import check_nonnegative_integers as f

    assert f(np.array([[0, 3]], dtype=np.int64))
    assert f(sparse.csr_matrix(np.array([[0.0, 3.0]], dtype=np.float32)))
    assert not f(np.array([[0.5, 3.0]]))
    assert not f(np.array([[-1, 3]]))
    assert not f(np.array([[-0.0, 3.0]]))  # signbit, as the reference

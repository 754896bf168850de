"""Analytic Pearson residuals on the H100: the reference's own tests (tests/test_normalization.py:98-323,
tests/test_highly_variable_genes.py:159-349) restated on the pbmc68k counts, the oracle (oracle/pearson.py) across
formats, dtypes and batches, NaN propagation, determinism across runs and chunk sizes, the chain into neighbors and
leiden, and one larger case."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import pca as opca, pearson as opr
from scanpy_b200 import _pearson
from scanpy_b200._compat import MiniAnnData, settings
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

PP = sb.experimental.pp
FMTS = {"csr": sparse.csr_matrix, "csc": sparse.csc_matrix, "dense": np.asarray}
DTYPES = [np.float32, np.float64, np.int32, np.int64]


def counts():
    """700 x 765 integer counts."""
    return ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts").tocsr().astype(np.float32)


def batches(n, seed=0):
    """Three unequal batches, labels out of np.unique order."""
    rng = np.random.default_rng(seed)
    return rng.choice(np.array(["s2", "s0", "s1"]), size=n, p=[0.5, 0.15, 0.35])


def pbmc(fmt="csr", dtype=np.float32):
    x = counts()
    x = FMTS[fmt](x if fmt != "dense" else x.toarray()).astype(dtype)
    ad = MiniAnnData(x, obs=pd.DataFrame(index=[f"c{i}" for i in range(x.shape[0])]),
                     var=pd.DataFrame(index=[f"g{i}" for i in range(x.shape[1])]))
    ad.obs["batch"] = batches(x.shape[0])
    return ad


def assert_close(got, ref):
    """float32: within one ulp of the fp64 oracle; float64: 1e-12 relative.  NaN exactly where the oracle has NaN."""
    assert got.shape == ref.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    g, r = got[ok].astype(np.float64), ref[ok]
    if got.dtype == np.float32:
        bad = np.abs(g - r) > np.spacing(np.abs(r).astype(np.float32)).astype(np.float64)
        assert not bad.any(), f"{bad.sum()} values beyond one float32 ulp: {g[bad][:4]} vs {r[bad][:4]}"
    else:
        np.testing.assert_allclose(g, r, rtol=1e-12, atol=1e-300)


# ------------------------------------------------------------------------------------------ the reference's tests
@pytest.mark.parametrize("sparsity_func", [np.array, sparse.csr_matrix])
@pytest.mark.parametrize("dtype", ["float32", "int64"])
@pytest.mark.parametrize("theta", [0.01, 1, 100, np.inf])
@pytest.mark.parametrize("clip", [None, 1, np.inf])
def test_normalize_pearson_residuals_values(sparsity_func, dtype, theta, clip):
    x = np.array([[3, 6], [2, 4], [1, 0]])
    ns, ps = np.sum(x, axis=1), np.sum(x, axis=0) / np.sum(x)
    mu = np.outer(ns, ps)
    reference = (x - mu) / np.sqrt(mu) if np.isinf(theta) else (x - mu) / np.sqrt(mu + mu**2 / theta)
    adata = MiniAnnData(sparsity_func(x).astype(dtype))
    output = PP.normalize_pearson_residuals(adata, theta=theta, clip=clip, inplace=False)
    output_x = output["X"]
    PP.normalize_pearson_residuals(adata, theta=theta, clip=clip, inplace=True)
    assert {"pearson_residuals_normalization"} <= adata.uns.keys()
    assert adata.uns["pearson_residuals_normalization"] == dict(theta=theta, clip=clip, computed_on="adata.X")
    np.testing.assert_array_equal(adata.X, output_x)
    assert output_x.dtype == (np.float32 if dtype == "float32" else np.float64)
    if clip is None:
        threshold = np.sqrt(adata.shape[0]).astype(np.float32)
        assert np.max(output_x) <= threshold and np.min(output_x) >= -threshold
    elif np.isinf(clip):
        assert np.allclose(output_x, reference)
    else:
        assert np.max(output_x) <= clip and np.min(output_x) >= -clip


@pytest.mark.parametrize(("params", "match"), [(dict(theta=0), r"Pearson residuals require theta > 0"),
                                               (dict(theta=-1), r"Pearson residuals require theta > 0"),
                                               (dict(clip=-1), r"Pearson residuals require `clip>=0` or `clip=None`.")])
def test_normalize_pearson_residuals_errors(params, match):
    with pytest.raises(ValueError, match=match):
        PP.normalize_pearson_residuals(pbmc(), **params)


def test_normalize_pearson_residuals_warnings():
    import warnings

    ad = pbmc("dense")
    i, j = np.nonzero(ad.X)
    ad.X[i[0], j[0]] = 0.5
    with pytest.warns(UserWarning, match=r"`normalize_pearson_residuals\(\)` expects raw count data"):
        PP.normalize_pearson_residuals(ad.copy())
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        PP.normalize_pearson_residuals(ad.copy(), check_values=False)


def _check_pearson_hvg_columns(output_df, n_top_genes):
    assert pd.api.types.is_float_dtype(output_df["residual_variances"].dtype)
    assert output_df["highly_variable"].to_numpy().dtype is np.dtype("bool")
    assert np.sum(output_df["highly_variable"]) == n_top_genes
    assert np.nanmax(output_df["highly_variable_rank"].to_numpy()) <= n_top_genes - 1


@pytest.mark.parametrize("subset", [True, False])
@pytest.mark.parametrize("clip", [None, np.inf, 30])
@pytest.mark.parametrize("theta", [100, np.inf])
@pytest.mark.parametrize("n_top_genes", [100, 200])
def test_pearson_residuals_general(subset, clip, theta, n_top_genes):
    adata = pbmc()
    adata.var = pd.DataFrame(index=adata.var.index)
    residuals_res = PP.normalize_pearson_residuals(adata, clip=clip, theta=theta, inplace=False)
    residual_variances_reference = np.var(residuals_res["X"], axis=0)
    if subset:
        top_n_idx = np.argsort(-residual_variances_reference)[:n_top_genes]
        residual_variances_reference = residual_variances_reference[top_n_idx]
    output_df = PP.highly_variable_genes(adata, flavor="pearson_residuals", n_top_genes=n_top_genes, subset=subset,
                                         inplace=False, clip=clip, theta=theta)
    PP.highly_variable_genes(adata, flavor="pearson_residuals", n_top_genes=n_top_genes, subset=subset, inplace=True,
                             clip=clip, theta=theta)
    pd.testing.assert_frame_equal(output_df, adata.var)
    for key in ["highly_variable", "means", "variances", "residual_variances", "highly_variable_rank"]:
        assert key in output_df.columns
    if subset:
        sort_output_idx = np.argsort(-output_df["residual_variances"].to_numpy())
        assert np.allclose(output_df["residual_variances"].to_numpy()[sort_output_idx], residual_variances_reference)
    else:
        assert np.allclose(output_df["residual_variances"].to_numpy(), residual_variances_reference)
    hvg_idx = np.where(output_df["highly_variable"])[0]
    topn_idx = np.sort(np.argsort(-output_df["residual_variances"].to_numpy())[:n_top_genes])
    assert np.all(hvg_idx == topn_idx)
    assert np.nanmin(output_df["highly_variable_rank"].to_numpy()) == 0
    _check_pearson_hvg_columns(output_df, n_top_genes)


@pytest.mark.parametrize("subset", [True, False])
@pytest.mark.parametrize("n_top_genes", [100, 200])
def test_pearson_residuals_batch(subset, n_top_genes):
    adata = pbmc()
    adata.var = pd.DataFrame(index=adata.var.index)
    output_df = PP.highly_variable_genes(adata, flavor="pearson_residuals", n_top_genes=n_top_genes,
                                         batch_key="batch", subset=subset, inplace=False)
    PP.highly_variable_genes(adata, flavor="pearson_residuals", n_top_genes=n_top_genes, batch_key="batch",
                             subset=subset, inplace=True)
    pd.testing.assert_frame_equal(output_df, adata.var)
    for key in ["highly_variable", "means", "variances", "residual_variances", "highly_variable_rank",
                "highly_variable_nbatches", "highly_variable_intersection"]:
        assert key in output_df.columns
    _check_pearson_hvg_columns(output_df, n_top_genes)
    nbatches = len(np.unique(adata.obs["batch"]))
    assert output_df["highly_variable_intersection"].to_numpy().dtype is np.dtype("bool")
    assert np.sum(output_df["highly_variable_intersection"]) <= n_top_genes * nbatches
    assert adata.uns["hvg"] == {"flavor": "pearson_residuals", "computed_on": "adata.X"}


@pytest.mark.parametrize("n_hvgs", [100, 200])
@pytest.mark.parametrize("n_comps", [30, 50])
@pytest.mark.parametrize(("do_hvg", "params", "n_var_copy_name"), [
    (False, dict(), "n_genes"), (True, dict(), "n_hvgs"), (True, dict(mask_var=None), "n_genes"),
    (False, dict(mask_var="test_mask"), "n_unmasked")])
def test_normalize_pearson_residuals_pca(n_hvgs, n_comps, do_hvg, params, n_var_copy_name):
    adata = pbmc()
    n_cells, n_genes = adata.shape
    n_unmasked = n_genes - 5
    adata.var["test_mask"] = np.r_[np.repeat(True, n_unmasked), np.repeat(False, n_genes - n_unmasked)]
    n_var_copy = dict(n_genes=n_genes, n_hvgs=n_hvgs, n_unmasked=n_unmasked)[n_var_copy_name]
    if do_hvg:
        PP.highly_variable_genes(adata, flavor="pearson_residuals", n_top_genes=n_hvgs)
    adata_pca = PP.normalize_pearson_residuals_pca(adata.copy(), inplace=False, n_comps=n_comps, **params)
    PP.normalize_pearson_residuals_pca(adata, inplace=True, n_comps=n_comps, **params)
    assert type(adata_pca) is type(adata)
    for ad, n_var_ret in ((adata_pca, n_var_copy), (adata, n_genes)):
        assert {"pearson_residuals_normalization", "pca"} <= ad.uns.keys()
        assert ad.obsm["X_pca"].shape == (n_cells, n_comps)
        assert ad.shape == (n_cells, n_var_ret)
        assert ad.varm["PCs"].shape == (n_var_ret, n_comps)
    assert sum(np.sum(np.abs(adata.varm["PCs"]), axis=1) == 0) == (n_genes - n_var_copy)
    np.testing.assert_array_equal(adata.obsm["X_pca"], adata_pca.obsm["X_pca"])
    df = adata.uns["pearson_residuals_normalization"]["pearson_residuals_df"]
    assert isinstance(df, pd.DataFrame) and df.shape == (n_cells, n_var_copy)
    assert (df.index == adata.obs.index).all()
    np.testing.assert_array_equal(df.to_numpy(), adata_pca.X)


@pytest.mark.parametrize("n_hvgs", [100, 200])
@pytest.mark.parametrize("n_comps", [30, 50])
def test_normalize_pearson_residuals_recipe(n_hvgs, n_comps):
    adata = pbmc()
    n_cells, n_genes = adata.shape
    adata_pca, hvg = PP.recipe_pearson_residuals(adata.copy(), inplace=False, n_comps=n_comps, n_top_genes=n_hvgs)
    assert adata_pca.obsm["X_pca"].shape == (n_cells, n_comps)
    assert adata_pca.shape == (n_cells, n_hvgs)
    assert adata_pca.varm["PCs"].shape == (n_hvgs, n_comps)
    assert {"means", "variances", "residual_variances", "highly_variable_rank", "highly_variable"} <= set(hvg.columns)
    assert np.sum(hvg["highly_variable"]) == n_hvgs
    assert hvg.shape[0] == n_genes
    PP.recipe_pearson_residuals(adata, inplace=True, n_comps=n_comps, n_top_genes=n_hvgs)
    assert adata.obsm["X_pca"].shape == (n_cells, n_comps)
    assert adata.shape == (n_cells, n_genes)
    assert adata.varm["PCs"].shape == (n_genes, n_comps)
    assert sum(np.sum(np.abs(adata.varm["PCs"]), axis=1) == 0) == n_genes - n_hvgs
    np.testing.assert_array_equal(adata.obsm["X_pca"], adata_pca.obsm["X_pca"])


# ------------------------------------------------------------------------------------------ against the oracle
def check_hvg(df, x, *, batch, n_top_genes, theta=100.0, clip=None):
    ref, _ = opr.highly_variable_pearson_residuals(x, theta=theta, clip=clip, n_top_genes=n_top_genes, batch=batch,
                                                   var_names=df.index)
    np.testing.assert_allclose(df["residual_variances"], ref["residual_variances"], rtol=1e-10, atol=0)
    keys = ("means", "variances") + (("highly_variable_nbatches", "highly_variable_intersection") if batch is not None
                                     else ())
    for key in keys:
        np.testing.assert_array_equal(df[key].to_numpy(), ref[key].to_numpy(), err_msg=key)
    # genes whose variance lies within 1e-9 of the n_top-th value could swap ranks; there are none here
    rv = ref["residual_variances"].to_numpy()
    cut = np.sort(rv)[::-1][n_top_genes - 1]
    near = np.abs(rv - cut) <= 1e-9 * abs(cut)
    assert near.sum() == 1, "ties at the selection cut-off"
    np.testing.assert_array_equal(df["highly_variable"].to_numpy(), ref["highly_variable"].to_numpy())
    return ref


@pytest.mark.parametrize("n_batches", [1, 3])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
def test_matches_oracle(fmt, dtype, n_batches):
    ad = pbmc(fmt, dtype)
    x = counts()
    key = "batch" if n_batches == 3 else None
    df = PP.highly_variable_genes(ad, n_top_genes=200, batch_key=key, inplace=False)
    check_hvg(df, x, batch=ad.obs["batch"].to_numpy() if key else None, n_top_genes=200)
    out = PP.normalize_pearson_residuals(ad, inplace=False)["X"]
    assert out.dtype == (np.float32 if dtype == np.float32 else np.float64)
    assert_close(out, opr.pearson_residuals(x))


@pytest.mark.parametrize("fmt", ["csr", "dense"])
def test_nan_where_the_oracle_has_nan(fmt):
    x = counts().toarray()
    x[5] = 0  # a zero-count cell
    x[:, 9] = 0  # a zero gene
    ad = MiniAnnData(FMTS[fmt](x))
    out = PP.normalize_pearson_residuals(ad, inplace=False)["X"]
    ref = opr.pearson_residuals(x)
    assert np.isnan(ref[5]).all() and np.isnan(ref[:, 9]).all()
    assert_close(out, ref)
    ad.obs["batch"] = batches(x.shape[0])
    df = PP.highly_variable_genes(ad, n_top_genes=100, batch_key="batch", inplace=False)
    _, var = opr.highly_variable_pearson_residuals(x, n_top_genes=100, batch=ad.obs["batch"].to_numpy())
    np.testing.assert_allclose(df["residual_variances"], var.mean(axis=0), rtol=1e-10, atol=0, equal_nan=True)
    assert np.isnan(df["residual_variances"]).any() and df["residual_variances"].iloc[9] == 0


def nb_counts(n, g, *, seed=0, dtype=np.float32):
    rng = np.random.default_rng(seed)
    mean = rng.lognormal(-1.5, 1.5, g)
    depth = rng.lognormal(0, 0.4, n)
    return sparse.csr_matrix(rng.negative_binomial(2, 2 / (2 + np.outer(depth, mean).clip(1e-6, 1e4))).astype(dtype))


@pytest.mark.parametrize("fmt", ["csr", "dense"])
def test_bit_identical_across_runs_and_chunk_sizes(fmt, monkeypatch):
    x = nb_counts(5000, 300, seed=1)
    batch = np.random.default_rng(2).choice(["a", "b", "c"], 5000, p=[0.5, 0.3, 0.2])

    def run():
        ad = MiniAnnData(FMTS[fmt](x if fmt == "csr" else x.toarray()))
        ad.obs["batch"] = batch
        df = PP.highly_variable_genes(ad, n_top_genes=50, batch_key="batch", inplace=False)
        return df, PP.normalize_pearson_residuals(ad, inplace=False)["X"]

    df0, x0 = run()
    df1, x1 = run()
    pd.testing.assert_frame_equal(df0, df1, check_exact=True)
    np.testing.assert_array_equal(x0, x1)
    monkeypatch.setattr(settings, "chunk_size", 1500)  # dense blocks of one subtile; several output blocks
    monkeypatch.setattr(_pearson, "PARTIAL_BYTES", 2 * 3 * 300 * 8)  # CSR: 2 subtiles
    df2, x2 = run()
    pd.testing.assert_frame_equal(df0, df2, check_exact=True)
    np.testing.assert_array_equal(x0, x2)


def test_recipe_neighbors_leiden_chain():
    ad = pbmc()
    PP.recipe_pearson_residuals(ad, n_top_genes=200, n_comps=20)
    hv = ad.var["highly_variable"].to_numpy()
    ref = opca.pca_arpack(opr.pearson_residuals(counts()[:, hv]), 20, dtype="float64")
    xp = opca.align_signs(ad.obsm["X_pca"].astype(np.float64), ref["X_pca"])
    rel = np.linalg.norm(xp - ref["X_pca"], axis=0) / np.linalg.norm(ref["X_pca"], axis=0)
    assert rel.max() < 1e-4, rel
    sb.pp.neighbors(ad, n_neighbors=15)
    sb.tl.leiden(ad, flavor="igraph", n_iterations=-1)
    assert ad.obs["leiden"].nunique() > 1


def test_larger_case_against_the_oracle():
    """50k x 4000 in 4 batches: many subtiles per batch and 16 slabs."""
    x = nb_counts(50_000, 4000, seed=3)
    batch = np.random.default_rng(4).choice(["p", "q", "r", "s"], 50_000, p=[0.4, 0.3, 0.2, 0.1])
    ad = MiniAnnData(x)
    ad.obs["batch"] = batch
    df = PP.highly_variable_genes(ad, n_top_genes=1000, batch_key="batch", inplace=False)
    check_hvg(df, x, batch=batch, n_top_genes=1000)

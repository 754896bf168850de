"""calculate_qc_metrics / filter_cells / filter_genes on the H100 against the oracle (oracle/qc.py) and the reference's
own tests (tests/test_qc_metrics.py, tests/test_preprocessing.py:611-676, the filter_cells docstring)."""
import logging

import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import preprocess as opp, qc as oqc
from scanpy_b200._compat import MiniAnnData, settings
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN
from test_qc_cpu import krumsiek11, mito_adata

pytestmark = pytest.mark.gpu

FMTS = {"csr": sparse.csr_matrix, "csc": sparse.csc_matrix, "dense": np.asarray}
COUNTS = GOLDEN / "pbmc68k_counts.zarr.zip"


def counts_adata():
    x = ZarrCSR(COUNTS, group="layers/counts").tocsr()
    var = pd.DataFrame(index=[f"g{i}" for i in range(x.shape[1])])
    var["mt"] = np.arange(x.shape[1]) % 17 == 0
    var["ribo"] = np.arange(x.shape[1]) < 40
    return MiniAnnData(x, obs=pd.DataFrame(index=[f"c{i}" for i in range(x.shape[0])]), var=var)


def assert_frames_match(got: pd.DataFrame, ref: pd.DataFrame, rtol=1e-12):
    assert list(got.columns) == list(ref.columns)
    assert list(got.index) == list(ref.index)
    for col in ref.columns:
        assert got[col].dtype == ref[col].dtype, (col, got[col].dtype, ref[col].dtype)
        a, b = got[col].to_numpy(), ref[col].to_numpy()
        if np.issubdtype(b.dtype, np.integer):
            np.testing.assert_array_equal(a, b, err_msg=col)
        else:
            np.testing.assert_allclose(a, b, rtol=rtol, atol=0, equal_nan=True, err_msg=col)


def oracle_qc(ad, **kw):
    return oqc.calculate_qc_metrics(ad.X, obs_names=ad.obs.index, var=ad.var, **kw)


# ------------------------------------------------------------------------------------------ the reference's tests
@pytest.mark.parametrize("fmt", FMTS)
def test_qc_metrics(fmt):
    ad = mito_adata(fmt=fmt)
    sb.pp.calculate_qc_metrics(ad, qc_vars=["mito", "negative"], inplace=True)
    obs, var = ad.obs, ad.var
    x = sparse.csr_matrix(ad.X)
    assert (obs["n_genes_by_counts"] < ad.shape[1]).all()
    assert (obs["n_genes_by_counts"] >= obs["log1p_n_genes_by_counts"]).all()
    assert (obs["total_counts"] == np.ravel(x.sum(axis=1))).all()
    assert (obs["total_counts"] >= obs["log1p_total_counts"]).all()
    assert (obs["total_counts_mito"] >= obs["log1p_total_counts_mito"]).all()
    assert (obs["total_counts_negative"] == 0).all()
    assert (obs["pct_counts_in_top_50_genes"] <= obs["pct_counts_in_top_100_genes"]).all()
    for col in filter(lambda c: "negative" not in c, obs.columns):
        assert (obs[col] >= 0).all()
        assert (obs[col] != 0).any()
        if col.startswith("pct_counts_in_top"):
            assert (obs[col] <= 100).all()
    for col in var.columns.drop(["mito", "negative"]):
        assert (var[col] >= 0).all()
    assert (var["mean_counts"] < np.ravel(x.max(axis=0).toarray())).all()
    assert (var["mean_counts"] >= var["log1p_mean_counts"]).all()
    assert (var["total_counts"] >= var["log1p_total_counts"]).all()
    ref_obs, ref_var = oracle_qc(mito_adata(fmt=fmt), qc_vars=["mito", "negative"])
    assert_frames_match(obs[ref_obs.columns], ref_obs)
    assert_frames_match(var[ref_var.columns], ref_var)


@pytest.mark.parametrize("fmt", FMTS)
def test_qc_metrics_idempotent_format_and_no_log1p(fmt):
    ad = mito_adata(fmt=fmt)
    sb.pp.calculate_qc_metrics(ad, qc_vars=["mito", "negative"], inplace=True)
    old_obs, old_var = ad.obs.copy(), ad.var.copy()
    sb.pp.calculate_qc_metrics(ad, qc_vars=["mito", "negative"], inplace=True)
    assert set(ad.obs.columns) == set(old_obs.columns) and set(ad.var.columns) == set(old_var.columns)
    for col in ad.obs:
        assert np.array_equal(ad.obs[col], old_obs[col], equal_nan=True)
    # str and list qc_vars, and CSR vs this format, give the same frames
    o1, v1 = sb.pp.calculate_qc_metrics(mito_adata(fmt=fmt), qc_vars="mito")
    o2, v2 = sb.pp.calculate_qc_metrics(mito_adata(fmt="csr"), qc_vars=["mito"])
    assert_frames_match(o1, o2, rtol=0)
    assert_frames_match(v1, v2, rtol=0)
    o3, v3 = sb.pp.calculate_qc_metrics(mito_adata(fmt=fmt), qc_vars=["mito"], log1p=False)
    assert not o3.columns.str.startswith("log1p_").any() and not v3.columns.str.startswith("log1p_").any()


def test_qc_metrics_percentage():
    ad = mito_adata()
    for pt in ([], (), None, [1], [1, 2, 3, 10], range(1, 101)):
        obs, _ = sb.pp.calculate_qc_metrics(ad, percent_top=pt)
        ref, _ = oracle_qc(ad, percent_top=pt)
        assert_frames_match(obs, ref)
    with pytest.raises(IndexError):
        sb.pp.calculate_qc_metrics(ad, percent_top=[1, 2, 3, -5])
    with pytest.raises(IndexError):
        sb.pp.calculate_qc_metrics(ad, percent_top=[20, 30, 1001])


def test_layer_equals_x():
    ad = mito_adata()
    ad.layers["counts"] = ad.X.copy()
    o1, v1 = sb.pp.calculate_qc_metrics(ad)
    sb.pp.log1p(ad)
    o2, v2 = sb.pp.calculate_qc_metrics(ad, layer="counts")
    assert_frames_match(o2, o1, rtol=0)
    assert_frames_match(v2, v1, rtol=0)


# ------------------------------------------------------------------------------------------ parity on real counts
@pytest.mark.parametrize("percent_top", [(50, 100, 200, 500), (50, 100, 200)], ids=["m500_padded", "m200_select"])
def test_pbmc68k_counts_match_the_oracle(percent_top):
    ad = counts_adata()
    obs, var = sb.pp.calculate_qc_metrics(ad, qc_vars=["mt", "ribo"], percent_top=percent_top)
    ref_obs, ref_var = oracle_qc(counts_adata(), qc_vars=["mt", "ribo"], percent_top=percent_top)
    assert_frames_match(obs, ref_obs)
    assert_frames_match(var, ref_var)
    # two runs are bit-identical
    obs2, var2 = sb.pp.calculate_qc_metrics(ad, qc_vars=["mt", "ribo"], percent_top=percent_top)
    assert_frames_match(obs2, obs, rtol=0)
    assert_frames_match(var2, var, rtol=0)


def test_on_disk_counts_match_in_core(monkeypatch):
    """Chunks of 128 rows (not a divisor of 700) from the zarr store: bit-identical to the in-core run, X untouched."""
    monkeypatch.setattr(settings, "chunk_size", 128)
    backed = sb.read_zarr_backed(COUNTS, group="layers/counts")
    backed.var = counts_adata().var
    backed.obs = counts_adata().obs
    obs_d, var_d = sb.pp.calculate_qc_metrics(backed, qc_vars=["mt", "ribo"])
    obs_m, var_m = sb.pp.calculate_qc_metrics(counts_adata(), qc_vars=["mt", "ribo"])
    assert isinstance(backed.X, ZarrCSR)
    assert_frames_match(obs_d, obs_m, rtol=0)
    assert_frames_match(var_d, var_m, rtol=0)


# ------------------------------------------------------------------------------------------ adversarial rows
def _rows_csr(rows, g):
    indptr = np.r_[0, np.cumsum([len(v) for v, _ in rows])]
    return sparse.csr_matrix((np.concatenate([v for v, _ in rows]).astype(np.float32),
                              np.concatenate([c for _, c in rows]).astype(np.int32), indptr), shape=(len(rows), g))


def test_adversarial_rows_match_the_oracle():
    rng = np.random.default_rng(7)
    g = 60_000
    m = 20

    def cols(k):
        return np.sort(rng.choice(g, k, replace=False))

    rows = [(np.full(k, 3.0), cols(k)) for k in (m - 1, m, m + 1, 45)]                 # ties at the n-th value
    rows += [(rng.integers(1, 50, k).astype(float), cols(k)) for k in (m - 1, m, m + 1)]
    rows += [(np.zeros(0), np.zeros(0, int))]                                         # empty row -> NaN shares
    rows += [(np.r_[np.zeros(5), rng.integers(1, 9, 18)].astype(float), cols(23))]    # explicit zeros
    rows += [(rng.integers(-5, 6, k).astype(float), cols(k)) for k in (7, 19, 20, 21, 60)]   # negative values
    rows += [(rng.gamma(0.7, 2.0, k), cols(k)) for k in (10, 300)]                    # non-integer values
    rows += [(rng.integers(1, 1000, 50_000).astype(float), cols(50_000))]             # beyond the shared-memory staging
    rows += [(rng.standard_normal(3000), cols(3000))]                                 # long row, negatives
    x = _rows_csr(rows, g)
    ref_x = x.copy()
    ad = MiniAnnData(x)
    for pt in ((1, 5, 10, 20), (1, 2, 20), (50, 100, 200, 500)):
        obs, var = sb.pp.calculate_qc_metrics(ad, percent_top=pt)
        ref_obs, ref_var = oqc.calculate_qc_metrics(ref_x, obs_names=ad.obs.index, var=ad.var, percent_top=pt)
        assert_frames_match(obs, ref_obs, rtol=1e-6)
        assert_frames_match(var, ref_var, rtol=1e-6)
        assert np.isnan(obs.iloc[7][[c for c in obs.columns if c.startswith("pct_")]].to_numpy(float)).all()
        assert obs["n_genes_by_counts"].iloc[8] == 18
        obs2, _ = sb.pp.calculate_qc_metrics(ad, percent_top=pt)
        assert_frames_match(obs2, obs, rtol=0)


def test_n_equals_n_vars_and_long_rows_with_large_m():
    rng = np.random.default_rng(3)
    x = sparse.random(40, 3000, density=0.8, format="csr", dtype=np.float32, random_state=4)
    x.data = rng.integers(-20, 100, x.nnz).astype(np.float32)
    x.eliminate_zeros()
    ad = MiniAnnData(x)
    for pt in ((3000,), (1, 1000, 2999, 3000)):
        obs, _ = sb.pp.calculate_qc_metrics(ad, percent_top=pt)
        ref_obs, _ = oqc.calculate_qc_metrics(x, obs_names=ad.obs.index, var=ad.var, percent_top=pt)
        assert_frames_match(obs, ref_obs)


# ------------------------------------------------------------------------------------------ filters
def test_krumsiek11_filter_cells_docstring():
    x, obs_names, var_names = krumsiek11()
    x[x < 0.3] = 0
    ad = MiniAnnData(x, obs=pd.DataFrame(index=obs_names), var=pd.DataFrame(index=var_names))
    sb.pp.filter_cells(ad, min_genes=0)
    assert ad.n_obs == 640 and int(ad.obs["n_genes"].min()) == 1
    sb.pp.filter_cells(ad, min_genes=3)
    assert ad.n_obs == 554 and int(ad.obs["n_genes"].min()) == 3


def _raw_x():
    d = np.load(GOLDEN / "pbmc68k_raw_seurat_hvg.npz")
    return sparse.csr_matrix((d["raw_data"], d["raw_indices"], d["raw_indptr"]), shape=(700, 765))


CELL_KW = [dict(max_genes=100), dict(max_counts=100), dict(min_genes=20), dict(min_counts=20)]
GENE_KW = [dict(max_cells=100), dict(max_counts=100), dict(min_cells=20), dict(min_counts=20)]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kw", CELL_KW, ids=lambda d: next(iter(d)))
def test_filter_cells_matrix(fmt, kw):
    raw = _raw_x()
    ad = MiniAnnData(FMTS[fmt](raw.toarray() if fmt == "dense" else raw))
    ref_keep, ref_number = oqc.filter_cells(raw, **kw)
    sb.pp.filter_cells(ad, **kw)
    key = "n_genes" if "genes" in next(iter(kw)) else "n_counts"
    np.testing.assert_array_equal(ad.obs[key].to_numpy(), ref_number[ref_keep])
    assert ad.obs[key].dtype == ref_number.dtype
    got = ad.X.toarray() if sparse.issparse(ad.X) else ad.X
    np.testing.assert_array_equal(got, raw[ref_keep].toarray())
    keep, number = sb.pp.filter_cells(FMTS[fmt](raw.toarray() if fmt == "dense" else raw), **kw)
    np.testing.assert_array_equal(keep, ref_keep)
    np.testing.assert_array_equal(number, ref_number)
    assert number.dtype == ref_number.dtype


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kw", GENE_KW, ids=lambda d: next(iter(d)))
def test_filter_genes_matrix(fmt, kw):
    raw = _raw_x()
    ad = MiniAnnData(FMTS[fmt](raw.toarray() if fmt == "dense" else raw))
    ref_keep, ref_number = oqc.filter_genes(raw, **kw)
    keep, number = sb.pp.filter_genes(ad, inplace=False, **kw)
    np.testing.assert_array_equal(keep, ref_keep)
    np.testing.assert_array_equal(number, ref_number)
    assert ad.n_vars == 765
    sb.pp.filter_genes(ad, **kw)
    key = "n_cells" if "cells" in next(iter(kw)) else "n_counts"
    np.testing.assert_array_equal(ad.var[key].to_numpy(), ref_number[ref_keep])
    got = ad.X.toarray() if sparse.issparse(ad.X) else ad.X
    np.testing.assert_array_equal(got, raw[:, ref_keep].toarray())


def test_filter_copy_log_and_subset_of_every_axis(caplog):
    raw = _raw_x()
    rng = np.random.default_rng(0)
    ad = MiniAnnData(raw.copy(), obsm={"X_pca": rng.standard_normal((700, 3))}, varm={"PCs": rng.standard_normal((765, 3))},
                     obsp={"distances": sparse.random(700, 700, density=0.01, format="csr", random_state=0)})
    ad.layers["counts"] = raw.copy()
    with caplog.at_level(logging.INFO, logger="scanpy_b200"):
        out = sb.pp.filter_cells(ad, max_genes=150, copy=True)
    assert "`copy` is deprecated, use `inplace` instead." in caplog.text
    keep, _ = oqc.filter_cells(raw, max_genes=150)
    assert f"filtered out {int((~keep).sum())} cells that have more than 150 genes expressed" in caplog.text
    assert ad.n_obs == 700 and out.n_obs == keep.sum()
    sb.pp.filter_cells(ad, max_genes=150)
    np.testing.assert_array_equal(ad.obsm["X_pca"], out.obsm["X_pca"])
    np.testing.assert_array_equal(ad.obsp["distances"].toarray(), out.obsp["distances"].toarray())
    np.testing.assert_array_equal(ad.layers["counts"].toarray(), raw[keep].toarray())
    gkeep, _ = oqc.filter_genes(ad.X, min_cells=20)
    sb.pp.filter_genes(ad, min_cells=20)
    np.testing.assert_array_equal(ad.varm["PCs"], out.varm["PCs"][gkeep])
    np.testing.assert_array_equal(ad.layers["counts"].toarray(), raw[keep][:, gkeep].toarray())


def test_filter_to_nothing():
    x, obs_names, var_names = krumsiek11()
    x[x < 0.3] = 0
    ad = MiniAnnData(sparse.csr_matrix(x), obs=pd.DataFrame(index=obs_names), var=pd.DataFrame(index=var_names))
    sb.pp.filter_cells(ad, max_genes=0)
    assert ad.shape == (0, 11) and len(ad.obs["n_genes"]) == 0
    ad = MiniAnnData(sparse.csr_matrix(x))
    sb.pp.filter_genes(ad, min_cells=10_000)
    assert ad.shape == (640, 0)


def test_chain_filter_qc_normalize_log1p():
    """filter_cells(min_genes=200) -> filter_genes(min_cells=3) -> calculate_qc_metrics -> normalize_total -> log1p
    against the oracle filters and the oracle normalize_total / log1p on the host-subset matrix."""
    ad = counts_adata()
    x = ad.X.copy()
    sb.pp.filter_cells(ad, min_genes=200)
    sb.pp.filter_genes(ad, min_cells=3)
    assert ad.n_obs == 693
    ckeep, _ = oqc.filter_cells(x, min_genes=200)
    gkeep, _ = oqc.filter_genes(x[ckeep], min_cells=3)
    xs = x[ckeep][:, gkeep]
    np.testing.assert_array_equal(ad.X.toarray(), xs.toarray())
    sb.pp.calculate_qc_metrics(ad, qc_vars=["mt"], inplace=True)
    ref_obs, ref_var = oqc.calculate_qc_metrics(xs, obs_names=ad.obs.index, var=ad.var, qc_vars=["mt"])
    assert_frames_match(ad.obs[ref_obs.columns], ref_obs)
    assert_frames_match(ad.var[ref_var.columns], ref_var)
    sb.pp.normalize_total(ad, target_sum=1e4)
    sb.pp.log1p(ad)
    ref, _, _ = opp.normalize_total(xs, target_sum=1e4)
    ref = opp.log1p(ref)
    np.testing.assert_allclose(ad.X.toarray(), ref.toarray(), rtol=1e-6, atol=1e-6)

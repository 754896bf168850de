"""CPU tests for calculate_qc_metrics / filter_cells / filter_genes: the oracle against the reference's own literal tests
(tests/test_qc_metrics.py, the filter_cells docstring, tests/test_preprocessing.py:611-676), and the argument errors the
public functions raise before touching a device."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import qc as oqc
from scanpy_b200 import _abi
from scanpy_b200._compat import MiniAnnData
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN


def _no_gpu():
    import torch

    return not torch.cuda.is_available()


def mito_adata(seed=0, *, fmt="csr"):
    """The reference's `adata` / `adata_mito` fixtures: binomial(100, 0.005) counts, 1000 x 1000, `mito` = first 100
    genes, `negative` = none."""
    a = np.random.default_rng(seed).binomial(100, 0.005, (1000, 1000))
    x = {"csr": sparse.csr_matrix, "csc": sparse.csc_matrix, "dense": np.asarray}[fmt](a)
    var = pd.DataFrame(index=[f"gene{i}" for i in range(1000)])
    var["mito"] = np.r_[np.ones(100, bool), np.zeros(900, bool)]
    var["negative"] = False
    return MiniAnnData(x, obs=pd.DataFrame(index=[f"cell{i}" for i in range(1000)]), var=var)


def krumsiek11():
    d = np.load(GOLDEN / "krumsiek11.npz")
    return d["X"].copy(), d["obs_names"], d["var_names"]


# ------------------------------------------------------------------------------------------ oracle vs the reference's tests
@pytest.mark.parametrize("a", [np.ones((100, 100)), sparse.csr_matrix(np.ones((100, 100)))], ids=["dense", "sparse"])
def test_proportions(a):
    prop = oqc.top_proportions(a, 100)
    assert (prop[:, -1] == 1).all()
    assert np.array_equal(np.sort(prop, axis=1), prop)
    assert np.apply_along_axis(lambda x: len(np.unique(x)) == 1, 0, prop).all()
    assert (prop[:, 49] == 0.5).all()


def test_segments_binary():
    rng = np.random.default_rng(0)
    a = np.concatenate([np.zeros((300, 50)), np.ones((300, 50))], 1)
    a = np.apply_along_axis(rng.permutation, 1, a)
    for m in (a, sparse.csr_matrix(a)):
        seg = oqc.top_segment_proportions(m, [25, 50, 100])
        assert (seg[:, 0] == 0.5).all()
        assert (oqc.top_segment_proportions(m, [25]) == 0.5).all()
        assert (seg[:, 1] == 1.0).all()
        assert (seg[:, 2] == 1.0).all()
        segfull = oqc.top_segment_proportions(m, np.arange(100) + 1)
        assert (segfull == oqc.top_proportions(a, 100)).all()


@pytest.mark.parametrize("fmt", [np.asarray, sparse.csr_matrix, sparse.csc_matrix, sparse.coo_matrix])
def test_top_segments(fmt):
    seg = oqc.top_segment_proportions(fmt(np.ones((300, 100))), [50, 100])
    assert (seg[:, 0] == 0.5).all()
    assert (seg[:, 1] == 1.0).all()


def test_top_segment_sums_match_brute_force_sort():
    """Ties, negatives, explicit zeros and rows on both sides of m against sorting the padded row."""
    rng = np.random.default_rng(1)
    rows = [rng.integers(-3, 4, size=k).astype(np.float32) for k in (0, 1, 5, 9, 10, 11, 40)]
    rows += [rng.standard_normal(k).astype(np.float32) for k in (3, 10, 25)]
    rows += [np.full(12, 2.5, np.float32), -np.abs(rng.standard_normal(14)).astype(np.float32)]
    indptr = np.r_[0, np.cumsum([len(r) for r in rows])]
    data = np.concatenate(rows)
    ns = [1, 2, 3, 7, 10]
    got = oqc.top_segment_sums_csr(data, indptr, ns)
    for i, r in enumerate(rows):
        r = r.astype(np.float64)
        vec = np.sort(-np.partition(-r, 10)[:10])[::-1] if len(r) > 10 else np.r_[r, np.zeros(10 - len(r))]
        vec = np.sort(vec)[::-1]
        np.testing.assert_array_equal(got[i], np.cumsum(vec)[np.array(ns) - 1])


def test_qc_metrics_properties_on_the_oracle():
    """tests/test_qc_metrics.py::test_qc_metrics (the property set) on the oracle."""
    ad = mito_adata()
    obs, var = oqc.calculate_qc_metrics(ad.X, obs_names=ad.obs.index, var=ad.var, qc_vars=["mito", "negative"])
    x = ad.X
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
    for col in var.columns:
        assert (var[col] >= 0).all()
    assert (var["mean_counts"] < np.ravel(x.max(axis=0).toarray())).all()
    assert (var["mean_counts"] >= var["log1p_mean_counts"]).all()
    assert (var["total_counts"] >= var["log1p_total_counts"]).all()
    # integer X: integer totals, as `stats.sum` gives for integer input
    assert obs["total_counts"].dtype == np.int64 and obs["n_genes_by_counts"].dtype == np.int64


def test_qc_metrics_percentage_on_the_oracle():
    """tests/test_qc_metrics.py::test_qc_metrics_percentage."""
    ad = mito_adata()
    for pt in ([], (), None, [1, 2, 3, 10], [1]):
        oqc.calculate_qc_metrics(ad.X, obs_names=ad.obs.index, var=ad.var, percent_top=pt)
    for pt in ([1, 2, 3, -5], [20, 30, 1001]):
        with pytest.raises(IndexError):
            oqc.calculate_qc_metrics(ad.X, obs_names=ad.obs.index, var=ad.var, percent_top=pt)


def test_krumsiek11_filter_cells_docstring():
    """src/scanpy/preprocessing/_simple.py:104-133."""
    x, _, var_names = krumsiek11()
    assert x.shape == (640, 11) and list(var_names[:2]) == ["Gata2", "Gata1"]
    x[x < 0.3] = 0
    keep, number = oqc.filter_cells(x, min_genes=0)
    assert keep.sum() == 640 and number.min() == 1
    keep, number = oqc.filter_cells(x, min_genes=3)
    assert keep.sum() == 554 and number[keep].min() == 3


def test_pbmc68k_counts_shape_of_the_golden():
    """The counts fixture exercises both top-n branches: with m = 200, 689 rows select and 11 pad (4 sit at 200)."""
    x = ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts").tocsr()
    nnz = np.diff(x.indptr)
    assert x.shape == (700, 765) and x.nnz == 174_400 and nnz.min() == 183 and nnz.max() == 409
    assert (nnz > 200).sum() == 689 and (nnz == 200).sum() == 4
    assert oqc.filter_cells(x, min_genes=200)[0].sum() == 693


@pytest.mark.parametrize(("kw", "kept"), [(dict(min_cells=20), 728), (dict(max_cells=100), 189),
                                          (dict(min_counts=20), 738), (dict(max_counts=100), 120)])
def test_pbmc68k_raw_filter_genes_counts(kw, kept):
    d = np.load(GOLDEN / "pbmc68k_raw_seurat_hvg.npz")
    x = sparse.csr_matrix((d["raw_data"], d["raw_indices"], d["raw_indptr"]), shape=(700, 765))
    assert oqc.filter_genes(x, **kw)[0].sum() == kept
    ckw = {k.replace("cells", "genes"): v for k, v in kw.items()}
    assert oqc.filter_cells(x, **ckw)[0].sum() == (700 if next(iter(ckw)).startswith("min") else 0)


# ------------------------------------------------------------------------------------------ argument errors, no device
def test_filter_option_count_errors():
    x = sparse.random(20, 10, density=0.3, format="csr", dtype=np.float32, random_state=0)
    with pytest.raises(ValueError, match=r"Provide exactly one of the optional parameters `min_counts`, `min_genes`, "
                                         r"`max_counts`, `max_genes` per call\."):
        sb.pp.filter_cells(x)
    with pytest.raises(ValueError, match=r"`min_counts`, `min_genes`"):
        sb.pp.filter_cells(MiniAnnData(x), min_genes=1, min_counts=2)
    with pytest.raises(ValueError, match=r"Provide exactly one of the optional parameters `min_counts`, `min_cells`, "
                                         r"`max_counts`, `max_cells` per call\."):
        sb.pp.filter_genes(x, min_cells=1, max_cells=3)


def test_filters_refuse_on_disk_x():
    ad = sb.read_zarr_backed(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts")
    with pytest.raises(NotImplementedError, match=r"filter_cells is not implemented for matrices of type "
                                                  r"<class 'scanpy_b200._io.ZarrCSR'>"):
        sb.pp.filter_cells(ad, min_genes=3)
    with pytest.raises(NotImplementedError, match=r"filter_genes is not implemented for matrices of type"):
        sb.pp.filter_genes(ad, min_cells=3)


def test_qc_argument_errors_before_the_device():
    ad = mito_adata()
    with pytest.raises(IndexError, match="Positions outside range of features."):
        sb.pp.calculate_qc_metrics(ad, percent_top=[1, 2, 3, -5])
    with pytest.raises(IndexError, match="Positions outside range of features."):
        sb.pp.calculate_qc_metrics(ad, percent_top=[20, 30, 1001])
    with pytest.raises(KeyError):
        sb.pp.calculate_qc_metrics(ad, qc_vars="not_a_column")
    with pytest.raises(ValueError, match="Cannot use expression from both layer and raw"):
        sb.pp.calculate_qc_metrics(ad, layer="counts", use_raw=True)


def test_qc_parallel_is_deprecated():
    ad = mito_adata()
    with pytest.warns(FutureWarning, match="Argument `parallel` is deprecated"):
        with pytest.raises(IndexError):  # stops before the device
            sb.pp.calculate_qc_metrics(ad, percent_top=[0], parallel=True)


def test_qc_and_filters_have_no_cpu_fallback():
    if not _no_gpu():
        pytest.skip("GPU present")
    ad = mito_adata()
    with pytest.raises(_abi.B200Error):
        sb.pp.calculate_qc_metrics(ad, qc_vars="mito")
    with pytest.raises(_abi.B200Error):
        sb.pp.filter_cells(ad, min_genes=3)
    with pytest.raises(_abi.B200Error):
        sb.pp.filter_genes(ad.X, min_cells=3)


def test_mini_anndata_inplace_subsetting():
    rng = np.random.default_rng(0)
    x = sparse.random(6, 5, density=0.5, format="csr", dtype=np.float32, random_state=1)
    ad = MiniAnnData(x, obsm={"X_pca": rng.standard_normal((6, 2))}, varm={"PCs": rng.standard_normal((5, 2))},
                     obsp={"distances": sparse.csr_matrix(rng.standard_normal((6, 6)))})
    ad.layers["counts"] = x.toarray() * 2
    full = (x.toarray(), ad.obsm["X_pca"].copy(), ad.varm["PCs"].copy(), ad.obsp["distances"].toarray())
    cells = np.array([True, False, True, True, False, True])
    genes = np.array([False, True, True, False, True])
    ad._inplace_subset_obs(cells)
    ad._inplace_subset_var(genes)
    assert ad.shape == (4, 3) and list(ad.obs.index) == ["0", "2", "3", "5"] and list(ad.var.index) == ["1", "2", "4"]
    np.testing.assert_array_equal(ad.X.toarray(), full[0][cells][:, genes])
    np.testing.assert_array_equal(ad.layers["counts"], 2 * full[0][cells][:, genes])
    np.testing.assert_array_equal(ad.obsm["X_pca"], full[1][cells])
    np.testing.assert_array_equal(ad.varm["PCs"], full[2][genes])
    np.testing.assert_array_equal(ad.obsp["distances"].toarray(), full[3][cells][:, cells])
    ad._inplace_subset_obs(np.zeros(4, bool))
    assert ad.shape == (0, 3) and ad.obsm["X_pca"].shape == (0, 2) and ad.obsp["distances"].shape == (0, 0)

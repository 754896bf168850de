"""regress_out on the H100: the reference's own tests (tests/test_preprocessing.py:360-503), the oracle
(oracle/regress.py) across formats, dtypes and branches, chunking, and the tutorial's preprocessing chain."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import pca as opca, preprocess as opp, regress as orr
from scanpy_b200._compat import MiniAnnData, settings
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN
from test_regress_out_cpu import pbmc68k_small

pytestmark = pytest.mark.gpu

FMTS = {"csr": sparse.csr_matrix, "csc": sparse.csc_matrix, "dense": np.asarray}
DTYPES = [np.float32, np.float64, np.int32, np.int64]


def assert_close(got, ref, x):
    """float32: within one ulp of the oracle; float64: 1e-12 relative, plus 1e-10 * max|x| for cancelled entries."""
    assert got.dtype == ref.dtype, (got.dtype, ref.dtype)
    scale = float(np.abs(x.toarray() if sparse.issparse(x) else np.asarray(x)).max())
    if got.dtype == np.float32:
        tol = np.spacing(np.abs(ref)) + 1e-12 * scale
        bad = np.abs(got.astype(np.float64) - ref.astype(np.float64)) > tol
        assert not bad.any(), f"{bad.sum()} entries beyond one ulp, e.g. {got[bad][:4]} vs {ref[bad][:4]}"
    else:
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-10 * scale)


def random_adata(n=1000, g=100, *, dtype=np.float64, seed=0):
    rng = np.random.default_rng(seed)
    x = sparse.random(n, g, density=0.6, format="csr", random_state=rng)
    if np.dtype(dtype).kind in "iu":
        x = sparse.random(n, g, density=0.6, format="csr", dtype=np.uint16, random_state=rng).astype(dtype)
    ad = MiniAnnData(x, obs=pd.DataFrame(index=[f"c{i}" for i in range(n)]))
    ad.obs["percent_mito"] = rng.random(n)
    ad.obs["n_counts"] = np.ravel(x.sum(axis=1))
    return ad


# ------------------------------------------------------------------------------------------ the reference's tests
def test_regress_out_ordinal():
    ad = random_adata()
    single = sb.pp.regress_out(ad, keys=["n_counts", "percent_mito"], n_jobs=1, copy=True)
    multi = sb.pp.regress_out(ad, keys=["n_counts", "percent_mito"], n_jobs=8, copy=True)
    assert ad.X.shape == single.X.shape
    np.testing.assert_array_equal(single.X, multi.X)


@pytest.mark.parametrize("dtype", [np.int64, np.float64, np.int32])
def test_regress_out_layer(dtype):
    ad = random_adata(dtype=dtype)
    cast = {np.int64: np.float64, np.float64: np.float64, np.int32: np.float32}[dtype]
    ad.layers["counts"] = ad.X.copy().astype(cast)
    single = sb.pp.regress_out(ad, keys=["n_counts", "percent_mito"], n_jobs=1, copy=True)
    layer = sb.pp.regress_out(ad, layer="counts", keys=["n_counts", "percent_mito"], n_jobs=1, copy=True)
    assert ad.X.shape == single.X.shape
    np.testing.assert_allclose(single.X, layer.layers["counts"])


def test_regress_out_categorical():
    rng = np.random.default_rng()
    ad = MiniAnnData(sparse.random(1000, 100, density=0.6, format="csr", random_state=rng))
    ad.obs["batch"] = pd.Categorical(rng.integers(1, 4, size=1000))
    multi = sb.pp.regress_out(ad, keys="batch", n_jobs=8, copy=True)
    assert ad.X.shape == multi.X.shape


def test_regress_out_constants():
    rng = np.random.default_rng()
    ad = MiniAnnData(np.hstack((np.full((10, 1), 0.0), np.full((10, 1), 1.0))))
    ad.obs["percent_mito"] = rng.random(10)
    ad.obs["n_counts"] = ad.X.sum(axis=1)
    before = ad.X.copy()
    sb.pp.regress_out(ad, keys=["n_counts", "percent_mito"])
    np.testing.assert_array_equal(ad.X, before)
    assert ad.X.dtype == before.dtype


@pytest.mark.parametrize(("keys", "golden", "atol"), [(["n_counts", "percent_mito"], "regress_test_small", 0.0),
                                                      (["bulk_labels"], "regress_test_small_cat", 1e-6)])
def test_regress_out_reproducible(keys, golden, atol):
    x, obs, d = pbmc68k_small()
    ad = MiniAnnData(x, obs=obs)
    sb.pp.regress_out(ad, keys=keys)
    np.testing.assert_allclose(ad.X, d[golden], atol=atol)


def test_regress_out_constants_equivalent():
    from sklearn.datasets import make_blobs

    x, cat = make_blobs(100, 20, random_state=0)
    a = MiniAnnData(np.hstack([x, np.zeros((100, 5))]), obs=pd.DataFrame({"cat": pd.Categorical(cat)}))
    b = MiniAnnData(x, obs=pd.DataFrame({"cat": pd.Categorical(cat)}))
    sb.pp.regress_out(a, "cat")
    sb.pp.regress_out(b, "cat")
    np.testing.assert_equal(a.X[:, :20], b.X)
    assert (a.X[:, 20:] == 0).all()


@pytest.mark.parametrize(("float_dtype", "int_dtype"), [(np.float32, np.uint32), (np.float64, np.uint64)])
def test_regress_out_int(float_dtype, int_dtype):
    """The dtype-invariance half of the reference's test_regress_out_int: integer counts give what their float cast
    gives.  Its golden (cat_regressor_for_int_input.npy) needs pbmc3k, which is a download; the pbmc68k counts stand in."""
    counts = ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts").tocsr()[:200, :200].toarray()
    labels = pd.Categorical(["A"] * 100 + ["B"] * 100)
    a = MiniAnnData(counts.astype(float_dtype), obs=pd.DataFrame({"labels": labels}))
    b = MiniAnnData(counts.astype(int_dtype), obs=pd.DataFrame({"labels": labels}))
    sb.pp.regress_out(a, keys=["labels"])
    sb.pp.regress_out(b, keys=["labels"])
    assert a.X.dtype == b.X.dtype == np.float64
    np.testing.assert_array_equal(a.X, b.X)


# ------------------------------------------------------------------------------------------ against the oracle
N, G = 2500, 300  # not multiples of the 16-row steps, the 1024-row subtiles or the 256-column slabs


def oracle_case(case, seed=0):
    """(x [N x G] float64 with ~30 % zeros, obs, keys, oracle kwargs)."""
    rng = np.random.default_rng(seed)
    x = rng.gamma(1.5, 2.0, (N, G)).round(1)
    x[rng.random((N, G)) < 0.3] = 0
    x[:, 7] = 0.0
    x[:, 11] = 3.0
    obs = pd.DataFrame({"k1": rng.random(N), "k2": rng.normal(size=N)})
    if case == "shortcut":
        keys = ["k1", "k2"]
    elif case == "duplicate":
        obs["k3"] = obs["k1"]
        keys = ["k1", "k2", "k3"]
    elif case == "constant_key":
        obs["k3"] = 0.5
        keys = ["k1", "k3"]
    else:
        n_cat = 300 if case == "cat300" else 12
        codes = rng.integers(0, n_cat, N)
        codes[codes == 4] = 5  # unused category
        if case == "cat_missing":
            codes[rng.random(N) < 0.1] = -1
        obs["cat"] = pd.Categorical.from_codes(codes, [f"c{i}" for i in range(n_cat)])
        return x, obs, ["cat"], dict(codes=codes, n_categories=n_cat, exact_means=True)
    return x, obs, keys, dict(regressors=orr.design(obs, keys))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("case", ["shortcut", "duplicate", "constant_key", "cat_missing", "cat", "cat300"])
def test_matches_oracle(case, fmt, dtype):
    x, obs, keys, kw = oracle_case(case)
    x = x.astype(dtype) if np.dtype(dtype).kind == "f" else np.rint(x).astype(dtype)
    ref = orr.regress_out(x, **kw)
    ad = MiniAnnData(FMTS[fmt](x), obs=obs)
    sb.pp.regress_out(ad, keys)
    assert isinstance(ad.X, np.ndarray) and ad.X.shape == (N, G)
    assert_close(ad.X, ref, x)
    if case != "shortcut":  # the GLM paths return constant genes unchanged
        assert (ad.X[:, 7] == 0).all() and (ad.X[:, 11] == 3).all()


@pytest.mark.parametrize("case", ["shortcut", "duplicate", "cat_missing"])
def test_explicit_stored_zeros(case):
    x, obs, keys, kw = oracle_case(case, seed=3)
    # store zeros explicitly: all of gene 7 (zero everywhere) and every zero of gene 20
    stored = x != 0
    stored[:, [7, 20]] = True
    xs = sparse.csr_matrix((x[stored], np.nonzero(stored)), shape=(N, G))
    assert (xs.data == 0).sum() >= N
    ad = MiniAnnData(xs, obs=obs)
    sb.pp.regress_out(ad, keys)
    assert_close(ad.X, orr.regress_out(x, **kw), x)


@pytest.mark.parametrize("fmt", ["csr", "dense"])
@pytest.mark.parametrize("case", ["shortcut", "duplicate", "cat_missing", "cat300"])
def test_chunk_size_is_bit_identical(case, fmt, monkeypatch):
    x, obs, keys, _ = oracle_case(case, seed=4)
    x = x.astype(np.float32)
    whole = MiniAnnData(FMTS[fmt](x), obs=obs)
    sb.pp.regress_out(whole, keys)
    monkeypatch.setattr(settings, "chunk_size", 700)  # several output blocks; dense pass-1 blocks of one subtile
    chunked = MiniAnnData(FMTS[fmt](x), obs=obs)
    sb.pp.regress_out(chunked, keys)
    np.testing.assert_array_equal(whole.X, chunked.X)


def test_tutorial_chain():
    """filter -> QC -> normalize_total -> log1p -> HVG subset -> regress_out(total_counts, pct_counts_mt) ->
    scale(max_value=10) -> pca, each device step checked against the oracle from the device's own input."""
    counts = ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts").tocsr().astype(np.float32)
    var = pd.DataFrame(index=[f"g{i}" for i in range(counts.shape[1])])
    var["mt"] = np.arange(counts.shape[1]) % 23 == 0
    ad = MiniAnnData(counts, obs=pd.DataFrame(index=[f"c{i}" for i in range(counts.shape[0])]), var=var)
    sb.pp.filter_cells(ad, min_genes=10)
    sb.pp.filter_genes(ad, min_cells=3)
    sb.pp.calculate_qc_metrics(ad, qc_vars=["mt"], inplace=True)
    sb.pp.normalize_total(ad, target_sum=1e4)
    sb.pp.log1p(ad)
    sb.pp.highly_variable_genes(ad, min_mean=0.0125, max_mean=3, min_disp=0.5)
    ad._inplace_subset_var(ad.var["highly_variable"].to_numpy())
    before = ad.X.copy()
    sb.pp.regress_out(ad, ["total_counts", "pct_counts_mt"])
    ref = orr.regress_out(before, regressors=orr.design(ad.obs, ["total_counts", "pct_counts_mt"]))
    assert_close(ad.X, ref, before)
    sb.pp.scale(ad, max_value=10)
    ref_scaled, _, _ = opp.scale(ref, max_value=10)
    np.testing.assert_allclose(ad.X, ref_scaled, rtol=1e-5, atol=1e-5)
    sb.pp.pca(ad, n_comps=20)
    ref_pca = opca.pca_arpack(ref_scaled.astype(np.float64), 20, dtype="float64")
    xp = opca.align_signs(ad.obsm["X_pca"].astype(np.float64), ref_pca["X_pca"])
    rel = np.linalg.norm(xp - ref_pca["X_pca"], axis=0) / np.linalg.norm(ref_pca["X_pca"], axis=0)
    assert rel[:10].max() < 1e-3, rel

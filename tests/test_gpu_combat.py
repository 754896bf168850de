"""combat on the H100: the oracle (oracle/combat.py) across formats, dtypes, batch counts and covariates, determinism
across runs and chunk sizes, the reference's own tests (tests/test_combat.py), a pbmc68k chain and a large case."""
import numpy as np
import pandas as pd
import pytest
from scipy import sparse

import scanpy_b200 as sb
from oracle import combat as oc
from scanpy_b200._compat import MiniAnnData, settings
from scanpy_b200._io import ZarrCSR

from conftest import GOLDEN
from test_combat_cpu import blobs, oracle_inputs

pytestmark = pytest.mark.gpu

FMTS = {"csr": sparse.csr_matrix, "csc": sparse.csc_matrix, "dense": np.asarray}
DTYPES = [np.float32, np.float64, np.int32, np.int64]
N, G = 2500, 300  # not multiples of the 16-row steps, the 1024-row subtiles or the 256-column slabs
TOL = 1e-10  # times max|x|


def oracle_case(case, seed=0):
    """(x [N x G] float64 with ~40 % zeros, obs, covariates).  Gene 7 is zero everywhere (zero variance); gene 13 is
    zero in batch 1 only."""
    rng = np.random.default_rng(seed)
    n_batch = {"one_batch": 1, "two_batches": 2}.get(case, 7)
    b = rng.integers(0, n_batch, N)
    if n_batch == 7:
        b[b == 6] = 5
        b[rng.choice(N, 2, replace=False)] = 6  # a batch of exactly 2 cells
    counts = rng.gamma(1.5, 3.0, (N, G)) * (rng.random((N, G)) > 0.4) * (1 + 0.5 * b[:, None] * rng.random(G))
    x = counts.round(0)
    x[:, 7] = 0.0
    x[b == 1, 13] = 0.0
    cats = [f"b{i}" for i in range(n_batch)]
    if case == "unused_categories":
        cats = ["gone"] + cats + ["never"]
    obs = pd.DataFrame({"batch": pd.Categorical.from_codes(b + (case == "unused_categories"), cats)},
                       index=[f"c{i}" for i in range(N)])
    covariates = []
    if case == "numeric":
        obs["num"] = rng.normal(size=N)
        obs["k"] = rng.integers(0, 4, N)
        x += np.rint(2 * (obs["num"].to_numpy() > 0))[:, None] * (x > 0)
        covariates = ["num", "k"]
    if case == "many_numeric":  # more than 4 covariate columns: the kernels' wide variant
        for k in range(6):
            obs[f"n{k}"] = rng.normal(size=N)
        x += np.rint(obs[["n0", "n3"]].to_numpy().sum(axis=1) > 0)[:, None] * (x > 0)
        covariates = [f"n{k}" for k in range(6)]
    if case == "categorical":
        obs["group"] = pd.Categorical(rng.choice(["p", "q", "r"], N))
        obs["flag"] = rng.random(N) < 0.3
        obs["num"] = rng.normal(size=N)
        covariates = ["group", "flag", "num"]
    return x, obs, covariates


def max_err(got, ref, x) -> float:
    scale = float(np.abs(x.toarray() if sparse.issparse(x) else np.asarray(x, dtype=np.float64)).max())
    return float(np.abs(got - ref).max() / scale)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("case", ["one_batch", "two_batches", "seven_batches", "numeric", "many_numeric",
                                  "unused_categories"])
def test_matches_oracle(case, fmt, dtype, capsys):
    x, obs, covariates = oracle_case(case)
    x = x.astype(dtype)
    design, idx = oracle_inputs(obs, "batch", covariates)
    ref, inter = oc.combat(x, design, idx)
    ad = MiniAnnData(FMTS[fmt](x), obs=obs)
    sb.pp.combat(ad, "batch", covariates=covariates or None)
    assert isinstance(ad.X, np.ndarray) and ad.X.dtype == np.float64 and ad.X.shape == (N, G)
    assert "Found 1 genes with zero variance." in capsys.readouterr().out
    err = max_err(ad.X, ref, x)
    print(f"combat {case} {fmt} {np.dtype(dtype).name}: max |device - oracle| / max|x| = {err:.3g}")
    assert err < TOL, err
    np.testing.assert_array_equal(ad.X[:, 7], inter["stand_mean"][:, 7])  # zero variance: stand_mean (here 0)


@pytest.mark.parametrize("fmt", FMTS)
def test_categorical_covariates_run(fmt):
    """A categorical covariate makes the reference's design rank-deficient: `~ 0 + Q(a)` codes every level of the first
    factor, and those columns sum to the batch columns' sum.  inv(DᵀD) is then finite but meaningless (condition
    ~1e17), and the reference's own result depends on the rounding of its expression order, so it is not compared to
    the oracle.  The design itself is pinned on the CPU; here the path runs end to end."""
    x, obs, covariates = oracle_case("categorical")
    ad = MiniAnnData(FMTS[fmt](x), obs=obs)
    out = sb.pp.combat(ad, "batch", covariates=covariates, inplace=False)
    assert out.shape == (N, G) and np.isfinite(out).all()


def test_bit_identical_across_runs_and_chunk_sizes(monkeypatch):
    x, obs, covariates = oracle_case("numeric", seed=4)
    x = x.astype(np.float32)
    results = []
    for fmt in ("csr", "dense"):
        for chunk in (settings.chunk_size, 1500, 700, 700):
            monkeypatch.setattr(settings, "chunk_size", chunk)
            results.append(sb.pp.combat(MiniAnnData(FMTS[fmt](x), obs=obs), "batch", covariates=covariates,
                                        inplace=False))
    for r in results[1:]:
        np.testing.assert_array_equal(r, results[0])


def test_nan_and_inf_are_rejected():
    x, obs, _ = oracle_case("two_batches")
    for bad in (np.nan, np.inf, -np.inf):
        y = x.copy()
        y[5, 3] = bad
        with pytest.raises(ValueError, match="requires finite values"):
            sb.pp.combat(MiniAnnData(sparse.csr_matrix(y), obs=obs), "batch")


# ------------------------------------------------------------------------------------------ the reference's tests
def test_covariates():
    rng = np.random.default_rng()
    ad = blobs()
    key = "blobs"
    x1 = sb.pp.combat(ad, key=key, inplace=False)
    ad.obs["cat1"] = rng.binomial(3, 0.5, size=ad.n_obs)
    ad.obs["cat2"] = rng.binomial(2, 0.1, size=ad.n_obs)
    ad.obs["num1"] = rng.standard_normal(ad.n_obs)
    x2 = sb.pp.combat(ad, key=key, covariates=["cat1", "cat2", "num1"], inplace=False)
    sb.pp.combat(ad, key=key, covariates=["cat1", "cat2", "num1"], inplace=True)
    assert x1.shape == x2.shape
    np.testing.assert_array_equal(ad.X, x2)


def test_combat_obs_names():
    """Non-unique obs names give what unique ones give."""
    rng = np.random.default_rng()
    x = rng.random((200, 100))
    batch = pd.Categorical(rng.integers(0, 2, (200,)))
    a = MiniAnnData(x.copy(), obs=pd.DataFrame({"batch": batch}, index=np.repeat(np.arange(100), 2).astype(str)))
    b = MiniAnnData(x.copy(), obs=pd.DataFrame({"batch": batch}, index=[str(i) for i in range(200)]))
    sb.pp.combat(a, "batch")
    sb.pp.combat(b, "batch")
    np.testing.assert_array_equal(a.X, b.X)


def test_combat_single_cell_batch():
    ad = blobs()
    ad.obs["batch"] = pd.Categorical(["single"] + ["other"] * (ad.n_obs - 1))
    with pytest.raises(ValueError, match="fewer than 2 cells"):
        sb.pp.combat(ad, key="batch")


def test_silhouette():
    from sklearn.metrics import silhouette_score

    ad = blobs()
    sb.pp.combat(ad, "blobs")
    sb.pp.pca(ad)
    sh = silhouette_score(ad.obsm["X_pca"][:, :2], ad.obs["blobs"].values)
    assert sh < 0.1


# ------------------------------------------------------------------------------------------ chains and scale
def test_pbmc68k_chain():
    """normalize_total -> log1p -> HVG subset -> combat on a synthetic batch with a per-batch shift -> pca -> neighbors
    -> leiden.  The batch silhouette in PCA space drops from above 0.15 (0.20 measured) to below 0.05 (about 0)."""
    from sklearn.metrics import silhouette_score

    counts = ZarrCSR(GOLDEN / "pbmc68k_counts.zarr.zip", group="layers/counts").tocsr().astype(np.float32)
    n = counts.shape[0]
    ad = MiniAnnData(counts, obs=pd.DataFrame(index=[f"c{i}" for i in range(n)]))
    sb.pp.normalize_total(ad, target_sum=1e4)
    sb.pp.log1p(ad)
    sb.pp.highly_variable_genes(ad, n_top_genes=500)
    ad._inplace_subset_var(ad.var["highly_variable"].to_numpy())
    rng = np.random.default_rng(0)
    batch = rng.integers(0, 3, n)
    ad.obs["batch"] = pd.Categorical(batch.astype(str))
    shift = rng.normal(0.0, 0.6, (3, ad.n_vars))
    x = ad.X.toarray() + shift[batch]  # the injected batch effect
    before = MiniAnnData(x.copy(), obs=ad.obs.copy())
    sb.pp.pca(before, n_comps=20)
    sh_before = silhouette_score(before.obsm["X_pca"], batch)
    ad.X = x
    design, idx = oracle_inputs(ad.obs, "batch")
    ref, _ = oc.combat(x, design, idx)
    sb.pp.combat(ad, "batch")
    assert max_err(ad.X, ref, x) < TOL
    sb.pp.pca(ad, n_comps=20)
    sh_after = silhouette_score(ad.obsm["X_pca"], batch)
    print(f"pbmc68k batch silhouette: {sh_before:.3f} before combat, {sh_after:.3f} after")
    assert sh_before > 0.15 and sh_after < 0.05
    sb.pp.neighbors(ad, n_neighbors=15)
    sb.tl.leiden(ad, flavor="igraph", n_iterations=-1)
    assert ad.obs["leiden"].nunique() > 1


def test_large_against_oracle_on_sampled_rows():
    """200k x 2000 log-normalised CSR with 16 batches; the oracle needs the whole matrix for the fit, the comparison
    uses 4000 sampled rows."""
    rng = np.random.default_rng(7)
    n, g, nb = 200_000, 2000, 16
    b = rng.integers(0, nb, n)
    x = sparse.random(n, g, density=0.1, format="csr", dtype=np.float32, random_state=rng)
    x.data = np.log1p(x.data * 30).astype(np.float32)
    x = sparse.csr_matrix(x.multiply((1 + 0.05 * b)[:, None]).astype(np.float32))
    obs = pd.DataFrame({"batch": pd.Categorical(b)})
    got = sb.pp.combat(MiniAnnData(x, obs=obs), "batch", inplace=False)
    design, idx = oracle_inputs(obs, "batch")
    ref, _ = oc.combat(x, design, idx)
    rows = rng.choice(n, 4000, replace=False)
    err = max_err(got[rows], ref[rows], x)
    print(f"combat 200k x 2000, 16 batches: max |device - oracle| / max|x| = {err:.3g}")
    assert err < TOL, err

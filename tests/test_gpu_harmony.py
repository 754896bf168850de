"""`pp.harmony_integrate` on the device against the reference's recorded outputs, the fp64 oracle and live sklearn."""
from __future__ import annotations

import numpy as np
import pandas as pd
import pytest

from oracle import harmony as oh
from scanpy_b200 import _harmony as hm
from scanpy_b200._compat import MiniAnnData
from test_harmony_cpu import case_args, golden_cases, pbmc68k

pytestmark = pytest.mark.gpu

NEG = dict(tol_harmony=-1.0, tol_clustering=-1.0)  # never converged: every schedule runs to its iteration caps


def device_fit(x, codes, n_levels, *, centers, rng, **kw):
    stats = {}
    z = hm.fit(x, codes, n_levels, gen=np.random.default_rng(rng), centers=centers, stats=stats, **kw)
    return z, stats["iterations"]


def full_args(**kw):
    args = dict(theta=2.0, sigma=0.1, n_clusters=None, max_iter_harmony=10, max_iter_clustering=200, tol_harmony=1e-4,
                tol_clustering=1e-5, ridge_lambda=1.0, block_proportion=0.05, tau=0, alpha=0.2,
                batch_prune_threshold=1e-5, stabilized_penalty=True, dynamic_lambda=True)
    args.update(kw)
    return args


@pytest.mark.parametrize("case", list(golden_cases()))
def test_golden_cases_from_recorded_centres(case):
    x, obs, g = pbmc68k()
    p = golden_cases()[case]
    codes, n_levels = hm.get_batch_codes(obs, p["keys"])
    args = case_args(p)
    rng = args.pop("rng")
    z, its = device_fit(x.astype(np.float64), codes, n_levels, centers=g[f"{case}/centers"], rng=rng, **args)
    assert its == g[f"{case}/iters"].tolist()
    err = np.abs(z[g["rows"]] - g[f"{case}/out"]).max() / np.abs(x).max()
    assert err <= 1e-8, err


def synthetic(n=1501, d=20, n_batches=(4,), seed=0, unused=False):
    """Three planted clusters plus a shift per batch level of every key."""
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, 3, size=n)
    centres = rng.normal(scale=4.0, size=(3, d))
    x = centres[lab] + rng.normal(size=(n, d))
    obs = {}
    for j, nb in enumerate(n_batches):
        b = rng.integers(0, nb, size=n)
        x += rng.normal(scale=2.0, size=(nb, d))[b]
        cats = [f"k{j}_{i}" for i in range(nb + (1 if unused and j == 0 else 0))]
        obs[f"key{j}"] = pd.Categorical.from_codes(b, cats)
    return x, pd.DataFrame(obs), lab


ORACLE_CASES = {
    "harmony2": dict(),
    "harmony1": dict(stabilized_penalty=False, dynamic_lambda=False, ridge_lambda=0.7),
    "two_keys": dict(keys=2, theta=[2.0, 0.5]),
    "two_keys_theta0": dict(keys=2, theta=[2.0, 0.0], stabilized_penalty=False, dynamic_lambda=False),
    "one_cluster": dict(n_clusters=1),
    "unused_category": dict(unused=True),
    "one_block": dict(block_proportion=1.0),
    "pruning": dict(batch_prune_threshold=0.2, n_clusters=8),
    "tau": dict(tau=3, sigma=0.2),
}


def oracle_case(name, dtype):
    spec = dict(ORACLE_CASES[name])
    keys = spec.pop("keys", 1)
    unused = spec.pop("unused", False)
    x, obs, _ = synthetic(n_batches=(4, 3)[:keys], unused=unused)
    codes, n_levels = hm.get_batch_codes(obs, list(obs.columns))
    args = full_args(n_clusters=6, max_iter_harmony=3, max_iter_clustering=5, **NEG)
    args.update(spec)
    x = x.astype(dtype)
    z64 = x.astype(np.float64)
    z64 /= np.linalg.norm(z64, axis=1, keepdims=True)
    centers, _ = oh.kmeans_start(z64, args["n_clusters"], hm.spawn_random_state(np.random.default_rng(11)))
    return x, codes, n_levels, centers, args


@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_device_matches_oracle_f64(name):
    x, codes, n_levels, centers, args = oracle_case(name, np.float64)
    z, its = device_fit(x, codes, n_levels, centers=centers, rng=11, **args)
    want, wits = oh.harmony(x, codes, n_levels, centers=centers, rng=11, **args)
    assert its == wits == [5, 5, 5]
    err = np.abs(z - want).max() / np.abs(x).max()
    assert err <= 1e-8, err


@pytest.mark.parametrize("name", ["harmony2", "harmony1", "two_keys", "pruning"])
def test_device_matches_oracle_f32(name):
    """float32 stores Z, R and the output in float32 and does the dots and the exponent in float32.  A float32 dot of
    unit rows is off by ~1e-7; times |term| = 2 / sigma = 20 that moves log r by ~2e-6, and r, the correction weights
    and z_hat follow with the same relative error, compounded over 3 outer x 5 clustering iterations.  1e-4 x max|x|
    allows for that growth; a schedule or indexing fault moves the result by more than 1e-2 x max|x|."""
    x, codes, n_levels, centers, args = oracle_case(name, np.float32)
    z, its = device_fit(x, codes, n_levels, centers=centers, rng=11, **args)
    want, _ = oh.harmony(x.astype(np.float64), codes, n_levels, centers=centers, rng=11, **args)
    assert z.dtype == np.float32
    err = np.abs(z - want).max() / np.abs(x).max()
    assert err <= 1e-4, err


@pytest.mark.parametrize("n_clusters", [2, 23, 50])
def test_kmeans_start_matches_sklearn(n_clusters):
    from sklearn.cluster import KMeans

    x, _, _ = pbmc68k()
    x = x.astype(np.float64)
    dev = hm._Dev(x, np.zeros((len(x), 1), dtype=np.int32), 1)
    got = hm.kmeans_start(dev, n_clusters, hm.spawn_random_state(np.random.default_rng(0)), np.float64)
    z = x / np.linalg.norm(x, axis=1, keepdims=True)
    want = KMeans(n_clusters, random_state=hm.spawn_random_state(np.random.default_rng(0)), max_iter=25).fit(z)
    np.testing.assert_allclose(got, want.cluster_centers_, rtol=0, atol=1e-10)


def _measure(x, base, norm):
    if norm == "r":
        return np.array([np.corrcoef(x[:, i], base[:, i])[0, 1] for i in range(x.shape[1])])
    return np.array([np.linalg.norm(x[:, i] - base[:, i]) / np.linalg.norm(base[:, i]) for i in range(x.shape[1])])


def test_public_call_quality_against_reference():
    from scanpy_b200 import pp

    x, obs, g = pbmc68k()
    adata = MiniAnnData(np.zeros((len(x), 1), dtype=np.float32), obs=obs, obsm={"X_pca": x})
    pp.harmony_integrate(adata, "bulk_labels", rng=0)
    got = adata.obsm["X_pca_harmony"]
    assert got.dtype == np.float64
    got = got[g["rows"]]
    base = g["harmony2/out"]
    assert _measure(base, got, "r").min() > 0.95
    assert _measure(base, got, "L2").max() < 0.1
    # the k-means start is sklearn's, so the run follows the reference's schedule
    assert np.abs(got - base).max() <= 1e-8 * np.abs(x).max()


def test_two_runs_same_bits():
    from scanpy_b200 import pp

    x, obs, _ = synthetic(n=4001, n_batches=(5, 3))
    outs = []
    for _ in range(2):
        adata = MiniAnnData(np.zeros((len(x), 1), dtype=np.float32), obs=obs, obsm={"X_pca": x})
        pp.harmony_integrate(adata, ["key0", "key1"], rng=3, max_iter_harmony=3)
        outs.append(adata.obsm["X_pca_harmony"])
    assert outs[0].tobytes() == outs[1].tobytes()


def test_end_to_end_pca_harmony_neighbors_leiden():
    from scipy import sparse
    from sklearn.metrics import adjusted_rand_score

    import scanpy_b200 as sb

    rng = np.random.default_rng(7)
    n, g, n_batch = 6000, 300, 4
    lab = rng.integers(0, 4, size=n)
    batch = rng.integers(0, n_batch, size=n)
    programs = rng.gamma(2.0, 1.0, size=(4, g)) * (rng.random((4, g)) < 0.2) * 6.0
    shifts = rng.gamma(2.0, 1.0, size=(n_batch, g)) * (rng.random((n_batch, g)) < 0.1)
    counts = rng.poisson(1.0 + programs[lab] + shifts[batch]).astype(np.float32)
    x = np.log1p(counts)
    adata = sb.MiniAnnData(sparse.csr_matrix(x),
                           obs=pd.DataFrame({"batch": pd.Categorical(batch.astype(str))}))
    sb.pp.pca(adata, n_comps=20)

    def same_batch_share(rep):
        sb.pp.neighbors(adata, n_neighbors=15, use_rep=rep)
        d = adata.obsp["distances"].tocoo()
        return float(np.mean(batch[d.row] == batch[d.col]))

    before = same_batch_share("X_pca")
    sb.pp.harmony_integrate(adata, "batch", rng=0)
    after = same_batch_share("X_pca_harmony")
    sb.tl.leiden(adata, flavor="igraph", n_iterations=-1)
    ari = adjusted_rand_score(lab, adata.obs["leiden"].to_numpy())
    print(f"same-batch kNN share {before:.3f} -> {after:.3f} (batch proportion {1 / n_batch:.3f}), ARI {ari:.3f}")
    assert before > 0.9
    assert after < 0.45  # the fp64 oracle from sklearn's start reaches 0.36 on these data
    assert ari > 0.9

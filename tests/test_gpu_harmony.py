"""`pp.harmony_integrate` on the device against the reference's recorded outputs, the fp64 oracle and live sklearn."""
from __future__ import annotations

import numpy as np
import pandas as pd
import pytest

from oracle import harmony as oh
from scanpy_b200 import _harmony as hm
from scanpy_b200._compat import MiniAnnData
from test_harmony_cpu import case_args, golden_cases, pbmc68k, repeated_points

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
    # real shapes: groups above CHUNK_ROWS = 2048 cells and K·(d+1) = 5,100 outputs (3 slices) in wsums
    "default_k": dict(n=12_000, d=50, levels=(5,), n_clusters=None),
    # more than 48 KB of shared memory in step, apply and wsums
    "wide_basis": dict(n=8000, d=100, levels=(4,), n_clusters=100),
    # the caps: K = d = 128 and 128 marginal codes (code_sums at 132 KB of shared memory), the multi-key solve
    "caps": dict(n=6000, d=128, levels=(64, 64), n_clusters=128),
    # 120 codes, thousands of code tuples of 1 to 3 cells
    "many_tuples": dict(n=20_000, d=30, levels=(40, 40, 40), n_clusters=20),
}
SHAPED = ["default_k", "wide_basis", "caps", "many_tuples"]


def oracle_case(name, dtype):
    """A case's data, codes, k-means centres and arguments.  `n`, `d` and `levels` (per key) shape the data; the
    schedule is NEG's, so every case runs max_iter_harmony x max_iter_clustering iterations."""
    spec = dict(ORACLE_CASES[name])
    keys = spec.pop("keys", 1)
    unused = spec.pop("unused", False)
    n, d = spec.pop("n", 1501), spec.pop("d", 20)
    x, obs, _ = synthetic(n=n, d=d, n_batches=spec.pop("levels", (4, 3)[:keys]), unused=unused)
    codes, n_levels = hm.get_batch_codes(obs, list(obs.columns))
    args = full_args(n_clusters=6, max_iter_harmony=3, max_iter_clustering=5, **NEG)
    args.update(spec)
    x = x.astype(dtype)
    z64 = x.astype(np.float64)
    z64 /= np.linalg.norm(z64, axis=1, keepdims=True)
    k = args["n_clusters"] or max(int(min(100, n / 30)), 2)
    centers, _ = oh.kmeans_start(z64, k, hm.spawn_random_state(np.random.default_rng(11)))
    return x, codes, n_levels, centers, args


def schedule(args):
    return [args["max_iter_clustering"]] * args["max_iter_harmony"]


@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_device_matches_oracle_f64(name):
    x, codes, n_levels, centers, args = oracle_case(name, np.float64)
    z, its = device_fit(x, codes, n_levels, centers=centers, rng=11, **args)
    want, wits = oh.harmony(x, codes, n_levels, centers=centers, rng=11, **args)
    assert its == wits == schedule(args)
    err = np.abs(z - want).max() / np.abs(x).max()
    assert err <= 1e-8, err


@pytest.mark.parametrize("name", ["harmony2", "harmony1", "two_keys", "pruning", *SHAPED])
def test_device_matches_oracle_f32(name):
    """float32 stores Z, R and the output in float32 and does the dots and the exponent in float32.  A float32 dot of
    unit rows is off by ~1e-7; times |term| = 2 / sigma = 20 that moves log r by ~2e-6, and r, the correction weights
    and z_hat follow with the same relative error, compounded over 3 outer x 5 clustering iterations.  1e-4 x max|x|
    allows for that growth; a schedule or indexing fault moves the result by more than 1e-2 x max|x|."""
    x, codes, n_levels, centers, args = oracle_case(name, np.float32)
    z, its = device_fit(x, codes, n_levels, centers=centers, rng=11, **args)
    want, wits = oh.harmony(x.astype(np.float64), codes, n_levels, centers=centers, rng=11, **args)
    assert its == wits == schedule(args)
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


def _dev_kmeans(z, n_clusters, seed):
    dev = hm._Dev(z, np.zeros((len(z), 1), dtype=np.int32), 1)
    return hm.kmeans_start(dev, n_clusters, hm.spawn_random_state(np.random.default_rng(seed)), z.dtype)


@pytest.mark.parametrize("d", [50, 128])
@pytest.mark.parametrize("n_clusters", [33, 100, 128])
@pytest.mark.parametrize("n", [1025, 20_000])
def test_kmeans_start_matches_oracle_at_real_shapes(n, n_clusters, d):
    """Clusters on every lane of `labels_kernel` (up to four per lane), Lloyd sums over several CHUNK_ROWS chunks and
    the segmented k-means++ search (n > 1024), against the oracle's k-means start, and live sklearn at one shape."""
    x, _, _ = synthetic(n=n, d=d, n_batches=(4,), seed=n + d)
    got = _dev_kmeans(x, n_clusters, 5)
    z = x / np.linalg.norm(x, axis=1, keepdims=True)
    want, _ = oh.kmeans_start(z, n_clusters, hm.spawn_random_state(np.random.default_rng(5)))
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)
    if (n, n_clusters, d) == (20_000, 100, 50):
        from sklearn.cluster import KMeans

        sk = KMeans(n_clusters, random_state=hm.spawn_random_state(np.random.default_rng(5)), max_iter=25).fit(z)
        np.testing.assert_allclose(got, sk.cluster_centers_, rtol=0, atol=1e-10)


def test_kmeans_start_with_fewer_distinct_points_than_clusters():
    """k-means++ at a potential of exactly 0, then Lloyd with 24 clusters that stay empty: sklearn leaves them
    unrelocated (every point sits on its centre) and places them at the largest cluster's centre."""
    from sklearn.cluster import KMeans
    from sklearn.exceptions import ConvergenceWarning

    x = repeated_points()
    assert len(np.unique(x, axis=0)) == 40
    got = _dev_kmeans(x, 64, 2)
    with pytest.warns(ConvergenceWarning, match="distinct clusters"):
        sk = KMeans(64, random_state=hm.spawn_random_state(np.random.default_rng(2)), max_iter=25).fit(x)
    want, _ = oh.kmeans_start(x, 64, hm.spawn_random_state(np.random.default_rng(2)))
    np.testing.assert_array_equal(want, sk.cluster_centers_)
    np.testing.assert_allclose(got, sk.cluster_centers_, rtol=0, atol=1e-12)


def _f32_start_case(name):
    if name == "pbmc68k":
        x, obs, _ = pbmc68k()
        return x.astype(np.float32), obs, "bulk_labels"
    x, obs, _ = synthetic(n=12_000, d=50, n_batches=(5,))
    return x.astype(np.float32), obs, "key0"


@pytest.mark.parametrize("name", ["pbmc68k", "default_k"])
def test_public_float32_call_against_scanpys_float32_start(name):
    """scanpy runs sklearn's KMeans on the float32 rows, in float32; the device runs its k-means start in float64 on
    the float32 rows.  The public float32 call against the oracle started from sklearn's float32 centres, with the
    float32 bar of the oracle tests.  Printed next to it: the same device fit from sklearn's centres, which separates
    the start's share of the error from the float32 schedule's."""
    from sklearn.cluster import KMeans

    from scanpy_b200 import pp

    x, obs, key = _f32_start_case(name)
    adata = MiniAnnData(np.zeros((len(x), 1), dtype=np.float32), obs=obs, obsm={"X_pca": x})
    pp.harmony_integrate(adata, key, dtype=np.float32, rng=0)
    got = adata.obsm["X_pca_harmony"]
    assert got.dtype == np.float32
    z = x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), np.float32(1e-12))
    k = max(int(min(100, len(x) / 30)), 2)
    sk = KMeans(k, random_state=hm.spawn_random_state(np.random.default_rng(0)), max_iter=25).fit(z).cluster_centers_
    assert sk.dtype == np.float32
    codes, n_levels = hm.get_batch_codes(obs, key)
    want, wits = oh.harmony(x.astype(np.float64), codes, n_levels, centers=sk, rng=0)
    scale = np.abs(x).max()
    err = np.abs(got - want).max() / scale
    from_sk, its = device_fit(x, codes, n_levels, centers=sk, rng=0, **full_args())
    err_sk = np.abs(from_sk - want).max() / scale
    centres = np.abs(_dev_kmeans(x, k, 0) - sk).max()
    print(f"[{name}] float32 public call vs oracle from sklearn float32 centres: {err:.2e} x max|x|; the device fit "
          f"from those centres: {err_sk:.2e} (iterations {its} vs {wits}); device start vs sklearn's: {centres:.2e}")
    assert err <= 1e-4, err


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

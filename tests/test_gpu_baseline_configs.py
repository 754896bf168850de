"""Parity ON the BASELINE.json configurations (need an H100: `pytest -m gpu`).

configs[0]  pbmc3k-shaped 2700 x 1838 CSR (pbmc3k itself needs a download; SURVEY.md 8d prescribes the generator at
            that shape, K = 8, plus the in-tree pbmc68k fixture for real data - see test_gpu_parity.py)
configs[1]  synthetic 100k x 2000, n_pcs 50, k 15
configs[2]  (1.3M x 2000) is checked inside bench.py after the timed region (stages.parity) - it is too large for a
            unit test's oracle.
Bars (BASELINE.json north_star): X_pca within 1e-4 relative up to sign, identical kNN index sets, Leiden ARI >= 0.99.
Oracles: PCA - float64 covariance-eigh ground truth (oracle.pca.pca_gram_f64) AND the reference's live float32 call
(sklearn ARPACK, src/scanpy/preprocessing/_pca/__init__.py:282-291); kNN - float64 brute force with exactly-rounded
distances (oracle.knn.knn_exact_f64), so "identical" means identical; Leiden - the sequential oracle.
Reference tests mirrored: tests/test_pca.py:225-233, tests/test_neighbors.py:151-192.
"""
import numpy as np
import pytest
from sklearn.metrics import adjusted_rand_score

import scanpy_b200 as sb
from oracle import knn as oknn, leiden as old, pca as opca
from scanpy_b200._synth import synth_scipy

pytestmark = pytest.mark.gpu


def _rel_err(a, b):
    a = opca.align_signs(np.asarray(a, np.float64), b)
    return np.linalg.norm(a - b, axis=0) / np.linalg.norm(b, axis=0)


def _run_pipeline(x, n_pcs, k):
    ad = sb.MiniAnnData(x)
    sb.pp.pca(ad, n_comps=n_pcs)
    sb.pp.neighbors(ad, n_neighbors=k)
    sb.tl.leiden(ad, flavor="igraph", n_iterations=-1)
    return ad


def _check_pca(ad, x, n_pcs, *, label):
    truth = opca.pca_gram_f64(x, n_pcs)
    ref32 = opca.pca_arpack(x, n_pcs)                       # the reference's own call, float32 ARPACK
    e64 = _rel_err(ad.obsm["X_pca"], truth["X_pca"])
    noise = _rel_err(ref32["X_pca"], truth["X_pca"])        # the reference's own float32 error per component
    e32 = _rel_err(ad.obsm["X_pca"], ref32["X_pca"].astype(np.float64))
    gaps = truth["gaps"]
    literal = int((e32 < 1e-4).sum())
    print(f"\n[{label}] X_pca rel. error vs fp64 truth: max {e64.max():.2e}; vs the live fp32 ARPACK call: max {e32.max():.2e} "
          f"({literal}/{n_pcs} components inside the literal 1e-4; the reference's own fp32 error vs truth: max {noise.max():.2e}); "
          f"relative spectrum gaps min {gaps.min():.2e} median {np.median(gaps):.2e}")
    # the bar, against ground truth, on EVERY component
    assert e64.max() < 1e-4, (e64.max(), gaps.min())
    # against the reference's float32 run: every component within the reference's own distance from the truth
    assert (e32 < np.maximum(1e-4, 2.0 * noise + 1e-5)).all(), (e32.max(), noise.max())
    np.testing.assert_allclose(ad.uns["pca"]["variance"], truth["variance"], rtol=1e-5)
    np.testing.assert_allclose(ad.uns["pca"]["variance_ratio"], truth["variance_ratio"], rtol=1e-5)
    return truth


def _knn_lists(ad, k):
    n = ad.obsm["X_pca"].shape[0]
    d = ad.obsp["distances"]
    idx = np.hstack([np.arange(n)[:, None], d.indices.reshape(n, k - 1)])
    return idx


def test_config_a_pbmc3k_shape_full_pipeline():
    n, g, n_pcs, k = 2700, 1838, 50, 15
    x, lab = synth_scipy(n, g, n_clusters=8, r=64)
    ad = _run_pipeline(x, n_pcs, k)
    _check_pca(ad, x, n_pcs, label="config A 2700x1838")
    # identical kNN index sets, every row, against float64 brute force on the embedding the neighbours were built from
    xp = ad.obsm["X_pca"]
    oi, od = oknn.knn_exact_f64(xp, np.arange(n), k)
    bad = oknn.exact_set_mismatches(_knn_lists(ad, k), oi, od, k)
    assert bad.sum() == 0, f"{bad.sum()} rows with a wrong neighbour set"
    np.testing.assert_allclose(ad.obsp["distances"].data.reshape(n, k - 1), np.sqrt(od[:, 1:k]), rtol=1e-6, atol=1e-7)
    # Leiden vs the sequential oracle on the same connectivities
    got = ad.obs["leiden"].to_numpy().astype(int)
    mo, qo, _ = old.leiden(ad.obsp["connectivities"], seed=0)
    ari = adjusted_rand_score(mo, got)
    print(f"[config A] Leiden ARI vs oracle {ari:.4f}, vs planted {adjusted_rand_score(lab, got):.4f}; "
          f"Q {ad.uns['leiden']['modularity']:.5f} (oracle {qo:.5f}); {got.max() + 1} communities (oracle {mo.max() + 1})")
    assert ari >= 0.99
    assert ad.uns["leiden"]["modularity"] >= qo - 1e-3


def test_config_b_100k_full_pipeline():
    n, g, n_pcs, k = 100_000, 2000, 50, 15
    x, lab = synth_scipy(n, g)
    ad = _run_pipeline(x, n_pcs, k)
    _check_pca(ad, x, n_pcs, label="config B 100k x 2000")
    xp = ad.obsm["X_pca"]
    rows = np.random.RandomState(0).choice(n, 5000, replace=False)
    oi, od = oknn.knn_exact_f64(xp, rows, k)
    bad = oknn.exact_set_mismatches(_knn_lists(ad, k)[rows], oi, od, k)
    assert bad.sum() == 0, f"{bad.sum()} of 5000 sampled rows with a wrong neighbour set"
    np.testing.assert_allclose(ad.obsp["distances"].data.reshape(n, k - 1)[rows], np.sqrt(od[:, 1:k]), rtol=1e-6, atol=1e-7)
    got = ad.obs["leiden"].to_numpy().astype(int)
    mo, qo, _ = old.leiden(ad.obsp["connectivities"], seed=0)
    ari = adjusted_rand_score(mo, got)
    print(f"[config B] Leiden ARI vs oracle {ari:.4f}, vs planted {adjusted_rand_score(lab, got):.4f}; "
          f"Q {ad.uns['leiden']['modularity']:.5f} (oracle {qo:.5f}); {got.max() + 1} communities (oracle {mo.max() + 1})")
    assert ari >= 0.99
    assert ad.uns["leiden"]["modularity"] >= qo - 1e-3

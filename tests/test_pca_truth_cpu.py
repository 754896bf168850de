"""The float64 PCA truth and the gap-aware comparator of oracle/pca.py (no GPU): the comparator accepts the truth against
itself under any signs and any rotation inside a degenerate eigenvalue cluster, and rejects a 1e-3 perturbation of an
isolated component, a swap of two well-separated components, and non-zero output on null components."""
import numpy as np
import pytest
from scipy import sparse

from oracle import pca as opca


def _planted(n=400, g=60, spectrum=(10.0, 5.0, 5.0, 5.0, 3.0, 2.0, 1.5, 1.2, 1.0), seed=0, offset=1.0):
    """Exactly known singular values: X = mu + U diag(s) V^T with U orthonormal and orthogonal to the ones vector."""
    rs = np.random.RandomState(seed)
    r = len(spectrum)
    u = rs.standard_normal((n, r))
    u -= u.mean(axis=0)
    u, _ = np.linalg.qr(u)
    v, _ = np.linalg.qr(rs.standard_normal((g, r)))
    return offset + u @ np.diag(spectrum) @ v.T


def _as_got(truth, k, signs=None, rot=None):
    comp = truth["components"][:k].copy()
    xp = opca.project(truth, np.arange(k))
    if rot is not None:
        a, b, q = rot
        comp[a:b] = q.T @ comp[a:b]
        xp[:, a:b] = xp[:, a:b] @ q
    if signs is not None:
        comp *= signs[:, None]
        xp *= signs[None, :]
    return dict(X_pca=xp, components=comp, variance=truth["variance"][:k].copy(),
                variance_ratio=truth["variance_ratio"][:k].copy(), mean=truth["mean"].copy())


@pytest.mark.parametrize("dense", [True, False])
def test_truth_recovers_a_planted_spectrum(dense):
    x = _planted()
    t = opca.pca_full_f64(sparse.csr_matrix(x), dense=dense)
    s = np.array([10.0, 5.0, 5.0, 5.0, 3.0, 2.0, 1.5, 1.2, 1.0])
    np.testing.assert_allclose(t["spectrum"][:9], s ** 2, rtol=1e-12)
    assert (np.abs(t["spectrum"][9:]) <= 1e-12 * t["spectrum"][0]).all()   # rank 9: the rest is null
    np.testing.assert_allclose(t["variance"][:9], s ** 2 / (x.shape[0] - 1), rtol=1e-12)
    np.testing.assert_allclose(t["mean"], x.mean(axis=0), rtol=1e-12)
    np.testing.assert_allclose(t["total_var"], x.var(axis=0, ddof=1).sum(), rtol=1e-12)
    ref = opca.pca_exact_f64(x, 5)
    np.testing.assert_allclose(t["components"][[0, 4]], ref["components"][[0, 4]], atol=1e-10)
    np.testing.assert_allclose(opca.project(t, [0, 4]), ref["X_pca"][:, [0, 4]], atol=1e-9)


def test_truncated_truth_matches_the_reference_call():
    x = sparse.csr_matrix(np.abs(_planted(300, 40, offset=0.5)))
    t = opca.pca_full_f64(x, zero_center=False)
    ref = opca.truncated_svd_arpack(x, 6)
    np.testing.assert_allclose(t["variance"][:6], ref["variance"], rtol=1e-9)
    np.testing.assert_allclose(t["variance_ratio"][:6], ref["variance_ratio"], rtol=1e-9)
    np.testing.assert_allclose(np.abs(opca.project(t, np.arange(6))), np.abs(ref["X_pca"]), atol=1e-9)


def test_svd_flip_tie_takes_the_first_index():
    vt = np.array([[-0.5, 0.5, 0.5, -0.5], [0.0, 0.6, -0.6, 0.0], [0.0, 0.0, 0.0, 0.0]])
    np.testing.assert_array_equal(opca.svd_flip_rows(vt), [-1.0, 1.0, 1.0])


def test_comparator_accepts_the_truth_under_signs_and_cluster_rotations():
    x = sparse.csr_matrix(_planted())
    t = opca.pca_full_f64(x)
    k = 7
    rep = opca.compare_pca(_as_got(t, k), t, k)
    assert rep["ok"], rep["failures"]
    assert rep["clusters"] == [(0, 0), (1, 3), (4, 4), (5, 5), (6, 6)]
    rs = np.random.RandomState(1)
    signs = rs.choice([-1.0, 1.0], k)
    signs[0] = -1.0
    rep = opca.compare_pca(_as_got(t, k, signs=signs), t, k, check_signs=False)
    assert rep["ok"], rep["failures"]
    # the same flipped output breaks svd_flip's sign rule
    rep = opca.compare_pca(_as_got(t, k, signs=signs), t, k)
    assert not rep["ok"] and any("sign rule" in f for f in rep["failures"])
    q, _ = np.linalg.qr(rs.standard_normal((3, 3)))
    got = _as_got(t, k, rot=(1, 4, q))
    got["components"][1:4] *= opca.svd_flip_rows(got["components"][1:4])[:, None]   # a valid output has flipped signs
    rep = opca.compare_pca(got, t, k)
    assert rep["ok"], rep["failures"]
    # a cluster cut by k (components 1..3, k = 3) is compared with its full truth subspace
    got = _as_got(t, 3, rot=(1, 3, np.linalg.qr(rs.standard_normal((2, 2)))[0]))
    rep = opca.compare_pca(got, t, 3, check_signs=False)
    assert rep["ok"], rep["failures"]
    assert rep["clusters"] == [(0, 0), (1, 3)]


def test_comparator_rejects_a_small_perturbation_and_a_swap():
    x = sparse.csr_matrix(_planted())
    t = opca.pca_full_f64(x)
    k = 7
    # 1e-3 of the next direction mixed into the isolated component 4
    got = _as_got(t, k)
    v = t["components"][4] + 1e-3 * t["components"][5]
    v /= np.linalg.norm(v)
    got["components"][4] = v
    got["X_pca"][:, 4] = opca.project(dict(t, components=v[None]), [0])[:, 0]
    rep = opca.compare_pca(got, t, k)
    assert not rep["ok"] and any("component 4" in f for f in rep["failures"]), rep["summary"]
    assert 5e-4 < rep["x_err"][4] < 2e-3
    # the same perturbation inside the degenerate cluster is a rotation of it, and fine
    got = _as_got(t, k)
    c = np.cos(1e-3); s = np.sin(1e-3)
    got["components"][1:3] = np.array([[c, s], [-s, c]]) @ got["components"][1:3]
    rep = opca.compare_pca(got, t, k, check_signs=False)
    assert rep["ok"], rep["failures"]
    # two well-separated components swapped
    got = _as_got(t, k)
    got["components"][[4, 5]] = got["components"][[5, 4]]
    got["X_pca"][:, [4, 5]] = got["X_pca"][:, [5, 4]]
    rep = opca.compare_pca(got, t, k)
    assert not rep["ok"] and any("component 4" in f for f in rep["failures"])
    # a variance off by 2e-5
    got = _as_got(t, k)
    got["variance"][5] *= 1 + 2e-5
    assert not opca.compare_pca(got, t, k)["ok"]


def test_comparator_null_components():
    x = sparse.csr_matrix(_planted(n=200, g=40, spectrum=(4.0, 2.0, 1.0)))
    t = opca.pca_full_f64(x)
    k = 6                                             # components 3..5 are null (rank 3)
    got = _as_got(t, k)
    assert opca.compare_pca(got, t, k)["null"] == [3, 4, 5]
    rs = np.random.RandomState(2)
    got["X_pca"][:, 3:] = 1e-7 * rs.standard_normal((200, 3))   # rounding-level projections are null
    got["variance"][3:] = [1e-12, 0.0, 0.0]
    got["components"][3:] *= opca.svd_flip_rows(got["components"][3:])[:, None]
    rep = opca.compare_pca(got, t, k)
    assert rep["ok"], rep["failures"]
    bad = dict(got, X_pca=got["X_pca"].copy())
    bad["X_pca"][:, 4] = 1e-3 * bad["X_pca"][:, 0]
    assert not opca.compare_pca(bad, t, k)["ok"]
    bad = dict(got, variance=got["variance"].copy())
    bad["variance"][5] = 1e-6 * t["variance"][0]
    assert not opca.compare_pca(bad, t, k)["ok"]

"""PCA oracle = the reference's arithmetic (test infrastructure only; see oracle/__init__.py).

scanpy's `pca()` for a scipy CSR input with zero_center=True and svd_solver in {None,'arpack'}
does exactly this (src/scanpy/preprocessing/_pca/__init__.py:282-291,308,338-363):

    pca_ = sklearn.decomposition.PCA(n_components=n_comps, svd_solver='arpack', random_state=0)
    x_pca = pca_.fit_transform(x);  x_pca = x_pca.astype('float32')

and reads `components_`, `explained_variance_`, `explained_variance_ratio_`.
`covariance_eigh` restates src/scanpy/preprocessing/_pca/_dask.py:24-132,143-213
(Gram -> cov with bias -> eigh -> project), in float64.
"""
from __future__ import annotations

import numpy as np


def pca_arpack(x, n_comps: int, *, random_state: int = 0, dtype="float32"):
    """Return dict(X_pca, components, variance, variance_ratio, mean) as scanpy would store them."""
    from sklearn.decomposition import PCA

    pca_ = PCA(n_components=n_comps, svd_solver="arpack", random_state=random_state)
    x_pca = pca_.fit_transform(x)
    if x_pca.dtype != np.dtype(dtype):
        x_pca = x_pca.astype(dtype)
    return dict(
        X_pca=np.ascontiguousarray(x_pca),
        components=pca_.components_,
        variance=pca_.explained_variance_,
        variance_ratio=pca_.explained_variance_ratio_,
        mean=np.asarray(pca_.mean_).ravel(),
        singular_values=pca_.singular_values_,
    )


def pca_exact_f64(x, n_comps: int):
    """Dense float64 PCA by eigh of the covariance: the 'true' answer both the reference's
    float32 ARPACK run and our CUDA path approximate (used to calibrate tolerances)."""
    import scipy.linalg as sla
    from scipy import sparse

    xd = x.toarray().astype(np.float64) if sparse.issparse(x) else np.asarray(x, np.float64)
    n = xd.shape[0]
    mu = xd.mean(axis=0)
    xc = xd - mu
    cov = xc.T @ xc / (n - 1)
    g = cov.shape[0]
    w, v = sla.eigh(cov, subset_by_index=[g - n_comps, g - 1])
    w, v = w[::-1], v[:, ::-1]
    vt = v.T.copy()
    # svd_flip(u_based_decision=False): largest-|.| entry of each row of Vt positive
    # (site-packages/sklearn/utils/extmath.py:974-981)
    sign = np.sign(vt[np.arange(n_comps), np.argmax(np.abs(vt), axis=1)])
    vt *= sign[:, None]
    total_var = xc.var(axis=0, ddof=1).sum()
    return dict(X_pca=xc @ vt.T, components=vt, variance=w, variance_ratio=w / total_var, mean=mu)


def align_signs(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Flip columns of `a` so that each correlates positively with the same column of `b`."""
    s = np.sign(np.einsum("ij,ij->j", a, b))
    s[s == 0] = 1
    return a * s


def gram_f64_blocked(x, *, block_rows: int = 16384):
    """(G = X^T X, column sums), both in float64, for a scipy CSR matrix, by dense row blocks through BLAS (a sparse-sparse product
    costs sum_r nnz_r^2 hashed updates on one core; densified syrk blocks use every core).  This is the host-side
    restatement of the reference's `csr_gram_dense` (src/scanpy/preprocessing/_pca/_kernels.py:14-58)."""
    n, g = x.shape
    gram = np.zeros((g, g), np.float64)
    colsum = np.zeros(g, np.float64)
    for r0 in range(0, n, block_rows):
        blk = x[r0:r0 + block_rows].toarray().astype(np.float64, copy=False)
        gram += blk.T @ blk
        colsum += blk.sum(axis=0)
    return gram, colsum


def pca_gram_f64(x, n_comps: int, *, rows=None):
    """Float64 ground truth through the covariance_eigh route (src/scanpy/preprocessing/_pca/_dask.py:143-213
    restated with ddof=1 like sklearn's explained_variance_): Gram -> covariance -> LAPACK eigh -> projection.
    Never densifies more than a row block, so it also serves the 100k and 1.3M configurations.
    `rows`: project only these rows (X_pca of a sample); None = all rows."""
    import scipy.linalg as sla

    n, g = x.shape
    gram, colsum = gram_f64_blocked(x)
    mu = colsum / n
    cov = (gram - n * np.outer(mu, mu)) / (n - 1)
    w, v = sla.eigh(cov, subset_by_index=[g - n_comps, g - 1])
    w, v = w[::-1], v[:, ::-1]
    vt = v.T.copy()
    sign = np.sign(vt[np.arange(n_comps), np.argmax(np.abs(vt), axis=1)])
    vt *= sign[:, None]
    xs = x if rows is None else x[np.asarray(rows)]
    x_pca = np.asarray(xs.astype(np.float64) @ vt.T) - mu @ vt.T
    total_var = float(np.trace(cov))
    # relative spectrum gaps (sigma_j - sigma_{j+1}) / sigma_j of the singular values, one more than n_comps
    w_all = sla.eigh(cov, subset_by_index=[g - n_comps - 1, g - 1], eigvals_only=True)[::-1]
    s = np.sqrt(np.maximum(w_all, 0.0))
    gaps = (s[:-1] - s[1:]) / s[:-1]
    return dict(X_pca=x_pca, components=vt, variance=w, variance_ratio=w / total_var, mean=mu, gaps=gaps)


def svd_flip_rows(vt: np.ndarray) -> np.ndarray:
    """Signs of svd_flip(u_based_decision=False) for the rows of `vt`: the largest-|.| entry of each row positive, the
    first such entry when the maximum is tied (np.argmax); an all-zero row keeps sign +1."""
    s = np.sign(vt[np.arange(vt.shape[0]), np.argmax(np.abs(vt), axis=1)])
    s[s == 0] = 1.0
    return s


def pca_full_f64(x, *, zero_center: bool = True, dense: bool | None = None):
    """Float64 truth with the FULL spectrum, so the rank of the data and its null components are known.

    zero_center=True: sklearn PCA (explained variance S^2/(n-1), ratio against the ddof-1 total variance).
    zero_center=False: sklearn TruncatedSVD (explained variance np.var(X V) with ddof 0, ratio against sum_g var_g ddof 0).
    `dense` (default: n*g <= 4e6) takes a dense SVD of the (centred) matrix; otherwise the covariance (or X^T X) is built by
    row blocks and diagonalised with LAPACK eigh, which resolves null eigenvalues to ~1e-16 of the largest.  Returns
    components [m x g] with svd_flip signs, `spectrum` [m] (eigenvalues of Xc^T Xc, descending), variance and
    variance_ratio [m], mean [g], `var_scale` (the variance unit the null bars refer to) and what `project` needs to form
    X_pca columns on demand.  m = min(n, g) for the SVD, g for eigh."""
    import scipy.linalg as sla
    from scipy import sparse

    n, g = x.shape
    if dense is None:
        dense = n * g <= 4_000_000
    if dense:
        xd = x.toarray().astype(np.float64) if sparse.issparse(x) else np.asarray(x, np.float64)
        mu = xd.mean(axis=0)
        shift = mu if zero_center else np.zeros(g)
        _, s, vt = np.linalg.svd(xd - shift, full_matrices=False)
        spectrum = s * s
        total_var = float(xd.var(axis=0, ddof=1 if zero_center else 0).sum())
    else:
        gram, colsum = gram_f64_blocked(x)
        mu = colsum / n
        shift = mu if zero_center else np.zeros(g)
        cov = gram - n * np.outer(shift, shift)
        w, v = sla.eigh(cov)
        spectrum, vt = w[::-1].copy(), v[:, ::-1].T.copy()
        diag = np.diag(gram) - n * mu * mu
        total_var = float(diag.sum() / ((n - 1) if zero_center else n))
    vt = vt * svd_flip_rows(vt)[:, None]
    if zero_center:
        variance = np.maximum(spectrum, 0.0) / (n - 1)
        var_scale = spectrum[0] / (n - 1)
    else:
        variance = np.maximum(spectrum, 0.0) / n - (mu @ vt.T) ** 2
        var_scale = spectrum[0] / n
    return dict(components=vt, spectrum=spectrum, variance=variance, variance_ratio=variance / total_var, mean=mu,
                var_scale=var_scale, total_var=total_var, x=x, shift=shift)


def project(truth, cols) -> np.ndarray:
    """X_pca columns `cols` of a `pca_full_f64` truth, in float64: X V - 1 (shift^T V)."""
    v = truth["components"][np.asarray(cols)].T
    x = truth["x"]
    xv = x.astype(np.float64) @ v if hasattr(x, "toarray") else np.asarray(x, np.float64) @ v
    return np.asarray(xv) - truth["shift"] @ v


def compare_pca(got, truth, k: int, *, gap: float = 1e-3, null: float = 1e-12, x_rtol: float = 1e-4,
                comp_atol: float = 2e-4, angle: float = 1e-4, null_x: float = 1e-5, null_var: float = 1e-9,
                var_rtol: float = 1e-5, check_signs: bool = True) -> dict:
    """Gap-aware comparison of a PCA result `got` (X_pca [n x k], components [k x g], variance, variance_ratio[, mean])
    with a `pca_full_f64` truth.

    - null components (truth eigenvalue <= null * the largest): |X_pca[:, j]| <= null_x * max|X_pca[:, 0]| and
      variance_j <= null_var * var_scale; their directions are not compared.
    - the other components fall into clusters: runs of eigenvalues whose relative gap (lam_j - lam_j+1) / lam_j is below
      `gap`.  A cluster may run past k; it is then compared with all of its truth directions.
    - an isolated component (a cluster of one) matches per component, up to one sign shared by its X_pca column and its
      component: X_pca relative error < x_rtol, component |.| error <= comp_atol.
    - a cluster is compared as a subspace: the largest principal-angle sine between the returned components and the
      truth's cluster directions must be < angle.
    - variance and variance_ratio to var_rtol on the non-null components; the mean (if returned) to 1e-6.
    - check_signs: every returned component has its largest-|.| entry (first one on ties) >= 0, > 0 unless null.
    Returns a report: per-component errors, cluster sines, null ratios, the worst value of each check next to its bar
    (`summary`) and the list of `failures` (empty = the bar is met)."""
    lam = np.asarray(truth["spectrum"], np.float64)
    m = lam.shape[0]
    lam0 = lam[0]
    is_null = lam <= null * lam0
    rel_gap = np.full(m, np.inf)
    nz = ~is_null[:-1]
    rel_gap[:-1][nz] = (lam[:-1][nz] - lam[1:][nz]) / lam[:-1][nz]
    xp = np.asarray(got["X_pca"], np.float64)
    comp = np.asarray(got["components"], np.float64)
    var = np.asarray(got["variance"], np.float64)
    ratio = np.asarray(got["variance_ratio"], np.float64)
    tvt = truth["components"]
    fail, rep = [], dict(x_err={}, comp_err={}, cluster_sine={}, null_x={}, null_var={}, clusters=[], null=[])
    # clusters of the non-null components < k (each may extend past k)
    j = 0
    while j < k:
        if is_null[j]:
            rep["null"].append(j)
            j += 1
            continue
        e = j
        while e + 1 < m and not is_null[e + 1] and rel_gap[e] < gap:
            e += 1
        rep["clusters"].append((j, e))
        j = e + 1
    scale0 = np.abs(xp[:, 0]).max() if xp.size else 0.0
    for a, b in rep["clusters"]:
        if a == b:
            t = project(truth, [a])[:, 0]
            c = comp[a]
            s = 1.0 if c @ tvt[a] >= 0 else -1.0
            ex = float(np.linalg.norm(s * xp[:, a] - t) / max(np.linalg.norm(t), 1e-300))
            ec = float(np.abs(s * c - tvt[a]).max())
            rep["x_err"][a], rep["comp_err"][a] = ex, ec
            if not ex < x_rtol:
                fail.append(f"component {a}: X_pca relative error {ex:.2e} >= {x_rtol:g}")
            if not ec <= comp_atol:
                fail.append(f"component {a}: loading error {ec:.2e} > {comp_atol:g}")
        else:
            hi = min(b, k - 1)
            q, _ = np.linalg.qr(comp[a:hi + 1].T)
            t = tvt[a:b + 1]
            resid = q - t.T @ (t @ q)
            sine = float(np.linalg.svd(resid, compute_uv=False).max()) if resid.size else 0.0
            rep["cluster_sine"][(a, b)] = sine
            if not sine < angle:
                fail.append(f"cluster {a}..{b}: principal-angle sine {sine:.2e} >= {angle:g}")
    for jn in rep["null"]:
        rx = float(np.abs(xp[:, jn]).max() / scale0) if scale0 > 0 else float(np.abs(xp[:, jn]).max())
        rv = float(var[jn] / truth["var_scale"])
        rep["null_x"][jn], rep["null_var"][jn] = rx, rv
        if not rx <= null_x:
            fail.append(f"null component {jn}: max|X_pca| / max|X_pca[:, 0]| = {rx:.2e} > {null_x:g}")
        if not rv <= null_var:
            fail.append(f"null component {jn}: variance / largest = {rv:.2e} > {null_var:g}")
    keep = np.array([j for j in range(k) if not is_null[j]], dtype=int)
    var_err = ratio_err = 0.0
    if keep.size:
        tv, tr = truth["variance"][keep], truth["variance_ratio"][keep]
        var_err = float((np.abs(var[keep] - tv) / np.abs(tv)).max())
        ratio_err = float((np.abs(ratio[keep] - tr) / np.abs(tr)).max())
        if not var_err <= var_rtol:
            fail.append(f"variance relative error {var_err:.2e} > {var_rtol:g}")
        if not ratio_err <= var_rtol:
            fail.append(f"variance_ratio relative error {ratio_err:.2e} > {var_rtol:g}")
    mean_err = 0.0
    if got.get("mean") is not None:
        mu = truth["mean"]
        mean_err = float((np.abs(np.asarray(got["mean"], np.float64) - mu) / (np.abs(mu) + 1e-3)).max())
        if not mean_err <= 1e-6:
            fail.append(f"mean error {mean_err:.2e} > 1e-06")
    if check_signs:
        lead = comp[np.arange(k), np.argmax(np.abs(comp), axis=1)]
        bad = [j for j in range(k) if lead[j] < 0 or (lead[j] == 0 and not is_null[j])]
        if bad:
            fail.append(f"svd_flip sign rule broken on components {bad[:8]}")
    worst = lambda d: max(d.values()) if d else 0.0  # noqa: E731
    rep.update(failures=fail, ok=not fail, var_err=var_err, ratio_err=ratio_err, mean_err=mean_err,
               min_gap=float(rel_gap[:k].min()) if k else np.inf)
    rep["summary"] = (f"X_pca {worst(rep['x_err']):.2e} (bar {x_rtol:g}), loadings {worst(rep['comp_err']):.2e} "
                      f"(bar {comp_atol:g}), cluster sine {worst(rep['cluster_sine']):.2e} (bar {angle:g}, "
                      f"{sum(1 for a, b in rep['clusters'] if b > a)} clusters), null |X_pca| {worst(rep['null_x']):.2e} "
                      f"(bar {null_x:g}) var {worst(rep['null_var']):.2e} (bar {null_var:g}, {len(rep['null'])} null), "
                      f"variance {var_err:.2e} ratio {ratio_err:.2e} (bar {var_rtol:g}), mean {mean_err:.2e}")
    return rep


def truncated_svd_arpack(x, n_comps: int, dtype="float64"):
    """The reference's `zero_center=False` call (src/scanpy/preprocessing/_pca/__init__.py:331-336) with the exact solver:
    sklearn TruncatedSVD(algorithm='arpack') -> dict(X_pca, components, variance, variance_ratio, singular_values)."""
    from sklearn.decomposition import TruncatedSVD

    t = TruncatedSVD(n_components=n_comps, algorithm="arpack", random_state=0)
    xp = t.fit_transform(x.astype(dtype))
    return dict(X_pca=xp, components=t.components_, variance=t.explained_variance_, variance_ratio=t.explained_variance_ratio_,
                singular_values=t.singular_values_)

"""Harmony oracle (test infrastructure only): a numpy fp64 restatement of the reference's
src/scanpy/preprocessing/_harmony/core.py, following its schedule step by step.

`harmony` starts from given k-means centres (sklearn's `cluster_centers_`) instead of running KMeans, and draws the
per-clustering-iteration permutations from `np.random.default_rng(rng)` exactly as the reference does: its k-means start
spawns a child stream, which does not advance the parent.  It returns the corrected matrix and, per outer iteration, the
number of clustering iterations run.  Every cell's o / e update is applied cell by cell, as `np.add.at` does.

`kmeans_start` restates sklearn's `KMeans(n_clusters, random_state=rs, max_iter=25).fit(x).cluster_centers_`
(k-means++ with 2 + int(ln K) local trials, then Lloyd with the tolerance mean(var) * 1e-4 and strict convergence).
"""
from __future__ import annotations

import numpy as np

SUPPRESS_PENALTY = 1e30


# ------------------------------------------------------------------------------------------ k-means start
def _sq_dists(c: np.ndarray, x: np.ndarray, xx: np.ndarray) -> np.ndarray:
    """||c - x_i||² as xx + cc - 2 x·c, clipped at 0 (sklearn's expansion)."""
    d = xx - 2.0 * (x @ c) + c @ c
    return np.maximum(d, 0.0)


def kmeans_start(x: np.ndarray, n_clusters: int, random_state: np.random.RandomState, max_iter: int = 25):
    """-> (cluster centres [K x d], Lloyd iterations)."""
    x = np.asarray(x, dtype=np.float64)
    n, d = x.shape
    tol = np.mean(np.var(x, axis=0)) * 1e-4
    mean = x.mean(axis=0)
    xc = x - mean
    xx = (xc * xc).sum(axis=1)

    # greedy k-means++
    n_trials = 2 + int(np.log(n_clusters))
    w = np.ones(n)
    first = random_state.choice(n, p=w / w.sum())
    centers = np.empty((n_clusters, d))
    centers[0] = xc[first]
    closest = _sq_dists(centers[0], xc, xx)
    pot = closest.sum()
    for c in range(1, n_clusters):
        u = random_state.uniform(size=n_trials) * pot
        cand = np.minimum(np.searchsorted(np.cumsum(closest), u), n - 1)
        dist = np.stack([np.minimum(closest, _sq_dists(xc[i], xc, xx)) for i in cand])
        pots = dist.sum(axis=1)
        best = int(np.argmin(pots))
        pot, closest = pots[best], dist[best]
        centers[c] = xc[cand[best]]

    # Lloyd
    labels_old = np.full(n, -1)
    it = 0
    for it in range(1, max_iter + 1):
        labels = np.argmin((centers * centers).sum(axis=1)[None, :] - 2.0 * xc @ centers.T, axis=1)
        counts = np.bincount(labels, minlength=n_clusters).astype(np.float64)
        sums = np.zeros_like(centers)
        np.add.at(sums, labels, xc)
        empty = np.flatnonzero(counts == 0)
        dist = ((xc - centers[labels]) ** 2).sum(axis=1) if empty.size else None
        # sklearn: the points farthest from their centres start the empty clusters, unless every point sits on its
        # centre (fewer distinct points than clusters); an empty cluster's centre is then 0
        if empty.size and dist.max() > 0:
            far = np.argpartition(dist, -empty.size)[: -empty.size - 1 : -1]
            for k, i in zip(empty, far):
                sums[labels[i]] -= xc[i]
                sums[k] = xc[i]
                counts[k] = 1.0
                counts[labels[i]] -= 1.0
        avg = sums * (1.0 / np.maximum(counts, 1.0))[:, None]
        # sklearn's _average_centers: a cluster still empty takes the centre of the largest one as the loop over the
        # clusters leaves it, averaged when it comes earlier and still a sum when it comes later
        big = int(np.argmax(counts))
        later = (np.arange(len(counts)) > big)[:, None]
        new = np.where(counts[:, None] > 0, avg, np.where(later, avg[big], sums[big]))
        shift = ((new - centers) ** 2).sum()
        centers = new
        if np.array_equal(labels, labels_old) or shift <= tol:
            break
        labels_old = labels
    return centers + mean, it


# ------------------------------------------------------------------------------------------ host pieces
def batch_codes(columns: list[np.ndarray], n_levels: list[int]) -> np.ndarray:
    """Per-key local codes -> marginal codes (each key gets its own range)."""
    offs = np.concatenate([[0], np.cumsum(n_levels)[:-1]])
    return np.stack([np.asarray(c) + o for c, o in zip(columns, offs)], axis=1).astype(np.int64)


def theta_array(theta, n_levels) -> np.ndarray:
    levels = np.asarray(n_levels, dtype=np.int64)
    t = np.asarray(theta, dtype=np.float64)
    if t.ndim == 0:
        return np.full(int(levels.sum()), float(t))
    t = t.ravel()
    return np.repeat(t, levels) if t.size == levels.size else t


def lambda_kb(e, o, n_b, *, alpha, threshold, ridge_lambda, dynamic_lambda):
    if not dynamic_lambda:
        lam = np.full_like(e, ridge_lambda)
    else:
        lam = alpha * e
        if threshold is not None:
            safe = np.where(n_b > 0, n_b, 1.0)
            mask = (o / safe[:, None]) < threshold
            mask |= n_b[:, None] == 0
            lam[mask] = SUPPRESS_PENALTY
    lam[(o + lam) == 0] = SUPPRESS_PENALTY
    return lam


def _normalize(x):
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-12)


def _objective(y_norm, z, r, theta, sigma, o, e, stabilized):
    kme = np.sum(r * 2.0 * (1.0 - z @ y_norm.T))
    rn = r / np.clip(r.sum(axis=1, keepdims=True), 1e-12, None)
    ent = sigma * np.sum(rn * np.log(rn + 1e-12))
    ratio = np.log((o + e + 1) / (e + 1)) if stabilized else np.log((o + 1) / (e + 1))
    return kme + ent + sigma * np.sum(theta @ (o * ratio))


def _correct_fast(x, codes, n_batches, r, o, lam):
    z = x.copy()
    for k in range(r.shape[1]):
        o_k, r_k = o[:, k], r[:, k]
        factor = 1.0 / (o_k + lam[:, k])
        c_inv = 1.0 / (np.sum(o_k) - np.sum(factor * o_k**2))
        p = np.eye(n_batches + 1)
        p[0, 1:] = -factor * o_k
        pb = np.zeros((n_batches + 1, n_batches + 1))
        pb[0, 0] = c_inv
        pb[1:, 1:] = np.diag(factor)
        pb[1:, 0] = p[0, 1:] * c_inv
        phi = np.zeros((n_batches + 1, x.shape[1]))
        phi[0] = r_k @ x
        for b in range(n_batches):
            m = codes == b
            phi[b + 1] = r_k[m] @ x[m]
        w = (pb @ p) @ phi
        w[0] = 0
        z -= r_k[:, None] * w[codes + 1]
    return z


def _correct_multi(x, codes, n_batches, r, lam):
    """Each cluster's ridge fit from the dense one-hot design [1 | keys]: gram = Dᵀ diag(r_k) D + diag(0, λ)."""
    n, d = x.shape
    design = np.zeros((n, n_batches + 1))
    design[:, 0] = 1
    for j in range(codes.shape[1]):
        design[np.arange(n), codes[:, j] + 1] = 1
    z = x.copy()
    for k in range(r.shape[1]):
        r_k = r[:, k]
        active = lam[:, k] < SUPPRESS_PENALTY
        keep = np.concatenate(([True], active))
        dk = design[:, keep]
        gram = dk.T @ (r_k[:, None] * dk)
        gram[np.arange(1, keep.sum()), np.arange(1, keep.sum())] += lam[active, k]
        rhs = dk.T @ (r_k[:, None] * x)
        if np.linalg.matrix_rank(gram) < gram.shape[0]:
            wk = np.linalg.lstsq(gram, rhs, rcond=None)[0]
        else:
            wk = np.linalg.solve(gram, rhs)
        w = np.zeros((n_batches + 1, d))
        w[keep] = wk
        w[0] = 0
        z -= r_k[:, None] * (design @ w)
    return z


# ------------------------------------------------------------------------------------------ harmony
def harmony(x, codes, n_levels, *, centers, rng, theta=2.0, sigma=0.1, n_clusters=None, max_iter_harmony=10,
            max_iter_clustering=200, tol_harmony=1e-4, tol_clustering=1e-5, ridge_lambda=1.0, block_proportion=0.05,
            tau=0, stabilized_penalty=True, dynamic_lambda=True, alpha=0.2, batch_prune_threshold=1e-5):
    """-> (z_hat [n x d] float64, clustering iterations per outer iteration).  `codes`: n x keys marginal codes."""
    gen = np.random.default_rng(rng)
    x = np.asarray(x, dtype=np.float64)
    codes = np.asarray(codes).reshape(len(x), -1)
    n = len(x)
    n_batches = int(np.sum(n_levels))
    z = _normalize(x)
    n_b = np.bincount(codes.ravel(), minlength=n_batches).astype(np.float64)
    pr_b = (n_b / n)[:, None]
    th = theta_array(theta, n_levels)[None, :]
    k = n_clusters if n_clusters is not None else max(int(min(100, n / 30)), 2)
    if tau > 0:
        th = th * (1 - np.exp(-n_b / (k * tau)) ** 2)
    term = -2.0 / sigma

    y_norm = _normalize(np.asarray(centers, dtype=np.float64))
    r = np.exp(term * (1.0 - z @ y_norm.T))
    r /= np.maximum(r.sum(axis=1, keepdims=True), 1e-12)
    e = pr_b @ r.sum(axis=0)[None, :]
    o = np.zeros((n_batches, k))
    for c in codes.T:
        np.add.at(o, c, r)
    objectives = [_objective(y_norm, z, r, th, sigma, o, e, stabilized_penalty)]

    n_blocks = int(min(n, 1 // block_proportion))
    iterations = []
    z_hat = x
    for _ in range(max_iter_harmony):
        objs = []
        obj = None
        it = 0
        for it in range(1, max_iter_clustering + 1):
            y_norm = _normalize(r.T @ z)
            for idx in np.array_split(gen.permutation(n), n_blocks):
                cc = codes[idx]
                r_old = r[idx]
                for c in cc.T:
                    np.add.at(o, c, -r_old)
                e -= pr_b * r_old.sum(axis=0)
                if stabilized_penalty:
                    pen = th.T * (np.log(e + 1.0) - np.log(o + e + 1.0))
                else:
                    pen = th.T * (np.log(e + 1.0) - np.log(o + 1.0))
                lr = term * (1.0 - z[idx] @ y_norm.T) + pen[cc].sum(axis=1)
                lr -= lr.max(axis=1, keepdims=True)
                r_new = np.exp(lr)
                r_new /= np.maximum(r_new.sum(axis=1, keepdims=True), 1e-12)
                r[idx] = r_new
                for c in cc.T:
                    np.add.at(o, c, r_new)
                e += pr_b * r_new.sum(axis=0)
            objs.append(_objective(y_norm, z, r, th, sigma, o, e, stabilized_penalty))
            if len(objs) >= 4 and sum(objs[-4:-1]) - sum(objs[-3:]) < tol_clustering * abs(sum(objs[-4:-1])):
                obj = objs[-1]
                break
        iterations.append(it)
        if obj is not None:
            objectives.append(obj)
        lam = lambda_kb(e, o, n_b, alpha=alpha, threshold=batch_prune_threshold, ridge_lambda=ridge_lambda,
                        dynamic_lambda=dynamic_lambda)
        if codes.shape[1] > 1:
            z_hat = _correct_multi(x, codes, n_batches, r, lam)
        else:
            z_hat = _correct_fast(x, codes[:, 0], n_batches, r, o, lam)
        z = _normalize(z_hat)
        if len(objectives) >= 2 and (objectives[-2] - objectives[-1]) < tol_harmony * abs(objectives[-2]):
            break
    return z_hat, iterations

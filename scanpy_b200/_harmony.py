"""`sc.pp.harmony_integrate` on the device.

Reference: src/scanpy/preprocessing/_harmony/ (`harmony_integrate` and `Harmony.fit`).  The schedule is the
reference's, step for step; the per-cell passes run in CUDA (csrc/harmony.cu) and everything sized clusters x codes
stays on the host: the penalty inputs, `_compute_lambda_kb`, the fast-path `inv_mat`, the multi-key gram and solve,
the diversity term of the objective and both convergence tests.

* Random stream: `rng = np.random.default_rng(rng)`.  The k-means start uses a RandomState on
  `rng.bit_generator.spawn(1)` (the reference's `_legacy_random_state(rng, always_state=True)`), which does not advance
  `rng`; after that `rng` is consumed only by one `rng.permutation(n)` per clustering iteration.  The stream does not
  depend on the data, so the next permutation is drawn on the host while the device works on the current one.
* k-means start: sklearn's `KMeans(n_clusters, random_state=..., max_iter=25)` on the centred rows, restated: greedy
  k-means++ with 2 + int(ln K) local trials (the uniforms drawn on the host in sklearn's order; the D² sums, candidate
  searches and potentials on the device), then Lloyd with the tolerance mean(var) * 1e-4 and strict convergence.
* Blocks: `n_blocks = min(n, 1 // block_proportion)` (floor division on a float: 0.05 gives 19 blocks) and the cells
  split like `np.array_split`.  Per block: remove the block's r from o and e, compute the penalty, compute r, add r back.
* Objective: Σ r 2(1 - z·y) = 2 Σ r - 2 Σ_k y_k · (Rᵀ Z)_k, so the centroid pass Rᵀ[Z | 1] that starts the next
  clustering iteration also gives the k-means error of the last one; the entropy comes from per-cell terms the block
  step writes.
* Correction: the cells are grouped once by their code tuple; per group c the device sums S_c = Σ r_i and
  T_c = Σ r_i ⊗ x_i, and every gram entry and right-hand side of both the single-key fast path (with the clustering's
  own o) and the multi-key solve is a host sum over c.

`dtype` sets how Z, R and the output are stored and the per-element arithmetic; every sum over cells is fp64.
"""
from __future__ import annotations

import numpy as np
import pandas as pd

from . import _abi, _ops
from ._abi import check, ptr
from ._compat import logger, warn

SUPPRESS_PENALTY = 1e30
MAX_K = 128  # SB2_HARMONY_MAX_K
MAX_D = 128  # SB2_HARMONY_MAX_D
MAX_CODES = 128  # SB2_HARMONY_MAX_CODES
MAX_TUPLES = 65536  # SB2_HARMONY_MAX_TUPLES
MAX_TRIALS = 8  # SB2_HARMONY_MAX_TRIALS


# ------------------------------------------------------------------------------------------ host helpers
def get_batch_codes(obs, key) -> tuple[np.ndarray, np.ndarray]:
    """Each key's categories as its own range of marginal codes -> (codes [n x keys] int32, levels per key)."""
    keys = [key] if isinstance(key, str) else list(key)
    if not keys:
        raise ValueError("batch_key must contain at least one column name")
    codes = np.empty((len(obs), len(keys)), dtype=np.int32)
    n_levels = np.empty(len(keys), dtype=np.int32)
    offset = 0
    for j, k in enumerate(keys):
        col = obs[k].astype("category")
        local = col.cat.codes.to_numpy(dtype=np.int32, copy=False)
        if np.any(local < 0):
            raise ValueError(f"Batch variable {k!r} contains missing values")
        n_levels[j] = col.cat.categories.size
        codes[:, j] = local + offset
        offset += int(n_levels[j])
    return codes, n_levels


def get_theta_array(theta, n_levels: np.ndarray, dtype) -> np.ndarray:
    """A scalar, one value per key or one per level -> [1 x levels]."""
    levels = n_levels.astype(np.int64, copy=False)
    try:
        t = np.asarray(theta, dtype=dtype)
    except (TypeError, ValueError) as e:
        raise ValueError("theta must be a scalar or an array-like collection of numeric values, "
                         f"got {type(theta).__name__}") from e
    if t.ndim == 0:
        return np.full((1, int(levels.sum())), t.item(), dtype=dtype)
    t = t.ravel()
    if t.size == levels.size:
        t = np.repeat(t, levels)
    elif t.size != int(levels.sum()):
        raise ValueError(f"theta array size ({t.size}) must match the number of batch variables ({levels.size}) or "
                         f"categorical levels ({int(levels.sum())})")
    return t.reshape(1, -1)


def compute_lambda_kb(e, *, o, n_b, alpha, threshold, ridge_lambda, dynamic_lambda) -> np.ndarray:
    """Per (code, cluster) ridge penalty; `SUPPRESS_PENALTY` marks the pairs that get no correction."""
    sentinel = e.dtype.type(SUPPRESS_PENALTY)
    if not dynamic_lambda:
        lam = np.full_like(e, ridge_lambda)
    else:
        lam = (alpha * e).astype(e.dtype)
        if threshold is not None:
            safe_n_b = np.where(n_b > 0, n_b, np.ones_like(n_b))
            prune = (o / safe_n_b[:, None]) < threshold
            prune |= n_b[:, None] == 0
            lam[prune] = sentinel
    lam[(o + lam) == 0] = sentinel
    return lam


def fast_weights(phi: np.ndarray, o: np.ndarray, lam: np.ndarray) -> np.ndarray:
    """Single key: W[k] = inv_mat_k @ phi[k] with the reference's factorised inverse, row 0 zeroed.
    phi [K x (B+1) x d]: row 0 Σ r_k x, row b+1 the same over the cells of code b.  o, lam [B x K]."""
    n_batches = o.shape[0]
    w = np.empty_like(phi)
    p = np.eye(n_batches + 1)
    for k in range(o.shape[1]):
        o_k, lam_k = o[:, k], lam[:, k]
        factor = 1.0 / (o_k + lam_k)
        c_inv = 1.0 / (np.sum(o_k) + np.sum(-factor * o_k**2))
        p[0, 1:] = -factor * o_k
        ptb = np.zeros((n_batches + 1, n_batches + 1))
        ptb[0, 0] = c_inv
        ptb[1:, 1:] = np.diag(factor)
        ptb[1:, 0] = p[0, 1:] * c_inv
        w[k] = (ptb @ p) @ phi[k]
        w[k, 0] = 0
    return w


def multi_weights(s: np.ndarray, t: np.ndarray, gcodes: np.ndarray, lam: np.ndarray) -> np.ndarray:
    """Several keys: the exact ridge solve of each cluster over the design [1 | one-hot per key].
    s [G x K], t [G x K x d]: Σ r and Σ r x per code tuple; gcodes [G x keys] marginal codes; lam [B x K]."""
    n_groups, n_clusters, d = t.shape
    n_batches = lam.shape[0]
    sentinel = SUPPRESS_PENALTY
    # one-hot [G x (B+1)] with column 0 the intercept: design rows of a group are all equal
    onehot = np.zeros((n_groups, n_batches + 1))
    onehot[:, 0] = 1
    for j in range(gcodes.shape[1]):
        onehot[np.arange(n_groups), gcodes[:, j] + 1] = 1
    w = np.zeros((n_clusters, n_batches + 1, d))
    for k in range(n_clusters):
        gram = onehot.T @ (s[:, k, None] * onehot)
        rhs = onehot.T @ t[:, k]
        active = lam[:, k] < sentinel
        retained = np.concatenate(([True], active))
        idx = np.flatnonzero(retained)
        gram[idx[1:], idx[1:]] += lam[active, k]
        g_red = gram[np.ix_(idx, idx)]
        rhs_red = rhs[retained]
        try:
            if np.linalg.matrix_rank(g_red) < g_red.shape[0]:
                raise np.linalg.LinAlgError
            w_red = np.linalg.solve(g_red, rhs_red)
        except np.linalg.LinAlgError:
            w_red = np.linalg.lstsq(g_red, rhs_red, rcond=None)[0]
        w[k, retained] = w_red
        w[k, 0] = 0
    return w


def diversity(o, e, theta, sigma, stabilized) -> float:
    ratio = np.log((o + e + 1) / (e + 1)) if stabilized else np.log((o + 1) / (e + 1))
    return float(sigma * np.sum(theta @ (o * ratio)))


def n_blocks_of(n: int, block_proportion: float) -> int:
    return int(min(n, 1 // block_proportion))


def block_bounds(n: int, n_blocks: int) -> np.ndarray:
    """`np.array_split` bounds: the first n % n_blocks blocks get one extra cell."""
    q, rem = divmod(n, n_blocks)
    sizes = np.full(n_blocks, q, dtype=np.int64)
    sizes[:rem] += 1
    return np.concatenate([[0], np.cumsum(sizes)])


def check_caps(d: int, n_clusters: int, n_batches: int, n_tuples: int) -> None:
    for what, v, cap in (("n_clusters", n_clusters, MAX_K), ("the basis width", d, MAX_D),
                         ("the number of batch levels over all keys", n_batches, MAX_CODES),
                         ("the number of distinct batch-key combinations", n_tuples, MAX_TUPLES)):
        if v > cap:
            raise NotImplementedError(f"harmony_integrate in scanpy_b200 supports {what} up to {cap}; got {v}")


def spawn_random_state(gen: np.random.Generator) -> np.random.RandomState:
    [bitgen] = gen.bit_generator.spawn(1)
    return np.random.RandomState(bitgen)


# ------------------------------------------------------------------------------------------ device passes
class _Dev:
    """The device arrays of one run and thin wrappers over the harmony entry points."""

    def __init__(self, x: np.ndarray, codes: np.ndarray, n_batches: int):
        import torch

        self.torch = torch
        self.ctx = _abi.default_context()
        self.lib = self.ctx.lib
        self.h = self.ctx.handle
        self.n, self.d = x.shape
        self.is_f64 = int(x.dtype == np.float64)
        self.tdt = torch.float64 if self.is_f64 else torch.float32
        self.keys = codes.shape[1]
        self.n_codes = n_batches
        self.x = _ops._to_device(x)
        self.z = torch.empty_like(self.x)
        self.codes = _ops._to_device(np.ascontiguousarray(codes, dtype=np.int32))
        check(self.lib.sb2_harmony_normalize(self.h, self.n, self.d, self.is_f64, ptr(self.x), ptr(self.z)))

    def f64(self, *shape):
        return self.torch.empty(shape, dtype=self.torch.float64, device="cuda")

    def wsums(self, bounds: np.ndarray, idx, z, mode: int, k: int, r=None, labels=None, is_f64=None):
        out = self.f64(len(bounds) - 1, k, self.d + 1)
        b = np.ascontiguousarray(bounds, dtype=np.int64)
        check(self.lib.sb2_harmony_wsums(self.h, len(b) - 1, ptr(b), ptr(idx), self.d, k,
                                         self.is_f64 if is_f64 is None else is_f64, ptr(z), mode, ptr(r),
                                         ptr(labels), ptr(out)))
        return out

    def code_sums(self, rows, idx, r, k, out):
        check(self.lib.sb2_harmony_code_sums(self.h, rows, ptr(idx), k, self.is_f64, ptr(r), self.keys,
                                             ptr(self.codes), self.n_codes, ptr(out)))

    def vsum(self, v, n):
        out = self.f64(1)
        check(self.lib.sb2_harmony_sum(self.h, n, ptr(v), ptr(out)))
        return out


def kmeans_start(dev: _Dev, n_clusters: int, rs: np.random.RandomState, dtype, max_iter: int = 25) -> np.ndarray:
    """sklearn's `KMeans(n_clusters, random_state=rs, max_iter=max_iter).fit(z).cluster_centers_` for the rows z of
    `dev.z`: centred data, greedy k-means++, Lloyd."""
    torch, lib, h = dev.torch, dev.lib, dev.h
    n, d = dev.n, dev.d
    sums = _ops._to_host(dev.wsums(np.array([0, n]), None, dev.z, 2, 1))[0, 0]
    mean = sums[:d] / n
    d_mean = _ops._to_device(mean)
    xc, xx = dev.f64(n, d), dev.f64(n)
    check(lib.sb2_harmony_center(h, n, d, dev.is_f64, ptr(dev.z), ptr(d_mean), ptr(xc), ptr(xx)))
    tol = float(_ops._to_host(dev.vsum(xx, n))[0]) / (n * d) * 1e-4

    n_trials = 2 + int(np.log(n_clusters))
    w = np.ones(n, dtype=dtype)
    ids = np.empty(n_clusters, dtype=np.int64)
    ids[0] = rs.choice(n, p=w / w.sum())
    dist = [dev.f64(n_trials, n), dev.f64(n_trials, n)]
    pots = dev.f64(n_trials)
    d_ids = torch.empty(n_trials, dtype=torch.int64, device="cuda")
    d_ids[:1].copy_(torch.from_numpy(ids[:1]))
    check(lib.sb2_harmony_kpp_dists(h, n, d, ptr(xc), ptr(xx), 1, ptr(d_ids), None, ptr(dist[0]), ptr(pots)))
    closest = dist[0][0]
    pot = float(_ops._to_host(pots)[0])
    for c in range(1, n_clusters):
        out = dist[c % 2]
        u = _ops._to_device(rs.uniform(size=n_trials) * pot)
        check(lib.sb2_harmony_kpp_search(h, n, ptr(closest), n_trials, ptr(u), ptr(d_ids)))
        check(lib.sb2_harmony_kpp_dists(h, n, d, ptr(xc), ptr(xx), n_trials, ptr(d_ids), ptr(closest), ptr(out),
                                        ptr(pots)))
        h_pots, h_ids = _ops._to_host(pots, d_ids)
        best = int(np.argmin(h_pots))
        pot = float(h_pots[best])
        closest = out[best]
        ids[c] = h_ids[best]
    centers = _ops._to_host(xc[torch.from_numpy(ids).cuda()])

    labels = [torch.full((n,), -1, dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")]
    changed = torch.zeros(1, dtype=torch.int32, device="cuda")
    bounds = np.array([0, n])
    for _ in range(max_iter):
        changed.zero_()
        d_c = _ops._to_device(np.ascontiguousarray(centers))
        check(lib.sb2_harmony_labels(h, n, d, n_clusters, ptr(xc), ptr(d_c), ptr(labels[0]), ptr(labels[1]),
                                     ptr(changed)))
        s = dev.wsums(bounds, None, xc, 1, n_clusters, labels=labels[1], is_f64=1)
        s, flag = _ops._to_host(s, changed)
        s = s[0]
        sums, counts = s[:, :d].copy(), s[:, d].copy()
        empty = np.flatnonzero(counts == 0)
        if empty.size:
            h_xc, lab = _ops._to_host(xc, labels[1])
            dist = ((h_xc - centers[lab]) ** 2).sum(axis=1)
        # sklearn: the points farthest from their centres start the empty clusters, unless every point sits on its
        # centre (fewer distinct points than clusters); an empty cluster's centre is then 0
        if empty.size and dist.max() > 0:
            far = np.argpartition(dist, -empty.size)[: -empty.size - 1 : -1]
            for k, i in zip(empty, far):
                sums[lab[i]] -= h_xc[i]
                sums[k] = h_xc[i]
                counts[k] = 1.0
                counts[lab[i]] -= 1.0
        avg = sums * (1.0 / np.maximum(counts, 1.0))[:, None]
        # sklearn's _average_centers: a cluster still empty takes the centre of the largest one as the loop over the
        # clusters leaves it, averaged when it comes earlier and still a sum when it comes later
        big = int(np.argmax(counts))
        later = (np.arange(len(counts)) > big)[:, None]
        new = np.where(counts[:, None] > 0, avg, np.where(later, avg[big], sums[big]))
        shift = ((new - centers) ** 2).sum()
        centers = new
        if not flag[0] or shift <= tol:
            break
        labels.reverse()
    return centers + mean


def _objective_sums(dev: _Dev, r, k: int, ent, y_norm: np.ndarray, sigma: float):
    """(Rᵀ[Z | 1] [K x (d+1)], k-means error + entropy term against `y_norm`)."""
    yr = dev.wsums(np.array([0, dev.n]), None, dev.z, 0, k, r=r)
    hent = dev.vsum(ent, dev.n)
    yr, hent = _ops._to_host(yr, hent)
    yr = yr[0]
    kme = 2.0 * yr[:, dev.d].sum() - 2.0 * np.sum(y_norm * yr[:, : dev.d])
    return yr, kme + sigma * float(hent[0])


def _normalize(y: np.ndarray) -> np.ndarray:
    return y / np.maximum(np.linalg.norm(y, axis=1, keepdims=True), 1e-12)


def fit(x: np.ndarray, codes: np.ndarray, n_levels: np.ndarray, *, gen: np.random.Generator, theta, sigma: float,
        n_clusters, max_iter_harmony: int, max_iter_clustering: int, tol_harmony: float, tol_clustering: float,
        ridge_lambda: float, block_proportion: float, tau, stabilized_penalty: bool, dynamic_lambda: bool,
        alpha: float, batch_prune_threshold, centers: np.ndarray | None = None, stats: dict | None = None):
    """`Harmony.fit` -> the corrected matrix in x's dtype.  `centers`: start from these k-means centres instead of
    running the k-means start (the random stream is the same either way).  `stats["iterations"]` receives the
    clustering iterations of every outer iteration."""
    import torch

    n, d = x.shape
    n_batches = int(n_levels.sum())
    n_b = np.bincount(codes.ravel(), minlength=n_batches).astype(x.dtype)
    pr_b = (n_b / n).astype(np.float64)
    theta_arr = get_theta_array(theta, n_levels, x.dtype)
    k = n_clusters if n_clusters is not None else max(int(min(100, n / 30)), 2)
    if tau > 0:
        theta_arr = theta_arr * (1 - np.exp(-n_b / (k * tau)) ** 2)
    theta64 = theta_arr.astype(np.float64)
    # cells grouped by their code tuple, once
    dims = (n_batches,) * codes.shape[1]
    tuples, gid = np.unique(np.ravel_multi_index(codes.T, dims), return_inverse=True)
    gcodes = np.stack(np.unravel_index(tuples, dims), axis=1).astype(np.int32)
    order = np.argsort(gid, kind="stable")
    gbounds = np.searchsorted(gid[order], np.arange(len(gcodes) + 1)).astype(np.int64)
    check_caps(d, k, n_batches, len(gcodes))

    rs = spawn_random_state(gen)
    dev = _Dev(x, codes, n_batches)
    if centers is None:
        centers = kmeans_start(dev, k, rs, x.dtype)
    y_norm = _normalize(np.asarray(centers, dtype=np.float64))
    term = -2.0 / sigma
    r = torch.empty((n, k), dtype=dev.tdt, device="cuda")
    ent = dev.f64(n)
    check(dev.lib.sb2_harmony_step(dev.h, n, None, d, k, dev.is_f64, ptr(dev.z), ptr(_ops._to_device(y_norm)), 0,
                                   None, None, term, ptr(r), ptr(ent)))
    sums = dev.f64(n_batches + 1, k)
    dev.code_sums(n, None, r, k, sums)
    h_sums = _ops._to_host(sums)
    o = dev.f64(n_batches, k).copy_(torch.from_numpy(h_sums[:n_batches]))
    e = _ops._to_device(np.ascontiguousarray(pr_b[:, None] * h_sums[n_batches][None, :]))
    pen = dev.f64(n_batches, k)
    d_pr_b, d_theta = _ops._to_device(pr_b), _ops._to_device(np.ascontiguousarray(theta64.ravel()))
    yr, part = _objective_sums(dev, r, k, ent, y_norm, sigma)
    h_o, h_e = _ops._to_host(o, e)
    objectives = [part + diversity(h_o, h_e, theta64, sigma, stabilized_penalty)]

    bounds = block_bounds(n, n_blocks_of(n, block_proportion))
    d_order, d_gcodes = _ops._to_device(order.astype(np.int64)), _ops._to_device(gcodes)
    zhat = torch.empty_like(dev.x)
    iterations = []
    perm = gen.permutation(n)

    def update(sign, rows, idx):
        dev.code_sums(rows, idx, r, k, sums)
        check(dev.lib.sb2_harmony_oe_update(dev.h, n_batches, k, sign, ptr(sums), ptr(d_pr_b), ptr(d_theta),
                                            int(stabilized_penalty), ptr(o), ptr(e), ptr(pen)))

    fresh_z = False  # yr holds Rᵀ[Z | 1] for the current Z and R
    for it_h in range(max_iter_harmony):
        objs, obj, it = [], None, 0
        for it in range(1, max_iter_clustering + 1):
            if fresh_z:
                yr = _ops._to_host(dev.wsums(np.array([0, n]), None, dev.z, 0, k, r=r))[0]
                fresh_z = False
            y_norm = _normalize(yr[:, :d])
            d_y = _ops._to_device(y_norm)
            d_perm = _ops._to_device(perm.astype(np.int64))
            for b0, b1 in zip(bounds[:-1], bounds[1:]):
                idx = d_perm[int(b0):]
                rows = int(b1 - b0)
                update(-1.0, rows, idx)
                check(dev.lib.sb2_harmony_step(dev.h, rows, ptr(idx), d, k, dev.is_f64, ptr(dev.z), ptr(d_y),
                                               dev.keys, ptr(dev.codes), ptr(pen), term, ptr(r), ptr(ent)))
                update(1.0, rows, idx)
            perm = gen.permutation(n)  # drawn while the device works: the stream does not depend on the data
            yr, part = _objective_sums(dev, r, k, ent, y_norm, sigma)
            h_o, h_e = _ops._to_host(o, e)
            objs.append(part + diversity(h_o, h_e, theta64, sigma, stabilized_penalty))
            if len(objs) >= 4 and sum(objs[-4:-1]) - sum(objs[-3:]) < tol_clustering * abs(sum(objs[-4:-1])):
                obj = objs[-1]
                break
        iterations.append(it)
        if obj is not None:
            objectives.append(obj)

        lam = compute_lambda_kb(h_e, o=h_o, n_b=n_b.astype(np.float64), alpha=alpha, threshold=batch_prune_threshold,
                                ridge_lambda=ridge_lambda, dynamic_lambda=dynamic_lambda)
        st = _ops._to_host(dev.wsums(gbounds, d_order, dev.x, 0, k, r=r))  # [G x K x (d+1)]
        if codes.shape[1] > 1:
            w = multi_weights(st[:, :, d], st[:, :, :d], gcodes, lam)
        else:
            phi = np.zeros((k, n_batches + 1, d))
            phi[:, 0] = st[:, :, :d].sum(axis=0)
            np.add.at(phi, (slice(None), gcodes[:, 0] + 1), st[:, :, :d].transpose(1, 0, 2))
            w = fast_weights(phi, h_o, lam)
        d_w = _ops._to_device(np.ascontiguousarray(w))
        b = np.ascontiguousarray(gbounds)
        check(dev.lib.sb2_harmony_apply(dev.h, len(gcodes), ptr(b), ptr(d_order), d, k, dev.is_f64, dev.keys,
                                        ptr(d_gcodes), n_batches, ptr(d_w), ptr(dev.x), ptr(r), ptr(zhat),
                                        ptr(dev.z)))
        fresh_z = True
        if len(objectives) >= 2 and (objectives[-2] - objectives[-1]) < tol_harmony * abs(objectives[-2]):
            logger.info(f"Harmony converged in {it_h + 1} iterations")
            break
    else:
        logger.info(f"Harmony did not converge after {max_iter_harmony} iterations.")
    if stats is not None:
        stats["iterations"] = iterations
        stats["objectives"] = objectives
    return _ops._to_host(zhat)


# ------------------------------------------------------------------------------------------ public
def harmony_integrate(adata, key, *, basis: str = "X_pca", adjusted_basis: str = "X_pca_harmony",
                      dtype=np.float64, flavor: str = "harmony2", n_clusters: int | None = None,
                      max_iter_harmony: int = 10, max_iter_clustering: int = 200, tol_harmony: float = 1e-4,
                      tol_clustering: float = 1e-5, sigma: float = 0.1, theta=2.0, tau: int = 0,
                      ridge_lambda: float = 1.0, alpha: float = 0.2, batch_prune_threshold: float | None = 1e-5,
                      correction_method: str = "fast", block_proportion: float = 0.05, rng=None) -> None:
    """Integrate batches with Harmony (signature of `scanpy.pp.harmony_integrate`).

    Writes `adata.obsm[adjusted_basis]` in `dtype` (float32 or float64)."""
    if flavor not in {"harmony1", "harmony2"}:
        raise ValueError(f"flavor must be 'harmony1' or 'harmony2', got {flavor!r}.")
    if correction_method != "fast":
        raise ValueError(f"correction_method must be 'fast', got {correction_method!r}.")
    stabilized_penalty = dynamic_lambda = flavor == "harmony2"
    if flavor == "harmony2" and ridge_lambda != 1.0:
        warn("ridge_lambda is ignored when flavor='harmony2'; use alpha to control regularization strength.",
             UserWarning)
    if flavor == "harmony1":
        if alpha != 0.2:
            warn("alpha is ignored when flavor='harmony1'; use ridge_lambda instead.", UserWarning)
        if batch_prune_threshold != 1e-5:
            warn("batch_prune_threshold is ignored when flavor='harmony1'.", UserWarning)
    if basis not in adata.obsm:
        raise ValueError(f"The specified basis {basis!r} is not available in `adata.obsm`. "
                         f"Available bases: {list(adata.obsm.keys())}")
    input_data = adata.obsm[basis]
    try:
        x = np.ascontiguousarray(input_data, dtype=dtype)
    except Exception as e:
        raise TypeError(f"Could not convert input of type {type(input_data).__name__} to NumPy array.") from e
    if np.isnan(x).any():
        raise ValueError("Input data contains NaN values. Please handle these before running harmony_integrate.")

    gen = np.random.default_rng(rng)
    if max_iter_harmony < 1:
        raise ValueError("max_iter_harmony must be >= 1")
    if dynamic_lambda:
        if not np.isfinite(alpha) or alpha <= 0:
            raise ValueError(f"alpha must be a finite positive number when dynamic_lambda=True, got {alpha}.")
        if batch_prune_threshold is not None and not (0 <= batch_prune_threshold <= 1):
            raise ValueError(f"batch_prune_threshold must be in [0, 1] or None, got {batch_prune_threshold}.")
    elif not np.isfinite(ridge_lambda) or ridge_lambda <= 0:
        raise ValueError(f"ridge_lambda must be a finite positive number when dynamic_lambda=False, got {ridge_lambda}.")
    obs = adata.obs if isinstance(adata.obs, pd.DataFrame) else pd.DataFrame(adata.obs)
    codes, n_levels = get_batch_codes(obs, key)
    if x.dtype not in (np.float32, np.float64):
        raise NotImplementedError(f"harmony_integrate in scanpy_b200 supports float32 and float64, not {x.dtype}")
    adata.obsm[adjusted_basis] = fit(
        x, codes, n_levels, gen=gen, theta=theta, sigma=sigma, n_clusters=n_clusters,
        max_iter_harmony=max_iter_harmony, max_iter_clustering=max_iter_clustering, tol_harmony=tol_harmony,
        tol_clustering=tol_clustering, ridge_lambda=ridge_lambda, block_proportion=block_proportion, tau=tau,
        stabilized_penalty=stabilized_penalty, dynamic_lambda=dynamic_lambda, alpha=alpha,
        batch_prune_threshold=batch_prune_threshold)

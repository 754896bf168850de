"""Each `sb2_harmony_*` entry point of csrc/harmony.cu against a short numpy float64 restatement, at the shapes where
the kernels change layout: clusters per lane (lane l owns clusters l, l + 32, l + 64, l + 96), columns per lane (the
same for d), the output slices of `wsums_kernel` (K·(d+1) > 2048), groups that span several CHUNK_ROWS = 2048 chunks,
the two-level cumsum of `kpp_search_kernel`, and dynamic shared memory above 48 KB at the caps K = d = 128 codes.

The restatements are checked against `oracle/harmony.py` and brute force by the unmarked tests, so they run without a
device; the device tests are marked `gpu`.

Tolerances come from the arithmetic.  ε is the unit round-off of the type (2⁻⁵³ for float64, 2⁻²⁴ for float32).  A
sum of m terms in any order is within γ_m·Σ|terms| of the exact sum, γ_m ≈ m·ε; the device and numpy each are, so
they agree to 2(m + 1)·ε·Σ|terms| (`sum_tol`).  A float32 dot of unit rows is within d·ε₃₂ of the exact dot, and one
float32 store or operation moves a value by ε₃₂ of itself.  Each test says which of these it adds up.
"""
from __future__ import annotations

import numpy as np
import pytest
from scipy import sparse

from oracle import harmony as oh
from scanpy_b200 import _harmony as hm

CHUNK = 2048  # CHUNK_ROWS in harmony.cu
EPS = {np.float64: 2.0**-53, np.float32: 2.0**-24}
E64 = EPS[np.float64]
DTYPES = [np.float64, np.float32]
D_EDGES = [1, 31, 32, 33, 64, 65, 96, 127, 128]
K_EDGES = [1, 2, 31, 32, 33, 63, 64, 65, 100, 127, 128]
GROUP_ROWS = [0, 1, 2047, 2048, 2049, 6145]


def sum_tol(mag, m):
    """Two orders of a sum of m terms whose magnitudes add up to `mag`."""
    return 2.0 * (m + 1) * E64 * mag


def unit_rows(rng, n, d, dtype=np.float64):
    x = rng.normal(size=(n, d))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(dtype)


# ------------------------------------------------------------------------------------------ restatements
def normalize_ref(x):
    x = np.asarray(x, dtype=np.float64)
    return x / np.maximum(np.sqrt((x * x).sum(axis=1, keepdims=True)), 1e-12)


def wsums_ref(bounds, idx, z, mode, k, r=None, labels=None):
    """-> (Σ w·[z | 1] per group [G x k x (d+1)], the same sum of |w·[z | 1]|).  Weights: r (mode 0), one-hot
    labels (mode 1), 1 (mode 2, k = 1).  Group g holds rows idx[bounds[g]:bounds[g+1]] (idx None: the positions)."""
    z1 = np.hstack([np.asarray(z, dtype=np.float64), np.ones((len(z), 1))])
    rows = np.arange(bounds[-1]) if idx is None else np.asarray(idx)
    out = np.zeros((len(bounds) - 1, k, z1.shape[1]))
    mag = np.zeros_like(out)
    for g, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        sel = rows[a:b]
        if mode == 0:
            w = np.asarray(r, dtype=np.float64)[sel]
        elif mode == 1:
            w = np.zeros((len(sel), k))
            w[np.arange(len(sel)), labels[sel]] = 1.0
        else:
            w = np.ones((len(sel), 1))
        out[g] = w.T @ z1[sel]
        mag[g] = np.abs(w).T @ np.abs(z1[sel])
    return out, mag


def step_ref(z, y, term, rows, codes=None, pen=None):
    """r and the entropy term of the cells `rows`: softmax over clusters of term·(1 - z·y) + Σ_keys pen[code]."""
    lr = term * (1.0 - np.asarray(z, dtype=np.float64)[rows] @ y.T)
    if pen is not None:
        lr = lr + pen[codes[rows]].sum(axis=1)
    lr = lr - lr.max(axis=1, keepdims=True)
    r = np.exp(lr)
    r /= np.maximum(r.sum(axis=1, keepdims=True), 1e-12)
    rn = r / np.maximum(r.sum(axis=1, keepdims=True), 1e-12)
    return r, (rn * np.log(rn + 1e-12)).sum(axis=1)


def code_sums_ref(rows, idx, r, codes, n_codes):
    """[(n_codes + 1) x k]: Σ r per marginal code over every key, then Σ r over the cells."""
    sel = np.arange(rows) if idx is None else np.asarray(idx)[:rows]
    rr = np.asarray(r, dtype=np.float64)[sel]
    cc = codes[sel]
    onehot = sparse.csr_matrix((np.ones(cc.size), (cc.ravel(), np.repeat(np.arange(len(sel)), cc.shape[1]))),
                               shape=(n_codes, len(sel)))
    return np.vstack([onehot @ rr, rr.sum(axis=0)])


def oe_update_ref(o, e, sums, pr_b, theta, sign, stabilized):
    n_codes = len(o)
    ov = o + sign * sums[:n_codes]
    ev = e + sign * pr_b[:, None] * sums[n_codes][None, :]
    pen = theta[:, None] * (np.log(ev + 1.0) - np.log((ov + ev if stabilized else ov) + 1.0))
    return ov, ev, pen


def center_ref(z, mean):
    xc = np.asarray(z, dtype=np.float64) - mean
    return xc, (xc * xc).sum(axis=1)


def kpp_search_ref(v, u):
    return np.minimum(np.searchsorted(np.cumsum(v), u, "left"), len(v) - 1)


def kpp_dists_ref(xc, xx, ids, closest=None):
    dist = np.stack([oh._sq_dists(xc[i], xc, xx) for i in ids])
    if closest is not None:
        dist = np.minimum(dist, closest[None, :])
    return dist, dist.sum(axis=1)


def labels_ref(xc, centers):
    """argmin_c ||c||² - 2 x·c; a centre equal to an earlier one never wins (the lowest index of equal values)."""
    _, first = np.unique(centers, axis=0, return_index=True)
    u = centers[np.sort(first)]
    d2 = (u * u).sum(axis=1)[None, :] - 2.0 * xc @ u.T
    return np.sort(first)[np.argmin(d2, axis=1)].astype(np.int32), d2


def apply_ref(bounds, idx, gcodes, w, x, r):
    """z_hat = x - r·Σ_keys W[:, code + 1] per code tuple, its row-normalised copy, and Σ|r·W| per element.
    w: [k x (n_codes + 1) x d]."""
    x64, r64 = np.asarray(x, dtype=np.float64), np.asarray(r, dtype=np.float64)
    zhat = np.zeros_like(x64)
    mag = np.zeros_like(x64)
    for g, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        sel = idx[a:b]
        wc = w[:, gcodes[g] + 1, :].sum(axis=1)
        zhat[sel] = x64[sel] - r64[sel] @ wc
        mag[sel] = np.abs(r64[sel]) @ np.abs(wc)
    return zhat, mag


# ------------------------------------------------------------------------------------------ the restatements' checks
def test_normalize_ref_is_the_oracles():
    x = np.random.default_rng(0).normal(size=(50, 7))
    x[3] = 0
    np.testing.assert_allclose(normalize_ref(x), oh._normalize(x), rtol=1e-15, atol=0)
    assert not normalize_ref(x)[3].any()


def _tuples(codes):
    gcodes, gid = np.unique(codes, axis=0, return_inverse=True)
    order = np.argsort(gid.ravel(), kind="stable")
    bounds = np.searchsorted(gid.ravel()[order], np.arange(len(gcodes) + 1))
    return gcodes, order, bounds


def _weights_inputs(keys, seed=5):
    rng = np.random.default_rng(seed)
    n, d, k, levels = 300, 6, 4, [3, 4, 2][:keys]
    codes = np.column_stack([rng.integers(0, lv, size=n) for lv in levels]) + np.concatenate([[0], np.cumsum(levels)[:-1]])
    x = rng.normal(size=(n, d))
    r = rng.random(size=(n, k))
    r /= r.sum(axis=1, keepdims=True)
    lam = rng.uniform(0.2, 1.0, size=(sum(levels), k))
    lam[1, 2] = oh.SUPPRESS_PENALTY
    return x, codes, r, lam, sum(levels)


@pytest.mark.parametrize("keys", [1, 2, 3])
def test_wsums_and_apply_refs_give_the_oracles_correction(keys):
    """The grouped sums of `wsums_ref` (mode 0 over code tuples) turned into weights by the host, then `apply_ref`,
    equal the oracle's correction from the cells (`_correct_fast` for one key, the dense design for several)."""
    x, codes, r, lam, n_codes = _weights_inputs(keys)
    gcodes, order, bounds = _tuples(codes)
    st, _ = wsums_ref(bounds, order, x, 0, r.shape[1], r=r)
    o = np.stack([r[codes[:, 0] == b].sum(axis=0) for b in range(n_codes)])
    if keys == 1:
        phi = np.zeros((r.shape[1], n_codes + 1, x.shape[1]))
        phi[:, 0] = st[:, :, :-1].sum(axis=0)
        phi[:, gcodes[:, 0] + 1] = st[:, :, :-1].transpose(1, 0, 2)
        w = hm.fast_weights(phi, o, lam)
        want = oh._correct_fast(x, codes[:, 0], n_codes, r, o, lam)
    else:
        w = hm.multi_weights(st[:, :, -1], st[:, :, :-1], gcodes, lam)
        want = oh._correct_multi(x, codes, n_codes, r, lam)
    got, _ = apply_ref(bounds, order, gcodes, w, x, r)
    np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-11)


def test_wsums_ref_lloyd_sums_and_plain_sums():
    rng = np.random.default_rng(2)
    z = rng.normal(size=(500, 9))
    labels = rng.integers(0, 6, size=500)
    labels[labels == 4] = 5  # label 4 has no rows
    got, _ = wsums_ref(np.array([0, 500]), None, z, 1, 6, labels=labels)
    sums = np.zeros((6, 9))
    np.add.at(sums, labels, z)
    np.testing.assert_allclose(got[0, :, :9], sums, rtol=1e-13, atol=1e-13)
    np.testing.assert_array_equal(got[0, :, 9], np.bincount(labels, minlength=6))
    perm = rng.permutation(500)
    got, _ = wsums_ref(np.array([0, 200, 200, 500]), perm, z, 2, 1)
    np.testing.assert_allclose(got[:, 0, :9], [z[perm[:200]].sum(0), np.zeros(9), z[perm[200:]].sum(0)], atol=1e-12)
    np.testing.assert_array_equal(got[:, 0, 9], [200, 0, 300])


def test_step_ref_entropy_and_penalty_are_the_oracles():
    """Without a penalty r is the oracle's first r; σ·Σ entropy terms + k-means error + diversity is the oracle's
    objective; the penalty from `oe_update_ref` is the oracle's."""
    rng = np.random.default_rng(3)
    n, k, n_codes, sigma = 400, 7, 5, 0.1
    z, y = unit_rows(rng, n, 12), unit_rows(rng, k, 12)
    term = -2.0 / sigma
    r, ent = step_ref(z, y, term, np.arange(n))
    want = np.exp(term * (1.0 - z @ y.T))
    want /= want.sum(axis=1, keepdims=True)
    np.testing.assert_allclose(r, want, rtol=1e-12, atol=1e-300)
    codes = rng.integers(0, n_codes, size=(n, 1))
    theta = np.full((1, n_codes), 2.0)
    pr_b = np.bincount(codes[:, 0], minlength=n_codes) / n
    sums = code_sums_ref(n, None, r, codes, n_codes)
    o, e, pen = oe_update_ref(np.zeros((n_codes, k)), np.zeros((n_codes, k)), sums, pr_b, theta[0], 1.0, True)
    o_want = np.zeros((n_codes, k))
    np.add.at(o_want, codes[:, 0], r)
    np.testing.assert_allclose(o, o_want, rtol=1e-13)
    np.testing.assert_allclose(e, pr_b[:, None] @ r.sum(axis=0)[None, :], rtol=1e-13)
    np.testing.assert_allclose(pen, theta.T * (np.log(e + 1.0) - np.log(o + e + 1.0)), rtol=1e-13)
    kme = np.sum(r * 2.0 * (1.0 - z @ y.T))
    ratio = np.log((o + e + 1) / (e + 1))
    got = kme + sigma * ent.sum() + sigma * np.sum(theta @ (o * ratio))
    np.testing.assert_allclose(got, oh._objective(y, z, r, theta, sigma, o, e, True), rtol=1e-12)
    # the penalty enters the exponent of each cell through its code
    r2, _ = step_ref(z, y, term, np.arange(n), codes, pen)
    lr = term * (1.0 - z @ y.T) + pen[codes[:, 0]]
    want = np.exp(lr - lr.max(axis=1, keepdims=True))
    np.testing.assert_allclose(r2, want / want.sum(axis=1, keepdims=True), rtol=1e-12, atol=1e-300)


def test_code_sums_ref_is_add_at():
    rng = np.random.default_rng(4)
    r = rng.random(size=(300, 5))
    codes = np.column_stack([rng.integers(0, 3, 300), rng.integers(3, 7, 300)])
    idx = rng.permutation(300)
    got = code_sums_ref(120, idx, r, codes, 7)
    want = np.zeros((8, 5))
    for c in codes[idx[:120]].T:
        np.add.at(want, c, r[idx[:120]])
    want[7] = r[idx[:120]].sum(axis=0)
    np.testing.assert_allclose(got, want, rtol=1e-13)


def test_kpp_search_ref_is_a_serial_scan():
    rng = np.random.default_rng(5)
    v = rng.integers(0, 3, size=200).astype(np.float64)
    c = np.cumsum(v)
    for u in [0.0, 0.5, c[17], c[17] + 0.5, c[-1], c[-1] + 1.0]:
        want = next((i for i in range(len(v)) if c[i] >= u), len(v) - 1)
        assert kpp_search_ref(v, np.array([u]))[0] == want


def test_kpp_dists_and_labels_refs_are_brute_force():
    rng = np.random.default_rng(6)
    xc = rng.normal(size=(300, 8))
    xx = (xc * xc).sum(axis=1)
    dist, pot = kpp_dists_ref(xc, xx, [3, 77])
    brute = np.stack([((xc - xc[i]) ** 2).sum(axis=1) for i in (3, 77)])
    np.testing.assert_allclose(dist, brute, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(pot, brute.sum(axis=1), rtol=1e-12)
    centers = xc[[5, 9, 5, 40, 9]]
    got, _ = labels_ref(xc, centers)
    want = np.argmin(((xc[:, None, :] - centers[None]) ** 2).sum(axis=2), axis=1)
    np.testing.assert_array_equal(centers[got], centers[want])
    assert not np.isin(got, [2, 4]).any()  # the later copies never win


# ------------------------------------------------------------------------------------------ device plumbing
def _lib():
    from scanpy_b200 import _abi

    ctx = _abi.default_context()
    return ctx.lib, ctx.handle


def dev(a):
    """A device copy of `a`.  Keep it in a variable until the entry point has run: a temporary freed while the
    arguments are still being built lets the next copy reuse its memory before the kernel reads it."""
    import torch

    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def empty(shape, dtype, fill=None):
    import torch

    t = torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), device="cuda")
    if fill is not None:
        t.fill_(fill)
    return t


def call(fn, *args):
    hm.check(fn(*args))


def ptr(t):
    return hm.ptr(t)


def is64(dtype):
    return int(dtype == np.float64)


# ------------------------------------------------------------------------------------------ normalize
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_normalize(dtype):
    """out = x / max(||x||, 1e-12) with the norm in float64: the restatement sees the same stored x, so the two differ by
    the final store (ε_T·|out|) and the reordered norm ((d + 2)·ε₆₄·|out|)."""
    lib, h = _lib()
    rng = np.random.default_rng(10)
    for d in D_EDGES:
        x = (rng.normal(size=(1003, d)) * rng.uniform(0.01, 100, size=(1003, 1))).astype(dtype)
        x[7] = 0
        d_x, out = dev(x), empty((1003, d), dtype)
        call(lib.sb2_harmony_normalize, h, 1003, d, is64(dtype), ptr(d_x), ptr(out))
        got, want = host(out), normalize_ref(x)
        assert not got[7].any(), d
        tol = (EPS[dtype] + (d + 2) * E64) * np.abs(want)
        assert (np.abs(got - want) <= tol).all(), (d, np.abs(got - want).max())


# ------------------------------------------------------------------------------------------ wsums
def _wsums(lib, h, bounds, idx, z, mode, k, dtype, r=None, labels=None):
    d = z.shape[1]
    out = empty((len(bounds) - 1, k, d + 1), np.float64, fill=np.nan)
    b = np.ascontiguousarray(bounds, dtype=np.int64)
    d_idx, d_z, d_r, d_labels = dev(None if idx is None else idx.astype(np.int64)), dev(z), dev(r), dev(labels)
    call(lib.sb2_harmony_wsums, h, len(b) - 1, ptr(b), ptr(d_idx), d, k, is64(dtype), ptr(d_z), mode, ptr(d_r),
         ptr(d_labels), ptr(out))
    return host(out)


WSUMS_SHAPES = [(16, 126), (16, 127), (17, 120), (128, 128)]  # K·(d+1) = 2032, 2048, 2057, the cap 16,512


@pytest.mark.gpu
@pytest.mark.parametrize("perm", [True, False], ids=["perm", "positions"])
@pytest.mark.parametrize(("mode", "dtype", "k", "d"),
                         [(0, t, k, d) for t in DTYPES for k, d in WSUMS_SHAPES]
                         + [(1, np.float64, k, d) for k, d in WSUMS_SHAPES]
                         + [(2, t, 1, d) for t in DTYPES for d in (1, 64, 128)])
def test_wsums(mode, dtype, k, d, perm):
    """Every output of every group against the restatement, to `sum_tol` over the group's rows (the weights and z are
    the same stored values on both sides, and every product and sum is float64).  Groups of 0, 1, 2047, 2048, 2049 and
    6145 rows: none, one and four chunks."""
    lib, h = _lib()
    rng = np.random.default_rng(11 + k + d)
    bounds = np.concatenate([[0], np.cumsum(GROUP_ROWS)]).astype(np.int64)
    n = int(bounds[-1])
    z = rng.normal(size=(n, d)).astype(dtype)
    idx = rng.permutation(n) if perm else None
    r = labels = None
    if mode == 0:
        r = rng.random(size=(n, k)).astype(dtype)
    if mode == 1:
        labels = rng.integers(0, k, size=n).astype(np.int32)
        labels[labels == k // 2] = 0  # one label without rows
    got = _wsums(lib, h, bounds, idx, z, mode, k, dtype, r=r, labels=labels)
    want, mag = wsums_ref(bounds, idx, z, mode, k, r=r, labels=labels)
    assert not got[0].any()
    if mode == 1:
        assert not got[:, k // 2].any()
        np.testing.assert_array_equal(got[..., d], want[..., d])  # counts are exact
    err = np.abs(got - want)
    assert (err <= sum_tol(mag, max(GROUP_ROWS))).all(), err.max()


# ------------------------------------------------------------------------------------------ step
def _step(lib, h, z, y, term, idx, n, k, dtype, codes=None, pen=None):
    d = z.shape[1]
    r = empty((n, k), dtype, fill=12345.0)
    ent = empty((n,), np.float64, fill=12345.0)
    keys = 0 if codes is None else codes.shape[1]
    d_idx, d_z, d_y, d_pen = dev(idx.astype(np.int64)), dev(z), dev(y), dev(pen)
    d_codes = dev(None if codes is None else codes.astype(np.int32))
    call(lib.sb2_harmony_step, h, len(idx), ptr(d_idx), d, k, is64(dtype), ptr(d_z), ptr(d_y), keys, ptr(d_codes),
         ptr(d_pen), term, ptr(r), ptr(ent))
    return host(r), host(ent)


def _check_step(got_r, got_ent, z, y, term, idx, dtype, codes=None, pen=None):
    """The exponent of cell i and cluster c is lr = term·(1 - z·y) + ps, ps the float64 penalty sum.  The device forms
    it in T: the dot of unit rows is within d·ε_T, 1 - dot, the product, the store of ps, the sum and the shift by the
    maximum each add ε_T of their size, so |Δlr| ≤ δ = ε_T·(|term|·(d + 4) + 3·|ps| + 2·|lr|) + 2d·ε₆₄·|term|.  r is
    exp(lr - max) over its float64 sum of k terms: within e^{2δ} - 1 of r, plus 2k·ε₆₄ for the two sums and 6ε_T for
    the two exponentials (2 ulp each), the division and the store (and the smallest float32 subnormal).  The entropy
    term Σ rn·log(rn + 1e-12) moves by at most (|log 1e-12| + 1)·2 ≤ 60 times Σ|Δr|, plus its float64 sum."""
    eps = EPS[dtype]
    n, k = got_r.shape
    d = z.shape[1]
    y_t = y.astype(dtype).astype(np.float64)  # the device stages y in T
    want_r, want_ent = step_ref(z, y_t, term, idx, codes, pen)
    lr = term * (1.0 - z.astype(np.float64)[idx] @ y_t.T)
    ps = np.zeros_like(lr) if pen is None else np.abs(pen)[codes[idx]].sum(axis=1)
    delta = (eps * (abs(term) * (d + 4) + 3 * ps + 2 * (np.abs(lr) + ps)) + 2 * d * E64 * abs(term)).max(axis=1)
    rtol = np.expm1(2 * delta + 2 * k * E64 + 6 * eps)[:, None]
    tol_r = rtol * want_r + (2.0**-148 if dtype == np.float32 else 0.0)
    err = np.abs(got_r[idx].astype(np.float64) - want_r)
    assert (err <= tol_r).all(), err.max()
    tol_h = 60.0 * tol_r.sum(axis=1) + sum_tol(np.abs(want_ent) + 1e-11, k)
    assert (np.abs(got_ent[idx] - want_ent) <= tol_h).all(), np.abs(got_ent[idx] - want_ent).max()
    rest = np.setdiff1d(np.arange(n), idx)
    assert (got_r[rest] == 12345.0).all() and (got_ent[rest] == 12345.0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("k", K_EDGES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_step_without_penalty(dtype, k):
    """Every cluster and basis width edge, on a block that is a subset of a permutation; the other rows keep the
    sentinel.  At K = 128, d ≥ 56 (float64) the kernel takes more than 48 KB of shared memory."""
    lib, h = _lib()
    rng = np.random.default_rng(20 + k)
    n = 1500
    for d in D_EDGES:
        z, y = unit_rows(rng, n, d, dtype), unit_rows(rng, k, d)
        idx = rng.permutation(n)[:1100]
        r, ent = _step(lib, h, z, y, -20.0, idx, n, k, dtype)
        _check_step(r, ent, z, y, -20.0, idx, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("sigma", [0.1, 0.05])
@pytest.mark.parametrize("keys", [1, 2, 3])
@pytest.mark.parametrize(("k", "d"), [(33, 20), (100, 65), (128, 128)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_step_with_penalty(dtype, k, d, keys, sigma):
    """The penalty of every key of the cell's codes; sigma = 0.05 spreads the exponents over 80 + |pen| units, so
    most of r is below 1e-30."""
    lib, h = _lib()
    rng = np.random.default_rng(30 + keys + k)
    n, n_codes = 2000, 128
    z, y = unit_rows(rng, n, d, dtype), unit_rows(rng, k, d)
    bounds = np.linspace(0, n_codes, keys + 1).astype(int)
    codes = np.column_stack([rng.integers(bounds[u], bounds[u + 1], size=n) for u in range(keys)])
    pen = rng.normal(scale=2.0, size=(n_codes, k))
    idx = rng.permutation(n)[:1700]
    r, ent = _step(lib, h, z, y, -2.0 / sigma, idx, n, k, dtype, codes, pen)
    _check_step(r, ent, z, y, -2.0 / sigma, idx, dtype, codes, pen)


# ------------------------------------------------------------------------------------------ code_sums, oe_update, sum
@pytest.mark.gpu
@pytest.mark.parametrize("keys", [1, 2, 3])
@pytest.mark.parametrize("rows", [1, 256, 257, 135_169])
@pytest.mark.parametrize("dtype", DTYPES)
def test_code_sums(dtype, rows, keys):
    """Σ r per code over the first `rows` entries of a permutation, 128 codes at K = 128 (132 KB of shared memory) and
    7 codes at K = 33; float64 sums of the stored r, to `sum_tol` over the rows."""
    lib, h = _lib()
    rng = np.random.default_rng(40 + keys)
    n = rows + 100
    for k, n_codes in ((128, 128), (33, 7)):
        r = rng.random(size=(n, k)).astype(dtype)
        bounds = np.linspace(0, n_codes, keys + 1).astype(int)
        codes = np.column_stack([rng.integers(bounds[u], bounds[u + 1], size=n) for u in range(keys)]).astype(np.int32)
        idx = rng.permutation(n)
        out = empty(((n_codes + 1) * k,), np.float64, fill=np.nan)
        d_idx, d_r, d_codes = dev(idx.astype(np.int64)), dev(r), dev(codes)
        call(lib.sb2_harmony_code_sums, h, rows, ptr(d_idx), k, is64(dtype), ptr(d_r), keys, ptr(d_codes), n_codes,
             ptr(out))
        want = code_sums_ref(rows, idx, r, codes, n_codes)
        err = np.abs(host(out).reshape(n_codes + 1, k) - want)
        assert (err <= sum_tol(want, rows)).all(), (k, err.max())


@pytest.mark.gpu
@pytest.mark.parametrize("stabilized", [0, 1])
@pytest.mark.parametrize("sign", [-1.0, 1.0])
def test_oe_update(sign, stabilized):
    """o += sign·sums and e += sign·pr_b·Σr round once or twice (2ε₆₄ and 4ε₆₄ of the terms' sizes); pen =
    θ·(log a - log b) with a = e + 1, b = o [+ e] + 1 then moves by Δa/a + Δb/b, plus 2 ulp per log and the
    subtraction and the product."""
    lib, h = _lib()
    rng = np.random.default_rng(50)
    n_codes, k = 128, 100
    o, e = rng.uniform(5, 50, size=(2, n_codes, k))
    sums = rng.uniform(0, 4, size=(n_codes + 1, k))
    sums[n_codes] = rng.uniform(0, 100, size=k)  # pr_b·Σr < 5: e stays positive
    pr_b = rng.dirichlet(np.ones(n_codes))
    theta = rng.uniform(0, 3, size=n_codes)
    d_o, d_e, d_pen = dev(o), dev(e), empty((n_codes, k), np.float64)
    d_sums, d_pr_b, d_theta = dev(sums), dev(pr_b), dev(theta)
    call(lib.sb2_harmony_oe_update, h, n_codes, k, sign, ptr(d_sums), ptr(d_pr_b), ptr(d_theta), stabilized,
         ptr(d_o), ptr(d_e), ptr(d_pen))
    ov, ev, pen = oe_update_ref(o, e, sums, pr_b, theta, sign, stabilized)
    tol_o = 2 * E64 * (o + sums[:n_codes])
    tol_e = 4 * E64 * (e + pr_b[:, None] * sums[n_codes][None, :])
    assert (np.abs(host(d_o) - ov) <= tol_o).all() and (np.abs(host(d_e) - ev) <= tol_e).all()
    a, b = ev + 1, ((ov + ev) if stabilized else ov) + 1
    da, db = tol_e + E64 * a, (tol_o + tol_e if stabilized else tol_o) + 2 * E64 * b
    tol = theta[:, None] * (da / a + db / b + 6 * E64 * (np.abs(np.log(a)) + np.abs(np.log(b)))) + 2 * E64 * np.abs(pen)
    assert (np.abs(host(d_pen) - pen) <= tol).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 135_168, 135_169, 1_000_003])
def test_sum(n):
    """Σ v in float64 to `sum_tol`; a second call gives the same bits."""
    import math

    lib, h = _lib()
    v = np.random.default_rng(n).normal(size=n) * 10.0
    d_v = dev(v)
    outs = []
    for _ in range(2):
        out = empty((1,), np.float64, fill=np.nan)
        call(lib.sb2_harmony_sum, h, n, ptr(d_v), ptr(out))
        outs.append(host(out)[0])
    assert abs(outs[0] - math.fsum(v)) <= sum_tol(np.abs(v).sum(), n) / 2
    assert outs[0].tobytes() == outs[1].tobytes()


# ------------------------------------------------------------------------------------------ k-means start
@pytest.mark.gpu
@pytest.mark.parametrize("with_closest", [False, True])
@pytest.mark.parametrize("d", [37, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_center_and_kpp_dists(dtype, d, with_closest):
    """xc = z - mean (one float64 rounding on each side, so equal bits) and xx = ||xc||² within 2(d + 1)ε₆₄·xx.  The
    D² of trials 1 to 8 candidates: xx + cc - 2 x·c, whose dot of d products is within 2(d + 1)ε₆₄·Σ|x_j c_j| ≤
    (d + 1)ε₆₄·(xx + cc) on each side, clipped at 0 and (with `closest`) taken as a minimum, both 1-Lipschitz; the
    potentials are float64 sums of those, to their error times n plus `sum_tol`.  n = 5003 is not a multiple of 256."""
    lib, h = _lib()
    rng = np.random.default_rng(60 + d)
    n = 5003
    z = unit_rows(rng, n, d, dtype)
    mean = z.astype(np.float64).mean(axis=0)
    xc, xx = empty((n, d), np.float64), empty((n,), np.float64)
    d_z, d_mean = dev(z), dev(mean)
    call(lib.sb2_harmony_center, h, n, d, is64(dtype), ptr(d_z), ptr(d_mean), ptr(xc), ptr(xx))
    want_xc, want_xx = center_ref(z, mean)
    np.testing.assert_array_equal(host(xc), want_xc)
    assert (np.abs(host(xx) - want_xx) <= 2 * (d + 1) * E64 * want_xx).all()
    closest = rng.uniform(0, 2, size=n) if with_closest else None
    d_closest = dev(closest)
    for trials in range(1, hm.MAX_TRIALS + 1):
        ids = rng.choice(n, size=trials, replace=False)
        dist, pot = empty((trials, n), np.float64, fill=np.nan), empty((trials,), np.float64, fill=np.nan)
        d_ids = dev(ids.astype(np.int64))
        call(lib.sb2_harmony_kpp_dists, h, n, d, ptr(xc), ptr(xx), trials, ptr(d_ids), ptr(d_closest), ptr(dist),
             ptr(pot))
        want_dist, want_pot = kpp_dists_ref(want_xc, want_xx, ids, closest)
        tol = 4 * (d + 2) * E64 * (want_xx[None, :] + want_xx[ids][:, None])
        err = np.abs(host(dist) - want_dist)
        assert (err <= tol).all(), (trials, err.max())
        assert (np.abs(host(pot) - want_pot) <= tol.sum(axis=1) + sum_tol(want_pot, n)).all(), trials


def _kpp_search(lib, h, v, u):
    ids = empty((len(u),), np.int64, fill=-1)
    d_v, d_u = dev(v), dev(u)
    call(lib.sb2_harmony_kpp_search, h, len(v), ptr(d_v), len(u), ptr(d_u), ptr(ids))
    return host(ids)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 1023, 1024, 1025, 4097, 1_000_003])
def test_kpp_search_is_exact(n):
    """Integer-valued v makes every prefix sum exact in float64, in the kernel's two-level order and in np.cumsum, so
    the candidate must be exactly np.searchsorted's: u on prefix boundaries, u = 0, u above the total, and runs of
    zeros that straddle the kernel's segments (ceil(n / 1024) values each)."""
    lib, h = _lib()
    rng = np.random.default_rng(70 + n)
    seg = -(-n // 1024)
    v = rng.integers(1, 5, size=n).astype(np.float64)
    for a in range(seg // 2, n, max(1, 7 * seg)):  # zero runs from the middle of one segment into the next ones
        v[a : a + 2 * seg + 1] = 0.0
    v[: min(n, seg + 1)] = 0.0  # a leading zero run: u = 0 must take index 0
    c = np.cumsum(v)
    pos = np.flatnonzero(v > 0)
    cases = [np.array([0.0, c[-1] + 1.0, c[-1], c[-1] / 2])]
    if len(pos):
        picks = rng.choice(pos, size=min(len(pos), 64), replace=False)
        cases += [c[picks], c[picks] - 0.5, c[np.maximum(picks - 1, 0)]]
    cases.append(rng.uniform(0, c[-1] + 1, size=64))
    every = np.concatenate(cases)
    for u in np.array_split(every, -(-len(every) // hm.MAX_TRIALS)):  # one CTA per uniform, up to 8 per launch
        u = np.ascontiguousarray(u, dtype=np.float64)
        np.testing.assert_array_equal(_kpp_search(lib, h, v, u), kpp_search_ref(v, u))


def _labels(lib, h, xc, centers, old):
    n, d = xc.shape
    labels = empty((n,), np.int32, fill=-7)
    changed = empty((1,), np.int32, fill=0)
    d_xc, d_centers, d_old = dev(xc), dev(centers), dev(old)
    call(lib.sb2_harmony_labels, h, n, d, len(centers), ptr(d_xc), ptr(d_centers), ptr(d_old), ptr(labels),
         ptr(changed))
    return host(labels), int(host(changed)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128])
@pytest.mark.parametrize("d", [50, 128])
def test_labels_are_exact(d, k):
    """The nearest centre, exactly: the data keep the best and second-best ||c||² - 2 x·c of every row 1e-6 apart, far
    beyond the 4(d + 1)ε₆₄ by which two orders of the dot can differ.  `changed` is 1 exactly when a label differs
    from `old`."""
    lib, h = _lib()
    rng = np.random.default_rng(80 + k + d)
    n = 3001
    centers = rng.normal(size=(k, d))
    xc = centers[rng.integers(0, k, size=n)] + 0.3 * rng.normal(size=(n, d))
    want, d2 = labels_ref(xc, centers)
    if k > 1:
        part = np.sort(d2, axis=1)
        assert (part[:, 1] - part[:, 0] > 1e-6).all()
    old = np.full(n, -1, dtype=np.int32)
    got, changed = _labels(lib, h, xc, centers, old)
    np.testing.assert_array_equal(got, want)
    assert changed == 1
    got, changed = _labels(lib, h, xc, centers, want)
    np.testing.assert_array_equal(got, want)
    assert changed == 0
    old = want.copy()
    old[n - 1] = (old[n - 1] + 1) % (k + 1)
    assert _labels(lib, h, xc, centers, old)[1] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("k", [33, 65, 128])
def test_labels_duplicated_centres_take_the_lowest_index(k):
    """Equal centres give equal distances bit for bit, so the lowest index must win: copies one lane apart (c, c + 1),
    one q apart (c, c + 32) and three q apart (c, c + 96), with the copy on either side."""
    lib, h = _lib()
    rng = np.random.default_rng(90 + k)
    d, n = 40, 4000
    centers = rng.normal(size=(k, d))
    for a, b in [(0, 1), (32, 3), (5, 37), (1, 97), (64, 2), (127, 31)]:
        if a < k and b < k:
            centers[b] = centers[a]
    xc = centers[rng.integers(0, k, size=n)] + 0.3 * rng.normal(size=(n, d))
    want, _ = labels_ref(xc, centers)
    got, _ = _labels(lib, h, xc, centers, np.full(n, -1, dtype=np.int32))
    np.testing.assert_array_equal(got, want)


# ------------------------------------------------------------------------------------------ apply
def _tuple_layout(rng, n, keys, n_codes):
    """Codes per cell over `keys` keys of n_codes // keys levels, with one tuple forced to 5,000 cells (three chunks)."""
    bounds = np.linspace(0, n_codes, keys + 1).astype(int)
    codes = np.column_stack([rng.integers(bounds[u], bounds[u + 1], size=n) for u in range(keys)])
    codes[: 5000] = codes[0]
    perm = rng.permutation(n)
    codes = codes[perm]
    return codes.astype(np.int32), *_tuples(codes)


@pytest.mark.gpu
@pytest.mark.parametrize("keys", [1, 2, 3])
@pytest.mark.parametrize(("k", "d", "n_codes"), [(40, 70, 9), (100, 100, 20), (128, 128, 128)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_apply(dtype, k, d, n_codes, keys):
    """z_hat = x - Σ_c r_c·Σ_keys W[c, code + 1] per code tuple: float64 sums of k products of the stored r and W,
    within `sum_tol` over k, then one store in T (ε_T·|z_hat|).  The normalised copy: z_hat's stores (ε_T each)
    move its norm by ε_T·||z_hat|| at most, and the division and its store add 2ε_T, so it is within
    4ε_T·|out| + (Δz_hat_j + ||Δz_hat||) / ||z_hat||.  A tuple of 5,000 cells spans three chunks."""
    lib, h = _lib()
    rng = np.random.default_rng(100 + k + keys)
    n = 9000
    codes, gcodes, order, gb = _tuple_layout(rng, n, keys, n_codes)
    x = (rng.normal(size=(n, d)) * 5).astype(dtype)
    r = rng.dirichlet(np.ones(k), size=n).astype(dtype)
    w = rng.normal(size=(k, n_codes + 1, d))
    zhat, znorm = empty((n, d), dtype, fill=np.nan), empty((n, d), dtype, fill=np.nan)
    b = np.ascontiguousarray(gb, dtype=np.int64)
    d_order, d_gcodes, d_w, d_x, d_r = dev(order.astype(np.int64)), dev(gcodes.astype(np.int32)), dev(w), dev(x), dev(r)
    call(lib.sb2_harmony_apply, h, len(gcodes), ptr(b), ptr(d_order), d, k, is64(dtype), keys, ptr(d_gcodes),
         n_codes, ptr(d_w), ptr(d_x), ptr(d_r), ptr(zhat), ptr(znorm))
    want, mag = apply_ref(gb, order, gcodes, w, x, r)
    eps = EPS[dtype]
    tol = sum_tol(mag, k) + eps * np.abs(want)
    err = np.abs(host(zhat) - want)
    assert (err <= tol).all(), err.max()
    nrm = np.linalg.norm(want, axis=1, keepdims=True)
    want_n = want / nrm
    tol_n = 4 * eps * np.abs(want_n) + (tol + np.linalg.norm(tol, axis=1, keepdims=True)) / nrm
    err = np.abs(host(znorm) - want_n)
    assert (err <= tol_n).all(), err.max()

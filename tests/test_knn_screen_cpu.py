"""CPU restatement of the kNN tile screen's arithmetic (knn_tc2.cu / knn.cu): the kd order's segments and its radix
select, the bound u(q) >= d_k(q) from the short sweep's proposals, the starting threshold it seeds, the screen's fp32
skip test with its margins, and the re-score's check d_k <= u.  The scores are perturbed anywhere inside the fp16
tier's rounding bound (knn_tc2_error_coefs), adversarially towards skipping, and every skip must still be right in
float64."""
import numpy as np
import pytest

CN = 128
U24 = 2.0 ** -24


def segments(n):
    """knn_tc2_kd_order's levels: [a, b) splits at a + 128 * floor(tiles / 2) while it holds more than one tile"""
    levels, cur = [], [(0, n)]
    while True:
        lv, nxt = [], []
        for a, b in cur:
            if b - a <= CN:
                continue
            m = a + CN * (((b - a + CN - 1) // CN) // 2)
            lv.append((a, m, b))
            nxt += [(a, m), (m, b)]
        if not lv:
            return levels
        levels.append(lv)
        cur = nxt


@pytest.mark.parametrize("n", [1, 128, 129, 300, 5000, 70_001, 1_300_000])
def test_kd_segments_end_in_single_tiles(n):
    levels = segments(n)
    leaves = [(0, n)]
    for lv in levels:
        split = {(a, b): m for a, m, b in lv}
        leaves = [x for a, b in leaves for x in (((a, split[(a, b)]), (split[(a, b)], b)) if (a, b) in split else ((a, b),))]
        for a, m, b in lv:
            assert a % CN == 0 and m % CN == 0 and a < m < b
    assert leaves == [(t * CN, min(n, t * CN + CN)) for t in range((n + CN - 1) // CN)]
    assert len(levels) == (0 if n <= CN else int(np.ceil(np.log2((n + CN - 1) // CN))))


def ord_bits(x):
    u = np.asarray(x, np.float32).view(np.uint32)
    return np.where(u & 0x80000000, u ^ np.uint32(0xFFFFFFFF), u ^ np.uint32(0x80000000)).astype(np.uint32)


def test_ord_bits_orders_like_floats():
    rs = np.random.RandomState(0)
    x = np.concatenate([rs.standard_normal(5000) * 10.0 ** rs.randint(-30, 30, 5000), [0.0, -np.inf, np.inf, 1e-45, -1e-45]])
    x = x.astype(np.float32)
    o = np.argsort(x, kind="stable")
    assert np.all(np.diff(ord_bits(x[o]).astype(np.int64)) >= 0)


def split(keys, P, need_left):
    """kd_split_kernel: 4-pass radix select of the pivot, then the stable partition"""
    prefix, rank = 0, need_left - 1
    for byte in (3, 2, 1, 0):
        hmask = 0 if byte == 3 else (0xFFFFFFFF << (8 * (byte + 1))) & 0xFFFFFFFF
        sel = keys[(keys & hmask) == prefix]
        hist = np.bincount((sel >> (8 * byte)) & 255, minlength=256)
        bin_ = 0
        while bin_ < 255 and rank >= hist[bin_]:
            rank -= hist[bin_]
            bin_ += 1
        prefix |= bin_ << (8 * byte)
    eq = keys == prefix
    eq_rank = np.cumsum(eq) - eq
    left = (keys < prefix) | (eq & (eq_rank < rank + 1))
    return np.concatenate([P[left], P[~left]]), left.sum()


@pytest.mark.parametrize("seed", range(6))
def test_radix_select_partition_is_a_stable_sort_split(seed):
    rs = np.random.RandomState(seed)
    n = rs.randint(129, 3000)
    v = rs.standard_normal(n).astype(np.float32)
    v[rs.randint(0, n, n // 3)] = v[0]          # many exact ties
    keys = ord_bits(v)
    need = CN * (((n + CN - 1) // CN) // 2)
    P = rs.permutation(n).astype(np.int64)
    out, nl = split(keys, P, need)
    assert nl == need
    order = np.argsort(keys, kind="stable")     # ties in position order
    assert set(out[:need]) == set(P[order[:need]])
    # both halves keep position order
    pos = {p: i for i, p in enumerate(P)}
    assert all(np.diff([pos[p] for p in out[:need]]) > 0) and all(np.diff([pos[p] for p in out[need:]]) > 0)


def coefs(kpad):
    acc = 1.6 * kpad * U24
    return acc, acc + 8.0 * U24      # c_q, c_n (fp16 operands)


def scale(R):
    e = int(np.floor(np.log2(np.float32(200.0) / np.float32(R))))
    return 2.0 ** max(-60, min(60, e))


def f32_ru(x):
    f = np.float32(x)
    return f if float(f) >= x else np.nextafter(f, np.float32(np.inf))


def f32_rd(x):
    f = np.float32(x)
    return f if float(f) <= x else np.nextafter(f, np.float32(-np.inf))


def _cloud(seed, n=2048, d=50, offset=0.0, labels=False):
    rs = np.random.RandomState(seed)
    c = 3.0 * rs.standard_normal((8, d))
    lab = rs.randint(0, 8, n)
    x = (c[lab] + rs.standard_normal((n, d)) + offset).astype(np.float32)
    return (x, lab) if labels else x


@pytest.mark.parametrize("seed,offset", [(0, 0.0), (1, 0.0), (2, 30.0)])
def test_row_bound_and_seed(seed, offset):
    x = _cloud(seed, offset=offset)
    xd = x.astype(np.float64)
    n, d = x.shape
    kpad = 64
    c_q, c_n = coefs(kpad)
    R = np.sqrt((xd ** 2).sum(1).max())
    s = scale(R * R)
    s2inv = 1.0 / (s * s)
    xs = x * np.float32(s)
    dn = np.sqrt(((xs.astype(np.float64) - xs.astype(np.float16).astype(np.float64)) ** 2).sum(1)) / s
    dmax = dn.max()
    rs = np.random.RandomState(seed + 10)
    k = 15
    for q in rs.choice(n, 40, replace=False):
        qn = (xd[q] ** 2).sum()
        cand = rs.choice(n, 1024, replace=False)
        cand[0] = q
        true = xd[cand] @ xd[q] - 0.5 * (xd[cand] ** 2).sum(1)
        eps = c_n * 0.5 * R * R + c_q * np.sqrt(qn) * R + dn[q] * R * (1 + 1e-6) + (np.sqrt(qn) + dn[q]) * dmax * (1 + 1e-6)
        comp = (true + rs.uniform(-1, 1, true.shape) * eps) / s2inv      # scaled units, anywhere inside the bound
        comp = comp.astype(np.float32)
        sk = np.sort(comp)[::-1][k - 1]
        u2 = qn - 2.0 * (float(sk) * s2inv - eps)
        u = f32_ru(np.sqrt(max(u2, 0.0)) * (1 + 1e-7))
        d2 = ((xd[cand] - xd[q]) ** 2).sum(1)
        assert np.sort(d2)[k - 1] <= float(u) ** 2                        # u bounds the k-th distance of the candidates
        sdd = ((qn - float(u) ** 2) * 0.5 - eps) / s2inv
        seed_ = f32_rd(sdd - abs(sdd) * 1e-6)
        within = d2 <= float(u) ** 2
        assert np.all(comp[within] >= seed_)                             # every point within u scores above the seed


@pytest.mark.parametrize("seed,offset", [(3, 0.0), (4, 0.0), (5, 25.0)])
def test_screen_skips_only_far_tiles(seed, offset):
    x, lab = _cloud(seed, n=4096, d=50, offset=offset, labels=True)
    xd = x.astype(np.float64)
    n, d = x.shape
    kpad = 64
    c_q, c_n = coefs(kpad)
    R = np.sqrt((xd ** 2).sum(1).max())
    s = scale(R * R)
    s32 = np.float32(s)
    order = np.lexsort((xd[:, 0], lab))        # tiles inside one cluster; the bound itself assumes nothing about them
    tiles = [order[t * CN:(t + 1) * CN] for t in range(n // CN)]
    # kd_tile_stats_kernel: fp16-exact centres in the scaled units, radii rounded up
    mu = np.stack([(np.float32(xd[t].mean(0).astype(np.float32) * s32).astype(np.float16).astype(np.float32) / s32) for t in tiles])
    rad = np.array([f32_ru(np.sqrt(((xd[t] - mu[i].astype(np.float64)) ** 2).sum(1).max()) * (1 + 1e-12)) for i, t in enumerate(tiles)],
                   np.float32)
    xs = x * s32
    dn = np.sqrt(((xs.astype(np.float64) - xs.astype(np.float16).astype(np.float64)) ** 2).sum(1)) / s
    rs = np.random.RandomState(seed)
    C = np.float32(1.0 + 1.0 / 65536.0)
    skips = 0
    for q in rs.choice(n, 64, replace=False):
        qn = (xd[q] ** 2).sum()
        qnorm = np.sqrt(qn)
        eps_c = c_n * 0.5 * R * R + c_q * qnorm * R + dn[q] * R * (1 + 1e-6)
        slack = 2.0 ** -19 * (qnorm + R) ** 2
        qlb = f32_rd((qn - 2.0 * eps_c - slack) * s * s)
        d2q = ((xd - xd[q]) ** 2).sum(1)
        u = f32_ru(np.sqrt(np.sort(d2q)[14]) * rs.uniform(1.0, 1.5))   # any u >= d_k
        us = np.float32(u) * s32
        mu64 = mu.astype(np.float64)
        true = (mu64 @ xd[q] - 0.5 * (mu64 ** 2).sum(1)) * s * s
        for sign in (-1.0, 1.0):     # -1: the computed scores err towards skipping
            acc = (true + sign * eps_c * s * s).astype(np.float32)
            D2 = (np.float64(-2.0) * acc.astype(np.float64) + np.float64(qlb)).astype(np.float32)   # fmaf: one rounding
            t = us + rad * s32
            skip = D2 > (t * t) * C
            for i in np.flatnonzero(skip):
                assert d2q[tiles[i]].min() > float(u) ** 2
                # the re-score's check: kth <= u^2 (1 - 1e-9) while fp64 keys of skipped points are >= d^2 (1 - 2e-13)
                assert d2q[tiles[i]].min() * (1 - 2e-13) > float(u) ** 2 * (1 - 1e-9)
            skips += int(skip.sum())
    if offset == 0.0:
        assert skips > 0      # the test exercises the skip branch

"""CPU restatement of the kd order's split rule and of its many-CTA split (knn_tc2.cu): kd_dir_kernel's direction (power
iterations on the centred sample's scatter from the coordinate of largest variance, the largest |v_j| made positive), the
keys ord_bits(fp32(x . v - mu . v)), and kd_wide_*: per-chunk counts, the per-segment scan and the chunked partition
give the permutation of the one-CTA split."""
import numpy as np
import pytest

CN = 128
POWER_ITERS = 12
CHUNK = 4096


def ord_bits(x):
    u = np.asarray(x, np.float32).view(np.uint32)
    return np.where(u & 0x80000000, u ^ np.uint32(0xFFFFFFFF), u ^ np.uint32(0x80000000)).astype(np.uint32)


def direction(s):
    """kd_dir_kernel on the sample s [ns, d]: (v, mu . v)"""
    s = s.astype(np.float64)
    mu = s.mean(0)
    c = s - mu
    v = np.zeros(s.shape[1])
    v[np.argmax((c * c).sum(0))] = 1.0
    for _ in range(POWER_ITERS):
        u = c.T @ (c @ v)
        nrm = np.sqrt(u @ u)
        if not (nrm > 0.0 and np.isfinite(nrm)):
            break
        v = u / nrm
    if v[np.argmax(np.abs(v))] < 0:
        v = -v
    return v, mu @ v


def keys(x, v, off):
    return ord_bits((x.astype(np.float64) @ v - off).astype(np.float32))


@pytest.mark.parametrize("seed", range(4))
def test_direction_reaches_the_top_eigenvector(seed):
    rs = np.random.RandomState(seed)
    d = 50
    scales = np.concatenate([[8.0, 4.0], rs.uniform(0.5, 2.0, d - 2)])
    q, _ = np.linalg.qr(rs.standard_normal((d, d)))
    s = (rs.standard_normal((512, d)) * scales) @ q.T + 5.0 * rs.standard_normal(d)
    v, off = direction(s.astype(np.float32))
    c = s.astype(np.float32).astype(np.float64)
    c -= c.mean(0)
    w = np.linalg.eigvalsh(c.T @ c)
    assert w[-1] > 2.0 * w[-2]                      # a clear gap
    assert abs(v @ (c.T @ (c @ v)) - w[-1]) <= 1e-6 * w[-1]
    assert abs(np.linalg.norm(v) - 1.0) < 1e-12
    assert v[np.argmax(np.abs(v))] > 0              # the sign rule


def test_direction_without_spread_keeps_the_start_coordinate():
    s = np.tile(np.arange(7, dtype=np.float32), (40, 1))
    v, off = direction(s)
    assert np.array_equal(v, np.eye(7)[0]) and off == 0.0


def test_keys_order_like_the_centred_projections():
    rs = np.random.RandomState(1)
    x = (rs.standard_normal((3000, 20)) + 100.0).astype(np.float32)   # far from the origin: the offset keeps resolution
    v, off = direction(x[:: 6])
    k = keys(x, v, off)
    p = x.astype(np.float64) @ v - off
    o = np.argsort(k, kind="stable")
    assert np.all(np.diff(p[o]) >= -1e-5 * np.abs(p).max())
    assert len(np.unique(k)) > 0.95 * len(k)       # without the offset, fp32 keys near 700 would tie far more often


def select(keys, need_left):
    """the 4-pass radix select: the pivot and how many keys equal to it go left"""
    prefix, rank = 0, need_left - 1
    for byte in (3, 2, 1, 0):
        hmask = 0 if byte == 3 else (0xFFFFFFFF << (8 * (byte + 1))) & 0xFFFFFFFF
        hist = np.bincount((keys[(keys & hmask) == prefix] >> (8 * byte)) & 255, minlength=256)
        b = 0
        while b < 255 and rank >= hist[b]:
            rank -= hist[b]
            b += 1
        prefix |= b << (8 * byte)
    return prefix, rank + 1


def split_one(keys, P, need_left):
    pivot, eq_take = select(keys, need_left)
    eq = keys == pivot
    left = (keys < pivot) | (eq & (np.cumsum(eq) - eq < eq_take))
    return np.concatenate([P[left], P[~left]])


def split_wide(keys, P, need_left):
    """kd_wide_count / kd_wide_scan / kd_wide_scatter: chunks of CHUNK keys, each placed from its scanned offsets"""
    pivot, eq_take = select(keys, need_left)
    out = np.empty_like(P)
    eq_before = left_before = 0
    for lo in range(0, len(keys), CHUNK):
        k, p = keys[lo:lo + CHUNK], P[lo:lo + CHUNK]
        eq = k == pivot
        left = (k < pivot) | (eq & (eq_before + np.cumsum(eq) - eq < eq_take))
        nl = int(left.sum())
        out[left_before:left_before + nl] = p[left]
        right0 = need_left + (lo - left_before)
        out[right0:right0 + len(k) - nl] = p[~left]
        left_before += int((k < pivot).sum()) + max(0, min(int(eq.sum()), eq_take - eq_before))
        eq_before += int(eq.sum())
    return out


@pytest.mark.parametrize("seed", range(5))
def test_chunked_partition_matches_the_one_cta_split(seed):
    rs = np.random.RandomState(seed)
    n = rs.randint(CHUNK + 1, 6 * CHUNK)
    v = rs.standard_normal(n).astype(np.float32)
    v[rs.randint(0, n, n // 2)] = v[rs.randint(n)]      # a flood of ties that straddles chunks
    k = ord_bits(v)
    P = rs.permutation(n)
    need = CN * (((n + CN - 1) // CN) // 2)
    assert np.array_equal(split_wide(k, P, need), split_one(k, P, need))

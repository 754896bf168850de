"""The exact-kNN certificate rests on rounding bounds for the tensor-core scores (scanpy_b200/csrc/knn_tc2.cu:
`knn_tc2_error_coefs`, `knn_tc2_prep_kernel`; scanpy_b200/csrc/knn.cu: `knn_rescore_kernel`).  This CPU test restates
the operand formats in numpy, emulates a PESSIMISTIC tensor pipe (exact fp16 x fp16 products, every 16-product
group and every accumulator update truncated towards zero to fp32) and checks that the bounds the kernels use hold
for every (query, candidate) pair tried - including data far from the origin, tiny and huge scales, sub-normal
halves and d up to the 150 the library accepts.  No GPU, no library call: it pins the arithmetic of the proof."""
import numpy as np
import pytest

U24 = 2.0 ** -24


def _trunc32(v):
    """float64 -> float32, rounded towards zero (worst case for a truncating accumulator)."""
    f = v.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(v)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def _scale(max_norm):
    # tc_scale_from_maxnorm: power of two s with s * R in [100, 200)
    if not np.isfinite(max_norm) or max_norm <= 0:
        return 1.0
    return float(2.0 ** np.clip(np.floor(np.log2(200.0 / max_norm)), -60, 60))


def _images(x, terms):
    """-> (A, B) fp16 operand rows on the concatenated K axis, scale s, per-point residual norms (units of x)."""
    n, d = x.shape
    r = float(np.sqrt((x.astype(np.float64) ** 2).sum(1).max()))
    s = _scale(np.float32(r))
    xs = (x * np.float32(s)).astype(np.float32)
    hi = xs.astype(np.float16)
    lo = (xs - hi.astype(np.float32)).astype(np.float16)
    hn = -0.5 * (xs.astype(np.float64) ** 2).sum(1)
    h0 = hn.astype(np.float32).astype(np.float16)
    r1 = hn - h0.astype(np.float64)
    h1 = r1.astype(np.float32).astype(np.float16)
    h2 = (r1 - h1.astype(np.float64)).astype(np.float32).astype(np.float16)
    ones = np.ones((n, 3), np.float16)
    hs = np.stack([h0, h1, h2], 1)
    if terms == 1:
        a, b = np.hstack([hi, ones]), np.hstack([hi, hs])
    else:
        a, b = np.hstack([hi, hi, lo, ones]), np.hstack([hi, lo, hi, hs])
    k = a.shape[1]
    kpad = -(-k // 16) * 16
    a = np.pad(a, ((0, 0), (0, kpad - k)))
    b = np.pad(b, ((0, 0), (0, kpad - k)))
    dnorm = np.sqrt(((xs.astype(np.float64) - hi.astype(np.float64)) ** 2).sum(1)) * (1 + 1e-12) / s
    return a, b, s, dnorm, kpad, r


def _tensor_pipe(a_rows, b_rows):
    """scores[i, j] = sum_k a[i,k] b[j,k]: exact products, truncated 16-product group sums, truncated fp32 updates."""
    a = a_rows.astype(np.float64)
    b = b_rows.astype(np.float64)
    acc = np.zeros((a.shape[0], b.shape[0]), np.float32)
    for k0 in range(0, a.shape[1], 16):
        grp = _trunc32(a[:, k0:k0 + 16] @ b[:, k0:k0 + 16].T)
        acc = _trunc32(acc.astype(np.float64) + grp.astype(np.float64))
    return acc.astype(np.float64)


def _cases():
    rs = np.random.RandomState(0)
    yield "pca-like d=50", rs.standard_normal((400, 50)).astype(np.float32) * (0.97 ** np.arange(50)).astype(np.float32) * 3
    yield "far from origin", (rs.standard_normal((300, 24)) * 0.05 + 40.0).astype(np.float32)
    yield "tiny scale", (rs.standard_normal((300, 10)) * 1e-20).astype(np.float32)
    yield "huge scale", (rs.standard_normal((300, 10)) * 1e15).astype(np.float32)
    x = rs.standard_normal((300, 150)).astype(np.float32)
    x[:100] *= 1e-4   # many sub-normal halves after scaling
    x[0] = 0
    yield "d=150 mixed magnitudes", x
    yield "one dimension", rs.standard_normal((200, 1)).astype(np.float32)
    y = rs.standard_normal((256, 33)).astype(np.float32)
    y[:, 0] += 1000.0
    yield "offset in one coordinate", y


@pytest.mark.parametrize("terms", [1, 3])
def test_score_error_bounds_hold(terms):
    for name, x in _cases():
        a, b, s, dnorm, kpad, r = _images(x, terms)
        if not (9801.0 <= (r * s) ** 2 <= 67600.0):
            # knn_rescore_kernel refuses to certify outside the scaled-norm regime the bounds are derived for
            # (the power-of-two scale is clamped to 2^+-60): such data goes to the exact scan
            assert name in ("tiny scale",), name
            continue
        q = np.arange(0, x.shape[0], 3)
        got = _tensor_pipe(a[q], b) / (s * s)                        # what the kernel's score * inv_s2 is
        x64 = x.astype(np.float64)
        true = x64[q] @ x64.T - 0.5 * (x64 ** 2).sum(1)[None, :]     # s(q,c) = q.c - |c|^2 / 2
        qn = np.sqrt((x64[q] ** 2).sum(1))
        acc = 1.6 * kpad * U24                                       # knn_tc_error_coefs
        c_n = acc + 8.0 * U24
        c_q = acc + (8.0 * U24 if terms == 3 else 0.0)
        eps = c_n * 0.5 * r * r + c_q * qn * r                       # knn_rescore_kernel
        if terms == 1:
            dq, dc = dnorm[q], dnorm.max()
            eps = eps + (dq * r + (qn + dq) * dc) * (1 + 1e-6)
        err = np.abs(got - true).max(1)
        assert (err <= eps).all(), (name, terms, float((err / np.maximum(eps, 1e-300)).max()))
        # the bound must also be worth something: within two orders of magnitude of the observed error for the
        # typical case (otherwise tier 1 could never certify a row)
        if name == "pca-like d=50":
            assert np.median(eps / np.maximum(err, 1e-300)) < 200, name


def test_certificate_logic_on_emulated_sweep():
    """End to end in numpy: proposals = top-32 by the emulated fp16 score, fp64 re-score, certificate
    kth_exact < |q|^2 - 2 (tau + eps); every certified row must equal the brute-force answer."""
    rs = np.random.RandomState(1)
    c = rs.standard_normal((6, 20)) * 4
    x = (c[rs.randint(0, 6, 700)] + rs.standard_normal((700, 20))).astype(np.float32)
    x[50:60] = x[49]  # a block of exact duplicates
    k, lm = 15, 32
    a, b, s, dnorm, kpad, r = _images(x, 1)
    scores = _tensor_pipe(a, b) / (s * s)
    x64 = x.astype(np.float64)
    d2 = ((x64[:, None, :] - x64[None, :, :]) ** 2).sum(-1)
    qn2 = (x64 ** 2).sum(1)
    n_cert = 0
    for i in range(x.shape[0]):
        prop = np.argsort(-scores[i], kind="stable")[:lm]
        tau = scores[i, prop].min()
        key = d2[i, prop].copy()
        key[prop == i] = -1.0
        order = np.lexsort((prop, key))
        top = prop[order][:k]
        kth = np.sort(key)[k - 1]
        qn = np.sqrt(qn2[i])
        eps = (1.6 * kpad + 8) * U24 * 0.5 * r * r + 1.6 * kpad * U24 * qn * r + (dnorm[i] * r + (qn + dnorm[i]) * dnorm.max()) * (1 + 1e-6)
        certified = top[0] == i and kth < qn2[i] - 2.0 * (tau + eps)
        if certified:
            n_cert += 1
            ref = np.lexsort((np.arange(x.shape[0]), np.where(np.arange(x.shape[0]) == i, -1.0, d2[i])))[:k]
            assert set(ref.tolist()) == set(top.tolist()), i
    assert n_cert > 0.9 * (x.shape[0] - 11)   # all but the duplicate block certify on this data

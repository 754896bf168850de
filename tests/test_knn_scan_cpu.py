"""The fast path of the tensor-core kNN sweep's examination (scanpy_b200/csrc/knn_tc2.cu: `chunk_imax`) asks "does any of
a chunk's 32 scores beat tau" on the raw bit patterns: signed-integer maximum of the patterns against tau's pattern.
This CPU test restates that test and its dispatch rule in numpy and checks the argument the kernel rests on: the integer
test equals the float test whenever tau's sign bit is clear, and every tau with the sign bit set (all tau < 0, and -0.0)
is sent to the float test.  No GPU, no library call."""
import numpy as np
import pytest

PAD = np.float32(-60000.0)          # score of a padding candidate
TINY = np.float32(1e-45)            # smallest sub-normal
SPECIAL = np.array([0.0, -0.0, TINY, -TINY, 1.1754942e-38, -1.1754942e-38, 1.17549435e-38, 1.0, -1.0, 3.4028235e38,
                    -3.4028235e38, PAD, 65504.0, 12.7, -12.7], dtype=np.float32)


def bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


def float_hit(v, tau):
    """chunk_max(v) > tau"""
    return bool(np.max(v) > np.float32(tau))


def chunk_imax(v):
    """the kernel's ternary tree over the 32 patterns: ten triples, three triples of those, (a9, v30, v31), the rest"""
    p = [int(b) for b in bits(v)]
    a = [max(p[3 * i], p[3 * i + 1], p[3 * i + 2]) for i in range(10)]
    b = [max(a[0], a[1], a[2]), max(a[3], a[4], a[5]), max(a[6], a[7], a[8]), max(a[9], p[30], p[31])]
    return max(max(b[0], b[1], b[2]), b[3])


def int_hit(v, tau):
    """chunk_imax(v) > __float_as_int(tau)"""
    return chunk_imax(v) > int(bits(tau))


def takes_float_path(tau0, tau1):
    """a thread holds two rows; one OR and one sign test decide for both"""
    return (int(bits(tau0)) | int(bits(tau1))) < 0


def _chunks(rs):
    """random and adversarial chunks of 32 finite float32 scores"""
    out = []
    for scale in (1e-40, 1e-3, 1.0, 300.0, 3e4):
        out.append((scale * rs.standard_normal(32)).astype(np.float32))                    # mixed signs
        out.append(-np.abs(scale * rs.standard_normal(32)).astype(np.float32))             # all negative
        out.append(np.abs(scale * rs.standard_normal(32)).astype(np.float32))              # all positive
    out.append(np.full(32, PAD))                                                           # a tile of padding
    out.append(np.full(32, np.float32(-0.0)))
    out.append(np.zeros(32, np.float32))
    for _ in range(40):
        v = rs.choice(SPECIAL, 32)
        out.append(v)
        w = (100.0 * rs.standard_normal(32)).astype(np.float32)
        w[rs.randint(0, 32, 6)] = rs.choice(SPECIAL, 6)
        w[rs.randint(0, 32, 3)] = PAD
        out.append(w)
    return out


def _taus(v, rs):
    """thresholds around every value of the chunk, the special values and both infinities"""
    with np.errstate(over="ignore"):     # the step up from the largest finite float is +inf
        near = np.concatenate([v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))])
    rnd = (50.0 * rs.standard_normal(8)).astype(np.float32)
    return np.concatenate([near, SPECIAL, rnd, np.array([np.inf, -np.inf], np.float32)]).astype(np.float32)


def test_tree_is_the_maximum_of_all_32_patterns():
    rs = np.random.RandomState(0)
    for v in _chunks(rs):
        assert chunk_imax(v) == int(bits(v).max())
    for i in range(32):          # every position reaches the root
        v = np.full(32, PAD)
        v[i] = np.float32(1.0)
        assert chunk_imax(v) == int(bits(np.float32(1.0)))


def test_integer_test_equals_float_test_when_sign_bit_of_tau_is_clear():
    rs = np.random.RandomState(1)
    n = 0
    for v in _chunks(rs):
        for tau in _taus(v, rs):
            if int(bits(tau)) >= 0:      # +0, sub-normals, every positive float, +inf
                assert int_hit(v, tau) == float_hit(v, tau), (v, tau)
                n += 1
    assert n > 5000


@pytest.mark.parametrize("tau", [0.0, TINY, np.inf])
def test_edge_thresholds(tau):
    tau = np.float32(tau)
    neg = np.array([-0.0, -TINY, -1.0, PAD] * 8, np.float32)
    assert not int_hit(neg, tau) and not float_hit(neg, tau)          # nothing negative (or -0) beats tau >= +0
    big = neg.copy()
    big[17] = np.float32(3.4028235e38)
    assert int_hit(big, tau) == float_hit(big, tau) == bool(np.isfinite(tau))   # +inf (rows past n_query) never hits
    eq = neg.copy()
    eq[5] = tau
    assert not int_hit(eq, tau) and not float_hit(eq, tau)            # a score equal to tau is not a hit


def test_every_negative_threshold_takes_the_float_path():
    rs = np.random.RandomState(2)
    pos = np.float32(12.7)
    for tau in np.concatenate([-np.abs(_taus((30.0 * rs.standard_normal(32)).astype(np.float32), rs)),
                               np.array([-np.inf, -TINY, -0.0], np.float32)]):
        if tau < 0 or np.signbit(tau):
            assert takes_float_path(tau, pos) and takes_float_path(pos, tau) and takes_float_path(tau, tau)
    for tau in (np.float32(0.0), TINY, pos, np.float32(np.inf)):
        assert not takes_float_path(tau, pos) and not takes_float_path(pos, tau)


def test_integer_test_is_wrong_for_negative_thresholds():
    # why the rule exists: among negative floats the patterns order the other way round, and -0.0 is INT_MIN
    v = np.full(32, np.float32(-5.0))
    assert float_hit(v, -7.0) and not int_hit(v, -7.0)               # a missed hit
    assert float_hit(v, -np.inf) and not int_hit(v, -np.inf)         # also at a cold start's -inf
    assert not float_hit(v, -3.0) and int_hit(v, -3.0)               # a false hit
    assert not float_hit(np.full(32, np.float32(-1.0)), -0.0) and int_hit(np.full(32, np.float32(-1.0)), -0.0)

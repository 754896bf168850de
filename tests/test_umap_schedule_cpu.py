"""The host restatement of the device UMAP layout (oracle/umap_schedule.py), checked without a GPU:

* the kernel's closed-form sampling schedule against umap's running counters (oracle.graph_tools._optimize's
  bookkeeping), arc by arc and epoch by epoch;
* the comparison tolerance of tests/test_gpu_umap_exact.py rejects a kernel that is wrong in any of the ways that barely
  change layout quality: one pull per sampled arc instead of two, one negative sample too many or too few, the old
  rounding of the negative count, the alpha of the next epoch, pruning with too small an epoch count, or Gauss-Seidel
  reads of the other end points - on every case that test runs;
* the rescale, the seed mix and the epoch-0 identity the GPU tests build on.
"""
import numpy as np
import pytest

import umap_exact_cases as uc
from oracle import umap_schedule as us

A, B = uc.A, uc.B

# on random weights, schedule mismatches are boundary rounding (fp32 wmax / w against umap's fp64 n_epochs / n_samples,
# and the drift of the running `+= eps`); they stay under this share of all (arc, epoch) samples
MISMATCH_RATE = 1e-4


N_DIV = 1000  # the first N_DIV weights are exact divisors of wmax


@pytest.fixture(scope="module")
def weights():
    rng = np.random.default_rng(0)
    w = rng.random(20000).astype(np.float32)
    # exact divisors of wmax = 1: sampled every 1, 2, 3, 5, 10 epochs
    w[:N_DIV] = np.tile(np.array([1, 1 / 2, 1 / 3, 1 / 5, 1 / 10], np.float32), N_DIV // 5)
    return w


@pytest.mark.parametrize("rate", [1, 5, 7])
@pytest.mark.parametrize("n_epochs", [11, 50, 200, 500])
def test_closed_form_schedule_matches_running_counters(weights, n_epochs, rate):
    prune = us.prune_epochs_for(len(weights), n_epochs)
    eps32 = us.epochs_per_sample(weights, len(weights), n_epochs)
    eps64 = us.umap_epochs_per_sample(weights, n_epochs, prune)
    np.testing.assert_array_equal(eps32 > 0, eps64 > 0)  # same arcs pruned
    s_k, n_k = us.closed_form_schedule(eps32, n_epochs, rate)
    s_u, n_u = us.running_counter_schedule(eps64, n_epochs, float(rate))
    # per arc, the same number of samples up to one and the same number of negatives up to one sample's worth
    assert np.abs(s_k.sum(1).astype(int) - s_u.sum(1)).max() <= 1
    assert np.abs(n_k.sum(1) - n_u.sum(1)).max() <= rate
    # random weights: mismatches are rare, and not a bias (as many samples early as late)
    sk, sn, uk, un = s_k[N_DIV:], n_k[N_DIV:], s_u[N_DIV:], n_u[N_DIV:]
    total = int(uk.sum())
    miss_s = int((sk != uk).sum())
    miss_n = int((sn[sk & uk] != un[sk & uk]).sum())
    print(f"n_epochs={n_epochs} rate={rate}: {total} samples of random-weight arcs, {miss_s} sample and {miss_n} "
          f"negative-count mismatches")
    assert miss_s <= MISMATCH_RATE * total and miss_n <= MISMATCH_RATE * total
    early, late = int((sk & ~uk).sum()), int((uk & ~sk).sum())
    assert abs(early - late) <= max(2, 0.2 * miss_s)
    # exact divisors: the kernel keeps the exact rational schedule - a sample every `period` epochs, rate - 1
    # negatives at the first and rate at every later one.  umap's counters agree on the samples; their running
    # `+= eps / rate` can lose a negative to rounding (e.g. eps = 5, rate = 7) and pay it back at a later sample.
    ep = np.arange(n_epochs)
    for r, period in enumerate([1, 2, 3, 5, 10]):
        want_s = (ep % period == 0) & (ep > 0)
        want_n = np.where(want_s, np.where(ep == period, rate - 1, rate), 0)
        for row in range(r, N_DIV, 5 * 40):
            np.testing.assert_array_equal(s_k[row], want_s)
            np.testing.assert_array_equal(s_u[row], want_s)
            np.testing.assert_array_equal(n_k[row], want_n)
            assert abs(int(n_u[row].sum()) - int(want_n.sum())) <= rate


def test_negative_count_clamp():
    # rate 70 on an arc sampled every epoch owes 69 negatives at its first sample and 70 later; the kernel clamps to 64
    # (a deliberate bound on per-arc work that umap does not have)
    s, nn = us.closed_form_schedule(np.array([1.0], np.float32), 5, 70)
    assert nn[0].tolist() == [0, 64, 64, 64, 64]
    _, nu = us.running_counter_schedule(np.array([1.0]), 5, 70.0)
    assert nu[0].tolist() == [0, 69, 70, 70, 70]


def test_seed_mix_and_rescale():
    assert us.seed_mix(0) == 12345
    assert us.seed_mix(1) == (2654435761 + 12345) & 0xFFFFFFFF
    # seeds past 2^32: the high word is folded in, not dropped
    assert us.seed_mix(2**32 + 1) == us.seed_mix(0) and us.seed_mix(2**32 + 2) != us.seed_mix(2)
    x = np.array([[1.0, 5.0, -2.0], [3.0, 5.0, 0.0], [2.0, 5.0, 6.0]], np.float32)
    r = us.rescale(x)
    assert r.dtype == np.float32
    np.testing.assert_array_equal(r[:, 0], [0.0, 10.0, 5.0])
    np.testing.assert_array_equal(r[:, 1], 0.0)  # a constant column maps to 0
    np.testing.assert_array_equal(r[:, 2], np.float32(10) * (x[:, 2] + 2) / np.float32(8))


def test_epoch_zero_samples_nothing():
    g = us.edge_case_graph(300, seed=1)
    init = np.random.default_rng(1).normal(size=(300, 2)).astype(np.float32)
    for dtype in (np.float32, np.float64):
        for ne in (0, 1):
            np.testing.assert_array_equal(us.umap_layout(g, init, n_epochs=ne, a=A, b=B, dtype=dtype),
                                          us.rescale(init, dtype))
    assert not np.array_equal(us.umap_layout(g, init, n_epochs=2, a=A, b=B), us.rescale(init, np.float64))


MUTATIONS = {
    "one pull per sampled arc": dict(pulls=1),
    "one negative sample too many": dict(neg_delta=1),
    "one negative sample too few": dict(neg_delta=-1),
    "negative count rounded as epoch * (rate / eps)": dict(rate_first=True),
    "alpha of the next epoch": dict(alpha_shift=1),
    "Gauss-Seidel reads across vertices": dict(gauss_seidel=True),
}


@pytest.mark.parametrize("case", uc.CASES, ids=uc.IDS)
def test_tolerance_rejects_each_mutation(case):
    """On every case of tests/test_gpu_umap_exact.py, each mutation either leaves the layout bit for bit unchanged (it
    cannot show in that case, e.g. no arc is sampled before epoch 1, or a count sits at 0 or at the clamp) or moves it by
    more than twice the tolerance."""
    kw = case["kw"]
    r64 = uc.restated(case)
    tol = us.tolerance(uc.restated(case, dtype=np.float32), r64)
    muts = dict(MUTATIONS)
    if kw["n_epochs"] >= 3:
        # pruning at an epoch count below n_epochs - 1 drops arcs that are due a sample; at n_epochs = 2 only the arcs of
        # weight wmax are ever sampled, so no pruning can change the layout there
        muts["pruning with too small an epoch count"] = dict(prune_epochs=(kw["n_epochs"] - 1) // 2)
    lines, silent = [], []
    for name, mut in muts.items():
        r = uc.restated(case, **mut)
        if np.array_equal(r, r64):
            silent.append(name)
            continue
        dev = float(np.abs(r - r64).max())
        lines.append(f"{name}: {dev / tol:.1f} x")
        assert dev > 2 * tol, (name, dev, tol)
    print(f"{case['id']}: tolerance {tol:.3g}; " + "; ".join(lines + [f"no effect: {', '.join(silent)}"] * bool(silent)))
    # the mutations that must show wherever an arc is sampled, and the negative counts wherever they are not 0 or clamped
    if kw["n_epochs"] >= 2:
        for name in ("one pull per sampled arc", "alpha of the next epoch", "Gauss-Seidel reads across vertices"):
            assert name not in silent, name
        if kw["negative_sample_rate"] not in (0, 70):
            assert "one negative sample too few" not in silent and "one negative sample too many" not in silent
    if kw["negative_sample_rate"] == 7 and kw["n_epochs"] > 45:
        assert "negative count rounded as epoch * (rate / eps)" not in silent


@pytest.mark.parametrize("n_epochs", [2, 3, 5, 10])
def test_pruning_at_the_epoch_count_changes_nothing(n_epochs):
    """For n_epochs <= 10 the kernel prunes at wmax / 500 (n <= 10000) or wmax / 200, umap's default epoch counts.
    Pruning at wmax / n_epochs instead gives the same layout bit for bit: an arc is first sampled in epoch ceil(eps),
    and any arc pruned at a count P >= n_epochs has eps > n_epochs, so it is never due within the run.  A wrong
    pruning count is only visible below n_epochs - 1 (test_tolerance_rejects_each_mutation)."""
    g = us.edge_case_graph(2000, seed=0, hub_degree=300)
    init = np.random.default_rng(2).normal(size=(2000, 2)).astype(np.float32)
    kw = dict(n_epochs=n_epochs, a=A, b=B, seed=7)
    assert (us.epochs_per_sample(g.data, 2000, n_epochs, n_epochs) != us.epochs_per_sample(g.data, 2000, n_epochs)).any()
    np.testing.assert_array_equal(us.umap_layout(g, init, prune_epochs=n_epochs, **kw), us.umap_layout(g, init, **kw))

"""The device UMAP layout (sb2_umap_layout_f32, csrc/umap.cu) coordinate by coordinate against the float64 host
restatement of its schedule (oracle/umap_schedule.py), on the cases of tests/umap_exact_cases.py.

The tolerance of each case is `oracle.umap_schedule.tolerance`: 16 times how far the same schedule in plain fp32 lands
from float64 (the device adds __powf and FMA contractions, roundings of the same size).  tests/test_umap_schedule_cpu.py
shows, on these same cases, that every mutation of the schedule that barely changes layout quality (one pull instead of
two, a negative sample more or less, the old rounding of the negative count, the next epoch's alpha, wrong pruning,
Gauss-Seidel reads) either changes nothing in that case or moves it by more than twice that tolerance.  Each case prints
its deviation; the module prints the worst.
"""
import numpy as np
import pytest

import umap_exact_cases as uc
from oracle import umap_schedule as us

pytestmark = pytest.mark.gpu

REPORT = []


@pytest.fixture(scope="module", autouse=True)
def _worst_case_report():
    yield
    if REPORT:
        name, err, tol, spread = max(REPORT, key=lambda r: r[1] / r[2])
        print(f"\nworst device-vs-float64 deviation: {err:.3g} = {err / tol:.3f} x tolerance "
              f"({err / max(spread, 1e-30):.2f} x the fp32 spread) in {name}; {len(REPORT)} cases")


def _device(case, **over):
    from scanpy_b200 import _ops

    kw = dict(case["kw"], **over)
    return _ops.umap_layout(uc.graph(case["graph"]), n_components=case["dim"], init=uc.init(case), a=uc.A, b=uc.B, **kw)


@pytest.mark.parametrize("case", uc.CASES, ids=uc.IDS)
def test_device_matches_float64_restatement(case):
    dev = _device(case)
    x0 = uc.init(case)
    assert dev.dtype == np.float32 and dev.shape == x0.shape and np.isfinite(dev).all()
    r64 = uc.restated(case)
    r32 = uc.restated(case, dtype=np.float32)
    spread = float(np.abs(r32 - r64).max())
    err = float(np.abs(dev - r64).max())
    tol = us.tolerance(r32, r64)
    REPORT.append((case["id"], err, tol, spread))
    print(f"{case['id']}: max |device - float64| {err:.3g}, fp32 spread {spread:.3g}, tolerance {tol:.3g} "
          f"({err / tol:.3f} x)")
    assert err <= tol, (case["id"], err, tol, spread)
    if case["kw"]["n_epochs"] <= 1:
        # epoch 0 samples no arc: the result is the fp32 rescale of the initialisation, bit for bit
        np.testing.assert_array_equal(dev, us.rescale(x0))
    if case["const_col"] is not None and case["kw"]["n_epochs"] <= 1:
        np.testing.assert_array_equal(dev[:, case["const_col"]], 0.0)


def test_seed_high_word_changes_the_negative_samples():
    case = next(c for c in uc.CASES if c["id"] == "seed=99")
    assert not np.array_equal(_device(case), _device(case, seed=2**32 + 99))


def test_identical_calls_are_bitwise_equal():
    case = next(c for c in uc.CASES if c["id"] == "big n_epochs=3")
    np.testing.assert_array_equal(_device(case, n_epochs=20), _device(case, n_epochs=20))

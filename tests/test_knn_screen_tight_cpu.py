"""CPU restatement of the tile screen's near lists (knn_tc2.cu, knn_near_lists_kernel): per query block the nt
consecutive tiles of the kd order around the tile of its first row, clamped into [0, n_tiles).  A wider list contains
every narrower one (also where it is clamped at either end of the order), which is what makes the wider short sweep's
bound u(q) at most the narrower one's: every proposal sub-list then ends at least as high.  This checks the formula,
not the kernel: tests/test_gpu_knn_screen_tight.py checks the kernel's lists through that consequence (u and the kept
tiles shrink as the width grows)."""
import numpy as np
import pytest


def near_list(own, n_tiles, nt):
    cnt = min(nt, n_tiles)
    first = max(0, min(own - (nt - 1) // 2, n_tiles - cnt))
    return np.arange(first, first + cnt)


@pytest.mark.parametrize("n_tiles", [1, 5, 8, 9, 31, 32, 33, 100, 10_157])
def test_near_lists_are_in_range_and_hold_the_own_tile(n_tiles):
    for nt in (1, 8, 32, 64):
        for own in range(n_tiles):
            t = near_list(own, n_tiles, nt)
            assert len(t) == min(nt, n_tiles) and t[0] >= 0 and t[-1] < n_tiles
            assert own in t


@pytest.mark.parametrize("n_tiles", [8, 9, 31, 33, 40, 100, 10_157])
def test_wider_near_lists_contain_narrower_ones(n_tiles):
    owns = range(n_tiles) if n_tiles < 1000 else np.r_[0:100, n_tiles - 100:n_tiles, 5000:5100]
    for own in owns:
        for a, b in ((8, 32), (8, 64), (32, 64), (16, 32)):
            assert set(near_list(own, n_tiles, a)) <= set(near_list(own, n_tiles, b)), (own, a, b)

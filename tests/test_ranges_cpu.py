"""The work split of the decode kernels (kivi_attn.cuh `Ranges`: one contiguous, cost-balanced range of (unit, item)
positions per warp) evaluated on the host through the kivi_debug_range_split hook: partition properties that the kernels'
workspace indexing relies on, and the balance the cost model is there for."""
import ctypes

import numpy as np
import pytest


@pytest.fixture(scope="module")
def split():
    from kivi_b200 import _lib, build
    build.build()
    fn = _lib.bind("kivi_debug_range_split", ctypes.c_int, [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_void_p])

    def run(n_units, n_b, n_w, w_cap, kernel):
        per_unit = n_b + n_w + 1
        lo = np.zeros((w_cap + 2, 2), np.int32)
        owner = np.zeros(n_units * per_unit, np.int32)
        W = fn(n_units, n_b, n_w, w_cap, kernel, lo.ctypes.data, owner.ctypes.data)
        assert W >= 1
        return W, lo[:W + 1], owner
    return run


CASES = [  # n_units, n_b, n_w, w_cap
    (1024, 31, 9, 2368),       # cfg 2 p.V at T = 4096
    (1024, 31, 2, 2368),       # cfg 2 q.K^T
    (512, 63, 9, 2368),        # cfg 3
    (128, 511, 5, 2368),       # cfg 4: few long units
    (128, 511, 5, 1776),       # cfg 4 as launched: 148 CTAs x 12 warps (kivi_attn.cuh WarpsPerCta<4, 4>)
    (512, 63, 9, 1776),
    (8192, 31, 9, 2368),       # cfg 5 on one GPU: the 64-bit arithmetic path
    (3, 0, 2, 2368),           # tiny: nothing packed yet, more warps than items
    (1, 0, 0, 2368),           # one unit, only the new token
    (7, 5, 0, 11),
    (2, 300, 17, 33),
]


@pytest.mark.parametrize("n_units,n_b,n_w,w_cap", CASES)
@pytest.mark.parametrize("kernel", [0, 1])
def test_ranges_partition_the_items(split, n_units, n_b, n_w, w_cap, kernel):
    per_unit = n_b + n_w + 1
    W, lo, owner = split(n_units, n_b, n_w, w_cap, kernel)
    assert W <= w_cap and W <= n_units * per_unit
    pos = lo[:, 0].astype(np.int64) * per_unit + lo[:, 1]
    assert pos[0] == 0 and pos[-1] == n_units * per_unit, "the ranges cover all items"
    assert (np.diff(pos) >= 1).all(), "every range is non-empty (the kernels index workspace slots by range number)"
    assert ((lo[:, 1] >= 0) & (lo[:, 1] < per_unit)).all()
    # owner() is the inverse of lo(): position p belongs to range w iff lo(w) <= p < lo(w + 1)
    exp = np.repeat(np.arange(W), np.diff(pos))
    np.testing.assert_array_equal(owner, exp)
    # a unit meets at most ceil(W / n_units) + 1 ranges: the bound of the statistics / partial-record slots
    per = owner.reshape(n_units, per_unit)
    assert int((per[:, -1] - per[:, 0] + 1).max()) <= -(-W // n_units) + 1


def test_default_split_is_equal_item_counts(split):
    """The shipped build weighs every item the same (KIVI_UNIFORM_RANGES = 1): range sizes differ by at most one item."""
    for kernel in (0, 1):
        W, lo, owner = split(1024, 31, 9, 2368, kernel)
        counts = np.bincount(owner, minlength=W)
        assert counts.max() - counts.min() <= 1

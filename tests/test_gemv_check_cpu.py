"""The oracle check of the dequant-GEMVs (tests/_gemv.py) on the oracle's own outputs: it accepts them, and it rejects each
single defect a kernel could make.  The only checks of the GEMV harness that run without a GPU."""
import numpy as np
import pytest

from oracle import ref
from tests._gemv import FLOOR_COEF, check_gemv, dequant, exact, kernel_layout, kernel_layout_case, l1, padded_rows, ulp16

B, H, HKV, K, N, G, BITS = 2, 4, 2, 96, 128, 32, 2                 # two query heads per KV head


def _case(layout, overflow=False, cancelling=False):
    """The oracle's output of one small case of `layout` and check_gemv's arguments for it.  overflow: batch 1, KV head 0
    gets a group of scale inf (row 5, channels 0-31).  cancelling: the rows of w come in equal pairs and x in opposite
    pairs, so every exact output is 0."""
    rng = np.random.default_rng(7)
    if layout == "kernel":
        x, w = kernel_layout_case(rng, B, H, HKV, K, N)
        code, scale, mn = ref.pack_lastdim(w, G, BITS)
        return ref.bgemv_outer_kernel_layout(x, *kernel_layout(code, scale, mn), BITS, G, H, HKV), \
            ("kernel", x, code, scale, mn, G, BITS, "kernel", H)
    if layout == "inner":
        x = rng.standard_normal((3, 512)).astype(np.float16)
        code, scale, mn = ref.pack_lastdim(rng.standard_normal((64, 512)).astype(np.float16), 64, 4)
        return ref.gemv_inner_w4(x, code, *padded_rows(scale, mn, 64), 64), ("inner", x, code, scale, mn, 64, 4, "inner")
    w = rng.standard_normal((B, HKV, K, N)).astype(np.float16)
    x = (rng.standard_normal((B, H, 1, K)) * 0.7).astype(np.float16)
    if overflow:
        w[1, 0, 5, 0], w[1, 0, 5, 1] = -60000.0, 60000.0
    if cancelling:
        w[:, :, 1::2] = w[:, :, 0::2]
        x[..., 1::2] = -x[..., 0::2]
    code, scale, mn = ref.pack_lastdim(w, G, BITS)
    return ref.bmm_fA_qB_outer(G, x, code, scale, mn, BITS), ("bmm", x, code, scale, mn, G, BITS, "bmm")


def _rejects(got, args, match):
    with pytest.raises(AssertionError, match=match):
        check_gemv(args[0], got, *args[1:])


@pytest.mark.parametrize("layout", ["bmm", "kernel", "inner"])
def test_accepts_the_oracle(layout):
    oracle, args = _case(layout)
    check_gemv(args[0], oracle, *args[1:])


def test_rejects_each_defect():
    oracle, args = _case("bmm", overflow=True)
    assert not np.isfinite(oracle[1, :2, 0, :32]).any() and np.isfinite(np.delete(oracle, 1, 0)).all(), "precondition"
    check_gemv(args[0], oracle, *args[1:])
    # one output 2 fp16 steps beyond the bar
    j = (0, 1, 0, int(np.argmax(oracle[0, 1, 0])))
    x, code, scale, mn = args[1:5]
    w = dequant(code, scale, mn, G, BITS)
    e = float(exact(x, w)[j])
    edge = np.float16(e + abs(float(oracle[j]) - e) + ulp16(e) + FLOOR_COEF * float(l1(x, w)[j]))
    got = oracle.copy()
    got[j] = (edge.view(np.uint16) + 2).view(np.float16)
    _rejects(got, args, "1 / .* out of tolerance")
    # a finite output where the oracle's is inf, and an inf where the oracle's is finite
    got = oracle.copy()
    got[1, 0, 0, 3] = 0.0
    _rejects(got, args, "non-finite positions")
    got = oracle.copy()
    got[0, 0, 0, 3] = np.inf
    _rejects(got, args, "non-finite positions")
    # query head h reading KV head h % HKV instead of h // (H / HKV)
    oracle, args = _case("bmm")
    x, code, scale, mn = args[1:5]
    swapped = ref.bmm_fA_qB_outer(G, np.ascontiguousarray(x[:, [0, 2, 1, 3]]), code, scale, mn, BITS)[:, [0, 2, 1, 3]]
    _rejects(swapped, args, "out of tolerance")


def test_rejects_a_floor_error_on_cancelling_outputs():
    """Every exact output is 0, so the bar is the floor: half of it passes, twice it fails."""
    oracle, args = _case("bmm", cancelling=True)
    x, code, scale, mn = args[1:5]
    floor = FLOOR_COEF * l1(x, dequant(code, scale, mn, G, BITS))
    assert (np.abs(oracle) + ulp16(0.0) < 0.1 * floor).all(), "precondition: the floor dominates the bar"
    for factor, ok in ((0.5, True), (2.0, False)):
        got = oracle.copy()
        got[1, 3, 0, 17] = np.float16(factor * floor[1, 3, 0, 17])
        if ok:
            check_gemv(args[0], got, *args[1:])
        else:
            _rejects(got, args, "1 / .* out of tolerance")

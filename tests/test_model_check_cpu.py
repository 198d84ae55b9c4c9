"""The model-level checks (tests/_model.py) on synthetic data, without a GPU: TupleBar accepts logits inside its bars and
rejects each single defect, and packed_parts_equal tells two 9-tuples apart by one bit of a packed field."""
import pytest
import torch

from tests._model import PACKED, TupleBar, packed_parts_equal


def _logits():
    """[3, 50] logits whose argmax (token 7) leads token 8 by 0.01 in every row."""
    ref = torch.randn(3, 50, generator=torch.Generator().manual_seed(0))
    ref[:, 7], ref[:, 8] = 5.0, 4.99
    return ref


def test_step_bar_accepts_inside_and_rejects_above():
    ref = _logits()
    limit = 3e-2 * 5.0 + 3e-2
    bar = TupleBar("synthetic")
    bar.step(ref.clone(), ref, "equal")
    inside = ref.clone()
    inside[1, 20] += 0.99 * limit
    bar.step(inside, ref, "inside")
    assert bar.agree == 2 and bar.worst["step"] == pytest.approx(0.99, rel=1e-4)
    for bad in (1.01 * limit, float("nan"), float("inf")):
        got = ref.clone()
        got[2, 30] += bad
        with pytest.raises(AssertionError, match="max\\|got - ref\\|"):
            bar.step(got, ref, "bad")
    assert bar.agree == 2


def test_prompt_bar_is_elementwise_allclose():
    ref = _logits()
    ref[0, 0] = 0.0
    top = 2e-2 + 2e-2 * 5.0                                           # the bar of an element whose ref is 5.0
    bar = TupleBar("synthetic")
    bar.prompt(ref.clone(), ref)
    inside = ref.clone()
    inside[0, 7] += 0.99 * top
    bar.prompt(inside, ref)
    assert bar.worst["prompt"] == pytest.approx(0.99, rel=1e-4)
    # over the bar at the largest element; at an element whose ref is 0, whose bar is atol alone; non-finite
    for at, add in (((0, 7), 1.01 * top), ((0, 0), 1.01 * 2e-2), ((2, 0), float("nan")), ((2, 0), float("inf"))):
        got = ref.clone()
        got[at] += add
        with pytest.raises(AssertionError, match="prompt"):
            bar.prompt(got, ref)


@pytest.mark.parametrize("flips", [3, 4])
def test_argmax_may_flip_in_three_of_ten_steps(flips):
    ref = _logits()
    bar = TupleBar("synthetic")
    for s in range(10):
        got = ref.clone()
        if s < flips:
            got[s % 3, 8] = 5.01                                      # inside the bar, argmax 8 instead of 7
        bar.step(got, ref, f"step {s}")
    assert bar.agree == 10 - flips
    if flips <= 3:
        bar.done(10)
    else:
        with pytest.raises(AssertionError, match="6 of 10 steps"):
            bar.done(10)


def _parts():
    """A 9-tuple with every field present: int32 codes, fp16 windows, scales and zero points (scales and zero points in
    [0.5, 1.5): a flip of the lowest mantissa bit changes the value)."""
    g = torch.Generator().manual_seed(1)
    codes = lambda *s: torch.randint(-2 ** 31, 2 ** 31 - 1, s, dtype=torch.int32, generator=g)   # noqa: E731
    halves = lambda *s: (torch.rand(s, generator=g) + 0.5).half()                            # noqa: E731
    return [codes(2, 2, 128, 4), halves(2, 2, 5, 128), halves(2, 2, 128, 4), halves(2, 2, 128, 4),
            codes(2, 2, 64, 8), halves(2, 2, 7, 128), halves(2, 2, 64, 4), halves(2, 2, 64, 4), 133]


def test_packed_parts_equal():
    fused = _parts()
    packed_parts_equal(fused, [t.clone() if torch.is_tensor(t) else t for t in fused], "copy")
    reshaped = [t.reshape(t.shape[0], -1) if torch.is_tensor(t) else t for t in fused]
    packed_parts_equal(fused, reshaped, "other view shape")
    for i in PACKED:
        ref = [t.clone() if torch.is_tensor(t) else t for t in fused]
        bits = ref[i].view(torch.int16) if ref[i].dtype == torch.float16 else ref[i]
        bits.view(-1)[37] ^= 1
        with pytest.raises(AssertionError, match=f"tuple\\[{i}\\]"):
            packed_parts_equal(fused, ref, "one bit")
        for a, b in ((None, ref[i]), (ref[i], None)):
            x, y = list(fused), list(fused)
            x[i], y[i] = a, b
            with pytest.raises(AssertionError, match="one side only"):
                packed_parts_equal(x, y, "None")
    none = list(fused)
    none[0] = none[2] = none[3] = None
    packed_parts_equal(none, list(none), "no packed K on either side")
    with pytest.raises(AssertionError, match="kv_seq_len"):
        packed_parts_equal(fused, fused[:8] + [134], "kv_seq_len")

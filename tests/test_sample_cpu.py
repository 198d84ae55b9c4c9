"""Sampling without a GPU: the numpy reference of kivi_sample_f32 (tests/_sample.py: Philox4x32-10 and the row semantics in
fp64, which the GPU tests compare the kernel with) checked on known answers and hand-made rows; the argument checks of
the C entry point; parameter validation of set_sampling / generate (sampling_rows) and request parsing of serve()."""
import numpy as np
import pytest

from tests._sample import M32, greedy_id, philox4x32_10, reference_pick, reference_row, uniform24

KIVI_ERR_SHAPE, KIVI_ERR_NULL = -2, -6
FAKE = 1 << 20                                       # never dereferenced: validation returns before any launch


# ------------------------------------------------------------------------------------------------ the reference itself
def test_philox_known_answers():
    """The known-answer vectors of the Random123 distribution for philox4x32_10."""
    assert philox4x32_10((0, 0, 0, 0), (0, 0)) == (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)
    assert philox4x32_10((M32,) * 4, (M32,) * 2) == (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)
    assert philox4x32_10((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0)) == \
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)
    assert uniform24(0, 0) == 0x6627e8
    assert len({uniform24(s, d) for s in range(30) for d in range(30)}) > 890


def test_reference_row_semantics():
    ln = np.log
    row = np.array([ln(4), ln(2), ln(2), 0.0, -np.inf, np.nan, ln(1)], dtype=np.float32)   # masses 4 2 2 1 - - 1 of 10
    full, _ = reference_row(row, 1.0, 0, 1.0)
    assert (full > 0).tolist() == [True, True, True, True, False, False, True]             # -inf and NaN are never kept
    np.testing.assert_allclose(full / full.sum(), [.4, .2, .2, .1, 0, 0, .1], atol=1e-7)
    assert (reference_row(row, 1.0, 2, 1.0)[0] > 0).sum() == 3                             # the tie at the 2nd largest stays
    assert (reference_row(row, 1.0, 1, 1.0)[0] > 0).sum() == 1
    assert (reference_row(row, 1.0, 7, 1.0)[0] > 0).sum() == 5                             # k >= vocab: off
    assert (reference_row(row, 1.0, 0, 0.3)[0] > 0).sum() == 1
    w, margin = reference_row(row, 1.0, 0, 0.5)                                            # .4 < .5: the tie joins whole
    assert (w > 0).sum() == 3 and abs(margin - 0.1) < 1e-6
    assert (reference_row(row, 1.0, 0, 0.85)[0] > 0).sum() == 5
    assert (reference_row(row, 1.0, 0, 0.0)[0] > 0).sum() == 1                             # p <= 0: the maximum only
    assert (reference_row(row, 1.0, 3, 0.95)[0] > 0).sum() == 3                            # top-p over what top-k kept
    sharp, _ = reference_row(row, 0.5, 0, 1.0)
    np.testing.assert_allclose(sharp / sharp.sum(), np.array([16, 4, 4, 1, 0, 0, 1]) / 26, atol=1e-6)
    assert reference_row(row, 0.0, 0, 1.0) is None
    assert reference_row(np.array([1.0, np.inf, 2.0]), 1.0, 0, 1.0) is None
    assert reference_row(np.array([-np.inf, np.nan]), 1.0, 0, 1.0) is None
    assert greedy_id([1.0, 3.0, 3.0]) == 1 and greedy_id([1.0, np.nan, 9.0, np.nan]) == 1
    assert greedy_id([-np.inf, -np.inf]) == 0


def test_reference_pick_walks_in_token_order():
    w = np.array([0.0, 2.0, 0.0, 1.0, 1.0])
    ids = [reference_pick(w, n)[0] for n in (0, (1 << 23) - 1, 1 << 23, (3 << 22) - 1, 3 << 22, (1 << 24) - 1)]
    assert ids == [1, 1, 3, 3, 4, 4]
    assert abs(reference_pick(w, 1 << 22)[1] - 0.25) < 1e-12


# ------------------------------------------------------------------------------------------------ the C entry point
def test_entry_point_validates_arguments():
    import ctypes
    from kivi_b200 import _lib, build
    build.build()
    L = _lib.lib()
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    f = L.kivi_sample_f32
    f.restype, f.argtypes = i32, [vp, i32, i32] + [vp] * 10
    ok = [FAKE, 4, 32000] + [FAKE] * 9 + [None]
    n0 = _lib.launch_count()
    for i in (0, 3, 4, 5, 6, 7, 8):                                       # every required pointer
        args = list(ok)
        args[i] = None
        assert f(*args) == KIVI_ERR_NULL, i
    for batch, vocab in ((-1, 32000), (4, 0), (4, -5), (4, (1 << 22) + 1)):
        args = list(ok)
        args[1], args[2] = batch, vocab
        assert f(*args) == KIVI_ERR_SHAPE, (batch, vocab)
    args = list(ok)
    args[1] = 0
    assert f(*args) == 0                                                  # an empty batch is fine
    assert _lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------ the Python surface
def test_sampling_rows_validation():
    from kivi_b200.choice import sampling_rows
    assert sampling_rows(3) == ([1.0] * 3, [50] * 3, [1.0] * 3, [0, 1, 2])
    t, k, p, s = sampling_rows(2, temperature=[0.0, 0.7], top_k=0, top_p=(0.9, 1.0), seed=[7, 2 ** 64 - 1])
    assert (t, k, p, s) == ([0.0, 0.7], [0, 0], [0.9, 1.0], [7, 2 ** 64 - 1])
    assert sampling_rows(2, seed=2 ** 64 - 1)[3] == [2 ** 64 - 1, 0]      # keys wrap
    for bad in (dict(temperature=-0.1), dict(temperature=float("nan")), dict(temperature=float("inf")),
                dict(top_p=1.5), dict(top_p=-0.01), dict(top_p=float("nan")), dict(top_k=2.5), dict(top_k=2 ** 31),
                dict(top_k="many"), dict(seed=-1), dict(seed=1.5), dict(temperature=[1.0, 1.0, 1.0]),
                dict(top_p=[0.5]), dict(seed=[1, 2, 3]), dict(top_k=[1])):
        with pytest.raises(ValueError):
            sampling_rows(2, **bad)


def test_generate_rejects_bad_parameters_before_any_work():
    import torch
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    model = LlamaForCausalLM_KIVI(default_config("tiny"))
    ids = torch.zeros((2, 4), dtype=torch.long)
    with pytest.raises(ValueError, match="temperature"):
        model.generate(ids, max_new_tokens=2, do_sample=True, temperature=-1.0)
    with pytest.raises(ValueError, match="top_p"):
        model.generate(ids, max_new_tokens=2, do_sample=True, top_p=[0.5, 1.2])
    assert model.cache is None


def test_serve_request_parsing():
    from kivi_b200.serve import Params, parse_requests
    reqs, params = parse_requests([([1, 2, 3], 4), (np.array([5]), 2)])
    assert [p.tolist() for p, _ in reqs] == [[1, 2, 3], [5]] and [m for _, m in reqs] == [4, 2]
    assert params == [Params(), Params()] and params[0] == (None,) * 4   # no params: serve() stays on the greedy step
    reqs, params = parse_requests([([1], 1, {"temperature": 0.8, "seed": 3}), ([2], 1), ([3], 1, None), ([4], 1, {})])
    assert [p.sampling for p in params] == [{"temperature": 0.8, "seed": 3}, None, None, {}]
    assert all(p.processing is None and p.logprobs is None and p.adapter is None for p in params)
    for bad in ([([1], 1, {"temperature": -1})], [([1], 1, {"top_p": 2})], [([1], 1, {"min_p": 0.1})],
                [([1], 1, {"top_k": [1, 2]})], [([], 1)], [([1], 0)], [([1],)], [([1], 1, {}, 0)]):
        with pytest.raises(ValueError):
            parse_requests(bad)


def test_serve_validates_params_before_touching_the_model():
    """serve() parses and validates every request first: bad params raise before the model is asked for anything, and a
    valid list reaches the cache set-up."""
    import torch
    from kivi_b200 import serve as ks

    class Stop(Exception):
        pass

    class Model:
        cache = None

        def init_cache(self, batch, max_tokens):
            raise Stop

        def __getattr__(self, name):
            raise AssertionError(f"serve() touched model.{name}")

    with pytest.raises(Stop):
        list(ks.serve(Model(), [(torch.tensor([1, 2]), 3)], 2, 64))
    with pytest.raises(ValueError, match="top_p"):
        list(ks.serve(Model(), [(torch.tensor([1, 2]), 3, {"top_p": 7})], 2, 64))

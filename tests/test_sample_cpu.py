"""Sampling without a GPU: a numpy restatement of Philox4x32-10 and of the row semantics of kivi_sample_f32 in fp64 (the
reference the GPU tests compare the kernel with), checked here on known answers and hand-made rows; the argument checks of
the C entry point; parameter validation of set_sampling / generate (sampling_rows) and request parsing of serve()."""
import numpy as np
import pytest

KIVI_ERR_SHAPE, KIVI_ERR_NULL = -2, -6
FAKE = 1 << 20                                       # never dereferenced: validation returns before any launch
M32 = 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------ the reference
def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., SC11): counter = 4 words, key = 2 words -> 4 words."""
    c0, c1, c2, c3 = counter
    k0, k1 = key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & M32, (p0 >> 32) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
    return c0, c1, c2, c3


def uniform24(seed: int, draw: int) -> int:
    """The 24-bit integer n of the kernel's uniform number u = n * 2^-24 for (seed, draw), both uint64."""
    return philox4x32_10((draw & M32, draw >> 32, 0, 0), (seed & M32, seed >> 32))[0] >> 8


def greedy_id(row) -> int:
    """torch.argmax's rule: the first NaN, else the first maximum."""
    row = np.asarray(row)
    nan = np.isnan(row)
    return int(nan.argmax()) if nan.any() else int(row.argmax())


def reference_row(row, temperature, top_k, top_p):
    """Row semantics in fp64.  Returns None for a row that takes the greedy id (temperature 0, a +inf, no finite logit), else
    (w, margin): w [vocab] fp64 the kept tokens' masses exp(x - max) (0 = not kept), margin the distance of the top-p
    decision from its nearest alternative as a fraction of the mass (inf when top-p is off)."""
    row = np.asarray(row, dtype=np.float32)
    if temperature == 0:
        return None
    with np.errstate(all="ignore"):
        x = (row / np.float32(temperature)).astype(np.float64)          # the fp32 quotient, as the kernel forms it
    x[np.isnan(x)] = -np.inf
    V, mx = x.size, x.max()
    if not np.isfinite(mx):
        return None
    kept = x > -np.inf
    if 0 < top_k < V:
        kept &= x >= np.partition(x, V - top_k)[V - top_k]
    w = np.where(kept, np.exp(x - mx), 0.0)
    margin = np.inf
    if top_p < 1:
        if top_p <= 0:
            thr = mx
        else:
            vals, inv = np.unique(x[kept], return_inverse=True)         # ascending distinct values; ties share a class
            mass = np.bincount(inv, weights=w[kept])[::-1]
            cum, target = np.cumsum(mass), top_p * w.sum()
            j = int(np.argmax(cum >= target)) if (cum >= target).any() else len(cum) - 1
            thr = vals[::-1][j]
            margin = np.abs(cum - target).min() / w.sum()
        w = np.where(x >= thr, w, 0.0)
    return w, margin


def reference_pick(w, n24: int):
    """The inverse CDF in token-id order: (first id whose cumulative mass exceeds u * S, distance of u * S from the nearest
    CDF step as a fraction of S)."""
    cdf = np.cumsum(w)
    S = cdf[-1]
    target = n24 * 2.0 ** -24 * S
    return int(np.argmax(cdf > target)), np.abs(cdf[w > 0] - target).min() / S


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
    from kivi_b200.llama_kivi import sampling_rows
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
    from kivi_b200.serve import parse_requests
    reqs, params = parse_requests([([1, 2, 3], 4), (np.array([5]), 2)])
    assert [p.tolist() for p, _ in reqs] == [[1, 2, 3], [5]] and [m for _, m in reqs] == [4, 2]
    assert params == [None, None]                                         # no params: serve() stays on the greedy step
    reqs, params = parse_requests([([1], 1, {"temperature": 0.8, "seed": 3}), ([2], 1), ([3], 1, None), ([4], 1, {})])
    assert params == [{"temperature": 0.8, "seed": 3}, None, None, {}]
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

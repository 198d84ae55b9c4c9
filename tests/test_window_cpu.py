"""Sliding-window decode without a GPU: the C entry kivi_decode_attention_window_f16 is exported and validates its window,
the producer and consumer walks of a windowed call stay in step and cover exactly the visible items (kivi_debug_window_items
replays both with the kernels' own functions), and the model reads config.sliding_window and refuses per-layer windows."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

BLOCK = 128                     # tokens per packed block (kivi_decode.cuh kBlockTokens)
KIVI_ERR_SHAPE, KIVI_ERR_NULL = -2, -6


@pytest.fixture(scope="module")
def lib():
    from kivi_b200 import _lib, build
    build.build()
    return _lib.lib()


def test_window_symbols_are_exported(lib):
    assert hasattr(lib, "kivi_decode_attention_window_f16")
    assert hasattr(lib, "kivi_debug_window_items")


def test_window_entry_validates_the_window(lib):
    from kivi_b200.cache import _CacheStruct
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    fn = lib.kivi_decode_attention_window_f16
    fn.restype = i32
    fn.argtypes = [ctypes.POINTER(_CacheStruct), vp, vp, vp, vp, i32, vp, vp, vp, i64, vp, vp, i64, i32, vp]
    f = dict(batch=2, num_heads=4, num_kv_heads=2, head_dim=128, k_bits=2, v_bits=2, group_size=32, residual_length=128,
             k_cap_blocks=4, v_cap_blocks=4, v_res_cap=129, flags=0)
    fake = 1 << 20                                   # never dereferenced: validation returns before any launch
    st = _CacheStruct(*[f[n] for n, _ in _CacheStruct._fields_[:12]], fake, fake, fake, fake, fake)

    def call(window, q=fake):
        return fn(ctypes.byref(st), q, fake, fake, None, window, None, fake, fake, 1 << 30, None, None, 0, 256, None)
    assert call(0) == KIVI_ERR_SHAPE
    assert call(-5) == KIVI_ERR_SHAPE
    assert call(64, q=None) == KIVI_ERR_NULL


def _window_items(lib, n_units, n_b, n_w, w_cap, kernel, starts, T, window):
    fn = lib.kivi_debug_window_items
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_int64, ctypes.c_void_p]
    cap = n_units * (n_b + n_w + 1) + 8
    st = None if starts is None else np.ascontiguousarray(starts, np.int32)
    issued = np.zeros((cap, 4), np.int32)
    consumed = np.zeros((cap, 4), np.int32)
    n = np.zeros(2, np.int64)
    W = fn(n_units, n_b, n_w, w_cap, kernel, None if st is None else st.ctypes.data, T, window, issued.ctypes.data,
           consumed.ctypes.data, cap, n.ctypes.data)
    assert W >= 1, W
    return W, issued[:n[0]], consumed[:n[1]]


def _visible_stages(n_units, n_b, n_w, starts, T, window):
    """Every (unit, item) that needs a stage: the window items, and the packed blocks not wholly below the visible start
    max(clamp(kv_start, 0, T - 1), T - window)."""
    out = []
    for u in range(n_units):
        s = min(max(int(starts[u]) if starts is not None else 0, 0), T - 1)
        s = max(s, T - window)
        out += [(u, j) for j in range(n_b) if (j + 1) * BLOCK > s] + [(u, n_b + i) for i in range(n_w)]
    return out


def _geometry(rng, kernel):
    n_units = int(rng.choice([1, 3, 8, 32, 200, 1024]))
    n_b = int(rng.integers(0, 40))
    n_w = int(rng.integers(0, 10)) if kernel == 0 else int(rng.integers(1, 18))
    w_cap = int(rng.choice([1, 7, 33, 132 * 12, 132 * 16, 5000]))
    tk = max(n_b * BLOCK - int(rng.choice([0, 0, 64, 96])), 0)            # the last packed block may be partial (R < 128)
    T = max(tk + n_w * 16 - int(rng.integers(0, 16)) if n_w else tk, tk) + 1
    return n_units, n_b, n_w, w_cap, T


def _windows(rng, T, R):
    """1, below R, inside a packed block, on a block edge, at / beyond T."""
    edge = T - BLOCK * int(rng.integers(0, T // BLOCK + 1))
    return [1, max(1, R - 1 - int(rng.integers(0, R - 1))), max(1, T - BLOCK * int(rng.integers(0, T // BLOCK + 1)) - 37),
            max(1, edge), T, T + int(rng.integers(1, 500))]


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("seed", range(8))
def test_window_walks_issue_exactly_the_visible_items(lib, kernel, seed, padded):
    """For every warp range the producer issues exactly the stages the consumer waits on, in the same order; no packed
    block below the window's first block j0 is issued; and the ranges together cover exactly the visible items."""
    rng = np.random.default_rng(seed * 4 + kernel * 2 + int(padded))
    n_units, n_b, n_w, w_cap, T = _geometry(rng, kernel)
    R = int(rng.choice([32, 64, 128, 256]))
    for window in _windows(rng, T, R):
        starts = None
        if padded:
            starts = np.array([int(rng.choice([0, 1, BLOCK * int(rng.integers(0, n_b + 1)) + 5, int(rng.integers(0, T + 1)),
                                               T + 300, -7])) for _ in range(n_units)], np.int32)
        W, issued, consumed = _window_items(lib, n_units, n_b, n_w, w_cap, kernel, starts, T, window)
        for w in range(W):
            np.testing.assert_array_equal(issued[issued[:, 0] == w], consumed[consumed[:, 0] == w],
                                          err_msg=f"warp {w}, window {window}")
        np.testing.assert_array_equal(issued, consumed)
        j0 = min(n_b, max(0, T - window) // BLOCK)
        blocks = issued[issued[:, 2] < n_b]
        assert (blocks[:, 2] >= j0).all(), f"window {window}: a block below j0 = {j0} was issued"
        got = [(int(u), int(j)) for u, j in issued[:, 1:3]]
        assert got == _visible_stages(n_units, n_b, n_w, starts, T, window), f"window {window}"
        assert (np.diff(issued[:, 0]) >= 0).all()                        # ranges in warp order: a partition


def test_window_split_counts_only_the_visible_blocks(lib):
    """At T = 32k and W = 4096 every warp range lies inside the last ~4096 tokens: the split has 1/8 of the packed items."""
    n_units, n_b, n_w, T, window = 128, 256, 4, 256 * BLOCK + 60, 4096
    W_full, full, _ = _window_items(lib, n_units, n_b, n_w, 132 * 16, 1, None, T, T + 1)
    W_win, win, _ = _window_items(lib, n_units, n_b, n_w, 132 * 16, 1, None, T, window)
    assert (full[:, 2] < n_b).sum() == n_units * n_b
    assert (win[:, 2] < n_b).sum() == n_units * (n_b - (T - window) // BLOCK)
    per_warp = np.bincount(win[:, 0], minlength=W_win)
    assert per_warp.min() >= 1                                           # no warp is left with skipped items only


def test_window_hook_validates(lib):
    n = np.zeros(2, np.int64)
    buf = np.zeros((8, 4), np.int32)
    fn = lib.kivi_debug_window_items
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_int64, ctypes.c_void_p]
    assert fn(1, 2, 1, 4, 0, None, 300, 0, buf.ctypes.data, buf.ctypes.data, 8, n.ctypes.data) == KIVI_ERR_SHAPE
    assert fn(1, 2, 1, 4, 0, None, 0, 10, buf.ctypes.data, buf.ctypes.data, 8, n.ctypes.data) == KIVI_ERR_SHAPE


# ---------------------------------------------------------------------------------------------------------------------
# config reading
# ---------------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from kivi_b200.llama_kivi import default_config
    return default_config("tiny", **kw)


def test_sliding_window_from_config():
    from kivi_b200.llama_kivi import sliding_window
    assert sliding_window(SimpleNamespace()) is None
    assert sliding_window(SimpleNamespace(sliding_window=None)) is None
    assert sliding_window(SimpleNamespace(sliding_window=4096)) == 4096
    assert sliding_window(SimpleNamespace(sliding_window=4096, layer_types=["sliding_attention"] * 4)) == 4096
    assert sliding_window(SimpleNamespace(sliding_window=4096, layer_types=["full_attention"] * 4)) is None
    with pytest.raises(NotImplementedError, match="layer_types"):
        sliding_window(SimpleNamespace(sliding_window=4096, layer_types=["sliding_attention", "full_attention"]))
    with pytest.raises(ValueError):
        sliding_window(SimpleNamespace(sliding_window=0))


def test_model_reads_the_window_and_refuses_mixed_layers():
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    assert LlamaForCausalLM_KIVI(_cfg()).sliding_window is None
    cfg = _cfg()
    cfg.sliding_window = 160
    assert LlamaForCausalLM_KIVI(cfg).sliding_window == 160
    cfg.layer_types = ["sliding_attention", "full_attention"] * (cfg.num_hidden_layers // 2)
    with pytest.raises(NotImplementedError, match="layer_types"):
        LlamaForCausalLM_KIVI(cfg)


def test_mistral_config_window():
    transformers = pytest.importorskip("transformers")
    from kivi_b200.llama_kivi import sliding_window
    assert sliding_window(transformers.MistralConfig(sliding_window=4096)) == 4096
    assert sliding_window(transformers.MistralConfig(sliding_window=None)) is None


def test_additive_mask_follows_the_transformers_window_rule():
    """kv_idx > q_idx - W on top of causal (and the padding mask), for the prompt pass and one decode query."""
    from kivi_b200.llama_kivi import _additive_mask
    n, W = 9, 4
    m = _additive_mask(None, n, n, torch.float32, "cpu", W, batch=2)
    q, k = torch.arange(n)[:, None], torch.arange(n)[None, :]
    assert m.shape == (2, 1, n, n)
    assert torch.equal(m[0, 0] == 0, (k <= q) & (k > q - W))
    d = _additive_mask(None, 1, n, torch.float32, "cpu", W, batch=3)
    assert d.shape == (3, 1, 1, n) and torch.equal(d[0, 0, 0] == 0, torch.arange(n) > n - 1 - W)
    assert _additive_mask(None, 1, W, torch.float32, "cpu", W) is None                     # the window covers everything
    pad = torch.tensor([[0, 0, 1, 1, 1, 1, 1, 1, 1]])
    p = _additive_mask(pad, n, n, torch.float32, "cpu", W)
    assert torch.equal(p[0, 0] == 0, (k <= q) & (k > q - W) & (k >= 2))
    assert _additive_mask(None, n, n, torch.float32, "cpu", None) is None

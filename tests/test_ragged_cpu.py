"""Left-padded decode without a GPU: the C entry kivi_decode_attention_ragged_f16 is exported and validates its arguments,
the skip decision of the two attention kernels keeps every warp's producer (bulk copies) and consumer (stage waits) in step
(kivi_debug_ragged_items replays both walks on the host with the kernels' own functions), and the HF-mask helper accepts
left padding only."""
import ctypes

import numpy as np
import pytest
import torch

BLOCK = 128                     # tokens per packed block (kivi_decode.cuh kBlockTokens)
KIVI_ERR_BITS, KIVI_ERR_NULL, KIVI_ERR_CAPACITY = -1, -6, -8


@pytest.fixture(scope="module")
def lib():
    from kivi_b200 import _lib, build
    build.build()
    return _lib.lib()


def test_ragged_symbols_are_exported(lib):
    assert hasattr(lib, "kivi_decode_attention_ragged_f16")
    assert hasattr(lib, "kivi_debug_ragged_items")


def _entry(lib):
    from kivi_b200.cache import _CacheStruct
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    fn = lib.kivi_decode_attention_ragged_f16
    fn.restype = i32
    fn.argtypes = [ctypes.POINTER(_CacheStruct), vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, i64, i32, vp]
    return fn


def _struct(**kw):
    from kivi_b200.cache import _CacheStruct
    f = dict(batch=2, num_heads=4, num_kv_heads=2, head_dim=128, k_bits=2, v_bits=2, group_size=32, residual_length=128,
             k_cap_blocks=4, v_cap_blocks=4, v_res_cap=129, flags=0)
    f.update(kw)
    fake = 1 << 20                                   # never dereferenced: validation returns before any launch
    return _CacheStruct(*[f[n] for n, _ in _CacheStruct._fields_[:12]], fake, fake, fake, fake, fake)


def test_ragged_entry_validates_arguments(lib):
    fn = _entry(lib)
    fake = 1 << 20
    starts = 1 << 21

    def call(st, q=fake, max_kv_len=256):
        return fn(ctypes.byref(st) if st is not None else None, q, fake, fake, starts, None, fake, fake, 1 << 30,
                  None, None, 0, max_kv_len, None)
    assert call(None) == KIVI_ERR_NULL
    assert call(_struct(), q=None) == KIVI_ERR_NULL
    assert call(_struct(k_bits=3)) == KIVI_ERR_BITS
    assert call(_struct(v_bits=8)) == KIVI_ERR_BITS
    assert call(_struct(), max_kv_len=4 * BLOCK + 1) == KIVI_ERR_CAPACITY


def _ragged_items(lib, n_units, n_b, n_w, w_cap, kernel, starts, kv_len):
    fn = lib.kivi_debug_ragged_items
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                        ctypes.c_void_p]
    cap = n_units * (n_b + n_w + 1) + 8
    st = np.ascontiguousarray(starts, np.int32)
    issued = np.zeros((cap, 4), np.int32)
    consumed = np.zeros((cap, 4), np.int32)
    n = np.zeros(2, np.int64)
    W = fn(n_units, n_b, n_w, w_cap, kernel, st.ctypes.data, kv_len, issued.ctypes.data, consumed.ctypes.data, cap,
           n.ctypes.data)
    assert W >= 1, W
    return W, issued[:n[0]], consumed[:n[1]]


def _expected_stages(n_units, n_b, n_w, starts, kv_len):
    """Every (unit, item) that needs a stage: the window items, and the packed blocks not wholly below the clamped start."""
    out = []
    for u in range(n_units):
        s = min(max(int(starts[u]), 0), kv_len)
        out += [(u, j) for j in range(n_b) if (j + 1) * BLOCK > s] + [(u, n_b + i) for i in range(n_w)]
    return out


def _random_starts(rng, n_units, n_b, tk, kv_len):
    kinds = [lambda: 0, lambda: 1, lambda: BLOCK * int(rng.integers(0, n_b + 1)), lambda: int(rng.integers(0, kv_len + 1)),
             lambda: BLOCK * int(rng.integers(0, n_b + 1)) + int(rng.integers(1, BLOCK)),      # mid-block
             lambda: tk + int(rng.integers(0, kv_len - tk + 1)),                               # inside the windows
             lambda: kv_len + int(rng.integers(0, 400)),                                      # at / beyond kv_len
             lambda: -int(rng.integers(1, 50))]
    return np.array([kinds[int(rng.integers(0, len(kinds)))]() for _ in range(n_units)], np.int32)


@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("seed", range(12))
def test_issued_copies_equal_consumed_stages(lib, kernel, seed):
    """For every warp range the producer issues exactly the stages the consumer waits on, in the same order -- the wholly
    padded blocks are left out of both -- and together they cover every stage-item of the job."""
    rng = np.random.default_rng(seed * 2 + kernel)
    n_units = int(rng.choice([1, 3, 8, 32, 200, 1024]))
    n_b = int(rng.integers(0, 40))
    n_w = int(rng.integers(0, 10)) if kernel == 0 else int(rng.integers(1, 18))
    w_cap = int(rng.choice([1, 7, 33, 148 * 12, 148 * 16, 5000]))
    tk = max(n_b * BLOCK - int(rng.choice([0, 0, 64, 96])), 0)            # the last packed block may be partial (R < 128)
    kv_len = tk + n_w * 16 - int(rng.integers(0, 16)) if n_w else tk
    kv_len = max(kv_len, tk)
    starts = _random_starts(rng, n_units, n_b, tk, kv_len)
    W, issued, consumed = _ragged_items(lib, n_units, n_b, n_w, w_cap, kernel, starts, kv_len)
    for w in range(W):
        np.testing.assert_array_equal(issued[issued[:, 0] == w], consumed[consumed[:, 0] == w], err_msg=f"warp {w}")
    np.testing.assert_array_equal(issued, consumed)
    assert (issued[:, 3] == 0).all()                                     # whole-block stages (kHalfChunks = 8)
    got = [(int(u), int(j)) for u, j in issued[:, 1:3]]
    assert got == _expected_stages(n_units, n_b, n_w, starts, kv_len)


def test_no_padding_consumes_every_stage(lib):
    n_units, n_b, n_w, kv_len = 64, 31, 9, 31 * BLOCK + 140
    W, issued, consumed = _ragged_items(lib, n_units, n_b, n_w, 2368, 1, np.zeros(n_units, np.int32), kv_len)
    assert len(issued) == n_units * (n_b + n_w)
    np.testing.assert_array_equal(issued, consumed)


def test_kv_start_from_mask():
    from kivi_b200.cache import kv_start_from_mask
    ones = torch.ones(3, 7, dtype=torch.long)
    assert kv_start_from_mask(ones).tolist() == [0, 0, 0]
    left = torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1], [0, 0, 0, 0, 1]])
    st = kv_start_from_mask(left)
    assert st.dtype == torch.int32 and st.tolist() == [2, 0, 4]
    assert kv_start_from_mask(left.bool()).tolist() == [2, 0, 4]
    with pytest.raises(ValueError, match="left padding"):
        kv_start_from_mask(torch.tensor([[1, 1, 1, 0, 0], [1, 1, 1, 1, 1]]))       # right padding
    with pytest.raises(ValueError, match="left padding"):
        kv_start_from_mask(torch.tensor([[1, 1, 0, 1, 1]]))                        # a hole in the middle
    with pytest.raises(ValueError, match="left padding"):
        kv_start_from_mask(torch.tensor([[0, 1, 0, 1, 1]]))
    with pytest.raises(ValueError):
        kv_start_from_mask(torch.tensor([[0, 0, 0]]))                              # no real token

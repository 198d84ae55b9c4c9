"""Continuous batching without a GPU: the three C entries of a slot refill and a timeline shift are exported and reject
every invalid argument by return code before any launch, and the admission / shift policy of kivi_b200.serve."""
import ctypes

import pytest

KIVI_ERR_SHAPE, KIVI_ERR_NULL, KIVI_ERR_CAPACITY = -2, -6, -8
FAKE = 1 << 20                                       # never dereferenced: validation returns before any launch


@pytest.fixture(scope="module")
def lib():
    from kivi_b200 import _lib, build
    build.build()
    L = _lib.lib()
    from kivi_b200.cache import _CacheStruct
    P, vp, i32 = ctypes.POINTER(_CacheStruct), ctypes.c_void_p, ctypes.c_int
    L.kivi_cache_refill_f16.restype = i32
    L.kivi_cache_refill_f16.argtypes = [P, i32, vp, vp] + [i32] * 6 + [vp]
    L.kivi_cache_shift_f16.restype = i32
    L.kivi_cache_shift_f16.argtypes = [P, i32, i32, i32, vp]
    L.kivi_cache_shift_state.restype = i32
    L.kivi_cache_shift_state.argtypes = [P, i32, vp, vp]
    return L


def _struct(**kw):
    from kivi_b200.cache import _CacheStruct
    f = dict(batch=4, num_heads=4, num_kv_heads=2, head_dim=128, k_bits=2, v_bits=2, group_size=32, residual_length=128,
             k_cap_blocks=4, v_cap_blocks=4, v_res_cap=129, flags=0)
    f.update(kw)
    return _CacheStruct(*[f[n] for n, _ in _CacheStruct._fields_[:12]], FAKE, FAKE, FAKE, FAKE, FAKE)


def test_symbols_are_exported(lib):
    for name in ("kivi_cache_refill_f16", "kivi_cache_shift_f16", "kivi_cache_shift_state"):
        assert hasattr(lib, name), name


def test_refill_validates_arguments(lib):
    st = _struct()                                   # R = 128, capacity 4 blocks = 512 tokens

    def call(seq=1, n=100, tk=256, r=44, tv=172, L=128, vhead=5, k=FAKE, v=FAKE, s=st):
        return lib.kivi_cache_refill_f16(ctypes.byref(s) if s is not None else None, seq, k, v, n, tk, r, tv, L, vhead,
                                         None)
    assert call(s=None) == KIVI_ERR_NULL
    assert call(seq=-1) == KIVI_ERR_SHAPE                                   # seq outside [0, B)
    assert call(seq=4) == KIVI_ERR_SHAPE
    assert call(n=0) == KIVI_ERR_SHAPE                                      # n < 1
    assert call(n=301) == KIVI_ERR_SHAPE                                    # n > T = 300
    assert call(tk=200, r=100, tv=172) == KIVI_ERR_SHAPE                    # tk % R
    assert call(tk=128, r=128, tv=128) == KIVI_ERR_SHAPE                    # r >= R
    assert call(tv=171, L=129) == KIVI_ERR_SHAPE                            # L > R
    assert call(tv=100) == KIVI_ERR_SHAPE                                   # tk + r != tv + L
    assert call(tk=256, r=44, tv=200, L=100) == KIVI_ERR_SHAPE              # a V store before the window is full
    assert call(vhead=129) == KIVI_ERR_SHAPE                                # ring head outside the ring
    assert call(vhead=-1) == KIVI_ERR_SHAPE
    assert call(tk=640, r=44, tv=556, n=10) == KIVI_ERR_CAPACITY            # 5 K blocks > 4
    assert call(k=None) == KIVI_ERR_NULL
    assert call(v=None) == KIVI_ERR_NULL


def test_shift_validates_arguments(lib):
    def call(shift=128, tk=384, tv=300, s=None):
        s = _struct() if s is None else s
        return lib.kivi_cache_shift_f16(ctypes.byref(s), shift, tk, tv, None)
    assert lib.kivi_cache_shift_f16(None, 128, 384, 300, None) == KIVI_ERR_NULL
    assert call(shift=0) == KIVI_ERR_SHAPE                                  # shift > 0
    assert call(shift=-128) == KIVI_ERR_SHAPE
    assert call(shift=64, s=_struct(group_size=32, residual_length=32)) == KIVI_ERR_SHAPE        # % max(128, R)
    assert call(shift=128, tk=512, tv=300, s=_struct(residual_length=256, v_res_cap=257)) == KIVI_ERR_SHAPE
    assert call(shift=256, tk=384, tv=200) == KIVI_ERR_SHAPE                # shift > tv
    assert call(shift=256, tk=128, tv=300) == KIVI_ERR_SHAPE                # shift > tk
    assert call(shift=128, tk=640, tv=600) == KIVI_ERR_CAPACITY             # 5 blocks > 4


def test_shift_state_validates_arguments(lib):
    st = _struct()
    assert lib.kivi_cache_shift_state(None, 128, FAKE, None) == KIVI_ERR_NULL
    assert lib.kivi_cache_shift_state(ctypes.byref(st), 0, FAKE, None) == KIVI_ERR_SHAPE
    assert lib.kivi_cache_shift_state(ctypes.byref(st), 96, FAKE, None) == KIVI_ERR_SHAPE
    st256 = _struct(residual_length=256, v_res_cap=257)
    assert lib.kivi_cache_shift_state(ctypes.byref(st256), 128, FAKE, None) == KIVI_ERR_SHAPE


def test_policy_admits_what_fits():
    from kivi_b200.serve import plan_admission
    # T = 1000, room for 500 more tokens: fits as it is
    assert plan_admission(1000, 872, 1500, 128, [300, 950], 200, 500, 600) == (0, True)
    # a prompt longer than T never fits before a shift could make it (the start-up pads to the longest prompt)
    assert plan_admission(1000, 872, 4096, 128, [300], 1001, 10, 1001) == (0, False)


def test_policy_shift_amounts():
    from kivi_b200.serve import plan_admission
    # needs T <= 900: the smallest live start (700) allows 640, the longest pending prompt (200) allows 800 -> 640
    assert plan_admission(1500, 1372, 1600, 128, [900, 700, 1499], 100, 700, 200) == (640, True)
    # the longest pending prompt binds: T - 1250 = 250 -> 128
    assert plan_admission(1500, 1372, 1600, 128, [900, 700], 100, 228, 1250) == (128, True)
    assert plan_admission(1500, 1372, 1600, 128, [900, 700], 100, 229, 1250) == (0, False)
    # R = 256: the quantum is 256 (700 -> 512)
    assert plan_admission(1500, 1244, 1600, 256, [700], 100, 550, 100) == (512, True)
    # the packed V length binds: a start near T cannot shift past tv
    assert plan_admission(1030, 902, 1100, 128, [1025], 5, 500, 5) == (896, True)


def test_policy_waits():
    from kivi_b200.serve import plan_admission
    # the smallest live start is below one quantum: nothing can be dropped yet
    assert plan_admission(1500, 1372, 1600, 128, [100, 900], 100, 700, 200) == (0, False)
    # a shift is possible but not enough: wait rather than move blocks for nothing
    assert plan_admission(1500, 1372, 1600, 128, [300], 100, 700, 200) == (0, False)


def test_policy_restarts_when_no_slot_is_live():
    from kivi_b200.serve import plan_admission
    assert plan_admission(1500, 1372, 1600, 128, [], 100, 700, 200) is None
    assert plan_admission(10, 0, 1600, 128, (), 1, 1, 1) is None

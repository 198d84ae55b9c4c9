"""The decode-step glue entries without a GPU: kivi_add_rmsnorm_f16, kivi_rope_split_f16, kivi_silu_mul_f16 and
kivi_greedy_sample_exchange_f32 reject every invalid argument by return code before any launch.  Every call here is
invalid in at least one argument (or has nothing to do), so none of them launches."""
import ctypes

import pytest

KIVI_OK, KIVI_ERR_SHAPE, KIVI_ERR_ALIGN, KIVI_ERR_NULL = 0, -2, -5, -6
FAKE = 1 << 20                                       # 16-byte aligned, never dereferenced: validation returns first


@pytest.fixture(scope="module")
def lib():
    from kivi_b200 import _lib, build, glue
    build.build()
    glue._bind()
    return _lib.lib()


def test_symbols_are_exported(lib):
    for name in ("kivi_add_rmsnorm_f16", "kivi_rope_split_f16", "kivi_silu_mul_f16", "kivi_greedy_sample_exchange_f32"):
        assert hasattr(lib, name), name


def test_add_rmsnorm_validates_arguments(lib):
    def call(x=FAKE, r=FAKE, w=FAKE, o=FAKE, rows=4, hidden=4096):
        return lib.kivi_add_rmsnorm_f16(x, r, w, o, rows, hidden, 1e-5, None)
    assert call(r=None) == KIVI_ERR_NULL
    assert call(w=None) == KIVI_ERR_NULL
    assert call(o=None) == KIVI_ERR_NULL
    assert call(hidden=4092) == KIVI_ERR_SHAPE                              # hidden % 8 (one uint4 = 8 halves)
    assert call(hidden=0) == KIVI_ERR_SHAPE
    assert call(hidden=16392) == KIVI_ERR_SHAPE                             # > 4 slices x 512 threads x 8
    assert call(rows=-1) == KIVI_ERR_SHAPE
    assert call(rows=-1, x=None) == KIVI_ERR_SHAPE
    # every uint4 operand must start on a 16-byte boundary; a 2-byte misaligned fp16 view is the usual culprit
    for off in (2, 8):
        assert call(x=FAKE + off) == KIVI_ERR_ALIGN
        assert call(r=FAKE + off) == KIVI_ERR_ALIGN
        assert call(r=FAKE + off, x=None) == KIVI_ERR_ALIGN
        assert call(w=FAKE + off) == KIVI_ERR_ALIGN
        assert call(o=FAKE + off) == KIVI_ERR_ALIGN
        assert call(o=FAKE + off, rows=0) == KIVI_ERR_ALIGN                 # checked before the empty early return
    assert call(rows=0) == KIVI_OK                                          # nothing to launch
    assert call(rows=0, x=None) == KIVI_OK


def test_rope_split_validates_arguments(lib):
    def call(qkv=FAKE, c=FAKE, s=FAKE, pos=FAKE, q=FAKE, k=FAKE, v=FAKE, B=4, H=32, Hkv=8, rows=33792):
        return lib.kivi_rope_split_f16(qkv, c, s, pos, q, k, v, B, H, Hkv, rows, None)
    for name in ("qkv", "c", "s", "pos", "q", "k", "v"):
        assert call(**{name: None}) == KIVI_ERR_NULL, name
    assert call(B=0) == KIVI_ERR_SHAPE
    assert call(B=65536) == KIVI_ERR_SHAPE                                  # grid.y
    assert call(H=0) == KIVI_ERR_SHAPE
    assert call(Hkv=0) == KIVI_ERR_SHAPE
    assert call(rows=0) == KIVI_ERR_SHAPE                                   # no row to clamp a position into
    assert call(rows=-5) == KIVI_ERR_SHAPE


def test_silu_mul_validates_arguments(lib):
    def call(gu=FAKE, o=FAKE, rows=4, inter=14336):
        return lib.kivi_silu_mul_f16(gu, o, rows, inter, None)
    assert call(gu=None) == KIVI_ERR_NULL
    assert call(o=None) == KIVI_ERR_NULL
    assert call(inter=11007) == KIVI_ERR_SHAPE                              # odd I: the half2 pairs straddle gate | up
    assert call(inter=0) == KIVI_ERR_SHAPE
    assert call(rows=0) == KIVI_ERR_SHAPE
    assert call(rows=-1) == KIVI_ERR_SHAPE
    assert call(rows=65536) == KIVI_ERR_SHAPE                               # grid.y
    assert call(gu=FAKE + 2) == KIVI_ERR_ALIGN                              # half2 accesses need 4-byte alignment
    assert call(o=FAKE + 2) == KIVI_ERR_ALIGN
    assert call(gu=FAKE + 6, o=FAKE + 4) == KIVI_ERR_ALIGN
    assert call(gu=FAKE + 2, inter=11007) == KIVI_ERR_SHAPE                 # shape first, as in the other entries


def test_greedy_sample_validates_arguments(lib):
    def call(logits=FAKE, B=4, V=32000, nxt=FAKE, peers=None, rank=0, world=1, step=None, err=None):
        return lib.kivi_greedy_sample_exchange_f32(logits, B, V, nxt, None, peers, rank, world, step, err, None)
    assert call(logits=None) == KIVI_ERR_NULL
    assert call(nxt=None) == KIVI_ERR_NULL
    assert call(B=0) == KIVI_ERR_SHAPE
    assert call(V=0) == KIVI_ERR_SHAPE
    assert call(peers=FAKE, world=2, step=None, err=FAKE) == KIVI_ERR_SHAPE         # the exchange needs its step counter
    assert call(peers=FAKE, world=2, step=FAKE, err=None) == KIVI_ERR_SHAPE
    assert call(peers=FAKE, world=2, rank=2, step=FAKE, err=FAKE) == KIVI_ERR_SHAPE
    assert call(peers=FAKE, world=257, step=FAKE, err=FAKE) == KIVI_ERR_SHAPE

"""The decode attention at GQA ratios that G = 4 query heads per work unit do not divide (3, 5, 6, 7: Llama-3.2-3B and the
Qwen2.5 family).  A KV head's heads form ceil(ratio / G) units, the last one partly filled: its missing heads compute on
q = 0 and must write nothing.  Every case is held to the shared oracle check (tests/_attn.py: checked_call /
checked_step), with the geometry's default G and with G = 2 and G = 4 forced through KIVI_CACHE_GQA_CHUNK; and the
out-of-range writes a missing head could make are caught with guard regions around `out` and the debug rows."""
import itertools

import numpy as np
import pytest
import torch

from oracle import ref
from tests._attn import BITS, GROUPS, RESIDUALS, checked_call, checked_step, make_cache, rand16

pytestmark = pytest.mark.gpu

D = 128
RATIOS = (3, 5, 6, 7)
MODES = ("unpadded", "ragged", "windowed")


def _cases():
    out = []
    for i, (ratio, kb, vb, g, mode) in enumerate(itertools.product(RATIOS, BITS, BITS, GROUPS, MODES)):
        Rs = [R for R in RESIDUALS if R % g == 0]
        R = Rs[i % len(Rs)]
        out.append(pytest.param(ratio, kb, vb, g, R, mode, id=f"ratio{ratio}-k{kb}v{vb}-g{g}-R{R}-{mode}"))
    return out


def _inputs(rng, B, H, Hkv):
    return (rand16(rng, (B, H, 1, D), 0.7), rand16(rng, (B, Hkv, 1, D)), rand16(rng, (B, Hkv, 1, D)))


@pytest.mark.parametrize("ratio,kb,vb,g,R,mode", _cases())
def test_partial_head_chunks_match_oracle(ratio, kb, vb, g, R, mode):
    """Two KV heads of `ratio` query heads each, B = 2, a prefill of 3R - 2 tokens, then three checked steps (the
    second completes the K window and flushes it) with G = default (4, or 2 at ratio 6), 2 and 4.  ragged: the second
    sequence starts at min(130, n0 / 2 + 1), inside the first packed block at every R (at R = 128 and 256 one token into
    the second); windowed: a window of half the prefill."""
    B, Hkv = 2, 2
    H = ratio * Hkv
    n0 = 3 * R - 2
    starts = [0, min(130, n0 // 2 + 1)] if mode == "ragged" else None
    window = n0 // 2 if mode == "windowed" else None
    for G in (0, 2, 4):
        rng = np.random.default_rng(ratio * 1000 + kb * 100 + vb * 10 + g + R + G)
        cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16, gqa_chunk=G)
        k, v = rand16(rng, (B, Hkv, n0, D)), rand16(rng, (B, Hkv, n0, D))
        cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(),
                      kv_start=None if starts is None else torch.tensor(starts))
        st = ref.prefill_cache(k, v, g, kb, vb, R)
        for step in range(3):
            try:
                st = checked_step(cache, st, *_inputs(rng, B, H, Hkv), (g, kb, vb, R), starts=starts, window=window)
            except AssertionError as e:
                raise AssertionError(f"G = {G or 'default'}, step {step}: {e}") from None


GUARD = 4096                    # halfs of sentinel before and after every output the call writes
SENTINEL = 0x7BCD               # an fp16 bit pattern no kernel writes by accident (a large finite value)


def _guarded(shape):
    """A view of `shape` in the middle of a flat fp16 buffer whose GUARD halfs on either side hold SENTINEL."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int16, device="cuda").view(torch.float16)
    view = buf[GUARD:GUARD + n].view(*shape)
    view.zero_()
    return buf, view


def _guards_intact(buf, what):
    bits = buf.view(torch.int16)
    for side, part in (("before", bits[:GUARD]), ("after", bits[-GUARD:])):
        bad = (part != SENTINEL).nonzero().flatten()
        assert bad.numel() == 0, f"{what}: {bad.numel()} halfs written {side} the buffer (first at {bad[:4].tolist()})"


@pytest.mark.parametrize("ratio,mode", list(itertools.product(RATIOS, MODES)))
def test_missing_heads_write_nothing(ratio, mode):
    """`out`, dbg_logits and dbg_probs are views inside larger buffers: after a call at G = 4 (a partial last unit on every
    KV head) every guard half holds its sentinel, the debug rows hold nothing past position T, and the output equals
    the call without debug pointers.  The last KV head's missing heads would write past the end of each buffer."""
    B, Hkv, kb, vb, g, R = 3, 2, 2, 2, 32, 64
    H = ratio * Hkv
    n0 = 3 * R + 7
    rng = np.random.default_rng(ratio)
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16, gqa_chunk=4)
    starts = [0, 70, 129] if mode == "ragged" else None
    if mode == "windowed":
        cache.sliding_window = 100
    k, v = rand16(rng, (B, Hkv, n0, D)), rand16(rng, (B, Hkv, n0, D))
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(),
                  kv_start=None if starts is None else torch.tensor(starts))
    for step in range(2):
        T = cache.kv_len + 1
        q, kn, vn = (torch.from_numpy(np.ascontiguousarray(a[:, :, 0])).cuda() for a in _inputs(rng, B, H, Hkv))
        ob, out = _guarded((B, H, D))
        sb, dbg_s = _guarded((B, H, T + 8))
        pb, dbg_p = _guarded((B, H, T + 8))
        plain = cache.decode_attention(0, q, kn, vn).clone()
        cache.decode_attention(0, q, kn, vn, out=out, dbg_logits=dbg_s, dbg_probs=dbg_p)
        torch.cuda.synchronize()
        for buf, what in ((ob, "out"), (sb, "dbg_logits"), (pb, "dbg_probs")):
            _guards_intact(buf, f"step {step} {what}")
        assert not dbg_s[..., T:].view(torch.int16).any() and not dbg_p[..., T:].view(torch.int16).any()
        assert torch.equal(out.view(torch.int16), plain.view(torch.int16)), "the debug pointers changed the output"
        assert torch.isfinite(out).all()
        cache.advance()


@pytest.mark.parametrize("ratio", RATIOS)
def test_every_head_is_computed(ratio):
    """A direct check that no head is skipped or swapped: each query head of a ratio-`ratio` KV head gets a q of its own
    magnitude, so the heads' outputs differ; at G = 4 the output of every head matches the oracle (checked_call), including
    the last unit's real heads, and no two of the kernel's output rows are equal."""
    B, Hkv, kb, vb, g, R = 1, 1, 4, 4, 64, 64
    H = ratio * Hkv
    n0 = 2 * R + 5
    rng = np.random.default_rng(100 + ratio)
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8, gqa_chunk=4)
    k, v = rand16(rng, (B, Hkv, n0, D)), rand16(rng, (B, Hkv, n0, D))
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    q = np.stack([rand16(rng, (B, 1, 1, D), 0.3 * (h + 1))[:, 0] for h in range(H)], axis=1)
    kn, vn = _inputs(rng, B, H, Hkv)[1:]
    checked_call(cache, st, q, kn, vn, (g, kb, vb, R))
    # the same call again (checked_call does not advance the cache): the kernel's own rows
    got = cache.decode_attention(0, *(torch.from_numpy(np.ascontiguousarray(a[:, :, 0])).cuda() for a in (q, kn, vn)))
    rows = got.reshape(H, D).view(torch.int16).cpu()
    assert len({tuple(r.tolist()) for r in rows}) == H, "two heads have the same output row"

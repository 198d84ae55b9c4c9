"""Sliding-window decode attention on the fused cache (kivi_decode_attention_window_f16): against the oracle's decode step
given the window as an additive finfo(fp16).min mask, a window that covers everything against the unpadded entry (bit for
bit), packed blocks below the window not read, the cache update, and the step captured in a CUDA graph while T moves."""
import numpy as np
import pytest
import torch

from oracle import ref
from tests._attn import NEG16, assert_e2e, checked_call, hidden_mask, make_cache, rand16, tuple_equal

pytestmark = pytest.mark.gpu

CASES = [  # kb, vb, g, R, H, Hkv  (G = 4 / 2 / 1 from H / Hkv; the 4-bit K G = 4 kernels run 12 warps per CTA)
    (2, 2, 32, 128, 4, 1),
    (2, 4, 64, 64, 2, 1),
    (4, 2, 128, 128, 2, 2),
    (4, 4, 64, 64, 8, 2),
    (4, 4, 32, 256, 2, 2),
    (2, 2, 128, 128, 4, 2),
    (4, 2, 32, 32, 4, 1),
    (2, 4, 32, 128, 3, 3),
]


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", CASES)
def test_window_matches_oracle(kb, vb, g, R, H, Hkv, padded):
    """Several windows per step (1, below R, inside a packed block, on a block edge, two blocks, beyond T), with and without
    kv_start, over steps that cross a K flush and a V-ring wrap: every window by the suite's check against the oracle with
    the equivalent mask (dbg_probs 0 below the window: the partly visible block writes zeros there, blocks that are not
    read leave the zeroed buffer as it is), and the cache after every step bit-identical to a twin driven by the unpadded
    entry."""
    dev = torch.device("cuda")
    rng = np.random.default_rng(kb * 1000 + vb * 100 + g + R + H + int(padded))
    B = 4
    n0 = max(3, -(-600 // R)) * R + R - 3                            # r = R - 3: the K window flushes at step 3
    steps = 6
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16, sliding_window=1)
    twin = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16)
    k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
    starts = [0, 130, 257, n0 - 50] if padded else None
    cache.prefill(0, torch.from_numpy(k).to(dev), torch.from_numpy(v).to(dev),
                  kv_start=None if starts is None else torch.tensor(starts))
    twin.prefill(0, torch.from_numpy(k).to(dev), torch.from_numpy(v).to(dev))
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    for step in range(steps):
        T = cache.kv_len + 1
        q, kn, vn = rand16(rng, (B, H, 1, 128), 0.7), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
        qd, kd, vd = (torch.from_numpy(np.ascontiguousarray(a[:, :, 0])).to(dev) for a in (q, kn, vn))
        for W in (1, R // 2, 200, 256, 384, T + 5):
            try:
                _, _, nxt, _ = checked_call(cache, st, q, kn, vn, (g, kb, vb, R), starts=starts, window=W)
            except AssertionError as e:
                raise AssertionError(f"step {step} W {W}: {e}") from None
        twin.decode_attention(0, qd, kd, vd)
        st = nxt
        cache.advance()
        twin.advance()
        tuple_equal(cache.export(0), twin.export(0), f"step {step}")
    assert cache.read_state() == twin.read_state()


@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", CASES[:4])
def test_window_covering_everything_is_the_unpadded_call(kb, vb, g, R, H, Hkv):
    """W >= T: the same work split and arithmetic as the unpadded entry, bit for bit."""
    dev = torch.device("cuda")
    rng = np.random.default_rng(5 + kb + g)
    B, n0 = 3, 5 * R + 17
    a, b = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8, sliding_window=n0 + 1), make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8)
    k, v = (torch.from_numpy(rand16(rng, (B, Hkv, n0, 128))).to(dev) for _ in range(2))
    a.prefill(0, k, v)
    b.prefill(0, k, v)
    for step in range(4):
        q, kn, vn = (torch.from_numpy(rand16(rng, s)).to(dev) for s in ((B, H, 128), (B, Hkv, 128), (B, Hkv, 128)))
        oa, ob = a.decode_attention(0, q, kn, vn), b.decode_attention(0, q, kn, vn)
        assert torch.equal(oa.view(torch.int16), ob.view(torch.int16)), f"step {step}"
        a.sliding_window += 1
        a.advance()
        b.advance()


def test_blocks_below_the_window_are_not_read():
    """NaN bytes in the codes, scales and zeros of every packed block wholly below the window: the windowed output is the
    clean cache's, bit for bit; the same poisoned cache through the mask path gives NaN (the poison landed)."""
    dev = torch.device("cuda")
    rng = np.random.default_rng(9)
    B, H, Hkv, kb, vb, g, R, n0, W = 3, 4, 2, 2, 4, 32, 128, 1000, 300
    clean = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8, sliding_window=W)
    k, v = (torch.from_numpy(rand16(rng, (B, Hkv, n0, 128))).to(dev) for _ in range(2))
    clean.prefill(0, k, v)
    T = clean.kv_len + 1
    nb = (T - W) // 128                                              # blocks wholly below T - W
    assert nb >= 2 and nb * 128 <= min(clean.tk, clean.tv)
    tup = [t.clone() if torch.is_tensor(t) else t for t in clean.export(0)]
    nan_word = torch.tensor(0x7E007E00, dtype=torch.int32)           # two fp16 NaN halves
    tup[0][..., :nb * 128 * kb // 32] = nan_word                     # K codes [B, Hkv, 128, tk * kb / 32]
    tup[2][..., :nb * 128 // g] = float("nan")                       # K scales / zeros [B, Hkv, 128, tk / g]
    tup[3][..., :nb * 128 // g] = float("nan")
    tup[4][:, :, :nb * 128] = nan_word                               # V codes [B, Hkv, tv, 128 * vb / 32]
    tup[6][:, :, :nb * 128] = float("nan")                           # V scales / zeros [B, Hkv, tv, 128 / g]
    tup[7][:, :, :nb * 128] = float("nan")
    bad = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8, sliding_window=W)
    bad.import_tuple(0, tuple(tup))
    q, kn, vn = (torch.from_numpy(rand16(rng, s)).to(dev) for s in ((B, H, 128), (B, Hkv, 128), (B, Hkv, 128)))
    out_clean = clean.decode_attention(0, q, kn, vn).clone()
    out_bad = bad.decode_attention(0, q, kn, vn).clone()
    torch.cuda.synchronize()
    assert not torch.isnan(out_clean).any()
    assert torch.equal(out_clean.view(torch.int16), out_bad.view(torch.int16)), "poisoned blocks below the window"
    bad.sliding_window = None                                        # the same cache through the additive-mask path
    m = torch.zeros((B, T), dtype=torch.float16, device=dev)
    m[:, :T - W] = float(NEG16)
    out_mask = bad.decode_attention(0, q, kn, vn, mask=m)
    torch.cuda.synchronize()
    assert torch.isnan(out_mask).any(), "the poison did not reach the mask path"


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", [(2, 2, 32, 128, 4, 1), (4, 4, 64, 64, 8, 2)])
def test_window_in_captured_step(kb, vb, g, R, H, Hkv, padded):
    """The attention call and the cache advance captured once in a CUDA graph, replayed while T (and with it the window's
    first block) moves across several packed blocks: every replay against the oracle."""
    dev = torch.device("cuda")
    rng = np.random.default_rng(21 + kb + int(padded))
    B, n0, W, steps = 3, 4 * R + R - 3, 160, 40
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + steps + 4, sliding_window=W)
    k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
    starts = [0, 70, n0 - 30] if padded else None
    cache.prefill(0, torch.from_numpy(k).to(dev), torch.from_numpy(v).to(dev),
                  kv_start=None if starts is None else torch.tensor(starts))
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    qb, kb_, vb_ = (torch.zeros(s, dtype=torch.float16, device=dev) for s in ((B, H, 128), (B, Hkv, 128), (B, Hkv, 128)))
    out = torch.zeros_like(qb)
    state0 = cache.state.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                       # warm-up outside the capture
        cache.decode_attention(0, qb, kb_, vb_, out=out)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cache.decode_attention(0, qb, kb_, vb_, out=out)
        cache._enqueue_advance()
    cache.state.copy_(state0)                                        # capture does not execute; the warm-up did not advance
    for step in range(steps):
        T = cache.kv_len + 1
        q, kn, vn = rand16(rng, (B, H, 1, 128), 0.7), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
        for dst, src in ((qb, q), (kb_, kn), (vb_, vn)):
            dst.copy_(torch.from_numpy(np.ascontiguousarray(src[:, :, 0])))
        graph.replay()
        cache._mirror_advance()
        torch.cuda.synchronize()
        exp_out, _, st = ref.decode_step(st, q, kn, vn, g, kb, vb, R, hidden_mask(B, T, starts, W))
        assert_e2e(out.cpu().numpy()[:, :, None, :], exp_out, f"replay {step}")
    assert cache.read_state()[:6] == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]

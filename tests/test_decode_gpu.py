"""Parity of the pre-allocated cache + fused decode-attention kernel (kivi_cache.cu, kivi_decode.cu)
with the restated attention hook of the reference (oracle/ref.py: models/llama_kivi.py:314-455).

Cache contents (codes, scale, mn, fp16 windows) are compared BIT-EXACTLY with the oracle's 9-tuple; the attention
output stage by stage and end to end by the suite's check (tests/_attn.py)."""
import numpy as np
import pytest
import torch

from oracle import ref
from tests._attn import (RAGGED_STARTS, _slab, assert_e2e, check_stages, checked_step, hidden_mask, instantiation_cases,
                         make_cache, mirror_lengths, rand16, tuple_equal)
from tests._util import to_np

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[0, 1], ids=["G-auto", "G-1"])
def gqa_chunk(request):
    """G-auto: the query heads of a KV head share the MMAs (chunks of up to 4, KIVI_CACHE_GQA_CHUNK = 0);
    G-1: one head per unit (KIVI_CACHE_GQA_CHUNK(1))."""
    return request.param


@pytest.mark.parametrize("n", [1, 5, 128, 200, 333, 640])
@pytest.mark.parametrize("kb,vb,g,R", [(2, 2, 32, 128), (4, 4, 64, 64), (2, 4, 32, 32), (4, 2, 128, 128)])
def test_prefill_matches_oracle(n, kb, vb, g, R):
    """kivi_cache_prefill_f16 == the prefill split + pack of models/llama_kivi.py:425-452, bit for bit."""
    rng = np.random.default_rng(n * 31 + kb + R)
    B, H, Hkv = 2, 4, 2
    k, v = rand16(rng, (B, Hkv, n, 128)), rand16(rng, (B, Hkv, n, 128))
    cache = make_cache(B, H, Hkv, kb, vb, g, R)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    tuple_equal(cache.export(0), ref.prefill_cache(k, v, g, kb, vb, R), "prefill")
    assert to_np(cache.state)[:6].tolist() == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]


DECODE_CASES = [  # B, H, Hkv, kb, vb, g, R, n_prefill, steps
    (1, 2, 2, 2, 2, 32, 128, 300, 140),     # crosses a K flush (r: 44 -> 128) and V ring wrap-around
    (2, 4, 1, 2, 2, 32, 32, 70, 40),        # GQA 4 (G = 4), R = 32: several flushes
    (1, 8, 1, 4, 4, 64, 64, 130, 70),       # ratio 8 -> two chunks of 4, 4-bit g64
    (1, 2, 1, 2, 4, 32, 64, 10, 80),        # G = 2, mixed bits, starts below R (no packed part at first)
    (1, 3, 3, 4, 2, 128, 128, 0, 135),      # decode from an EMPTY cache, g = 128
    (1, 2, 1, 4, 2, 64, 256, 250, 20),      # R = 256: a K flush fills two 128-token blocks (step 6)
    (2, 2, 2, 2, 2, 128, 256, 250, 20),     # R = 256, g = 128, 2-bit: flush at step 6 into blocks 0 and 1
]


@pytest.mark.parametrize("B,H,Hkv,kb,vb,g,R,n0,steps", DECODE_CASES)
def test_decode_steps_match_oracle(B, H, Hkv, kb, vb, g, R, n0, steps, gqa_chunk):
    """Every step: the production and instrumented epilogues give the same bits and the output meets the oracle end to
    end.  For time, only some steps (the first and last three, every 9th, and those around a K flush) are fully checked
    (checked_step: every stage, and the exported cache bit for bit)."""
    rng = np.random.default_rng(n0 * 13 + H + R)
    cfg = (g, kb, vb, R)
    cache = make_cache(B, H, Hkv, kb, vb, g, R, 512, gqa_chunk=gqa_chunk)
    if n0 > 0:
        k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
        cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
        st = ref.prefill_cache(k, v, *cfg)
    else:
        st = (None, None, None, None, None, np.zeros((B, Hkv, 0, 128), np.float16), None, None, 0)
    dbg_s = torch.zeros((B, H, 512), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    for step in range(steps):
        q, k_new, v_new = rand16(rng, (B, H, 1, 128), 0.7), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
        if step < 3 or step % 9 == 0 or step >= steps - 3 or st[1] is None or st[1].shape[2] >= R - 2:
            st = checked_step(cache, st, q, k_new, v_new, cfg)
            continue
        qd, kd, vd = (torch.from_numpy(a[:, :, 0]).cuda() for a in (q, k_new, v_new))
        # the production epilogue first (no debug pointers: the branch bench.py runs), then the instrumented one on the
        # same state -- every instantiation the cases reach (<2,4,32>, G = 2, g = 128, ...) must give the same bits
        out_fast = cache.decode_attention(0, qd, kd, vd).clone()
        out = cache.decode_attention(0, qd, kd, vd, dbg_logits=dbg_s, dbg_probs=dbg_p)
        assert torch.equal(out_fast, out), f"step {step}: fast and instrumented epilogues disagree"
        cache.advance()
        exp_out, _, st = ref.decode_step(st, q, k_new, v_new, *cfg)
        assert_e2e(to_np(out)[:, :, None, :], exp_out, f"step {step}")
    assert cache.read_state()[:6] == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]


# ---------------------------------------------------------------------------------------------------
# every attention instantiation against the oracle: k_bits x v_bits x g x G x {unpadded, ragged}
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kb,vb,g,G,R,ratio,ragged", instantiation_cases("ragged"))
def test_every_instantiation_matches_oracle(kb, vb, g, G, R, ratio, ragged):
    """Every (k_bits, v_bits, g, G, RAGGED) kernel pair the dispatcher can pick, against the C oracle: prefill to
    r = R - 3, then six steps that cross a K flush and move the V ring head, every step fully checked (checked_step).
    Ragged cases: one sequence unpadded, the others with whole 128-token blocks skipped, partly padded blocks, and
    starts inside the fp16 K and V windows; the oracle runs with the equivalent additive mask."""
    Hkv = 2 if ratio == G else 1
    H = ratio * Hkv
    n0 = max(3, -(-540 // R)) * R + R - 3
    rng = np.random.default_rng(1000 * kb + 100 * vb + g + 7 * G + R + ratio + 3 * ragged)
    B = 6 if ragged else 2
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16, gqa_chunk=G)
    k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
    starts = None
    if ragged:
        tk, r, tv, L = mirror_lengths(n0, R)
        starts = RAGGED_STARTS + [tk + r // 2, tv + L // 2]
        assert len(starts) == B and max(starts) < n0
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(),
                  kv_start=None if starts is None else torch.tensor(starts))
    assert cache.ragged == ragged
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    r0 = cache.r
    for step in range(6):
        q, k_new, v_new = rand16(rng, (B, H, 1, 128), 0.7), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
        st = checked_step(cache, st, q, k_new, v_new, (g, kb, vb, R), starts=starts)
    assert r0 == R - 3 and cache.r == 3 and cache.vhead != 0, "the steps crossed a K flush and moved the V ring head"
    assert cache.read_state()[:6] == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]


def test_decode_with_mask(gqa_chunk):
    """Additive mask + max with finfo.min (models/llama_kivi.py:364-372), e.g. left padding."""
    rng = np.random.default_rng(4)
    B, H, Hkv, kb, vb, g, R, n0 = 2, 2, 2, 2, 2, 32, 128, 200
    cache = make_cache(B, H, Hkv, kb, vb, g, R, 512, gqa_chunk=gqa_chunk)
    k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    T = n0 + 1
    mask = hidden_mask(B, T, [17, 3])                                # sequence 0 is left-padded by 17 tokens, 1 by 3
    q, k_new, v_new = rand16(rng, (B, H, 1, 128)), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
    dbg_s = torch.zeros((B, H, 512), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out = cache.decode_attention(0, torch.from_numpy(q[:, :, 0]).cuda(), torch.from_numpy(k_new[:, :, 0]).cuda(),
                                 torch.from_numpy(v_new[:, :, 0]).cuda(), mask=torch.from_numpy(mask).cuda(),
                                 dbg_logits=dbg_s, dbg_probs=dbg_p)
    torch.cuda.synchronize()
    check_stages(st, q, k_new, v_new, (g, kb, vb, R), to_np(out)[:, :, None, :], to_np(dbg_s)[:, :, None, :],
                 to_np(dbg_p)[:, :, None, :], mask)


def test_multi_layer_shared_state():
    """All layers share one device state; decode of layer l must not disturb layer m."""
    rng = np.random.default_rng(8)
    B, H, Hkv, g, R, n0, NL = 1, 2, 2, 32, 128, 150, 3
    cache = make_cache(B, H, Hkv, 2, 2, g, R, 512, n_layers=NL)
    sts = []
    for l in range(NL):
        k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
        cache.prefill(l, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
        sts.append(ref.prefill_cache(k, v, g, 2, 2, R))
    for step in range(4):
        for l in range(NL):
            q, kn, vn = rand16(rng, (B, H, 1, 128)), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
            cache.decode_attention(l, torch.from_numpy(q[:, :, 0]).cuda(), torch.from_numpy(kn[:, :, 0]).cuda(),
                                   torch.from_numpy(vn[:, :, 0]).cuda())
            _, _, sts[l] = ref.decode_step(sts[l], q, kn, vn, g, 2, 2, R)
        cache.advance()
    for l in range(NL):
        tuple_equal(cache.export(l), sts[l], f"layer {l}")


def test_full_size_consistency(gqa_chunk):
    """BASELINE cfg 2 layer shape (B32, H32, T = 4096, K2V2 g32 R128): too big for the CPU oracle end to
    end, so (1) a slab of units is checked stage-by-stage against the oracle, (2) the fused kernel must
    agree with the library's own generic-layout kernels run on the exported cache for ALL units
    (two independent code paths), (3) probabilities sum to 1."""
    from kivi_b200 import matmul
    gen = torch.Generator(device="cuda").manual_seed(3)
    B, H, Hkv, g, R, n0 = 32, 32, 32, 32, 128, 4095
    cache = make_cache(B, H, Hkv, 2, 2, g, R, 4352, gqa_chunk=gqa_chunk)
    k = torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16)
    v = torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16)
    cache.prefill(0, k, v)
    del k, v
    tup = cache.export(0)
    q = torch.randn((B, H, 128), generator=gen, device="cuda", dtype=torch.float16)
    kn = torch.randn((B, Hkv, 128), generator=gen, device="cuda", dtype=torch.float16)
    vn = torch.randn((B, Hkv, 128), generator=gen, device="cuda", dtype=torch.float16)
    dbg_s = torch.zeros((B, H, 4352), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out = cache.decode_attention(0, q, kn, vn, dbg_logits=dbg_s, dbg_probs=dbg_p)
    torch.cuda.synchronize()
    T = n0 + 1
    assert cache.tk == 3968 and cache.r == 127 and cache.tv == 3967 and cache.L == 128
    # (3)
    psum = dbg_p[..., :T].float().sum(-1)
    assert bool(((psum - 1).abs() < 2e-2).all())
    # (2) generic kernels on the exported (reference-layout) cache
    lq = matmul.cuda_bmm_fA_qB_outer(g, q[:, :, None, :], tup[0], tup[2], tup[3], 2)[:, :, 0]
    s_generic = (lq.float() * (1.0 / 11.313708)).half()
    diff = (dbg_s[..., :3968].float() - s_generic.float()).abs()
    assert bool((diff <= 1e-3 * s_generic.float().abs() + 2e-3).all()), float(diff.max())
    oq = matmul.cuda_bmm_fA_qB_outer(g, dbg_p[:, :, None, :3967], tup[4], tup[6], tup[7], 2)[:, :, 0]
    vfull = torch.cat([tup[5], vn[:, :, None, :]], dim=2)
    orr = torch.matmul(dbg_p[:, :, None, 3967:T].float(), vfull.float())[:, :, 0].half()
    exp = (oq + orr)
    d2 = (out.float() - exp.float()).abs()
    assert bool((d2 <= 2e-3 * exp.float().abs() + 2e-4).all()), float(d2.max())
    # (1) oracle on a slab
    sl = slice(7, 8)
    st = tuple(None if t is None else (t if isinstance(t, int) else to_np(t[sl, :2])) for t in tup[:8]) + (tup[8],)
    check_stages(st, to_np(q[sl, :2])[:, :, None, :], to_np(kn[sl, :2])[:, :, None, :], to_np(vn[sl, :2])[:, :, None, :],
                 (g, 2, 2, R), to_np(out[sl, :2])[:, :, None, :], to_np(dbg_s[sl, :2])[:, :, None, :],
                 to_np(dbg_p[sl, :2])[:, :, None, :], None)


@pytest.mark.parametrize("B,H,Hkv,kb,vb,g,R,n0", [(1, 8, 2, 4, 4, 64, 64, 20000),      # cfg-4-like: few, long units, GQA 4, 4-bit
                                                  (2, 4, 4, 2, 2, 32, 128, 9000)])     # MHA, more ranges per unit than warps of a CTA
def test_long_context_many_ranges_per_unit(B, H, Hkv, kb, vb, g, R, n0):
    """Few long units: every unit is cut into many warp ranges (more than 32 statistic slots and partial records per
    unit), far beyond what a logits row in shared memory could hold.  Checked against the library's generic-layout
    kernels run on the exported cache (an independent code path) and against the softmax identities."""
    from kivi_b200 import matmul
    gen = torch.Generator(device="cuda").manual_seed(11)
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 64)
    k = torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16)
    v = torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16)
    cache.prefill(0, k, v)
    del k, v
    tup = cache.export(0)
    q = (torch.randn((B, H, 128), generator=gen, device="cuda", dtype=torch.float32) * 0.5).half()
    kn = torch.randn((B, Hkv, 128), generator=gen, device="cuda", dtype=torch.float16)
    vn = torch.randn((B, Hkv, 128), generator=gen, device="cuda", dtype=torch.float16)
    T = n0 + 1
    dbg_s = torch.zeros((B, H, T + 8), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out = cache.decode_attention(0, q, kn, vn, dbg_logits=dbg_s, dbg_probs=dbg_p)
    out2 = cache.decode_attention(0, q, kn, vn)                     # same state (no advance): the fast path, same result
    torch.cuda.synchronize()
    assert torch.equal(out, out2), "debug and fast paths disagree"
    tk, tv, L = cache.tk, cache.tv, cache.L
    psum = dbg_p[..., :T].float().sum(-1)
    assert bool(((psum - 1).abs() < 2e-2).all())
    lq = matmul.cuda_bmm_fA_qB_outer(g, q[:, :, None, :], tup[0], tup[2], tup[3], kb)[:, :, 0]
    s_generic = (lq.float() * (1.0 / 11.313708)).half()
    diff = (dbg_s[..., :tk].float() - s_generic.float()).abs()
    assert bool((diff <= 1e-3 * s_generic.float().abs() + 2e-3).all()), float(diff.max())
    # softmax of the kernel's own logits
    p_ref = torch.softmax(dbg_s[..., :T].float(), -1)
    assert bool(((dbg_p[..., :T].float() - p_ref).abs() <= 2e-3 * p_ref + 1e-6).all())
    oq = matmul.cuda_bmm_fA_qB_outer(g, dbg_p[:, :, None, :tv], tup[4], tup[6], tup[7], vb)[:, :, 0]
    rep = H // Hkv
    vfull = torch.cat([tup[5], vn[:, :, None, :]], dim=2).repeat_interleave(rep, dim=1)
    orr = torch.matmul(dbg_p[:, :, None, tv:T].float(), vfull.float())[:, :, 0].half()
    exp = (oq + orr)
    d2 = (out.float() - exp.float()).abs()
    assert bool((d2 <= 2e-3 * exp.float().abs() + 2e-4).all()), float(d2.max())


# ---------------------------------------------------------------------------------------------------
# BASELINE.json configs at full size: the fused path against the oracle on slabs of units, fast == instrumented on all
# ---------------------------------------------------------------------------------------------------
FULL_CONFIGS = {   # name: B, H, Hkv, kb, vb, g, R, kv length after the step, slabs (batch, kv head)
    "cfg2-llama2-7b-bs32-4k": (32, 32, 32, 2, 2, 32, 128, 4096, [(0, 0), (13, 17), (31, 31)]),
    "cfg3-llama3-8b-gqa-bs64-8k": (64, 32, 8, 2, 2, 32, 128, 8192, [(0, 0), (37, 5), (63, 7)]),
    "cfg4-mistral-7b-k4v4-bs16-32k": (16, 32, 8, 4, 4, 64, 64, 32768, [(0, 0), (9, 3), (15, 7)]),
    "cfg5-shard-bs128-4k": (128, 32, 32, 2, 2, 32, 128, 4096, [(0, 0), (127, 31)]),
}


@pytest.mark.parametrize("name", list(FULL_CONFIGS))
def test_baseline_configs_full_size(name):
    """The shapes BASELINE.json quotes its metric on (cfg 4 as g64 / R64: the reference rejects R32 with g64,
    models/mistral_kivi.py:402).  One decode step of one layer through the fused path at FULL size:
      * three slabs (first, middle, last unit -- different warps, different range cuts) by the suite's check (stage by
        stage against the C oracle of the reference kernels, end to end) and bit-exactly on the updated cache;
      * the production epilogue (no debug pointers) equals the instrumented one on ALL units, bit for bit;
      * every probability row sums to 1 and the device-side guard word stays clear."""
    B, H, Hkv, kb, vb, g, R, T, slabs = FULL_CONFIGS[name]
    n0 = T - 1
    ratio = H // Hkv
    gen = torch.Generator(device="cuda").manual_seed(len(name))
    cache = make_cache(B, H, Hkv, kb, vb, g, R, T + 64)
    k = torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16)
    v = torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16)
    cache.prefill(0, k, v)
    del k, v
    tup = cache.export(0)
    q = (torch.randn((B, H, 128), generator=gen, device="cuda", dtype=torch.float32) * 0.6).half()
    kn = torch.randn((B, Hkv, 128), generator=gen, device="cuda", dtype=torch.float16)
    vn = torch.randn((B, Hkv, 128), generator=gen, device="cuda", dtype=torch.float16)
    dbg_s = torch.zeros((B, H, T + 8), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out_fast = cache.decode_attention(0, q, kn, vn).clone()
    out = cache.decode_attention(0, q, kn, vn, dbg_logits=dbg_s, dbg_probs=dbg_p)
    torch.cuda.synchronize()
    assert torch.equal(out_fast, out), "production and instrumented epilogues disagree"
    psum = dbg_p[..., :T].float().sum(-1)
    assert bool(((psum - 1).abs() < 2e-2).all())
    after = {}
    for b, hk in slabs:
        st, q4, kn4, vn4, out4, s4, p4 = _slab(tup, q, kn, vn, out, dbg_s, dbg_p, b, hk, ratio)
        _, _, after[b, hk], _ = check_stages(st, q4, kn4, vn4, (g, kb, vb, R), out4, s4, p4, None)
    cache.advance()
    assert cache.read_state()[6] == 0
    tup2 = cache.export(0)
    for b, hk in slabs[:2]:                                        # the cache update of the step, bit for bit
        got = tuple(None if t is None else t[b:b + 1, hk:hk + 1] for t in tup2[:8]) + (tup2[8],)
        tuple_equal(got, after[b, hk], f"slab ({b}, {hk})")


# ---------------------------------------------------------------------------------------------------
# the ATen boundary (models/llama_kivi.py:337, :339, :375, :384): cuBLAS batched matmul on the fp16 windows and ATen's
# fp32 softmax are third-party arithmetic the reference's tests never pin; the GPU box runs those exact ops
# ---------------------------------------------------------------------------------------------------
def _ulp_steps(a, b):
    """Distance in fp16 representable steps between two fp16 tensors of the same sign structure."""
    ai = a.view(torch.int16).to(torch.int32)
    bi = b.view(torch.int16).to(torch.int32)
    ai = torch.where(ai < 0, -(ai & 0x7fff), ai)
    bi = torch.where(bi < 0, -(bi & 0x7fff), bi)
    return (ai - bi).abs()


@pytest.mark.parametrize("B,H,Hkv,n0", [(2, 4, 4, 100), (3, 8, 2, 127), (1, 4, 1, 60)])
def test_window_and_softmax_against_aten(B, H, Hkv, n0):
    """No packed part yet (n0 < R = 128): the whole step is the reference's ATen code -- torch.matmul on fp16 (:337),
    `/ math.sqrt(head_dim)` (:339), F.softmax(dtype=float32).to(fp16) (:375), torch.matmul (:380).  Run exactly those
    ops on the GPU and compare (a) the kernel, (b) the C oracle's restatement, pinning both at this boundary."""
    import math
    import torch.nn.functional as F
    from kivi_b200.llama_kivi import repeat_kv
    g, R = 32, 128
    rng = np.random.default_rng(n0)
    k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
    q, kn, vn = rand16(rng, (B, H, 1, 128), 0.8), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
    cache = make_cache(B, H, Hkv, 2, 2, g, R, 256)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    T = n0 + 1
    dbg_s = torch.zeros((B, H, 256), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out = cache.decode_attention(0, torch.from_numpy(q[:, :, 0]).cuda(), torch.from_numpy(kn[:, :, 0]).cuda(),
                                 torch.from_numpy(vn[:, :, 0]).cuda(), dbg_logits=dbg_s, dbg_probs=dbg_p)
    rep = H // Hkv
    qd = torch.from_numpy(q).cuda()
    Kf = torch.cat([torch.from_numpy(k).cuda(), torch.from_numpy(kn).cuda()], dim=2)
    Vf = torch.cat([torch.from_numpy(v).cuda(), torch.from_numpy(vn).cuda()], dim=2)
    # ---- the reference's ops, verbatim
    att = torch.matmul(qd, repeat_kv(Kf, rep).transpose(2, 3))                       # :337 (cuBLAS, fp16 out)
    s_aten = att / math.sqrt(128)                                                     # :339
    p_aten = F.softmax(s_aten, dim=-1, dtype=torch.float32).to(torch.float16)         # :375
    o_aten = torch.matmul(p_aten, repeat_kv(Vf, rep))                                 # :380
    # (a) kernel: scaled logits equal ATen's except where the two fp32 summation orders round the fp16 logit apart
    s_k = dbg_s[:, :, None, :T]
    steps = _ulp_steps(s_k.contiguous(), s_aten.contiguous())
    assert int(steps.max()) <= 2, f"scaled window logits: {int(steps.max())} fp16 steps from ATen"
    assert float((steps == 0).float().mean()) > 0.9
    # softmax of the kernel's own logits == ATen's softmax of the same logits, to one fp16 step
    p_own = F.softmax(s_k.contiguous(), dim=-1, dtype=torch.float32).to(torch.float16)
    p_k = dbg_p[:, :, None, :T].contiguous()
    st2 = _ulp_steps(p_k, p_own)
    assert int(st2.max()) <= 1, f"probabilities: {int(st2.max())} fp16 steps from ATen softmax"
    assert float((st2 == 0).float().mean()) > 0.9
    # output from the kernel's own probabilities with ATen's matmul
    o_own = torch.matmul(p_k, repeat_kv(Vf, rep))
    err = (out[:, :, None, :].float() - o_own.float()).abs()
    assert bool((err <= 1e-3 * o_own.float().abs() + 2e-4).all()), float(err.max())
    assert_e2e(to_np(out)[:, :, None, :], to_np(o_aten), "kernel against ATen")
    # (b) the C oracle's restatement of these ATen ops (fp32 accumulate in index order, one fp16 rounding)
    att_o = ref.residual_qk(q, np.concatenate([k, kn], axis=2))
    so = _ulp_steps(torch.from_numpy(att_o).cuda(), att.contiguous())
    assert int(so.max()) <= 1 and float((so == 0).float().mean()) > 0.9, "oracle residual_qk vs torch.matmul"
    p_o = ref.scale_softmax(to_np(att), 128)
    sp = _ulp_steps(torch.from_numpy(p_o).cuda(), p_aten.contiguous())
    assert int(sp.max()) <= 1 and float((sp == 0).float().mean()) > 0.9, "oracle scale_softmax vs ATen div + softmax"
    o_o = ref.residual_pv(to_np(p_aten), np.concatenate([v, vn], axis=2))
    eo = (torch.from_numpy(o_o).cuda().float() - o_aten.float()).abs()
    assert bool((eo <= 1e-3 * o_aten.float().abs() + 2e-4).all()), "oracle residual_pv vs torch.matmul"


# ---------------------------------------------------------------------------------------------------
# import of the reference's 9-tuple, device-side capacity guard, second device
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,Hkv,kb,vb,g,R,n0,steps", [(2, 4, 2, 2, 2, 32, 128, 300, 5), (1, 8, 2, 4, 4, 64, 64, 200, 70),
                                                        (2, 2, 2, 2, 4, 32, 32, 20, 3), (1, 2, 1, 4, 2, 128, 128, 0, 0)])
def test_import_tuple_roundtrip(B, H, Hkv, kb, vb, g, R, n0, steps):
    """KiviCache.import_tuple is the inverse of export (models/llama_kivi.py:454-455): export -> import into a fresh
    cache -> export gives the same tuple bit for bit, and both caches then decode identically."""
    gen = torch.Generator(device="cuda").manual_seed(n0 + R)
    a = make_cache(B, H, Hkv, kb, vb, g, R, 512)
    if n0:
        a.prefill(0, torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16),
                  torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16))
    mk = lambda *s: torch.randn(s, generator=gen, device="cuda", dtype=torch.float16)   # noqa: E731
    for _ in range(steps):                                           # ring wrap / flushes before the export
        a.decode_attention(0, mk(B, H, 128), mk(B, Hkv, 128), mk(B, Hkv, 128))
        a.advance()
    tup = a.export(0)
    b = make_cache(B, H, Hkv, kb, vb, g, R, 512)
    b.import_tuple(0, tup)
    assert b.read_state()[:6] == [a.tk, a.r, a.tv, a.L, 0, a.kv_len]
    tup_b = b.export(0)
    assert tup_b[8] == tup[8]
    for i in range(8):
        if tup[i] is None:
            assert tup_b[i] is None
        else:
            assert torch.equal(tup[i], tup_b[i]), f"tuple[{i}]"
    for _ in range(R + 3):                                           # continue on both, flushes included
        q, kn, vn = mk(B, H, 128), mk(B, Hkv, 128), mk(B, Hkv, 128)
        oa, ob = a.decode_attention(0, q, kn, vn), b.decode_attention(0, q, kn, vn)
        # same cache CONTENTS, but the imported V ring starts at slot 0: its 16-token window items are cut at other
        # places, so the fp32 partial sums are added in another order (bit-equal only when the ring heads coincide)
        if a.vhead == b.vhead:
            assert torch.equal(oa, ob)
        err = (oa.float() - ob.float()).abs()
        assert bool((err <= 1e-3 * oa.float().abs() + 1e-3 * float(oa.float().abs().max())).all()), float(err.max())
        a.advance(), b.advance()
    ta, tb = a.export(0), b.export(0)
    for i in range(8):
        assert (ta[i] is None and tb[i] is None) or torch.equal(ta[i], tb[i]), f"tuple[{i}] after decoding on"


def test_import_continues_a_reference_style_cache():
    """A cache grown by the reference's hook semantics (kivi_prefill_tuple / kivi_decode_attention_tuple: torch.cat
    growth, per-op launches) is imported and the fused path continues where the tuple path would: outputs within the
    end-to-end tolerance, packed cache contents bit-equal."""
    from kivi_b200.llama_kivi import kivi_decode_attention_tuple, kivi_prefill_tuple
    B, H, Hkv, kb, vb, g, R, n0 = 2, 8, 2, 2, 2, 32, 128, 260
    gen = torch.Generator(device="cuda").manual_seed(5)
    mk = lambda *s: torch.randn(s, generator=gen, device="cuda", dtype=torch.float16)   # noqa: E731
    past = kivi_prefill_tuple(mk(B, Hkv, n0, 128), mk(B, Hkv, n0, 128), g, kb, vb, R)
    for _ in range(7):
        _, past = kivi_decode_attention_tuple(mk(B, H, 1, 128), mk(B, Hkv, 1, 128), mk(B, Hkv, 1, 128), past, g, kb, vb, R)
    cache = make_cache(B, H, Hkv, kb, vb, g, R, 512)
    cache.import_tuple(0, past)
    for _ in range(130):
        q, kn, vn = mk(B, H, 1, 128) * 0.7, mk(B, Hkv, 1, 128), mk(B, Hkv, 1, 128)
        exp, past = kivi_decode_attention_tuple(q, kn, vn, past, g, kb, vb, R)
        out = cache.decode_attention(0, q[:, :, 0].contiguous(), kn[:, :, 0].contiguous(), vn[:, :, 0].contiguous())
        cache.advance()
        assert_e2e(to_np(out), to_np(exp[:, :, 0]), "fused against the tuple path")
    tup = cache.export(0)
    for i in (0, 2, 3, 4, 6, 7, 1, 5):
        assert (tup[i] is None and past[i] is None) or torch.equal(tup[i], past[i].view_as(tup[i])), f"tuple[{i}]"
    assert tup[8] == past[8]


def test_device_side_capacity_guard():
    """A C-ABI caller whose device-side lengths run past the sizes it declared gets NO memory traffic and an error
    word (KIVI_STATE_ERR_CAPACITY in state[6]) instead of silent out-of-bounds writes."""
    B, H, Hkv = 1, 2, 2
    cache = make_cache(B, H, Hkv, 2, 2, 32, 128, 256)
    gen = torch.Generator(device="cuda").manual_seed(0)
    mk = lambda *s: torch.randn(s, generator=gen, device="cuda", dtype=torch.float16)   # noqa: E731
    cache.prefill(0, mk(B, Hkv, 200, 128), mk(B, Hkv, 200, 128))
    q, kn, vn = mk(B, H, 128), mk(B, Hkv, 128), mk(B, Hkv, 128)
    good = cache.decode_attention(0, q, kn, vn).clone()
    assert cache.read_state()[6] == 0
    before = [b.clone() for b in cache._bufs[0]]
    st = cache.state.clone()
    cache.state[0] = 384                                              # tk: 384 + r 72 + 1 > max_kv_len 256 (the host mirror is bypassed)
    out = torch.full_like(good, 7.0)
    cache.decode_attention(0, q, kn, vn, out=out)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()), "the guarded call must not write the output"
    for x, y in zip(before, cache._bufs[0]):
        assert torch.equal(x, y), "the guarded call must not touch the cache"
    with pytest.raises(RuntimeError, match="refused to run"):
        cache.read_state()
    cache.state.copy_(st)                                             # clears the error word as well
    assert torch.equal(cache.decode_attention(0, q, kn, vn), good)


@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_second_device_in_one_process():
    """Per-device opt-ins (dynamic shared memory) and limits are cached per device ordinal: the same process drives
    cuda:0 and cuda:1 (the reference supports this through device_map="auto")."""
    from kivi_b200.cache import KiviCache
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        gen = torch.Generator(device=dev).manual_seed(3)
        cache = KiviCache(1, 2, 4, 2, 128, 2, 2, 32, 128, 512, device=dev)
        mk = lambda *s: torch.randn(s, generator=gen, device=dev, dtype=torch.float16)   # noqa: E731
        cache.prefill(0, mk(2, 2, 300, 128), mk(2, 2, 300, 128))
        outs.append(cache.decode_attention(0, mk(2, 4, 128), mk(2, 2, 128), mk(2, 2, 128)).cpu())
        torch.cuda.synchronize(dev)
    assert torch.equal(outs[0], outs[1])

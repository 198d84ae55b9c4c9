"""The sliding-window decode attention (kivi_decode_attention_window_f16) against the C oracle, swept the way the ragged and
unpadded entries are: every instantiation at every window-edge position, value magnitudes at the window's edge, long
windows cut into many warp ranges per unit, the benchmarked Mistral-7B layer, the window combined with an additive mask,
and a captured step replayed over a long walk.

Each window is checked as checked_step checks a step (tests/_attn.py), except that the cache is advanced only after the
step's last window: the production and instrumented epilogues give the same bits, every stage matches the oracle
applied to the kernel's previous stage with the equivalent finfo(fp16).min mask below the per-sequence visible start
max(clamp(kv_start), T - W), the output matches end to end at the suite's bar, and the kernel's probabilities are exactly 0
wherever the mask hides a position.  After the step the exported cache equals the oracle's 9-tuple bit for bit.

The window's start s = T - W is placed on purpose, from the host mirror of the lengths (tk, r, tv, L, vhead): on the
edges where the kernels switch between a wholly hidden, a partly visible and a wholly visible item, in every kind of item
(packed K / V block, fp16 K window row, V ring row of either ring segment)."""
import numpy as np
import pytest
import torch

from oracle import ref
from tests._attn import (E2E_ATOL_FRAC, E2E_RTOL, NEG16, _slab, assert_e2e, check_stages, checked_call, hidden_mask,
                         instantiation_cases, make_cache, mirror_lengths, rand16, tuple_equal)
from tests._util import to_np

pytestmark = pytest.mark.gpu

D = 128
SQRT_D = 11.313708


def _step_inputs(rng, B, H, Hkv):
    return rand16(rng, (B, H, 1, D), 0.7), rand16(rng, (B, Hkv, 1, D)), rand16(rng, (B, Hkv, 1, D))


# ---------------------------------------------------------------------------------------------------
# 1. every instantiation x every window-edge class
# ---------------------------------------------------------------------------------------------------
EDGE_CLASSES = ("W=T", "W>T", "block 0", "128j-1", "128j", "128j+1", "tv-1", "tv", "tv+1", "last V block", "[tv,tk)",
                "tk-1", "tk", "tk+1", "ring wrap", "T-2", "T-1")


def _edge_windows(cache):
    """{class: W} for the cache's lengths before a step: W places s = T - W on each edge the kernels treat differently.
    Classes whose edge does not exist at these lengths are left out (the test asserts that its steps reach them all)."""
    tk, tv, L, vhead, T = cache.tk, cache.tv, cache.L, cache.vhead, cache.kv_len + 1
    j = max(1, min(tk, tv) // 256)                                   # a middle block, wholly packed in K and V
    s = {"W=T": 0, "block 0": 37, "128j-1": 128 * j - 1, "128j": 128 * j, "128j+1": 128 * j + 1,
         "tv-1": tv - 1, "tv": tv, "tv+1": tv + 1, "tk-1": tk - 1, "tk": tk, "tk+1": tk + 1, "T-2": T - 2, "T-1": T - 1}
    if tv % 128 >= 2:                                                # inside the last, partly filled packed V block
        s["last V block"] = tv - tv % 128 + (tv % 128) // 2
    if tv < tk:                                                      # K still has a partly visible block; V is in its ring
        x = -(-tv // 128) * 128                                      # where the V items start past the last packed block
        s["[tv,tk)"] = x if x < tk else (tv + tk) // 2
    seg1 = min(L, cache.v_res_cap - vhead)
    if L > seg1:                                                     # the ring's second (wrapped) segment
        s["ring wrap"] = tv + seg1 + (L - seg1) // 2
    out = {k: T - x for k, x in s.items() if 0 <= x <= T - 1}
    out["W>T"] = T + 5
    return out


@pytest.mark.parametrize("kb,vb,g,G,R,ratio,padded", instantiation_cases("padded"))
def test_every_instantiation_at_every_window_edge(kb, vb, g, G, R, ratio, padded):
    """Prefill to r = R - 3 at 600-1000 tokens, then six steps that cross a K flush and wrap the V ring; at every step a
    window per edge class (_edge_windows).  Padded: one unpadded sequence, one start in a partly padded block, one in
    [tv, tk), one in the fp16 K window, so that over the windows both arms of visible_start decide."""
    Hkv = 2 if ratio == G else 1
    H = ratio * Hkv
    n0 = max(3, -(-600 // R)) * R + R - 3
    rng = np.random.default_rng(1000 * kb + 100 * vb + g + 7 * G + R + ratio + 3 * padded)
    B = 4 if padded else 2
    tk0, r0, tv0, _ = mirror_lengths(n0, R)
    starts = [0, 130, tv0 + 1, tk0 + r0 // 2] if padded else None
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16, gqa_chunk=G)
    k, v = rand16(rng, (B, Hkv, n0, D)), rand16(rng, (B, Hkv, n0, D))
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(),
                  kv_start=None if starts is None else torch.tensor(starts))
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    reached, arms = set(), set()
    for step in range(6):
        T = cache.kv_len + 1
        q, kn, vn = _step_inputs(rng, B, H, Hkv)
        by_w = {}
        for cls, W in _edge_windows(cache).items():
            by_w.setdefault(W, []).append(cls)
        for W, classes in sorted(by_w.items()):
            try:
                _, _, nxt, _ = checked_call(cache, st, q, kn, vn, (g, kb, vb, R), starts=starts, window=W)
            except AssertionError as e:
                raise AssertionError(f"step {step}, s = T - W = {T - W} {classes}: {e}") from None
            reached.update(classes)
            for x in (starts or []):
                if 0 < x < T - 1 and T - W > 0:
                    arms.add("window" if T - W > x else "kv_start" if x > T - W else "equal")
        cache.advance()
        st = nxt
        tuple_equal(cache.export(0), st, f"step {step}")
    assert reached == set(EDGE_CLASSES), f"edge classes never reached: {sorted(set(EDGE_CLASSES) - reached)}"
    assert r0 == R - 3 and cache.r == 3 and cache.vhead >= 2, "the steps crossed a K flush and wrapped the V ring"
    if padded:
        assert {"window", "kv_start"} <= arms, f"both arms of visible_start: {arms}"
    assert cache.read_state()[:6] == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]


# ---------------------------------------------------------------------------------------------------
# 2. magnitudes at the window edge
# ---------------------------------------------------------------------------------------------------
EDGE_KERNELS = {   # name: k_bits, v_bits, g, R, G (Hkv = 2, one sequence)
    "cfg2-k2v2-g32-R128-G1": (2, 2, 32, 128, 1),
    "cfg3-k2v2-g32-R128-G4": (2, 2, 32, 128, 4),
    "cfg4-k4v4-g64-R64-G4": (4, 4, 64, 64, 4),
    "k4v2-g128-R128-G2": (4, 2, 128, 128, 2),
}
# where the peaked token p lies: the K item / V item it belongs to
PLACES = ("kblock-vblock", "kblock-vring", "kwindow-vring")
PEAK_LOGIT = 120.0      # scaled logit of the peaked token (the others: about N(0, 0.5))
PEAK_GAP = 100.0        # its least advantage: exp(-PEAK_GAP) is 0 in fp32, so a peak leaked into the maximum zeroes the rest
VBIG = 3.0e4            # |V| of the rows just below the peak: finite scales (range < 65504), large enough to show any leak


def _peak_position(place, tk, tv, g):
    if place == "kblock-vblock":                                     # a middle block; p the last token of a K group (g < 128)
        return 128 * max(1, tv // 256) + (63 if g <= 64 else 100)
    if place == "kblock-vring":
        return tk - 2                                                # packed K, V ring (tv <= tk - 2 in both steps)
    return tk + 1                                                    # fp16 K window row, V ring


@pytest.mark.parametrize("place", PLACES)
@pytest.mark.parametrize("kname", list(EDGE_KERNELS))
def test_magnitudes_at_the_window_edge(kname, place):
    """A token p whose logit exceeds every other by PEAK_GAP, and V rows of magnitude VBIG at p - 3 .. p - 1.  Window
    start s = p + 1 hides the peak just outside (a leak into the running maximum would zero the visible probabilities,
    one into the probabilities would move the output to V[p]); s = p shows it just inside (an off-by-one hiding it moves
    almost all of the mass).  Either way the VBIG rows are hidden, so probabilities of exactly 0 must keep them out.  Two
    steps; the V-token pack of each step packs a VBIG row in the kblock-vring case."""
    kb, vb, g, R, G = EDGE_KERNELS[kname]
    B, Hkv = 1, 2
    H = G * Hkv
    n0 = max(3, -(-900 // R)) * R + R - 3
    tk, r, tv, L = mirror_lengths(n0, R)
    p = _peak_position(place, tk, tv, g)
    rng = np.random.default_rng(PLACES.index(place) * 31 + kb * 7 + vb + g + G)
    k = rng.standard_normal((B, Hkv, n0, D))
    v = rng.standard_normal((B, Hkv, n0, D))
    qbase = rng.standard_normal((B, Hkv, D)) * 0.5
    for hk in range(Hkv):                                            # q . K[p] / sqrt(D) = PEAK_LOGIT for every head
        k[0, hk, p] = PEAK_LOGIT * SQRT_D / float(qbase[0, hk] @ qbase[0, hk]) * qbase[0, hk]
        v[0, hk, p - 3:p] = rng.uniform(-VBIG, VBIG, (3, D))
        v[0, hk, p - 3:p, 0], v[0, hk, p - 3:p, 1] = -VBIG, VBIG
    k, v = k.astype(np.float16), v.astype(np.float16)
    assert np.isfinite(k).all() and np.isfinite(v).all()
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16, gqa_chunk=G)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    cfg = (g, kb, vb, R)
    ratio = H // Hkv
    for step in range(2):
        T = cache.kv_len + 1
        kind_k = "packed" if p < cache.tk else "window"
        kind_v = "packed" if p < cache.tv else "ring"
        assert f"k{'block' if kind_k == 'packed' else 'window'}-v{'block' if kind_v == 'packed' else 'ring'}" == place
        assert p // 128 == (p + 1) // 128 or kind_k == "window", "s = p + 1 lies in the peak's block: partly visible"
        q = np.repeat(qbase[:, :, None, :], ratio, axis=1) + rng.standard_normal((B, H, 1, D)) * 0.01
        q = q.astype(np.float16)
        kn, vn = rand16(rng, (B, Hkv, 1, D)), rand16(rng, (B, Hkv, 1, D))
        # just inside: the peak carries almost all of the mass, and its logit leads every other visible one by PEAK_GAP
        exp_out, exp_p, _, got_s = checked_call(cache, st, q, kn, vn, cfg, window=T - p)
        assert np.isfinite(exp_out).all(), "precondition: the oracle output is finite"
        assert (exp_p[..., p] > 0.99).all(), "precondition: the visible peak carries the mass"
        rest = np.delete(got_s.astype(np.float64), p, axis=-1).max(-1)
        assert (got_s[..., p].astype(np.float64) - rest > PEAK_GAP).all(), "precondition: the peak's logit advantage"
        # just outside: the peak and the VBIG rows hidden
        exp_out, exp_p, nxt, _ = checked_call(cache, st, q, kn, vn, cfg, window=T - p - 1)
        assert np.isfinite(exp_out).all(), "precondition: the oracle output is finite"
        assert (exp_p[..., p - 3:p + 1] == 0).all() and (exp_p.max(-1) < 0.5).all(), "precondition: a spread softmax"
        assert np.abs(exp_out).max() < 10.0, "precondition: the VBIG rows do not reach the oracle output"
        cache.advance()
        st = nxt
        tuple_equal(cache.export(0), st, f"step {step}")
        if st[6] is not None:
            assert np.isfinite(st[6]).all(), "precondition: finite V scales"


# ---------------------------------------------------------------------------------------------------
# 3. long windows: many warp ranges per unit
# ---------------------------------------------------------------------------------------------------
LONG = {   # name: B, H, Hkv, k_bits, v_bits, g, R, G, T, starts
    "k4v4-g64-R64-G4-T20000": (1, 8, 2, 4, 4, 64, 64, 4, 20000, None),
    "k4v4-g64-R64-G4-T32768": (1, 8, 2, 4, 4, 64, 64, 4, 32768, None),
    "mha-k2v2-g32-R128-T20000": (2, 4, 4, 2, 2, 32, 128, 1, 20000, None),
    "mha-k2v2-g32-R128-T32768": (2, 4, 4, 2, 2, 32, 128, 1, 32768, None),
    "mha-k2v2-g32-R128-T20000-padded": (2, 4, 4, 2, 2, 32, 128, 1, 20000, [9000, 0]),
    "k4v4-g64-R64-G4-ratio8-T32768": (1, 8, 1, 4, 4, 64, 64, 4, 32768, None),
}


@pytest.mark.parametrize("name", list(LONG))
def test_long_windows_many_ranges_per_unit(name):
    """Few long units: a window of up to 32k tokens is cut into many warp ranges per unit (more than 32 statistic slots
    and partial records, counted from the window's first block).  W in {T - 1, 16384, 4097, 129}, each against the
    oracle stage by stage; then the step's cache update bit for bit."""
    B, H, Hkv, kb, vb, g, R, G, T, starts = LONG[name]
    n0 = T - 1
    rng = np.random.default_rng(T + H + Hkv + kb)
    k, v = rand16(rng, (B, Hkv, n0, D)), rand16(rng, (B, Hkv, n0, D))
    cache = make_cache(B, H, Hkv, kb, vb, g, R, T + 16, gqa_chunk=G)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(),
                  kv_start=None if starts is None else torch.tensor(starts))
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    del k, v
    q, kn, vn = rand16(rng, (B, H, 1, D), 0.5), rand16(rng, (B, Hkv, 1, D)), rand16(rng, (B, Hkv, 1, D))
    for W in (T - 1, 16384, 4097, 129):
        _, _, nxt, _ = checked_call(cache, st, q, kn, vn, (g, kb, vb, R), starts=starts, window=W)
    cache.advance()
    tuple_equal(cache.export(0), nxt, "after the step")


# ---------------------------------------------------------------------------------------------------
# 4. the benchmarked windowed shape: one Mistral-7B layer, K4V4 g64 R64, B = 16, T = 32768, W = 4096
# ---------------------------------------------------------------------------------------------------
def _dequant_lastdim(code, scale, mn, g, bits):
    """c * s + z in float64 along the last dim of the reference layout (codes packed 32 / bits per int32 word)."""
    fpi = 32 // bits
    sh = torch.arange(fpi, device=code.device, dtype=torch.int64) * bits
    c = ((code.to(torch.int64)[..., None] >> sh) & ((1 << bits) - 1)).reshape(*code.shape[:-1], code.shape[-1] * fpi)
    s = scale.double().repeat_interleave(g, dim=-1)
    z = mn.double().repeat_interleave(g, dim=-1)
    return c.double() * s + z


def test_mistral_layer_window_4096_at_32k():
    """Every unit against a float64 reference on the device that dequantises the window's slice of the exported cache and
    computes softmax(q K^T / sqrt(128)) V over it (end-to-end bar); a slab of units stage by stage against the oracle; the
    probabilities sum to 1 over the window and are 0 below it; the slab's cache update bit for bit."""
    B, H, Hkv, kb, vb, g, R, T, W = 16, 32, 8, 4, 4, 64, 64, 32768, 4096
    n0, ratio = T - 1, H // Hkv
    gen = torch.Generator(device="cuda").manual_seed(4096)
    cache = make_cache(B, H, Hkv, kb, vb, g, R, T + 64, sliding_window=W)
    k = torch.randn((B, Hkv, n0, D), generator=gen, device="cuda", dtype=torch.float16)
    v = torch.randn((B, Hkv, n0, D), generator=gen, device="cuda", dtype=torch.float16)
    cache.prefill(0, k, v)
    del k, v
    torch.cuda.empty_cache()
    tup = cache.export(0)
    q = (torch.randn((B, H, D), generator=gen, device="cuda", dtype=torch.float32) * 0.6).half()
    kn = torch.randn((B, Hkv, D), generator=gen, device="cuda", dtype=torch.float16)
    vn = torch.randn((B, Hkv, D), generator=gen, device="cuda", dtype=torch.float16)
    dbg_s = torch.zeros((B, H, T + 8), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out_fast = cache.decode_attention(0, q, kn, vn).clone()
    out = cache.decode_attention(0, q, kn, vn, dbg_logits=dbg_s, dbg_probs=dbg_p)
    torch.cuda.synchronize()
    assert torch.equal(out_fast.view(torch.int16), out.view(torch.int16)), "production and instrumented epilogues"
    s0 = T - W
    tk, tv = cache.tk, cache.tv
    assert 0 < s0 < tv < tk, (s0, tv, tk)
    # probabilities: 0 below the window, summing to 1 over it
    assert not bool(dbg_p[..., :s0].any()), "probabilities below the window"
    psum = dbg_p[..., s0:T].double().sum(-1)
    assert bool(((psum - 1).abs() < 2e-2).all()), float((psum - 1).abs().max())
    # float64 reference over the window's slice of the exported cache, every unit
    assert s0 % g == 0
    Kq = _dequant_lastdim(tup[0][..., s0 * kb // 32:], tup[2][..., s0 // g:], tup[3][..., s0 // g:], g, kb)   # [B, Hkv, D, tk - s0]
    Kw = torch.cat([Kq.transpose(2, 3), tup[1].double(), kn[:, :, None].double()], dim=2)   # [B, Hkv, W, D]
    del Kq
    Vq = _dequant_lastdim(tup[4][:, :, s0:], tup[6][:, :, s0:], tup[7][:, :, s0:], g, vb)   # [B, Hkv, tv - s0, D]
    Vw = torch.cat([Vq, tup[5].double(), vn[:, :, None].double()], dim=2)
    del Vq
    assert Kw.shape[2] == W and Vw.shape[2] == W
    qg = q.double().view(B, Hkv, ratio, D)
    prob = torch.softmax(qg @ Kw.transpose(2, 3) / np.sqrt(D), dim=-1)                 # [B, Hkv, ratio, W]
    exp = (prob @ Vw).reshape(B, H, D)
    del Kw, Vw, prob
    err = (out.double() - exp).abs()
    tol = E2E_RTOL * exp.abs() + E2E_ATOL_FRAC * exp.abs().amax(-1, keepdim=True)
    assert bool((err <= tol).all()), f"float64 reference: worst err / bar {float((err / tol.clamp_min(1e-30)).max()):.2f}"
    # a slab of units stage by stage against the oracle, then its cache update
    after = {}
    for b, hk in [(0, 0), (9, 3), (15, 7)]:
        st4, q4, kn4, vn4, out4, s4, p4 = _slab(tup, q, kn, vn, out, dbg_s, dbg_p, b, hk, ratio)
        _, _, after[b, hk], _ = check_stages(st4, q4, kn4, vn4, (g, kb, vb, R), out4, s4, p4, hidden_mask(1, T, window=W))
    cache.advance()
    tup2 = cache.export(0)
    for b, hk in [(0, 0), (15, 7)]:
        got = tuple(None if t is None else t[b:b + 1, hk:hk + 1] for t in tup2[:8]) + (tup2[8],)
        tuple_equal(got, after[b, hk], f"slab ({b}, {hk})")


# ---------------------------------------------------------------------------------------------------
# 5. the window combined with an additive mask
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("kb,vb,g,R,G,H,Hkv", [(2, 4, 32, 64, 2, 4, 2), (4, 2, 64, 128, 1, 2, 2)])
def test_window_with_mask(kb, vb, g, R, G, H, Hkv, padded):
    """An additive finfo.min mask that hides random positions inside and below the window and a run across its start,
    passed together with the window: against the oracle given the combined mask (hidden wherever either one hides)."""
    B = 4
    n0 = max(3, -(-600 // R)) * R + R - 3
    rng = np.random.default_rng(kb + 10 * vb + g + R + padded)
    tk0, r0, tv0, _ = mirror_lengths(n0, R)
    starts = [0, 200, tv0 + 1, 50] if padded else None
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 16, gqa_chunk=G)
    k, v = rand16(rng, (B, Hkv, n0, D)), rand16(rng, (B, Hkv, n0, D))
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(),
                  kv_start=None if starts is None else torch.tensor(starts))
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    for step in range(4):                                            # the third step flushes the K window
        T = cache.kv_len + 1
        q, kn, vn = _step_inputs(rng, B, H, Hkv)
        for W in (T - 150, 333, 130, 40):
            s = T - W
            user = np.where(rng.random((B, T)) < 0.15, NEG16, 0).astype(np.float16)
            user[:, max(s - 6, 0):s + 6] = NEG16                    # a run across the window's start
            user[:, T - 1] = 0                                       # the new token stays visible
            vis = (hidden_mask(B, T, starts, W)[:, 0, 0] == NEG16).sum(-1)      # the first visible position
            assert all((user[b, x:T - 1] == NEG16).any() for b, x in enumerate(vis)), "the mask hides visible positions"
            assert all((user[b, :x] == NEG16).any() for b, x in enumerate(vis) if x > 0), "the mask hides hidden ones"
            _, _, nxt, _ = checked_call(cache, st, q, kn, vn, (g, kb, vb, R), starts=starts, window=W, user=user)
        cache.advance()
        st = nxt
        tuple_equal(cache.export(0), st, f"step {step}")


# ---------------------------------------------------------------------------------------------------
# 6. a captured step replayed over a long walk
# ---------------------------------------------------------------------------------------------------
def test_captured_window_step_over_a_long_walk():
    """The window call and the cache advance captured once in a CUDA graph, replayed 300 times with W = 1000 on a
    left-padded batch whose KV head spans two work units (ratio = 2G): the window's first block crosses several K and V
    blocks and the K window flushes several times.  Every replay end to end against the oracle; the cache bit for bit at
    the end."""
    kb, vb, g, R, G, H, Hkv, B, W = 4, 2, 64, 64, 2, 4, 1, 3, 1000
    n0, steps = 1100 + R - 3, 300
    rng = np.random.default_rng(300)
    starts = [0, 300, n0 - 200]                                      # below T - W, crossed by it mid-walk, above it
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + steps + 8, gqa_chunk=G, sliding_window=W)
    k, v = rand16(rng, (B, Hkv, n0, D)), rand16(rng, (B, Hkv, n0, D))
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), kv_start=torch.tensor(starts))
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    qb, kb_, vb_ = (torch.zeros(s, dtype=torch.float16, device="cuda") for s in ((B, H, D), (B, Hkv, D), (B, Hkv, D)))
    out = torch.zeros_like(qb)
    state0 = cache.state.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                                    # warm-up outside the capture
        cache.decode_attention(0, qb, kb_, vb_, out=out)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cache.decode_attention(0, qb, kb_, vb_, out=out)
        cache._enqueue_advance()
    cache.state.copy_(state0)
    j0s, flushes = set(), 0
    for step in range(steps):
        T = cache.kv_len + 1
        tk0 = cache.tk
        q, kn, vn = _step_inputs(rng, B, H, Hkv)
        for dst, src in ((qb, q), (kb_, kn), (vb_, vn)):
            dst.copy_(torch.from_numpy(np.ascontiguousarray(src[:, :, 0])))
        graph.replay()
        cache._mirror_advance()
        torch.cuda.synchronize()
        exp_out, _, st = ref.decode_step(st, q, kn, vn, g, kb, vb, R, hidden_mask(B, T, starts, W))
        assert_e2e(to_np(out)[:, :, None, :], exp_out, f"replay {step}")
        j0s.add((T - W) // 128)
        flushes += cache.tk != tk0
    assert len(j0s) >= 3 and flushes >= 4, (j0s, flushes)
    assert cache.read_state()[:6] == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]
    tuple_equal(cache.export(0), st, "after the walk")

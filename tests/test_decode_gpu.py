"""Parity of the pre-allocated cache + fused decode-attention kernel (kivi_cache.cu, kivi_decode.cu)
with the restated attention hook of the reference (oracle/ref.py: models/llama_kivi.py:314-455).

Cache contents (codes, scale, mn, fp16 windows) are compared BIT-EXACTLY with the oracle's 9-tuple.
The attention output passes through the reference's fp16 rounding points (fp16 logits -> fp16 scale
-> fp32 softmax -> fp16 probs -> fp16 partial outputs), where a 1-ulp flip of an fp16 logit (ulp up
to 2^-7 at |s| ~ 8) legitimately moves a probability by ~1%; so every stage is checked against the
oracle applied to the kernel's OWN previous-stage values (rtol 1e-3 + fp32 accumulation floor), and
the end-to-end output against the full oracle chain with the looser, stated E2E tolerance."""
import itertools

import numpy as np
import pytest
import torch

from oracle import ref
from tests._util import assert_gemv_close, l1_mass_ref_layout, to_np

pytestmark = pytest.mark.gpu

E2E_RTOL, E2E_ATOL_FRAC = 2e-2, 5e-3       # end-to-end |err| <= 2e-2*|ref| + 5e-3*max|ref|


def _tuple_equal(got, exp):
    assert got[8] == exp[8]
    for i in range(8):
        a, b = got[i], exp[i]
        if b is None or b.size == 0:
            assert a is None or a.numel() == 0, f"tuple[{i}] should be empty"
            continue
        a = to_np(a)
        assert a.shape == b.shape, (i, a.shape, b.shape)
        if a.dtype == np.float16:
            np.testing.assert_array_equal(a.view(np.uint16), b.view(np.uint16), err_msg=f"tuple[{i}]")
        else:
            np.testing.assert_array_equal(a, b, err_msg=f"tuple[{i}]")


def _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=1024, n_layers=1, mode=None):
    from kivi_b200.cache import KiviCache
    return KiviCache(n_layers, B, H, Hkv, 128, kb, vb, g, R, max_tokens, gqa_chunk=1 if mode == "G-1" else 0)


@pytest.fixture(params=["G-auto", "G-1"])
def mode(request):
    """G-auto: the query heads of a KV head share the MMAs (chunks of up to 4, KIVI_CACHE_GQA_CHUNK = 0);
    G-1: one head per unit (KIVI_CACHE_GQA_CHUNK(1))."""
    return request.param


@pytest.mark.parametrize("n", [1, 5, 128, 200, 333, 640])
@pytest.mark.parametrize("kb,vb,g,R", [(2, 2, 32, 128), (4, 4, 64, 64), (2, 4, 32, 32), (4, 2, 128, 128)])
def test_prefill_matches_oracle(n, kb, vb, g, R):
    """kivi_cache_prefill_f16 == the prefill split + pack of models/llama_kivi.py:425-452, bit for bit."""
    rng = np.random.default_rng(n * 31 + kb + R)
    B, H, Hkv = 2, 4, 2
    k = rng.standard_normal((B, Hkv, n, 128)).astype(np.float16)
    v = rng.standard_normal((B, Hkv, n, 128)).astype(np.float16)
    cache = _mk_cache(B, H, Hkv, kb, vb, g, R)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    exp = list(ref.prefill_cache(k, v, g, kb, vb, R))
    # the oracle packs K and V with their own bit widths
    if exp[0] is not None:
        nq = exp[0].shape[-1] * (32 // kb)
        exp[0], exp[2], exp[3] = ref.pack_lastdim(np.ascontiguousarray(k[:, :, :nq].transpose(0, 1, 3, 2)), g, kb)
    if exp[4] is not None:
        exp[4], exp[6], exp[7] = ref.pack_lastdim(np.ascontiguousarray(v[:, :, :-R]), g, vb)
    _tuple_equal(cache.export(0), tuple(exp))
    assert to_np(cache.state)[:6].tolist() == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]


def _step16(x):
    """Bound of one fp16 rounding step of x: 2^-10 |x|, and the subnormal step 2^-24 below 2^-14."""
    return np.maximum(2.0 ** -10 * np.abs(np.asarray(x, np.float64)), 2.0 ** -24)


def _stage_checks(cache_tuple_before, q, k_new, v_new, g, kb, vb, R, got_out, got_s, got_p, mask=None):
    """cache_tuple_before: oracle 9-tuple BEFORE the step (numpy)."""
    Kq, Kfull, Ks, Kz, Vq, Vfull, Vs, Vz, kv_len = cache_tuple_before
    B, H, _, D = q.shape
    T = kv_len + 1
    # ---- stage 1: logits (fp16 kernel outputs), then the fp16 scale
    Kf = np.concatenate([Kfull, k_new], axis=2) if Kfull is not None else k_new
    parts, l1 = [], []
    if Kq is not None:
        parts.append(ref.bmm_fA_qB_outer(g, q, Kq, Ks, Kz, kb))
        l1.append(np.broadcast_to(l1_mass_ref_layout(q, Ks, Kz, 2 ** kb - 1), parts[-1].shape))
    parts.append(ref.residual_qk(q, Kf))
    rep = H // Kf.shape[1]
    l1r = np.einsum("bhd,bhtd->bht", np.abs(q[:, :, 0].astype(np.float64)),
                    np.abs(np.repeat(Kf, rep, axis=1).astype(np.float64)))[:, :, None, :]
    l1.append(l1r)
    logits = np.concatenate(parts, -1)
    l1 = np.concatenate(l1, -1)
    exp_s = (logits.astype(np.float32) * (np.float32(1.0) / np.float32(11.313708))).astype(np.float16)
    if mask is not None:
        exp_s = (exp_s.astype(np.float32) + mask.astype(np.float32)).astype(np.float16)
        exp_s = np.maximum(exp_s, np.float16(-65504))
    # The kernel output that the 1e-3 rtol bar applies to is the UNSCALED fp16 logit (the reference
    # kernel's output); the fp16 scale that follows re-rounds it.  Accept exactly the scaled images of
    # the oracle logit and of its two fp16 neighbours (a 1-ulp flip = 2^-10 relative <= 1e-3), or the
    # fp32 accumulation floor for logits that cancel to ~0.
    def _sc(x):
        y = (x.astype(np.float32) * (np.float32(1.0) / np.float32(11.313708))).astype(np.float16)
        if mask is not None:
            y = np.maximum((y.astype(np.float32) + mask.astype(np.float32)).astype(np.float16), np.float16(-65504))
        return y
    gs = got_s[..., :T]
    ok = np.zeros(gs.shape, bool)
    for cand in (logits, np.nextafter(logits, np.float16(-np.inf)), np.nextafter(logits, np.float16(np.inf))):
        ok |= (gs == _sc(cand))
    ok |= np.abs(gs.astype(np.float64) - exp_s.astype(np.float64)) <= 1e-6 * l1 / 11.3
    if mask is not None:      # masked positions are not part of the kernel's result (fp16(s + finfo.min) depends on s)
        ok |= np.broadcast_to(mask == np.finfo(np.float16).min, ok.shape)
    assert ok.all(), f"scaled logits: {(~ok).sum()} / {ok.size} differ by more than one fp16 ulp of the kernel output"
    # ---- stage 2: softmax of the kernel's own scaled logits
    exp_p = ref.scale_softmax(np.ascontiguousarray(got_s[..., :T]), 1)
    pe = np.abs(got_p[..., :T].astype(np.float64) - exp_p.astype(np.float64))
    assert (pe <= 1e-3 * exp_p.astype(np.float64) + 1e-7).all(), f"softmax stage: max err {pe.max():.3e}"
    # ---- stage 3: p.V with the kernel's own probabilities
    p_own = np.ascontiguousarray(got_p[..., :T])
    Vf = np.concatenate([Vfull, v_new], axis=2)
    L = Vf.shape[2]
    out_r = ref.residual_pv(np.ascontiguousarray(p_own[..., -L:]), Vf)
    l1o = np.einsum("bht,bhtd->bhd", np.abs(p_own[:, :, 0, -L:].astype(np.float64)),
                    np.abs(np.repeat(Vf, rep, axis=1).astype(np.float64)))[:, :, None, :]
    if Vq is not None:
        pq = np.ascontiguousarray(p_own[..., :-L])
        out_q = ref.bmm_fA_qB_outer(g, pq, Vq, Vs, Vz, vb)
        exp_out = ref.add_f16(out_q, out_r)
        l1o = l1o + l1_mass_ref_layout(pq, Vs, Vz, 2 ** vb - 1)
        # the two fp16 partial sums may each flip by one ulp before the fp16 add (one step is 2^-24 in the subnormals)
        l1o = l1o + (1 / 1e-6) * (_step16(out_q) + _step16(out_r))
    else:
        exp_out = out_r
    # rtol covers one rounding step of a normal fp16 output (2^-10 relative at most); a subnormal output's step is 2^-24
    l1o = l1o + np.where(np.abs(exp_out.astype(np.float64)) < 2.0 ** -14, 2.0 ** -24 / 1e-6, 0.0)
    assert_gemv_close(got_out, exp_out, l1o, "attention output (own probs)")


DECODE_CASES = [  # B, H, Hkv, kb, vb, g, R, n_prefill, steps
    (1, 2, 2, 2, 2, 32, 128, 300, 140),     # crosses a K flush (r: 44 -> 128) and V ring wrap-around
    (2, 4, 1, 2, 2, 32, 32, 70, 40),        # GQA 4 (G = 4), R = 32: several flushes
    (1, 8, 1, 4, 4, 64, 64, 130, 70),       # ratio 8 -> two chunks of 4, 4-bit g64
    (1, 2, 1, 2, 4, 32, 64, 10, 80),        # G = 2, mixed bits, starts below R (no packed part at first)
    (1, 3, 3, 4, 2, 128, 128, 0, 135),      # decode from an EMPTY cache, g = 128
    (1, 2, 1, 4, 2, 64, 256, 250, 20),      # R = 256: a K flush fills two 128-token blocks (step 6)
    (2, 2, 2, 2, 2, 128, 256, 250, 20),     # R = 256, g = 128, 2-bit: flush at step 6 into blocks 0 and 1
]


def _oracle_prefill(k, v, g, kb, vb, R):
    """ref.prefill_cache with K and V packed at their own bit widths (the oracle's prefill uses one width for both)."""
    st = list(ref.prefill_cache(k, v, g, kb, vb, R))
    if st[0] is not None:
        nq = st[0].shape[-1] * (32 // kb)
        st[0], st[2], st[3] = ref.pack_lastdim(np.ascontiguousarray(k[:, :, :nq].transpose(0, 1, 3, 2)), g, kb)
    if st[4] is not None:
        st[4], st[6], st[7] = ref.pack_lastdim(np.ascontiguousarray(v[:, :, :-R]), g, vb)
    return tuple(st)


@pytest.mark.parametrize("B,H,Hkv,kb,vb,g,R,n0,steps", DECODE_CASES)
def test_decode_steps_match_oracle(B, H, Hkv, kb, vb, g, R, n0, steps, mode):
    rng = np.random.default_rng(n0 * 13 + H + R)
    cache = _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=512, mode=mode)
    if n0 > 0:
        k = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
        v = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
        cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
        st = _oracle_prefill(k, v, g, kb, vb, R)
    else:
        st = (None, None, None, None, None, np.zeros((B, Hkv, 0, 128), np.float16), None, None, 0)
    tmax = 512
    dbg_s = torch.zeros((B, H, tmax), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    worst = 0.0
    for step in range(steps):
        q = (rng.standard_normal((B, H, 1, 128)) * 0.7).astype(np.float16)
        k_new = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
        v_new = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
        qd, kd, vd = (torch.from_numpy(a[:, :, 0]).cuda() for a in (q, k_new, v_new))
        # the production epilogue first (no debug pointers: the branch bench.py runs), then the instrumented one on the
        # same state -- every instantiation the cases reach (<2,4,32>, G = 2, g = 128, ...) must give the same bits
        out_fast = cache.decode_attention(0, qd, kd, vd).clone()
        out = cache.decode_attention(0, qd, kd, vd, dbg_logits=dbg_s, dbg_probs=dbg_p)
        assert torch.equal(out_fast, out), f"step {step}: fast and instrumented epilogues disagree"
        cache.advance()
        torch.cuda.synchronize()
        got_out = to_np(out)[:, :, None, :]
        got_s, got_p = to_np(dbg_s)[:, :, None, :], to_np(dbg_p)[:, :, None, :]
        check = step < 3 or step % 9 == 0 or step >= steps - 3 or st[1] is None or (st[1].shape[2] >= R - 2)
        if check:
            _stage_checks(st, q, k_new, v_new, g, kb, vb, R, got_out, got_s, got_p)
        # oracle step (K and V may use different bit widths: restate with the per-tensor widths)
        exp_out, exp_p, st = _oracle_step(st, q, k_new, v_new, g, kb, vb, R)
        err = np.abs(got_out.astype(np.float64) - exp_out.astype(np.float64))
        tol = E2E_RTOL * np.abs(exp_out.astype(np.float64)) + E2E_ATOL_FRAC * np.abs(exp_out.astype(np.float64)).max()
        assert (err <= tol).all(), f"step {step}: end-to-end err {err.max():.3e}"
        worst = max(worst, float(err.max()))
        if check:
            _tuple_equal(cache.export(0), st)
    assert cache.read_state()[:6] == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]


def _oracle_step(st, q, k_new, v_new, g, kb, vb, R, mask=None):
    return ref.decode_step(st, q, k_new, v_new, g, kb, vb, R, mask)


NEG16 = np.finfo(np.float16).min


def _start_mask(starts, B, T):
    """The additive finfo(fp16).min mask [B, 1, 1, T] that per-sequence starts stand for (the new token stays visible)."""
    m = np.zeros((B, 1, 1, T), np.float16)
    for b, s in enumerate(starts):
        m[b, ..., :min(max(s, 0), T - 1)] = NEG16
    return m


def _checked_step(cache, st, q, k_new, v_new, g, kb, vb, R, starts=None):
    """One decode step of `cache` (oracle 9-tuple `st` before it) with every check of the oracle suite:
      * the production epilogue (no debug pointers) and the instrumented one give the same bits;
      * every stage against the oracle applied to the kernel's own previous stage (_stage_checks);
      * the output end to end against ref.decode_step;
      * the exported cache equals the oracle's 9-tuple bit for bit.
    starts: per-sequence first visible positions (the cache must be in ragged mode); the oracle then runs with the
    equivalent additive mask, and the kernel's logits of excluded positions, which are not part of its result (wholly padded
    blocks are not even computed), are replaced by the masked value before the stage checks.  Returns the new tuple."""
    B, H = q.shape[:2]
    T = st[8] + 1
    qd, kd, vd = (torch.from_numpy(np.ascontiguousarray(a[:, :, 0])).cuda() for a in (q, k_new, v_new))
    dbg_s = torch.zeros((B, H, T + 8), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out_fast = cache.decode_attention(0, qd, kd, vd).clone()
    out = cache.decode_attention(0, qd, kd, vd, dbg_logits=dbg_s, dbg_probs=dbg_p)
    cache.advance()
    torch.cuda.synchronize()
    assert torch.equal(out_fast.view(torch.int16), out.view(torch.int16)), "production and instrumented epilogues disagree"
    got_out = to_np(out)[:, :, None, :]
    got_s, got_p = to_np(dbg_s)[:, :, None, :T].copy(), to_np(dbg_p)[:, :, None, :T]
    mask = None
    if starts is not None:
        mask = _start_mask(starts, B, T)
        got_s[np.broadcast_to(mask == NEG16, got_s.shape)] = NEG16
    _stage_checks(st, q, k_new, v_new, g, kb, vb, R, got_out, got_s, got_p,
                  mask=None if mask is None else np.broadcast_to(mask, (B, H, 1, T)))
    exp_out, _, st = _oracle_step(st, q, k_new, v_new, g, kb, vb, R, mask)
    e, x = got_out.astype(np.float64), exp_out.astype(np.float64)
    err = np.abs(e - x)
    tol = E2E_RTOL * np.abs(x) + E2E_ATOL_FRAC * np.abs(x).max()
    assert (err <= tol).all(), f"end-to-end: worst err / bar {(err / np.maximum(tol, 1e-30)).max():.2f}"
    _tuple_equal(cache.export(0), st)
    return st


# ---------------------------------------------------------------------------------------------------
# every attention instantiation against the oracle: k_bits x v_bits x g x G x {unpadded, ragged}
# ---------------------------------------------------------------------------------------------------
def _header_set(name):
    """A supported-value set as include/kivi_b200.h documents it, e.g. `group_size in {32,64,128}`."""
    import os
    import re
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kivi_b200.h")) as f:
        m = re.search(name + r" in \{([0-9, ]+)\}", f.read())
    assert m, name
    return tuple(int(x) for x in m.group(1).split(","))


BITS = (2, 4)
GROUPS = _header_set("group_size")
RESIDUALS = _header_set("residual_length")
GQA_CHUNKS = (1, 2, 4)                                    # KIVI_CACHE_GQA_CHUNK: 1 / 2 / 4 query heads per work unit
RAGGED_STARTS = [0, 300, 129, 512]                        # whole blocks skipped, blocks partly padded (as test_padded_blocks_are_not_read)


def _instantiation_cases():
    cases = []
    for (ik, kb), (iv, vb), g, (iG, G), ragged in itertools.product(enumerate(BITS), enumerate(BITS), GROUPS,
                                                                      enumerate(GQA_CHUNKS), (False, True)):
        Rs = [R for R in RESIDUALS if R % g == 0]
        # as (k_bits, v_bits) run through their four values for a fixed (g, G), R runs through every residual length
        R = Rs[(2 * ik + iv + iG + ragged) % len(Rs)]
        ratio = 2 * G if (2 * ik + iv + iG + GROUPS.index(g)) % 5 == 0 else G   # a few: one KV head spans two units
        cases.append(pytest.param(kb, vb, g, G, R, ratio, ragged,
                                  id=f"k{kb}v{vb}-g{g}-G{G}-R{R}-ratio{ratio}-{'ragged' if ragged else 'unpadded'}"))
    return cases


@pytest.mark.parametrize("kb,vb,g,G,R,ratio,ragged", _instantiation_cases())
def test_every_instantiation_matches_oracle(kb, vb, g, G, R, ratio, ragged):
    """Every (k_bits, v_bits, g, G, RAGGED) kernel pair the dispatcher can pick, against the C oracle: prefill to
    r = R - 3, then six steps that cross a K flush and move the V ring head, every step fully checked (_checked_step).
    Ragged cases: one sequence unpadded, the others with whole 128-token blocks skipped, partly padded blocks, and
    starts inside the fp16 K and V windows; the oracle runs with the equivalent additive mask."""
    from kivi_b200.cache import KiviCache
    Hkv = 2 if ratio == G else 1
    H = ratio * Hkv
    n0 = max(3, -(-540 // R)) * R + R - 3
    rng = np.random.default_rng(1000 * kb + 100 * vb + g + 7 * G + R + ratio + 3 * ragged)
    B = 6 if ragged else 2
    cache = KiviCache(1, B, H, Hkv, 128, kb, vb, g, R, n0 + 16, gqa_chunk=G)
    k = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    v = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    starts = None
    if ragged:
        tk, r, tv, L = _mirror_lengths(n0, R)
        starts = RAGGED_STARTS + [tk + r // 2, tv + L // 2]
        assert len(starts) == B and max(starts) < n0
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(),
                  kv_start=None if starts is None else torch.tensor(starts))
    assert cache.ragged == ragged
    st = _oracle_prefill(k, v, g, kb, vb, R)
    r0 = cache.r
    for step in range(6):
        q = (rng.standard_normal((B, H, 1, 128)) * 0.7).astype(np.float16)
        k_new = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
        v_new = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
        st = _checked_step(cache, st, q, k_new, v_new, g, kb, vb, R, starts)
    assert r0 == R - 3 and cache.r == 3 and cache.vhead != 0, "the steps crossed a K flush and moved the V ring head"
    assert cache.read_state()[:6] == [cache.tk, cache.r, cache.tv, cache.L, cache.vhead, cache.kv_len]


def _mirror_lengths(n, R):
    """(tk, r, tv, L) after a prefill of n tokens (models/llama_kivi.py:425-452)."""
    nqk = (0 if n < R else n - n % R) if n % R != 0 else n
    nqv = 0 if n <= R else n - R
    return nqk, n - nqk, nqv, n - nqv


def test_decode_with_mask(mode):
    """Additive mask + max with finfo.min (models/llama_kivi.py:364-372), e.g. left padding."""
    rng = np.random.default_rng(4)
    B, H, Hkv, kb, vb, g, R, n0 = 2, 2, 2, 2, 2, 32, 128, 200
    cache = _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=512, mode=mode)
    k = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    v = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    T = n0 + 1
    mask = np.zeros((B, 1, 1, T), np.float16)
    mask[0, :, :, :17] = np.finfo(np.float16).min                   # sequence 0 is left-padded by 17 tokens
    mask[1, :, :, :3] = np.finfo(np.float16).min
    q = rng.standard_normal((B, H, 1, 128)).astype(np.float16)
    k_new = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
    v_new = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
    dbg_s = torch.zeros((B, H, 512), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out = cache.decode_attention(0, torch.from_numpy(q[:, :, 0]).cuda(), torch.from_numpy(k_new[:, :, 0]).cuda(),
                                 torch.from_numpy(v_new[:, :, 0]).cuda(), mask=torch.from_numpy(mask).cuda(),
                                 dbg_logits=dbg_s, dbg_probs=dbg_p)
    torch.cuda.synchronize()
    got_p = to_np(dbg_p)[:, :, None, :T]
    assert (got_p[0, :, :, :17] == 0).all() and (got_p[1, :, :, :3] == 0).all()
    _stage_checks(st, q, k_new, v_new, g, kb, vb, R, to_np(out)[:, :, None, :], to_np(dbg_s)[:, :, None, :],
                  to_np(dbg_p)[:, :, None, :], mask=np.broadcast_to(mask, (B, H, 1, T)))


def test_multi_layer_shared_state():
    """All layers share one device state; decode of layer l must not disturb layer m."""
    rng = np.random.default_rng(8)
    B, H, Hkv, g, R, n0, NL = 1, 2, 2, 32, 128, 150, 3
    cache = _mk_cache(B, H, Hkv, 2, 2, g, R, max_tokens=512, n_layers=NL)
    sts = []
    for l in range(NL):
        k = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
        v = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
        cache.prefill(l, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
        sts.append(ref.prefill_cache(k, v, g, 2, 2, R))
    for step in range(4):
        for l in range(NL):
            q = rng.standard_normal((B, H, 1, 128)).astype(np.float16)
            kn = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
            vn = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
            cache.decode_attention(l, torch.from_numpy(q[:, :, 0]).cuda(), torch.from_numpy(kn[:, :, 0]).cuda(),
                                   torch.from_numpy(vn[:, :, 0]).cuda())
            _, _, sts[l] = ref.decode_step(sts[l], q, kn, vn, g, 2, 2, R)
        cache.advance()
    for l in range(NL):
        _tuple_equal(cache.export(l), sts[l])


def test_full_size_consistency(mode):
    """BASELINE cfg 2 layer shape (B32, H32, T = 4096, K2V2 g32 R128): too big for the CPU oracle end to
    end, so (1) a slab of units is checked stage-by-stage against the oracle, (2) the fused kernel must
    agree with the library's own generic-layout kernels run on the exported cache for ALL units
    (two independent code paths), (3) probabilities sum to 1."""
    from kivi_b200 import matmul
    gen = torch.Generator(device="cuda").manual_seed(3)
    B, H, Hkv, g, R, n0 = 32, 32, 32, 32, 128, 4095
    cache = _mk_cache(B, H, Hkv, 2, 2, g, R, max_tokens=4352, mode=mode)
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
    _stage_checks(st, to_np(q[sl, :2])[:, :, None, :], to_np(kn[sl, :2])[:, :, None, :], to_np(vn[sl, :2])[:, :, None, :],
                  g, 2, 2, R, to_np(out[sl, :2])[:, :, None, :], to_np(dbg_s[sl, :2])[:, :, None, :],
                  to_np(dbg_p[sl, :2])[:, :, None, :])


@pytest.mark.parametrize("B,H,Hkv,kb,vb,g,R,n0", [(1, 8, 2, 4, 4, 64, 64, 20000),      # cfg-4-like: few, long units, GQA 4, 4-bit
                                                  (2, 4, 4, 2, 2, 32, 128, 9000)])     # MHA, more ranges per unit than warps of a CTA
def test_long_context_many_ranges_per_unit(B, H, Hkv, kb, vb, g, R, n0):
    """Few long units: every unit is cut into many warp ranges (more than 32 statistic slots and partial records per
    unit), far beyond what a logits row in shared memory could hold.  Checked against the library's generic-layout
    kernels run on the exported cache (an independent code path) and against the softmax identities."""
    from kivi_b200 import matmul
    gen = torch.Generator(device="cuda").manual_seed(11)
    cache = _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=n0 + 64)
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
def _slab(tup, q, kn, vn, out, dbg_s, dbg_p, b, hk, ratio):
    """Cut (batch b, KV head hk) and its `ratio` query heads out of the full-size tensors, as numpy."""
    sb, sk, sq = slice(b, b + 1), slice(hk, hk + 1), slice(hk * ratio, (hk + 1) * ratio)
    st = tuple(None if t is None else to_np(t[sb, sk]) for t in tup[:8]) + (tup[8],)
    four = lambda t, hs: to_np(t[sb, hs])[:, :, None, :]           # noqa: E731
    return st, four(q, sq), four(kn, sk), four(vn, sk), four(out, sq), four(dbg_s, sq), four(dbg_p, sq)


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
      * three slabs (first, middle, last unit -- different warps, different range cuts) stage by stage against the
        C oracle of the reference kernels (1e-3 rtol + fp32 accumulation floor) and bit-exactly on the updated cache;
      * the production epilogue (no debug pointers) equals the instrumented one on ALL units, bit for bit;
      * every probability row sums to 1 and the device-side guard word stays clear."""
    B, H, Hkv, kb, vb, g, R, T, slabs = FULL_CONFIGS[name]
    n0 = T - 1
    ratio = H // Hkv
    gen = torch.Generator(device="cuda").manual_seed(len(name))
    cache = _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=T + 64)
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
    for b, hk in slabs:
        st, q4, kn4, vn4, out4, s4, p4 = _slab(tup, q, kn, vn, out, dbg_s, dbg_p, b, hk, ratio)
        _stage_checks(st, q4, kn4, vn4, g, kb, vb, R, out4, s4, p4)
    cache.advance()
    assert cache.read_state()[6] == 0
    tup2 = cache.export(0)
    for b, hk in slabs[:2]:                                        # the cache update of the step, bit for bit
        st, q4, kn4, vn4, *_ = _slab(tup, q, kn, vn, out, dbg_s, dbg_p, b, hk, ratio)
        _, _, exp = ref.decode_step(st, q4, kn4, vn4, g, kb, vb, R)
        got = tuple(None if t is None else t[b:b + 1, hk:hk + 1] for t in tup2[:8]) + (tup2[8],)
        _tuple_equal(got, exp)


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
    k = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    v = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    q = (rng.standard_normal((B, H, 1, 128)) * 0.8).astype(np.float16)
    kn = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
    vn = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
    cache = _mk_cache(B, H, Hkv, 2, 2, g, R, max_tokens=256)
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
    e2e = (out[:, :, None, :].float() - o_aten.float()).abs()
    assert bool((e2e <= E2E_RTOL * o_aten.float().abs() + E2E_ATOL_FRAC * float(o_aten.float().abs().max())).all())
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
    a = _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=512)
    if n0:
        a.prefill(0, torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16),
                  torch.randn((B, Hkv, n0, 128), generator=gen, device="cuda", dtype=torch.float16))
    mk = lambda *s: torch.randn(s, generator=gen, device="cuda", dtype=torch.float16)   # noqa: E731
    for _ in range(steps):                                           # ring wrap / flushes before the export
        a.decode_attention(0, mk(B, H, 128), mk(B, Hkv, 128), mk(B, Hkv, 128))
        a.advance()
    tup = a.export(0)
    b = _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=512)
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
    cache = _mk_cache(B, H, Hkv, kb, vb, g, R, max_tokens=512)
    cache.import_tuple(0, past)
    for _ in range(130):
        q, kn, vn = mk(B, H, 1, 128) * 0.7, mk(B, Hkv, 1, 128), mk(B, Hkv, 1, 128)
        exp, past = kivi_decode_attention_tuple(q, kn, vn, past, g, kb, vb, R)
        out = cache.decode_attention(0, q[:, :, 0].contiguous(), kn[:, :, 0].contiguous(), vn[:, :, 0].contiguous())
        cache.advance()
        err = (out.float() - exp[:, :, 0].float()).abs()
        assert bool((err <= E2E_RTOL * exp[:, :, 0].float().abs() + E2E_ATOL_FRAC * float(exp.float().abs().max())).all())
    tup = cache.export(0)
    for i in (0, 2, 3, 4, 6, 7, 1, 5):
        assert (tup[i] is None and past[i] is None) or torch.equal(tup[i], past[i].view_as(tup[i])), f"tuple[{i}]"
    assert tup[8] == past[8]


def test_device_side_capacity_guard():
    """A C-ABI caller whose device-side lengths run past the sizes it declared gets NO memory traffic and an error
    word (KIVI_STATE_ERR_CAPACITY in state[6]) instead of silent out-of-bounds writes."""
    B, H, Hkv = 1, 2, 2
    cache = _mk_cache(B, H, Hkv, 2, 2, 32, 128, max_tokens=256)
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

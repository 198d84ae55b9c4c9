"""The oracle check of the fused decode attention, shared by every test of the fused cache.

The attention output passes through the reference's fp16 rounding points (fp16 logits -> fp16 scale -> fp32 softmax ->
fp16 probs -> fp16 partial outputs), where a 1-ulp flip of an fp16 logit (ulp up to 2^-7 at |s| ~ 8) legitimately moves a
probability by ~1%.  So every stage is checked against the oracle applied to the kernel's OWN previous-stage values
(rtol 1e-3 + fp32 accumulation floor), and the end-to-end output against the full oracle chain with the looser, stated
E2E bar.  A call's state is the oracle's 9-tuple before it; `cfg` is (group_size, k_bits, v_bits, residual_length).

This module imports without CUDA (collection runs on machines without one): kivi_b200 is imported inside the functions."""
import itertools
import os
import re

import numpy as np
import pytest
import torch

from oracle import ref
from tests._gemv import OUTLIER_CHANNELS, edge_rows, rtol_bar  # noqa: F401  (the tests use OUTLIER_CHANNELS)
from tests._util import to_np

E2E_RTOL, E2E_ATOL_FRAC = 2e-2, 5e-3       # end-to-end |err| <= 2e-2*|ref| + 5e-3*max|ref|
NEG16 = np.finfo(np.float16).min


def _header_set(name):
    """A supported-value set as include/kivi_b200.h documents it, e.g. `group_size in {32,64,128}`."""
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kivi_b200.h")) as f:
        m = re.search(name + r" in \{([0-9, ]+)\}", f.read())
    assert m, name
    return tuple(int(x) for x in m.group(1).split(","))


BITS = (2, 4)
GROUPS = _header_set("group_size")
RESIDUALS = _header_set("residual_length")
GQA_CHUNKS = (1, 2, 4)                                    # KIVI_CACHE_GQA_CHUNK: 1 / 2 / 4 query heads per work unit
RAGGED_STARTS = [0, 300, 129, 512]                        # whole blocks skipped, blocks partly padded (as test_padded_blocks_are_not_read)


# ---------------------------------------------------------------------------------------------------
# small shared helpers
# ---------------------------------------------------------------------------------------------------
def make_cache(B, H, Hkv, kb, vb, g, R, max_tokens=1024, n_layers=1, gqa_chunk=0, sliding_window=None):
    from kivi_b200.cache import KiviCache
    return KiviCache(n_layers, B, H, Hkv, 128, kb, vb, g, R, max_tokens, gqa_chunk=gqa_chunk, sliding_window=sliding_window)


def rand16(rng, shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float16)


def mirror_lengths(n, R):
    """(tk, r, tv, L) after a prefill of n tokens (models/llama_kivi.py:425-452)."""
    nqk = (0 if n < R else n - n % R) if n % R != 0 else n
    nqv = 0 if n <= R else n - R
    return nqk, n - nqk, nqv, n - nqv


def instantiation_cases(label):
    """Every (k_bits, v_bits, g, G) kernel, unpadded and with per-sequence starts (named `label` in the ids: "ragged" or
    "padded"), as params (kb, vb, g, G, R, ratio, with_starts).  As (k_bits, v_bits) run through their four values for a
    fixed (g, G), R runs through every residual length; in a few cases one KV head spans two work units (ratio = 2G)."""
    cases = []
    for (ik, kb), (iv, vb), g, (iG, G), padded in itertools.product(enumerate(BITS), enumerate(BITS), GROUPS,
                                                                      enumerate(GQA_CHUNKS), (False, True)):
        Rs = [R for R in RESIDUALS if R % g == 0]
        R = Rs[(2 * ik + iv + iG + padded) % len(Rs)]
        ratio = 2 * G if (2 * ik + iv + iG + GROUPS.index(g)) % 5 == 0 else G
        cases.append(pytest.param(kb, vb, g, G, R, ratio, padded,
                                  id=f"k{kb}v{vb}-g{g}-G{G}-R{R}-ratio{ratio}-{label if padded else 'unpadded'}"))
    return cases


def tiny_model(seed=0, **kw):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config("tiny", **kw)
    torch.manual_seed(seed)
    return LlamaForCausalLM_KIVI(cfg).half().cuda().eval(), cfg


def left_padded(cfg, lengths, n, seed=0, low=1):
    """Ids [B, n] drawn from [low, vocab) and the attention mask of sequences of `lengths` tokens, left-padded with id 0."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(low, cfg.vocab_size, (len(lengths), n), device="cuda", generator=g)
    mask = torch.zeros((len(lengths), n), dtype=torch.long, device="cuda")
    for b, ln in enumerate(lengths):
        mask[b, n - ln:] = 1
        ids[b, :n - ln] = 0
    return ids, mask


def _slab(tup, q, kn, vn, out, dbg_s, dbg_p, b, hk, ratio):
    """Cut (batch b, KV head hk) and its `ratio` query heads out of the full-size tensors, as numpy."""
    sb, sk, sq = slice(b, b + 1), slice(hk, hk + 1), slice(hk * ratio, (hk + 1) * ratio)
    st = tuple(None if t is None else to_np(t[sb, sk]) for t in tup[:8]) + (tup[8],)
    four = lambda t, hs: to_np(t[sb, hs])[:, :, None, :]           # noqa: E731
    return st, four(q, sq), four(kn, sk), four(vn, sk), four(out, sq), four(dbg_s, sq), four(dbg_p, sq)


# ---------------------------------------------------------------------------------------------------
# edge values (the rows of test_pack_edge_values, tests/_gemv.py) as K and V
# ---------------------------------------------------------------------------------------------------
def _put_k_edges(k, pos0, kb):
    """K channel 3 + 17e of token t (absolute position pos0 + t) = row e at t mod 64: whole quantisation groups along
    tokens.  Sequence 0 gets the finite rows, sequence 1 all of them."""
    for b in range(k.shape[0]):
        rows = edge_rows(kb, finite=(b == 0))
        for e, row in enumerate(rows):
            k[b, :, :, 3 + 17 * e] = row[(pos0 + np.arange(k.shape[2])) % 64]


def _put_v_edges(v, pos0, vb):
    """Token t with (pos0 + t) % 5 == 2 of every sequence is an edge row over its 128 channels (two rows of 64)."""
    for b in range(v.shape[0]):
        rows = edge_rows(vb, finite=(b == 0))
        for t in range(v.shape[2]):
            p = pos0 + t
            if p % 5 == 2:
                e = (p // 5) % len(rows)
                v[b, :, t, :] = np.concatenate([rows[e], rows[(e + 1) % len(rows)]])


# ---------------------------------------------------------------------------------------------------
# the check
# ---------------------------------------------------------------------------------------------------
def hidden_mask(B, T, starts=None, window=None, user=None):
    """The additive finfo(fp16).min mask [B, 1, 1, T] of what a call hides: the positions below
    max(clamp(kv_start, 0, T - 1), T - W) (visible_start() of kivi_attn.cuh), so never the new token, and wherever the
    user mask [B, T] is finfo.min.  None when the call hides nothing."""
    if starts is None and window is None and user is None:
        return None
    m = np.zeros((B, 1, 1, T), np.float16)
    for b in range(B):
        s = min(max(0 if starts is None else int(starts[b]), 0), T - 1)
        m[b, ..., :s if window is None else max(s, T - window)] = NEG16
    if user is not None:
        m[np.asarray(user).reshape(B, 1, 1, T) == NEG16] = NEG16
    return m


def tuple_equal(got, exp, what):
    """Two 9-tuples bit for bit; either may hold torch or numpy arrays, and None counts as an empty entry."""
    assert int(got[8]) == int(exp[8]), f"{what}: kv_len {got[8]} != {exp[8]}"
    for i in range(8):
        a, b = (None if t is None else to_np(t) if torch.is_tensor(t) else np.asarray(t) for t in (got[i], exp[i]))
        if a is None or a.size == 0 or b is None or b.size == 0:
            assert (a is None or a.size == 0) and (b is None or b.size == 0), f"{what}: tuple[{i}] only one side empty"
            continue
        assert a.shape == b.shape and a.dtype == b.dtype, (what, i, a.shape, b.shape, a.dtype, b.dtype)
        if a.dtype == np.float16:
            a, b = a.view(np.uint16), b.view(np.uint16)
        np.testing.assert_array_equal(a, b, err_msg=f"{what}: tuple[{i}]")


def assert_e2e(got, exp, what):
    """The end-to-end bar, where the oracle output is finite; elsewhere the kernel's must be non-finite too."""
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    fin = np.isfinite(exp)
    np.testing.assert_array_equal(np.isfinite(got), fin, err_msg=f"{what}: non-finite positions differ from the oracle's")
    e, x = got[fin], exp[fin]
    err = np.abs(e - x)
    tol = E2E_RTOL * np.abs(x) + E2E_ATOL_FRAC * np.abs(x).max(initial=0.0)
    assert (err <= tol).all(), f"{what}: end-to-end worst err / bar {(err / np.maximum(tol, 1e-30)).max():.2f}"


def l1_mass_ref_layout(fA, scales, zeros, maxq):
    """Upper bound of sum_k |x_k| * max_n |s*c+z| per (b, head): fA [B,H,1,K], scales/zeros [B,Hkv,K,G]."""
    x = np.abs(np.asarray(fA, np.float64))[:, :, 0, :]                                  # [B,H,K]
    w = (np.abs(np.asarray(scales, np.float64)) * maxq + np.abs(np.asarray(zeros, np.float64))).max(-1)  # [B,Hkv,K]
    rep = x.shape[1] // w.shape[1]
    w = np.repeat(w, rep, axis=1)
    return (x * w).sum(-1)[:, :, None, None]                                            # [B,H,1,1]


def _step16(x):
    """Bound of one fp16 rounding step of x: 2^-10 |x|, and the subnormal step 2^-24 below 2^-14."""
    return np.maximum(2.0 ** -10 * np.abs(np.asarray(x, np.float64)), 2.0 ** -24)


def _stage_checks(st, q, k_new, v_new, cfg, got_out, got_s, got_p, mask=None):
    """Every stage of one call against the oracle applied to the kernel's own previous stage."""
    g, kb, vb, R = cfg
    Kq, Kfull, Ks, Kz, Vq, Vfull, Vs, Vz, kv_len = st
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
        ok |= np.broadcast_to(mask == NEG16, ok.shape)
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
    rtol_bar(got_out, exp_out, l1o, "attention output (own probs)")


def check_stages(st, q, kn, vn, cfg, got_out, got_s, got_p, mask, bad=()):
    """Every check of one call, given the oracle 9-tuple `st` before it, the inputs q [B,H,1,D] / kn, vn [B,Hkv,1,D], the
    kernel's output [B,H,1,D], scaled logits and probabilities [B,H,1,>=T] and the mask of what the call hides (None:
    nothing):
      * the probabilities are exactly 0 wherever the mask hides a position;
      * every stage against the oracle applied to the kernel's own previous stage, the hidden logits (not part of the
        kernel's result: wholly hidden blocks are not even computed) replaced by the masked value, on the sequences not
        in `bad` (those whose oracle output may be non-finite);
      * the output end to end against ref.decode_step (assert_e2e).
    Returns the oracle's (output, probabilities, 9-tuple after the step) and the kernel's scaled logits as checked."""
    B, H = q.shape[:2]
    T = st[8] + 1
    got_s, got_p = got_s[..., :T].copy(), got_p[..., :T]
    full = None
    if mask is not None:
        full = np.broadcast_to(mask, (B, H, 1, T))
        hidden = full == NEG16
        assert not got_p[hidden].any(), "probabilities at hidden positions"
        got_s[hidden] = NEG16
    good = [b for b in range(B) if b not in bad] if bad else slice(None)
    _stage_checks(tuple(None if t is None else t[good] for t in st[:8]) + (st[8],), q[good], kn[good], vn[good], cfg,
                  got_out[good], got_s[good], got_p[good], None if full is None else full[good])
    exp_out, exp_p, st_next = ref.decode_step(st, q, kn, vn, *cfg, mask)
    assert_e2e(got_out, exp_out, "attention output")
    return exp_out, exp_p, st_next, got_s


def checked_call(cache, st, q, kn, vn, cfg, starts=None, window=None, user=None, bad=()):
    """One decode-attention call on layer 0 of `cache` (no advance): the production epilogue (no debug pointers), then the
    instrumented one on the same state, which must give the same bits; then check_stages.  starts: the cache's
    per-sequence kv_start (ragged mode); window: the sliding window the call runs with; user: an additive fp16 mask [B, T]
    (0 or finfo.min) passed with the call.  Returns what check_stages returns."""
    B, H = q.shape[:2]
    T = st[8] + 1
    if window is not None:
        cache.sliding_window = window
    qd, kd, vd = (torch.from_numpy(np.ascontiguousarray(a[:, :, 0])).cuda() for a in (q, kn, vn))
    md = None if user is None else torch.from_numpy(user).cuda()
    dbg_s = torch.zeros((B, H, T + 8), dtype=torch.float16, device="cuda")
    dbg_p = torch.zeros_like(dbg_s)
    out_fast = cache.decode_attention(0, qd, kd, vd, mask=md).clone()
    out = cache.decode_attention(0, qd, kd, vd, mask=md, dbg_logits=dbg_s, dbg_probs=dbg_p)
    torch.cuda.synchronize()
    assert torch.equal(out_fast.view(torch.int16), out.view(torch.int16)), "production and instrumented epilogues disagree"
    return check_stages(st, q, kn, vn, cfg, to_np(out)[:, :, None, :], to_np(dbg_s)[:, :, None, :],
                        to_np(dbg_p)[:, :, None, :], hidden_mask(B, T, starts, window, user), bad)


def checked_step(cache, st, q, kn, vn, cfg, **call):
    """checked_call (keywords passed through), then cache.advance(); the exported cache must equal the oracle's 9-tuple
    after the step bit for bit.  Returns that tuple."""
    _, _, st, _ = checked_call(cache, st, q, kn, vn, cfg, **call)
    cache.advance()
    tuple_equal(cache.export(0), st, "exported cache")
    return st

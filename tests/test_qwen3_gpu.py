"""The decode step's RoPE + split kernel with Qwen3's per-head q / k RMSNorm folded in (kivi_qk_norm_rope_split_f16),
against exact references, at the Qwen3 head counts and across value magnitudes, and its wiring into the decode step.

The bar for q and k.  For one head x (fp16, 128 channels) and its weight w, r64 = x / sqrt(mean(x^2) + float32(eps)) in
fp64, and a <= r64 <= b are the adjacent fp16 values; the normalised value the kernel may hold is fp16(w*a) or fp16(w*b)
(fp32 statistics may round the inner value either way, the weight product must be rounded correctly).  Each output
element reads two channels (i and i +- 64) and must equal the fp16 RoPE (x*cos + rotate_half(x)*sin, every op rounded to
fp16) of one of the candidates of each.  Non-finite positions equal those of the torch chain (LlamaRMSNorm's rounding,
then apply_rotary_pos_emb); v is a bit-exact copy; the plain entry still equals rope_ref bit for bit."""
import numpy as np
import pytest
import torch

from tests._util import to_np
from tests.test_glue_numerics_gpu import (EPS, TABLE_ROWS, _positions, _tables, assert_bits, check_rounded_product,
                                          f16_neighbours, rmsnorm_inner64, rope_ref)

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------
def _rope16(n, partner, c, s):
    """fp16 RoPE of n (fp16 [..., 128]) whose rotate_half reads `partner` in place of n."""
    rot = np.concatenate([-partner[..., 64:], partner[..., :64]], -1)
    with np.errstate(over="ignore", invalid="ignore"):
        return n * c + rot * s


def check_norm_rope(got, x16, w16, c, s, what):
    """The bar of the module docstring.  got, x16 [B, heads, 128]; w16 [heads, 128]; c, s [B, 1, 128] (fp16 rows)."""
    got = np.asarray(got, np.float16)
    a, b = f16_neighbours(rmsnorm_inner64(x16))
    w = w16.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        cands = [(w * t.astype(np.float64)).astype(np.float16) for t in (a, b)]
    outs = [_rope16(n, p, c, s) for n in cands for p in cands]
    g = got.astype(np.float64)
    ok = np.zeros(got.shape, bool)
    for o in outs:
        ok |= (g == o.astype(np.float64)) | (np.isnan(got) & np.isnan(o))
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError(f"{what}: {(~ok).sum()} / {ok.size} outputs are no rounding of the normalised RoPE; first at "
                             f"{i}: got {got[i]!r}, allowed {[o[i] for o in outs]}")


def torch_chain(x, w, cos_rows, sin_rows):
    """LlamaRMSNorm / Qwen3RMSNorm then apply_rotary_pos_emb, on the device: x [B, heads, 128], w [heads, 128] fp16."""
    from kivi_b200.llama_kivi import _rotate_half
    h = x.float()
    h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + EPS)
    n = w * h.to(x.dtype)
    return n * cos_rows + _rotate_half(n) * sin_rows


# ---------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------
REGIMES = ["unit", "tiny", "std300", "zero_head", "outlier", "nan", "inf", "near_max"]


def _qkv(rng, B, H, Hkv, regime):
    n = H + 2 * Hkv
    if regime == "near_max":                      # |x| near 65504: x^2 only fits the fp32 statistics
        x = rng.uniform(60000.0, 65504.0, (B, n, 128)) * rng.choice([-1.0, 1.0], (B, n, 128))
    else:
        std = {"unit": 1.0, "tiny": 2.0 ** -20, "std300": 300.0, "zero_head": 1.0, "outlier": 1.0, "nan": 1.0,
               "inf": 1.0}[regime]
        x = rng.standard_normal((B, n, 128)) * std
    if regime == "zero_head":                     # a q head and a k head of zeros in every row
        x[:, rng.integers(0, H)] = 0.0
        x[:, H + rng.integers(0, Hkv)] = 0.0
    if regime == "outlier":                       # one channel per head at 2000 ... 60000
        ch = rng.integers(0, 128, (B, n))
        x[np.arange(B)[:, None], np.arange(n)[None], ch] = np.exp(rng.uniform(np.log(2000.0), np.log(60000.0), (B, n)))
    if regime == "nan":                           # one NaN channel in some heads
        x[:, rng.choice(n, n // 3, replace=False), rng.integers(0, 128)] = np.nan
    if regime == "inf":                           # one +-inf channel in some heads: NaN there, +-0 elsewhere in the head
        x[:, rng.choice(n, n // 3, replace=False), rng.integers(0, 128)] = np.inf * rng.choice([-1.0, 1.0])
    return x.astype(np.float16).reshape(B, n * 128)


def _weights(rng, kind):
    """q and k norm weights [128] each: U(0.2, 3), or U(0.2, 3) with random signs."""
    w = rng.uniform(0.2, 3.0, (2, 128))
    if kind == "signed":
        w *= rng.choice([-1.0, 1.0], (2, 128))
    return w.astype(np.float16)


def _run(qkv16, cos, sin, pos, H, Hkv, w16):
    from kivi_b200 import glue
    B = qkv16.shape[0]
    qkv = torch.from_numpy(qkv16).cuda()
    p = torch.as_tensor(pos, dtype=torch.int64).cuda()
    q = torch.full((B, H, 128), float("nan"), device="cuda", dtype=torch.float16)
    k = torch.full((B, Hkv, 128), float("nan"), device="cuda", dtype=torch.float16)
    v = torch.full_like(k, float("nan"))
    wq, wk = (torch.from_numpy(w).cuda() for w in w16)
    glue.rope_split(qkv, cos, sin, p, q, k, v, wq, wk, EPS)
    return qkv, p, q, k, v, wq, wk


def _check(B, H, Hkv, pos, regime, wkind, seed, theta=1e6):
    rng = np.random.default_rng(seed)
    cos, sin, cn, sn = _tables(theta)
    qkv16 = _qkv(rng, B, H, Hkv, regime)
    w16 = _weights(rng, wkind)
    qkv, p, q, k, v, wq, wk = _run(qkv16, cos, sin, pos, H, Hkv, w16)
    what = f"qk_norm rope B={B} H={H}/{Hkv} {regime} {wkind}"
    x = qkv16.reshape(B, H + 2 * Hkv, 128)
    rows = np.clip(np.asarray(pos, np.int64), 0, TABLE_ROWS - 1)
    c, s = cn[rows][:, None], sn[rows][:, None]
    wh = np.concatenate([np.repeat(w16[:1], H, 0), np.repeat(w16[1:], Hkv, 0)])     # [H + Hkv, 128]
    got = np.concatenate([to_np(q), to_np(k)], 1)
    check_norm_rope(got, x[:, :H + Hkv], wh, c, s, what)
    ev = x[:, H + Hkv:]
    assert np.array_equal(to_np(v).view(np.uint16), ev.view(np.uint16)), what + ": v is not an exact copy"
    xt = qkv.view(B, H + 2 * Hkv, 128)
    tr = p.clamp(0, TABLE_ROWS - 1)
    exp = torch_chain(xt[:, :H + Hkv], torch.cat([wq.expand(H, 128), wk.expand(Hkv, 128)]), cos[tr][:, None],
                      sin[tr][:, None])
    got_nf, exp_nf = ~np.isfinite(got.astype(np.float64)), ~np.isfinite(to_np(exp).astype(np.float64))
    assert (got_nf == exp_nf).all(), f"{what}: non-finite at {got_nf.sum()} positions, torch chain at {exp_nf.sum()}"
    at0 = rows == 0             # cos 1, sin 0: the output is the normalised value itself (a NaN partner would leak in)
    if at0.any() and np.isfinite(x).all():
        check_rounded_product(got[at0], wh[None], rmsnorm_inner64(x[at0, :H + Hkv]), what + ": at position 0")
    # the plain entry on the same operands is unchanged
    from kivi_b200 import glue
    q2, k2, v2 = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    glue.rope_split(qkv, cos, sin, p, q2, k2, v2)
    eq, ek, _ = rope_ref(qkv16, cn, sn, pos, H, Hkv)
    assert_bits(to_np(q2), eq, what + ": plain q")
    assert_bits(to_np(k2), ek, what + ": plain k")
    return got


HEADS = [(16, 8), (32, 8), (40, 8), (64, 8)]


@pytest.mark.parametrize("B", [1, 32, 64])
@pytest.mark.parametrize("H,Hkv", HEADS)
def test_qk_norm_rope_shapes(H, Hkv, B):
    """Every Qwen3 head count, per-row positions including the first and last table rows."""
    rng = np.random.default_rng(H * 7 + B)
    _check(B, H, Hkv, _positions(rng, B), "unit", "signed", seed=int(rng.integers(1 << 30)))


@pytest.mark.parametrize("wkind", ["positive", "signed"])
@pytest.mark.parametrize("regime", REGIMES)
def test_qk_norm_rope_magnitudes(regime, wkind):
    rng = np.random.default_rng(REGIMES.index(regime) * 31 + len(wkind))
    pos = _positions(rng, 64)
    pos[:3] = 0                                   # rows where the output is the normalised value
    got = _check(64, 40, 8, pos, regime, wkind, seed=int(rng.integers(1 << 30)))
    if regime in ("unit", "std300", "near_max", "outlier", "tiny"):
        assert np.isfinite(got.astype(np.float64)).all()
    if regime == "near_max":                      # normalised: far inside the fp16 range
        assert np.abs(got.astype(np.float64)).max() < 100
    if regime in ("nan", "inf"):
        assert np.isnan(got.astype(np.float64)).any() and np.isfinite(got.astype(np.float64)).any()


def test_qk_norm_rope_zero_head_is_zero():
    rng = np.random.default_rng(5)
    qkv16 = np.zeros((4, (32 + 16) * 128), np.float16)
    cos, sin, _, _ = _tables(1e6)
    _, _, q, k, _, _, _ = _run(qkv16, cos, sin, [0, 7, 4095, 40000], 32, 8, _weights(rng, "signed"))
    assert (to_np(q) == 0).all() and (to_np(k) == 0).all()


def test_qk_norm_rope_clamps_positions():
    """Out-of-table positions read the nearest row, as the plain entry."""
    pos = np.array([-1, TABLE_ROWS, 10 ** 9, -(10 ** 12), TABLE_ROWS - 1, 0, TABLE_ROWS + 1, 2 ** 62], np.int64)
    _check(len(pos), 32, 8, pos, "unit", "signed", seed=14)


def test_qk_norm_rope_arbitrary_tables_and_weights_per_head_kind():
    """Random tables tell the halves apart; q heads must read the q weight and k heads the k weight."""
    from kivi_b200 import glue
    rng = np.random.default_rng(11)
    rows = 300
    cn = rng.uniform(-1, 1, (rows, 128)).astype(np.float16)
    sn = rng.uniform(-1, 1, (rows, 128)).astype(np.float16)
    cos, sin = torch.from_numpy(cn).cuda(), torch.from_numpy(sn).cuda()
    B, H, Hkv = 16, 32, 8
    qkv16 = _qkv(rng, B, H, Hkv, "unit")
    pos = rng.integers(0, rows, B)
    w16 = _weights(rng, "signed")
    _, _, q, k, _, _, _ = _run(qkv16, cos, sin, pos, H, Hkv, w16)
    x = qkv16.reshape(B, H + 2 * Hkv, 128)
    c, s = cn[pos][:, None], sn[pos][:, None]
    check_norm_rope(to_np(q), x[:, :H], np.repeat(w16[:1], H, 0), c, s, "q with the q weight")
    check_norm_rope(to_np(k), x[:, H:H + Hkv], np.repeat(w16[1:], Hkv, 0), c, s, "k with the k weight")
    with pytest.raises(AssertionError):
        check_norm_rope(to_np(k), x[:, H:H + Hkv], np.repeat(w16[:1], Hkv, 0), c, s, "k with the q weight")
    # eps reaches the kernel: a tiny head normalises differently with eps 0
    tiny = (rng.standard_normal((1, (H + 2 * Hkv) * 128)) * 2.0 ** -12).astype(np.float16)
    outs = []
    for eps in (EPS, 0.0):
        qq = torch.empty(1, H, 128, device="cuda", dtype=torch.float16)
        kk, vv = (torch.empty(1, Hkv, 128, device="cuda", dtype=torch.float16) for _ in range(2))
        glue.rope_split(torch.from_numpy(tiny).cuda(), cos, sin, torch.zeros(1, dtype=torch.int64, device="cuda"), qq, kk,
                        vv, torch.from_numpy(w16[0]).cuda(), torch.from_numpy(w16[1]).cuda(), eps)
        outs.append(to_np(qq))
    assert not np.array_equal(outs[0], outs[1])


def test_qk_norm_rope_wrapper_checks():
    from kivi_b200 import glue
    dev, h = "cuda", torch.float16
    B, H, Hkv = 2, 4, 2
    qkv = torch.zeros(B, (H + 2 * Hkv) * 128, device=dev, dtype=h)
    cos, sin = torch.ones(8, 128, device=dev, dtype=h), torch.zeros(8, 128, device=dev, dtype=h)
    pos = torch.zeros(B, dtype=torch.int64, device=dev)
    q, k, v = (torch.empty(B, n, 128, device=dev, dtype=h) for n in (H, Hkv, Hkv))
    w = torch.ones(128, device=dev, dtype=h)
    for bad in (dict(wq=w.float()), dict(wk=torch.ones(64, device=dev, dtype=h)), dict(wq=w.cpu()),
                dict(eps=float("nan")), dict(eps=float("inf")), dict(eps=-1e-6), dict(eps=None),
                dict(wk=torch.ones(256, device=dev, dtype=h)[::2])):
        a = dict(wq=w, wk=w, eps=1e-6)
        a.update(bad)
        with pytest.raises((ValueError, RuntimeError)):
            glue.rope_split(qkv, cos, sin, pos, q, k, v, a["wq"], a["wk"], a["eps"])
    glue.rope_split(qkv, cos, sin, pos, q, k, v, w, w, 0.0)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------
# production wiring
# ---------------------------------------------------------------------------------------------------
def _one_layer(model_type):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config("qwen3-8b", num_hidden_layers=1, rms_norm_eps=EPS, model_type=model_type)
    torch.manual_seed(5)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg)
    return cfg, model.half().eval()


def test_decode_step_qk_norm_wiring():
    """One layer with Qwen3-8B layer shapes (H 32, Hkv 8, head_dim 128, hidden 4096; eps set to the bar's 1e-5): a
    left-padded batch of 8 is prefilled, then decoded through the CUDA graph; q and k of every step meet the bar against
    the step's own q|k|v and the layer's q_norm / k_norm weights, v is their copy.  The norm adds no launch to the step."""
    cfg, model = _one_layer("qwen3")
    a = model.model.layers[0].self_attn
    gen = np.random.default_rng(3)
    with torch.no_grad():
        a.q_norm.weight.copy_(torch.from_numpy(_weights(gen, "signed")[0]))
        a.k_norm.weight.copy_(torch.from_numpy(_weights(gen, "positive")[1]))
    B, n = 8, 180
    starts = torch.tensor([0, 3, 17, 64, 100, 127, 128, 179])
    mask = (torch.arange(n)[None, :] >= starts[:, None]).long().cuda()
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda")
    model.init_cache(B, n + 8)
    logits = model.prefill(ids, attention_mask=mask)
    cos_t, sin_t = model._tables(torch.device("cuda"))
    cn, sn = to_np(cos_t), to_np(sin_t)
    H, Hkv = cfg.num_attention_heads, cfg.num_key_value_heads
    wh = np.concatenate([np.repeat(to_np(a.q_norm.weight)[None], H, 0), np.repeat(to_np(a.k_norm.weight)[None], Hkv, 0)])
    tok = logits.argmax(-1, keepdim=True)
    exp_pos = (n - starts).numpy()
    for step in range(3):
        model.decode_step(tok)                                               # graph captured at step 0, replayed after
        torch.cuda.synchronize()
        f = model._fast
        pos = to_np(model._pos).ravel() - 1
        assert np.array_equal(pos, exp_pos + step), (step, pos)
        x = to_np(f.qkv).reshape(B, H + 2 * Hkv, 128)
        got = np.concatenate([to_np(f.q), to_np(f.k)], 1)
        check_norm_rope(got, x[:, :H + Hkv], wh, cn[pos][:, None], sn[pos][:, None], f"step {step}: q, k")
        assert np.array_equal(to_np(f.v).view(np.uint16), x[:, H + Hkv:].view(np.uint16)), f"step {step}: v"
        tok = model.next_tokens.view(B, 1).clone()
    twin_cfg, twin = _one_layer("llama")                                     # the same shapes, no q / k norms
    assert twin.model.layers[0].self_attn.q_norm is None
    twin.init_cache(B, n + 8)
    twin.prefill(ids, attention_mask=mask)
    twin.decode_step(tok)
    assert model.launches_per_step is not None and model.launches_per_step == twin.launches_per_step

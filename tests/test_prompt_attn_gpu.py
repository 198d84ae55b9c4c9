"""The prompt-attention kernel (kivi_prompt_attention_f16, glue.prompt_attention) and the model's prompt pass on it.

Kernel: against a float64 reference -- an explicit masked softmax of the rule lo <= j <= i, lo = max(s_b, i - W + 1) --
on strided q / k / v laid out as the model's projections leave them.  The bar is twice the error of today's call, SDPA
with an additive fp16 mask over K / V expanded to the query heads, on the same fp16 inputs, plus 1e-3; rows with no
visible key are exactly zero.  Model: the padded and the windowed prompt pass against the same model with the kernel
replaced by that SDPA call, against transformers (tests/_hf.py), and the memory the pass holds."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests._hf import (Bar, checkpoints, exports, hf_kw, hf_positions, load_kivi, pad_mask,  # noqa: F401
                       reference_models, reference_step)
from tests._model import TupleBar, small_cfg

pytestmark = pytest.mark.gpu

D = 128


def _qkv(B, H, Hkv, n, seed, q_std=1.0, k_std=1.0, v_std=1.0, v_clip=None):
    """q [B, H, n, 128], k / v [B, Hkv, n, 128] fp16: transposed views of [B, n, heads, 128] storage, the layout of
    LlamaFlashAttention_KIVI._qkv."""
    gen = torch.Generator(device="cuda").manual_seed(seed)

    def make(heads, std):
        return (torch.randn((B, n, heads, D), generator=gen, device="cuda") * std).half().transpose(1, 2)
    q, k, v = make(H, q_std), make(Hkv, k_std), make(Hkv, v_std)
    if v_clip is not None:
        v = v.clamp_(-v_clip, v_clip)
    return q, k, v


def _visible(n, starts, window, device="cuda"):
    """keep [B, n, n]: query i of row b sees key j."""
    i = torch.arange(n, device=device)
    s = torch.tensor([min(max(int(x), 0), n) for x in starts], device=device)
    lo = s[:, None].expand(-1, n)
    if window:
        lo = torch.maximum(lo, (i - window + 1)[None, :])
    return (i[None, None, :] >= lo[:, :, None]) & (i[None, None, :] <= i[None, :, None])


def _ref64(q, k, v, keep):
    """float64 reference [B, n, H, 128]; rows with no visible key are 0."""
    B, H, n, _ = q.shape
    G = H // k.shape[1]
    out = torch.zeros((B, n, H, D), dtype=torch.float64, device=q.device)
    for b in range(B):
        for h in range(H):
            s = (q[b, h].double() @ k[b, h // G].double().T) / math.sqrt(D)
            s = s.masked_fill(~keep[b], float("-inf"))
            p = torch.softmax(s, -1).nan_to_num(0.0)
            out[b, :, h] = p @ v[b, h // G].double()
    return out


def _sdpa16(q, k, v, keep):
    """Today's prompt attention with a mask: SDPA over K / V expanded to the query heads, an additive fp16 mask."""
    from kivi_b200.llama_kivi import repeat_kv
    G = q.shape[1] // k.shape[1]
    mask = torch.zeros(keep.shape, dtype=torch.float16, device=q.device).masked_fill(~keep, torch.finfo(torch.float16).min)
    o = F.scaled_dot_product_attention(q, repeat_kv(k, G), repeat_kv(v, G), attn_mask=mask[:, None])
    return o.transpose(1, 2)


def _run(q, k, v, starts=None, window=0):
    from kivi_b200 import glue
    B, H, n, _ = q.shape
    out = torch.empty((B, n, H, D), dtype=torch.float16, device="cuda")
    ks = None if starts is None else torch.tensor(starts, dtype=torch.int32, device="cuda")
    return glue.prompt_attention(q, k, v, out, ks, window)


def _check(q, k, v, starts, window, what):
    keep = _visible(q.shape[2], starts, window)
    ours = _run(q, k, v, starts, window)
    assert torch.isfinite(ours).all(), what
    ref = _ref64(q, k, v, keep)
    rows = keep.any(-1)                                                     # [B, n]: queries with a visible key
    assert torch.equal(ours[~rows], torch.zeros_like(ours[~rows])), f"{what}: rows with no visible key are not zero"
    if rows.any():
        sdpa = _sdpa16(q, k, v, keep)
        err = (ours[rows].double() - ref[rows]).abs().max().item()
        base = (sdpa[rows].double() - ref[rows]).abs().max().item()
        assert err <= 2 * base + 1e-3, f"{what}: max|ours - ref64| {err:.3g} > 2 * {base:.3g} + 1e-3"


NS = [1, 63, 64, 65, 127, 128, 129, 1000, 4097]
GS = [1, 2, 4, 7, 8]


def _start_set(n):
    return [0, 1, 63, 64, 65, 127, 128, 129, n - 1, n, n + 7]


@pytest.mark.parametrize("G", GS)
@pytest.mark.parametrize("n", NS)
def test_kernel_matches_float64(n, G):
    """Every window of {0, 1, 63, 64, 65, n - 1, n, n + 5}; three rows with different starts, which walk through
    {0, 1, tile edges +- 1, n - 1, n, > n} as the window changes."""
    Hkv = 2 if G <= 4 else 1
    q, k, v = _qkv(3, G * Hkv, Hkv, n, seed=n * 10 + G)
    S = _start_set(n)
    for w_i, W in enumerate([0, 1, 63, 64, 65, n - 1, n, n + 5]):
        if W < 0:
            continue
        starts = [S[(3 * w_i + r) % len(S)] for r in range(3)]
        if w_i == 0:
            starts[0] = 0
        _check(q, k, v, starts, W, f"n {n} G {G} W {W} starts {starts}")


@pytest.mark.parametrize("G", [65, 128])
@pytest.mark.parametrize("n", [1, 129, 1000])
def test_kernel_matches_float64_large_groups(n, G):
    """More than 64 query heads per KV head: the group is split over CTAs of 64 heads each (G = 65: a last CTA of one
    head)."""
    q, k, v = _qkv(2, G, 1, n, seed=n + G)
    for starts, W in (([0, 0], 0), ([1, 64], 0), ([0, n - 1], 65), ([129, n + 7], 1)):
        _check(q, k, v, starts, W, f"n {n} G {G} W {W} starts {starts}")


@pytest.mark.parametrize("case", ["peaked", "flat", "large_v"])
def test_kernel_magnitudes(case):
    """Logits q.k / sqrt(128) of std ~30 (one key dominates), ~1e-4 (uniform weights), and V up to 3e4."""
    kw = dict(peaked=dict(q_std=5.5, k_std=5.5), flat=dict(q_std=0.01, k_std=0.01),
              large_v=dict(v_std=1.2e4, v_clip=3e4))[case]
    q, k, v = _qkv(3, 8, 2, 1000, seed=7, **kw)
    for starts, W in (([0, 0, 0], 0), ([0, 129, 500], 0), ([5, 64, 900], 200)):
        _check(q, k, v, starts, W, f"{case} starts {starts} W {W}")


def test_padding_blocks_are_never_read():
    """K / V NaN in the 128-token blocks wholly before each row's start: the same bits as with clean K / V."""
    n, starts = 1000, [0, 300, 777]
    q, k, v = _qkv(3, 8, 2, n, seed=11)
    clean = _run(q, k, v, starts)
    kn, vn = k.clone(), v.clone()
    for b, s in enumerate(starts):
        kn[b, :, : s // 128 * 128] = float("nan")
        vn[b, :, : s // 128 * 128] = float("nan")
    assert torch.equal(_run(q, kn, vn, starts), clean)
    assert torch.equal(_run(q, kn, vn, starts, 200), _run(q, k, v, starts, 200))


def test_deterministic_and_graph_capturable():
    from kivi_b200 import glue
    q, k, v = _qkv(3, 16, 4, 1000, seed=5)
    ks = torch.tensor([0, 130, 600], dtype=torch.int32, device="cuda")
    a, b = (glue.prompt_attention(q, k, v, torch.empty((3, 1000, 16, D), dtype=torch.float16, device="cuda"), ks, 300)
            for _ in range(2))
    assert torch.equal(a, b)
    out = torch.zeros_like(a)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        glue.prompt_attention(q, k, v, out, ks, 300)                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        glue.prompt_attention(q, k, v, out, ks, 300)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)


def test_64bit_offsets():
    """B * H * n * 128 > 2^31 elements in q and out: the rows of the last sequence and head against the reference."""
    B, H, Hkv, n, W = 17, 32, 8, 32768, 512
    assert B * H * n * D > 2 ** 31
    q, k, v = _qkv(B, H, Hkv, n, seed=3)
    starts = [0] * (B - 1) + [1000]
    ours = _run(q, k, v, starts, W)
    b, h = B - 1, H - 1
    i = torch.cat([torch.arange(990, 1010), torch.arange(n - 200, n)]).cuda()
    got = ours[b, i, h].double()
    for r, t in enumerate(i.tolist()):
        lo = max(1000, t - W + 1)
        if t < lo:
            assert torch.equal(got[r], torch.zeros_like(got[r]))
            continue
        s = (q[b, h, t].double() @ k[b, h // 4, lo:t + 1].double().T) / math.sqrt(D)
        exp = torch.softmax(s, -1) @ v[b, h // 4, lo:t + 1].double()
        assert (got[r] - exp).abs().max().item() <= 2e-3, f"token {t}"
    del ours, q, k, v
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ model level
def _old_prompt_attention(q, k, v, out, kv_start=None, window=None):
    """glue.prompt_attention replaced by the call the model made before the kernel: SDPA with the additive mask."""
    B, H, n, _ = q.shape
    starts = [0] * B if kv_start is None else kv_start.tolist()
    keep = _visible(n, starts, window or 0)
    out.copy_(_sdpa16(q, k, v, keep))
    return out


def _spy(monkeypatch):
    from kivi_b200 import glue
    calls = []
    real = glue.prompt_attention

    def spy(*a, **kw):
        calls.append(1)
        return real(*a, **kw)
    monkeypatch.setattr(glue, "prompt_attention", spy)
    return calls


@pytest.mark.parametrize("kind", ["padded", "windowed"])
def test_prefill_matches_masked_sdpa(monkeypatch, kind):
    """A left-padded prompt, and an unpadded one 5x longer than the window, through prefill(): the kernel against the
    same model with the kernel replaced by the masked SDPA call, at TupleBar's prompt bar; the K / V bits of layer 0
    are the same."""
    from kivi_b200 import glue
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    cfg = small_cfg(sliding_window=64) if kind == "windowed" else small_cfg()
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    B, n = 3, 320
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda")
    mask = pad_mask([0, 37, 250], n) if kind == "padded" else None
    results = []
    for old in (False, True):
        with monkeypatch.context() as m:
            calls = _spy(m) if not old else None
            if old:
                m.setattr(glue, "prompt_attention", _old_prompt_attention)
            model.init_cache(B, n + 8)
            logits = model.prefill(ids, attention_mask=mask)
            if calls is not None:
                assert len(calls) == cfg.num_hidden_layers
            results.append((logits, model.cache.export(0)))
    (ours, kv), (ref, kv_ref) = results
    TupleBar(f"prompt kernel {kind}").prompt(ours, ref)
    for a, b in zip(kv, kv_ref):                                      # eight tensors (or None) and kv_seq_len
        assert torch.equal(a, b) if torch.is_tensor(a) else a == b


def test_generate_matches_transformers(checkpoints, monkeypatch):
    """The windowed Mistral checkpoint of the parity tests, a left-padded prompt longer than the window: prefill and the
    prompt of forward() on the 9-tuple path run the kernel and agree with transformers at the parity bar.  generate()'s
    tokens are then replayed step by step: each step's logits against transformers seeded with the model's own cache at
    that step (tests/_hf.py reference_step), and each generated token against transformers' argmax where the bar
    decides it."""
    bar = Bar()
    window, R = 160, 64
    path = checkpoints("mistral", sliding_window=window)
    ref64, hf16 = reference_models("mistral", path)
    model = load_kivi("mistral", path, residual_length=R)
    B, n = 3, window + 150
    gen = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, model.config.vocab_size, (B, n), device="cuda", generator=gen)
    pads = [0, 17, n - 5]
    mask = pad_mask(pads, n)
    kw = dict(attention_mask=mask, position_ids=hf_positions(mask))
    ref = ref64(input_ids=ids, **hf_kw(kw, torch.float64, window)).logits
    hf = hf16(input_ids=ids, **hf_kw(kw, torch.float16, window)).logits
    calls = _spy(monkeypatch)
    model.fused_forward = False
    real = mask.bool()
    bar.check("kernel forward", model(input_ids=ids, **kw).logits[real], ref[real], hf[real])
    assert len(calls) == model.config.num_hidden_layers
    model.fused_forward = True
    model.init_cache(B, n + 16)
    bar.check("kernel prefill", model.prefill(ids, attention_mask=mask), ref[:, -1], hf[:, -1])
    steps = 12
    out = model.generate(ids, attention_mask=mask, max_new_tokens=steps + 1)
    assert out.shape == (B, n + steps + 1)
    bar.argmax_agrees("generate token 0", out[:, n], ref[:, -1], hf[:, -1])
    model.prefill(ids, attention_mask=mask)                       # the same prompt pass, then generate()'s tokens
    pos = [n - p for p in pads]
    for s in range(steps):
        tok = out[:, n + s]
        r, h = reference_step(ref64, hf16, exports(model), model.config, tok, pos, pads)
        bar.check(f"generate step {s}", model.decode_step(tok.view(B, 1)).clone(), r, h)
        bar.argmax_agrees(f"generate token {s + 1}", out[:, n + s + 1], r, h)
        pos = [p + 1 for p in pos]
    bar.report("prompt kernel against transformers")


@pytest.mark.parametrize("kind", ["right_padded", "holes", "empty_row", "4d"])
def test_windowed_tuple_prompt_keeps_other_masks(monkeypatch, kind):
    """A windowed model (n > W) on the 9-tuple path with a mask the kernel's rule does not state -- right padding,
    holes, a row with no real token, a 4-D additive mask -- runs today's additive mask combined with the window: the
    kernel is not called and the logits and K / V are those of the model made to take the additive mask."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, _additive_mask
    cfg = small_cfg(sliding_window=48)
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    model.fused_forward = False
    B, n = 2, 200
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda")
    mask = torch.ones((B, n), dtype=torch.long, device="cuda")
    if kind == "right_padded":
        mask[1, n - 30:] = 0
    elif kind == "holes":
        mask[0, 50:60] = 0
    elif kind == "empty_row":
        mask[1] = 0
    else:
        mask = _additive_mask(None, n, n, torch.float16, ids.device, 48, B).clone()
        mask[1, :, :, :20] = torch.finfo(torch.float16).min
    calls = _spy(monkeypatch)
    logits, pasts = model(input_ids=ids, attention_mask=mask, return_dict=False)
    assert not calls, "the prompt-attention kernel ran for a mask it does not state"
    monkeypatch.setattr(model, "_tuple_prompt_mask", lambda *a: None)
    ref_logits, ref_pasts = model(input_ids=ids, attention_mask=mask, return_dict=False)
    same = lambda a, b: torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)    # noqa: E731 (bits)
    same(logits, ref_logits)
    for a, b in zip(pasts[-1], ref_pasts[-1]):
        if torch.is_tensor(a):
            same(a, b)
        else:
            assert a == b


def test_long_padded_prompt_memory():
    """B 2, n 32768, left-padded: B * n is 4 chunks.  The pass holds the residual stream, q, k, v, the attention output,
    the cache's contiguous K / V copies and one chunk's temporaries, with no B * n^2 mask and no [B * n, intermediate]
    tensor: its peak above the weights and the cache stays under that bound (today's mask alone is 4.3 GB)."""
    from kivi_b200.llama_kivi import PROMPT_CHUNK_ROWS, LlamaForCausalLM_KIVI
    cfg = small_cfg(num_hidden_layers=2)
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    B, n = 2, 32768
    rows = B * n
    assert rows > PROMPT_CHUNK_ROWS
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda")
    mask = pad_mask([0, 5000], n)
    model.init_cache(B, n + 8)
    model._tables(ids.device)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    logits = model.prefill(ids, attention_mask=mask)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    hid, H, Hkv, inter = cfg.hidden_size, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.intermediate_size
    f16 = 2
    whole = rows * f16 * (2 * hid + 2 * H * D + 4 * Hkv * D + 2 * D) + rows * 8 * 4   # residual x2, q, out, k, v + copies,
    chunk = PROMPT_CHUNK_ROWS * (f16 * (6 * hid + 2 * (H + 2 * Hkv) * D + 4 * inter) + 4 * 3 * hid)  # cos/sin, ids, positions
    bound = whole + chunk + (64 << 20)
    mask_bytes = B * n * n * f16
    print(f"\n[prompt memory] peak above weights + cache {peak / 2**20:.0f} MiB, bound {bound / 2**20:.0f} MiB, "
          f"dense mask {mask_bytes / 2**20:.0f} MiB")
    assert torch.isfinite(logits).all()
    assert peak <= bound < mask_bytes

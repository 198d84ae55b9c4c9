"""Model-level parity: the fused cache path (one launch per layer) against the tuple path that restates
the reference hook op for op (kivi_decode_attention_tuple), and the tuple path against the CPU oracle."""
import numpy as np
import pytest
import torch

from oracle import ref
from tests._model import TupleBar, packed_parts_equal, tuple_prompt, tuple_steps
from tests._util import to_np

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H,Hkv,kb,vb,g,R,n0,steps", [(4, 4, 2, 2, 32, 128, 200, 70), (8, 2, 4, 4, 64, 64, 100, 40)])
def test_tuple_hook_matches_oracle(H, Hkv, kb, vb, g, R, n0, steps):
    """kivi_decode_attention_tuple / kivi_prefill_tuple == oracle decode_step / prefill_cache
    (models/llama_kivi.py:314-455): cache tuple bit-exact, outputs within the end-to-end tolerance."""
    from kivi_b200.llama_kivi import kivi_decode_attention_tuple, kivi_prefill_tuple
    rng = np.random.default_rng(H * 10 + R)
    B = 2
    k = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    v = rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)
    past = kivi_prefill_tuple(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), g, kb, vb, R)
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    for step in range(steps):
        q = (rng.standard_normal((B, H, 1, 128)) * 0.7).astype(np.float16)
        kn = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
        vn = rng.standard_normal((B, Hkv, 1, 128)).astype(np.float16)
        out, past = kivi_decode_attention_tuple(torch.from_numpy(q).cuda(), torch.from_numpy(kn).cuda(),
                                                torch.from_numpy(vn).cuda(), past, g, kb, vb, R)
        exp, _, st = ref.decode_step(st, q, kn, vn, g, kb, vb, R)
        err = np.abs(to_np(out).astype(np.float64) - exp.astype(np.float64))
        assert (err <= 2e-2 * np.abs(exp.astype(np.float64)) + 5e-3 * np.abs(exp).max()).all(), (step, err.max())
    assert past[8] == st[8]
    for i in (0, 2, 3, 4, 6, 7, 1, 5):
        if st[i] is None:
            assert past[i] is None
            continue
        a = to_np(past[i])
        np.testing.assert_array_equal(a.view(np.uint16) if a.dtype == np.float16 else a,
                                      st[i].view(np.uint16) if st[i].dtype == np.float16 else st[i])


_GQA_K4V4 = dict(num_attention_heads=4, num_key_value_heads=1, hidden_size=512, k_bits=4, v_bits=4, group_size=64,
                 residual_length=64)


@pytest.mark.parametrize("name,kw", [("tiny", {}), ("tiny", _GQA_K4V4), ("tiny", dict(attention_bias=True))])
def test_fused_model_matches_tuple_model(name, kw, request):
    """LlamaForCausalLM_KIVI: prefill + greedy decode through the fused cache path (CUDA graph) and through
    the reference-style forward with per-layer 9-tuples give the same logits (two independent code paths).  With
    attention biases the tuple path keeps the module linears, the decode step adds the fused biases in its GEMMs."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config(name, **kw)
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    with torch.no_grad():
        for pname, p in model.named_parameters():
            if pname.endswith(".bias"):
                p.uniform_(-1.0, 1.0)                 # as large as the projections' outputs: a dropped bias must show
    ids = torch.randint(0, cfg.vocab_size, (2, 150), device="cuda")
    _decode_against_tuple_path(model, ids, 40, request.node.name)


def test_one_token_prompt_is_prefilled():
    """A one-token prompt is a prompt like any other: prefill() and forward() write it into the fused cache, the decode
    steps after it match the 9-tuple path, and a prompt pass on a cache that still holds an earlier sequence reads none
    of it."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config("tiny", **_GQA_K4V4)
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    B = 2
    ids = torch.randint(0, cfg.vocab_size, (B, 150), device="cuda")
    one = ids[:, :1]
    model.init_cache(B, 8)
    model.prefill(one)
    assert model.cache.kv_len == 1
    assert model(input_ids=one).past_key_values[0][-1] == 1
    # 70 steps cross a K flush (R = 64) and move the V window
    _decode_against_tuple_path(model, one, 70, "test_one_token_prompt_is_prefilled")
    # after a generate() of a longer prompt the same one-token prefill gives the bits it gives on a new cache
    model.generate(ids, max_new_tokens=8)
    got = model.prefill(one).clone()
    assert model.cache.kv_len == 1
    model.init_cache(B, 8)
    assert torch.equal(got, model.prefill(one))


def _decode_against_tuple_path(model, ids, steps, site):
    """Prefill `ids`, then `steps` teacher-forced decode steps on the fused cache and through forward() on the reference's
    9-tuples (tests/_model.py: TupleBar), and the packed cache parts equal."""
    bar = TupleBar(site)
    model.init_cache(ids.shape[0], ids.shape[1] + steps + 4)
    pasts = tuple_steps(model, *tuple_prompt(model, ids, bar), steps, bar)
    bar.done(steps)
    packed_parts_equal(model.cache.export(0), pasts[0], "layer 0")


def test_forward_loop_runs_on_the_fused_cache():
    """The reference's calling convention -- `out = model(input_ids=..., past_key_values=out.past_key_values)` in a loop,
    models/llama_kivi.py:815-905 -- lands on the pre-allocated cache: the per-layer past is a KiviPast view ([-1] =
    kv_seq_len, tensors exported on access), logits equal the decode_step path bit for bit, a cache grown by the tuple path is
    imported once and continued, and anything the fused path does not cover (padding mask) falls back to real 9-tuples."""
    from kivi_b200.llama_kivi import KiviPast, LlamaForCausalLM_KIVI, default_config
    cfg = default_config("tiny", num_attention_heads=4, num_key_value_heads=2, hidden_size=512)
    torch.manual_seed(3)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    B, n = 2, 140
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda")
    out = model(input_ids=ids)
    logits, past = out
    assert logits.shape == (B, n, cfg.vocab_size) and logits.dtype == torch.float32
    assert all(isinstance(p_, KiviPast) for p_ in past) and past[0][-1] == n and len(past[0]) == 9
    inp = model.prepare_inputs_for_generation(torch.cat([ids, logits[:, -1].argmax(-1, keepdim=True)], 1), past_key_values=past)
    assert inp["input_ids"].shape == (B, 1)
    # the same steps through decode_step on a second model object with the same weights
    twin = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    twin.load_state_dict(model.state_dict())
    twin.init_cache(B, n + 64)
    l2 = twin.prefill(ids)
    assert torch.allclose(l2, logits[:, -1], rtol=1e-2, atol=1e-2)      # lm_head on [B, n, hid] vs [B, hid]: other GEMM shape
    tok = logits[:, -1].argmax(-1, keepdim=True)
    for step in range(20):
        logits, past = model(input_ids=tok, past_key_values=past)
        l2 = twin.decode_step(tok)
        assert logits.shape == (B, 1, cfg.vocab_size) and torch.equal(logits[:, 0], l2), step
        tok = logits[:, -1].argmax(-1, keepdim=True)
    assert past[0][8] == n + 20
    snap = past[1]
    fields = snap.materialise()                                        # a 9-tuple snapshot of layer 1
    assert fields[8] == n + 20 and fields[5].shape[2] == min(n + 20, cfg.residual_length)
    old_view = past[0]
    logits, past = model(input_ids=tok, past_key_values=past)          # the cache moves on: unmaterialised older views are stale
    with pytest.raises(RuntimeError, match="stale"):
        old_view[0]
    assert snap[4] is fields[4]                                        # the materialised snapshot stays readable
    # a cache grown on the tuple path continues on the fused path after one import
    model.fused_forward = False
    lt, tp = model(input_ids=ids)
    assert isinstance(tp[0], tuple) and not isinstance(tp[0], KiviPast)
    tok_t = lt[:, -1].argmax(-1, keepdim=True)
    lt, tp = model(input_ids=tok_t, past_key_values=tp)
    model.fused_forward = True
    tok_t = lt[:, -1].argmax(-1, keepdim=True)
    lf, fp_ = model(input_ids=tok_t, past_key_values=tp)               # plain tuples in -> imported -> KiviPast out
    model.fused_forward = False
    lt2, tp2 = model(input_ids=tok_t, past_key_values=tp)
    assert isinstance(fp_[0], KiviPast) and fp_[0][-1] == tp2[0][-1] == n + 2
    bar = TupleBar("test_forward_loop_runs_on_the_fused_cache")
    bar.step(lf, lt2, "the step after the import")
    bar.report()
    packed_parts_equal(fp_[0], tp2[0], "layer 0")
    # a padding mask is outside the fused path: real 9-tuples come back
    model.fused_forward = True
    mask = torch.ones(B, n, dtype=torch.long, device="cuda")
    mask[0, :5] = 0
    lm, pm = model(input_ids=ids, attention_mask=mask)
    assert not isinstance(pm[0], KiviPast) and pm[0][8] == n


def test_generate_runs():
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config("tiny")
    torch.manual_seed(1)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    ids = torch.randint(0, cfg.vocab_size, (3, 140), device="cuda")
    out = model.generate(ids, max_new_tokens=10)
    assert out.shape == (3, 150) and torch.equal(out[:, :140], ids)


def test_glue_kernels_match_torch():
    """The decode-step glue kernels reproduce the fp16 op chains of the HF Llama modules."""
    from kivi_b200 import glue
    from kivi_b200.llama_kivi import _rope_tables, _rotate_half
    torch.manual_seed(0)
    B, H, Hkv, hid, inter = 5, 4, 2, 512, 1408
    # residual-add + RMSNorm (LlamaRMSNorm: fp32 statistics, cast, multiply by the fp16 weight)
    x = torch.randn(B, hid, device="cuda", dtype=torch.float16)
    res = torch.randn(B, hid, device="cuda", dtype=torch.float16)
    w = (torch.rand(hid, device="cuda") + 0.5).half()
    r2 = res.clone()
    out = torch.empty_like(x)
    glue.add_rmsnorm(x, r2, w, out, 1e-5)
    exp_res = res + x
    hs = exp_res.float()
    exp = w * (hs * torch.rsqrt(hs.pow(2).mean(-1, keepdim=True) + 1e-5)).half()
    assert torch.equal(r2, exp_res)
    assert (out.float() - exp.float()).abs().max() <= 2e-3 * exp.float().abs().max()
    # RoPE + split
    qkv = torch.randn(B, (H + 2 * Hkv) * 128, device="cuda", dtype=torch.float16)
    cos_t, sin_t = _rope_tables(128, 64, 10000.0, torch.device("cuda"))
    pos = torch.full((B, 1), 37, dtype=torch.long, device="cuda")
    q = torch.empty(B, H, 128, device="cuda", dtype=torch.float16)
    k = torch.empty(B, Hkv, 128, device="cuda", dtype=torch.float16)
    v = torch.empty_like(k)
    glue.rope_split(qkv, cos_t, sin_t, pos, q, k, v)
    q0, k0, v0 = qkv.view(B, H + 2 * Hkv, 128).split([H, Hkv, Hkv], dim=1)
    c, s = cos_t[37], sin_t[37]
    assert torch.equal(q, q0 * c + _rotate_half(q0) * s)
    assert torch.equal(k, k0 * c + _rotate_half(k0) * s)
    assert torch.equal(v, v0)
    # SiLU * mul
    gu = torch.randn(B, 2 * inter, device="cuda", dtype=torch.float16)
    act = torch.empty(B, inter, device="cuda", dtype=torch.float16)
    glue.silu_mul(gu, act)
    exp = torch.nn.functional.silu(gu[:, :inter]) * gu[:, inter:]
    assert (act.float() - exp.float()).abs().max() <= 2e-3 * exp.float().abs().max() + 1e-4

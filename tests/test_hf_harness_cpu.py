"""The transformers parity harness (tests/_hf.py) on the CPU: the bar accepts hf16 and rejects each single defect,
reference_step is transformers' own next position, the fp64 K / V of a packed 9-tuple is the packed data, and the prompt
mask keeps exactly the causal or banded set.  Tiny transformers models in float64."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests._hf import ALPHA, BETA, Bar, hf_kw, hf_positions, hf_prompt_mask, kv_fp64, pad_mask, reference_step

VOCAB, N = 97, 20


def _tiny(kind, **fields):
    """A random transformers Llama / Mistral in float64 with eager attention, head_dim 128, q_proj and k_proj scaled up so
    attention is peaked (a position or mask error then moves the logits well beyond fp64 rounding)."""
    import transformers
    cfg = getattr(transformers, f"{kind}Config")(hidden_size=256, intermediate_size=256, num_hidden_layers=2,
                                                 num_attention_heads=2, num_key_value_heads=1, vocab_size=VOCAB,
                                                 max_position_embeddings=256, rms_norm_eps=1e-5, **fields)
    torch.manual_seed(0)
    model = getattr(transformers, f"{kind}ForCausalLM")._from_config(cfg, attn_implementation="eager", dtype=torch.float64)
    with torch.no_grad():
        for layer in model.model.layers:
            layer.self_attn.q_proj.weight.mul_(4.0)
            layer.self_attn.k_proj.weight.mul_(4.0)
    return model.eval()


def _logits(seed=0):
    """ref [64, 50] with top-2 margins from none to wide, and hf = ref plus a little noise."""
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(64, 50, generator=g, dtype=torch.float64)
    ref[:, 7] += torch.linspace(0.0, 8.0, 64, dtype=torch.float64)
    return ref, ref + 1e-2 * torch.randn(64, 50, generator=g, dtype=torch.float64)


def test_check_accepts_hf16_and_rejects_each_defect():
    ref, hf = _logits()
    limit = ALPHA * (hf - ref).abs().max().item() + BETA * ref.abs().max().item()
    top2 = ref.topk(2, dim=-1).values
    decided = torch.nonzero(top2[:, 0] - top2[:, 1] > 2 * limit).flatten().tolist()
    undecided = torch.nonzero(top2[:, 0] - top2[:, 1] <= 2 * limit).flatten().tolist()
    assert decided and undecided
    bar = Bar()
    bar.check("hf16 step 3", hf, ref, hf)
    assert bar.worst == {"hf16": [1.0, pytest.approx((hf - ref).abs().max().item() / ref.abs().max().item())]}
    assert bar.decided == [len(decided), 64]
    bar.assert_decided([0, 0])
    with pytest.raises(AssertionError, match="only"):
        bar.assert_decided([0, 0], share=0.99)

    over = ref.clone()
    over[5, 11] += 1.01 * limit
    with pytest.raises(AssertionError, match=r"max\|ours - ref64\| = "):
        bar.check("above the bar", over, ref, hf)
    flip = ref.clone()
    r = decided[0]
    a, b = ref[r].topk(2).indices.tolist()
    flip[r, a], flip[r, b] = ref[r, b], ref[r, a]
    with pytest.raises(AssertionError):
        bar.check("argmax flip", flip, ref, hf)
    for bad in (float("nan"), float("inf")):
        odd = hf.clone()
        odd[9, 3] = bad
        with pytest.raises(AssertionError, match="^non-finite$"):
            bar.check("non-finite", odd, ref, hf)

    ids = ref.argmax(-1)
    bar.argmax_agrees("ids", ids, ref, hf)
    ids[undecided[0]] = (ids[undecided[0]] + 1) % 50              # a row the margin does not decide may differ
    bar.argmax_agrees("ids", ids, ref, hf)
    ids[r] = b
    with pytest.raises(AssertionError, match=f"argmax differs on rows \\[{r}\\]"):
        bar.argmax_agrees("ids", ids, ref, hf)


def _kv_tuples(model, ids, kw):
    """transformers' own post-RoPE K / V of a prompt pass, as 9-tuples with no packed part."""
    from transformers import DynamicCache
    cache = DynamicCache()
    model(input_ids=ids, past_key_values=cache, use_cache=True, **hf_kw(kw, torch.float64))
    n = ids.shape[1]
    return [(None, lay.keys, None, None, None, lay.values, None, None, n) for lay in cache.layers]


@pytest.mark.parametrize("case", ["unpadded", "left-padded", "released", "windowed"])
def test_reference_step_is_transformers_next_position(case):
    """reference_step seeded with the K / V of ids[:, :N] gives the logits of transformers' full forward of ids[:, :N + 1]
    at its last position; a released slot (start None) gives those of its token alone."""
    model = _tiny("Mistral", sliding_window=8) if case == "windowed" else _tiny("Llama")
    B = 3
    ids = torch.randint(0, VOCAB, (B, N + 1), generator=torch.Generator().manual_seed(1))
    pads = [0, 5, N - 3] if case == "left-padded" else [0] * B
    full = pad_mask(pads, N + 1, "cpu")
    kw = dict(attention_mask=full, position_ids=hf_positions(full)) if any(pads) else {}
    want = model(input_ids=ids, **hf_kw(kw, torch.float64)).logits[:, -1]
    prompt = pad_mask(pads, N, "cpu")
    kw = dict(attention_mask=prompt, position_ids=hf_positions(prompt)) if any(pads) else {}
    tuples = _kv_tuples(model, ids[:, :N], kw)
    start, pos = list(pads), [N - p for p in pads]
    if case == "released":
        start[1], pos[1] = None, 4
        want[1] = model(input_ids=ids[1:2, N:], position_ids=torch.tensor([[4]])).logits[0, -1]
    got, again = reference_step(model, model, tuples, model.config, ids[:, N], pos, start)
    assert torch.equal(got, again)
    assert (got - want).abs().max().item() <= 1e-9 * want.abs().max().item()
    if case == "windowed":                      # the window matters: attention over the whole prompt gives other logits
        assert (_tiny("Mistral", sliding_window=None)(input_ids=ids).logits[:, -1] - want).abs().max() > 1e-3


def test_kv_fp64_of_an_oracle_packed_tuple():
    """K packed along tokens, V along channels, as the cache exports them: the fp64 K and V are [B, Hkv, T, 128], the packed
    part the oracle's fp16 dequant to within its two fp16 roundings and the packed data to within half a quantisation
    step, the windows exactly the windows."""
    from oracle import ref
    B, Hkv, D, g, kbits, vbits = 2, 2, 128, 32, 2, 4
    tk, r, tv, L = 64, 16, 77, 3
    rng = np.random.default_rng(0)
    K = rng.standard_normal((B, Hkv, tk + r, D)).astype(np.float16)
    V = rng.standard_normal((B, Hkv, tv + L, D)).astype(np.float16)
    kc, ks, km = ref.pack_lastdim(np.ascontiguousarray(K[:, :, :tk].transpose(0, 1, 3, 2)), g, kbits)
    vc, vs, vm = ref.pack_lastdim(V[:, :, :tv], g, vbits)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))                              # noqa: E731
    k, v = kv_fp64((t(kc), t(K[:, :, tk:]), t(ks), t(km), t(vc), t(V[:, :, tv:]), t(vs), t(vm), tk + r),
                   SimpleNamespace(k_bits=kbits, v_bits=vbits, group_size=g))
    assert k.shape == v.shape == (B, Hkv, tk + r, D) and k.dtype == v.dtype == torch.float64
    assert torch.equal(k[:, :, tk:], t(K[:, :, tk:]).double()) and torch.equal(v[:, :, tv:], t(V[:, :, tv:]).double())
    for got, data, (code, s, z), bits, along_tokens in ((k[:, :, :tk], K[:, :, :tk], (kc, ks, km), kbits, True),
                                                         (v[:, :, :tv], V[:, :, :tv], (vc, vs, vm), vbits, False)):
        deq = ref.unpack_dequant_lastdim(code, s, z, g, bits)
        s, z = (np.repeat(a.astype(np.float64), g, -1) for a in (s, z))
        if along_tokens:
            deq, s, z = (a.transpose(0, 1, 3, 2) for a in (deq, s, z))
        got = got.numpy()
        # the oracle rounds c * s and then (c * s) + z to fp16: half an fp16 ulp each, 2^-24 at the subnormals
        assert (np.abs(deq - got) <= 2.0 ** -11 * (np.abs(got - z) + np.abs(got)) + 2.0 ** -24).all()
        # rounding to the nearest code, plus the fp16 roundings of the quantiser's own arithmetic
        assert (np.abs(got - data) <= s * (0.5 + 3 * (2 ** bits - 1) * 2.0 ** -11)).all()


@pytest.mark.parametrize("window", [None, 4])
def test_hf_prompt_mask_keeps_exactly_the_causal_or_banded_set(window):
    pads, n = [0, 3, 9], 12
    mask = pad_mask(pads, n, "cpu")
    assert hf_positions(mask).tolist() == [[1] * p + list(range(n - p)) for p in pads]
    add = hf_prompt_mask(mask, torch.float64, window)
    assert add.shape == (3, 1, n, n) and add.dtype == torch.float64
    seen = add[:, 0] == 0
    assert (add[:, 0][~seen] == torch.finfo(torch.float64).min).all()
    for b, p in enumerate(pads):
        for i in range(n):
            want = {i} if i < p else {j for j in range(p, i + 1) if window is None or j > i - window}
            assert set(torch.nonzero(seen[b, i]).flatten().tolist()) == want, (b, i)
    assert hf_kw({}, torch.float64, window) == {}                 # an unpadded prompt: transformers' own mask

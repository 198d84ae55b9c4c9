"""LlamaForCausalLM_KIVI on Qwen2 checkpoints against transformers' Qwen2ForCausalLM (save_pretrained, with q / k / v biases
drawn from U(-1, 1) so a dropped bias shows), under the bar and method of tests/test_hf_parity_gpu.py: ratios 7 and 5,
and a tied-embedding case at ratio 3.  Prompt pass unpadded and left-padded, decode across K flushes and the V ring,
insert / release / shift under serve()-style continuous batching, and the tensor-parallel loader at world 1."""
import pytest
import torch

from tests._hf import Bar, Decoder, hf_kw, hf_positions, pad_mask
from tests._qwen import load_kivi, qwen_checkpoints, reference_models  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

bar = Bar()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    bar.report("qwen2 hf parity")


def _prompt(name, model, ref64, hf16, ids, pads, forward=True, tag=""):
    B, n = ids.shape
    mask = pad_mask(pads, n)
    padded = any(pads)
    kw = dict(attention_mask=mask, position_ids=hf_positions(mask)) if padded else {}
    ref = ref64(input_ids=ids, **hf_kw(kw, torch.float64)).logits
    hf = hf16(input_ids=ids, **hf_kw(kw, torch.float16)).logits
    real = mask.bool()
    if forward:
        model.fused_forward = False
        ours = model(input_ids=ids, **kw).logits
        model.fused_forward = True
        bar.check(f"{name} forward{tag}", ours[real], ref[real], hf[real])
    last = model.prefill(ids, attention_mask=mask if padded else None)
    bar.check(f"{name} prefill{tag}", last, ref[:, -1], hf[:, -1])
    return last


@pytest.mark.parametrize("name,tp", [("qwen-ratio7", False), ("qwen-ratio5", False), ("qwen-tied", False),
                                     ("qwen-ratio7", True)])
def test_prompt_and_decode_match_transformers(qwen_checkpoints, name, tp):
    decided0 = list(bar.decided)
    path = qwen_checkpoints(name)
    ref64, hf16 = reference_models(path)
    model = load_kivi(name, path, tensor_parallel=tp)
    assert model.model.layers[0].self_attn.o_proj.bias is None
    if tp:
        name += " tp"
    R = model.config.residual_length
    B, n = 3, 150
    steps = 2 * R + 3
    gen = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, model.config.vocab_size, (B, n), device="cuda", generator=gen)
    for pads in ([0] * B, [0, 17, n - 5]):
        tag = " padded" if any(pads) else ""
        model.init_cache(B, n + steps + 8)
        _prompt(name, model, ref64, hf16, ids, pads, forward=not tp, tag=tag)
        dec = Decoder(bar, model, ref64, hf16, T=n, pos=[n - p for p in pads], start=pads,
                      gen=torch.Generator(device="cuda").manual_seed(sum(pads)))
        dec.run(steps, f"{name} decode{tag}")
        assert dec.flushes >= 2 and model.cache.vhead != 0
    bar.assert_decided(decided0)


def test_continuous_batching_matches_transformers(qwen_checkpoints):
    """insert into slot 2, release slot 1, shift the timeline by 128, keep decoding (as the Llama parity test does)."""
    name = "qwen-ratio5"
    decided0 = list(bar.decided)
    path = qwen_checkpoints(name)
    ref64, hf16 = reference_models(path)
    model = load_kivi(name, path)
    R = model.config.residual_length
    B, n = 4, 200
    pads = [128, 5, 0, 136]
    gen = torch.Generator(device="cuda").manual_seed(2)
    ids = torch.randint(0, model.config.vocab_size, (B, n), device="cuda", generator=gen)
    model.init_cache(B, n + 3 * R + 64)
    _prompt(name, model, ref64, hf16, ids, pads, forward=False, tag=" batch")
    dec = Decoder(bar, model, ref64, hf16, T=n, pos=[n - p for p in pads], start=pads,
                  gen=torch.Generator(device="cuda").manual_seed(3))
    dec.run(10, f"{name} decode batch")
    n_new = 40
    prompt = torch.randint(0, model.config.vocab_size, (1, n_new), device="cuda", generator=gen)
    got = model.insert(2, prompt)
    bar.check(f"{name} insert", got[None], ref64(input_ids=prompt).logits[:, -1], hf16(input_ids=prompt).logits[:, -1])
    dec.pos[2], dec.start[2] = n_new, dec.T - n_new
    dec.run(R // 2, f"{name} decode inserted")
    model.release(1)
    dec.pos[1], dec.start[1] = 0, None
    dec.run(10, f"{name} decode released")
    tk0 = model.cache.tk
    model.cache.shift(128)
    dec.T -= 128
    dec.start = [None if s is None else s - 128 for s in dec.start]
    dec.run(2 * R + 3, f"{name} decode shifted")
    assert model.cache.tk > tk0 - 128 and dec.flushes >= 2
    bar.assert_decided(decided0)


def test_serve_first_tokens_match_transformers(qwen_checkpoints):
    """serve() on the ratio-7 checkpoint with 2 slots and 5 requests (inserts, releases and shifts mid-decode): every
    request gets its max_new_tokens tokens, and its first token is transformers' argmax on the prompt alone wherever the
    ref64 margin decides it."""
    from kivi_b200.serve import serve
    name = "qwen-ratio7"
    path = qwen_checkpoints(name)
    ref64, hf16 = reference_models(path)
    model = load_kivi(name, path)
    gen = torch.Generator(device="cuda").manual_seed(5)
    prompts = [torch.randint(0, model.config.vocab_size, (n,), device="cuda", generator=gen) for n in (30, 70, 50, 90, 20)]
    reqs = [(p, 6 + 3 * i) for i, p in enumerate(prompts)]
    stats = {}
    got = dict(serve(model, reqs, batch=2, max_tokens=384, stats=stats))
    assert sorted(got) == list(range(len(reqs))) and stats["inserts"] == 3
    for i, (p, m) in enumerate(reqs):
        assert got[i].shape == (m,), i
        bar.argmax_agrees(f"{name} serve first token", got[i][:1], ref64(input_ids=p[None]).logits[:, -1],
                          hf16(input_ids=p[None]).logits[:, -1])

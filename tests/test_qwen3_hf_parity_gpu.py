"""LlamaForCausalLM_KIVI on Qwen3 checkpoints against transformers' Qwen3ForCausalLM (save_pretrained, with q_norm / k_norm
weights drawn from U(1, 3) so a dropped weight shows), under the bar and method of tests/test_hf_parity_gpu.py: ratios 2,
4 and 8 with head_dim 128 and hidden_size below heads x 128, tied embeddings with the Qwen vocabulary, and one Mistral
checkpoint with an explicit head_dim 128 != hidden / heads.  Prompt pass unpadded, left-padded and chunked, decode across
K flushes and the V ring, insert / release / shift, serve() with and without a PrefixCache, and the tensor-parallel loader
at world 1 and (with two GPUs) at world 2."""
import os

import pytest
import torch

from tests._hf import Bar, Decoder, hf_kw, hf_positions, pad_mask
from tests._model import same_on_all_ranks, spawn_ranks
from tests._qwen3 import load_kivi, qwen3_checkpoints, reference_models, write_checkpoint  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

bar = Bar()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    bar.report("qwen3 hf parity")


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


@pytest.mark.parametrize("name,tp", [("qwen3-narrow-ratio2", False), ("qwen3-ratio4", False),
                                     ("qwen3-narrow-ratio8", False), ("mistral-narrow", False),
                                     ("qwen3-narrow-ratio2", True)])
def test_prompt_and_decode_match_transformers(qwen3_checkpoints, name, tp):
    decided0 = list(bar.decided)
    path = qwen3_checkpoints(name)
    ref64, hf16 = reference_models(name, path)
    model = load_kivi(name, path, tensor_parallel=tp)
    a = model.model.layers[0].self_attn
    assert a.head_dim == 128 and (a.q_norm is None) == name.startswith("mistral")
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


def test_chunked_prompt_matches_transformers(qwen3_checkpoints, monkeypatch):
    """PROMPT_CHUNK_ROWS lowered to 64: the prompt's norms, projections and q / k norms run in chunks (_qkv_rows)."""
    from kivi_b200 import llama_kivi
    monkeypatch.setattr(llama_kivi, "PROMPT_CHUNK_ROWS", 64)
    name = "qwen3-narrow-ratio8"
    decided0 = list(bar.decided)
    path = qwen3_checkpoints(name)
    ref64, hf16 = reference_models(name, path)
    model = load_kivi(name, path)
    B, n = 3, 150
    gen = torch.Generator(device="cuda").manual_seed(7)
    ids = torch.randint(0, model.config.vocab_size, (B, n), device="cuda", generator=gen)
    for pads in ([0] * B, [0, 33, n - 9]):
        tag = " chunked padded" if any(pads) else " chunked"
        model.init_cache(B, n + 40)
        _prompt(name, model, ref64, hf16, ids, pads, tag=tag)
        dec = Decoder(bar, model, ref64, hf16, T=n, pos=[n - p for p in pads], start=pads,
                      gen=torch.Generator(device="cuda").manual_seed(8))
        dec.run(12, f"{name} decode{tag}")
    bar.assert_decided(decided0)


def test_continuous_batching_matches_transformers(qwen3_checkpoints):
    """insert into slot 2, release slot 1, shift the timeline by 128, keep decoding (as the Llama parity test does)."""
    name = "qwen3-ratio4"
    decided0 = list(bar.decided)
    path = qwen3_checkpoints(name)
    ref64, hf16 = reference_models(name, path)
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


@pytest.mark.parametrize("prefix", [False, True], ids=["no_cache", "prefix_cache"])
def test_serve_first_tokens_match_transformers(qwen3_checkpoints, prefix):
    """serve() on the ratio-2 checkpoint with 2 slots and 5 requests (inserts, releases and shifts mid-decode): every
    request gets its tokens, and its first token is transformers' argmax on the prompt alone wherever the ref64 margin
    decides it.  prefix_cache: the prompts share a system prompt of MIN_REUSE + 40 tokens, so the later inserts run
    their prompt pass on the suffix over the stored K / V."""
    from kivi_b200.prefix import MIN_REUSE, PrefixCache
    from kivi_b200.serve import serve
    name = "qwen3-narrow-ratio2"
    path = qwen3_checkpoints(name)
    ref64, hf16 = reference_models(name, path)
    model = load_kivi(name, path)
    gen = torch.Generator(device="cuda").manual_seed(5)
    head = MIN_REUSE + 40 if prefix else 0
    system = torch.randint(0, model.config.vocab_size, (head,), device="cuda", generator=gen)
    prompts = [torch.cat([system, torch.randint(0, model.config.vocab_size, (n,), device="cuda", generator=gen)])
               for n in (30, 70, 50, 90, 20)]
    reqs = [(p, 6 + 3 * i) for i, p in enumerate(prompts)]
    stats = {}
    pc = PrefixCache(1 << 30) if prefix else None
    got = dict(serve(model, reqs, batch=2, max_tokens=head + 384, stats=stats, prefix_cache=pc))
    assert sorted(got) == list(range(len(reqs))) and stats["inserts"] == 3
    if prefix:                                  # the first insert stores the system prompt, the other two reuse it
        assert stats["prefix_hits"] == 2 and stats["prefix_tokens"] == 2 * head
    for i, (p, m) in enumerate(reqs):
        assert got[i].shape == (m,), i
        bar.argmax_agrees(f"{name} serve first token{' prefix' if prefix else ''}", got[i][:1],
                          ref64(input_ids=p[None]).logits[:, -1], hf16(input_ids=p[None]).logits[:, -1])


def _tp_worker(rank, ws, out_dir, path, name):
    import torch.distributed as dist
    torch.cuda.set_device(torch.device("cuda", rank))
    model = load_kivi(name, path, tensor_parallel=True)
    assert model.tp_world == ws and model.model.layers[0].self_attn.num_heads == 8 // ws
    ref64, hf16 = reference_models(name, path)
    local = Bar()
    dev = torch.device("cuda", rank)
    gen = torch.Generator(device=dev).manual_seed(1)
    B, n = 3, 150
    ids = torch.randint(0, model.config.vocab_size, (B, n), device=dev, generator=gen)
    model.init_cache(B, n + 40)
    last = model.prefill(ids)
    local.check(f"{name} tp{ws} prefill", last, ref64(input_ids=ids).logits[:, -1], hf16(input_ids=ids).logits[:, -1])
    tok = last.argmax(-1, keepdim=True)
    for _ in range(20):                         # the cache holds this rank's heads: it exports no whole-model 9-tuple
        logits = model.decode_step(tok)
        assert torch.isfinite(logits).all() and same_on_all_ranks(logits)
        tok = model.next_tokens.view(B, 1).clone()
    torch.cuda.synchronize()
    dist.barrier()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")
    dist.destroy_process_group()


@pytest.mark.parametrize("ws", [2])
def test_tensor_parallel_multi_gpu(tmp_path, ws):
    """The tensor-parallel loader at world 2 on the ratio-4 checkpoint: each rank holds 4 query heads' q rows, 1 KV head's
    k / v rows and the whole q_norm / k_norm; the prompt meets the bar on every rank, and every rank decodes the same
    logits."""
    if torch.cuda.device_count() < ws:
        pytest.skip(f"needs {ws} GPUs")
    name = "qwen3-ratio4"
    path = tmp_path / "ckpt"
    write_checkpoint(name, path)
    spawn_ranks(_tp_worker, ws, tmp_path, str(path), name)

"""Prefix reuse on the GPU: the suffix prompt-attention entry (kivi_prompt_attention_suffix_f16) against a float64 masked
softmax and bit for bit against the full entry's rows, the model's insert over a stored prefix against transformers,
the tensor-parallel model, serve() with and without a PrefixCache, and the memory the cache holds."""
import math
import os

import pytest
import torch

from kivi_b200.prefix import MIN_REUSE
from tests._hf import Bar, Decoder, checkpoints, load_kivi, reference_models  # noqa: F401
from tests._model import same_logits, same_on_all_ranks, sharded_model, small_cfg, spawn_ranks, world_one_pair
from tests.test_prompt_attn_gpu import _qkv, _sdpa16, _visible

pytestmark = pytest.mark.gpu

D = 128


# ------------------------------------------------------------------------------------------------ kernel
def _ref64_rows(q, k, v, keep, lo):
    """float64 reference of the query rows lo .. n-1 [B, n - lo, H, 128]; rows with no visible key are 0."""
    B, H, n, _ = q.shape
    G = H // k.shape[1]
    out = torch.zeros((B, n - lo, H, D), dtype=torch.float64, device=q.device)
    for b in range(B):
        for h in range(H):
            s = (q[b, h, lo:].double() @ k[b, h // G].double().T) / math.sqrt(D)
            s = s.masked_fill(~keep[b, lo:], float("-inf"))
            out[b, :, h] = torch.softmax(s, -1).nan_to_num(0.0) @ v[b, h // G].double()
    return out


def _suffix(q, k, v, m, starts, window):
    from kivi_b200 import glue
    B, H, n, _ = q.shape
    out = torch.empty((B, m, H, D), dtype=torch.float16, device="cuda")
    ks = torch.tensor(starts, dtype=torch.int32, device="cuda")
    return glue.prompt_attention_suffix(q[:, :, n - m:], k, v, out, ks, window)


def _full(q, k, v, starts, window):
    from kivi_b200 import glue
    B, H, n, _ = q.shape
    out = torch.empty((B, n, H, D), dtype=torch.float16, device="cuda")
    return glue.prompt_attention(q, k, v, out, torch.tensor(starts, dtype=torch.int32, device="cuda"), window)


def _check_suffix(q, k, v, m, starts, window, what, fp64=True):
    """The suffix entry's rows equal the full entry's rows n - m .. n - 1 bit for bit, and meet the float64 bar."""
    n = q.shape[2]
    ours = _suffix(q, k, v, m, starts, window)
    assert torch.equal(ours, _full(q, k, v, starts, window)[:, n - m:]), f"{what}: not the full entry's rows"
    if not fp64:
        return
    keep = _visible(n, starts, window)
    rows = keep[:, n - m:].any(-1)                                      # [B, m]
    assert torch.equal(ours[~rows], torch.zeros_like(ours[~rows])), f"{what}: rows with no visible key are not zero"
    if rows.any():
        ref = _ref64_rows(q, k, v, keep, n - m)
        sdpa = _sdpa16(q, k, v, keep)[:, n - m:]
        err = (ours[rows].double() - ref[rows]).abs().max().item()
        base = (sdpa[rows].double() - ref[rows]).abs().max().item()
        assert err <= 2 * base + 1e-3, f"{what}: max|ours - ref64| {err:.3g} > 2 * {base:.3g} + 1e-3"


def _suffix_lengths(n):
    """m in {1, 63, 64, 65, n - 1, n}, and the prefix n - m on and around tile edges (63, 64, 65, 127, 128, 129)."""
    ms = {1, 63, 64, 65, n - 1, n} | {n - r for r in (63, 64, 65, 127, 128, 129)}
    return sorted(m for m in ms if 1 <= m <= n)


@pytest.mark.parametrize("G", [1, 2, 4, 7, 8, 65])
@pytest.mark.parametrize("n", [1, 64, 130, 1000, 4097])
def test_suffix_matches_float64_and_the_full_entry(n, G):
    """Every suffix length of _suffix_lengths with every window of {0, 1, 64, n - m, n}; row 0 starts inside the prefix,
    row 1 inside the suffix.  Bit identity on every case; the float64 bar on every case up to n = 1000 and on a subset at
    4097 (m <= 65 or m >= n - 1)."""
    Hkv = 1 if G >= 7 else 2
    q, k, v = _qkv(2, G * Hkv, Hkv, n, seed=n * 100 + G)
    for m in _suffix_lengths(n):
        r = n - m
        starts = [r // 2, r + m // 2]
        for W in sorted({0, 1, 64, n - m, n}):
            fp64 = n <= 1000 or m <= 65 or m >= n - 1
            _check_suffix(q, k, v, m, starts, W, f"n {n} G {G} m {m} W {W} starts {starts}", fp64)


@pytest.mark.parametrize("case", ["peaked", "flat"])
def test_suffix_magnitudes(case):
    """Logits q.k / sqrt(128) of std ~30 (one key dominates) and ~1e-4 (uniform weights)."""
    kw = dict(peaked=dict(q_std=5.5, k_std=5.5), flat=dict(q_std=0.01, k_std=0.01))[case]
    q, k, v = _qkv(2, 8, 2, 1000, seed=7, **kw)
    for m, starts, W in ((300, [0, 0], 0), (300, [129, 800], 0), (65, [5, 950], 200), (999, [64, 500], 64)):
        _check_suffix(q, k, v, m, starts, W, f"{case} m {m} starts {starts} W {W}")


def test_suffix_skips_tiles_below_the_window_and_the_start():
    """K / V NaN in the 64-key tiles wholly below every suffix query's window and below the start: the same bits."""
    n, m, W = 2000, 300, 256
    q, k, v = _qkv(2, 8, 2, n, seed=3)
    starts = [0, 1800]
    clean = _suffix(q, k, v, m, starts, W)
    kn, vn = k.clone(), v.clone()
    first = n - m - W + 1                                                 # the lowest key any suffix query sees
    kn[0, :, : first // 64 * 64] = float("nan")
    vn[0, :, : first // 64 * 64] = float("nan")
    kn[1, :, :1792] = float("nan")
    vn[1, :, :1792] = float("nan")
    assert torch.equal(_suffix(q, kn, vn, m, starts, W), clean)


# ------------------------------------------------------------------------------------------------ model
bar = Bar()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    bar.report("prefix reuse against transformers")


def _prompts(vocab, gen, head, tails):
    system = torch.randint(0, vocab, (head,), device="cuda", generator=gen)
    return [torch.cat([system, torch.randint(0, vocab, (t,), device="cuda", generator=gen)]) for t in tails]


@pytest.mark.parametrize("name,chunked", [("llama3", False), ("mistral", False), ("llama3", True)])
def test_insert_over_a_stored_prefix_matches_transformers(checkpoints, monkeypatch, name, chunked):
    """Two requests share a system prompt of MIN_REUSE + 76 tokens.  The first insert stores it, the second reuses it
    and runs its last tokens only; its logits and the decode steps of both slots after it meet the transformers bar.
    mistral: a 160-token window that cuts the prompts.  chunked: PROMPT_CHUNK_ROWS lowered to 32, so the suffix runs
    in chunks."""
    from kivi_b200 import llama_kivi
    from kivi_b200.prefix import PrefixCache
    if chunked:
        monkeypatch.setattr(llama_kivi, "PROMPT_CHUNK_ROWS", 32)
    path = checkpoints(name, sliding_window=160) if name == "mistral" else checkpoints(name)
    ref64, hf16 = reference_models(name, path)
    model = load_kivi(name, path, residual_length=64)
    head = MIN_REUSE + 76
    B, T = 2, head + 120
    gen = torch.Generator(device="cuda").manual_seed(4)
    model.init_cache(B, T + 200)
    model.prefill(torch.randint(0, model.config.vocab_size, (B, T), device="cuda", generator=gen))
    pc = PrefixCache(1 << 30)
    a, b = _prompts(model.config.vocab_size, gen, head, [50, 97])
    for slot, p in ((0, a), (1, b)):
        got = model.insert(slot, p, pc)
        ids = p.view(1, -1)
        bar.check(f"{name} prefix insert {slot}", got[None], ref64(input_ids=ids).logits[:, -1],
                  hf16(input_ids=ids).logits[:, -1])
    assert pc.hits == 1 and pc.reused_tokens == head
    n = [a.numel(), b.numel()]
    dec = Decoder(bar, model, ref64, hf16, T=T, pos=n, start=[T - x for x in n],
                  gen=torch.Generator(device="cuda").manual_seed(5))
    dec.run(80, f"{name} prefix decode")


def test_prefix_insert_stores_what_one_pass_computes():
    """The slot after an insert over a stored prefix against the slot after the same prompt in one pass: the same refill
    of K / V that differ only through the GEMM row count -- the 9-tuples agree within fp16 rounding of the codes' inputs,
    and the logits at the prompt bar."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    from kivi_b200.prefix import PrefixCache
    from tests._model import TupleBar
    cfg = small_cfg()
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    head = MIN_REUSE + 66
    model.init_cache(2, head + 300)
    model.prefill(torch.randint(0, cfg.vocab_size, (2, head + 200), device="cuda"))
    gen = torch.Generator(device="cuda").manual_seed(1)
    a, b = _prompts(cfg.vocab_size, gen, head, [20, 70])
    pc = PrefixCache(1 << 30)
    model.insert(0, a, pc)
    got = model.insert(1, b, pc)
    assert pc.hits == 1 and pc.reused_tokens == head
    reused = [model.cache.export(i) for i in range(cfg.num_hidden_layers)]
    ref = model.insert(1, b)
    TupleBar("prefix insert").prompt(got[None], ref[None])
    for layer, tup in enumerate(reused):
        fresh = model.cache.export(layer)
        for x, y in zip(tup, fresh):
            if torch.is_tensor(x) and x.dtype == torch.float16:
                assert (x.float() - y.float()).abs().max().item() <= 2e-2 * y.float().abs().max().item() + 2e-2


def test_tensor_parallel_at_world_one_with_a_prefix_cache():
    """The plain model and the tensor-parallel model at world 1, each with its own PrefixCache used the same way: the
    inserts' logits and the decode steps after them equal bit for bit."""
    from kivi_b200.prefix import PrefixCache
    cfg = small_cfg()
    plain, tpm = world_one_pair(cfg)
    gen = torch.Generator(device="cuda").manual_seed(2)
    head = MIN_REUSE + 86
    prompts = _prompts(cfg.vocab_size, gen, head, [30, 70, 5])
    start = torch.randint(0, cfg.vocab_size, (3, head + 110), device="cuda", generator=gen)
    caches, logits = [], []
    for m in (plain, tpm):
        m.init_cache(3, head + 250)
        m.prefill(start)
        pc = PrefixCache(1 << 30)
        caches.append(pc)
        logits.append([m.insert(slot, p, pc).clone() for slot, p in enumerate(prompts)])
    assert caches[0].hits == caches[1].hits == 2
    for x, y in zip(*logits):
        assert torch.equal(x, y)
    ids = torch.stack([x.argmax() for x in logits[0]]).view(3, 1)
    same_logits(plain, tpm, 40, ids)


def _tp_prefix_worker(rank, ws, out_dir):
    import torch.distributed as dist
    from kivi_b200.prefix import PrefixCache
    from kivi_b200.serve import serve
    cfg = small_cfg()
    model, _ = sharded_model(cfg, rank, ws)
    dev = torch.device("cuda", rank)
    gen = torch.Generator().manual_seed(3)
    head = MIN_REUSE + 36
    system = [torch.randint(0, cfg.vocab_size, (head,), generator=gen) for _ in range(2)]
    reqs = [(torch.cat([system[i % 2], torch.randint(0, cfg.vocab_size, (10 + 7 * i,), generator=gen)]), 6 + i)
            for i in range(8)]
    pc = PrefixCache(1 << 30)
    stats = {}
    got = dict(serve(model, reqs, 2, head + 300, stats=stats, prefix_cache=pc))
    assert stats["prefix_hits"] > 0
    for i in range(len(reqs)):
        assert same_on_all_ranks(got[i].to(dev)), i
    assert same_on_all_ranks(torch.tensor([pc.hits, pc.reused_tokens, pc.stored_bytes, len(pc)], device=dev))
    torch.cuda.synchronize()
    dist.barrier()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")
    dist.destroy_process_group()


@pytest.mark.parametrize("ws", [2])
def test_tensor_parallel_prefix_multi_gpu(tmp_path, ws):
    """Each rank stores its own KV heads and decides matches and evictions from token ids alone: every rank returns the
    same tokens and holds a tree of the same shape."""
    if torch.cuda.device_count() < ws:
        pytest.skip(f"needs {ws} GPUs")
    spawn_ranks(_tp_prefix_worker, ws, tmp_path)


# ------------------------------------------------------------------------------------------------ serve()
MARGIN = 0.1        # top-2 log-probability margin below which a greedy token may flip between the two prompt passes
SYSTEM = MIN_REUSE + 86                             # the system prompts' length
SERVE_TOKENS = SYSTEM + 250                         # the serve() calls' max_tokens


def _serve_requests(cfg, seed, n_req=12):
    gen = torch.Generator().manual_seed(seed)
    system = [torch.randint(1, cfg.vocab_size, (SYSTEM,), generator=gen) for _ in range(3)]
    reqs = []
    for i in range(n_req):
        user = torch.randint(1, cfg.vocab_size, (int(torch.randint(10, 60, (1,), generator=gen)),), generator=gen)
        reqs.append((torch.cat([system[i % 3], user]), int(torch.randint(16, 40, (1,), generator=gen)), {"logprobs": 2}))
    return reqs


def _agree_until_close(plain, cached):
    """Each request's tokens agree up to its first step whose top-2 margin (without the cache) is under MARGIN.
    Returns the number of tokens compared and the total."""
    compared = total = 0
    for i, (ids, lp) in plain.items():
        ids2 = cached[i][0]
        margin = lp.top[:, 0] - lp.top[:, 1]
        close = torch.nonzero(margin < MARGIN).flatten().tolist()
        upto = close[0] if close else ids.numel()
        assert torch.equal(ids[:upto], ids2[:upto]), f"request {i}: tokens differ before step {upto}"
        if not close:
            assert torch.equal(ids, ids2), f"request {i}"
        compared += upto
        total += ids.numel()
    return compared, total


def test_serve_with_a_prefix_cache():
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    from kivi_b200.prefix import PrefixCache
    from kivi_b200.serve import serve
    cfg = small_cfg()
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    model.lm_head.weight.data.mul_(8)                   # default-init logits are flat: most top-2 margins would be tiny
    reqs = _serve_requests(cfg, seed=1)

    def run(pc):
        stats = {}
        out = {i: (ids, lp) for i, ids, lp in serve(model, reqs, 3, SERVE_TOKENS, stats=stats, prefix_cache=pc)}
        return out, stats
    plain, s0 = run(None)
    assert s0["prefix_hits"] == 0 and s0["prefix_tokens"] == 0
    pc = PrefixCache(1 << 30)
    cached, s1 = run(pc)
    # 9 inserts after the first group's prefill; the first insert of each of the 3 system prompts stores it
    assert s1["inserts"] == 9 and s1["prefix_hits"] == 6 and s1["prefix_tokens"] == 6 * SYSTEM
    assert pc.hits == 6 and pc.stored_bytes > 0
    compared, total = _agree_until_close(plain, cached)
    assert compared >= total // 3, f"only {compared} of {total} tokens had a clear margin"
    again, _ = run(PrefixCache(1 << 30))                                 # two runs with a cache: identical
    for i in cached:
        assert torch.equal(cached[i][0], again[i][0])
        assert torch.equal(cached[i][1].top, again[i][1].top) and torch.equal(cached[i][1].top_ids, again[i][1].top_ids)
    # the cache outlives the call: a second stream with the same system prompts hits on every insert
    reqs2 = [(torch.cat([r[0][:SYSTEM], torch.randint(1, cfg.vocab_size, (25,))]), 8 + 3 * (i % 4), r[2])
             for i, r in enumerate(reqs)]
    stats = {}
    out2 = {i: (ids, lp) for i, ids, lp in serve(model, reqs2, 3, SERVE_TOKENS, stats=stats, prefix_cache=pc)}
    assert stats["inserts"] > 0 and stats["prefix_hits"] == stats["inserts"]
    assert stats["prefix_tokens"] == SYSTEM * stats["inserts"]
    base = {i: (ids, lp) for i, ids, lp in serve(model, reqs2, 3, SERVE_TOKENS)}
    _agree_until_close(base, out2)


def test_prefix_memory_stays_within_max_bytes():
    """Inserts of prompts that share and diverge from a few heads, with a budget of ~3.5 prompts: after every insert the
    memory allocated above the model and its cache never exceeds max_bytes, and evictions happen."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    from kivi_b200.prefix import PrefixCache
    cfg = small_cfg()
    torch.manual_seed(0)
    model = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    head = MIN_REUSE + 176                                # cut by up to 111 tokens: still reused
    model.init_cache(2, 2 * head + 300)
    model.prefill(torch.randint(0, cfg.vocab_size, (2, 2 * head + 200), device="cuda"))
    gen = torch.Generator(device="cuda").manual_seed(6)
    heads = [torch.randint(0, cfg.vocab_size, (head,), device="cuda", generator=gen) for _ in range(3)]
    prompts = [torch.cat([heads[i % 3][: head - 37 * (i % 4)],
                          torch.randint(0, cfg.vocab_size, (40 + 13 * (i % 5),), device="cuda", generator=gen)])
               for i in range(24)]                      # made before the base, so that only the cache grows
    warm = torch.cat([heads[0], heads[1]])
    first_use = PrefixCache(1 << 30)                     # one-time allocations of both insert paths, outside the count
    model.insert(0, warm, first_use)
    model.insert(0, warm, first_use)
    del first_use
    pc = PrefixCache(cfg.num_hidden_layers * 2 * cfg.num_key_value_heads * 256 * int(3.5 * (head + 66)))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    for i, prompt in enumerate(prompts):
        model.insert(i % 2, prompt, pc)
        torch.cuda.synchronize()
        grown = torch.cuda.memory_allocated() - base
        assert pc.stored_bytes <= pc.max_bytes
        assert grown <= pc.max_bytes, f"insert {i}: {grown} bytes above the base, budget {pc.max_bytes}"
    assert pc.evictions > 0 and pc.hits > 0

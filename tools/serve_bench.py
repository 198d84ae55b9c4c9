"""A stream of requests on one H100: static batching through generate() against continuous batching through serve().

    python tools/serve_bench.py [--requests 128] [--batch 32] [--max-tokens 4096] [--model llama-2-7b]

Workload: the Llama-2-7B shape (random-init fp16 weights), K2V2 g32 R128, `batch` slots, a cache of `max-tokens`
positions.  Prompt lengths are uniform in [--prompt-min, --prompt-max] and requested output lengths in [--out-min,
--out-max] (seeded), prompt ids random.  Greedy decoding without EOS, so every request produces exactly its budget.
  static: groups of `batch` requests in arrival order, each left-padded and run through generate() to its longest output
  serve : kivi_b200.serve.serve() with the same requests
Prints one JSON line per mode and one with the kernel times:
  useful_tokens_per_s  requested tokens only, over the makespan (host clock around the whole mode, ending in a synchronise)
  occupancy            requested tokens / (batch x decode steps): the share of the step rows that did useful work
  insert_ms            serve: total time of the B = 1 prompt passes of inserted requests (CUDA events)
  refill_ms_per_layer  one kivi_cache_refill_f16 call (CUDA events, median) for a --refill-len prompt at the final length
  shift_ms_per_layer   one kivi_cache_shift_f16 call of one 128-token block (CUDA events, median) at --shift-len positions
and the device name and power limit read in the same run.  Nothing is written to the repository.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except Exception:                                          # the number is still reported, without its power limit
        return "unknown"


def refill_bytes(cache, n):
    """Algorithmic HBM bytes of one refill call: the prompt's K and V read, the slot's packed blocks and windows written."""
    per_tok = 128 * (cache.k_bits / 8 + 4 / cache.group_size), 128 * (cache.v_bits / 8 + 4 / cache.group_size)
    return cache.num_kv_heads * (2 * n * 256 + cache.tk * per_tok[0] + cache.tv * per_tok[1] + (cache.r + cache.L) * 256)


def shift_bytes(cache, tokens):
    """Algorithmic HBM bytes of one shift call (one layer): every kept block of both stores read and written once."""
    U, d = cache.batch * cache.num_kv_heads, tokens // 128
    kb = 4096 * cache.k_bits // 2 + 8 * (128 // cache.group_size) * 64
    vb = 4096 * cache.v_bits // 2 + 8 * (128 // cache.group_size) * 64
    nk, nv = -(-cache.tk // 128), -(-cache.tv // 128)
    return 2 * U * ((nk - d) * kb + (nv - d) * vb)


def make_requests(args, vocab):
    g = torch.Generator().manual_seed(args.seed)
    lens = torch.randint(args.prompt_min, args.prompt_max + 1, (args.requests,), generator=g)
    outs = torch.randint(args.out_min, args.out_max + 1, (args.requests,), generator=g)
    return [(torch.randint(1, vocab, (int(n),), generator=g), int(m)) for n, m in zip(lens, outs)]


def run_static(model, reqs, B):
    steps = 0
    for i in range(0, len(reqs), B):
        group = reqs[i:i + B]
        P = max(p.numel() for p, _ in group)
        ids = torch.zeros((B, P), dtype=torch.long)
        mask = torch.zeros((B, P), dtype=torch.long)
        mask[:, -1] = 1                                        # rows without a request (last group): one token
        for b, (p, _) in enumerate(group):
            ids[b, P - p.numel():] = p
            mask[b, P - p.numel():] = 1
        m = max(n for _, n in group)
        model.generate(ids.cuda(), max_new_tokens=m, attention_mask=mask.cuda())
        steps += m - 1
    return steps


def median_event_ms(fn, reps):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-2-7b")
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--max-tokens", type=int, default=4096)
    ap.add_argument("--prompt-min", type=int, default=512)
    ap.add_argument("--prompt-max", type=int, default=2048)
    ap.add_argument("--out-min", type=int, default=64)
    ap.add_argument("--out-max", type=int, default=1024)
    ap.add_argument("--refill-len", type=int, default=1024)
    ap.add_argument("--shift-len", type=int, default=3072)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--modes", default="static,serve")
    args = ap.parse_args()
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    from kivi_b200.serve import serve

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, T_max = args.batch, args.max_tokens
    cfg = default_config(args.model)
    torch.manual_seed(0)
    with torch.device(dev):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p_ in model.parameters():
        p_.requires_grad_(False)
    model.eval()
    reqs = make_requests(args, cfg.vocab_size)
    useful = sum(m for _, m in reqs)
    model.init_cache(B, T_max)
    warm = torch.randint(1, cfg.vocab_size, (B, 64), device=dev)      # cuBLAS algorithms, the padded step graph
    wmask = torch.ones_like(warm)
    wmask[0, :3] = 0
    model.generate(warm, max_new_tokens=8, attention_mask=wmask)
    torch.cuda.synchronize()
    common = {"workload": f"{args.model} K{cfg.k_bits}V{cfg.v_bits} g{cfg.group_size} R{cfg.residual_length}, {B} slots, "
                          f"max_tokens {T_max}, {len(reqs)} requests, prompts [{args.prompt_min}, {args.prompt_max}], "
                          f"outputs [{args.out_min}, {args.out_max}]",
              "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "useful_tokens": useful}
    for mode in args.modes.split(","):
        if mode == "static":
            t0 = time.perf_counter()
            steps = run_static(model, reqs, B)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            print(json.dumps(dict(common, mode="static", useful_tokens_per_s=useful / dt, makespan_s=dt, decode_steps=steps,
                                  occupancy=(useful - len(reqs)) / (B * steps))), flush=True)
        elif mode == "serve":
            events = []
            orig = model.insert

            def timed_insert(seq, ids):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = orig(seq, ids)
                e1.record()
                events.append((e0, e1))
                return out
            model.insert = timed_insert
            stats = {}
            t0 = time.perf_counter()
            got = 0
            for _, toks in serve(model, reqs, B, T_max, stats=stats):
                got += toks.numel()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            del model.insert
            assert got == useful, (got, useful)
            insert_ms = sum(a.elapsed_time(b) for a, b in events)
            print(json.dumps(dict(common, mode="serve", useful_tokens_per_s=useful / dt, makespan_s=dt,
                                  decode_steps=stats["steps"], occupancy=stats["slot_steps"] / (B * stats["steps"]),
                                  insert_ms=insert_ms, inserts=stats["inserts"], prefills=stats["prefills"],
                                  shifts=stats["shifts"], shifted_tokens=stats["shifted_tokens"])), flush=True)
    # kernel times at a fixed length: refill of one slot, shift of one block (layer 0; all slots idle for the shift)
    cache = model.cache
    model.prefill_synthetic(args.shift_len, seed=1)
    n = min(args.refill_len, cache.kv_len)
    k = torch.randn((cache.num_kv_heads, n, 128), device=dev, dtype=torch.float16)
    v = torch.randn_like(k)
    cache.refill(0, 1, k, v)
    refill_ms = median_event_ms(lambda: cache.refill(0, 1, k, v), 10)
    rb = refill_bytes(cache, n)
    cache.set_kv_start(torch.full((B,), 1 << 30, dtype=torch.int32))
    sb = shift_bytes(cache, 128)
    shift_ms = median_event_ms(lambda: cache.shift(128), 5) / cache.n_layers   # all layers + the state update
    print(json.dumps(dict(common, mode="kernels", refill_len=n, refill_at_len=args.shift_len, refill_ms_per_layer=refill_ms,
                          refill_bytes=rb, refill_GBps=rb / refill_ms / 1e6, shift_tokens=128,
                          shift_at_len=f"{args.shift_len} down to {args.shift_len - 4 * 128}",
                          shift_ms_per_layer=shift_ms, shift_bytes_first=sb, shift_GBps_first=sb / shift_ms / 1e6)))
    return 0


if __name__ == "__main__":
    sys.exit(main())

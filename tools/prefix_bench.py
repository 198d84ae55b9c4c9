"""Prefix reuse measurements on one GPU: one JSON line per measurement, the card's name and power limit in every line.

    python tools/prefix_bench.py [--models llama-2-7b,llama-3-8b] [--parts a,b,c]

Models: the Llama-2-7B and Llama-3-8B shapes, random-init fp16 weights, K2V2 g32 R128.
  (a) a serve() stream: 128 requests on 32 slots, max_tokens 4096.  Each prompt is one of 4 system prompts of 1024 tokens
      plus a user part of uniform length in [64, 512]; outputs uniform in [64, 512], greedy, no EOS (seeded).  The same
      stream without and with a PrefixCache of --prefix-gb GiB (a fresh one per run), alternated in this process.
      Reports useful tokens/s (requested tokens over the makespan, host clock ending in a synchronise), the total insert
      time (CUDA events around every insert), the reused share of the inserted prompts' tokens and the peak bytes held.
  (b) one insert: its time (CUDA events, median of --reps) at n = 2048, 4096 and 8192: without a cache (SDPA over the
      whole prompt), as a miss that stores the whole prompt, and as a hit on r stored tokens for r from 64 (one key
      tile, below the shipped MIN_REUSE) to n - 64.
  (c) the kernel alone: kivi_prompt_attention_suffix_f16 at (n 4096, m 512) and (n 8192, m 1024), B = 1, against
      kivi_prompt_attention_f16 over all n queries (CUDA events, median of 50 calls).
Nothing is written to the repository.
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


def card():
    dev = torch.cuda.current_device()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                          # the number is still reported, without its power limit
        out = ""
    return {"gpu": torch.cuda.get_device_name(dev), "power_limit": out or "unknown"}


def emit(**kw):
    print(json.dumps(kw), flush=True)


def cuda_ms(fn, reps):
    """Median time of fn() over `reps` calls, CUDA events around each, after one warm-up call."""
    fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def make_model(name):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config(name)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p in model.parameters():
        p.requires_grad_(False)
    return model.eval(), cfg


def stream(cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    system = [torch.randint(1, cfg.vocab_size, (1024,), generator=g) for _ in range(4)]
    reqs = []
    for i in range(128):
        user = torch.randint(1, cfg.vocab_size, (int(torch.randint(64, 513, (1,), generator=g)),), generator=g)
        reqs.append((torch.cat([system[int(torch.randint(0, 4, (1,), generator=g))], user]),
                     int(torch.randint(64, 513, (1,), generator=g))))
    return reqs


def part_a(model, cfg, name, info, args):
    from kivi_b200.prefix import PrefixCache
    from kivi_b200.serve import serve
    reqs = stream(cfg)
    useful = sum(m for _, m in reqs)
    B, T = 32, 4096
    model.init_cache(B, T)
    warm = torch.randint(1, cfg.vocab_size, (B, 64), device="cuda")
    wmask = torch.ones_like(warm)
    wmask[0, :3] = 0
    model.generate(warm, max_new_tokens=8, attention_mask=wmask)
    orig = model.insert
    for rnd in range(args.rounds):
        for on in (False, True):
            events, inserted = [], [0]

            def timed(seq, ids, prefix_cache=None):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = orig(seq, ids, prefix_cache)
                e1.record()
                events.append((e0, e1))
                inserted[0] += ids.numel()
                return out
            model.insert = timed
            pc = PrefixCache(int(args.prefix_gb * 2 ** 30)) if on else None
            stats = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = sum(toks.numel() for _, toks in serve(model, reqs, B, T, stats=stats, prefix_cache=pc))
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            del model.insert
            assert got == useful, (got, useful)
            emit(part="a", model=name, round=rnd, prefix_cache=on, useful_tokens_per_s=useful / dt, makespan_s=dt,
                 insert_ms=sum(a.elapsed_time(b) for a, b in events), inserts=stats["inserts"],
                 prefix_hits=stats["prefix_hits"], reused_share=stats["prefix_tokens"] / max(inserted[0], 1),
                 peak_prefix_bytes=pc.peak_bytes if on else 0, evictions=pc.evictions if on else 0,
                 decode_steps=stats["steps"], **info)
            del pc
            torch.cuda.empty_cache()


def part_b(model, cfg, name, info, args):
    """Every insert of one prompt of n tokens: without a cache, as a miss (an empty cache: the whole prompt is computed
    and stored) and as a hit on r stored tokens.  MIN_REUSE is lowered to one key tile here so that reuse below the
    shipped threshold is timed too: those rows are what place it."""
    from kivi_b200 import prefix
    from kivi_b200.prefix import PrefixCache
    shipped, prefix.MIN_REUSE = prefix.MIN_REUSE, 64
    model.init_cache(1, 8192 + 64)
    model.prefill_synthetic(8192 + 64)
    try:
        for n in (2048, 4096, 8192):
            ids = torch.randint(1, cfg.vocab_size, (n,), device="cuda",
                                generator=torch.Generator(device="cuda").manual_seed(n))
            rs = sorted({r for r in (64, 256, 512, 1024, 1536, 2048, 3072, n // 2, n - 64) if r < n})
            for kind, r in [("none", 0), ("miss", 0)] + [("hit", r) for r in rs]:
                times = []
                for _ in range(args.reps + 1):
                    pc = None if kind == "none" else PrefixCache(1 << 40)
                    if r:
                        model.insert(0, ids[:r], pc)                    # stores the first r tokens
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    model.insert(0, ids, pc)
                    e1.record()
                    e1.synchronize()
                    times.append(e0.elapsed_time(e1))
                    if pc is not None:
                        assert pc.hits == (1 if r else 0) and pc.reused_tokens == r
                    del pc
                emit(part="b", model=name, n=n, cache=kind, r=r, insert_ms=statistics.median(times[1:]),
                     spread_ms=max(times[1:]) - min(times[1:]), shipped_min_reuse=shipped, **info)
            torch.cuda.empty_cache()
    finally:
        prefix.MIN_REUSE = shipped


def part_c(cfg, name, info):
    from kivi_b200 import glue
    H, Hkv = cfg.num_attention_heads, cfg.num_key_value_heads
    for n, m in ((4096, 512), (8192, 1024)):
        g = torch.Generator(device="cuda").manual_seed(n)
        q = torch.randn((1, n, H, 128), device="cuda", generator=g).half().transpose(1, 2)
        k = torch.randn((1, n, Hkv, 128), device="cuda", generator=g).half().transpose(1, 2)
        v = torch.randn((1, n, Hkv, 128), device="cuda", generator=g).half().transpose(1, 2)
        full_out = torch.empty((1, n, H, 128), dtype=torch.float16, device="cuda")
        suf_out = torch.empty((1, m, H, 128), dtype=torch.float16, device="cuda")
        suf = cuda_ms(lambda: glue.prompt_attention_suffix(q[:, :, n - m:], k, v, suf_out), 50)
        full = cuda_ms(lambda: glue.prompt_attention(q, k, v, full_out), 50)
        assert torch.equal(suf_out, full_out[:, n - m:])
        emit(part="c", model=name, n=n, m=m, suffix_us=suf * 1e3, full_us=full * 1e3, ratio=suf / full, **info)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama-2-7b,llama-3-8b")
    ap.add_argument("--parts", default="a,b,c")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--prefix-gb", type=float, default=8.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prefix_bench needs a CUDA device")
    info = card()
    parts = args.parts.split(",")
    for name in args.models.split(","):
        from kivi_b200.llama_kivi import default_config
        if "c" in parts:
            part_c(default_config(name), name, info)
        if "a" in parts or "b" in parts:
            model, cfg = make_model(name)
            with torch.no_grad():
                if "b" in parts:
                    part_b(model, cfg, name, info, args)
                if "a" in parts:
                    part_a(model, cfg, name, info, args)
            del model
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

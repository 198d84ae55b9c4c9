"""Decode of a LEFT-padded batch on one H100: tokens/s and the attention of one layer (CUDA events).

    python tools/padded_bench.py [--spread 0.5] [--batch 32] [--seq 4096] [--steps 32] [--warmup 4]

The workload of bench.py's headline (Llama-2-7B, K2V2 g32 R128, random-init fp16 weights, the cache pre-filled with
synthetic K/V by the prefill pack kernels so that the timed steps end at kv length `seq`), but each sequence's prompt
length is drawn uniformly from [(1 - spread) * seq, seq] (seeded) and the batch is left-padded to `seq`
(KiviCache.set_kv_start): every decode step runs kivi_decode_attention_ragged_f16.  Prints one JSON line with
  value             tokens/s of the padded batch (whole decode step, CUDA graph)
  ragged_ms         one layer's attention call through the left-padded entry
  mask_ms           the same batch through kivi_decode_attention_f16 with the equivalent additive finfo.min mask
  unpadded_ms       the unpadded batch (no offsets, no mask) at the same lengths
  live_bytes        HBM bytes of the call counting only each sequence's visible tokens; padded_bytes: all tokens
Nothing is written to the repository.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def attention_bytes(cache, H, starts=None):
    """HBM bytes one attention call of one layer reads and writes: packed K / V codes + scales / mins, the fp16 windows,
    q / out / k_new / v_new.  With starts, only each sequence's visible tokens (positions >= its start) count."""
    B, Hkv = cache.batch, cache.num_kv_heads
    tok_k = 128 * (cache.k_bits / 8 + 4 / cache.group_size)
    tok_v = 128 * (cache.v_bits / 8 + 4 / cache.group_size)
    total = (2 * B * H + 2 * B * Hkv) * 256
    for s in (starts if starts is not None else [0] * B):
        s = min(max(int(s), 0), cache.kv_len)
        kw = cache.r - min(max(s - cache.tk, 0), cache.r)
        vw = cache.L - min(max(s - cache.tv, 0), cache.L)
        total += Hkv * (max(cache.tk - s, 0) * tok_k + max(cache.tv - s, 0) * tok_v + (kw + vw) * 256)
    return total


def attention_times(model, cache, starts, rounds=5, calls=8):
    """Layer 0, three variants timed in alternating rounds (one layer's cache >> L2: every call streams from HBM);
    median over the rounds of the mean of `calls` back-to-back calls."""
    cfg = model.config
    dev = cache.device
    B, H, Hkv = cache.batch, cfg.num_attention_heads, cfg.num_key_value_heads
    q = torch.randn((B, H, 128), device=dev, dtype=torch.float16)
    kn = torch.randn((B, Hkv, 128), device=dev, dtype=torch.float16)
    vn = torch.randn_like(kn)
    out = torch.empty_like(q)
    while cache.r == cache.residual_length - 1:          # stay off the K-flush step (once per R steps)
        model.decode_step()
    T = cache.kv_len + 1
    mask = torch.zeros((B, T), dtype=torch.float16, device=dev)
    for b, s in enumerate(starts.tolist()):
        mask[b, :min(s, T - 1)] = torch.finfo(torch.float16).min
    variants = {"ragged": (starts, None), "mask": (None, mask), "unpadded": (None, None)}
    times = {k: [] for k in variants}
    for rnd in range(rounds + 1):                        # round 0 settles clocks and caches, not counted
        for name, (st, m) in variants.items():
            cache.set_kv_start(st)
            cache.decode_attention(0, q, kn, vn, mask=m, out=out)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls):
                cache.decode_attention(0, q, kn, vn, mask=m, out=out)
            e1.record()
            torch.cuda.synchronize()
            if rnd > 0:
                times[name].append(e0.elapsed_time(e1) / calls)
    cache.set_kv_start(starts)
    return {k: statistics.median(v) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spread", type=float, default=0.5, help="prompt lengths uniform in [(1-spread)*seq, seq]")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    if not 0.0 <= args.spread < 1.0:
        ap.error("--spread must be in [0, 1)")
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, seq, K, W = args.batch, args.seq, args.steps, max(args.warmup, 3)
    cfg = default_config("llama-2-7b")
    cfg.max_position_embeddings = max(cfg.max_position_embeddings, seq + 64)
    torch.manual_seed(0)
    with torch.device(dev):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p_ in model.parameters():
        p_.requires_grad_(False)
    model.eval()
    n0 = seq - (W + K)                                   # the K timed steps end at kv length `seq`
    model.init_cache(B, max_tokens=seq + cfg.residual_length + 16)
    model.prefill_synthetic(n0, seed=0)
    cache = model.cache
    gen = torch.Generator().manual_seed(args.seed)
    lens = torch.randint(int((1.0 - args.spread) * seq), seq + 1, (B,), generator=gen)
    starts = (seq - lens).to(torch.int32)
    cache.set_kv_start(starts)
    model._pos.copy_((n0 - starts.long()).clamp(min=0).view(B, 1))
    model.decode_step(torch.randint(0, cfg.vocab_size, (B, 1), device=dev))   # captures the step graph
    for _ in range(W - 1):
        model.decode_step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        model.decode_step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    t = attention_times(model, cache, starts)
    live, padded = attention_bytes(cache, cfg.num_attention_heads, starts.tolist()), attention_bytes(cache, cfg.num_attention_heads)
    line = {"workload": f"Llama-2-7B K2V2 g32 R128 bs{B}, left-padded to seq {seq}, spread {args.spread}",
            "gpu": torch.cuda.get_device_name(dev), "value": B * K / (ms / 1e3), "unit": "tokens/s", "ms_per_step": ms / K,
            "prompt_len": {"min": int(lens.min()), "max": int(lens.max()), "mean": float(lens.float().mean())},
            "ragged_ms": t["ragged"], "mask_ms": t["mask"], "unpadded_ms": t["unpadded"],
            "ragged_over_mask": t["ragged"] / t["mask"], "ragged_over_unpadded": t["ragged"] / t["unpadded"],
            "live_bytes": live, "padded_bytes": padded, "live_share": live / padded,
            "state": [cache.tk, cache.r, cache.tv, cache.L]}
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())

"""Sliding-window decode on one H100: the windowed attention against whole-cache attention, Mistral-7B shape.

    python tools/window_bench.py [--batch 16] [--seqs 8192,32768] [--window 4096] [--rounds 5] [--steps 16] [--out DIR]

Mistral-7B (32 layers, 32 query / 8 KV heads, random-init fp16 weights), K4V4 g64 R64, B = 16, the cache pre-filled with
synthetic K/V by the prefill pack kernels to each length T.  For every T the two arms -- W = --window
(kivi_decode_attention_window_f16) and no window (kivi_decode_attention_f16) -- are warmed up, then timed in alternating
rounds in this one process, so the spread between rounds shows next to the difference between the arms:
  attn_ms          one layer's attention call, CUDA-graph timed (a graph of --calls back-to-back calls of layer 0)
  step_ms          the whole decode step (the model's captured step graph), --steps steps per round
  bytes            the algorithmic HBM bytes of one attention call (attention_bytes below); GB/s = bytes / attn_ms
  rounds           every round's value, so the run-to-run spread is visible
Then, for a rolling generate() (W = --window, prompt --prompt tokens, --new generated tokens):
  cache_bytes      of the rolling cache (max(prompt, W) + 2 max(128, R) positions) against a full-size one (prompt + new)
  shift_ms         one KiviCache.shift of the rolling cache at capacity, and per_step_ms = shift_ms / positions shifted,
                   the amortised cost per decode step.
The card's name and power limit are read in the same run and printed with the numbers (one JSON line on stdout; with
--out, also written there).  Nothing is written to the repository.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def block_bytes(bits, g):
    """One packed 128 x 128 block: codes + scales / zeros (kivi_decode.cuh lay_block_bytes)."""
    return (4096 if bits == 2 else 8192) + 8 * (128 // g) * 64


def attention_bytes(cache, H, window=None):
    """HBM bytes one attention call of one layer moves, from the cache's lengths: per unit (sequence x KV head) the packed K
    / V blocks the call reads (from block j0 = min(n_blocks, max(0, T - W) // 128) with a window), the fp16 K / V windows,
    the logits row (written by q.K^T, read by p.V for the packed V blocks), and q / out / k_new / v_new."""
    B, Hkv = cache.batch, cache.num_kv_heads
    T = cache.kv_len + 1
    n_kb, n_vb = -(-cache.tk // 128), -(-cache.tv // 128)
    j0k = j0v = 0
    if window is not None:
        j0k, j0v = min(n_kb, max(0, T - window) // 128), min(n_vb, max(0, T - window) // 128)
    g, rep = cache.group_size, H // Hkv
    per_unit = ((n_kb - j0k) * block_bytes(cache.k_bits, g) + (n_vb - j0v) * block_bytes(cache.v_bits, g)
                + (cache.r + cache.L) * 256
                + rep * 2 * ((n_kb - j0k) * 128 + cache.r + 1)           # logits written
                + rep * 2 * ((n_vb - j0v) * 128 + cache.L + 1))          # logits read
    return B * Hkv * per_unit + (2 * B * H + 2 * B * Hkv) * 256


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unavailable ({e})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def graph_of(fn, calls):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    return g


def timed(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def one_length(model, T, window, args):
    cfg, cache = model.config, None
    B = args.batch
    steps_total = (args.rounds + 1) * 2 * args.steps + 8
    model.init_cache(B, T + steps_total + 8)
    cache = model.cache
    model.prefill_synthetic(T - 1, seed=0)
    dev = cache.device
    H, Hkv = cfg.num_attention_heads, cfg.num_key_value_heads
    q = torch.randn((B, H, 128), device=dev, dtype=torch.float16)
    kn = torch.randn((B, Hkv, 128), device=dev, dtype=torch.float16)
    vn = torch.randn_like(kn)
    out = torch.empty_like(q)
    arms = {"window": window, "full": None}
    attn_graphs, step_graphs = {}, {}
    for name, w in arms.items():                          # warm up and capture every shape before any timing
        cache.sliding_window = w
        attn_graphs[name] = graph_of(lambda: cache.decode_attention(0, q, kn, vn, out=out), args.calls)
        model._graph = None
        model.decode_step(torch.zeros((B, 1), dtype=torch.long, device=dev))
        step_graphs[name] = model._graph
    bytes_ = {name: attention_bytes(cache, H, w) for name, w in arms.items()}
    res = {name: {"attn_ms": [], "step_ms": []} for name in arms}
    for rnd in range(args.rounds + 1):                    # round 0 settles clocks, not counted
        for name, w in arms.items():
            cache.sliding_window = w
            model._graph, model._graph_ragged = step_graphs[name], cache.ragged
            a = timed(attn_graphs[name].replay, 2) / (2 * args.calls)
            s = timed(model.decode_step, args.steps) / args.steps
            if rnd:
                res[name]["attn_ms"].append(a)
                res[name]["step_ms"].append(s)
    out_ = {"T": T}
    for name in arms:
        a, s = statistics.median(res[name]["attn_ms"]), statistics.median(res[name]["step_ms"])
        out_[name] = {"attn_ms": round(a, 4), "step_ms": round(s, 3), "bytes": bytes_[name],
                      "GBps": round(bytes_[name] / a / 1e6, 1),
                      "rounds": {k: [round(x, 4) for x in v] for k, v in res[name].items()}}
    out_["attn_speedup"] = round(out_["full"]["attn_ms"] / out_["window"]["attn_ms"], 3)
    out_["bytes_ratio"] = round(bytes_["window"] / bytes_["full"], 4)
    model.cache, model._graph = None, None
    del cache, attn_graphs, step_graphs
    torch.cuda.empty_cache()
    return out_


def rolling(model, window, args):
    """Cache bytes of a rolling generate() against a full-size cache, and the amortised cost of its shifts."""
    from kivi_b200.cache import KiviCache
    cfg = model.config
    B, R = args.batch, cfg.residual_length
    q = max(128, R)
    cap = max(args.prompt, window) + 2 * q
    sizes = {}
    for name, tokens in (("rolling", cap), ("full", args.prompt + args.new)):
        c = KiviCache(cfg.num_hidden_layers, B, cfg.num_attention_heads, cfg.num_key_value_heads, 128, cfg.k_bits,
                      cfg.v_bits, cfg.group_size, R, tokens, sliding_window=window)
        sizes[name] = c.nbytes() + c._ws.numel()
        del c
        torch.cuda.empty_cache()
    model.init_cache(B, cap)
    model.cache.sliding_window = window                  # (the model's config has no window: the cache gets it here)
    shifts = []
    for _ in range(args.rounds + 1):
        model.prefill_synthetic(cap, seed=1)
        c = model.cache
        tokens = min([c.tk, c.tv] + list(c.live_starts().values())) // q * q
        ms = timed(lambda: c.shift(tokens))
        shifts.append((ms, tokens))
    shifts = shifts[1:]
    ms = statistics.median(m for m, _ in shifts)
    tokens = shifts[0][1]
    model.cache, model._graph = None, None
    torch.cuda.empty_cache()
    return {"cap_tokens": cap, "cache_bytes": sizes, "shift_tokens": tokens, "shift_ms": round(ms, 3),
            "shift_ms_per_step": round(ms / tokens, 5), "shift_rounds": [round(m, 3) for m, _ in shifts]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seqs", default="8192,32768")
    ap.add_argument("--window", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--calls", type=int, default=8)
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--new", type=int, default=32768)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--out", default=None, help="directory that receives window_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("window_bench.py measures on a CUDA device; none is visible")
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    seqs = [int(x) for x in args.seqs.split(",")]
    cfg = default_config("mistral-7b", k_bits=4, v_bits=4, group_size=64, residual_length=64,
                         num_hidden_layers=args.layers)
    cfg.max_position_embeddings = max(seqs) + 4096
    torch.manual_seed(0)
    with torch.device(dev):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p_ in model.parameters():
        p_.requires_grad_(False)
    model.eval()
    result = {"workload": f"mistral-7b shape, K4V4 g64 R64, B={args.batch}, W={args.window}, layers={args.layers}",
              "card": card(), "lengths": [one_length(model, T, args.window, args) for T in seqs],
              "rolling": rolling(model, args.window, args)}
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "window_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

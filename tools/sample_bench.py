"""Sampling measurements: one JSON line per measurement, the card's name and power limit in every line.

    python tools/sample_bench.py [--only kernel|step] [--rounds R] [--steps K] [--warmup W]

kernel  kivi_sample_f32 alone next to kivi_greedy_sample_exchange_f32 (one GPU, no exchange): 100 calls captured in one
        CUDA graph, the graph replayed between CUDA events, microseconds per call, at (B, vocab) = (32, 32000), (64, 128256),
        (1, 128256) for temperature only / top-k 50 / top-p 0.9 / both.  Logits are N(0, 3^2), one seed per row.
step    Llama-2-7B, batch 32, K2V2 g32 R128, cache filled by prefill_synthetic to about 4096 tokens: milliseconds per
        graph-replayed decode step with the greedy kernel and with the sampling kernel (top-k 50, top-p 0.9, temperature
        0.8) as the step's last launch, alternated R times in one process (the order swaps every round; the cache grows by
        one token per step, so a round's two numbers are taken a few dozen tokens apart).
Needs a GPU: there is no CPU path.  Nothing is written outside the system's temporary directory.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SHAPES = [(32, 32000), (64, 128256), (1, 128256)]
MODES = [("temperature", 0, 1.0), ("top_k 50", 50, 1.0), ("top_p 0.9", 0, 0.9), ("top_k 50 + top_p 0.9", 50, 0.9)]


def card():
    import torch
    idx = torch.cuda.current_device()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(idx)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return {"gpu": torch.cuda.get_device_name(idx), "power_limit_w": power}


def _graph_us_per_call(fn, calls=100, replays=20):
    """fn enqueues one call; `calls` of them in one graph, microseconds per call over `replays` replays (best and median)."""
    import torch
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
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(replays):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / calls)
    times.sort()
    return {"us_per_call_min": round(times[0], 2), "us_per_call_median": round(times[len(times) // 2], 2)}


def bench_kernel(info):
    import torch
    from kivi_b200 import glue
    for B, V in SHAPES:
        gen = torch.Generator(device="cuda").manual_seed(B + V)
        logits = torch.randn((B, V), generator=gen, device="cuda") * 3.0
        nxt, fb = torch.zeros(B, dtype=torch.long, device="cuda"), torch.zeros(B, dtype=torch.long, device="cuda")
        r = _graph_us_per_call(lambda: glue.greedy_sample(logits, nxt, fb))
        print(json.dumps({"measurement": "kernel", "kernel": "kivi_greedy_sample_exchange_f32", "batch": B, "vocab": V,
                          **r, **info}), flush=True)
        seed, draw = torch.arange(B, device="cuda"), torch.zeros(B, dtype=torch.long, device="cuda")
        for name, k, p in MODES:
            t = torch.full((B,), 0.8, device="cuda")
            tk = torch.full((B,), k, dtype=torch.int32, device="cuda")
            tp = torch.full((B,), p, device="cuda")
            r = _graph_us_per_call(lambda: glue.sample(logits, t, tk, tp, seed, draw, nxt, fb))
            print(json.dumps({"measurement": "kernel", "kernel": "kivi_sample_f32", "mode": name, "batch": B, "vocab": V,
                              **r, **info}), flush=True)


def bench_step(info, rounds, K, W):
    import torch
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    B, seq = 32, 4096
    cfg = default_config("llama-2-7b")
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p in model.parameters():
        p.requires_grad_(False)
    model.eval()
    per_phase = W + K + 1                                                 # + the warm-up step of a capture
    total = 2 * rounds * per_phase
    model.init_cache(B, seq + total // 2 + 16)
    model.prefill_synthetic(seq - total // 2, seed=0)
    model._ids.copy_(torch.randint(0, cfg.vocab_size, (B, 1), device="cuda"))

    def phase(sampled):
        if sampled:
            model.set_sampling(temperature=0.8, top_k=50, top_p=0.9, seed=1)
        else:
            model.set_sampling(None)
        for _ in range(W):
            model.decode_step()
        torch.cuda.synchronize()
        start = model.cache.kv_len
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(K):
            model.decode_step()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / K, start

    res = {"greedy": [], "sampled": []}
    for r in range(rounds):
        for sampled in ((False, True) if r % 2 == 0 else (True, False)):
            ms, start = phase(sampled)
            res["sampled" if sampled else "greedy"].append(ms)
            print(json.dumps({"measurement": "step", "model": "llama-2-7b", "batch": B, "kv_len_start": start, "steps": K,
                              "round": r, "last_kernel": "kivi_sample_f32" if sampled else "kivi_greedy_sample_exchange_f32",
                              "ms_per_step": round(ms, 4), "launches_per_step": model.launches_per_step, **info}), flush=True)
    mean = {k: sum(v) / len(v) for k, v in res.items()}
    print(json.dumps({"measurement": "step summary", "model": "llama-2-7b", "batch": B, "seq": seq, "rounds": rounds,
                      "greedy_ms_per_step": round(mean["greedy"], 4), "sampled_ms_per_step": round(mean["sampled"], 4),
                      "greedy_spread_ms": round(max(res["greedy"]) - min(res["greedy"]), 4),
                      "sampled_minus_greedy_pct": round(100 * (mean["sampled"] / mean["greedy"] - 1), 3), **info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=("kernel", "step"))
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("sample_bench.py measures on a GPU; none is available")
    info = card()
    if args.only != "step":
        bench_kernel(info)
    if args.only != "kernel":
        bench_step(info, args.rounds, args.steps, args.warmup)


if __name__ == "__main__":
    main()

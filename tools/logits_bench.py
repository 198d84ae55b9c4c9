"""Logits-processing measurements: one JSON line per measurement, the card's name and power limit in every line.

    python tools/logits_bench.py [--only kernel|step] [--rounds R] [--steps K] [--warmup W]

kernel  kivi_logits_process_f32 + kivi_logits_record (every penalty on, so the counts are read; EOS suppression on) as
        100 pairs captured in one CUDA graph, the graph replayed between CUDA events, microseconds per pair, at
        (B, vocab) = (32, 32000), (64, 128256), (1, 128256); GB/s over the bytes the pair needs: logits and counts read and
        scores written (12 B per token) plus the prompt bits.
step    Llama-2-7B batch 32 and Llama-3-8B batch 64, K2V2 g32 R128, cache filled by prefill_synthetic to about 4096
        tokens: milliseconds per graph-replayed greedy decode step with processing off and on (repetition 1.2,
        presence 0.5, frequency 0.5, two EOS ids suppressed for the whole run), alternated R times in one process (the
        order swaps every round).
Needs a GPU: there is no CPU path.  Nothing is written outside the system's temporary directory.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from sample_bench import _graph_us_per_call, card  # noqa: E402

SHAPES = [(32, 32000), (64, 128256), (1, 128256)]
ON = dict(repetition_penalty=1.2, presence_penalty=0.5, frequency_penalty=0.5, min_new_tokens=1 << 30)


def bytes_needed(B, V):
    """logits + counts read, scores written (4 B each per token), the prompt bits read, and the record's few bytes."""
    return B * V * 12 + B * ((V + 31) // 32) * 4 + B * (8 + 4 + 4 + 1)


def bench_kernel(info):
    import torch
    from kivi_b200 import glue
    for B, V in SHAPES:
        gen = torch.Generator(device="cuda").manual_seed(B + V)
        dev = "cuda"
        logits = torch.randn((B, V), generator=gen, device=dev) * 3.0
        scores = torch.empty_like(logits)
        counts = torch.randint(0, 3, (B, V), generator=gen, device=dev, dtype=torch.int32)
        seen = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, (V + 31) // 32), generator=gen, device=dev, dtype=torch.int32)
        n_new = torch.zeros(B, dtype=torch.int32, device=dev)
        finished = torch.zeros(B, dtype=torch.uint8, device=dev)
        rep, pres, freq = (torch.full((B,), v, device=dev) for v in (1.2, 0.5, 0.5))
        min_new = torch.full((B,), 1 << 30, dtype=torch.int32, device=dev)
        eos = torch.tensor([2, 13], dtype=torch.long, device=dev)
        nxt = torch.zeros(B, dtype=torch.long, device=dev)

        def pair():
            glue.logits_process(logits, scores, counts, seen, n_new, finished, rep, pres, freq, min_new, eos, 0)
            glue.logits_record(nxt, counts, n_new, finished, eos)
        r = _graph_us_per_call(pair)
        gbs = bytes_needed(B, V) / (r["us_per_call_min"] * 1e-6) / 1e9
        print(json.dumps({"measurement": "kernel", "kernels": "kivi_logits_process_f32 + kivi_logits_record", "batch": B,
                          "vocab": V, **r, "bytes": bytes_needed(B, V), "GB_per_s_at_min": round(gbs, 1), **info}),
              flush=True)


def bench_step(info, name, B, seq, rounds, K, W):
    import torch
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config(name)
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

    def phase(on):
        if on:
            model.set_processing(**ON, eos_token_id=[2, 13])
        else:
            model.set_processing(None)
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

    res = {"off": [], "on": []}
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            ms, start = phase(on)
            res["on" if on else "off"].append(ms)
            print(json.dumps({"measurement": "step", "model": name, "batch": B, "kv_len_start": start, "steps": K,
                              "round": r, "processing": on, "ms_per_step": round(ms, 4),
                              "launches_per_step": model.launches_per_step, **info}), flush=True)
    mean = {k: sum(v) / len(v) for k, v in res.items()}
    print(json.dumps({"measurement": "step summary", "model": name, "batch": B, "seq": seq, "rounds": rounds,
                      "off_ms_per_step": round(mean["off"], 4), "on_ms_per_step": round(mean["on"], 4),
                      "off_spread_ms": round(max(res["off"]) - min(res["off"]), 4),
                      "on_spread_ms": round(max(res["on"]) - min(res["on"]), 4),
                      "on_minus_off_pct": round(100 * (mean["on"] / mean["off"] - 1), 3), **info}), flush=True)
    del model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=("kernel", "step"))
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("logits_bench.py measures on a GPU; none is available")
    info = card()
    if args.only != "step":
        bench_kernel(info)
    if args.only != "kernel":
        bench_step(info, "llama-2-7b", 32, 4096, args.rounds, args.steps, args.warmup)
        bench_step(info, "llama-3-8b", 64, 4096, args.rounds, args.steps, args.warmup)


if __name__ == "__main__":
    main()

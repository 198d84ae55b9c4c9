"""Qwen3's per-head q / k RMSNorm in the decode step, on one H100: the RoPE + split kernel with the norm folded in
(kivi_qk_norm_rope_split_f16) against the plain kernel (kivi_rope_split_f16), and the whole decode step with the norms
against the same shapes without them.

    python tools/qwen3_bench.py [--seq 4096] [--calls 64] [--reps 20] [--rounds 5] [--steps 16] [--out DIR]

Kernel: B in {32, 64} x query / KV heads {32/8 (Qwen3-4B / 8B), 64/8 (Qwen3-32B)}.  Each arm is a CUDA graph of --calls
launches on the same operands, timed with CUDA events over --reps replays; the two arms alternate for --rounds rounds
(round 0 settles clocks and is not counted), and the median is reported with every round listed.
  us     one launch
  bytes  the algorithmic HBM bytes of one launch from the shapes: qkv read once, q / k / v written once, one cos and
         one sin row per sequence, the positions, and (with the norm) the two 128-channel weights
  GBps   bytes / us.  These operands (at most 3 MB) fit in the H100's L2, and the replayed launches read them from
         there, so the rate is not an HBM rate.
Decode step: the random-init qwen3-8b and qwen3-4b shapes (36 layers, 32 / 8 heads, head_dim 128; the 4b shape has
hidden 2560 != 32 x 128) at B 32, T = --seq, K2V2 g32 R128.  The step is captured twice on one model: with the norms, and
with every layer's q_norm / k_norm detached (the step then calls the plain kernel), and the two graphs are replayed
alternately, --steps steps per sample, for --rounds rounds.
The card's name and power limit are read in the same run (one JSON line on stdout; with --out, also written there).
Nothing is written to the repository.
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

KERNEL_SHAPES = [(32, 32, 8), (64, 32, 8), (32, 64, 8), (64, 64, 8)]       # (B, H, Hkv)
MODELS = ["qwen3-8b", "qwen3-4b"]


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


def rope_bytes(B, H, Hkv, norm):
    io = 2 * B * (H + 2 * Hkv) * 128 * 2                 # qkv in, q / k / v out, fp16
    return io + B * (2 * 128 * 2 + 8) + (2 * 128 * 2 if norm else 0)


def one_kernel(B, H, Hkv, args):
    from kivi_b200 import glue
    from kivi_b200.llama_kivi import _rope_tables
    gen = torch.Generator(device="cuda").manual_seed(0)
    cos, sin = _rope_tables(128, 40960, 1e6, torch.device("cuda"))
    qkv = torch.randn((B, (H + 2 * Hkv) * 128), generator=gen, device="cuda").half()
    pos = torch.randint(0, 40960, (B,), generator=gen, device="cuda")
    wq, wk = (torch.rand(128, generator=gen, device="cuda").half() + 0.5 for _ in range(2))
    outs = {name: [torch.empty((B, n, 128), device="cuda", dtype=torch.float16) for n in (H, Hkv, Hkv)]
            for name in ("plain", "qk_norm")}
    arms = {"plain": lambda o=outs["plain"]: glue.rope_split(qkv, cos, sin, pos, *o),
            "qk_norm": lambda o=outs["qk_norm"]: glue.rope_split(qkv, cos, sin, pos, *o, wq, wk, 1e-6)}
    graphs = {name: graph_of(fn, args.calls) for name, fn in arms.items()}
    res = {name: [] for name in arms}
    for rnd in range(args.rounds + 1):
        for name, g in graphs.items():
            us = timed(g.replay, args.reps) / (args.reps * args.calls) * 1e3
            if rnd:
                res[name].append(us)
    out = {"B": B, "heads": f"{H}/{Hkv}"}
    for name in arms:
        us = statistics.median(res[name])
        by = rope_bytes(B, H, Hkv, name == "qk_norm")
        out[name] = {"us": round(us, 3), "bytes": by, "GBps": round(by / us / 1e3, 1),
                     "rounds": [round(x, 3) for x in res[name]]}
    out["qk_norm_minus_plain_us"] = round(out["qk_norm"]["us"] - out["plain"]["us"], 3)
    assert torch.equal(outs["plain"][2], outs["qk_norm"][2])                 # v is the same copy in both
    return out


def model_step(name, args):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config(name)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p_ in model.parameters():
        p_.requires_grad_(False)
    model.eval()
    B, T = 32, args.seq
    model.init_cache(B, T + (args.rounds + 1) * 2 * args.steps + 16)
    model.prefill_synthetic(T - 1, seed=0)
    tok = torch.zeros((B, 1), dtype=torch.long, device="cuda")
    attn = [layer.self_attn for layer in model.model.layers]
    norms = [(a.q_norm, a.k_norm) for a in attn]
    graphs, launches = {}, {}
    for arm in ("qk_norm", "plain"):
        for a, (qn, kn) in zip(attn, norms):
            a.q_norm, a.k_norm = (qn, kn) if arm == "qk_norm" else (None, None)
        model._graph = None
        model.decode_step(tok)
        graphs[arm], launches[arm] = model._graph, model.launches_per_step
    for a, (qn, kn) in zip(attn, norms):
        a.q_norm, a.k_norm = qn, kn
    res = {arm: [] for arm in graphs}
    for rnd in range(args.rounds + 1):
        for arm, g in graphs.items():
            model._graph = g
            ms = timed(lambda: model.decode_step(tok), args.steps) / args.steps
            if rnd:
                res[arm].append(ms)
    out = {"model": f"{name} shape (random init), K2V2 g32 R128, {cfg.num_hidden_layers} layers, hidden "
                    f"{cfg.hidden_size}", "B": B, "T": T}
    for arm in graphs:
        out[arm] = {"step_ms": round(statistics.median(res[arm]), 3), "rounds": [round(x, 3) for x in res[arm]],
                    "launches_per_step": launches[arm]}
    out["qk_norm_over_plain"] = round(out["qk_norm"]["step_ms"] / out["plain"]["step_ms"], 4)
    spread = [max(res[arm]) - min(res[arm]) for arm in graphs]
    out["spread_ms"] = round(max(spread), 3)
    del model, graphs
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--calls", type=int, default=64, help="kernel launches per captured graph")
    ap.add_argument("--reps", type=int, default=20, help="graph replays per timed kernel sample")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--no-model", action="store_true", help="skip the decode steps")
    ap.add_argument("--out", default=None, help="directory that receives qwen3_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qwen3_bench.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    result = {"card": card(), "rope_split": [one_kernel(B, H, Hkv, args) for B, H, Hkv in KERNEL_SHAPES]}
    if not args.no_model:
        result["decode_step"] = [model_step(name, args) for name in MODELS]
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "qwen3_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

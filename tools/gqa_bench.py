"""Decode attention at GQA ratios 3, 5, 6 and 7 on one H100: G = 4 query heads per work unit (a partly filled last unit
where 4 does not divide the ratio), G = 2 and G = 1, forced through KIVI_CACHE_GQA_CHUNK, ratio 4 as the control.  The
geometry's default is G = 4 at ratios 3, 4, 5 and 7 and G = 2 at ratio 6; the output's "default" names that arm.

    python tools/gqa_bench.py [--batch 32] [--seq 4096] [--calls 8] [--reps 16] [--rounds 5] [--steps 16] [--out DIR]

Before G = 4 with a partial last unit, the geometry picked the largest G in {1, 2, 4} dividing the ratio: G = 1 for
ratios 3, 5 and 7, G = 2 for ratio 6, G = 4 for ratio 4.  Every shape runs all three arms (G4, G2, G1); the output names
the geometry's default arm and that previous selection, and gives the default's and G = 4's speed-up over the previous one.
Shapes (query / KV heads): 24/8 (ratio 3, Llama-3.2-3B), 40/8 (5, Qwen2.5-14B/32B), 12/2 (6, Qwen2.5-1.5B) at B and at
4 B, 28/4 (7, Qwen2.5-7B), 32/8 (4, the control), each at K2V2 g32 R128 and K4V4 g64 R64, B = --batch, the cache pre-filled
with random K/V by the prefill pack kernels to --seq tokens.  Per shape the arms are warmed up and captured (a CUDA graph
of --calls calls of one layer's attention), then timed in alternating rounds in this one process, each sample --reps
replays of the graph:
  attn_ms   one call (median of the rounds; every round is listed, so the spread shows next to the difference)
  bytes     the algorithmic HBM bytes of one call from the shapes: every packed K / V block and fp16 window row once, the
            logits rows, q / out / k_new / v_new
  streamed  what the work units request: each of the B * Hkv * ceil(ratio / G) units streams all of its KV head's packed
            blocks and windows, so G = 1 requests them ratio times and G = 4 ceil(ratio / 4) times (repeats may hit L2)
  GBps      bytes / attn_ms
  l2_resident  bytes < 50 MB: the whole cache fits in the H100's L2, and the replayed calls read it from there, so the rate
            of such a shape is not an HBM rate (the 12/2 shape at 4 B is the one that does not fit)
Then the whole decode step of the random-init qwen2.5-7b shape (28 layers, 28 / 4 heads, K2V2 g32 R128), default against
G = 1, its previous selection.
The card's name and power limit are read in the same run (one JSON line on stdout; with --out, also written there).
Nothing is written to the repository.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(24, 8, 1), (40, 8, 1), (12, 2, 1), (12, 2, 4), (28, 4, 1), (32, 8, 1)]     # (H, Hkv, batch multiple)
L2_BYTES = 50 * 2 ** 20
CFGS = [(2, 2, 32, 128), (4, 4, 64, 64)]


def block_bytes(bits, g):
    """One packed 128 x 128 block: codes + scales / zeros (kivi_decode.cuh lay_block_bytes)."""
    return (4096 if bits == 2 else 8192) + 8 * (128 // g) * 64


def default_chunk(ratio):
    """The geometry's G (kivi_decode.cu gqa_chunk): the largest G in {1, 2, 4} dividing the ratio, 4 for odd ratios above 2."""
    return 4 if ratio % 4 == 0 else 2 if ratio % 2 == 0 else 4 if ratio >= 3 else 1


def previous_chunk(ratio):
    """The G the geometry picked before partial units: the largest G in {1, 2, 4} that divides the ratio."""
    return 4 if ratio % 4 == 0 else 2 if ratio % 2 == 0 else 1


def attention_bytes(cache, H, G):
    """(algorithmic bytes, bytes the work units stream) of one call"""
    B, Hkv = cache.batch, cache.num_kv_heads
    ratio = H // Hkv
    chunks = -(-ratio // G)
    n_kb, n_vb = -(-cache.tk // 128), -(-cache.tv // 128)
    g = cache.group_size
    per_unit = (n_kb * block_bytes(cache.k_bits, g) + n_vb * block_bytes(cache.v_bits, g) + (cache.r + cache.L) * 256)
    logits = ratio * 2 * ((n_kb * 128 + cache.r + 1) + (n_vb * 128 + cache.L + 1))      # written by q.K^T, read by p.V
    io = (2 * B * H + 2 * B * Hkv) * 256
    return B * Hkv * (per_unit + logits) + io, B * Hkv * (chunks * per_unit + logits) + io


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unavailable ({e})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def set_chunk(cache, G):
    """Run `cache`'s decode attention with G query heads per unit (KIVI_CACHE_GQA_CHUNK; 0 = the geometry's choice), with
    a workspace sized for it."""
    from kivi_b200 import _lib
    for st in cache._structs:
        st.flags = (st.flags & ~0x70) | (G << 4)
    need = int(_lib.lib().kivi_decode_workspace_bytes(ctypes.byref(cache._structs[0]), cache.max_tokens))
    _lib.check(need if need < 0 else 0, "kivi_decode_workspace_bytes")
    if cache._ws.numel() < need:
        cache._ws = torch.zeros(need, dtype=torch.uint8, device=cache.device)


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


def one_shape(H, Hkv, mult, kb, vb, g, R, args):
    from kivi_b200.cache import KiviCache
    B, T = args.batch * mult, args.seq
    arms = {"G4": 4, "G2": 2, "G1": 1}
    caches, graphs, outs = {}, {}, {}
    gen = torch.Generator(device="cuda").manual_seed(0)
    k = torch.randn((B, Hkv, T - 1, 128), generator=gen, device="cuda", dtype=torch.float16)
    v = torch.randn((B, Hkv, T - 1, 128), generator=gen, device="cuda", dtype=torch.float16)
    q = torch.randn((B, H, 128), generator=gen, device="cuda", dtype=torch.float16)
    kn = torch.randn((B, Hkv, 128), generator=gen, device="cuda", dtype=torch.float16)
    vn = torch.randn_like(kn)
    for name, G in arms.items():                          # warm up and capture every arm before any timing
        c = KiviCache(1, B, H, Hkv, 128, kb, vb, g, R, T + 8, gqa_chunk=G)
        c.prefill(0, k, v)
        outs[name] = torch.empty_like(q)
        graphs[name] = graph_of(lambda c=c, o=outs[name]: c.decode_attention(0, q, kn, vn, out=o), args.calls)
        caches[name] = c
    torch.cuda.synchronize()
    diff = max((outs["G4"].float() - outs[n].float()).abs().max().item() for n in arms)
    res = {name: [] for name in arms}
    for rnd in range(args.rounds + 1):                    # round 0 settles clocks, not counted
        for name in arms:
            a = timed(graphs[name].replay, args.reps) / (args.reps * args.calls)
            if rnd:
                res[name].append(a)
    ratio = H // Hkv
    out = {"heads": f"{H}/{Hkv}", "ratio": ratio, "cfg": f"K{kb}V{vb} g{g} R{R}", "B": B, "T": T,
           "max_abs_out_diff": diff}
    for name, G in arms.items():
        a = statistics.median(res[name])
        by, streamed = attention_bytes(caches[name], H, G)
        out[name] = {"G": G, "units_per_kv_head": -(-ratio // G), "attn_ms": round(a, 4), "bytes": by,
                     "streamed": streamed, "GBps": round(by / a / 1e6, 1), "rounds": [round(x, 4) for x in res[name]]}
    out["default"], out["previous"] = f"G{default_chunk(ratio)}", f"G{previous_chunk(ratio)}"
    d = out[out["default"]]["attn_ms"]
    out["speedup_vs_previous"] = round(out[out["previous"]]["attn_ms"] / d, 3)
    out["speedup_vs_G1"] = round(out["G1"]["attn_ms"] / d, 3)
    out["G4_vs_previous"] = round(out[out["previous"]]["attn_ms"] / out["G4"]["attn_ms"], 3)
    out["l2_resident"] = out["G4"]["bytes"] < L2_BYTES
    del caches, graphs
    torch.cuda.empty_cache()
    return out


def model_step(args):
    """The whole decode step of the random-init qwen2.5-7b shape, default selection against forced G = 1."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config("qwen2.5-7b", num_hidden_layers=args.layers)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p_ in model.parameters():
        p_.requires_grad_(False)
    model.eval()
    B, T = args.batch, args.seq
    steps_total = (args.rounds + 1) * 2 * args.steps + 16
    model.init_cache(B, T + steps_total)
    model.prefill_synthetic(T - 1, seed=0)
    set_chunk(model.cache, 4)                             # the larger of the two workspaces, allocated once
    assert previous_chunk(cfg.num_attention_heads // cfg.num_key_value_heads) == 1
    tok = torch.zeros((B, 1), dtype=torch.long, device="cuda")
    arms = {"default": 0, "G1": 1}
    step_graphs = {}
    for name, G in arms.items():
        set_chunk(model.cache, G)
        model._graph = None
        model.decode_step(tok)
        step_graphs[name] = model._graph
    res = {name: [] for name in arms}
    for rnd in range(args.rounds + 1):
        for name, G in arms.items():
            set_chunk(model.cache, G)
            model._graph = step_graphs[name]
            s = timed(lambda: model.decode_step(tok), args.steps) / args.steps
            if rnd:
                res[name].append(s)
    out = {"model": f"qwen2.5-7b shape (random init), K2V2 g32 R128, {args.layers} layers", "B": B, "T": T}
    for name in arms:
        out[name] = {"step_ms": round(statistics.median(res[name]), 3), "rounds": [round(x, 3) for x in res[name]]}
    out["speedup_vs_G1"] = round(out["G1"]["step_ms"] / out["default"]["step_ms"], 3)
    del model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--calls", type=int, default=8)
    ap.add_argument("--reps", type=int, default=16, help="graph replays per timed sample")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--no-model", action="store_true", help="skip the end-to-end decode step")
    ap.add_argument("--out", default=None, help="directory that receives gqa_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gqa_bench.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    result = {"card": card(), "attention": [one_shape(H, Hkv, m, *c, args) for H, Hkv, m in SHAPES for c in CFGS]}
    if not args.no_model:
        result["decode_step"] = model_step(args)
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gqa_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

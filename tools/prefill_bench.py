"""Prompt-pass measurements on one H100: the prompt-attention kernel against today's masked SDPA call, and whole prompt
passes at the long-context shapes.  One JSON line per measurement, each with the card's name and power limit.

    python tools/prefill_bench.py [--only kernel,window,a,b,c,d] [--rounds 5]

kernel   Llama-2-7B attention shape (B 32, H = Hkv = 32, n 4096), left-padded with starts spread over [0, n/2) (seeded):
         kivi_prompt_attention_f16 against SDPA with the additive fp16 [B, 1, n, n] mask, alternated in the same process;
         and the unpadded batch against SDPA is_causal, for the record.  TFLOP/s count the visible (query, key) pairs
         only: 4 * 128 FLOP per pair and query head.
window   Mistral-7B attention shape (B 1, H 32, Hkv 8, n 32768): the kernel at W = 4096 against W = 0.
a, b     Llama-2-7B, B 32, n 4096, prefill() left-padded as above (a) and unpadded (b, the SDPA path).
c        Llama-3-8B, B 64, n 8192, prefill() unpadded.
d        Mistral-7B K4V4 g64 R64, B 16, n 32768, W 4096, generate(max_new_tokens=128): time to first token (the prompt
         pass) and decode tok/s (B * 127 tokens over the rest of the call).
Random-init fp16 weights, as bench.py.  Times are CUDA events after a warm-up call of the same shape; peak memory is
torch.cuda.max_memory_allocated over the timed call, in total and above the weights and the cache.  Nothing is written
to the repository.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    idx = torch.cuda.current_device()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(idx)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return {"gpu": torch.cuda.get_device_name(idx), "power_limit_w": power}


def emit(rec):
    print(json.dumps(dict(rec, **card())), flush=True)


def timed(fn, calls=1):
    """ms per call of fn over `calls` back-to-back calls (CUDA events)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def starts_spread(B, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, n // 2, (B,), generator=g, dtype=torch.int32)


def visible_pairs(n, starts, window=0):
    """Visible (query, key) pairs summed over the batch: query i sees max(s, i - W + 1) <= j <= i."""
    i = torch.arange(n, dtype=torch.int64)
    total = 0
    for s in starts.tolist():
        lo = torch.full_like(i, min(max(s, 0), n))
        if window:
            lo = torch.maximum(lo, i - window + 1)
        total += int((i - lo + 1).clamp(min=0).sum())
    return total


def qkv(B, H, Hkv, n):
    """Strided [B, heads, n, 128] views of [B, n, heads, 128] storage, as the model's projections leave them."""
    def make(h):
        return torch.randn((B, n, h, 128), device="cuda", dtype=torch.float16).transpose(1, 2)
    return make(H), make(Hkv), make(Hkv)


def kernel_vs_sdpa(rounds):
    from kivi_b200 import glue
    from kivi_b200.llama_kivi import repeat_kv
    B, H, n = 32, 32, 4096
    q, k, v = qkv(B, H, H, n)
    out = torch.empty((B, n, H, 128), device="cuda", dtype=torch.float16)
    for padded in (True, False):
        starts = starts_spread(B, n) if padded else torch.zeros(B, dtype=torch.int32)
        ks = starts.cuda() if padded else None
        if padded:
            i = torch.arange(n, device="cuda")
            keep = (i[None, None, :] >= ks[:, None, None]) & (i[None, None, :] <= i[None, :, None])
            mask = torch.zeros(keep.shape, dtype=torch.float16, device="cuda").masked_fill(~keep, torch.finfo(torch.float16).min)
            mask = mask[:, None]
            del keep
            sdpa = lambda: F.scaled_dot_product_attention(q, repeat_kv(k, 1), repeat_kv(v, 1), attn_mask=mask)  # noqa: E731
        else:
            sdpa = lambda: F.scaled_dot_product_attention(q, repeat_kv(k, 1), repeat_kv(v, 1), is_causal=True)  # noqa: E731
        ours = lambda: glue.prompt_attention(q, k, v, out, ks, 0)                                               # noqa: E731
        ours(), sdpa()
        t = {"kernel": [], "sdpa": []}
        for _ in range(rounds):
            t["kernel"].append(timed(ours, 3))
            t["sdpa"].append(timed(sdpa, 3))
        flop = 4 * 128 * H * visible_pairs(n, starts)
        km, sm = statistics.median(t["kernel"]), statistics.median(t["sdpa"])
        emit({"what": "kernel vs sdpa", "padded": padded, "B": B, "H": H, "n": n, "kernel_ms": round(km, 3),
              "sdpa_ms": round(sm, 3), "speedup": round(sm / km, 3), "kernel_tflops_visible": round(flop / km / 1e9, 1),
              "sdpa_tflops_visible": round(flop / sm / 1e9, 1), "kernel_ms_rounds": [round(x, 3) for x in t["kernel"]],
              "sdpa_ms_rounds": [round(x, 3) for x in t["sdpa"]]})
        if padded:
            del mask


def window_vs_full(rounds):
    from kivi_b200 import glue
    B, H, Hkv, n, W = 1, 32, 8, 32768, 4096
    q, k, v = qkv(B, H, Hkv, n)
    out = torch.empty((B, n, H, 128), device="cuda", dtype=torch.float16)
    zero = torch.zeros(B, dtype=torch.int32)
    fns = {w: (lambda w=w: glue.prompt_attention(q, k, v, out, None, w)) for w in (W, 0)}
    for f in fns.values():
        f()
    t = {w: [] for w in fns}
    for _ in range(rounds):
        for w, f in fns.items():
            t[w].append(timed(f, 3))
    med = {w: statistics.median(x) for w, x in t.items()}
    pairs = {w: visible_pairs(n, zero, w) for w in fns}
    emit({"what": "window vs full", "B": B, "H": H, "Hkv": Hkv, "n": n, "W": W, "window_ms": round(med[W], 3),
          "full_ms": round(med[0], 3), "time_ratio": round(med[W] / med[0], 3),
          "pair_ratio": round(pairs[W] / pairs[0], 3),
          "window_tflops_visible": round(4 * 128 * H * pairs[W] / med[W] / 1e9, 1),
          "full_tflops_visible": round(4 * 128 * H * pairs[0] / med[0] / 1e9, 1)})


def build(name, **kw):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config(name, **kw)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p in model.parameters():
        p.requires_grad_(False)
    return model.eval()


def prompt_pass(tag, name, B, n, padded, kivi=None):
    model = build(name, **(kivi or {}))
    ids = torch.randint(1, model.config.vocab_size, (B, n), device="cuda")
    mask = None
    if padded:
        s = starts_spread(B, n).cuda()
        mask = (torch.arange(n, device="cuda")[None, :] >= s[:, None]).long()
    model.init_cache(B, n + 8)
    model.prefill(ids, attention_mask=mask)                            # warm-up of the same shape
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ms = timed(lambda: model.prefill(ids, attention_mask=mask))
    peak = torch.cuda.max_memory_allocated()
    emit({"what": "prompt pass", "case": tag, "model": name, "B": B, "n": n, "padded": padded, "ms": round(ms, 1),
          "prompt_tokens_per_s": round(B * n / ms * 1e3), "peak_gib": round(peak / 2 ** 30, 2),
          "peak_above_weights_cache_gib": round((peak - base) / 2 ** 30, 2)})
    del model
    torch.cuda.empty_cache()


def mistral_generate():
    B, n, W, new = 16, 32768, 4096, 128
    model = build("mistral-7b", k_bits=4, v_bits=4, group_size=64, residual_length=64, sliding_window=W)
    ids = torch.randint(1, model.config.vocab_size, (B, n), device="cuda")
    prefill, t_prefill = model.prefill, []

    def timed_prefill(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = prefill(*a, **kw)
        e1.record()
        t_prefill.append((e0, e1))
        return r
    model.prefill = timed_prefill
    model.generate(ids, max_new_tokens=new)                            # warm-up: the same shapes, the step's graph
    torch.cuda.synchronize()
    t_prefill.clear()
    torch.cuda.reset_peak_memory_stats()
    total = timed(lambda: model.generate(ids, max_new_tokens=new))
    ttft = t_prefill[0][0].elapsed_time(t_prefill[0][1])
    peak = torch.cuda.max_memory_allocated()
    decode_ms = total - ttft
    emit({"what": "generate", "case": "d", "model": "mistral-7b K4V4 g64 R64", "B": B, "n": n, "W": W,
          "max_new_tokens": new, "ttft_ms": round(ttft, 1), "decode_ms": round(decode_ms, 1),
          "decode_tok_s": round(B * (new - 1) / decode_ms * 1e3, 1), "peak_gib": round(peak / 2 ** 30, 2)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="kernel,window,a,b,c,d")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefill_bench.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    parts = set(args.only.split(","))
    with torch.no_grad():
        if "kernel" in parts:
            kernel_vs_sdpa(args.rounds)
        if "window" in parts:
            window_vs_full(args.rounds)
        if "a" in parts:
            prompt_pass("a", "llama-2-7b", 32, 4096, True)
        if "b" in parts:
            prompt_pass("b", "llama-2-7b", 32, 4096, False)
        if "c" in parts:
            prompt_pass("c", "llama-3-8b", 64, 8192, False)
        if "d" in parts:
            mistral_generate()


if __name__ == "__main__":
    main()

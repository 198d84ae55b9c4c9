"""Memory / speed harness in the shape of the reference's mem_spd_test.py (`mem_spd_test.py:8-70`): a batch of
identical-length prompts, greedy generation of a fixed number of new tokens, mean wall time over a few repeats and the
peak allocated device memory.

    python tools/mem_spd_test.py                       # the reference's case: bs 96, 160 + 338 tokens, Llama-2-7B K2V2
    python tools/mem_spd_test.py --batch 32 --prompt 2048 --new 2048 --model llama-3-8b

Differences from the reference script, forced by the offline box: weights are random-init from the architecture table
(`kivi_b200.llama_kivi.default_config`), the prompt is random token ids instead of the tokenised "t,t,t," string, and
generation is this package's greedy `generate()` (pre-allocated KiviCache, CUDA-graph decode step) instead of HF
`generate`.  Prints the reference's two lines ("used time", "peak mem") and one JSON line.

`--fp16-baseline` runs the OTHER arm of the reference's script (`mem_spd_test.py:33-42`: K_BITS = 16 -> stock Hugging Face
`LlamaForCausalLM`, fp16 KV cache, HF `generate`) on the same random-init architecture, so that the README's peak-memory and
throughput ratios (`README.md:29`) have a counterpart on this implementation."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--model", default="llama-2-7b", choices=["llama-2-7b", "llama-3-8b", "mistral-7b", "tiny"])
    ap.add_argument("--batch", type=int, default=96)          # mem_spd_test.py:12
    ap.add_argument("--prompt", type=int, default=160)        # :54
    ap.add_argument("--new", type=int, default=338)           # :55
    ap.add_argument("--repeats", type=int, default=3)         # :56
    ap.add_argument("--k-bits", type=int, default=2, choices=[2, 4])
    ap.add_argument("--v-bits", type=int, default=2, choices=[2, 4])
    ap.add_argument("--group-size", type=int, default=32)
    ap.add_argument("--residual-length", type=int, default=128)
    ap.add_argument("--no-graph", action="store_true", help="run the decode step eagerly instead of replaying a CUDA graph")
    ap.add_argument("--fp16-baseline", action="store_true",
                    help="the reference script's K_BITS=16 arm: transformers' LlamaForCausalLM with an fp16 KV cache")
    ap.add_argument("--out", default=None, help="append the JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mem_spd_test.py needs a CUDA device (the KIVI path has no CPU fallback)")
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config

    cfg = default_config(a.model, k_bits=a.k_bits, v_bits=a.v_bits, group_size=a.group_size,
                         residual_length=a.residual_length)
    if a.fp16_baseline:
        return fp16_baseline(a, cfg)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p in model.parameters():
        p.requires_grad_(False)
    model.eval()
    ids = torch.randint(0, cfg.vocab_size, (a.batch, a.prompt), device="cuda")
    print(f"bs: {a.batch}, seqlen: {a.prompt}+{a.new}\nmodel:{a.model} (random-init), K{a.k_bits}V{a.v_bits} "
          f"g{a.group_size} residual {a.residual_length}")

    weights_gb = torch.cuda.memory_allocated() / 1024 ** 3
    torch.cuda.reset_peak_memory_stats()
    times = []
    with torch.no_grad():
        for _ in range(a.repeats):
            model.init_cache(a.batch, a.prompt + a.new + 8)   # a fresh cache (and decode graph) per request batch
            torch.cuda.synchronize()
            st = time.time()
            out = model.generate(ids, max_new_tokens=a.new, use_graph=not a.no_graph)
            torch.cuda.synchronize()
            times.append(time.time() - st)
            assert out.shape == (a.batch, a.prompt + a.new)
    used = sum(times) / len(times)
    peak_gb = torch.cuda.max_memory_allocated() / 1024 ** 3
    print(f"used time: {used * 1000} ms")
    print(f"peak mem: {peak_gb} GB")
    emit(a, {"arm": "kivi_b200", "model": a.model, "batch": a.batch, "prompt": a.prompt, "new_tokens": a.new, "repeats": a.repeats,
             "k_bits": a.k_bits, "v_bits": a.v_bits, "group_size": a.group_size,
             "residual_length": a.residual_length, "used_time_ms": used * 1000, "best_time_ms": min(times) * 1000,
             "tokens_per_s": a.batch * a.new / used, "peak_mem_gb": peak_gb, "weights_gb": weights_gb,
             "kv_cache_gb": model.cache.nbytes() / 1024 ** 3,
             "cuda_graph": not a.no_graph, "data": "synthetic ids, random-init weights"})
    return 0


def emit(a, rec):
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


def fp16_baseline(a, cfg):
    """mem_spd_test.py:33-42, :63-70 with K_BITS = 16: transformers' own LlamaForCausalLM (fp16 KV cache, its generate())."""
    import torch
    from transformers import LlamaConfig, LlamaForCausalLM
    hf = LlamaConfig(hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                     num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                     num_key_value_heads=cfg.num_key_value_heads, vocab_size=cfg.vocab_size, rope_theta=cfg.rope_theta,
                     rms_norm_eps=cfg.rms_norm_eps, max_position_embeddings=max(4096, a.prompt + a.new + 8))
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM(hf).half()
    model.eval()
    ids = torch.randint(0, cfg.vocab_size, (a.batch, a.prompt), device="cuda")
    print(f"bs: {a.batch}, seqlen: {a.prompt}+{a.new}\nmodel:{a.model} (random-init), fp16 KV cache (transformers LlamaForCausalLM)")
    weights_gb = torch.cuda.memory_allocated() / 1024 ** 3
    torch.cuda.reset_peak_memory_stats()
    times = []
    with torch.no_grad():
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            st = time.time()
            out = model.generate(input_ids=ids, attention_mask=torch.ones_like(ids), max_new_tokens=a.new,
                                 min_new_tokens=a.new, do_sample=False, pad_token_id=0)
            torch.cuda.synchronize()
            times.append(time.time() - st)
            assert out.shape == (a.batch, a.prompt + a.new)
    used = sum(times) / len(times)
    peak_gb = torch.cuda.max_memory_allocated() / 1024 ** 3
    print(f"used time: {used * 1000} ms")
    print(f"peak mem: {peak_gb} GB")
    kv_gb = a.batch * (a.prompt + a.new) * cfg.num_hidden_layers * 2 * cfg.num_key_value_heads * 128 * 2 / 1024 ** 3
    emit(a, {"arm": "fp16 baseline (transformers LlamaForCausalLM.generate)", "model": a.model, "batch": a.batch, "prompt": a.prompt,
             "new_tokens": a.new, "repeats": a.repeats, "used_time_ms": used * 1000, "best_time_ms": min(times) * 1000,
             "tokens_per_s": a.batch * a.new / used, "peak_mem_gb": peak_gb, "weights_gb": weights_gb, "kv_cache_gb": kv_gb,
             "data": "synthetic ids, random-init weights"})
    return 0


if __name__ == "__main__":
    sys.exit(main())

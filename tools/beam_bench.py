"""Beam-search measurements on the fused cache: one JSON line per prompt batch, the card's name and power limit in every
line.

    python tools/beam_bench.py [--model llama-2-7b] [--batches 1,4,8] [--beams 4] [--prompt 2048] [--new 128]

The model is random-init fp16 with K2V2, g32, R128.  The beam loop is that of LlamaForCausalLM_KIVI.generate(num_beams=K)
(_generate_many) with CUDA events around its three parts: the decode-step graph, the selection (kivi_b200.beam plus the
one device-to-host read) and the reorder graph (KiviCache._enqueue_reorder and the position gather).  No EOS id is set,
so every run takes all `new` steps.  The reorder's bytes are counted from the lengths and the rows it rewrites and
stages (read + write of the live packed blocks and the whole fp16 windows of every unit of every layer); its share is of
the H100 SXM data sheet's 3.35 TB/s.  The prompt pass is timed once per prompt (prompt-once, what generate does) and,
for comparison, with the prompt expanded to B * K rows as transformers runs it.
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

HBM_GBS = 3350.0


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


def row_bytes(cache):
    """Bytes of one row that a reorder copies at the cache's current lengths (all layers)."""
    kbb = cache._bytes[0] // (cache.batch * cache.num_kv_heads * cache.k_cap_blocks)
    vbb = cache._bytes[1] // (cache.batch * cache.num_kv_heads * cache.v_cap_blocks)
    unit = -(-cache.tk // 128) * kbb + -(-cache.tv // 128) * vbb + (cache._bytes[2] + cache._bytes[3]) // (
        cache.batch * cache.num_kv_heads)
    return cache.n_layers * cache.num_kv_heads * unit


def staged(src):
    readers = {s for b, s in enumerate(src) if s != b}
    return sum(1 for s in readers if src[s] != s)


def timed_prompt(model, ids, copies):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    model.lm_head(model._prompt_pass(ids, None, copies=copies)[:, -1]).float()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def beam_run(model, ids, K, new):
    import torch
    from kivi_b200.beam import BeamSearch
    B, n = ids.shape
    rows = B * K
    ev = lambda: torch.cuda.Event(enable_timing=True)       # noqa: E731
    model.set_sampling(None)
    logits = model.lm_head(model._prompt_pass(ids, None, copies=K)[:, -1]).float()
    search = BeamSearch(ids, K, n + new)
    model.cache.reorder_scratch()
    t_sel, t_reo, t_step, rewritten, stage, moved = [], [], [], [], [], 0
    first = True
    torch.cuda.synchronize()
    start, end = ev(), ev()
    start.record()
    while True:
        e0, e1, e2, e3 = ev(), ev(), ev(), ev()
        e0.record()
        beam_idx, tok, done = search.step(logits)
        host = torch.cat([beam_idx, done.view(1).long()]).tolist()
        e1.record()
        if host[-1]:
            break
        src = host[:-1]
        model._ids.copy_(tok.view(rows, 1))
        if not first:
            model._reorder_rows(beam_idx, src)
            rw, st = sum(1 for b, s in enumerate(src) if s != b), staged(src)
            rewritten.append(rw)
            stage.append(st)
            moved += 2 * (rw + st) * row_bytes(model.cache)
        e2.record()
        logits = model.decode_step()
        e3.record()
        torch.cuda.synchronize()
        t_sel.append(e0.elapsed_time(e1))
        if not first:
            t_reo.append(e1.elapsed_time(e2))
        t_step.append(e2.elapsed_time(e3))
        first = False
    end.record()
    torch.cuda.synchronize()
    total = start.elapsed_time(end)
    mean = lambda x: sum(x) / max(len(x), 1)                 # noqa: E731
    reo_s = sum(t_reo) / 1e3
    return {"steps": len(t_step), "beam_tokens_per_s": rows * len(t_step) / (total / 1e3),
            "ms_step_graph": mean(t_step), "ms_selection": mean(t_sel), "ms_reorder_graph": mean(t_reo),
            "rows_rewritten_per_step": mean(rewritten), "rows_staged_per_step": mean(stage),
            "reorder_gb_per_step": moved / max(len(t_reo), 1) / 1e9,
            "reorder_gbs": moved / reo_s / 1e9 if reo_s > 0 else None,
            "reorder_share_of_3_35_tbs": moved / reo_s / 1e9 / HBM_GBS if reo_s > 0 else None,
            "launches_per_beam_step": (model.launches_per_step or 0) + (model.launches_per_reorder or 0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-2-7b")
    ap.add_argument("--batches", default="1,4,8")
    ap.add_argument("--beams", type=int, default=4)
    ap.add_argument("--prompt", type=int, default=2048)
    ap.add_argument("--new", type=int, default=128)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("beam_bench needs a CUDA device")
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    info = card()
    cfg = default_config(a.model, k_bits=2, v_bits=2, group_size=32, residual_length=128)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg).half()
    for p in model.parameters():
        p.requires_grad_(False)
    model.eval()
    K = a.beams
    with torch.no_grad():
        for B in [int(x) for x in a.batches.split(",")]:
            ids = torch.randint(1, cfg.vocab_size, (B, a.prompt), device="cuda")
            model.init_cache(B * K, a.prompt + a.new)
            timed_prompt(model, ids, K)                          # warm-up
            once = timed_prompt(model, ids, K)
            try:
                expanded = timed_prompt(model, ids.repeat_interleave(K, 0), 1)
            except torch.cuda.OutOfMemoryError:
                expanded = None                                  # not measured
            torch.cuda.empty_cache()
            beam_run(model, ids[:, : a.prompt // 4], K, 8)      # warm-up: captures both graphs, kept for the timed run
            res = beam_run(model, ids, K, a.new)
            line = dict(info, model=a.model, batch=B, beams=K, prompt=a.prompt, new=a.new,
                        ms_prompt_once=once, ms_prompt_expanded=expanded, **res)
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

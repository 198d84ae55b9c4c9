"""LoRA adapters per request on one H100: the shrink / expand kernels per projection group, the same delta from torch
gather + bmm, the decode step with and without adapters, and serve() over mixed- and single-adapter streams.

    python tools/lora_bench.py [--reps 20] [--steps 16] [--rounds 3] [--serve-layers 8] [--out DIR]

Kernels: the four groups of Llama-2-7B (B 32) and Llama-3-8B (B 64) with 1, 4 and 16 distinct adapters spread round-robin
over the rows and r in {8, 16, 64}.  Each arm is a CUDA graph of 20 calls timed with CUDA events over --reps replays.
  shrink_us / expand_us   one launch of each kernel
  bmm_us                  the same delta with torch: gather the rows' A and B, two bmm, add (fp32 intermediate)
  GBps                    algorithmic bytes / (shrink + expand): each present adapter's A and B once, x, t (fp32) and y
                          read and written once.
Decode step (B and T of the shape, K2V2 g32 R128, random init): no adapter loaded, adapters loaded but every row without
one, and 4 distinct r = 16 all-linear adapters across the batch: --rounds rounds of the first arm, then the other two
alternating for --rounds rounds (the first round of each arm settles clocks and is not counted), --steps replays per
sample, median ms reported.
serve(): the Llama-2-7B shape cut to --serve-layers layers (the time is the step's, so fewer layers keep the run short),
B 32, 96 requests of 256-token prompts and 64 new tokens: one stream with every request on one adapter, one cycling
through 4 adapters; tokens per second of wall time.
The card's name and power limit are read in the same run (one JSON line on stdout; with --out, also written there).
Nothing is written to the repository."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"llama-2-7b": (32, 4096), "llama-3-8b": (64, 8192)}       # (B, T)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unavailable ({e})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def timed(fn, calls=20, reps=20):
    """us per call of fn, captured `calls` times in one graph and replayed reps times."""
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
    g.replay()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        g.replay()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / (reps * calls)


def kernels(cfg, B, reps):
    import ctypes
    from kivi_b200 import _lib, glue, lora
    sh = lora.module_shapes(cfg)
    rows = []
    for group, mods in lora.GROUPS.items():
        n_in, segs = sh[mods[0]][1], lora.seg_offsets(group, sh)
        out, n_seg = segs[-1], len(mods)
        for r in (8, 16, 64):
            for S in (1, 4, 16):
                A = torch.randn((S, n_seg, r, n_in), device="cuda").half() * 0.02
                Bw = torch.randn((S, out, r), device="cuda").half() * 0.02
                scale = torch.ones(S, device="cuda")
                idx = (torch.arange(B, device="cuda") % S).to(torch.int32)
                x = torch.randn((B, n_in), device="cuda").half()
                y = torch.randn((B, out), device="cuda").half()
                ws = torch.empty(glue.lora_workspace_bytes(B, n_in, n_seg, r) // 4, device="cuda")
                glue.lora_apply(x, y, A, Bw, scale, segs, idx, ws)           # binds and checks the operands
                L = _lib.lib()
                c_segs = (ctypes.c_int * (n_seg + 1))(*segs)

                def shrink():                 # the stream is read at each call: capture runs on a side stream
                    _lib.check(L.kivi_lora_shrink_f16(x.data_ptr(), B, n_in, A.data_ptr(), S, n_seg, r, idx.data_ptr(),
                                                      ws.data_ptr(), _lib.stream_ptr()), "kivi_lora_shrink_f16")

                def expand():
                    _lib.check(L.kivi_lora_expand_f16(ws.data_ptr(), B, n_in, Bw.data_ptr(), scale.data_ptr(), S, n_seg, r,
                                                      c_segs, idx.data_ptr(), y.data_ptr(), out, _lib.stream_ptr()),
                               "kivi_lora_expand_f16")
                us_s, us_e = timed(shrink, reps=reps), timed(expand, reps=reps)
                seg_of = torch.repeat_interleave(torch.arange(n_seg, device="cuda"),
                                                 torch.tensor([segs[g + 1] - segs[g] for g in range(n_seg)], device="cuda"))
                lidx = idx.long()

                def bmm():
                    t = torch.bmm(A[lidx].float().view(B, n_seg * r, n_in), x.float().view(B, n_in, 1)).view(B, n_seg, r)
                    d = torch.bmm(Bw[lidx].float(), t.transpose(1, 2)).gather(2, seg_of.view(1, -1, 1).expand(B, -1, 1))
                    d = d.squeeze(-1)
                    y.add_((d * scale[lidx].view(B, 1)).half())
                us_b = timed(bmm, calls=4, reps=max(2, reps // 4))
                nbytes = S * (n_seg * r * n_in + out * r) * 2 + B * n_in * 2 + 2 * B * out * 2 + \
                    2 * B * n_seg * r * 4 * -(-n_in // 512)
                rows.append(dict(group=group, r=r, adapters=S, shrink_us=round(us_s, 2), expand_us=round(us_e, 2),
                                 bmm_us=round(us_b, 2), bytes=nbytes, GBps=round(nbytes / (us_s + us_e) / 1e3, 1)))
                del A, Bw, ws
    return rows


def decode_steps(name, steps, rounds, tmp):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    from tests._lora import adapter_state, write_adapter
    B, T = SHAPES[name]
    cfg = default_config(name)
    torch.manual_seed(0)
    m = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    m.init_cache(B, T + 64 + 4 * steps * rounds)
    m.prefill_synthetic(T)
    tok = torch.zeros((B, 1), dtype=torch.long, device="cuda")
    ms = {}

    def sample(label):
        m.decode_step(tok)                                                 # captures when the arm is new
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(steps):
            m.decode_step(tok)
        t1.record()
        t1.synchronize()
        ms.setdefault(label, []).append(t0.elapsed_time(t1) / steps)
    for _ in range(rounds):
        sample("no_adapter")
    launches = {"no_adapter": m.launches_per_step}
    for i in range(4):
        st = adapter_state(cfg, 16, ["q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"],
                           seed=i, gain=0.1)
        m.load_adapter(write_adapter(tmp / f"{name}-{i}", st, 16, 32, "all-linear"), f"a{i}")
    for _ in range(rounds):
        m.set_adapters(None)
        sample("loaded_unused")
        m.set_adapters([f"a{b % 4}" for b in range(B)])
        sample("four_adapters")
    launches["with_adapters"] = m.launches_per_step
    res = {k: dict(median_ms=round(statistics.median(v[1:] or v), 4), rounds=[round(x, 4) for x in v]) for k, v in ms.items()}
    res["launches_per_step"] = launches
    del m
    torch.cuda.empty_cache()
    return res


def serve_rate(layers, tmp):
    import time
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    from kivi_b200.serve import serve
    from tests._lora import adapter_state, write_adapter
    cfg = default_config("llama-2-7b", num_hidden_layers=layers)
    torch.manual_seed(0)
    m = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    for i in range(4):
        st = adapter_state(cfg, 16, ["q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"],
                           seed=i, gain=0.1)
        m.load_adapter(write_adapter(tmp / f"serve-{i}", st, 16, 32, "all-linear"), f"a{i}")
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(0, cfg.vocab_size, (256,), generator=g) for _ in range(96)]
    out = {}
    for label, names in (("single_adapter", ["a0"] * 96), ("mixed_4_adapters", [f"a{i % 4}" for i in range(96)])) * 2:
        reqs = [(p, 64, dict(adapter=a)) for p, a in zip(prompts, names)]
        torch.cuda.synchronize()
        t = time.perf_counter()
        n = sum(len(ids) for _, ids in serve(m, reqs, batch=32, max_tokens=1024))
        torch.cuda.synchronize()
        out[label] = round(n / (time.perf_counter() - t), 1)               # the second pass of each stream is kept
    return out


def main():
    import pathlib
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--serve-layers", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_bench needs a CUDA device")
    from kivi_b200.llama_kivi import default_config
    res = {"card": card(), "kernels": {}, "decode_step": {}}
    with tempfile.TemporaryDirectory() as tmp:
        tmp = pathlib.Path(tmp)
        for name, (B, _) in SHAPES.items():
            res["kernels"][name] = kernels(default_config(name), B, a.reps)
        for name in SHAPES:
            res["decode_step"][name] = decode_steps(name, a.steps, a.rounds, tmp)
        res["serve_tokens_per_s"] = serve_rate(a.serve_layers, tmp)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lora_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""Tensor-parallel decode measurements: one JSON line per workload.

    python tools/tp_bench.py [--workloads a,b,c,kernel] [--tp 1,2,4,8] [--steps K] [--warmup W]

Every rank builds its shard directly on its GPU from a seed (random weights; nothing full-size is materialised), fills its
cache with `prefill_synthetic` so that the K timed steps end at the workload's length, and times K replays of the captured
decode step with CUDA events (max over ranks).  A separate torch.profiler run of a few replays gives the time spent in the
all-reduce kernels.  Workloads (K2V2 g32 R128):
  a       Llama-3-8B, B = 1, T = 32k: the single-sequence latency case, TP 1 / 2 / 4 / 8
  b       Llama-2-70B shape, B = 32, T = 4096, TP 4 / 8 (the 70B weights do not fit one GPU)
  c       Llama-2-7B, global batch 32, T = 4096: TP 2 against two data-parallel replicas of 16, same run
  kernel  kivi_allreduce_add_rmsnorm_f16 alone with N ranks emulated on one GPU (partials in local HBM, not over NVLink):
          the cluster widths 1 / 2 / 4 / 8 per row at B = 1 and 32
TP 1 is the unsharded model.  A configuration that needs more GPUs than the box has prints a line with "not measured".
Nothing is written outside the system's temporary directory.
"""
from __future__ import annotations

import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

WORKLOADS = {
    "a": dict(model="llama-3-8b", batch=1, seq=32768, tps=(1, 2, 4, 8)),
    "b": dict(model="llama-2-70b", batch=32, seq=4096, tps=(4, 8)),
    "c": dict(model="llama-2-7b", batch=32, seq=4096, tps=(2,)),
}


def card():
    import torch
    idx = torch.cuda.current_device()
    name = torch.cuda.get_device_name(idx)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(idx)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return {"gpu": name, "power_limit_w": power}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _build(model_name, dev, tensor_parallel, seq, margin):
    import torch
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config(model_name)
    cfg.max_position_embeddings = max(cfg.max_position_embeddings, seq + margin)
    torch.manual_seed(0)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float16)
    try:
        with torch.device(dev):                                          # this rank's shard only, built on its GPU
            model = LlamaForCausalLM_KIVI(cfg, tensor_parallel=tensor_parallel)
    finally:
        torch.set_default_dtype(prev)
    for p in model.parameters():
        p.requires_grad_(False)
    return model.eval(), cfg


def _time_steps(model, K, W, ids):
    """Warm up (the first step captures the graph), then K graph replays between CUDA events; returns ms per step."""
    import torch
    from kivi_b200 import dist as kdist
    model.decode_step(ids)
    for _ in range(W - 1):
        model.decode_step()
    torch.cuda.synchronize()
    kdist.barrier()
    g = model._graph
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        g.replay()
        model.cache._mirror_advance()
    e1.record()
    torch.cuda.synchronize()
    if model._allreduce is not None:
        model._allreduce.check()
    return kdist.max_over_ranks(e0.elapsed_time(e1) / K)


def _allreduce_kernel_ms(model, reps=4):
    """Device time per step of the kernels named allreduce_add_rmsnorm, from a torch.profiler run of `reps` replays."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    g = model._graph
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            g.replay()
            model.cache._mirror_advance()
        torch.cuda.synchronize()
    tot, n = 0.0, 0
    for e in prof.key_averages():
        if "allreduce_add_rmsnorm" in e.key:
            tot += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            n += e.count
    if model._allreduce is not None:
        model._allreduce.check()
    return tot / 1e3 / reps, n // reps


def _rank_main(rank, ws, port, job, out_path):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(ws), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch
    from types import SimpleNamespace
    from kivi_b200 import dist as kdist
    import bench
    kdist.init()
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    K, W, B, seq, mode = job["steps"], job["warmup"], job["batch"], job["seq"], job["mode"]
    margin = W + K + 64 + 128
    model, cfg = _build(job["model"], dev, mode == "tp" and ws > 1, seq, margin)
    if mode == "dp":
        B //= ws
    model.init_cache(B, seq + margin)
    model.prefill_synthetic(seq - (W + K), seed=rank)
    if mode == "dp" and ws > 1:
        model.enable_token_allgather(ws, mode="p2p")
    ids = torch.randint(0, cfg.vocab_size, (B, 1), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    ms = _time_steps(model, K, W, ids)
    ar_ms, ar_calls = _allreduce_kernel_ms(model)
    cache = model.cache
    shim = SimpleNamespace(config=SimpleNamespace(num_attention_heads=cache.num_heads, num_key_value_heads=cache.num_kv_heads),
                           decode_step=model.decode_step)
    roof = bench.attention_roofline(shim, cache, ms)
    Bg = B * ws if mode == "dp" else B
    line = {"workload": job["name"], "model": job["model"], "parallelism": f"{mode}{ws}" if ws > 1 else "1 GPU (unsharded)",
            "global_batch": Bg, "seq_len": seq, "k_bits": 2, "v_bits": 2, "group_size": 32, "residual_length": 128,
            "tok_s": Bg / (ms / 1e3), "ms_per_step": ms, "steps": K,
            "attention_roofline_per_rank": {k: roof[k] for k in ("achieved", "peak", "unit", "frac", "launch_ms",
                                                                  "share_of_step", "peak_source")},
            "allreduce_kernel_ms_per_step": ar_ms if ar_calls else 0.0, "allreduce_calls_per_step": ar_calls,
            "nvlink_bytes_read_per_call": (ws - 1) * B * cfg.hidden_size * 2 if mode == "tp" else 0,
            **card()}
    torch.cuda.synchronize()
    kdist.barrier()
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(line, f)
    if ws > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


def run_job(job, ngpu):
    ws = job["tp"]
    if ws > ngpu:
        print(json.dumps({"workload": job["name"], "model": job["model"], "parallelism": f"{job['mode']}{ws}",
                          "result": f"not measured: needs {ws} GPUs, this box has {ngpu}"}), flush=True)
        return
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "line.json")
        mp.spawn(_rank_main, args=(ws, _free_port(), job, out), nprocs=ws, join=True)
        with open(out) as f:
            print(f.read(), flush=True)


def kernel_alternatives(reps=100):
    """The all-reduce + RMSNorm kernel at every cluster width, N ranks emulated in one allocation on this GPU."""
    import torch
    from types import SimpleNamespace
    from kivi_b200 import glue
    for hidden in (4096, 8192):
        for world in (2, 4, 8):
            for rows in (1, 32):
                slot_words = rows * hidden * 2 // 8
                buf = torch.zeros(world, 2 * slot_words + world, dtype=torch.int64, device="cuda")
                for p in range(world):
                    buf[p].view(torch.float16)[: 2 * rows * hidden].normal_()
                buf[0, 2 * slot_words:] = 1 << 40                          # every rank has arrived at every call
                ar = SimpleNamespace(peer_ptrs=torch.tensor([buf[p].data_ptr() for p in range(world)], dtype=torch.int64,
                                                            device="cuda"),
                                     rank=0, world=world, rows_max=rows, hidden=hidden,
                                     epoch=torch.zeros(1, dtype=torch.int64, device="cuda"),
                                     err=torch.zeros(1, dtype=torch.int32, device="cuda"))
                res = torch.randn((rows, hidden), device="cuda").half()
                w = torch.ones(hidden, dtype=torch.float16, device="cuda")
                out = torch.empty_like(res)
                x = torch.randn((rows, hidden), device="cuda").half()

                def graph_ms(fn):
                    """Device time of one call: `reps` calls captured in a CUDA graph, the graph replayed 5 times."""
                    s_ = torch.cuda.Stream()
                    s_.wait_stream(torch.cuda.current_stream())
                    with torch.cuda.stream(s_):
                        for i in range(3):
                            fn(i)
                    torch.cuda.current_stream().wait_stream(s_)
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        for i in range(reps):
                            fn(i)
                    g.replay()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(5):
                        g.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    return e0.elapsed_time(e1) / (5 * reps) * 1e3

                times = {str(cl): graph_ms(lambda i, cl=cl: glue.allreduce_add_rmsnorm(res, w, out, 1e-5, ar, call=i,
                                                                                       cluster=cl))
                         for cl in (1, 2, 4, 8)}
                local = graph_ms(lambda i: glue.add_rmsnorm(x, res, w, out, 1e-5))
                assert int(ar.err.item()) == 0
                print(json.dumps({"workload": "kivi_allreduce_add_rmsnorm_f16, N ranks emulated on one GPU (local HBM)",
                                  "hidden": hidden, "world": world, "rows": rows, "us_per_call_by_cluster": times,
                                  "add_rmsnorm_us_per_call": local,
                                  "bytes_read_per_call": world * rows * hidden * 2,
                                  **card()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="a,b,c,kernel")
    ap.add_argument("--tp", default="1,2,4,8", help="tensor-parallel degrees to try (each workload keeps its own list)")
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=4)
    args = ap.parse_args()
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu == 0:
        raise SystemExit("tp_bench needs CUDA GPUs")
    allowed = {int(t) for t in args.tp.split(",")}
    for name in args.workloads.split(","):
        if name == "kernel":
            kernel_alternatives()
            continue
        w = WORKLOADS[name]
        for t in w["tps"]:
            if t not in allowed:
                continue
            job = dict(name=name, model=w["model"], batch=w["batch"], seq=w["seq"], tp=t, mode="tp",
                       steps=args.steps, warmup=args.warmup)
            run_job(job, ngpu)
            if name == "c":                                               # the same global batch as 2 data-parallel replicas
                run_job(dict(job, mode="dp"), ngpu)


if __name__ == "__main__":
    main()

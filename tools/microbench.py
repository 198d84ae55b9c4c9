"""Kernel micro-benchmarks on one H100 (CUDA events, L2 flushed between iterations).

    python tools/microbench.py [--ref] [--out microbench.json]

Times the generic-layout GEMVs (cuda_bmm_fA_qB_outer) and the pack kernel at the BASELINE cfg 2
per-layer shapes; with --ref also the UNMODIFIED reference extension (oracle/_ref/kivi_gemv.so),
kernel-only and wrapper-inclusive (its three transpose().contiguous() copies, quant/matmul.py:205-214).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timeit_graph(fn, reps=8, iters=10):
    """Kernel-bound timing for calls that are SHORTER than their Python wrapper (~80 us of ctypes + torch per call): `reps`
    back-to-back calls captured in one CUDA graph and replayed; ms per call (median, best).  The operands of the cfg shapes
    (~200 MB per call) exceed the 50 MB L2, so consecutive calls on the same operands still stream from HBM."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        g.replay()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) / reps)
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def timeit(fn, iters=20, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--H", type=int, default=32)
    ap.add_argument("--Hkv", type=int, default=32)
    ap.add_argument("--T", type=int, default=4096)
    ap.add_argument("--bits", type=int, default=2)
    ap.add_argument("--g", type=int, default=32)
    ap.add_argument("--R", type=int, default=128)
    ap.add_argument("--only-fused", action="store_true", help="time only the decode attention on the blocked cache")
    a = ap.parse_args()
    from kivi_b200 import matmul, new_pack
    dev = "cuda"
    B, H, Hkv, D, T, bits, g, R = a.B, a.H, a.Hkv, 128, a.T, a.bits, a.g, a.R
    Tk = (T - 1) // R * R
    Tv = T - 1 - R
    gen = torch.Generator(device=dev).manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)      # > 50 MB L2
    res = {"config": vars(a), "Tk": Tk, "Tv": Tv, "gpu": torch.cuda.get_device_name(0)}

    # calibration: plain copy
    src = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    ms, best = timeit(lambda: dst.copy_(src), iters=10)
    res["copy_GBps"] = 2 * src.numel() / best / 1e6
    del src, dst

    if not a.only_fused:
        generic_part(a, res, gen, flush, dev)
    fused_part(a, res, gen, flush, dev)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


def generic_part(a, res, gen, flush, dev):
    from kivi_b200 import matmul, new_pack
    B, H, Hkv, D, T, bits, g, R = a.B, a.H, a.Hkv, 128, a.T, a.bits, a.g, a.R
    Tk = (T - 1) // R * R
    Tv = T - 1 - R
    kT = torch.randn((B, Hkv, D, Tk), generator=gen, device=dev, dtype=torch.float16)
    kc, ks, kz = new_pack.triton_quantize_and_pack_along_last_dim(kT, g, bits)
    del kT
    v = torch.randn((B, Hkv, Tv, D), generator=gen, device=dev, dtype=torch.float16)
    vc, vs, vz = new_pack.triton_quantize_and_pack_along_last_dim(v, g, bits)
    del v
    q = torch.randn((B, H, 1, D), generator=gen, device=dev, dtype=torch.float16)
    p = torch.softmax(torch.randn((B, H, 1, T), generator=gen, device=dev), -1).half()
    pq = p[:, :, :, :Tv]

    bytes_qk = B * Hkv * Tk * D * (bits / 8 + 4 / g) + B * H * D * 2 + B * H * Tk * 2
    bytes_sv = B * Hkv * Tv * D * (bits / 8 + 4 / g) + B * H * Tv * 2 + B * H * D * 2
    ms, best = timeit_graph(lambda: matmul.cuda_bmm_fA_qB_outer(g, q, kc, ks, kz, bits))
    res["ours_qk_ms"] = ms
    res["ours_qk_GBps"] = bytes_qk / ms / 1e6
    ms, best = timeit_graph(lambda: matmul.cuda_bmm_fA_qB_outer(g, pq, vc, vs, vz, bits))
    res["ours_sv_ms"] = ms
    res["ours_sv_GBps"] = bytes_sv / ms / 1e6
    ms, _ = timeit(lambda: matmul.cuda_bmm_fA_qB_outer(g, q, kc, ks, kz, bits), flush=flush)
    res["ours_qk_single_call_ms"] = ms          # one eager call incl. its Python wrapper (CPU-bound below ~0.08 ms)

    # pack: decode V token and K flush
    vnew = torch.randn((B, Hkv, 1, D), generator=gen, device=dev, dtype=torch.float16)
    ms, _ = timeit(lambda: new_pack.triton_quantize_and_pack_along_last_dim(vnew, g, bits), flush=flush)
    res["ours_pack_v_token_ms"] = ms
    kres = torch.randn((B, Hkv, D, R), generator=gen, device=dev, dtype=torch.float16)
    ms, _ = timeit(lambda: new_pack.triton_quantize_and_pack_along_last_dim(kres, g, bits), flush=flush)
    res["ours_pack_k_flush_ms"] = ms
    res["ours_pack_k_flush_GBps"] = (kres.numel() * 2 * (1 + (bits / 8 + 4 / g) / 2)) / ms / 1e6

    if a.ref:
        reference_part(a, res, gen, flush, dev, q, pq, bytes_qk, bytes_sv)


def fused_part(a, res, gen, flush, dev):
    """decode attention on the blocked cache (two launches: q.K^T + statistics, p.V + output + cache update)"""
    from kivi_b200.cache import KiviCache
    B, H, Hkv, D, T, bits, g, R = a.B, a.H, a.Hkv, 128, a.T, a.bits, a.g, a.R
    # launched as inside a decoder layer (the q.K^T prologue may overlap the previous kernel: results are not checked here)
    cache = KiviCache(1, B, H, Hkv, 128, bits, bits, g, R, max_tokens=T + 256,
                      overlap_prologue=True)
    nfill = T - 1 - R // 2                                            # mid-window state (no K flush in the timed call)
    kk = torch.randn((B, Hkv, nfill, D), generator=gen, device=dev, dtype=torch.float16)
    vv = torch.randn((B, Hkv, nfill, D), generator=gen, device=dev, dtype=torch.float16)
    cache.prefill(0, kk, vv)
    # prompt -> blocked stores (models/llama_kivi.py:425-452 fused: transpose + quantise + fragment pack of K, pack of V)
    ms_p, _ = timeit(lambda: cache.prefill(0, kk, vv), flush=flush, iters=5)
    res["prefill_pack_ms"] = ms_p
    res["prefill_pack_GBps"] = 2 * B * Hkv * nfill * D * (2 + bits / 8 + 4 / g) / ms_p / 1e6   # fp16 K and V read, packed written
    del kk, vv
    qd = torch.randn((B, H, D), generator=gen, device=dev, dtype=torch.float16)
    kn = torch.randn((B, Hkv, D), generator=gen, device=dev, dtype=torch.float16)
    vn = torch.randn((B, Hkv, D), generator=gen, device=dev, dtype=torch.float16)
    outd = torch.empty_like(qd)
    per_tok = D * (bits / 8 + 4 / g)
    bytes_fused = B * Hkv * (cache.tk * per_tok + cache.tv * per_tok + (cache.r + cache.L) * D * 2) + 2 * B * H * D * 2
    ms, best = timeit(lambda: cache.decode_attention(0, qd, kn, vn, out=outd), flush=flush, iters=30)
    res["fused_state"] = [cache.tk, cache.r, cache.tv, cache.L]
    res["fused_decode_ms"] = ms
    res["fused_decode_best_ms"] = best
    res["fused_decode_GBps"] = bytes_fused / ms / 1e6
    res["fused_bytes"] = bytes_fused
    ms2, _ = timeit(lambda: cache.decode_attention(0, qd, kn, vn, out=outd), iters=30)   # no L2 flush (cache >> L2 anyway)
    res["fused_decode_noflush_ms"] = ms2
    ms3, best3 = timeit_graph(lambda: cache.decode_attention(0, qd, kn, vn, out=outd))   # 8 back-to-back calls in one CUDA graph
    res["fused_decode_graph_ms"] = ms3
    res["fused_decode_graph_GBps"] = bytes_fused / ms3 / 1e6


def reference_part(a, res, gen, flush, dev, q, pq, bytes_qk, bytes_sv):
    from kivi_b200 import matmul, new_pack
    B, H, Hkv, D, T, bits, g, R = a.B, a.H, a.Hkv, 128, a.T, a.bits, a.g, a.R
    Tk = (T - 1) // R * R
    Tv = T - 1 - R
    if True:
        kT = torch.randn((B, Hkv, D, Tk), generator=gen, device=dev, dtype=torch.float16)
        kc, ks, kz = new_pack.triton_quantize_and_pack_along_last_dim(kT, g, bits)
        del kT
        v = torch.randn((B, Hkv, Tv, D), generator=gen, device=dev, dtype=torch.float16)
        vc, vs, vz = new_pack.triton_quantize_and_pack_along_last_dim(v, g, bits)
        del v
        from oracle import build_ref
        refmod = build_ref.load()
        if refmod is None:
            res["ref"] = "unavailable"
        else:
            def ref_wrapper(fA, qB, scales, zeros):              # quant/matmul.py:199-218 restated for timing
                Bq, nh, M, K = fA.shape
                nh_kv = qB.shape[1]
                fA2 = fA.reshape(-1, M, K).contiguous()
                qB2 = qB.reshape(-1, K, qB.shape[-1]).transpose(1, 2).contiguous()
                s2 = scales.reshape(-1, scales.shape[-2], scales.shape[-1]).transpose(1, 2).contiguous()
                z2 = zeros.reshape(-1, zeros.shape[-2], zeros.shape[-1]).transpose(1, 2).contiguous()
                return refmod.gemv_forward_cuda_outer_dim(fA2, qB2, s2, z2, bits, g, nh, nh_kv)
            ms, _ = timeit(lambda: ref_wrapper(q, kc, ks, kz), flush=flush, iters=10)
            res["ref_qk_wrapper_ms"] = ms
            ms, _ = timeit(lambda: ref_wrapper(pq, vc, vs, vz), flush=flush, iters=10)
            res["ref_sv_wrapper_ms"] = ms
            q2 = q.reshape(-1, 1, D).contiguous()
            kc2 = kc.reshape(-1, D, kc.shape[-1]).transpose(1, 2).contiguous()
            ks2 = ks.reshape(-1, D, ks.shape[-1]).transpose(1, 2).contiguous()
            kz2 = kz.reshape(-1, D, kz.shape[-1]).transpose(1, 2).contiguous()
            # (the reference extension launches on the legacy default stream: not capturable, timed call by call)
            ms, _ = timeit(lambda: refmod.gemv_forward_cuda_outer_dim(q2, kc2, ks2, kz2, bits, g, H, Hkv), flush=flush, iters=10)
            res["ref_qk_kernel_ms"] = ms
            res["ref_qk_kernel_GBps"] = bytes_qk / ms / 1e6
            del kc2, ks2, kz2
            p2 = pq.reshape(-1, 1, Tv).contiguous()
            vc2 = vc.reshape(-1, Tv, vc.shape[-1]).transpose(1, 2).contiguous()
            vs2 = vs.reshape(-1, Tv, vs.shape[-1]).transpose(1, 2).contiguous()
            vz2 = vz.reshape(-1, Tv, vz.shape[-1]).transpose(1, 2).contiguous()
            ms, _ = timeit(lambda: refmod.gemv_forward_cuda_outer_dim(p2, vc2, vs2, vz2, bits, g, H, Hkv), flush=flush, iters=10)
            res["ref_sv_kernel_ms"] = ms
            res["ref_sv_kernel_GBps"] = bytes_sv / ms / 1e6


if __name__ == "__main__":
    main()

"""The reference-layout dequant-GEMV (cuda_bmm_fA_qB_outer) and the other GEMV surfaces against an exact reference, on
every kernel the dispatch can choose and across value magnitudes.  Reference and bar: tests/_gemv.py (exact_bar).

Routes.  The tensor-core kernels (kivi_bgemv_mma.cu) contract x*s split into hi = fp16(x*s) and lo = fma(x, s, -hi); that
split overflows for large scales and loses the residual in the fp16 denormals for small products.  ROUTES reaches every
MMA instantiation (tall at cluster sizes 1, 2, 4 and 8, wide at one and two head chunks and both scale granules), the SIMT
wide / tall kernels at 1, 2 and 4 heads per lane, the generic, kernel-layout and inner kernels, and the edges where copies
are zero-filled or masked; test_routes_reach_every_kernel checks in a profiler trace that each named kernel ran.

Magnitudes.  Named regimes, each on its own seed: q.K^T on the four reachable wide MMA instantiations and SIMT wide, p.V on
every tall instantiation at 600, 4096 and 32768 tokens of one KV unit (cluster sizes 1, 4 and 8), a reduced set on the
SIMT routes, and the edge rows of test_pack_edge_values as K and V groups."""
import json

import numpy as np
import pytest
import torch

from oracle import ref
from tests._gemv import (OUTLIER_CHANNELS, checked_gemv, edge_rows, kernel_layout_case, run_bmm, run_inner,
                         run_kernel_layout)

pytestmark = pytest.mark.gpu


def softmax16(logits):
    p = np.exp(logits - logits.max(-1, keepdims=True))
    return (p / p.sum(-1, keepdims=True)).astype(np.float16)


# ---------------------------------------------------------------------------------------------------
# routes
# ---------------------------------------------------------------------------------------------------
# kind "qk": fA = q [B,H,1,K], w [B,Hkv,K,N] ~ K^T; kind "pv": fA = softmax probabilities, w ~ V.
# name: kind, B, H, Hkv, K, N, g, bits, options, expected kernel (demangled name prefix), tall cluster size (grid.y)
ROUTES = {
    # MMA tall: every instantiation, cluster sizes 1, 2, 4, 8; K in {1, 127, 129, 128 n + 5}
    "tall-2-1-32-K1": ("pv", 2, 2, 2, 1, 128, 32, 2, {}, "kivi::bgm::tall_kernel<2, 1, 32>", 1),
    "tall-2-1-32-K600": ("pv", 1, 1, 1, 600, 128, 32, 2, {}, "kivi::bgm::tall_kernel<2, 1, 32>", 1),
    "tall-2-1-32-K389-meta4": ("pv", 1, 2, 2, 389, 128, 32, 2, {"meta_offset": 2}, "kivi::bgm::tall_kernel<2, 1, 32>", 1),
    "tall-4-1-32-S2": ("pv", 1, 1, 1, 2048 + 5, 128, 32, 4, {}, "kivi::bgm::tall_kernel<4, 1, 32>", 2),
    "tall-2-1-64-S4": ("pv", 1, 1, 1, 4096, 128, 64, 2, {}, "kivi::bgm::tall_kernel<2, 1, 64>", 4),
    "tall-4-1-64-S8-ratio3": ("pv", 1, 3, 1, 8192 + 77, 128, 64, 4, {}, "kivi::bgm::tall_kernel<4, 1, 64>", 8),
    "tall-2-2-64-K129": ("pv", 1, 2, 1, 129, 128, 64, 2, {}, "kivi::bgm::tall_kernel<2, 2, 64>", 1),
    "tall-4-2-64-K127": ("pv", 2, 4, 2, 127, 128, 64, 4, {}, "kivi::bgm::tall_kernel<4, 2, 64>", 1),
    "tall-4-2-64-S8-gqa": ("pv", 2, 32, 8, 8192 + 77, 128, 64, 4, {}, "kivi::bgm::tall_kernel<4, 2, 64>", 8),
    "tall-2-1-32-contiguous-fA": ("pv", 1, 2, 2, 777, 128, 32, 2, {"strided_pad": 0}, "kivi::bgm::tall_kernel<2, 1, 32>", 1),
    # MMA wide: ratio 2 at g32 (G = 1), ratio 2 / 4 at g64 (G = 2, one / two head chunks); N = 64 (three idle warps),
    # N % 512 != 0 (a partial last tile); scale rows of N / g % 4 == 0 (8-byte granule) and == 2 (4-byte granule)
    "wide-2-1-32-gran8": ("qk", 2, 4, 2, 128, 1024, 32, 2, {}, "kivi::bgm::wide_kernel<2, 1, 32>", None),
    "wide-4-1-32-N64-gran4": ("qk", 1, 2, 1, 128, 64, 32, 4, {}, "kivi::bgm::wide_kernel<4, 1, 32>", None),
    "wide-2-2-64-Z1-partial-gran4": ("qk", 1, 2, 1, 128, 1664, 64, 2, {}, "kivi::bgm::wide_kernel<2, 2, 64>", None),
    "wide-4-2-64-Z2-partial-gran8": ("qk", 2, 8, 2, 128, 2304, 64, 4, {}, "kivi::bgm::wide_kernel<4, 2, 64>", None),
    "wide-2-2-64-Z2-gran8": ("qk", 1, 4, 1, 128, 1024, 64, 2, {}, "kivi::bgm::wide_kernel<2, 2, 64>", None),
    # SIMT fast kernels: wide (N > 256) and tall (N <= 256) at G = 1, 2, 4 query heads per lane
    "simt-wide-G1": ("qk", 2, 4, 4, 128, 1024, 32, 2, {}, "void kivi::bgemv_ref_wide_kernel<2, 1>", None),
    "simt-wide-G2-g128": ("qk", 1, 4, 2, 128, 768, 128, 4, {}, "void kivi::bgemv_ref_wide_kernel<4, 2>", None),
    "simt-wide-G4": ("qk", 1, 8, 2, 128, 1536, 32, 2, {}, "void kivi::bgemv_ref_wide_kernel<2, 4>", None),
    "simt-tall-G1-N256": ("pv", 1, 2, 2, 1000, 256, 32, 4, {}, "void kivi::bgemv_ref_tall_kernel<4, 1>", None),
    "simt-tall-G2-N64": ("pv", 1, 4, 2, 333, 64, 32, 2, {}, "void kivi::bgemv_ref_tall_kernel<2, 2>", None),
    "simt-tall-G4-g128": ("pv", 2, 8, 2, 700, 128, 128, 2, {}, "void kivi::bgemv_ref_tall_kernel<2, 4>", None),
    # generic kernel: g % 32 != 0
    "generic-2-g16": ("pv", 1, 4, 2, 50, 48, 16, 2, {}, "void kivi::bgemv_ref_generic_kernel<2>", None),
    "generic-4-g24": ("qk", 2, 2, 1, 77, 48, 24, 4, {}, "void kivi::bgemv_ref_generic_kernel<4>", None),
}


def _route_inputs(name):
    kind, B, H, Hkv, K, N, g, bits, opt, _, _ = ROUTES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    w = rng.standard_normal((B, Hkv, K, N)).astype(np.float16)
    if kind == "qk":
        fA = rng.standard_normal((B, H, 1, K)).astype(np.float16)
    else:
        fA = softmax16(rng.standard_normal((B, H, 1, K)) * 2)
    opts = {"strided_pad": 5 if kind == "pv" else 0, "meta_offset": 0}
    opts.update(opt)
    return fA, w, g, bits, opts


@pytest.mark.parametrize("name", list(ROUTES))
def test_route_matches_exact(name):
    fA, w, g, bits, opts = _route_inputs(name)
    checked_gemv("bmm", fA, w, g, bits, name, group_floor=True, **opts)     # previous floor: MMA sums x*s*c, x*z apart


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("mqa", [False, True])
def test_kernel_layout_matches_exact(bits, mqa):
    B, nh, IC, OC = 2, 8, 739, 128
    x, w = kernel_layout_case(np.random.default_rng(40 + bits + 2 * mqa), B, nh, 1 if mqa else nh, IC, OC)
    checked_gemv("kernel", x, w, 32, bits, f"kernel layout b{bits} mqa {mqa}", nh=nh)


@pytest.mark.parametrize("g", [64, 128])
def test_inner_gemv_matches_exact(g):
    rng = np.random.default_rng(70 + g)
    Bn, IC, OC = 4, 1024, 96
    x = rng.standard_normal((Bn, IC)).astype(np.float16)
    w = rng.standard_normal((OC, IC)).astype(np.float16)
    checked_gemv("inner", x, w, g, 4, f"inner g{g}")


def _trace_kernels(path):
    """(name, grid) of every kernel event of a chrome trace."""
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    return [(e["name"], tuple(e.get("args", {}).get("grid", ()))) for e in events if e.get("cat") == "kernel"]


def test_routes_reach_every_kernel(tmp_path):
    """One profiler trace around every route case: each expected kernel ran, and each tall case at its cluster size."""
    from torch.profiler import ProfilerActivity, profile
    prepared = []
    for name in ROUTES:
        fA, w, g, bits, opts = _route_inputs(name)
        prepared.append((name, fA, ref.pack_lastdim(w, g, bits), g, bits, opts))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)      # the trace's first kernel: the profiler may not record the very first
        torch.cuda.synchronize()
        for name, fA, (code, scale, mn), g, bits, opts in prepared:
            run_bmm(fA, code, scale, mn, g, bits, **opts)
        for bits in (2, 4):
            x, w = kernel_layout_case(np.random.default_rng(40 + bits), 2, 8, 8, 739, 128)    # as test_kernel_layout_matches_exact
            run_kernel_layout(x, *ref.pack_lastdim(w, 32, bits), 32, bits, 8)
        run_inner(np.zeros((2, 512), np.float16), np.zeros((64, 64), np.int32), *[np.zeros((64, 8), np.float16)] * 2, 64)
        torch.cuda.synchronize()
    path = tmp_path / "routes_trace.json"
    prof.export_chrome_trace(str(path))
    ran = _trace_kernels(path)
    names = [n for n, _ in ran]
    expected = {ROUTES[n][9] for n in ROUTES} | {"void kivi::bgemv_kernel_layout_kernel<2>",
                                                 "void kivi::bgemv_kernel_layout_kernel<4>", "void kivi::gemv_inner_kernel<4>"}
    missing = sorted(k for k in expected if not any(k in n for n in names))
    assert not missing, f"kernels that never ran: {missing}; ran: {sorted(set(names))}"
    for name in ROUTES:
        kname, S = ROUTES[name][9], ROUTES[name][10]
        if S is not None:
            grids_y = {gr[1] for n, gr in ran if kname in n and len(gr) == 3}
            assert S in grids_y, f"{name}: no {kname} launch with cluster size {S} (grid.y seen: {sorted(grids_y)})"
    tall_s = {gr[1] for n, gr in ran if "tall_kernel<" in n and "bgm" in n and len(gr) == 3}
    assert {1, 2, 4, 8} <= tall_s, f"tall cluster sizes seen: {sorted(tall_s)}"


# ---------------------------------------------------------------------------------------------------
# magnitude sweep
# ---------------------------------------------------------------------------------------------------
QK_KERNELS = {   # name: B, H, Hkv, Tk, g, bits
    "wide-2-1-32": (1, 2, 1, 2048, 32, 2),
    "wide-4-1-32": (1, 2, 1, 2048, 32, 4),
    "wide-2-2-64": (1, 2, 1, 2048 + 128, 64, 2),
    "wide-4-2-64": (1, 4, 1, 2048, 64, 4),
    "simt-wide-G1": (1, 2, 2, 2048, 32, 2),
}
QK_REGIMES = {   # name: seed, q std, K std, extras
    "unit": (1, 1.0, 1.0, {}),
    "q-2^-6": (2, 2.0 ** -6, 1.0, {}),
    "q-8": (3, 8.0, 1.0, {}),
    "q-zero": (4, 0.0, 1.0, {}),
    "k-2^-6": (5, 1.0, 2.0 ** -6, {}),
    "k-2^-10": (6, 1.0, 2.0 ** -10, {}),
    "k-1e-4": (7, 1.0, 1e-4, {}),
    "k-16": (8, 1.0, 16.0, {}),
    "k-outliers-x32": (9, 1.0, 1.0, {"outliers": 32.0}),
    "k-outliers-x1000": (10, 2.0 ** -4, 1.0, {"outliers": 1000.0}),
    "k-range-thousands": (11, 2.0 ** -6, 2500.0, {}),          # 2-bit scales ~3k-20k, 4-bit group ranges ~ 20k-60k
    "k-range-near-max": (12, 2.0 ** -8, 1.0, {"near_max": True}),
    "q-tiny": (13, 2.0 ** -20, 1.0, {}),                        # max|q| < 2^-16: below what the row prescale can lift
    "k-inf-beside-large": (14, 2.0 ** -8, 1.0, {"inf_beside_large": True}),
}


def _qk_inputs(kname, rname):
    B, H, Hkv, Tk, g, bits = QK_KERNELS[kname]
    seed, qs, ks, extra = QK_REGIMES[rname]
    rng = np.random.default_rng(seed * 1009 + len(kname))
    k = rng.standard_normal((B, Hkv, 128, Tk)) * ks
    if "outliers" in extra:
        k[:, :, OUTLIER_CHANNELS] *= extra["outliers"]
    if "near_max" in extra:                                       # one group per channel spans about +-30000
        k[:, :, :, 0] = 30000.0
        k[:, :, :, 1] = -30000.0
    if "inf_beside_large" in extra:                               # per 64 tokens: a group whose range overflows (scale inf),
        k[:, :, :, 0::64], k[:, :, :, 1::64] = 60000.0, -60000.0     # then at g32 a finite group of range 32000
        k[:, :, :, 32::64], k[:, :, :, 33::64] = 16000.0, -16000.0
    k = np.clip(k, -60000, 60000).astype(np.float16)
    q = (rng.standard_normal((B, H, 1, 128)) * qs).astype(np.float16)
    return q, k, g, bits


@pytest.mark.parametrize("kname", list(QK_KERNELS))
@pytest.mark.parametrize("rname", list(QK_REGIMES))
def test_qk_magnitude_sweep(kname, rname):
    q, k, g, bits = _qk_inputs(kname, rname)
    checked_gemv("bmm", q, k, g, bits, f"qk {kname} {rname}", group_floor=True)     # previous floor: as routes


PV_KERNELS = {   # name: H (one KV unit), g, bits -- the tall instantiation <bits, H, g>
    "tall-2-1-32": (1, 32, 2),
    "tall-4-1-32": (1, 32, 4),
    "tall-2-1-64": (1, 64, 2),
    "tall-4-1-64": (1, 64, 4),
    "tall-2-2-64": (2, 64, 2),
    "tall-4-2-64": (2, 64, 4),
}
PV_REGIMES = {   # name: seed, logit std ("peaked": +12 on one token), V std, extras
    "unit": (1, 2.0, 1.0, {}),
    "flat": (2, 0.0, 1.0, {}),
    "logit-4": (3, 4.0, 1.0, {}),
    "peaked": (4, "peaked", 1.0, {}),
    "v-2^-6": (5, 2.0, 2.0 ** -6, {}),
    "v-0.02": (6, 2.0, 0.02, {}),
    "v-2^-10-flat": (7, 0.0, 2.0 ** -10, {}),
    "v-2^-10-logit-4": (8, 4.0, 2.0 ** -10, {}),
    "v-1e-4": (9, 2.0, 1e-4, {}),
    "v-1e-4-peaked": (10, "peaked", 1e-4, {}),
    "v-large": (11, 2.0, 3500.0, {}),                          # std 2000-5000, clipped finite
    "v-large-peaked": (12, "peaked", 2000.0, {}),
    "fA-not-prob": (13, None, 1.0, {}),                        # arbitrary fp16 x, max|x| > 32, small elements mixed in
    "v-inf-beside-large": (14, 2.0, 1.0, {"inf_beside_large": True}),   # channels 0-31 / 0-63: scale inf; 64-95: range 32000
}
PV_T = (600, 4096, 32768)
LONG_PV_REGIMES = list(PV_REGIMES)


def _pv_inputs(H, Tv, rname, N=128):
    seed, ls, vs, extra = PV_REGIMES[rname]
    rng = np.random.default_rng(seed * 7919 + Tv + H)
    v = np.clip(rng.standard_normal((1, 1, Tv, N)) * vs, -60000, 60000).astype(np.float16)
    if "inf_beside_large" in extra:
        v[..., 0], v[..., 1], v[..., 64], v[..., 65] = 60000.0, -60000.0, 16000.0, -16000.0
    if ls is None:
        x = rng.standard_normal((1, H, 1, Tv)) * 30.0
        x[..., ::2] *= 1e-5
        p = x.astype(np.float16)
    elif ls == "peaked":
        logits = rng.standard_normal((1, H, 1, Tv))
        logits[..., Tv // 3] += 12.0
        p = softmax16(logits)
    else:
        p = softmax16(rng.standard_normal((1, H, 1, Tv)) * ls)
    return p, v


def _pv_cases():
    return [pytest.param(k, r, T, id=f"{k}-{r}-T{T}") for T in PV_T for k in PV_KERNELS for r in PV_REGIMES]


@pytest.mark.parametrize("kname,rname,Tv", _pv_cases())
def test_pv_magnitude_sweep(kname, rname, Tv):
    H, g, bits = PV_KERNELS[kname]
    p, v = _pv_inputs(H, Tv, rname)
    # previous floor: the MMA kernels sum x*s*c and x*z apart
    checked_gemv("bmm", p, v, g, bits, f"pv {kname} {rname} T{Tv}", group_floor=True, strided_pad=3)


@pytest.mark.parametrize("kname", ["tall-2-2-64", "tall-4-2-64"])
@pytest.mark.parametrize("Tv", [4096, 32768])
@pytest.mark.parametrize("peaked_head", [0, 1])
def test_pv_mixed_heads(kname, Tv, peaked_head):
    """Two query heads in one CTA (G = 2) with different softmaxes over the same small V: one peaked (+12 on one token, a
    long low tail), one flat.  Each head's tiles must get the window they need, whatever the other head's."""
    H, g, bits = PV_KERNELS[kname]
    rng = np.random.default_rng(Tv + 31 * peaked_head + bits)
    v = (rng.standard_normal((1, 1, Tv, 128)) * 1e-4).astype(np.float16)
    logits = np.zeros((1, H, 1, Tv))
    logits[:, peaked_head] = rng.standard_normal(Tv)
    logits[:, peaked_head, :, Tv // 3] += 12.0
    checked_gemv("bmm", softmax16(logits), v, g, bits, f"pv mixed heads {kname} T{Tv} peaked {peaked_head}", strided_pad=3)


SIMT_PV = {   # name: H, Hkv, N, g, bits (N / g keep these off the tensor-core path)
    "simt-tall-G1-g128": (1, 1, 128, 128, 2),
    "simt-tall-G2-N64": (2, 1, 64, 32, 4),
}
SIMT_PV_REGIMES = ["unit", "peaked", "v-2^-10-logit-4", "v-1e-4-peaked", "v-large", "fA-not-prob"]


@pytest.mark.parametrize("kname", list(SIMT_PV))
@pytest.mark.parametrize("rname", SIMT_PV_REGIMES)
def test_pv_magnitude_sweep_simt(kname, rname):
    H, Hkv, N, g, bits = SIMT_PV[kname]
    p, v = _pv_inputs(H, 4096, rname, N)
    checked_gemv("bmm", p, v, g, bits, f"pv {kname} {rname}", strided_pad=3)


# ---------------------------------------------------------------------------------------------------
# edge rows as K and V groups
# ---------------------------------------------------------------------------------------------------
EDGE_KERNELS = {   # name: kind, B, H, Hkv, K, N, g, bits
    "wide-2-1-32": ("qk", 1, 2, 1, 128, 1024, 32, 2),
    "wide-4-2-64": ("qk", 1, 4, 1, 128, 1024, 64, 4),
    "simt-wide-G1": ("qk", 1, 1, 1, 128, 1024, 32, 4),
    "tall-2-1-32": ("pv", 1, 1, 1, 700, 128, 32, 2),
    "tall-4-2-64-S4": ("pv", 1, 2, 1, 4096, 128, 64, 4),
    "simt-tall-G1-g128": ("pv", 1, 1, 1, 700, 128, 128, 4),
}


@pytest.mark.parametrize("finite", [True, False], ids=["finite", "overflowing"])
@pytest.mark.parametrize("kname", list(EDGE_KERNELS))
def test_edge_groups(kname, finite):
    """K: chosen channels carry the edge rows along tokens (whole groups of 32 / 64).  V: every fifth token is two edge rows
    (the 128 channels).  The rows whose range overflows fp16 (finite=False) make scale = inf: the non-finite rule."""
    kind, B, H, Hkv, K, N, g, bits = EDGE_KERNELS[kname]
    rng = np.random.default_rng(len(kname) * 17 + finite)
    rows = edge_rows(bits, finite)
    w = rng.standard_normal((B, Hkv, K, N)).astype(np.float16)
    if kind == "qk":
        for e, row in enumerate(rows):
            w[:, :, 3 + 17 * e, :] = row[np.arange(N) % 64]
        fA = (rng.standard_normal((B, H, 1, K)) * 0.7).astype(np.float16)
    else:
        for t in range(2, K, 5):
            e = (t // 5) % len(rows)
            w[:, :, t, :] = np.concatenate([rows[e], rows[(e + 1) % len(rows)]])
        fA = softmax16(rng.standard_normal((B, H, 1, K)) * 2)
    checked_gemv("bmm", fA, w, g, bits, f"edges {kname} finite={finite}", strided_pad=3 if kind == "pv" else 0)

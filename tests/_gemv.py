"""The oracle check of every dequant-GEMV surface; imports without CUDA (kivi_b200 is imported inside the functions).

`exact` is the fp64 contraction of the oracle pack's codes, scale and zero, dequantised in fp64; `oracle` is the C oracle
(the reference kernel's fp32 order, fp16 output).  exact_bar: where the oracle's output is finite,
    |got - exact| <= |oracle - exact| + ulp16(exact) + FLOOR_COEF * l1,      ulp16(v) = 2^(floor(log2 max(|v|, 2^-14)) - 10)
with l1 = sum_k |x_k| * |w_kn|: one output rounding step plus the fp32 accumulation noise beyond the reference kernel;
elsewhere (a quantisation group whose range overflows fp16) the kernel's output must be non-finite too.  rtol_bar (rtol 1e-3
plus the same floor) is ill-posed in the fp16 subnormals, where one rounding step is far more than 1e-3 of the value; it is
kept where there is no exact result: the stored outputs of the unmodified reference extension, and the 8-bit surface."""
import numpy as np
import torch

from oracle import ref
from tests._util import to_np

RTOL, FLOOR_COEF = 1e-3, 1e-6      # BASELINE.json's "within 1e-3 rtol fp16"; the floor: a few fp32 ulps of the L1 mass
OUTLIER_CHANNELS = [5, 37, 77, 120]


def edge_rows(bits, finite):
    """The rows of test_pack_edge_values (64 values each: two groups of 32).  finite=False adds the rows whose group range
    overflows fp16 (large magnitudes, +-60000: the scale becomes inf)."""
    rng = np.random.default_rng(5)
    rows = [np.full(64, 1.25),                                                        # constant -> degenerate group
            np.zeros(64),
            np.concatenate([np.linspace(0, 3, 32), np.linspace(-7, 8, 32)]),         # ties / grid points
            rng.standard_normal(64) * 6e-6,                                           # fp16 subnormals
            np.arange(64) % (2 ** bits) * 0.5]                                        # exact levels
    if not finite:
        rows += [rng.standard_normal(64) * 2e4,
                 np.concatenate([[-60000.0, 60000.0], rng.standard_normal(62)])]
    return [r.astype(np.float16) for r in rows]


def kernel_layout_case(rng, B, nh, nh_kv, IC, OC):
    """x [B*nh,1,IC] and w [B*nh_kv,IC,OC], drawn as the reference's kernel-layout tests draw them (quant/gemv.py:93-165)."""
    x = rng.standard_normal((B * nh, 1, IC)).astype(np.float16)
    return x, rng.standard_normal((B * nh_kv, IC, OC)).astype(np.float16)


def kernel_layout(code, scale, mn):
    """The oracle pack [nkv, IC, *] of kernel-layout weights, transposed for the kernel: [nkv, *, IC] (quant/gemv.py:113)."""
    return [np.ascontiguousarray(a.transpose(0, 2, 1)) for a in (code, scale, mn)]


def reference_extension_inputs(bits):
    """test_against_reference_cuda_extension's seeded cases: shape, inp, the oracle pack and its kernel_layout."""
    rng = np.random.default_rng(1)
    for (B, nh, nh_kv, IC, OC, GS) in [(2, 8, 8, 739, 128, 32), (2, 8, 2, 128, 1024, 32), (1, 4, 1, 333, 128, 64)]:
        inp, w = kernel_layout_case(rng, B, nh, nh_kv, IC, OC)
        packed = ref.pack_lastdim(w, GS, bits)
        yield (B, nh, nh_kv, IC, OC, GS), inp, packed, kernel_layout(*packed)


def padded_rows(scale, mn, g):
    """scale / zero [OC, IC/g] in rows padded to 16 (g64) or 8 (g128) as the reference indexes them (gemv_cuda.cu:75,145)."""
    m = 16 if g == 64 else 8
    return [np.pad(a, ((0, 0), (0, -(-a.shape[1] // m) * m - a.shape[1]))) for a in (scale, mn)]


def dequant(code, scale, mn, g, bits):
    """fp64 s * c + z of an oracle pack along its last dim (a scale of inf times a zero code is NaN)."""
    c = ref.unpack_codes_lastdim(code, bits).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return c * np.repeat(scale.astype(np.float64), g, -1) + np.repeat(mn.astype(np.float64), g, -1)


def exact(fA, w):
    """fp64 sum_k x_k * w_kn: fA [B,H,1,K], dequantised w [B,Hkv,K,N] -> [B,H,1,N]; head h reads KV head h // (H / Hkv)."""
    B, H = fA.shape[:2]
    x = np.asarray(fA, np.float64)[:, :, 0].reshape(B, w.shape[1], H // w.shape[1], -1)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.einsum("bgrk,bgkn->bgrn", x, w).reshape(B, H, 1, -1)


def l1(fA, w):
    """sum_k |x_k| * |w_kn| per output, in fp64, for the operands of `exact`."""
    return exact(np.abs(np.asarray(fA, np.float64)), np.abs(w))


def ulp16(v):
    a = np.maximum(np.abs(np.asarray(v, np.float64)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


def _within(err, tol, what, detail=""):
    """err <= tol everywhere; returns the worst err / tol (a NaN bar rejects nothing and is left out)."""
    worst = float(np.nanmax(err / np.maximum(tol, 1e-30), initial=0.0))
    bad = err > tol
    assert not bad.any(), (f"{what}: {bad.sum()} / {bad.size} elements out of tolerance; max err {err.max():.3e}, "
                           f"worst ratio {worst:.2f}{detail}")
    return worst


def exact_bar(got, exact, oracle, l1, what):
    """The bar of the module docstring; returns the worst error / bar at the finite positions."""
    got, exact, oracle = (np.asarray(a, np.float64) for a in (got, exact, oracle))
    assert got.shape == exact.shape == oracle.shape, (what, got.shape, exact.shape, oracle.shape)
    fin = np.isfinite(oracle)
    bad_nf = np.isfinite(got) != fin
    assert not bad_nf.any(), (f"{what}: non-finite positions differ from the oracle's at {bad_nf.sum()} of {got.size} "
                              f"(kernel non-finite: {(~np.isfinite(got)).sum()}, oracle: {(~fin).sum()})")
    g, e, o, l = got[fin], exact[fin], oracle[fin], np.broadcast_to(np.asarray(l1, np.float64), got.shape)[fin]
    err, u = np.abs(g - e), ulp16(e)
    return _within(err, np.abs(o - e) + u + FLOOR_COEF * l, what, f"; worst {np.max(err / u, initial=0.0):.2f} ulp16 "
                   f"(oracle's own {np.max(np.abs(o - e) / u, initial=0.0):.2f})")


def rtol_bar(got, ref, l1, what=""):
    """|got - ref| <= RTOL * |ref| + FLOOR_COEF * l1 (l1 broadcastable); returns the worst error / bar."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return _within(np.abs(got - ref), RTOL * np.abs(ref) + FLOOR_COEF * np.asarray(l1, np.float64), what)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _meta_view(a, offset):
    """The same values in a view whose base sits `offset` fp16 elements into a row-padded buffer (row stride G + offset)."""
    t = torch.zeros(a.shape[:-1] + (a.shape[-1] + offset,), dtype=torch.float16, device="cuda")
    t[..., offset:] = _cuda(a)
    return t[..., offset:]


def run_bmm(fA, code, scale, mn, g, bits, strided_pad=0, meta_offset=0, triton=False):
    """cuda_bmm_fA_qB_outer (triton_bmm_fA_qB_outer if `triton`); fA as probs[..., :-strided_pad] of a longer row (the
    hook's view); with meta_offset > 0 scale / zero as views whose base is only (2 * meta_offset)-byte aligned."""
    from kivi_b200 import matmul
    fa_t = _cuda(np.concatenate([fA, np.ones(fA.shape[:-1] + (strided_pad,), np.float16)], -1))[..., :fA.shape[-1]]
    s_t, z_t = (_meta_view(a, meta_offset) if meta_offset else _cuda(a) for a in (scale, mn))
    f = matmul.triton_bmm_fA_qB_outer if triton else matmul.cuda_bmm_fA_qB_outer
    return to_np(f(g, fa_t, _cuda(code), s_t, z_t, bits))


def run_kernel_layout(x, code, scale, mn, g, bits, nh):
    """gemv_forward_cuda_outer_dim on x [B*nh,1,IC] and the oracle pack [B*nh_kv,IC,*] of w, transposed for the kernel."""
    from kivi_b200 import kivi_gemv
    args = map(_cuda, [x] + kernel_layout(code, scale, mn))
    return to_np(kivi_gemv.gemv_forward_cuda_outer_dim(*args, bits, g, nh, code.shape[0] * nh // x.shape[0]))


def run_inner(x, code, scale, mn, g, bits=4):
    """gemv_forward_cuda (4-bit, whatever `bits`) on x [Bn,IC] and the oracle pack of w [OC,IC], scale / zero in padded rows."""
    from kivi_b200 import kivi_gemv
    return to_np(kivi_gemv.gemv_forward_cuda(*map(_cuda, [x, code] + padded_rows(scale, mn, g)), 4, g))


def run_gemv_fwd(x, code, scale, mn, g, bits):
    """gemv_fwd on x [Bn,IC] and the oracle pack of w [OC,IC], scale / zero unpadded."""
    from kivi_b200 import gemv
    return to_np(gemv.gemv_fwd(bits, g, *map(_cuda, (x, code, mn, scale))))


def check_gemv(layout, got, fA, code, scale, mn, g, bits, what, nh=None, group_floor=False):
    """exact_bar on a surface's output `got` for input fA and the oracle pack code / scale / mn of w.  layout "bmm": fA
    [B,H,1,K], w [B,Hkv,K,N]; "kernel" (nh heads per sequence): fA [B*nh,1,IC], w [B*nh_kv,IC,OC]; "inner" (4-bit): fA
    [Bn,IC], w [OC,IC] -- these map onto "bmm" by a reshape / transpose.  group_floor ("bmm" only): the floor's mass is
    sum_k |x_k| * max_n (|s| * maxq + |z|), which bounds the noise of kernels that sum x*s*c and x*z apart where l1 does
    not.  Returns the oracle's output."""
    w = dequant(code, scale, mn, g, bits)
    if layout == "kernel":
        B = fA.shape[0] // nh
        oracle = ref.bgemv_outer_kernel_layout(fA, *kernel_layout(code, scale, mn), bits, g, nh, code.shape[0] // B)
        fA, w = fA.reshape(B, nh, 1, -1), w.reshape(B, -1, *w.shape[1:])
    elif layout == "inner":
        assert bits == 4, "the C oracle of the inner GEMV is 4-bit"
        oracle = ref.gemv_inner_w4(fA, code, *padded_rows(scale, mn, g), g)
        fA, w = fA[None, :, None, :], w.T[None, None]
    else:
        oracle = ref.bmm_fA_qB_outer(g, fA, code, scale, mn, bits)
    bound = (np.abs(scale.astype(np.float64)) * (2 ** bits - 1) + np.abs(mn.astype(np.float64))).max(-1, keepdims=True)
    mass = l1(fA, bound) if group_floor else l1(fA, w).reshape(oracle.shape)
    exact_bar(got, exact(fA, w).reshape(oracle.shape), oracle, mass, what)
    return oracle


def checked_gemv(surface, fA, w, g, bits, what, group_floor=False, **opts):
    """Pack w with the oracle, run `surface` ("bmm", "kernel", "inner" or "gemv_fwd", which has the inner layout) on fA with
    the runner's keywords `opts` and apply check_gemv.  Returns the kernel's and the oracle's output."""
    code, scale, mn = ref.pack_lastdim(w, g, bits)
    run = {"bmm": run_bmm, "kernel": run_kernel_layout, "inner": run_inner, "gemv_fwd": run_gemv_fwd}[surface]
    got = run(fA, code, scale, mn, g, bits, **opts)
    layout = "inner" if surface == "gemv_fwd" else surface
    return got, check_gemv(layout, got, fA, code, scale, mn, g, bits, what, opts.get("nh"), group_floor)

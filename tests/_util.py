"""Shared helpers for the parity tests."""
import hashlib

import numpy as np
import torch

# Tolerance of the floating-point parity tests (BASELINE.json north_star: "within 1e-3 rtol fp16").
# rtol alone is ill-posed for outputs that cancel to ~0 (the reference's own tests divide by |ref|+1e-5,
# quant/gemv.py:125), so the absolute floor is the fp32 accumulation-order noise of the contraction:
# FLOOR_COEF * sum_k |x_k| * max|dequantised weight|  (a few fp32 ulps of the L1 mass of the dot product).
RTOL = 1e-3
FLOOR_COEF = 1e-6


def to_np(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().numpy()


def assert_gemv_close(got, ref, l1_mass, what=""):
    """got/ref: arrays [..., N] (fp16); l1_mass: broadcastable upper bound of sum_k |x_k|*|w_kn|."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    tol = RTOL * np.abs(ref) + FLOOR_COEF * np.asarray(l1_mass, np.float64)
    err = np.abs(got - ref)
    bad = err > tol
    assert not bad.any(), (f"{what}: {bad.sum()} / {bad.size} elements out of tolerance; "
                           f"max err {err.max():.3e}, worst ratio {(err / np.maximum(tol, 1e-30)).max():.2f}")
    return float((err / (np.abs(ref) + 1e-5)).mean())          # the reference's printed metric


def l1_mass_ref_layout(fA, scales, zeros, maxq):
    """Upper bound of sum_k |x_k| * max_n |s*c+z| per (b, head): fA [B,H,1,K], scales/zeros [B,Hkv,K,G]."""
    x = np.abs(np.asarray(fA, np.float64))[:, :, 0, :]                                  # [B,H,K]
    w = (np.abs(np.asarray(scales, np.float64)) * maxq + np.abs(np.asarray(zeros, np.float64))).max(-1)  # [B,Hkv,K]
    rep = x.shape[1] // w.shape[1]
    w = np.repeat(w, rep, axis=1)
    return (x * w).sum(-1)[:, :, None, None]                                            # [B,H,1,1]


def rand_quantised(rng, shape_rows_T, g, bits):
    """Random fp16 data -> oracle pack (codes/scale/mn as numpy)."""
    from oracle import ref
    x = rng.standard_normal(shape_rows_T).astype(np.float16)
    return (x,) + ref.pack_lastdim(x, g, bits)


EXT_CASES = [(2, 8, 8, 739, 128, 32), (2, 8, 2, 128, 1024, 32), (1, 4, 1, 333, 128, 64)]   # (B, nh, nh_kv, IC, OC, GS)


def reference_extension_inputs(BIT):
    """The seeded inputs of test_against_reference_cuda_extension, case by case: the packed weights in the reference
    layout (code, scale, mn [nkv, IC, *]) and in the kernel layout (qw_t, sc_t, mn_t [nkv, *, IC])."""
    from oracle import ref
    rng = np.random.default_rng(1)
    for (B, nh, nh_kv, IC, OC, GS) in EXT_CASES:
        nkv = B * nh_kv
        inp = rng.standard_normal((B * nh, 1, IC)).astype(np.float16)
        w = rng.standard_normal((nkv, IC, OC)).astype(np.float16)
        code, scale, mn = ref.pack_lastdim(w, GS, BIT)
        kernel_layout = [np.ascontiguousarray(a.transpose(0, 2, 1)) for a in (code, scale, mn)]
        yield (B, nh, nh_kv, IC, OC, GS), inp, (code, scale, mn), kernel_layout


def input_digest(*arrays):
    return hashlib.sha256(b"".join(np.ascontiguousarray(a).tobytes() for a in arrays)).digest()

"""Parity of the CUDA dequant-GEMVs (kivi_bgemv.cu through the C ABI / Python surface) with the oracle
(reference summation order, oracle/kivi_oracle.c) and with the stored outputs of the UNMODIFIED reference CUDA
extension on the same inputs.  Check and bars: tests/_gemv.py."""
import os

import numpy as np
import pytest
import torch

from oracle import ref
from tests._gemv import (check_gemv, checked_gemv, dequant, exact, kernel_layout_case, l1, reference_extension_inputs,
                         rtol_bar, run_bmm, run_kernel_layout)
from tests._util import input_digest, to_np

pytestmark = pytest.mark.gpu


QK_CASES = [  # (B, H, Hkv, D, Tk, g, bits)
    (2, 4, 4, 128, 128, 32, 2),
    (2, 4, 4, 128, 1024, 32, 2),
    (1, 8, 8, 128, 3968, 32, 2),      # cfg 2 token count at T=4096
    (2, 8, 2, 128, 1152, 32, 2),      # GQA ratio 4
    (1, 8, 1, 128, 640, 32, 2),       # MQA ratio 8 (two chunks of 4)
    (1, 6, 2, 128, 384, 32, 2),       # ratio 3 -> G = 1
    (1, 4, 2, 128, 2176, 64, 4),      # cfg 4 style: 4-bit g64, ratio 2
    (2, 2, 2, 128, 512, 128, 4),
    (1, 2, 2, 64, 320, 32, 2),        # head_dim 64
    (1, 2, 2, 200, 256, 64, 2),       # K not a multiple of anything nice
]


@pytest.mark.parametrize("B,H,Hkv,D,Tk,g,bits", QK_CASES)
def test_qk_shape_matches_oracle(B, H, Hkv, D, Tk, g, bits):
    """q.K^T shape of cuda_bmm_fA_qB_outer (models/llama_kivi.py:324-325): K = head_dim, N = Tk."""
    rng = np.random.default_rng(Tk * 7 + H)
    k = rng.standard_normal((B, Hkv, D, Tk)).astype(np.float16)
    q = rng.standard_normal((B, H, 1, D)).astype(np.float16)
    got, _ = checked_gemv("bmm", q, k, g, bits, f"qk {B,H,Hkv,D,Tk,g,bits}")
    assert got.shape == (B, H, 1, Tk)


SV_CASES = [  # (B, H, Hkv, Tv, D, g, bits)
    (2, 4, 4, 1, 128, 32, 2),
    (2, 4, 4, 7, 128, 32, 2),
    (1, 8, 8, 333, 128, 32, 2),
    (1, 4, 4, 3967, 128, 32, 2),      # cfg 2 at T=4096
    (2, 8, 2, 1000, 128, 32, 2),      # GQA 4
    (1, 8, 1, 129, 128, 32, 2),       # MQA 8
    (1, 4, 2, 2048, 128, 64, 4),      # 4-bit g64
    (1, 2, 2, 100, 64, 32, 2),        # head_dim 64
    (1, 2, 2, 50, 256, 128, 4),       # head_dim 256
    (1, 3, 3, 77, 96, 32, 2),         # N = 96 (3 cells)
]


@pytest.mark.parametrize("B,H,Hkv,Tv,D,g,bits", SV_CASES)
def test_sv_shape_matches_oracle(B, H, Hkv, Tv, D, g, bits):
    """p.V shape (models/llama_kivi.py:382-383): K = Tv, N = head_dim, fA = a strided slice of the probs."""
    rng = np.random.default_rng(Tv * 3 + H)
    v = rng.standard_normal((B, Hkv, Tv, D)).astype(np.float16)
    L = 5
    logits = rng.standard_normal((B, H, 1, Tv + L)).astype(np.float32) * 2
    p = (np.exp(logits) / np.exp(logits).sum(-1, keepdims=True)).astype(np.float16)
    # previous floor: the MMA kernels sum x*s*c and x*z apart
    checked_gemv("bmm", p[..., :-L], v, g, bits, f"sv {B,H,Hkv,Tv,D,g,bits}", group_floor=True, strided_pad=L)


@pytest.mark.parametrize("bits,g,N", [(2, 16, 48), (2, 48, 96), (4, 8, 40), (4, 24, 48), (8, 64, 128), (8, 4, 20)])
def test_generic_group_sizes(bits, g, N):
    """Every group_size % fpi == 0 the reference kernel accepts (gemv_cuda.cu:357) plus the 8-bit Triton surface."""
    rng = np.random.default_rng(bits * 1000 + g)
    B, H, Hkv, K = 2, 4, 2, 50
    w = rng.standard_normal((B, Hkv, K, N)).astype(np.float16)
    x = rng.standard_normal((B, H, 1, K)).astype(np.float16)
    if bits != 8:
        checked_gemv("bmm", x, w, g, bits, "generic g")
    else:                           # the C oracle covers bits 2 / 4 only: against the fp16-rounded exact result
        code, scale, mn = ref.pack_lastdim(w, g, bits)
        wd = dequant(code, scale, mn, g, bits)
        rtol_bar(run_bmm(x, code, scale, mn, g, bits, triton=True), exact(x, wd).astype(np.float16), l1(x, wd), "generic g")


@pytest.mark.parametrize("BIT", [2, 4])
@pytest.mark.parametrize("mqa", [False, True])
def test_kernel_layout_reference_test_case(BIT, mqa):
    """The reference's own pinned case: B, nh, IC, OC = 8, 32, 739, 128, g32, seeds 0 (quant/gemv.py:14,
    :93-165, :270-276) through the `kivi_gemv` module surface; IC = 739 exercises the tail masks."""
    B, nh, IC, OC, GS = 8, 32, 739, 128, 32
    nh_kv = 1 if mqa else nh                                          # (the script's stale `False` would divide by 0)
    x, w = kernel_layout_case(np.random.default_rng(0), B, nh, nh_kv, IC, OC)
    got, oracle = (a.astype(np.float64) for a in checked_gemv("kernel", x, w, GS, BIT, f"kernel layout b{BIT} mqa {mqa}", nh=nh))
    assert (np.abs(got - oracle) / (np.abs(oracle) + 1e-5)).mean() < 1e-4    # the reference's printed metric (quant/gemv.py:125)


@pytest.mark.parametrize("BIT", [2, 4])
def test_against_reference_cuda_extension(BIT, golden_dir):
    """Kernel-vs-kernel (the only place the 1e-3 rtol bar is meaningful, SURVEY section 4): our library and the
    oracle against the outputs of the UNMODIFIED reference extension (gemv_forward_cuda_outer_dim) on the same seeded
    inputs, stored in tests/golden/reference_ext_gemv.npz by tests/golden/make_golden_ext.py.  Each of our kernels is also
    held to the exact result (the oracle being the stored output)."""
    gold = np.load(os.path.join(golden_dir, "reference_ext_gemv.npz"))
    for i, ((B, nh, nh_kv, IC, OC, GS), inp, (code, scale, mn), _) in enumerate(reference_extension_inputs(BIT)):
        assert input_digest(inp, code, scale, mn) == bytes(gold[f"digest_b{BIT}_{i}"]), "inputs differ from the stored run's"
        ref_out = gold[f"out_b{BIT}_{i}"]
        ours_k = run_kernel_layout(inp, code, scale, mn, GS, BIT, nh)
        orc = check_gemv("kernel", ours_k, inp, code, scale, mn, GS, BIT, "kernel layout vs exact", nh=nh)
        # (1) the C oracle reproduces the reference kernel BIT FOR BIT (same order, fmaf contraction)
        np.testing.assert_array_equal(orc.view(np.uint16), ref_out.view(np.uint16))
        # (2) our kernels, both layouts, against the reference kernel
        x, ref_layout = inp.reshape(B, nh, 1, IC), [a.reshape(B, nh_kv, IC, -1) for a in (code, scale, mn)]
        mass = l1(x, dequant(*ref_layout, GS, BIT)).reshape(B * nh, 1, OC)
        rtol_bar(ours_k, ref_out, mass, "kernel layout vs reference ext")
        ours_r = run_bmm(x, *ref_layout, GS, BIT)
        rtol_bar(ours_r.reshape(B * nh, 1, OC), ref_out, mass, "reference layout vs reference ext")
        check_gemv("bmm", ours_r, x, *ref_layout, GS, BIT, "reference layout vs exact")


@pytest.mark.parametrize("g", [64, 128])
def test_inner_gemv_matches_oracle(g):
    """gemv_forward_cuda (quant/csrc/gemv_cuda.cu:201-246): 4-bit inner-dim GEMV with padded scale rows."""
    rng = np.random.default_rng(g)
    Bn, IC, OC = 8, 1024, 128
    x = rng.standard_normal((Bn, IC)).astype(np.float16)
    w = rng.standard_normal((OC, IC)).astype(np.float16)
    checked_gemv("inner", x, w, g, 4, f"inner g{g}")


def test_gemv_fwd_surface():
    """gemv_fwd (quant/gemv.py:77-90) with unpadded [OC, IC/g] scale/mn, against the oracle of the inner GEMV."""
    from kivi_b200 import gemv
    rng = np.random.default_rng(3)
    Bn, IC, OC, g, bit = 4, 512, 64, 64, 4
    x = rng.standard_normal((Bn, IC)).astype(np.float16)
    w = rng.standard_normal((OC, IC)).astype(np.float16)
    checked_gemv("gemv_fwd", x, w, g, bit, "gemv_fwd")
    code, scale, mn = ref.pack_lastdim(w, g, bit)
    deq = gemv.dequant_weight(torch.from_numpy(ref.unpack_codes_lastdim(code, bit)).cuda(), torch.from_numpy(scale).cuda(),
                              torch.from_numpy(mn).cuda(), g)
    np.testing.assert_array_equal(to_np(deq).view(np.uint16), ref.unpack_dequant_lastdim(code, scale, mn, g, bit).view(np.uint16))


def test_argument_errors():
    from kivi_b200 import _lib, matmul
    q = torch.zeros((1, 3, 1, 128), dtype=torch.float16, device="cuda")
    code = torch.zeros((1, 2, 128, 8), dtype=torch.int32, device="cuda")
    sc = torch.zeros((1, 2, 128, 4), dtype=torch.float16, device="cuda")
    with pytest.raises(AssertionError):                              # nh % nh_kv (quant/matmul.py:216)
        matmul.cuda_bmm_fA_qB_outer(32, q, code, sc, sc, 2)
    with pytest.raises(AssertionError):                              # bits (quant/matmul.py:215)
        matmul.cuda_bmm_fA_qB_outer(32, q[:, :2], code, sc, sc, 3)
    L = _lib.lib()
    assert L.kivi_bgemv_outer_f16(q.data_ptr(), 128, code.data_ptr(), 1024, 8, sc.data_ptr(), sc.data_ptr(), 512, 4,
                                  q.data_ptr(), 1, 2, 2, 128, 128, 2, 24, 0, None) == -4      # KIVI_ERR_GROUP
    assert L.kivi_bgemv_outer_f16(q.data_ptr(), 128, code.data_ptr(), 1024, 8, sc.data_ptr(), sc.data_ptr(), 512, 4,
                                  q.data_ptr(), 1, 2, 2, 128, 128, 2, 32, 7, None) == -7      # KIVI_ERR_LAYOUT
    assert L.kivi_bgemv_outer_f16(None, 128, code.data_ptr(), 1024, 8, sc.data_ptr(), sc.data_ptr(), 512, 4,
                                  q.data_ptr(), 1, 2, 2, 128, 128, 2, 32, 0, None) == -6      # KIVI_ERR_NULL


@pytest.mark.parametrize("kind", ["qk", "sv"])
def test_full_size_linearity(kind):
    """BASELINE cfg 2 per-layer sizes (B32 H32 T=4096: Tk=3968 / Tv=3967) -- too big for the CPU oracle, so
    parity is checked through size-independent properties: linearity in the fp16 input (x and 2x give
    exactly 2x outputs barring overflow: scaling by 2 is exact in every fp32 step) and agreement with
    the oracle on a slab of units."""
    from kivi_b200 import matmul, new_pack
    gen = torch.Generator(device="cuda").manual_seed(0)
    B, H, D, g, bits = 32, 32, 128, 32, 2
    if kind == "qk":
        T = 3968
        kT = torch.randn((B, H, D, T), generator=gen, device="cuda", dtype=torch.float16)
        code, scale, mn = new_pack.triton_quantize_and_pack_along_last_dim(kT, g, bits)
        del kT
        x = torch.randn((B, H, 1, D), generator=gen, device="cuda", dtype=torch.float16)
    else:
        T = 3967
        v = torch.randn((B, H, T, D), generator=gen, device="cuda", dtype=torch.float16)
        code, scale, mn = new_pack.triton_quantize_and_pack_along_last_dim(v, g, bits)
        del v
        x = torch.softmax(torch.randn((B, H, 1, T), generator=gen, device="cuda") * 2, -1).half()
    y1 = matmul.cuda_bmm_fA_qB_outer(g, x, code, scale, mn, bits)
    y2 = matmul.cuda_bmm_fA_qB_outer(g, x * 2, code, scale, mn, bits)
    normal = y1.abs() >= 1e-4                                         # fp16 subnormals do not scale exactly
    assert torch.equal(y2.float()[normal], y1.float()[normal] * 2)
    assert bool(((y2.float() - 2 * y1.float()).abs() <= 2.0 ** -23).all())
    sl = slice(5, 7)
    slab = (to_np(t[sl, :4]) for t in (y1, x, code, scale, mn))
    # previous floor: the MMA kernels sum x*s*c and x*z apart
    check_gemv("bmm", *slab, g, bits, f"full-size {kind} slab", group_floor=True)

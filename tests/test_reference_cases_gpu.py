"""The reference's own pinned test cases (SURVEY section 4): the seeds / shapes / bit widths of quant/test.py, run
through this package's public surface (the names the reference's script imports) and ASSERTED, where the reference
only prints a mean relative error.  quant/gemv.py's cases live in tests/test_bgemv_gpu.py."""
import math

import numpy as np
import pytest
import torch

from oracle import ref, torch_ref
from tests._gemv import check_gemv
from tests._util import to_np

pytestmark = pytest.mark.gpu


def _roundtrip_bound(x, deq, scale_g, group_size, bits):
    """|dequant - x| <= scale/2 (rounding of the code) + the fp16 roundings of the chain (x - mn, / scale, code * scale,
    + mn: four roundings of quantities bounded by the group's range + |x|), per element; mean error ~ scale/4."""
    s = scale_g.float().repeat_interleave(group_size, dim=-1)
    err = (deq.float() - x.float()).abs()
    tol = 0.5 * s + 2.0 ** -9 * (s * (2 ** bits - 1) + x.float().abs()) + 1e-6
    worst = float((err - tol).max())
    mean_ok = float(err.mean()) <= 0.3 * float(s.mean()) + 2.0 ** -9 * float(x.float().abs().mean() + (s * (2 ** bits - 1)).mean())
    return bool((err <= tol).all()) and mean_ok, worst


@pytest.mark.parametrize("bits", [2, 4, 8])
def test_vcache_roundtrip_reference_case(bits):
    """quant/test.py:21-36 `test_vcache`: seed 0, v [555, 32, 433, 128] (T = 433 is deliberately odd), g 64, bits
    {2, 4, 8}; pack along channels then unpack_and_dequant_vcache.  The reference asserts "no NaN" and prints
    mean |gap / v|; here additionally: codes / scale / mn equal the reference's ATen chain on this GPU bit for bit
    (oracle/torch_ref.py) and the round-trip error respects the half-step bound."""
    from quant.new_pack import triton_quantize_and_pack_along_last_dim, unpack_and_dequant_vcache
    torch.manual_seed(0)
    B, nh, T, hd = 555, 32, 433, 128
    group_size = 64
    v = torch.randn((B, nh, T, hd), device="cuda", dtype=torch.float16)
    code, scale, mn = triton_quantize_and_pack_along_last_dim(v, group_size, bits)
    assert code.shape == (B, nh, T, hd * bits // 32) and scale.shape == mn.shape == (B, nh, T, hd // group_size)
    ec, es, em = torch_ref.pack_lastdim(v, group_size, bits)
    assert torch.equal(code, ec) and torch.equal(scale.view(torch.int16), es.view(torch.int16))
    assert torch.equal(mn.view(torch.int16), em.view(torch.int16))
    del ec, es, em
    deq = unpack_and_dequant_vcache(code, scale.unsqueeze(-1), mn.unsqueeze(-1), group_size, bits)
    assert not bool(deq.isnan().any())                                              # :33
    ok, worst = _roundtrip_bound(v, deq, scale, group_size, bits)
    assert ok, worst
    gap = torch.nan_to_num((deq - v) / v)                                            # :34-36, the printed metric
    assert math.isfinite(float(gap.float().abs().mean()))


@pytest.mark.parametrize("bits", [2, 4, 8])
def test_kcache_roundtrip_reference_case(bits):
    """quant/test.py:39-54 `test_kcache`: seed 0, k [11, 32, 4096, 128] packed per channel along tokens
    (k.transpose(2, 3).contiguous()), g 64, bits {2, 4, 8}."""
    from quant.new_pack import triton_quantize_and_pack_along_last_dim, unpack_and_dequant_vcache
    torch.manual_seed(0)
    BS, nh, T, D = 11, 32, 4096, 128
    group_size = 64
    k = torch.randn((BS, nh, T, D), device="cuda", dtype=torch.float16)
    kt = k.transpose(2, 3).contiguous()
    code, scale, mn = triton_quantize_and_pack_along_last_dim(kt, group_size, bits)
    ec, es, em = torch_ref.pack_lastdim(kt, group_size, bits)
    assert torch.equal(code, ec) and torch.equal(scale.view(torch.int16), es.view(torch.int16))
    assert torch.equal(mn.view(torch.int16), em.view(torch.int16))
    del ec, es, em
    deq = unpack_and_dequant_vcache(code, scale.unsqueeze(-1), mn.unsqueeze(-1), group_size, bits)
    assert not bool(deq.isnan().any())                                              # :51
    ok, worst = _roundtrip_bound(kt, deq, scale, group_size, bits)
    assert ok, worst
    # a slab through the C oracle as well (pack + the reference's fp16 dequant, bit for bit)
    sl = to_np(kt[3:4, 5:7])
    oc, os_, om = ref.pack_lastdim(sl, group_size, bits)
    np.testing.assert_array_equal(to_np(code[3:4, 5:7]), oc)
    np.testing.assert_array_equal(to_np(scale[3:4, 5:7]).view(np.uint16), os_.view(np.uint16))
    np.testing.assert_array_equal(to_np(deq[3:4, 5:7]).view(np.uint16),
                                  ref.unpack_dequant_lastdim(oc, os_, om, group_size, bits).view(np.uint16))


@pytest.mark.parametrize("bits", [8, 4, 2])
def test_4d_qmatmul_reference_case(bits):
    """quant/test.py:173-202 `test_4d_qmatmul`: seed 0, integer-valued k = randint(10) [16, 32, 1024, 128] and
    q = randint(5), g 64; quant_and_pack_kcache -> transpose to the "trans" layout (:190-193) -> q.K^T through
    triton_bmm_fA_qB_outer, against torch.matmul on the unquantised k.  Asserted: no NaN (:197-198); the kernel equals
    the fp32 evaluation of sum q*(s*c+z) on its own packed operands (1e-3 rtol + floor) on ALL units, the exact bar of
    tests/_gemv.py on a slab; and the distance to the unquantised matmul stays within the quantisation step."""
    from quant.matmul import triton_bmm_fA_qB_outer
    from quant.new_pack import quant_and_pack_kcache, unpack_and_dequant_kcache
    torch.manual_seed(0)
    BS, nh, T, D = 16, 32, 1024, 128
    group_size = 64
    k = torch.randint(10, (BS, nh, T, D), device="cuda").to(torch.float16)
    query_state = torch.randint(5, (BS, nh, 1, D), device="cuda").to(torch.float16)
    code, scale, mn = quant_and_pack_kcache(k, group_size, bits)                       # :187
    dequant_k = unpack_and_dequant_kcache(code, scale, mn, group_size, bits)           # :188
    code_t = code.transpose(2, 3)                                                      # :190
    scale_t = scale.view(BS, nh, -1, D).transpose(2, 3)                                # :192
    mn_t = mn.view(BS, nh, -1, D).transpose(2, 3)                                      # :193
    our_out = triton_bmm_fA_qB_outer(group_size, query_state, code_t, scale_t, mn_t, bits)
    ref_out = torch.matmul(query_state, k.transpose(2, 3))
    assert not bool(our_out.isnan().any()) and not bool(ref_out.isnan().any())       # :197-198
    # fp32 evaluation on the packed operands, on the device: the only check of all 16 x 32 units (too many for the C oracle)
    fpi = 32 // bits
    shifts = torch.arange(fpi, device="cuda", dtype=torch.int32) * bits
    c = ((code.unsqueeze(3) >> shifts.view(1, 1, 1, fpi, 1)) & (2 ** bits - 1)).reshape(BS, nh, T, D).float()
    s = scale.view(BS, nh, T // group_size, D).float().repeat_interleave(group_size, dim=2)
    z = mn.view(BS, nh, T // group_size, D).float().repeat_interleave(group_size, dim=2)
    w = s * c + z                                                                      # [BS, nh, T, D]
    exact = torch.einsum("bhd,bhtd->bht", query_state[:, :, 0].double(), w.double())
    l1 = torch.einsum("bhd,bhtd->bht", query_state[:, :, 0].double().abs(), w.double().abs())
    err = (our_out[:, :, 0].double() - exact).abs()
    assert bool((err <= 1e-3 * exact.abs() + 1e-6 * l1 + 2 ** -11 * exact.abs()).all()), float(err.max())
    if bits != 8:                    # the C oracle of the reference kernel (the same sum, fp32 accumulate) on a slab
        sb = slice(4, 5)
        slab = (to_np(t[sb, :2].contiguous()) for t in (our_out, query_state, code_t, scale_t, mn_t))
        check_gemv("bmm", *slab, group_size, bits, "4d qmatmul slab")
    # the printed metric (:199-202): relative gap to the unquantised product, bounded by the step size
    gap = torch.nan_to_num((our_out - ref_out) / ref_out)
    assert float(gap.float().abs().mean()) < {8: 0.01, 4: 0.05, 2: 0.3}[bits]
    assert bool(((dequant_k.float() - k.float()).abs() <= 0.5 * 9 / (2 ** bits - 1) + 0.02).all())


def test_streaming_kvcache_reference_case():
    """quant/test.py:125-170 `test_streaming_kvcache`: [1, 32, 340, 128], g 64, 2-bit, 16 decode steps of the test's
    own streaming policy (K: the first 320 tokens packed per channel, the rest + every new token in fp16; V: every
    token packed per token as it arrives; the query of step i > 0 is the previous output).  Each step is compared with
    (a) the same flow evaluated by the C oracle on the same inputs (kernel parity), (b) fp16 attention on the
    unquantised tensors, as the reference prints (bounded here)."""
    from quant.matmul import triton_bmm_fA_qB_outer
    from quant.new_pack import triton_quantize_and_pack_along_last_dim
    torch.manual_seed(114514)                                                         # :206
    BS, nh, T, D = 1, 32, 340, 128
    group_size, bits = 64, 2
    key_states = torch.randn((BS, nh, T, D), device="cuda", dtype=torch.float16)
    value_states = torch.randn((BS, nh, T, D), device="cuda", dtype=torch.float16)
    nq = T - T % group_size
    key_q, key_full = key_states[:, :, :nq].contiguous(), key_states[:, :, nq:].contiguous()
    # the reference packs all 340 V tokens along channels (last dim 128): legal, T is not the packed axis
    v_code, v_scale, v_mn = triton_quantize_and_pack_along_last_dim(value_states, group_size, bits)
    k_code, k_scale, k_mn = triton_quantize_and_pack_along_last_dim(key_q.transpose(2, 3).contiguous(), group_size, bits)
    out = None
    for i in range(16):
        q = torch.randn((BS, nh, 1, D), device="cuda", dtype=torch.float16) if out is None else out
        k_new = torch.randn((BS, nh, 1, D), device="cuda", dtype=torch.float16)
        v_new = torch.randn((BS, nh, 1, D), device="cuda", dtype=torch.float16)
        att_q = triton_bmm_fA_qB_outer(group_size, q, k_code, k_scale, k_mn, bits)
        key_full = torch.cat([key_full, k_new], dim=2)
        att_f = torch.matmul(q, key_full.transpose(2, 3))
        w = torch.softmax(torch.cat([att_q, att_f], dim=-1) / math.sqrt(D), dim=-1)
        c, s, m = triton_quantize_and_pack_along_last_dim(v_new, group_size, bits)
        v_code, v_scale, v_mn = torch.cat([v_code, c], 2), torch.cat([v_scale, s], 2), torch.cat([v_mn, m], 2)
        out = triton_bmm_fA_qB_outer(group_size, w, v_code, v_scale, v_mn, bits)
        # (a) oracle on the same operands
        check_gemv("bmm", to_np(att_q), *map(to_np, (q, k_code, k_scale, k_mn)), group_size, bits, f"step {i} q.K^T")
        check_gemv("bmm", to_np(out), *map(to_np, (w, v_code, v_scale, v_mn)), group_size, bits, f"step {i} p.V")
        ec, es, em = ref.pack_lastdim(to_np(v_new), group_size, bits)
        np.testing.assert_array_equal(to_np(c), ec)
        # (b) against fp16 attention on the unquantised tensors
        key_states = torch.cat([key_states, k_new], dim=2)
        value_states = torch.cat([value_states, v_new], dim=2)
        rw = torch.softmax(torch.matmul(q, key_states.transpose(2, 3)) / math.sqrt(D), dim=-1)
        ro = torch.matmul(rw, value_states)
        assert not bool(out.isnan().any())
        assert float((rw.float() - w.float()).abs().sum(-1).max()) < 1.0              # total-variation of the weights
        assert float((ro.float() - out.float()).abs().mean()) < 0.25

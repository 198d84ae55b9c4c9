"""Drop-in surface of the reference's quant/matmul.py, backed by libkivi_b200 (sm_90a CUDA)."""
from __future__ import annotations

import torch

from . import _lib

KIVI_LAYOUT_REFERENCE = 0
KIVI_LAYOUT_KERNEL = 1


def _uniform_rows(t: torch.Tensor):
    """Return (tensor, unit_stride, row_stride) for a [B, H, R, C] tensor whose (B, H) dims collapse to
    one uniform stride and whose last dim is contiguous; copy only when the view cannot be expressed."""
    B, H, R, C = t.shape
    ok = (t.stride(3) == 1 or C == 1) and (B == 1 or t.stride(0) == H * t.stride(1))
    if not ok:
        t = t.contiguous()
    return t, t.stride(1), t.stride(2)


def _bmm_outer(group_size, fA, qB, scales, zeros, bits, fn_name):
    assert len(fA.shape) == 4 and len(qB.shape) == 4             # quant/matmul.py:198
    _lib.require_cuda(fA, qB, scales, zeros)
    assert fA.dtype == torch.float16 and scales.dtype == torch.float16 and zeros.dtype == torch.float16
    assert qB.dtype == torch.int32
    B, nh, M, K = fA.shape
    nh_kv = qB.shape[1]                                          # :200
    feat_per_int = 32 // bits
    N = qB.shape[-1] * feat_per_int                              # :204
    assert nh % nh_kv == 0                                       # :216
    if M != 1:
        raise NotImplementedError("only M == 1 (decode) is supported, as in the reference kernel "
                                  "(quant/csrc/gemv_cuda.cu:538 ignores blockIdx.z)")
    fA, a_us, _ = _uniform_rows(fA)
    qB, qb_us, qb_rs = _uniform_rows(qB)
    scales, s_us, s_rs = _uniform_rows(scales)
    zeros, z_us, z_rs = _uniform_rows(zeros)
    if (z_us, z_rs) != (s_us, s_rs):
        zeros = zeros.contiguous()
        scales = scales.contiguous()
        s_us, s_rs = scales.stride(1), scales.stride(2)
    c = torch.empty((B, nh, 1, N), device=fA.device, dtype=torch.float16)
    with torch.cuda.device(fA.device):
        _lib.check(_lib.lib().kivi_bgemv_outer_f16(
            fA.data_ptr(), a_us, qB.data_ptr(), qb_us, qb_rs, scales.data_ptr(), zeros.data_ptr(), s_us, s_rs,
            c.data_ptr(), B, nh, nh_kv, K, N, bits, group_size, KIVI_LAYOUT_REFERENCE, _lib.stream_ptr(fA.device)),
            fn_name)
    return c


def cuda_bmm_fA_qB_outer(group_size: int, fA: torch.Tensor, qB: torch.Tensor, scales: torch.Tensor,
                         zeros: torch.Tensor, bits: int) -> torch.Tensor:
    """quant/matmul.py:178-219.  C = fA @ dequant(qB), packing/groups along the last dim of qB.

    fA (B, nh, 1, K) fp16; qB (B, nh_kv, K, N // feat_per_int) int32; scales, zeros (B, nh_kv, K, N // group_size)
    fp16.  Returns (B, nh, 1, N) fp16.  Unlike the reference wrapper no operand is transposed or copied
    (its :205,213-214 re-layout is gone): the kernel reads the cache layout directly, strided views
    (e.g. attn_weights[..., :-L], models/llama_kivi.py:382) included."""
    assert bits in [2, 4]                                        # :215
    return _bmm_outer(group_size, fA, qB, scales, zeros, bits, "cuda_bmm_fA_qB_outer")


def triton_bmm_fA_qB_outer(group_size: int, fA: torch.Tensor, qB: torch.Tensor, scales: torch.Tensor,
                           zeros: torch.Tensor, bits: int) -> torch.Tensor:
    """quant/matmul.py:112-175 (Triton qbvm_kernel :9-93).  Same contraction on the same layout; the
    name is kept for the reference's test scripts (quant/test.py:85,147,194).  8-bit is accepted like
    the Triton original; its `N % 64`, `group_size % 64`, no-GQA restrictions (:142-145) are lifted."""
    assert bits in [2, 4, 8]
    return _bmm_outer(group_size, fA, qB, scales, zeros, bits, "triton_bmm_fA_qB_outer")

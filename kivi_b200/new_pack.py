"""Drop-in surface of the reference's quant/new_pack.py, backed by libkivi_b200 (sm_90a CUDA).

Same names, argument order, return shapes/dtypes and assert behaviour as the reference
(jy-yuan/KIVI quant/new_pack.py).  All functions require CUDA tensors.
"""
from __future__ import annotations

import torch

from . import _lib


def _pack_lastdim(data: torch.Tensor, group_size: int, bit: int):
    """data [..., T] fp16 -> code [..., T/fpi] int32, scale/mn [..., T/g] fp16 (one fused kernel)."""
    _lib.require_cuda(data)
    assert data.dtype == torch.float16, "KIVI pack operates on fp16 tensors"
    T = data.shape[-1]
    assert T % group_size == 0                                   # quant/new_pack.py:222
    fpi = 32 // bit
    data = data.contiguous()
    rows = data.numel() // T if T > 0 else 0
    code = torch.empty(data.shape[:-1] + (T // fpi,), dtype=torch.int32, device=data.device)
    scale = torch.empty(data.shape[:-1] + (T // group_size,), dtype=torch.float16, device=data.device)
    mn = torch.empty_like(scale)
    with torch.cuda.device(data.device):
        _lib.check(_lib.lib().kivi_pack_lastdim_f16(data.data_ptr(), rows, T, group_size, bit, code.data_ptr(),
                                                     scale.data_ptr(), mn.data_ptr(), _lib.stream_ptr(data.device)),
                   "kivi_pack_lastdim_f16")
    return code, scale, mn


def triton_quantize_and_pack_along_last_dim(data: torch.Tensor, group_size: int, bit: int):
    """quant/new_pack.py:217-252.  data [B, nh, D, T] fp16 -> (code [B,nh,D,T/fpi] int32,
    scale [B,nh,D,T/g] fp16, mn [B,nh,D,T/g] fp16).  The name is kept for drop-in compatibility;
    the implementation is one hand-written CUDA kernel (kivi_pack.cu), not Triton."""
    assert len(data.shape) == 4                                  # :218
    return _pack_lastdim(data, group_size, bit)


quantize_and_pack_along_last_dim = triton_quantize_and_pack_along_last_dim


def quant_and_pack_kcache(k: torch.Tensor, group_size: int, bits: int):
    """quant/new_pack.py:8-27.  k [B,nh,T,D] -> code [B,nh,T/fpi,D], scale/mn [B,nh,T/g,1,D]."""
    assert len(k.shape) == 4
    B, nh, T, D = k.shape
    assert T % group_size == 0                                   # :13
    code, scale, mn = _pack_lastdim(k.transpose(2, 3), group_size, bits)
    return (code.transpose(2, 3).contiguous(), scale.transpose(2, 3).unsqueeze(-2).contiguous(),
            mn.transpose(2, 3).unsqueeze(-2).contiguous())


def quant_and_pack_vcache(v: torch.Tensor, group_size: int, bits: int):
    """quant/new_pack.py:30-48.  v [B,nh,T,D] -> code [B,nh,T,D/fpi], scale/mn [B,nh,T,D/g,1]."""
    assert len(v.shape) == 4
    assert v.shape[-1] % group_size == 0                         # :33
    code, scale, mn = _pack_lastdim(v, group_size, bits)
    return code, scale.unsqueeze(-1), mn.unsqueeze(-1)


def _unpack_dequant_lastdim(code: torch.Tensor, scale: torch.Tensor, mn: torch.Tensor, group_size: int, bits: int):
    _lib.require_cuda(code, scale, mn)
    fpi = 32 // bits
    code, scale, mn = code.contiguous(), scale.contiguous(), mn.contiguous()
    T = code.shape[-1] * fpi
    rows = code.numel() // code.shape[-1] if code.shape[-1] > 0 else 0
    out = torch.empty(code.shape[:-1] + (T,), dtype=torch.float16, device=code.device)
    with torch.cuda.device(code.device):
        _lib.check(_lib.lib().kivi_unpack_dequant_lastdim_f16(code.data_ptr(), scale.data_ptr(), mn.data_ptr(), rows, T,
                                                               group_size, bits, out.data_ptr(),
                                                               _lib.stream_ptr(code.device)),
                   "kivi_unpack_dequant_lastdim_f16")
    return out


def unpack_and_dequant_kcache(k_code, scale, mn, group_size: int, bits: int):
    """quant/new_pack.py:51-66.  k_code [B,nh,T/fpi,D], scale/mn [B,nh,T/g,1,D] -> [B,nh,T,D] fp16."""
    assert bits in [2, 4, 8]
    assert len(k_code.shape) == 4
    out = _unpack_dequant_lastdim(k_code.transpose(2, 3), scale.squeeze(-2).transpose(2, 3),
                                  mn.squeeze(-2).transpose(2, 3), group_size, bits)
    return out.transpose(2, 3).contiguous()


def unpack_and_dequant_vcache(v_code, scale, mn, group_size: int, bits: int):
    """quant/new_pack.py:69-83.  v_code [B,nh,T,D/fpi], scale/mn [B,nh,T,D/g,1] -> [B,nh,T,D] fp16."""
    assert bits in [2, 4, 8]
    assert len(v_code.shape) == 4
    return _unpack_dequant_lastdim(v_code, scale.squeeze(-1), mn.squeeze(-1), group_size, bits)


def pack_tensor(data: torch.Tensor, bits: int, pack_dim: int):
    """quant/new_pack.py:86-107: OR-pack integer codes along pack_dim (element i of a word at bit
    i*bits).  Pure integer tensor utility (test-data helper in the reference); vectorised torch ops."""
    shape = data.shape
    feat_per_int = 32 // bits
    assert bits in [2, 4, 8], "Only 2, 4, 8 bits are supported"
    assert shape[pack_dim] % feat_per_int == 0, "Dimension length must be divisible by number of features per int"
    d = data.to(torch.int32).movedim(pack_dim, -1)
    d = d.reshape(d.shape[:-1] + (shape[pack_dim] // feat_per_int, feat_per_int))
    shifts = torch.arange(feat_per_int, device=data.device, dtype=torch.int32) * bits
    code = torch.zeros(d.shape[:-1], dtype=torch.int32, device=data.device)
    for j in range(feat_per_int):
        code |= d[..., j] << shifts[j]
    return code.movedim(-1, pack_dim).contiguous()


def unpack_tensor(v_code: torch.Tensor, bits: int, pack_dim: int):
    """quant/new_pack.py:110-129: inverse of pack_tensor (int16 result, as in the reference)."""
    assert bits in [2, 4, 8]
    feat_per_int = 32 // bits
    if pack_dim not in (2, 3):
        raise NotImplementedError                                # :127-128
    c = v_code.movedim(pack_dim, -1)
    shifts = torch.arange(feat_per_int, device=v_code.device, dtype=torch.int32) * bits
    num = 0xFF >> (8 - bits)
    out = ((c.unsqueeze(-1) >> shifts).to(torch.int16)) & num
    out = out.reshape(c.shape[:-1] + (c.shape[-1] * feat_per_int,))
    return out.movedim(-1, pack_dim).contiguous()

"""Tensor-parallel placement of a Llama model: attention heads and MLP columns sharded over the GPUs of a box.

Rank r of N holds the q rows of query heads [r*H/N, (r+1)*H/N), the k / v rows of KV heads [r*Hkv/N, ...) (a KV head and
its query group stay on one rank, so the KIVI cache and attention kernels run unchanged on H/N, Hkv/N heads), the o_proj
input columns of its query heads, the gate and up rows of intermediate channels [r*I/N, ...) and the matching down_proj
input columns.  The embedding, the norms and lm_head are replicated.  o_proj and down_proj then produce partial sums that
every rank adds up in fp32 in rank order: kivi_allreduce_add_rmsnorm_f16 in the decode step, `sum_partials` off it.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def check_divisible(config, world: int):
    """ValueError unless the heads, KV heads and intermediate channels split evenly over `world` ranks."""
    H, Hkv, inter = config.num_attention_heads, config.num_key_value_heads, config.intermediate_size
    if world < 1 or H % world or Hkv % world or inter % world:
        raise ValueError(f"tensor parallelism over {world} ranks needs num_attention_heads ({H}), num_key_value_heads "
                         f"({Hkv}) and intermediate_size ({inter}) divisible by {world}")
    if getattr(config, "attention_bias", False) or getattr(config, "mlp_bias", False):
        raise ValueError("tensor parallelism supports bias-free projections only (a sharded o_proj / down_proj bias "
                         "would be added once per rank)")


def shard_of(name: str, config, rank: int, world: int):
    """(dim, lo, hi): the slice of parameter `name` (HF Llama naming) that rank `rank` holds, or None if it is replicated."""
    hd = config.hidden_size // config.num_attention_heads
    q = config.num_attention_heads // world * hd
    kv = config.num_key_value_heads // world * hd
    inter = config.intermediate_size // world
    for suffix, dim, n in ((".self_attn.q_proj.weight", 0, q), (".self_attn.k_proj.weight", 0, kv),
                           (".self_attn.v_proj.weight", 0, kv), (".self_attn.o_proj.weight", 1, q),
                           (".mlp.gate_proj.weight", 0, inter), (".mlp.up_proj.weight", 0, inter),
                           (".mlp.down_proj.weight", 1, inter)):
        if name.endswith(suffix):
            return dim, rank * n, (rank + 1) * n
    return None


def shard_tensor(t, spec):
    """Apply a `shard_of` result to a tensor (or to a safetensors slice: only the selected bytes are read)."""
    if spec is None:
        return t[:]
    dim, lo, hi = spec
    return t[lo:hi] if dim == 0 else t[:, lo:hi]


def shard_state_dict(state: dict, config, rank: int, world: int) -> dict:
    """Rank `rank`'s part of a full HF Llama state dict (see the module docstring); ValueError if the shapes do not split."""
    check_divisible(config, world)
    return {k: shard_tensor(v, shard_of(k, config, rank, world)).contiguous() for k, v in state.items()}


def sum_partials(x: torch.Tensor) -> torch.Tensor:
    """The o_proj / down_proj reduction of the prompt pass: gather every rank's partial sum and add them in fp32 in rank
    order, rounded once to x's dtype -- the numerics of kivi_allreduce_add_rmsnorm_f16, so every rank holds the same bits."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return x
    ws = dist.get_world_size()
    parts = torch.empty((ws,) + tuple(x.shape), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(parts, x.contiguous())
    acc = parts[0].float()
    for p in range(1, ws):
        acc += parts[p].float()
    return acc.to(x.dtype)

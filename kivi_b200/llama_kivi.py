"""Drop-in surface of the reference's models/llama_kivi.py (and, by config, models/mistral_kivi.py).

* `kivi_decode_attention_tuple`  -- the decode branch of LlamaFlashAttention_KIVI.forward
  (models/llama_kivi.py:314-399) on the reference's own 9-tuple cache, op for op, with every KIVI op
  routed to libkivi_b200 (cuda_bmm_fA_qB_outer without re-layout copies, fused pack kernel).
* `kivi_prefill_tuple`           -- the prefill split + pack (:425-455) producing that 9-tuple.
* `LlamaFlashAttention_KIVI`     -- attention module: same projections / RoPE / cache policy on the
  reference's 9-tuple; a prompt pass may instead hand its rotated K/V to the pre-allocated `KiviCache`
  (`store_kv`).
* `LlamaForCausalLM_KIVI`        -- decoder-only LM with HF Llama parameter names (state dicts of
  LlamaForCausalLM / MistralForCausalLM load unchanged), config attrs k_bits, v_bits, group_size,
  residual_length (models/llama_kivi.py:34-38).  Host code is PyTorch (linears = cuBLAS); the decode
  step runs on the `KiviCache` (fused attention, kivi_decode.cu) and is captured in a CUDA graph.

The reference's forks star-import transformers 4.43 internals and do not import under the installed
transformers 5.5 (SURVEY 8c); this module depends on torch only and accepts any config object with the
usual Llama fields.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Callable, NamedTuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import glue
from .cache import KiviCache, kv_start_from_mask
from .choice import TokenChoice, processing_rows, sampling_rows
from .matmul import cuda_bmm_fA_qB_outer
from .new_pack import triton_quantize_and_pack_along_last_dim
from .tp import check_divisible, shard_of, shard_state_dict, shard_tensor, sum_partials  # noqa: F401 (re-export)


def repeat_kv(hidden_states: torch.Tensor, n_rep: int) -> torch.Tensor:
    """transformers' repeat_kv, used by the reference at models/llama_kivi.py:337,384."""
    if n_rep == 1:
        return hidden_states
    b, h, t, d = hidden_states.shape
    return hidden_states[:, :, None, :, :].expand(b, h, n_rep, t, d).reshape(b, h * n_rep, t, d)


# ---------------------------------------------------------------------------------------------------
# the reference's cache policy on its own 9-tuple (functional form of the hook)
# ---------------------------------------------------------------------------------------------------
def _cat(old, new, dim):
    return new if old is None else torch.cat([old, new], dim=dim)


def kivi_prefill_tuple(key_states, value_states, group_size, k_bits, v_bits, residual_length):
    """Prefill split + pack of models/llama_kivi.py:425-455: key/value_states [B, Hkv, n, D] -> 9-tuple.
    K: the leading n - n % R tokens are packed per channel (none if n < R), the rest stays fp16;
    V: everything but the newest R tokens is packed per token."""
    n, R = key_states.shape[-2], residual_length
    n_kq = n - n % R if n >= R else 0
    k_code = k_scale = k_mn = None
    if n_kq:
        k_code, k_scale, k_mn = triton_quantize_and_pack_along_last_dim(
            key_states[:, :, :n_kq].transpose(2, 3).contiguous(), group_size, k_bits)
    k_full = key_states[:, :, n_kq:].contiguous() if n_kq < n else None
    n_vq = max(n - R, 0)
    v_code = v_scale = v_mn = None
    if n_vq:
        v_code, v_scale, v_mn = triton_quantize_and_pack_along_last_dim(value_states[:, :, :n_vq].contiguous(),
                                                                        group_size, v_bits)
    v_full = value_states[:, :, n_vq:].contiguous() if n_vq else value_states
    return (k_code, k_full, k_scale, k_mn, v_code, v_full, v_scale, v_mn, n)


def kivi_decode_attention_tuple(query_states, key_states, value_states, past_key_value, group_size, k_bits, v_bits,
                                residual_length, attention_mask=None):
    """Decode branch of the reference hook (models/llama_kivi.py:314-399, tuple :454-455) on the
    reference's own 9-tuple, with the same rounding points; every KIVI op runs in libkivi_b200.
    query_states [B,H,1,D], key/value_states [B,Hkv,1,D] (post-RoPE) -> (attn_output [B,H,1,D], new 9-tuple)."""
    k_code, k_full, k_scale, k_mn, v_code, v_full, v_scale, v_mn, seen = past_key_value
    B, H, q_len, D = query_states.shape
    rep = H // key_states.shape[1]
    R = residual_length
    total = seen + key_states.shape[-2]

    # logits = [ q . dequant(K_packed)^T | q . K_window^T ] / sqrt(D)            (:323-341)
    k_full = _cat(k_full, key_states, 2)
    pieces = []
    if k_code is not None:
        pieces.append(cuda_bmm_fA_qB_outer(group_size, query_states, k_code, k_scale, k_mn, k_bits))
    pieces.append(torch.matmul(query_states, repeat_kv(k_full, rep).transpose(2, 3)))
    scores = (torch.cat(pieces, dim=-1) if len(pieces) > 1 else pieces[0]) / math.sqrt(D)
    if scores.shape != (B, H, q_len, total):                                     # (:358-362)
        raise ValueError(f"Attention weights should be of size {(B, H, q_len, total)}, but is {tuple(scores.shape)}")

    # a full window is packed per channel and appended along the token axis      (:343-356)
    if k_full.shape[-2] == R:
        assert R % group_size == 0
        c, sc, mn = triton_quantize_and_pack_along_last_dim(k_full.transpose(2, 3).contiguous(), group_size, k_bits)
        k_code, k_scale, k_mn, k_full = _cat(k_code, c, 3), _cat(k_scale, sc, 3), _cat(k_mn, mn, 3), None

    if attention_mask is not None:                                               # (:364-372)
        if attention_mask.shape != (B, 1, q_len, total):
            raise ValueError(f"Attention mask should be of size {(B, 1, q_len, total)}, but is {tuple(attention_mask.shape)}")
        floor = torch.tensor(torch.finfo(scores.dtype).min, device=scores.device)
        scores = torch.max(scores + attention_mask, floor)
    probs = F.softmax(scores, dim=-1, dtype=torch.float32).to(query_states.dtype)   # (:375)

    # out = probs[:tv] . dequant(V_packed) + probs[tv:] . V_window                  (:377-384)
    v_full = _cat(v_full, value_states, 2)
    L = v_full.shape[-2]
    window_part = torch.matmul(probs[..., -L:], repeat_kv(v_full, rep))
    if v_code is None:
        attn_output = window_part
    else:
        attn_output = cuda_bmm_fA_qB_outer(group_size, probs[..., :-L], v_code, v_scale, v_mn, v_bits)
        attn_output += window_part

    # the window keeps R tokens: its oldest one is packed per token                  (:386-399)
    if L > R:
        assert L == R + 1
        c, sc, mn = triton_quantize_and_pack_along_last_dim(v_full[:, :, :1].contiguous(), group_size, v_bits)
        v_code, v_scale, v_mn = _cat(v_code, c, 2), _cat(v_scale, sc, 2), _cat(v_mn, mn, 2)
        v_full = v_full[:, :, 1:].contiguous()
    return attn_output, (k_code, k_full, k_scale, k_mn, v_code, v_full, v_scale, v_mn, total)


# ---------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------
def default_config(name: str = "llama-2-7b", **kw):
    """Architecture shapes of the BASELINE configs (weights are random-init; no checkpoints offline)."""
    table = {
        "llama-2-7b": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                           num_key_value_heads=32, vocab_size=32000, rope_theta=10000.0, rms_norm_eps=1e-5),
        "llama-3-8b": dict(hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32,
                           num_key_value_heads=8, vocab_size=128256, rope_theta=500000.0, rms_norm_eps=1e-5),
        "mistral-7b": dict(hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32,
                           num_key_value_heads=8, vocab_size=32000, rope_theta=1000000.0, rms_norm_eps=1e-5),
        "llama-2-13b": dict(hidden_size=5120, intermediate_size=13824, num_hidden_layers=40, num_attention_heads=40,
                            num_key_value_heads=40, vocab_size=32000, rope_theta=10000.0, rms_norm_eps=1e-5),
        "llama-2-70b": dict(hidden_size=8192, intermediate_size=28672, num_hidden_layers=80, num_attention_heads=64,
                            num_key_value_heads=8, vocab_size=32000, rope_theta=10000.0, rms_norm_eps=1e-5),
        "qwen2.5-7b": dict(model_type="qwen2", hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                           num_attention_heads=28, num_key_value_heads=4, vocab_size=152064, rope_theta=1000000.0,
                           rms_norm_eps=1e-6),
        "qwen3-8b": dict(model_type="qwen3", hidden_size=4096, intermediate_size=12288, num_hidden_layers=36,
                         num_attention_heads=32, num_key_value_heads=8, head_dim=128, vocab_size=151936,
                         rope_theta=1000000.0, rms_norm_eps=1e-6),
        # hidden 2560 != 32 heads x 128
        "qwen3-4b": dict(model_type="qwen3", hidden_size=2560, intermediate_size=9728, num_hidden_layers=36,
                         num_attention_heads=32, num_key_value_heads=8, head_dim=128, vocab_size=151936,
                         rope_theta=1000000.0, rms_norm_eps=1e-6),
        "llama-3.2-3b": dict(hidden_size=3072, intermediate_size=8192, num_hidden_layers=28, num_attention_heads=24,
                             num_key_value_heads=8, vocab_size=128256, rope_theta=500000.0, rms_norm_eps=1e-5),
        "tiny": dict(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                     num_key_value_heads=2, vocab_size=512, rope_theta=10000.0, rms_norm_eps=1e-5),
    }
    cfg = dict(table[name], k_bits=2, v_bits=2, group_size=32, residual_length=128, use_flash=True,
               max_position_embeddings=32768 + 1024)
    cfg.update(kw)
    return SimpleNamespace(**cfg)


class LlamaRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        # HF LlamaRMSNorm: fp32 statistics, the normalised value rounded to x's dtype, THEN the weight product (rounded
        # again).  F.rms_norm multiplies by the weight in fp32 and rounds once, which differs in ~1/4 of fp16 outputs;
        # the decode step's add_rmsnorm kernel rounds like this chain.
        h = x.float()
        h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + self.variance_epsilon)
        return self.weight * h.to(x.dtype)


ROPE_TYPES = ("default", "linear", "llama3")


def rope_settings(config):
    """The RoPE settings of a config object or a config.json dict -> (theta, scaling).  transformers 5.x writes them as
    `rope_parameters` {"rope_theta", "rope_type", ...}; 4.x as a top-level `rope_theta` plus `rope_scaling` (None, or a dict
    naming its type under "type" or "rope_type").  scaling is None for plain RoPE, else the parameters with "rope_type"
    set.  Raises NotImplementedError for a RoPE type outside ROPE_TYPES and for a partial rotary embedding."""
    get = config.get if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))
    params = dict(get("rope_parameters") or get("rope_scaling") or {})
    theta = float(params.get("rope_theta", get("rope_theta", 10000.0)))
    kind = params.get("rope_type", params.get("type", "default"))
    if kind not in ROPE_TYPES:
        raise NotImplementedError(f"RoPE type {kind!r} is not supported (supported: {', '.join(ROPE_TYPES)})")
    partial = params.get("partial_rotary_factor", get("partial_rotary_factor"))
    if partial is not None and float(partial) != 1.0:
        raise NotImplementedError(f"partial_rotary_factor {partial}: only a rotary embedding over the whole head is supported")
    if kind == "default":
        return theta, None
    need = ("factor",) if kind == "linear" else ("factor", "low_freq_factor", "high_freq_factor")
    missing = [k for k in need if k not in params]
    if missing:
        raise ValueError(f"RoPE type {kind!r} needs {', '.join(missing)}")
    scaling = {k: float(params[k]) for k in need}
    scaling["rope_type"] = kind
    if kind == "llama3":        # transformers falls back to max_position_embeddings as well
        scaling["original_max_position_embeddings"] = params.get("original_max_position_embeddings",
                                                                 get("max_position_embeddings"))
    return theta, scaling


def sliding_window(config):
    """The sliding window W of a config (config.sliding_window; None or absent = attention over the whole cache).  A
    config whose `layer_types` mixes attention kinds (per-layer windows) raises NotImplementedError; one whose layers are
    all full attention has no window.  A Qwen2 config.json names its window next to `use_sliding_window`, which decides:
    false means no window whatever `sliding_window` says; true puts windows on layers max_window_layers and above (as
    transformers' Qwen2Config derives `layer_types`), so a max_window_layers between 0 and the layer count is refused."""
    use = getattr(config, "use_sliding_window", None)
    if use is not None and not use:
        return None
    kinds = set(getattr(config, "layer_types", None) or ())
    if not kinds and use:
        n, first = config.num_hidden_layers, getattr(config, "max_window_layers", config.num_hidden_layers)
        kinds = {"sliding_attention" if i >= first else "full_attention" for i in range(n)}
    if len(kinds) > 1:
        raise NotImplementedError(f"layer_types {sorted(kinds)}: per-layer attention kinds (sliding windows on some layers "
                                  "only) are not supported")
    w = getattr(config, "sliding_window", None)
    if w is None or kinds == {"full_attention"}:
        return None
    if int(w) != w or int(w) < 1:
        raise ValueError(f"sliding_window must be a positive number of tokens or None, got {w!r}")
    return int(w)


def _rope_tables(head_dim, max_pos, theta, device, scaling=None):
    """fp16 cos / sin [max_pos, head_dim].  The inverse frequencies follow transformers' RoPE initialisers (default, linear,
    llama3) op for op in fp32, so the tables are the ones its rotary embedding produces."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32, device=device) / head_dim))
    kind = "default" if scaling is None else scaling["rope_type"]
    if kind == "linear":
        inv_freq = inv_freq / scaling["factor"]
    elif kind == "llama3":
        factor, low, high = scaling["factor"], scaling["low_freq_factor"], scaling["high_freq_factor"]
        old_context_len = scaling["original_max_position_embeddings"]
        low_freq_wavelen, high_freq_wavelen = old_context_len / low, old_context_len / high
        wavelen = 2 * math.pi / inv_freq
        inv_freq_llama = torch.where(wavelen > low_freq_wavelen, inv_freq / factor, inv_freq)
        smooth_factor = (old_context_len / wavelen - low) / (high - low)
        smoothed_inv_freq = (1 - smooth_factor) * inv_freq_llama / factor + smooth_factor * inv_freq_llama
        is_medium_freq = ~(wavelen < high_freq_wavelen) * ~(wavelen > low_freq_wavelen)
        inv_freq = torch.where(is_medium_freq, smoothed_inv_freq, inv_freq_llama)
    elif kind != "default":
        raise NotImplementedError(f"RoPE type {kind!r} is not supported (supported: {', '.join(ROPE_TYPES)})")
    freqs = torch.outer(torch.arange(max_pos, dtype=torch.float32, device=device), inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().half(), emb.sin().half()


def _rotate_half(x):
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


# Rows of B * n that the per-token part of a prompt pass (norms, projections, RoPE, MLP) runs on at a time: a longer prompt
# holds one chunk's [rows, intermediate] temporaries instead of the whole prompt's.  Every model-level prompt of the test
# suite (B * n <= 1500) stays one chunk and runs the unchunked code.
PROMPT_CHUNK_ROWS = 16384


class PromptMask(NamedTuple):
    """The mask of a prompt pass in the form kivi_prompt_attention_f16 takes it, in place of an additive [B, 1, n, n]
    tensor: query i of sequence b sees the keys max(kv_start[b], i - window + 1) <= j <= i.  kv_start: int32 [B] on the
    device, or None (no padding); window: 0 = none."""
    kv_start: torch.Tensor | None
    window: int


class PrefixMask(NamedTuple):
    """The mask of a prompt pass over tokens r .. n-1 of a prompt whose K / V at positions 0 .. r-1 are stored
    (LlamaForCausalLM_KIVI.insert with a PrefixCache).  Each layer places its suffix K / V after the prefix's in one
    [1, Hkv, n, 128] buffer (`extend`(layer, k, v) -> (k, v)), runs kivi_prompt_attention_suffix_f16 on it with `mask`
    (query t at position r + t) and stores that buffer."""
    mask: PromptMask
    extend: Callable


def attention_biases(config):
    """(q / k / v bias, o_proj bias) of a config: Qwen2 (model_type "qwen2") has biases on q, k and v and none on o_proj;
    Llama and Mistral have one `attention_bias` flag for all four projections."""
    if getattr(config, "model_type", None) == "qwen2":
        return True, False
    bias = bool(getattr(config, "attention_bias", False))
    return bias, bias


def qk_norm(config):
    """Whether the attention layers normalise every q and k head (Qwen3's q_norm / k_norm, an RMSNorm over head_dim
    channels before RoPE)."""
    return getattr(config, "model_type", None) == "qwen3"


def head_dim(config):
    """config.head_dim when the config names one (Qwen3 and Mistral-NeMo have hidden_size != heads x head_dim), else
    hidden_size / num_attention_heads."""
    return getattr(config, "head_dim", None) or config.hidden_size // config.num_attention_heads


def _linear(owner, name: str, layer: int, x, lora):
    """owner.<name>(x), plus the LoRA delta of each token's adapter when `lora` = (kivi_b200.lora.LoraState, adapter slot
    of each token [tokens]) is given (the prompt pass and forward(); the decode step runs the LoRA kernels instead)."""
    y = getattr(owner, name)(x)
    if lora is not None:
        lora[0].add(layer, name, x, y, lora[1])
    return y


class LlamaFlashAttention_KIVI(nn.Module):
    """Attention layer of the reference (models/llama_kivi.py:264-466), KIVI ops on libkivi_b200."""

    def __init__(self, config, layer_idx: int = 0, tp_world: int = 1):
        super().__init__()
        self.config = config
        self.layer_idx = layer_idx
        self.hidden_size = config.hidden_size
        self.head_dim = head_dim(config)
        self.num_heads = config.num_attention_heads // tp_world              # this rank's heads (kivi_b200.tp)
        self.num_key_value_heads = config.num_key_value_heads // tp_world
        self.num_key_value_groups = self.num_heads // self.num_key_value_heads
        self.k_bits, self.v_bits = config.k_bits, config.v_bits            # models/llama_kivi.py:34-38
        self.group_size, self.residual_length = config.group_size, config.residual_length
        qkv_bias, o_bias = attention_biases(config)
        self.q_proj = nn.Linear(self.hidden_size, self.num_heads * self.head_dim, bias=qkv_bias)
        self.k_proj = nn.Linear(self.hidden_size, self.num_key_value_heads * self.head_dim, bias=qkv_bias)
        self.v_proj = nn.Linear(self.hidden_size, self.num_key_value_heads * self.head_dim, bias=qkv_bias)
        self.o_proj = nn.Linear(self.num_heads * self.head_dim, self.hidden_size, bias=o_bias)
        if qk_norm(config):                                                 # Qwen3: replicated under tensor parallelism
            self.q_norm = LlamaRMSNorm(self.head_dim, config.rms_norm_eps)
            self.k_norm = LlamaRMSNorm(self.head_dim, config.rms_norm_eps)
        else:
            self.q_norm = self.k_norm = None

    def _qk_normed(self, q, k):
        """q and k [..., heads, D] through q_norm / k_norm (per head, before RoPE), when the model has them."""
        if self.q_norm is None:
            return q, k
        return self.q_norm(q), self.k_norm(k)

    def _qkv(self, hidden_states, cos, sin, lora=None):
        bsz, q_len, _ = hidden_states.shape
        proj = lambda name: _linear(self, name, self.layer_idx, hidden_states, lora)   # noqa: E731
        q = proj("q_proj").view(bsz, q_len, self.num_heads, self.head_dim)
        k = proj("k_proj").view(bsz, q_len, self.num_key_value_heads, self.head_dim)
        v = proj("v_proj").view(bsz, q_len, self.num_key_value_heads, self.head_dim).transpose(1, 2)
        q, k = (t.transpose(1, 2) for t in self._qk_normed(q, k))
        q = q * cos + _rotate_half(q) * sin                                 # apply_rotary_pos_emb (:311)
        k = k * cos + _rotate_half(k) * sin
        return q, k, v

    def _qkv_rows(self, x, cos, sin, lora=None):
        """_qkv on rows of tokens: x [rows, hidden], cos / sin [rows, 1, D] -> q [rows, H, D], k and v [rows, Hkv, D],
        q and k rotated."""
        rows = x.shape[0]
        q = _linear(self, "q_proj", self.layer_idx, x, lora).view(rows, self.num_heads, self.head_dim)
        k = _linear(self, "k_proj", self.layer_idx, x, lora).view(rows, self.num_key_value_heads, self.head_dim)
        v = _linear(self, "v_proj", self.layer_idx, x, lora).view(rows, self.num_key_value_heads, self.head_dim)
        q, k = self._qk_normed(q, k)
        return q * cos + _rotate_half(q) * sin, k * cos + _rotate_half(k) * sin, v

    def _prompt_attention(self, q, k, v, attention_mask):
        """Attention over the prompt itself (the reference calls flash-attn here, models/llama_kivi.py:401-423) -> [B,
        q_len, H * D].  A PromptMask (a left-padded batch or a sliding window that cuts the prompt, fp16 on CUDA) runs
        kivi_prompt_attention_f16 on the strided q / k / v, with no mask tensor and no K / V copy per query head.
        Otherwise SDPA: causal, plus an additive mask [B, 1, q_len, q_len] when one is given."""
        B, H, n, D = q.shape
        if isinstance(attention_mask, PromptMask):
            out = torch.empty((B, n, H, D), dtype=q.dtype, device=q.device)
            run = glue.prompt_attention if k.shape[2] == n else glue.prompt_attention_suffix     # a stored prefix
            run(q, k, v, out, attention_mask.kv_start, attention_mask.window)
            return out.view(B, n, H * D)
        kk, vv = repeat_kv(k, self.num_key_value_groups), repeat_kv(v, self.num_key_value_groups)
        if attention_mask is None:
            o = F.scaled_dot_product_attention(q, kk, vv, is_causal=True)
        else:
            o = F.scaled_dot_product_attention(q, kk, vv, attn_mask=attention_mask.to(q.dtype))
        return o.transpose(1, 2).reshape(B, n, H * D)

    def _prompt_core(self, q, k, v, attention_mask, store_kv):
        """The prompt pass between the projections and o_proj: attention ([B, q_len, H * D]) and the 9-tuple, or
        store_kv(layer, k, v) and None.  With a PrefixMask, k and v first take the stored prefix in front."""
        if isinstance(attention_mask, PrefixMask):
            k, v = attention_mask.extend(self.layer_idx, k, v)
            attention_mask = attention_mask.mask
        attn_output = self._prompt_attention(q, k, v, attention_mask)
        if store_kv is None:
            return attn_output, kivi_prefill_tuple(k, v, self.group_size, self.k_bits, self.v_bits, self.residual_length)
        store_kv(self.layer_idx, k, v)
        return attn_output, None

    def forward(self, hidden_states, cos, sin, past_key_value=None, attention_mask=None, store_kv=None, lora=None):
        """hidden_states [B, q_len, hidden]; cos/sin broadcastable to [B, 1, q_len, D].  lora: see _linear.
        past_key_value: None (a prompt pass, returns a 9-tuple) or the reference's 9-tuple (decode, returns the next one).
        store_kv: with a prompt pass, a callable store_kv(layer, k, v) that takes the rotated K and V [B, Hkv, q_len, D] in
        place of the 9-tuple (the fused cache: KiviCache.prefill, or a refill of one slot); the pass then returns None.
        attention_mask: None or additive [B, 1, q_len, kv_len] (models/llama_kivi.py:364-372); in a prompt pass also a
        PromptMask or a PrefixMask."""
        bsz, q_len, _ = hidden_states.shape
        q, k, v = self._qkv(hidden_states, cos, sin, lora)
        if past_key_value is not None:                                      # reference 9-tuple, decode
            attn_output, past = kivi_decode_attention_tuple(q, k, v, past_key_value, self.group_size, self.k_bits,
                                                            self.v_bits, self.residual_length, attention_mask)
            attn_output = attn_output.transpose(1, 2).contiguous().reshape(bsz, q_len, self.num_heads * self.head_dim)
        else:                                                               # prompt (:401-455)
            attn_output, past = self._prompt_core(q, k, v, attention_mask, store_kv)
        return _linear(self, "o_proj", self.layer_idx, attn_output, lora), None, past


LlamaAttention_KIVI = LlamaFlashAttention_KIVI      # models/llama_kivi.py:19 (unreachable in the reference: ctor asserts use_flash)


class LlamaMLP(nn.Module):
    def __init__(self, config, tp_world: int = 1):
        super().__init__()
        inter = config.intermediate_size // tp_world                          # this rank's channels (kivi_b200.tp)
        self.gate_proj = nn.Linear(config.hidden_size, inter, bias=False)
        self.up_proj = nn.Linear(config.hidden_size, inter, bias=False)
        self.down_proj = nn.Linear(inter, config.hidden_size, bias=False)

    def forward(self, x, lora=None, layer: int = 0):
        """lora, layer: the LoRA deltas of the rows' adapters (_linear) in decoder layer `layer`."""
        act = F.silu(_linear(self, "gate_proj", layer, x, lora)) * _linear(self, "up_proj", layer, x, lora)
        return _linear(self, "down_proj", layer, act, lora)


class LlamaDecoderLayer_KIVI(nn.Module):
    def __init__(self, config, layer_idx, tp_world: int = 1):
        super().__init__()
        self.self_attn = LlamaFlashAttention_KIVI(config, layer_idx, tp_world)
        self.mlp = LlamaMLP(config, tp_world)
        self.input_layernorm = LlamaRMSNorm(config.hidden_size, config.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNorm(config.hidden_size, config.rms_norm_eps)
        self.tp_world = tp_world

    def forward(self, hidden_states, cos, sin, past_key_value=None, attention_mask=None, store_kv=None, lora=None):
        """lora: None, or (kivi_b200.lora.LoraState, adapter slot of each batch row [B]) -- every token of row b takes the
        LoRA deltas of adapter slot b (< 0: none)."""
        if past_key_value is None and hidden_states.shape[0] * hidden_states.shape[1] > PROMPT_CHUNK_ROWS:
            return self._prompt_in_chunks(hidden_states, cos, sin, attention_mask, store_kv, lora)
        if lora is not None:
            lora = (lora[0], lora[1].repeat_interleave(hidden_states.shape[1]))        # a slot per token
        residual = hidden_states
        h, _, past = self.self_attn(self.input_layernorm(hidden_states), cos, sin, past_key_value, attention_mask,
                                    store_kv, lora)
        if self.tp_world > 1:                                                 # partial sums of the sharded projections
            h = sum_partials(h)
        hidden_states = residual + h
        h = self.mlp(self.post_attention_layernorm(hidden_states), lora, self.self_attn.layer_idx)
        if self.tp_world > 1:
            h = sum_partials(h)
        hidden_states = hidden_states + h
        return hidden_states, past

    def _prompt_in_chunks(self, x, cos, sin, attention_mask, store_kv, lora=None):
        """forward() of a prompt pass in bounded memory: the per-token work -- input norm, q|k|v, RoPE; after the
        attention o_proj, the residual add, the post-attention norm, the MLP and its residual add -- runs on
        PROMPT_CHUNK_ROWS rows of B * n at a time, the attention between the two halves on the whole prompt.  The layer
        holds the residual stream, q, k, v, the attention output and one chunk's temporaries.  x [B, n, hidden] is the
        residual stream, updated in place."""
        a = self.self_attn
        B, n, hidden = x.shape
        rows, D = B * n, a.head_dim
        flat = x.view(rows, hidden)
        cos, sin = (t.expand(B, 1, n, D).reshape(rows, 1, D) for t in (cos, sin))
        q = x.new_empty((rows, a.num_heads, D))
        k = x.new_empty((rows, a.num_key_value_heads, D))
        v = torch.empty_like(k)
        chunks = [slice(lo, min(lo + PROMPT_CHUNK_ROWS, rows)) for lo in range(0, rows, PROMPT_CHUNK_ROWS)]
        slots = None if lora is None else lora[1].repeat_interleave(n)          # a slot per token
        part = lambda c: None if lora is None else (lora[0], slots[c])        # noqa: E731
        for c in chunks:
            q[c], k[c], v[c] = a._qkv_rows(self.input_layernorm(flat[c]), cos[c], sin[c], part(c))
        heads = lambda t: t.view(B, n, -1, D).transpose(1, 2)                # noqa: E731 ([B, heads, n, D], as _qkv)
        attn, past = a._prompt_core(heads(q), heads(k), heads(v), attention_mask, store_kv)
        del q, k, v
        attn = attn.view(rows, -1)
        for c in chunks:
            h = _linear(a, "o_proj", a.layer_idx, attn[c], part(c))
            if self.tp_world > 1:
                h = sum_partials(h)
            r = flat[c] + h
            h = self.mlp(self.post_attention_layernorm(r), part(c), a.layer_idx)
            if self.tp_world > 1:
                h = sum_partials(h)
            flat[c] = r + h
        return x, past


class LlamaModel_KIVI(nn.Module):
    def __init__(self, config, tp_world: int = 1):
        super().__init__()
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size)
        self.layers = nn.ModuleList([LlamaDecoderLayer_KIVI(config, i, tp_world) for i in range(config.num_hidden_layers)])
        self.norm = LlamaRMSNorm(config.hidden_size, config.rms_norm_eps)


class KiviPast(tuple):
    """The per-layer `past_key_value` that forward() hands out while the cache lives in the pre-allocated KiviCache.
    It indexes like the reference's 9-tuple (models/llama_kivi.py:454-455): [8] / [-1] is kv_seq_len (what
    prepare_inputs_for_generation reads, :917) and costs nothing; the eight tensors are exported from the blocked cache
    on first access (a snapshot).  Passing it back to forward() continues on the fused path; it is valid for that as long
    as the cache has not moved on (one step per forward call, like the reference's functional tuples)."""

    def __new__(cls, cache, layer: int, kv_len: int):
        self = super().__new__(cls, ())
        self.cache, self.layer, self.kv_len, self._fields = cache, layer, kv_len, None
        return self

    def materialise(self):
        if self._fields is None:
            if self.cache.kv_len != self.kv_len:
                raise RuntimeError(f"stale KIVI cache view: it describes {self.kv_len} tokens, the cache now holds "
                                   f"{self.cache.kv_len} (export a view before decoding further if you need a snapshot)")
            self._fields = self.cache.export(self.layer)
        return self._fields

    def __len__(self):
        return 9

    def __getitem__(self, i):
        if isinstance(i, int) and i in (8, -1):
            return self.kv_len
        return self.materialise()[i]

    def __iter__(self):
        return iter(self.materialise())

    def __repr__(self):
        return f"KiviPast(layer={self.layer}, kv_seq_len={self.kv_len})"


class _Output(tuple):
    """What forward() returns when no transformers ModelOutput class is wanted: a (logits, past_key_values) tuple that
    also answers to the attribute names of CausalLMOutputWithPast."""
    __slots__ = ()
    loss = None
    logits = property(lambda self: self[0])
    past_key_values = property(lambda self: self[1])


_P2P_SAMPLING = ("sampling with enable_token_allgather(mode='p2p'): the fused argmax + peer-store exchange is greedy only; "
                 "use mode='nccl', which gathers the sampled ids")


def _additive_mask(attention_mask, q_len: int, total: int, dtype, device, window: int | None = None, batch: int = 1):
    """HF padding mask [B, total] (1 = attend; None = no padding) -> additive [B, 1, q_len, total] with the causal
    structure, or None when nothing is masked; a 4-D additive mask passes through (what the reference's hook receives,
    :364-372).  window = W (a sliding window): query i, at position total - q_len + i, also drops the keys at or below
    its position - W (transformers' kv_idx > q_idx - W); `batch` sizes the mask when there is no padding mask."""
    if attention_mask is not None and attention_mask.dim() == 4:
        return attention_mask
    cut = window is not None and total > window                           # some query loses keys to the window
    if attention_mask is None:
        if not cut:
            return None
        B = batch
        keep = torch.ones((1, 1, 1, total), dtype=torch.bool, device=device)
    else:
        keep = attention_mask[:, None, None, :total].to(torch.bool)
        B = keep.shape[0]
    if q_len == 1 and not cut and bool(keep.all()):
        return None
    if q_len > 1 or cut:
        causal = torch.ones((q_len, total), dtype=torch.bool, device=device).tril(total - q_len)
        if cut:
            causal = causal & ~causal.tril(total - q_len - window)
        keep = keep & causal
        if attention_mask is None:
            keep = keep.expand(B, 1, q_len, total)
    else:
        keep = keep.expand(-1, 1, 1, total)
    return torch.zeros(keep.shape, dtype=dtype, device=device).masked_fill(~keep, torch.finfo(dtype).min)


def _processing_args(n: int, repetition_penalty=None, min_length=None, min_new_tokens=None, eos_token_id=None,
                     pad_token_id=None):
    """generate()'s logits-processing arguments (prompt of n positions, left padding included, as transformers counts
    min_length) as set_processing keyword arguments, or None when they ask for nothing: no repetition penalty other than 1,
    and no eos_token_id.  min_length / min_new_tokens without eos_token_id is a ValueError."""
    floors = [m for m in (min_new_tokens, None if min_length is None else min_length - n) if m is not None]
    min_new = max(floors + [0])
    if eos_token_id is None and (min_new_tokens or min_length):
        raise ValueError("min_length and min_new_tokens suppress eos_token_id until they are reached: pass eos_token_id "
                         "(the config's EOS is not used as a default)")
    rep = 1.0 if repetition_penalty is None else repetition_penalty
    if rep == 1.0 and eos_token_id is None:
        return None
    return dict(repetition_penalty=rep, min_new_tokens=min_new, eos_token_id=eos_token_id, pad_token_id=pad_token_id)


def _trace_add(trace, logits, scores, clone: bool = False):
    """One new token's entries of generate()'s output_logits / output_scores lists (either may be None: not asked for);
    clone: the tensors are the step's static buffers.  With processing off the scores are the logits: one copy serves both."""
    if trace is None:
        return
    lg = logits.reshape(-1, logits.shape[-1])
    if clone and trace.logits is not None:
        lg = lg.clone()
    if trace.logits is not None:
        trace.logits.append(lg)
    if trace.scores is not None:
        sc = scores.reshape(-1, scores.shape[-1])
        if scores is logits:
            sc = lg.clone() if clone and trace.logits is None else lg
        elif clone:
            sc = sc.clone()
        trace.scores.append(sc)


def _trace_pop(trace):
    for t in (trace.scores, trace.logits):
        if t is not None:
            t.pop()


def _generate_output(sequences, trace):
    """transformers' GenerateDecoderOnlyOutput of a greedy or sampled generate(): the fields not asked for are None."""
    from transformers.generation.utils import GenerateDecoderOnlyOutput
    tup = lambda t: None if t is None else tuple(t)                       # noqa: E731
    return GenerateDecoderOnlyOutput(sequences=sequences, scores=tup(trace.scores), logits=tup(trace.logits))


class LlamaForCausalLM_KIVI(nn.Module):
    """models/llama_kivi.py:785.  `forward` keeps the reference's contract (HF argument names, per-layer 9-tuples as
    past_key_values, fp32 logits, `prepare_inputs_for_generation`, `_reorder_cache`); `decode_step` / `generate` use
    the fused cache path (pre-allocated KiviCache, the step captured in a CUDA graph).

    tensor_parallel=True: one rank of a model sharded over the GPUs of a box (kivi_b200.tp; rank and world from
    kivi_b200.dist.init(), i.e. torchrun's environment).  The modules are built at this rank's shapes, the cache holds its
    heads, and the decode step reduces the o_proj / down_proj partial sums with kivi_allreduce_add_rmsnorm_f16 inside its
    CUDA graph.  generate / decode_step / prefill / insert / serve run on every rank with the same inputs and give every
    rank the same tokens; forward() (9-tuples), 9-tuple import / export and enable_token_allgather are rejected."""

    def __init__(self, config, tensor_parallel: bool = False):
        super().__init__()
        if getattr(config, "model_type", None) == "qwen3_moe":
            raise NotImplementedError("model_type 'qwen3_moe': mixture-of-experts MLPs are not supported")
        hd = getattr(config, "head_dim", None)                  # transformers configs carry it explicitly
        if hd is not None and hd != 128:
            raise NotImplementedError(f"head_dim {hd} (hidden_size {config.hidden_size}, {config.num_attention_heads} "
                                      "heads): only head_dim 128 is supported")
        rope_settings(config)                                   # an unsupported RoPE type is refused here, not at the first forward
        self.sliding_window = sliding_window(config)            # per-layer windows are refused here
        self.config = config
        self.vocab_size = config.vocab_size
        self.tensor_parallel = tensor_parallel
        self.tp_rank, self.tp_world = 0, 1
        if tensor_parallel:
            from . import dist as kdist
            self.tp_rank, self.tp_world, _ = kdist.init()
            check_divisible(config, self.tp_world)
        self.model = LlamaModel_KIVI(config, self.tp_world)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self._rope = None
        self.cache: KiviCache | None = None
        self._graph = None
        self._graph_ragged = False          # the captured step calls the left-padded attention entry
        self._reorder_graph = None          # beam search: the cache's row reorder + the position gather, captured
        self.launches_per_reorder = None
        self._fast = None
        self._dist_tokens = None            # [world * B] ids gathered inside the step (greedy sampling, world > 1)
        self._dist_in_graph = True
        self._exchange = None               # kivi_b200.dist.PeerTokenExchange: ids stored into the peers' buffers by the sampling kernel
        self._allreduce = None              # kivi_b200.dist.PeerAllReduce of the tensor-parallel decode step
        self.choice: TokenChoice | None = None   # the cache's rows' sampling, logits processing and logprobs (init_cache)
        self._lora = None                   # kivi_b200.lora.LoraState once an adapter is loaded (load_adapter)
        self._adapter_sel = None            # set_adapters(): None, one slot, or a slot per row
        self._adapter_idx = None            # int32 [batch]: each cache row's adapter slot (-1: none), read by the step

    # ------------------------------------------------------------------ HF-style construction
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, config=None, torch_dtype=torch.float16, device_map=None,
                        tensor_parallel: bool = False, **unused):
        """Load a LOCAL Hugging Face Llama / Mistral / Qwen2 / Qwen3 checkpoint directory (config.json + *.safetensors or
        pytorch_model*.bin; there is no network here) into the KIVI model, as the reference's
        LlamaForCausalLM_KIVI.from_pretrained(config=...) does (example.py:22-28, mem_spd_test.py:24-31).  `config` is
        the user's config object carrying k_bits / v_bits / group_size / residual_length (models/llama_kivi.py:34-38);
        without one, config.json is read and the KIVI attributes default to K2V2 g32 R128.
        tensor_parallel=True: this rank's shard only (kivi_b200.tp): safetensors files are read slice by slice
        (safe_open(...).get_slice), .bin files are sharded after loading; the modules are built without initialising the
        full-size weights."""
        import glob
        import json
        import os
        path = str(pretrained_model_name_or_path)
        if not os.path.isdir(path):
            raise FileNotFoundError(f"{path}: from_pretrained needs a local checkpoint directory (no network on this box)")
        if config is None:
            with open(os.path.join(path, "config.json")) as f:
                raw = json.load(f)
            config = SimpleNamespace(**raw)
        for name, dflt in (("k_bits", 2), ("v_bits", 2), ("group_size", 32), ("residual_length", 128), ("use_flash", True)):
            if not hasattr(config, name):
                setattr(config, name, dflt)
        if tensor_parallel:
            from . import dist as kdist
            kdist.init()                                                  # the process group, outside the meta context
            with torch.device("meta"):                                   # parameters come from the checkpoint (assign)
                model = cls(config, tensor_parallel=True)
            rank, world = model.tp_rank, model.tp_world
        else:
            model = cls(config)
        state = {}
        files = sorted(glob.glob(os.path.join(path, "*.safetensors")))
        if files:
            if tensor_parallel:
                from safetensors import safe_open
                for fn in files:
                    with safe_open(fn, framework="pt") as f:
                        for k in f.keys():
                            state[k] = shard_tensor(f.get_slice(k), shard_of(k, config, rank, world))
            else:
                from safetensors.torch import load_file
                for fn in files:
                    state.update(load_file(fn))
        else:
            for fn in sorted(glob.glob(os.path.join(path, "pytorch_model*.bin"))):
                part = torch.load(fn, map_location="cpu", weights_only=True)
                state.update(shard_state_dict(part, config, rank, world) if tensor_parallel else part)
        if not state:
            raise FileNotFoundError(f"{path}: no *.safetensors / pytorch_model*.bin weights found")
        if "lm_head.weight" not in state and getattr(config, "tie_word_embeddings", False):
            state["lm_head.weight"] = state["model.embed_tokens.weight"]
        state = {k: v for k, v in state.items() if not k.endswith("rotary_emb.inv_freq")}
        model.load_state_dict(state, strict=True, assign=tensor_parallel)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        if device_map is not None:          # "auto" / "cuda" / {"": device}: this rank's model on the current GPU (dp or tp)
            model = model.cuda()
        return model.eval()

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    def _apply(self, fn, *args, **kwargs):
        # .to() / .half() / .cuda() re-create every parameter: the fused decode buffers and the captured graph would keep
        # pointing at the old storage
        self._fast, self._graph, self._rope = None, None, None
        return super()._apply(fn, *args, **kwargs)

    # ------------------------------------------------------------------ helpers
    def _tables(self, device, positions: int = 0):
        """cos / sin tables with a row for every position the cache can reach, and at least `positions` rows (a rolling
        generate() reaches positions beyond its cache).  Rebuilding them drops the captured step, which reads them."""
        rows = max(getattr(self.config, "max_position_embeddings", 4096), positions)
        if self.cache is not None:
            rows = max(rows, self.cache.max_tokens + 1)   # a cache longer than the config's context still has its rows
        if self._rope is None or self._rope[0].device != device or self._rope[0].shape[0] < rows:
            theta, scaling = rope_settings(self.config)
            self._rope = _rope_tables(head_dim(self.config), rows, theta, device, scaling)
            self._graph = None
        return self._rope

    def _run_layers(self, input_ids, positions, pasts, attention_mask=None, store_kv=None, adapters=None):
        """adapters: None, or the adapter slot of each batch row (int32 [B]; -1: none)."""
        cos_t, sin_t = self._tables(input_ids.device)
        lora = None if adapters is None or self._lora is None else (self._lora, adapters.to(input_ids.device))
        cos = cos_t.index_select(0, positions.reshape(-1)).view(positions.shape[0], 1, positions.shape[1], -1)
        sin = sin_t.index_select(0, positions.reshape(-1)).view(positions.shape[0], 1, positions.shape[1], -1)
        h = self.model.embed_tokens(input_ids)
        new_pasts = []
        for i, layer in enumerate(self.model.layers):
            h, past = layer(h, cos, sin, pasts[i] if pasts is not None else None, attention_mask, store_kv, lora)
            new_pasts.append(past)
        rows = h.shape[0] * h.shape[1]
        if rows > PROMPT_CHUNK_ROWS:                   # a long prompt: the norm's fp32 temporaries one chunk at a time
            flat = h.view(rows, -1)
            for lo in range(0, rows, PROMPT_CHUNK_ROWS):
                flat[lo:lo + PROMPT_CHUNK_ROWS] = self.model.norm(flat[lo:lo + PROMPT_CHUNK_ROWS])
        else:
            h = self.model.norm(h)
        return h, new_pasts

    # ------------------------------------------------------------------ reference-style forward (9-tuples)
    @torch.no_grad()
    def forward(self, input_ids=None, past_key_values=None, attention_mask=None, position_ids=None, use_cache=None,
                return_dict=None, **unused):
        """models/llama_kivi.py:815-905.  Returns logits [B, q_len, vocab] fp32 (:881) and past_key_values = per-layer
        9-tuples (:696-698, :911-916); prefill when past_key_values is None.  attention_mask: HF padding mask
        [B, kv_len] or an additive [B, 1, q_len, kv_len].  The result unpacks as (logits, past_key_values) and has the
        attributes of CausalLMOutputWithPast; with return_dict=True (or config.use_return_dict) it IS one."""
        if self.tensor_parallel:
            raise NotImplementedError("forward() returns the reference's per-layer 9-tuples, which hold every head; a "
                                      "tensor-parallel rank holds its share: use generate / decode_step / serve")
        B, q_len = input_ids.shape
        if past_key_values is not None and len(past_key_values) == 0:
            past_key_values = None
        start = 0 if past_key_values is None else past_key_values[0][-1]
        fused = self._fused_forward_ok(input_ids, past_key_values, attention_mask, position_ids, start)
        if fused:
            logits, pasts = self._forward_fused(input_ids, past_key_values, start)
        else:
            if past_key_values is not None and isinstance(past_key_values[0], KiviPast):
                past_key_values = [tuple(p.materialise()) for p in past_key_values]     # leave the fused path: plain 9-tuples
            if position_ids is None:
                position_ids = torch.arange(start, start + q_len, device=input_ids.device).unsqueeze(0).expand(B, -1)
            rows = self._tables(input_ids.device)[0].shape[0]
            if start + q_len > rows:            # the slow path's index_select would raise; say why
                raise ValueError(f"{start + q_len} positions exceed config.max_position_embeddings = {rows}")
            dtype = self.lm_head.weight.dtype
            mask = None
            if past_key_values is None:                                   # the prompt: the kernel's mask where it applies
                mask = self._tuple_prompt_mask(attention_mask, B, q_len, input_ids.device)
            if mask is None:
                mask = _additive_mask(attention_mask, q_len, start + q_len, dtype, input_ids.device, self.sliding_window, B)
            h, pasts = self._run_layers(input_ids, position_ids, past_key_values, mask, adapters=self._rows_for(B))
            logits = self.lm_head(h).float()                                     # logits.float() (:881)
        if return_dict is None:
            return_dict = getattr(self.config, "use_return_dict", False)
        if return_dict:
            from transformers.modeling_outputs import CausalLMOutputWithPast
            return CausalLMOutputWithPast(loss=None, logits=logits, past_key_values=tuple(pasts))
        return _Output((logits, pasts))

    def _kernel_mask(self, starts, n: int, device):
        """The PromptMask of a prompt at positions 0 .. n-1 whose sequences start at `starts` (int32 [B] on `device`, or
        None: no padding), or None where the prompt-attention kernel does not apply: weights other than fp16 on CUDA, a
        head_dim other than 128, or nothing to mask (no padding, and no sliding window shorter than the prompt).  The
        masks the model would otherwise build with _additive_mask -- left padding, a window that cuts the prompt, or
        both -- are exactly these."""
        cut = self.sliding_window is not None and n > self.sliding_window
        if (device.type != "cuda" or self.lm_head.weight.dtype != torch.float16
                or self.model.layers[0].self_attn.head_dim != 128 or (starts is None and not cut)):
            return None
        return PromptMask(None if starts is None else starts.to(device), self.sliding_window if cut else 0)

    def _tuple_prompt_mask(self, attention_mask, B: int, n: int, device):
        """The PromptMask of forward()'s prompt on the 9-tuple path, or None to keep the additive mask.  Only masks the
        kernel's rule states exactly go to it: no mask, an all-ones [B, n] mask, or a left-padding [B, n] mask (then with
        the sequences' starts) -- each with the window when it cuts the prompt.  A 4-D mask, a 2-D mask that is not left
        padding (right padding, holes, a row with no real token) or of another shape keeps _additive_mask, which applies
        it as given together with the window."""
        if attention_mask is None:
            return self._kernel_mask(None, n, device)
        if attention_mask.dim() != 2 or tuple(attention_mask.shape) != (B, n):
            return None
        try:
            starts = kv_start_from_mask(attention_mask)
        except ValueError:
            return None
        return self._kernel_mask(starts if bool(starts.any()) else None, n, device)

    # ------------------------------------------------------------------ forward() on the fused cache path
    fused_forward = True        # False: forward() always uses the reference's own 9-tuples (torch.cat growth, per-op launches)

    def _fused_forward_ok(self, input_ids, past_key_values, attention_mask, position_ids, start):
        """forward() may run on the pre-allocated cache when nothing asks for what only the tuple path offers: CUDA fp16
        weights, head_dim 128, equal-length sequences (no padding mask), default positions, and -- with a past -- one new
        token."""
        if not (self.fused_forward and input_ids.is_cuda and self.lm_head.weight.dtype == torch.float16
                and self.model.layers[0].self_attn.head_dim == 128):
            return False
        B, q_len = input_ids.shape
        if attention_mask is not None and (attention_mask.dim() != 2 or not bool(attention_mask.to(torch.bool).all())):
            return False
        if position_ids is not None:
            exp = torch.arange(start, start + q_len, device=position_ids.device).unsqueeze(0).expand(B, -1)
            if position_ids.shape != exp.shape or not bool((position_ids == exp).all()):
                return False
        if past_key_values is None:
            return True
        if q_len != 1 or len(past_key_values) != len(self.model.layers):
            return False
        if isinstance(past_key_values[0], KiviPast):
            return all(isinstance(p, KiviPast) and p.cache is self.cache and p.kv_len == self.cache.kv_len
                       for p in past_key_values)
        return past_key_values[0][5] is not None and past_key_values[0][5].shape[0] == B      # plain 9-tuples: import once

    def _forward_fused(self, input_ids, past_key_values, start):
        B, q_len = input_ids.shape
        n_layers = len(self.model.layers)
        reserve = int(getattr(self.config, "kivi_cache_reserve", 1024))      # head-room allocated beyond the current length
        if past_key_values is None:                                          # prefill into the blocked cache
            if self.cache is None or self.cache.batch != B or self.cache.max_tokens < q_len + 1:
                self.init_cache(B, q_len + reserve)
            logits = self.lm_head(self._prompt_pass(input_ids)).float()
        else:
            if not isinstance(past_key_values[0], KiviPast):                 # a cache grown elsewhere (reference hook): one re-layout
                self.import_cache(past_key_values, max_tokens=start + reserve)
            elif self.cache.kv_len + 1 > self.cache.max_tokens:              # out of room: re-allocate at twice the size
                tuples = [self.cache.export(i) for i in range(n_layers)]
                self.import_cache(tuples, max_tokens=2 * self.cache.max_tokens)
            logits = self.decode_step(input_ids).unsqueeze(1).clone()
        kv = self.cache.kv_len
        return logits, [KiviPast(self.cache, i, kv) for i in range(n_layers)]

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None,
                                      **kwargs):
        """models/llama_kivi.py:908-948: feed only the tokens the cache has not seen (its length is the last element
        of a layer's tuple), positions from the padding mask."""
        if past_key_values is not None and len(past_key_values) == 0:
            past_key_values = None
        if past_key_values is not None:
            seen = past_key_values[0][-1]
            drop = seen if input_ids.shape[1] > seen else input_ids.shape[1] - 1
            input_ids = input_ids[:, drop:]
        position_ids = kwargs.get("position_ids")
        if attention_mask is not None and position_ids is None:
            position_ids = attention_mask.long().cumsum(-1) - 1
            position_ids.masked_fill_(attention_mask == 0, 1)
            if past_key_values:
                position_ids = position_ids[:, -input_ids.shape[1]:]
        return {"input_ids": input_ids, "position_ids": position_ids, "past_key_values": past_key_values,
                "use_cache": kwargs.get("use_cache"), "attention_mask": attention_mask}

    @staticmethod
    def _reorder_cache(past_key_values, beam_idx):
        """models/llama_kivi.py:950-957 (beam search): select batch rows of every tensor of every layer's tuple; the
        reference's version fails on the None entries and the trailing int of the 9-tuple -- they pass through here.
        Views of the fused cache (KiviPast, every layer, one cache at its current length) stay on the fused path: the cache
        reorders its rows on the device (KiviCache.reorder) and fresh views are returned."""
        if past_key_values and all(isinstance(p, KiviPast) for p in past_key_values):
            cache = past_key_values[0].cache
            if all(p.cache is cache and p.kv_len == cache.kv_len for p in past_key_values):
                cache.reorder(beam_idx)
                return tuple(KiviPast(cache, p.layer, cache.kv_len) for p in past_key_values)
        return tuple(tuple(t.index_select(0, beam_idx.to(t.device)) if torch.is_tensor(t) else t for t in layer_past)
                     for layer_past in past_key_values)

    # ------------------------------------------------------------------ fused cache path
    def init_cache(self, batch: int, max_tokens: int):
        """Allocate the fused KIVI cache for `batch` sequences of up to `max_tokens` tokens.  The fused path runs fp16
        weights only (ValueError otherwise: convert the model with .half())."""
        cfg = self.config
        dev, dtype = self.lm_head.weight.device, self.lm_head.weight.dtype
        if dtype != torch.float16:
            raise ValueError(f"the fused KIVI cache path needs fp16 weights, the model's are {dtype}: call .half() first")
        n_top = None if self.choice is None else self.choice.n_top
        self.cache, self._graph, self.choice = None, None, None   # release the previous cache before the new one is allocated
        a = self.model.layers[0].self_attn                  # this rank's heads
        self.cache = KiviCache(cfg.num_hidden_layers, batch, a.num_heads, a.num_key_value_heads,
                               a.head_dim, cfg.k_bits, cfg.v_bits, cfg.group_size,
                               cfg.residual_length, max_tokens, device=dev,
                               overlap_prologue=True,       # the attention call follows the layer's RoPE kernel
                               sliding_window=self.sliding_window)
        if self.tensor_parallel:
            self.cache.tensor_parallel = True
            if self._allreduce is None or self._allreduce.rows_max != batch:
                from . import dist as kdist
                self._allreduce = None
                self._allreduce = kdist.PeerAllReduce(batch, cfg.hidden_size, dev)
        self._graph, self._graph_ragged, self._reorder_graph = None, False, None
        self._pos = torch.zeros((batch, 1), dtype=torch.long, device=dev)
        self._ids = torch.zeros((batch, 1), dtype=torch.long, device=dev)
        self._logits = torch.zeros((batch, cfg.vocab_size), dtype=torch.float32, device=dev)
        self.next_tokens = torch.zeros((batch,), dtype=torch.long, device=dev)   # the step's argmax or sample (in-graph)
        # greedy and without processing until set_sampling() / set_processing(); the logprobs mode outlives the cache
        self.choice = TokenChoice(batch, cfg.vocab_size, dev)
        self.choice.set_logprobs(n_top)
        self._tables(dev)                                   # rows for every position the cache can reach
        self._adapter_idx = torch.full((batch,), -1, dtype=torch.int32, device=dev)
        if self._lora is not None:
            self.cache.adapter_idx = self._adapter_idx       # KiviCache.reorder gathers it with the rows
            sel = self._adapter_sel
            if isinstance(sel, int):
                self._adapter_idx.fill_(sel)
            elif sel is not None and len(sel) == batch:
                self._adapter_idx.copy_(torch.tensor(sel, dtype=torch.int32))
        return self.cache

    def import_cache(self, past_key_values, max_tokens: int | None = None):
        """Continue on the fused path from the reference's per-layer 9-tuples (models/llama_kivi.py:454-455)."""
        if self.tensor_parallel:
            raise NotImplementedError("import_cache: the reference's 9-tuples hold every head; a tensor-parallel rank "
                                      "holds its share")
        seen = past_key_values[0][-1]
        B = past_key_values[0][5].shape[0]
        if self.cache is None or self.cache.batch != B or max(max_tokens or 0, seen + 1) > self.cache.max_tokens:
            self.init_cache(B, max(max_tokens or 0, seen + 1024))
        for i, past in enumerate(past_key_values):
            self.cache.import_tuple(i, past)
        self._pos.fill_(seen)
        return self.cache

    @torch.no_grad()
    def prefill(self, input_ids, attention_mask=None):
        """Run the prompt, fill the cache (models/llama_kivi.py:401-452), return last-position logits.
        attention_mask: None or an HF padding mask [B, n] of a LEFT-padded batch (ValueError otherwise).  The prompt
        attention then skips each sequence's padding (kivi_prompt_attention_f16 with the sequences' starts; the additive
        mask of the tuple path for weights other than fp16), positions follow HF (cumsum - 1, pad positions 1), and
        the decode steps skip each sequence's padding (KiviCache.set_kv_start).  An all-ones mask is no mask.  Every
        prompt, a one-token one included, replaces what the cache held."""
        assert self.cache is not None, "call init_cache() first"
        return self.lm_head(self._prompt_pass(input_ids, attention_mask)[:, -1]).float()

    def _prompt_pass(self, input_ids, attention_mask=None, copies: int = 1):
        """prefill() up to the final norm: the hidden states [B, n, hidden] of every position.  copies = K: the layers run
        on the B prompts once and the cache's rows b * K .. b * K + K - 1 (the beams or samples of prompt b) each receive
        prompt b's K / V, starts and positions."""
        B, n = input_ids.shape
        store = self.cache.prefill
        if copies > 1:
            def store(layer, k, v):
                self.cache.prefill(layer, k.repeat_interleave(copies, 0), v.repeat_interleave(copies, 0))
        starts = None
        if attention_mask is not None:
            starts = kv_start_from_mask(attention_mask)
            if not bool(starts.any()):
                starts = None
        self.choice.mark_prompt(input_ids, starts, slice(None), copies)
        rows = None if self._lora is None else self._adapter_idx[::copies].contiguous()     # prompt b's adapter
        if starts is None:
            positions = torch.arange(n, device=input_ids.device).unsqueeze(0).expand(B, -1)
            mask = self._kernel_mask(None, n, input_ids.device)
            if mask is None:
                mask = _additive_mask(None, n, n, self.lm_head.weight.dtype, input_ids.device, self.sliding_window, B)
            h, _ = self._run_layers(input_ids, positions, None, mask, store_kv=store, adapters=rows)
            self._pos.fill_(n)
        else:
            am = attention_mask.to(input_ids.device)
            positions = am.long().cumsum(-1) - 1                            # prepare_inputs_for_generation (:908-948)
            positions.masked_fill_(am == 0, 1)
            mask = self._kernel_mask(starts, n, input_ids.device)
            if mask is None:
                mask = _additive_mask(am, n, n, self.lm_head.weight.dtype, input_ids.device, self.sliding_window)
            h, _ = self._run_layers(input_ids, positions, None, mask, store_kv=store, adapters=rows)
            starts = starts.to(self._pos.device).repeat_interleave(copies)
            self._pos.copy_((n - starts).to(torch.long).view(B * copies, 1))
            self.cache.set_kv_start(starts)
        return h

    @torch.no_grad()
    def insert(self, seq: int, prompt_ids, prefix_cache=None, adapter=None):
        """Start a new sequence in slot `seq` of the running batch (continuous batching): a B = 1 prompt pass at positions
        0 .. n-1 whose K/V go into that slot right-aligned to the shared length T (KiviCache.refill), then
        kv_start[seq] = T - n and the slot's position = n.  The other slots are not touched.  Returns the prompt's
        last-position logits [vocab] fp32; the caller writes the first token into the slot's input (`_ids[seq]`).
        prefix_cache: a kivi_b200.prefix.PrefixCache.  When it holds the prompt's first r >= MIN_REUSE tokens (r <= n - 1,
        prefix.reuse_length), the pass runs on tokens r .. n-1 only, at positions r .. n-1, over the stored K / V and
        its own (PrefixMask); otherwise it runs the whole prompt as without a cache.  Either way the prompt's tokens past
        the stored path are stored.  A stored prefix is reused only under the adapter it was stored with.
        adapter: the name of a loaded LoRA adapter for the new sequence (load_adapter), or None for none."""
        assert self.cache is not None, "call init_cache() / prefill() first"
        ids = torch.as_tensor(prompt_ids, device=self.cache.device).reshape(1, -1)
        n, T = ids.shape[1], self.cache.kv_len
        if not 1 <= n <= T:
            raise ValueError(f"a prompt of {n} tokens does not fit the shared length {T} (1 <= n <= length)")
        rows = None
        if self._lora is not None:
            self._adapter_idx[seq] = self._lora.slot(adapter)
            rows = self._adapter_idx[seq:seq + 1]
        elif adapter is not None:
            raise ValueError(f"adapter {adapter!r}: no LoRA adapter is loaded (load_adapter)")
        r, store = 0, lambda layer, k, v: self.cache.refill(layer, seq, k, v)       # noqa: E731
        if prefix_cache is not None:
            r, store, record = self._prefix_insert(prefix_cache, ids, store, adapter)
        positions = torch.arange(r, n, device=ids.device).unsqueeze(0)
        mask = self._kernel_mask(None, n, ids.device)
        if r:
            mask = PrefixMask(PromptMask(None, 0) if mask is None else mask,
                              self._prefix_extend(prefix_cache, record[1], r, n))
        elif mask is None:
            mask = _additive_mask(None, n, n, self.lm_head.weight.dtype, ids.device, self.sliding_window)
        h, _ = self._run_layers(ids[:, r:], positions, None, mask, store_kv=store, adapters=rows)
        if prefix_cache is not None:
            prefix_cache.insert(*record)
        self._pos[seq] = n
        self.cache.set_seq_start(seq, T - n)
        self.choice.mark_prompt(ids, None, slice(seq, seq + 1))
        return self.lm_head(h[0, -1]).float()

    def _prefix_insert(self, prefix_cache, ids, refill, adapter=None):
        """insert()'s use of a PrefixCache: bind it, find the prompt's stored prefix and reserve room for the rest.
        Returns r (the tokens to reuse, 0 for none), the store_kv that refills the slot and copies the new tokens' K / V
        into the reserved storage, and the arguments of prefix_cache.insert once the pass is done."""
        from .prefix import reuse_length
        a = self.model.layers[0].self_attn
        prefix_cache.bind(self, len(self.model.layers), a.num_key_value_heads, ids.device)
        tokens = ids[0].tolist()
        n = len(tokens)
        match = prefix_cache.match(tokens, adapter)
        r = reuse_length(match.length, n)
        if r:
            prefix_cache.hits += 1
            prefix_cache.reused_tokens += r
        storage = prefix_cache.reserve(match, n - match.length)
        store = refill
        if storage is not None:
            def store(layer, k, v):
                storage[layer, 0].copy_(k[0, :, match.length:])
                storage[layer, 1].copy_(v[0, :, match.length:])
                refill(layer, k, v)
        return r, store, (tokens, match, storage, adapter)

    @staticmethod
    def _prefix_extend(prefix_cache, match, r: int, n: int):
        """PrefixMask.extend of an insert that reuses r stored tokens of an n-token prompt: per layer, a fresh
        [1, Hkv, n, 128] K and V holding the stored prefix, then the suffix's k / v [1, Hkv, n - r, 128]."""
        def extend(layer, k, v):
            kk = k.new_empty((1, k.shape[1], n, k.shape[3]))
            vv = torch.empty_like(kk)
            prefix_cache.copy_prefix(match, r, layer, kk[0], vv[0])
            kk[:, :, r:].copy_(k)
            vv[:, :, r:].copy_(v)
            return kk, vv
        return extend

    def release(self, seq: int):
        """Make slot `seq` idle (KiviCache.release): it keeps its row of every step but reads no cached byte."""
        self.cache.release(seq)
        self._pos[seq] = 0
        if self._lora is not None:
            self._adapter_idx[seq] = -1
        self.choice.release(seq)

    @torch.no_grad()
    def prefill_synthetic(self, n: int, seed: int = 0):
        """Fill every layer's cache with n random K/V tokens (benchmarks: the prompt's attention itself is
        off the decode hot path; the cache contents are produced by the real prefill pack kernels)."""
        assert self.cache is not None
        c = self.cache
        gen = torch.Generator(device=c.device).manual_seed(seed)
        for l in range(c.n_layers):
            k = torch.randn((c.batch, c.num_kv_heads, n, c.head_dim), generator=gen, device=c.device, dtype=torch.float16)
            v = torch.randn((c.batch, c.num_kv_heads, n, c.head_dim), generator=gen, device=c.device, dtype=torch.float16)
            c.prefill(l, k, v)
        self._pos.fill_(n)

    def enable_token_allgather(self, world_size: int, in_graph: bool = True, mode: str = "nccl"):
        """Data-parallel replicas (kivi_b200.dist): every rank's sampled ids end up in `all_tokens` [world_size * B].
        mode "p2p": the sampling kernel itself stores the ids into every peer's symmetric buffer (PeerTokenExchange; one
        fused compute + collective kernel inside the step's CUDA graph).  mode "nccl": an NCCL all-gather of the ids, inside
        the graph (in_graph) or right after the replay.  Call before the first decode_step (the step is captured once)."""
        if self.tensor_parallel:
            raise NotImplementedError("data-parallel replicas of a tensor-parallel model are not supported")
        self._exchange, self._dist_tokens = None, None
        if world_size > 1 and mode == "p2p":
            if self._sampling:
                raise NotImplementedError(_P2P_SAMPLING)
            from . import dist as kdist
            self._exchange = kdist.PeerTokenExchange(self.cache.batch, self.cache.device)
        elif world_size > 1:
            self._dist_tokens = torch.zeros(world_size * self.cache.batch, dtype=torch.long, device=self.cache.device)
        self._dist_in_graph = in_graph
        self._graph = None

    # ------------------------------------------------------------------ sampling
    def set_sampling(self, temperature=1.0, top_k=50, top_p=1.0, seed=0):
        """Sample the next token of every decode step on the device (kivi_sample_f32, the step's last kernel, inside its
        CUDA graph): temperature, then top-k, then top-p, then one draw.  Scalars, or one value per batch row; row b draws
        from the Philox stream of key seed + b (an int seed) or seed[b], starting at draw 0.  temperature 0 makes a row
        greedy.  set_sampling(None) returns the whole step to the greedy kernel.  The captured step is dropped when the
        mode changes, not when only parameters do.  Under tensor parallelism every rank calls this with the same arguments."""
        assert self.cache is not None, "call init_cache() first"
        if temperature is not None and self._exchange is not None:
            raise NotImplementedError(_P2P_SAMPLING)
        if self.choice.set_sampling(temperature, top_k, top_p, seed):
            self._graph = None

    def set_slot_sampling(self, seq: int, temperature=1.0, top_k=50, top_p=1.0, seed=0):
        """The sampling parameters of batch row `seq` alone (a slot given to a new request), its draw counter back to 0; the
        row's key is `seed` itself.  The captured step reads them on the device: no recapture."""
        self.choice.set_slot_sampling(seq, temperature, top_k, top_p, seed)

    def sample_first(self, logits, seq: int | None = None):
        """first_tokens() under sampling: the prompt's last-position logits ([B, vocab] of prefill, or [vocab] of
        insert(seq)) go through the step's own sampling kernel with the rows' parameters and consume their next draw
        (draw 0 after set_sampling / set_slot_sampling).  Rank 0's ids under tensor parallelism, like first_tokens."""
        if not self._sampling:
            raise RuntimeError("sample_first: the step is greedy; call set_sampling() first")
        logits = logits.reshape(-1, logits.shape[-1]).float().contiguous()
        tok = torch.empty(logits.shape[0], dtype=torch.long, device=logits.device)
        tok = self._rank0(self.choice.sample(logits, slice(None) if seq is None else slice(seq, seq + 1), tok))
        return tok if seq is None else tok[0]

    # ------------------------------------------------------------------ logits processing
    def set_processing(self, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0, min_new_tokens=0,
                       eos_token_id=None, pad_token_id=None):
        """Process the logits of every decode step on the device before the token choice (kivi_logits_process_f32 and, after
        the choice, kivi_logits_record, inside the step's CUDA graph): the repetition penalty over the prompt's and the
        generated tokens, the frequency and presence penalties over the generated ones, EOS suppression while a row has
        fewer than min_new_tokens new tokens, and after a row's EOS only pad_token_id (default: the first EOS id).  The
        greedy kernel or the sampler then chooses from the processed scores; decode_step still returns the raw logits.
        Scalars, or one value per batch row (processing_rows); eos_token_id: an int or up to 8 ids, for every row.
        Call before prefill() / insert(): they record the prompt tokens and reset the rows' counts, lengths and flags.
        set_processing(None) returns the step to what it was without processing and frees the state.  The captured step is
        dropped when processing turns on or off or pad_token_id changes, not when the other parameters do.  Under tensor
        parallelism every rank calls this with the same arguments."""
        assert self.cache is not None, "call init_cache() first"
        if self.choice.set_processing(repetition_penalty, presence_penalty, frequency_penalty, min_new_tokens, eos_token_id,
                                      pad_token_id):
            self._graph = None

    def set_slot_processing(self, seq: int, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0,
                            min_new_tokens=0):
        """The processing parameters of batch row `seq` alone (a slot given to a new request); its counts, length and flag
        are reset by insert().  The captured step reads them on the device: no recapture."""
        self.choice.set_slot_processing(seq, repetition_penalty, presence_penalty, frequency_penalty, min_new_tokens)

    def choose_first(self, logits, seq: int | None = None, return_scores: bool = False):
        """The first token(s) from the prompt's last-position logits ([B, vocab] of prefill, or [vocab] of insert(seq)), as
        the decode step chooses: processed (set_processing) with the rows' state, then the argmax (first_tokens) or a draw
        (sample_first), then recorded; with set_logprobs() on, the rows' logprobs buffers receive the raw log-probabilities
        of these tokens.  Returns [B] ids, or a 0-d id for `seq`; return_scores: (ids, the scores the choice read, in the
        shape of `logits`: the processed ones, or `logits` itself with processing off)."""
        flat = logits.reshape(-1, logits.shape[-1]).float().contiguous()

        def pick(scores):
            if self._sampling:
                return self.sample_first(scores, seq)
            return self.first_tokens(scores if seq is None else scores[0])
        tok, scores = self.choice.choose(flat, slice(None) if seq is None else slice(seq, seq + 1), pick)
        if not return_scores:
            return tok
        return tok, logits if scores is None else scores if seq is None else scores[0]

    # ------------------------------------------------------------------ log-probabilities
    def set_logprobs(self, n_top=0):
        """Log-probabilities of the chosen tokens, computed inside every decode step (kivi_token_logprobs_f32, after the
        token choice, inside the step's CUDA graph) and by choose_first for the first token: `logprobs` [B] fp32 receives
        each row's log-probability of its new token and `top_ids` [B, n_top] int64 / `top_logprobs` [B, n_top] fp32 the row's
        n_top most likely tokens (descending, ties by ascending id), 0 <= n_top <= 20.  These are raw log-probabilities, the
        log-softmax of the logits decode_step() returns: before logits processing, temperature, top-k and top-p.  The
        buffers are static, overwritten by the next step, and reallocated for the new batch by init_cache(), which keeps
        the mode (so does generate(), which may call it).  set_logprobs(None) turns the mode off and frees them; the
        captured step is dropped when the mode turns on or off or n_top changes.  Under tensor parallelism every rank
        computes the same values (the logits are replicated)."""
        assert self.cache is not None, "call init_cache() first"
        if self.choice.set_logprobs(n_top):
            self._graph = None

    logprobs = property(lambda self: None if self.choice is None else self.choice.logprobs)
    top_ids = property(lambda self: None if self.choice is None else self.choice.top_ids)
    top_logprobs = property(lambda self: None if self.choice is None else self.choice.top_logprobs)
    _sampling = property(lambda self: self.choice.sampling)     # the token choice's modes and state, read by the step
    _samp = property(lambda self: self.choice.samp)
    _proc = property(lambda self: self.choice.proc)

    # ------------------------------------------------------------------ LoRA adapters
    def load_adapter(self, path, adapter_name: str):
        """Load the PEFT LoRA adapter in the local directory `path` under `adapter_name` (kivi_b200.lora: what is supported
        and what is refused with a ValueError).  It is stacked beside the other loaded adapters on the model's device; the
        base weights are not touched.  Rows choose it with set_adapters, insert(adapter=), generate(adapter=) or a serve()
        request's "adapter".  Once an adapter is loaded the decode step adds two LoRA launches per projection group (8 per
        layer); rows without an adapter come out bit-equal to the step without them.  The captured steps are dropped.
        Load adapters after moving the model to its device and dtype.  NotImplementedError under tensor_parallel."""
        if self.tensor_parallel:
            raise NotImplementedError("load_adapter: LoRA under tensor parallelism (sharded A / B and their reduction) is "
                                      "not supported")
        from . import lora
        adapter = lora.read_adapter(path, self.config)                    # every check before anything changes
        state = self._lora if self._lora is not None else lora.LoraState(self.config, self.lm_head.weight.device)
        state.load(adapter_name, adapter)
        self._lora = state
        self._graph = self._reorder_graph = None
        if self.cache is not None:
            self.cache.adapter_idx = self._adapter_idx
        return state.names[adapter_name]

    @property
    def adapters(self):
        """The names of the loaded LoRA adapters, in slot order."""
        return [] if self._lora is None else list(self._lora.names)

    def set_adapters(self, adapters=None):
        """The LoRA adapter of every batch row: None (none), one name for every row, or a list of one name (or None) per
        row of the cache.  forward(), prefill() and the decode step read it; init_cache() keeps a selection that fits the
        new batch.  Unknown names are a KeyError, a list of the wrong length a ValueError."""
        if adapters is None:
            sel = None
        elif self._lora is None:
            raise ValueError("set_adapters: no LoRA adapter is loaded (load_adapter)")
        elif isinstance(adapters, str):
            sel = self._lora.slot(adapters)
        else:
            sel = [self._lora.slot(a) for a in adapters]
            if self.cache is not None and len(sel) != self.cache.batch:
                raise ValueError(f"set_adapters: {len(sel)} names for a batch of {self.cache.batch}")
        self._adapter_sel = sel
        if self._adapter_idx is not None:
            if sel is None or isinstance(sel, int):
                self._adapter_idx.fill_(-1 if sel is None else sel)
            else:
                self._adapter_idx.copy_(torch.tensor(sel, dtype=torch.int32))

    def _rows_for(self, B: int):
        """The adapter slot of each of B rows of a forward() pass (None: no adapter loaded or selected)."""
        if self._lora is None:
            return None
        if self.cache is not None and self.cache.batch == B:
            return self._adapter_idx
        sel = self._adapter_sel
        if sel is None:
            return None
        if isinstance(sel, int):
            sel = [sel] * B
        if len(sel) != B:
            raise ValueError(f"set_adapters named {len(sel)} rows, the batch has {B}")
        return torch.tensor(sel, dtype=torch.int32)

    def _lora_ws(self):
        """The decode step's LoRA workspace: fp32, the largest of the four groups' needs at this batch and rank."""
        from . import glue
        from .lora import GROUPS
        lo, B = self._lora, self.cache.batch
        need = max(glue.lora_workspace_bytes(B, lo.shapes[mods[0]][1], len(mods), lo.rank) for mods in GROUPS.values())
        ws = getattr(self._fast, "lora_ws", None)
        if ws is None or ws.numel() * 4 < need:
            ws = self._fast.lora_ws = torch.empty(need // 4, dtype=torch.float32, device=self.cache.device)
        return ws

    @property
    def all_tokens(self):
        if self._exchange is not None:
            return self._exchange.tokens()
        return self.next_tokens if self._dist_tokens is None else self._dist_tokens

    def _ensure_fast(self):
        """Fused q|k|v, o and gate|up weights in [in, out] layout, the fused q|k|v bias (None without attention biases)
        + static activation buffers for the 9-launch-per-layer step.  At M = B rows cuBLAS streams the weights faster from
        this layout (tools/gemm_probe.py compares the two layouts; down is layout-neutral).  The fused buffers OWN the
        storage: the nn.Linear parameters become (transposed) views of them, so there is one copy of every weight (the
        reference's mem_spd_test reports peak memory) and load_state_dict / in-place edits reach the decode path."""
        if self._fast is not None and self._fast.B == self.cache.batch:
            return self._fast
        cfg, dev, B = self.config, self.cache.device, self.cache.batch
        a0 = self.model.layers[0].self_attn                                  # this rank's shapes (all of them at world 1)
        H, Hkv, hid = a0.num_heads, a0.num_key_value_heads, cfg.hidden_size
        inter = self.model.layers[0].mlp.gate_proj.weight.shape[0]
        f = self._fast if self._fast is not None else SimpleNamespace(wqkv=None)
        f.B = B
        if f.wqkv is None:
            def view_param(buf, lo, hi):
                return nn.Parameter(buf.t()[lo:hi], requires_grad=False)
            f.wqkv, f.bqkv, f.wgu, f.wo = [], [], [], []
            for l in self.model.layers:
                a, m = l.self_attn, l.mlp
                nq, nk = a.q_proj.weight.shape[0], a.k_proj.weight.shape[0]
                w = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0).t().contiguous()
                a.q_proj.weight, a.k_proj.weight = view_param(w, 0, nq), view_param(w, nq, nq + nk)
                a.v_proj.weight = view_param(w, nq + nk, w.shape[1])
                f.wqkv.append(w)
                b = None
                if a.q_proj.bias is not None:
                    b = torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias])
                    a.q_proj.bias, a.k_proj.bias = view_param(b, 0, nq), view_param(b, nq, nq + nk)
                    a.v_proj.bias = view_param(b, nq + nk, b.shape[0])
                f.bqkv.append(b)
                w = torch.cat([m.gate_proj.weight, m.up_proj.weight], 0).t().contiguous()
                m.gate_proj.weight, m.up_proj.weight = view_param(w, 0, inter), view_param(w, inter, 2 * inter)
                f.wgu.append(w)
                w = a.o_proj.weight.t().contiguous()
                a.o_proj.weight = view_param(w, 0, w.shape[1])
                f.wo.append(w)
        e = lambda *shape: torch.empty(shape, dtype=torch.float16, device=dev)  # noqa: E731
        f.res, f.h, f.o, f.d = e(B, hid), e(B, hid), e(B, hid), e(B, hid)
        f.qkv, f.q, f.k, f.v = e(B, (H + 2 * Hkv) * 128), e(B, H, 128), e(B, Hkv, 128), e(B, Hkv, 128)
        f.attn, f.gu, f.act = e(B, H, 128), e(B, 2 * inter), e(B, inter)
        f.logits16 = e(B, cfg.vocab_size)
        self._fast = f
        return f

    def _step_body(self):
        """One decode step with 9 launches per layer: 4 cuBLAS GEMMs (q|k|v, o, gate|up, down), RoPE+split (Qwen3's
        q_norm / k_norm folded in), fused KIVI attention, SiLU*mul and two residual-add+RMSNorm kernels; then lm_head, the cache advance and the argmax
        or sampling kernel, which set_processing() frames with the logits-processing kernel before it and the record
        kernel after it; set_logprobs() adds the log-probability kernel after the choice.  A model with attention biases adds them in the q|k|v and o GEMMs (addmm).
        Tensor-parallel (self._allreduce is a PeerAllReduce): the same launches on this rank's heads and channels, but o_proj
        and down_proj write their partial sums into the PeerAllReduce slots, and the two residual-add + RMSNorm kernels of a
        layer become kivi_allreduce_add_rmsnorm_f16 (calls 2i and 2i + 1 of the step), which add up every rank's partials.
        The embedding's RMSNorm and lm_head are replicated: every rank computes the same logits."""
        from . import glue
        f, ar = self._ensure_fast(), self._allreduce
        cfg, cache = self.config, self.cache
        cos_t, sin_t = self._tables(cache.device)
        eps = cfg.rms_norm_eps
        layers = self.model.layers

        def partial(call):                      # where o_proj (call 2i of the step) or down_proj (2i + 1) writes
            return (f.o, f.d)[call & 1] if ar is None else ar.slot(call, f.B)

        def add_rmsnorm(call, weight):          # f.res += the sum of the call's partials; f.h = RMSNorm(f.res) * weight
            if ar is None:
                glue.add_rmsnorm(partial(call), f.res, weight, f.h, eps)
            else:
                glue.allreduce_add_rmsnorm(f.res, weight, f.h, eps, ar, call=call)

        def linear(x, w, bias, out):
            if bias is None:
                torch.mm(x, w, out=out)
            else:
                torch.addmm(bias, x, w, out=out)

        lo = self._lora
        if lo is not None:                                   # LoRA: shrink + expand after each GEMM, 8 launches per layer
            ws = self._lora_ws()

            def lora(i, group, x, y):
                A, B = lo.stacks[i][group]
                glue.lora_apply(x, y, A, B, lo.scale, lo.segs[group], self._adapter_idx, ws)
        else:
            def lora(i, group, x, y):
                pass

        f.res.copy_(self.model.embed_tokens(self._ids)[:, 0])
        glue.add_rmsnorm(None, f.res, layers[0].input_layernorm.weight, f.h, eps)
        for i, l in enumerate(layers):
            linear(f.h, f.wqkv[i], f.bqkv[i], f.qkv)
            lora(i, "qkv", f.h, f.qkv)                       # after the bias, before q_norm / RoPE (as PEFT)
            a = l.self_attn
            if a.q_norm is None:
                glue.rope_split(f.qkv, cos_t, sin_t, self._pos, f.q, f.k, f.v)
            else:                                            # the same kernel, normalising each q / k head first
                glue.rope_split(f.qkv, cos_t, sin_t, self._pos, f.q, f.k, f.v, a.q_norm.weight, a.k_norm.weight,
                                a.q_norm.variance_epsilon)
            cache.decode_attention(i, f.q, f.k, f.v, out=f.attn)
            linear(f.attn.view(f.B, -1), f.wo[i], l.self_attn.o_proj.bias, partial(2 * i))
            lora(i, "o", f.attn.view(f.B, -1), partial(2 * i))
            add_rmsnorm(2 * i, l.post_attention_layernorm.weight)
            torch.mm(f.h, f.wgu[i], out=f.gu)
            lora(i, "gu", f.h, f.gu)
            glue.silu_mul(f.gu, f.act)
            torch.mm(f.act, l.mlp.down_proj.weight.t(), out=partial(2 * i + 1))
            lora(i, "down", f.act, partial(2 * i + 1))
            nxt = layers[i + 1].input_layernorm.weight if i + 1 < len(layers) else self.model.norm.weight
            add_rmsnorm(2 * i + 1, nxt)
        if ar is not None:
            ar.epoch.add_(2 * len(layers))                                   # the next step's calls continue the count
        torch.mm(f.h, self.lm_head.weight.t(), out=f.logits16)
        self._logits.copy_(f.logits16)                                       # logits.float() (:881)
        cache._enqueue_advance()                             # decode_step advances the host mirror after each replay
        self._pos.add_(1)

        # greedy sampling inside the step (and inside its CUDA graph): the argmax of a sequence needs only that
        # sequence's logits, so with data-parallel replicas the exchange is the sampled ids, 8 B per sequence
        def pick(scores):
            if self._sampling:            # in the argmax kernel's place, one kernel as well: a draw per sequence
                return self.choice.sample(scores, slice(None), self.next_tokens, self._ids.view(-1))
            if self._exchange is not None:
                self._exchange.step.add_(1)                  # the step number the peers' arrival counters are compared with
            # one kernel: argmax per sequence, the feed-back copy for the next step, and (replicas) the ids stored straight
            # into every peer's buffer over NVLink + arrival counters
            return glue.greedy_sample(scores, self.next_tokens, self._ids.view(-1), self._exchange)
        # with processing, the choice reads the processed scores; decode_step returns the raw logits
        self.choice.choose(self._logits, None, pick)
        if self._dist_tokens is not None and self._dist_in_graph:
            from . import dist as kdist
            kdist.gather_tokens(self.next_tokens, out=self._dist_tokens)

    def first_tokens(self, logits):
        """Greedy ids of prompt logits (prefill / insert) -- under tensor parallelism rank 0's, broadcast, so the ranks can
        never start from different tokens."""
        return self._rank0(logits.argmax(-1))

    def _rank0(self, tok):
        if self.tensor_parallel and self.tp_world > 1:
            import torch.distributed as dist
            dist.broadcast(tok, src=0)
        return tok

    @torch.no_grad()
    def decode_step(self, input_ids=None, use_graph: bool = True):
        """One decode step for the whole batch: input_ids [B, 1] (device) -> logits [B, vocab] fp32 (device,
        a static buffer); `next_tokens` [B] holds their argmax, or after set_sampling() one sampled id per sequence (and
        `all_tokens` every rank's, see enable_token_allgather).  The step (32 x [norm, qkv, rope, fused KIVI attention,
        o_proj, MLP], lm_head, cache advance, argmax or sampling, token all-gather) is captured once in a CUDA graph and
        replayed."""
        assert self.cache is not None
        if self.cache.kv_len + 1 > self.cache.max_tokens:
            raise ValueError("KIVI cache capacity exceeded")
        if input_ids is not None:
            self._ids.copy_(input_ids.view(-1, 1))
        if not use_graph:
            self._step_body()
        else:
            if self._graph is not None and self._graph_ragged != self.cache.ragged:
                self._graph = None                                           # captured with the other attention entry
            if self._graph is None:
                # warm-up on a side stream (cuBLAS workspaces, lazy module loading, NCCL channels), then capture
                saved = self.choice.snapshot(self.cache.state, self._pos, self._ids)
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    self._step_body()
                torch.cuda.current_stream().wait_stream(s)
                torch.cuda.synchronize()
                # undo the warm-up step's effect on the lengths, positions, ids and token choice.  Everything it wrote
                # lies BEYOND the lengths -- the new token's window slots (K slot r, the free slot of the V ring), a flushed
                # K block past tk, the packed V token at tv -- and is rewritten with the same bytes by the first replay.
                self.choice.restore(saved)
                from . import _lib
                n0 = _lib.launch_count()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._step_body()
                self.launches_per_step = _lib.launch_count() - n0            # libkivi_b200 launches replayed by every step
                # capture does not execute: state is still the pre-step state
                self._graph, self._graph_ragged = g, self.cache.ragged
            self._graph.replay()
        if self._dist_tokens is not None and not self._dist_in_graph:
            from . import dist as kdist
            kdist.gather_tokens(self.next_tokens, out=self._dist_tokens)
        if self._allreduce is not None:
            self._allreduce.check()
        self.cache._mirror_advance()
        return self._logits

    def _roll(self):
        """Make room for one more step of a windowed model: drop the largest multiple of max(128, R) positions that no
        live sequence sees at the next step (KiviCache.live_starts) and that the packed stores hold."""
        c = self.cache
        if c.sliding_window is None:
            raise ValueError("KIVI cache capacity exceeded")
        q = max(128, c.residual_length)
        tokens = min([c.tk, c.tv] + list(c.live_starts().values())) // q * q
        if tokens <= 0:
            raise ValueError(f"KIVI cache capacity exceeded: no multiple of {q} positions lies below every window")
        c.shift(tokens)

    @torch.no_grad()
    def generate(self, input_ids=None, max_new_tokens: int | None = None, use_graph: bool = True, attention_mask=None,
                 max_length: int | None = None, do_sample: bool = False, temperature=1.0, top_k=50, top_p=1.0, seed=0,
                 num_beams: int = 1, num_return_sequences: int = 1, length_penalty: float = 1.0, early_stopping=False,
                 eos_token_id=None, pad_token_id=None, return_dict_in_generate: bool = False, repetition_penalty=None,
                 min_length: int | None = None, min_new_tokens: int | None = None, output_scores: bool = False,
                 output_logits: bool = False, adapter=None, **unused):
        """Decoding on the fused path with the call shape of HF generate (`model.generate(**inputs,
        max_new_tokens=n)`, example.py:60-61, mem_spd_test.py:66): returns [B, prompt + new] ids.  Greedy by default;
        do_sample=True samples every token, the first included, on the device with temperature / top_k / top_p (HF's
        defaults; scalars or one value per sequence, set_sampling) from the Philox streams of `seed`: the same seed gives
        the same ids, with or without the CUDA graph.  generate() sets the step's mode (set_sampling) to what this call asks
        for and leaves it so: a later decode_step() samples after do_sample=True and takes the argmax after do_sample=False.  attention_mask: an HF padding mask of a LEFT-padded batch
        (prefill(); the decode steps skip each sequence's padding); right padding raises ValueError.
        A model with a sliding window W rolls its cache: it holds about max(prompt, W) + 2 max(128, R) positions, and
        before a step that would not fit, the positions that fell out of every window are dropped (KiviCache.shift), so
        the generated length is bounded by the RoPE tables rather than by cache memory.
        num_beams > 1 or num_return_sequences > 1: several sequences per prompt, see _generate_many; the other arguments
        of that mode (length_penalty, early_stopping, return_dict_in_generate) are read there only.
        Logits processing (greedy and sampled decoding, set_processing): repetition_penalty (transformers'
        RepetitionPenaltyLogitsProcessor over the prompt, left padding excluded, and the generated tokens), min_length
        (counted as transformers does, from the padded prompt length) and min_new_tokens (EOS suppressed until then), and
        EOS stopping: with eos_token_id (an int or a list) a row that emits one of them is finished and continues with
        pad_token_id (default: the first EOS id), and decoding stops once every row has finished; the ids are then as long
        as transformers' greedy or sampled generate returns them.  Unlike transformers, the config's EOS is not a default:
        without eos_token_id the output has max_new_tokens new tokens, as it always had.  min_length or min_new_tokens
        without eos_token_id is a ValueError, and beam search with a processor a NotImplementedError (transformers applies
        them to log-probabilities there), both before any work.  Without these arguments the step is the one without
        processing, launch for launch.
        return_dict_in_generate=True returns transformers' GenerateDecoderOnlyOutput(sequences, scores, logits), its
        unrequested fields None.  output_logits=True: a tuple with one fp32 [rows, vocab] tensor per new token, the raw
        logits it was chosen from (the prompt's last position for the first token, then each decode_step's logits).
        output_scores=True (greedy only): the scores the argmax read, i.e. the processed scores with logits processing on
        and the logits without it; unlike transformers, a row that has finished gets the pad-only scores of the processing
        kernel (0 at the pad id, -inf elsewhere) rather than further processed logits.  Both tuples have exactly one entry
        per new token, also when decoding stops at EOS.  They stay on the device: rows * vocab * 4 bytes per new token
        each, as in transformers.  compute_transition_scores() turns them into per-token scores.  output_scores with
        do_sample=True (transformers returns the scores after its warpers, which the sampler never materialises) and either
        output with beam search are NotImplementedError, before any work.
        adapter: a loaded LoRA adapter's name for every prompt, or a list with one name (or None) per prompt; a prompt's
        beams and num_return_sequences copies take its adapter.  None: no adapter on any row."""
        names = self._adapter_names(adapter, input_ids.shape[0])
        if (output_scores or output_logits) and num_beams > 1:
            raise NotImplementedError("output_scores and output_logits in beam search are not supported")
        if output_scores and do_sample:
            raise NotImplementedError("output_scores with do_sample=True is not supported: the sampler never materialises "
                                      "the warped scores transformers returns; use output_logits")
        trace = SimpleNamespace(scores=[] if output_scores else None, logits=[] if output_logits else None)
        proc = _processing_args(input_ids.shape[1], repetition_penalty, min_length, min_new_tokens, eos_token_id,
                                pad_token_id)
        sampling = (temperature, top_k, top_p, seed) if do_sample else None
        if num_beams != 1 or num_return_sequences != 1:
            if num_beams > 1 and proc is not None and (proc["repetition_penalty"] != 1.0 or proc["min_new_tokens"]):
                raise NotImplementedError("repetition_penalty, min_length and min_new_tokens in beam search are not "
                                          "supported: transformers applies them to log-probabilities there")
            return self._generate_many(input_ids, max_new_tokens, use_graph, attention_mask, max_length, sampling,
                                       num_beams, num_return_sequences, length_penalty, early_stopping, eos_token_id,
                                       pad_token_id, return_dict_in_generate, proc, trace, names)
        max_new_tokens = self._generate_setup(input_ids, 1, max_new_tokens, max_length, attention_mask, sampling, proc,
                                              names)
        logits = self.prefill(input_ids, attention_mask)
        tok, scores = self.choose_first(logits, return_scores=True)
        _trace_add(trace, logits, scores)
        seq = torch.cat([input_ids, self._decode(tok.view(-1, 1), max_new_tokens, use_graph, trace)], 1)
        return _generate_output(seq, trace) if return_dict_in_generate else seq

    def _generate_setup(self, input_ids, copies: int, max_new_tokens, max_length, attention_mask, sampling, proc, names):
        """generate()'s set-up for `copies` rows per prompt: the argument checks (ValueError before any work), the cache,
        the RoPE tables, the modes (sampling: set_sampling's arguments, proc: set_processing's; None: off) and the rows'
        adapters (a prompt's copies take its adapter).  Returns max_new_tokens."""
        n, rows = input_ids.shape[1], input_ids.shape[0] * copies
        if sampling is not None:
            sampling_rows(rows, *sampling)
        if proc is not None:
            processing_rows(rows, proc["repetition_penalty"], eos_token_id=proc["eos_token_id"], vocab=self.config.vocab_size)
        if attention_mask is not None:
            kv_start_from_mask(attention_mask)                               # ValueError unless left-padded
        if max_new_tokens is None:
            if max_length is None:
                raise ValueError("generate() needs max_new_tokens or max_length")
            max_new_tokens = max_length - n
        cap = n + max_new_tokens
        if self.sliding_window is not None:
            cap = min(cap, max(n, self.sliding_window) + 2 * max(128, self.config.residual_length))
        if self.cache is None or self.cache.batch != rows or self.cache.max_tokens < cap:
            self.init_cache(rows, cap)
        self._tables(self.cache.device, n + max_new_tokens)                 # positions beyond a rolling cache
        # generate() owns the step's mode; it changes (and the captured step is dropped) only when do_sample does
        if sampling is not None:
            self.set_sampling(*sampling)
        else:
            self.set_sampling(None)
        if proc is not None:
            self.set_processing(**proc)
        else:
            self.set_processing(None)
        if self._lora is not None:
            self.set_adapters(None if names is None else [a for a in names for _ in range(copies)])
        return max_new_tokens

    def _adapter_names(self, adapter, B: int):
        """generate()'s adapter argument as a list of B names (None: no adapter), checked before any work."""
        if adapter is None:
            return None
        names = [adapter] * B if isinstance(adapter, str) else list(adapter)
        if len(names) != B:
            raise ValueError(f"adapter: expected one name or {B} names, got {len(names)}")
        if self._lora is None:
            raise ValueError("adapter: no LoRA adapter is loaded (load_adapter)")
        for a in names:
            self._lora.slot(a)
        return names

    def compute_transition_scores(self, sequences, scores, beam_indices=None, normalize_logits: bool = False):
        """transformers' GenerationMixin.compute_transition_scores for greedy and sampled outputs: the score of each
        generated token, [rows, len(scores)], from generate()'s `scores` (or `logits`) tuple.  normalize_logits=True takes
        the log-softmax of every step's row first (then, with output_logits, these are the tokens' raw log-probabilities).
        On the host's torch, in the tensors' own dtype and device.  beam_indices (beam search) is NotImplementedError."""
        if beam_indices is not None:
            raise NotImplementedError("compute_transition_scores with beam_indices: beam search returns no per-step scores")
        V, steps = self.config.vocab_size, len(scores)
        s = torch.stack(scores).reshape(steps, -1).transpose(0, 1)          # [rows * vocab, steps], transformers' layout
        if normalize_logits:
            s = torch.nn.functional.log_softmax(s.reshape(-1, V, steps), dim=1).reshape(-1, steps)
        rows = torch.arange(s.shape[0] // V, device=sequences.device).view(-1, 1) * V
        return s.gather(0, sequences[:, sequences.shape[-1] - steps:] + rows)

    def _decode(self, tok, max_new_tokens: int, use_graph: bool, trace=None):
        """The new tokens [rows, k] of a greedy or sampled generate(), from the first ones tok [rows, 1]: k = max_new_tokens,
        or, when processing stops rows at EOS, the number of steps until every row had finished.  The finished flags of
        token i are copied to the host asynchronously and read after step i + 1 has been launched, so the device never
        waits for the host; the step launched past the last row's EOS is dropped.  trace (generate's output_scores /
        output_logits lists, already holding the first token's entries): each step's scores and logits are cloned after
        its replay, and dropped with the step that is."""
        out = [tok]
        proc = self._proc
        stops = proc is not None and proc.stops
        if stops:
            flags = [torch.empty(tok.shape[0], dtype=torch.uint8, pin_memory=True) for _ in range(2)]
            events = [torch.cuda.Event(), torch.cuda.Event()]

            def copy_flags(i):
                flags[i & 1].copy_(proc.finished, non_blocking=True)
                events[i & 1].record()
            copy_flags(0)
        for i in range(1, max_new_tokens):
            if self.cache.kv_len + 1 > self.cache.max_tokens:
                self._roll()
            logits = self.decode_step(out[-1], use_graph=use_graph)
            out.append(self.next_tokens.view(-1, 1).clone())
            if trace is not None:
                _trace_add(trace, logits, logits if proc is None else proc.scores, clone=True)
            if stops:
                copy_flags(i)
                events[(i - 1) & 1].synchronize()
                if bool(flags[(i - 1) & 1].all()):
                    out.pop()                                        # every row had finished at token i - 1
                    if trace is not None:
                        _trace_pop(trace)
                    break
        return torch.cat(out, dim=1)

    def _generate_many(self, input_ids, max_new_tokens, use_graph, attention_mask, max_length, sampling, num_beams,
                       num_return_sequences, length_penalty, early_stopping, eos_token_id, pad_token_id,
                       return_dict_in_generate, proc=None, trace=None, names=None):
        """generate() with K = num_beams (beam search, kivi_b200.beam) or K = num_return_sequences (do_sample) sequences per
        prompt, in the cache's rows b * K .. b * K + K - 1.  The prompt pass runs once per prompt and its K / V fill the K
        rows (_prompt_pass(copies=K)).
        Beam search (transformers' _beam_search semantics: length_penalty, early_stopping True / False / "never",
        num_return_sequences <= num_beams, EOS = eos_token_id or config.eos_token_id, finished sequences padded with
        pad_token_id, default the EOS): every step replays the decode-step graph, selects the beams on its logits, reads the
        chosen rows and tokens back in one copy, and replays a second graph that reorders the cache's rows
        (KiviCache._enqueue_reorder: launches_per_reorder launches) and their positions.  Returns [B * n, length] ids, or
        with return_dict_in_generate an object with `sequences` and `sequences_scores`.
        do_sample (sampling: set_sampling's arguments, else None): row b * n + j samples from the Philox key seed + b * n + j
        (set_sampling over the B * n rows), its first token from prompt b's logits, with the logits processing `proc` (generate()'s, set_processing) on every row.
        Returns [B * n, prompt + new] ids, or with return_dict_in_generate generate()'s GenerateDecoderOnlyOutput (`trace`:
        its output_logits, per row).
        Refused before any work: beam sampling (NotImplementedError), num_return_sequences > num_beams and several greedy
        sequences per prompt (ValueError), beams with enable_token_allgather replicas (NotImplementedError)."""
        beams, do_sample = num_beams > 1, sampling is not None
        if num_beams < 1 or num_return_sequences < 1:
            raise ValueError(f"num_beams ({num_beams}) and num_return_sequences ({num_return_sequences}) must be >= 1")
        if beams and do_sample:
            raise NotImplementedError("beam sampling (num_beams > 1 with do_sample=True) is not supported")
        if beams and num_return_sequences > num_beams:
            raise ValueError(f"num_return_sequences ({num_return_sequences}) must not exceed num_beams ({num_beams})")
        if not beams and not do_sample:
            raise ValueError(f"greedy decoding returns one sequence per prompt, num_return_sequences is "
                             f"{num_return_sequences}: use do_sample=True or num_beams >= num_return_sequences")
        if beams and early_stopping not in (True, False, "never"):
            raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
        if beams and (self._exchange is not None or self._dist_tokens is not None):
            raise NotImplementedError("beam search with enable_token_allgather data-parallel replicas is not supported")
        K = num_beams if beams else num_return_sequences
        B, n = input_ids.shape
        rows = B * K
        proc = proc if do_sample else None                  # beam search reads eos_token_id itself
        max_new_tokens = self._generate_setup(input_ids, K, max_new_tokens, max_length, attention_mask, sampling, proc,
                                              names)
        logits = self.lm_head(self._prompt_pass(input_ids, attention_mask, copies=K)[:, -1]).float()    # [B, vocab]
        if do_sample:
            first = logits.repeat_interleave(K, 0)
            tok = self.choose_first(first).view(rows, 1)
            _trace_add(trace, first, first)
            seq = torch.cat([input_ids.repeat_interleave(K, 0), self._decode(tok, max_new_tokens, use_graph, trace)], 1)
            scores = None
        else:
            from .beam import BeamSearch
            if eos_token_id is None:
                eos_token_id = getattr(self.config, "eos_token_id", None)
            search = BeamSearch(input_ids, K, n + max_new_tokens, eos_token_id, pad_token_id, length_penalty,
                                early_stopping, num_return_sequences)
            self.cache.reorder_scratch()
            first = True
            while True:
                beam_idx, tok, done = search.step(logits)
                host = torch.cat([beam_idx, done.view(1).long()]).tolist()   # the one device-to-host read of a step
                if host[-1]:
                    break
                self._ids.copy_(tok.view(rows, 1))
                if not first:        # after the prompt pass the K rows of a prompt hold the same bytes: nothing to copy
                    self._reorder_rows(beam_idx, host[:-1], use_graph)
                first = False
                if self.cache.kv_len + 1 > self.cache.max_tokens:
                    self._roll()
                logits = self.decode_step(use_graph=use_graph)
            seq, scores = search.finalize()
        if not return_dict_in_generate:
            return seq
        from transformers.generation.utils import GenerateBeamDecoderOnlyOutput
        if scores is None:
            return _generate_output(seq, trace)
        return GenerateBeamDecoderOnlyOutput(sequences=seq, sequences_scores=scores)

    def _reorder_rows(self, beam_idx, rows, use_graph: bool = True):
        """Row r of the cache and of the positions becomes a copy of row beam_idx[r] (device [B], any integer dtype; `rows`:
        the same map on the host).  The copy (KiviCache._enqueue_reorder, reading cache.reorder_src) and the position gather
        are captured once in a CUDA graph: the first call runs them eagerly, which also loads the kernels, then captures."""
        c = self.cache
        c.reorder_src.copy_(beam_idx)

        def body():
            c._enqueue_reorder()
            self._pos.copy_(self._pos.index_select(0, c.reorder_src))
        if not use_graph:
            body()
        elif self._reorder_graph is not None and self._reorder_graph[1] == c.ragged:
            self._reorder_graph[0].replay()
        else:
            body()
            from . import _lib
            n0 = _lib.launch_count()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body()
            self.launches_per_reorder = _lib.launch_count() - n0
            self._reorder_graph = (g, c.ragged)
        c._mirror_reorder(rows)


MistralForCausalLM_KIVI = LlamaForCausalLM_KIVI       # models/mistral_kivi.py:921 -- same hook; GQA is handled in-kernel
MistralFlashAttention_KIVI = LlamaFlashAttention_KIVI  # (no repeat_kv_quant copies, models/mistral_kivi.py:58-67)

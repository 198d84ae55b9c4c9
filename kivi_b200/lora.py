"""LoRA adapters beside the base weights: read a local PEFT LoRA directory, check it against the model, and stack every
loaded adapter per layer and per projection group into the layout of kivi_lora_shrink_f16 / kivi_lora_expand_f16
(include/kivi_b200.h).  A batch row names its adapter by slot (LlamaForCausalLM_KIVI.load_adapter / set_adapters); the
decode step applies the rows' deltas with those kernels, the prompt pass and the 9-tuple forward() with torch matmuls per
adapter (LoraState.add).

Supported: LoRA on any of q/k/v/o/gate/up/down_proj (or "all-linear"), layers_to_transform, lora_alpha with or without
use_rslora (scale alpha / r or alpha / sqrt(r)), ranks 1 .. 128.  Refused at load with a ValueError naming the field:
DoRA, rank_pattern, alpha_pattern, bias other than "none", fan_in_fan_out, modules_to_save, embedding / lm_head or regex
targets, and weights whose shapes do not match the model.  A module or layer the adapter does not target gets zeros."""
from __future__ import annotations

import json
import math
import os
import re
from typing import NamedTuple

import torch

MAX_RANK = 128
RANK_ALIGN = 8                      # the kernels' rank granularity: ranks are zero-padded to a multiple of it
LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
# the decode step's four GEMMs and their segments, in the order of the fused weights' columns
GROUPS = {"qkv": ("q_proj", "k_proj", "v_proj"), "o": ("o_proj",), "gu": ("gate_proj", "up_proj"), "down": ("down_proj",)}
MODULE_GROUP = {m: (g, i) for g, ms in GROUPS.items() for i, m in enumerate(ms)}
_KEY = re.compile(r"^base_model\.model\.model\.layers\.(\d+)\.(self_attn|mlp)\.(\w+)\.lora_(A|B)(?:\.[^.]+)?\.weight$")


class LoraConfig(NamedTuple):
    rank: int
    scale: float
    targets: frozenset
    layers: frozenset | None          # layers_to_transform (None: every layer)


def parse_config(cfg: dict) -> LoraConfig:
    """The parts of a PEFT adapter_config.json the kernels honour; ValueError naming the field for anything else."""
    def refuse(field, why):
        raise ValueError(f"LoRA adapter_config.json: {field}: {why}")

    if cfg.get("peft_type", "LORA") != "LORA":
        refuse("peft_type", f"{cfg['peft_type']!r} is not LORA")
    if cfg.get("use_dora"):
        refuse("use_dora", "DoRA is not supported")
    for field in ("rank_pattern", "alpha_pattern"):
        if cfg.get(field):
            refuse(field, "per-module ranks or alphas are not supported")
    if cfg.get("bias", "none") != "none":
        refuse("bias", f"{cfg['bias']!r}: only 'none' is supported")
    if cfg.get("lora_bias"):
        refuse("lora_bias", "a bias on lora_B is not supported")
    if cfg.get("fan_in_fan_out"):
        refuse("fan_in_fan_out", "transposed (Conv1D) weights are not supported")
    if cfg.get("modules_to_save"):
        refuse("modules_to_save", "fully trained modules are not supported")
    r = cfg.get("r", 8)
    if isinstance(r, bool) or not isinstance(r, int) or not 1 <= r <= MAX_RANK:
        refuse("r", f"expected an int in [1, {MAX_RANK}], got {r!r}")
    alpha = cfg.get("lora_alpha", 8)
    if isinstance(alpha, bool) or not isinstance(alpha, (int, float)) or not math.isfinite(alpha):
        refuse("lora_alpha", f"expected a finite number, got {alpha!r}")
    scale = alpha / math.sqrt(r) if cfg.get("use_rslora") else alpha / r
    tm = cfg.get("target_modules")
    if tm == "all-linear":
        targets = frozenset(LINEARS)
    elif isinstance(tm, str) or not isinstance(tm, (list, tuple)) or not tm:
        refuse("target_modules", f"{tm!r}: expected a list of module names or 'all-linear' (regex targets are not "
                                 "supported)")
    else:
        bad = [m for m in tm if m not in LINEARS]
        if bad:
            refuse("target_modules", f"{bad}: only {', '.join(LINEARS)} are supported (no embedding or lm_head)")
        targets = frozenset(tm)
    lt = cfg.get("layers_to_transform")
    if lt is None:
        layers = None
    else:
        lt = [lt] if isinstance(lt, int) else lt
        if not isinstance(lt, (list, tuple)) or any(isinstance(i, bool) or not isinstance(i, int) or i < 0 for i in lt):
            refuse("layers_to_transform", f"expected layer indices, got {cfg['layers_to_transform']!r}")
        layers = frozenset(lt)
    return LoraConfig(r, float(scale), targets, layers)


def module_shapes(config) -> dict:
    """(out, in) of every projection of one layer of `config` (the whole model: tensor parallelism is not supported)."""
    from .llama_kivi import head_dim
    D, hid = head_dim(config), config.hidden_size
    q, kv, inter = config.num_attention_heads * D, config.num_key_value_heads * D, config.intermediate_size
    return {"q_proj": (q, hid), "k_proj": (kv, hid), "v_proj": (kv, hid), "o_proj": (hid, q), "gate_proj": (inter, hid),
            "up_proj": (inter, hid), "down_proj": (hid, inter)}


def read_state(path: str) -> dict:
    """The tensors of adapter_model.safetensors, else adapter_model.bin."""
    st = os.path.join(path, "adapter_model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file
        return load_file(st)
    b = os.path.join(path, "adapter_model.bin")
    if os.path.exists(b):
        return torch.load(b, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"{path}: no adapter_model.safetensors or adapter_model.bin")


class Adapter(NamedTuple):
    rank: int
    scale: float
    weights: dict                    # (layer, module) -> (A [r, in], B [out, r]) on the host


def read_adapter(path: str, config) -> Adapter:
    """A local PEFT LoRA directory checked against the model's `config`: ValueError naming what does not fit."""
    path = str(path)
    if not os.path.isdir(path):
        raise FileNotFoundError(f"{path}: expected a local PEFT adapter directory")
    with open(os.path.join(path, "adapter_config.json")) as f:
        cfg = parse_config(json.load(f))
    shapes, n_layers = module_shapes(config), config.num_hidden_layers
    parts: dict = {}
    for key, t in read_state(path).items():
        m = _KEY.match(key)
        if m is None:
            raise ValueError(f"LoRA weights: {key}: not a lora_A / lora_B weight of a decoder layer's projection "
                             "(embedding, lm_head and DoRA weights are not supported)")
        layer, module, ab = int(m.group(1)), m.group(3), m.group(4)
        if module not in cfg.targets:
            raise ValueError(f"LoRA weights: {key}: {module} is not in target_modules")
        if layer >= n_layers or (cfg.layers is not None and layer not in cfg.layers):
            raise ValueError(f"LoRA weights: {key}: layer {layer} is outside the model's {n_layers} layers or "
                             "layers_to_transform")
        out, n_in = shapes[module]
        want = (cfg.rank, n_in) if ab == "A" else (out, cfg.rank)
        if tuple(t.shape) != want:
            raise ValueError(f"LoRA weights: {key}: shape {tuple(t.shape)} does not match the model's {want}")
        parts.setdefault((layer, module), {})[ab] = t
    weights = {}
    for (layer, module), ab in parts.items():
        if set(ab) != {"A", "B"}:
            raise ValueError(f"LoRA weights: layer {layer} {module} has lora_{''.join(ab)} without its pair")
        weights[(layer, module)] = (ab["A"], ab["B"])
    return Adapter(cfg.rank, cfg.scale, weights)


def padded_rank(ranks) -> int:
    return max(RANK_ALIGN, -(-max(ranks) // RANK_ALIGN) * RANK_ALIGN)


def stack_group(adapters, layer: int, group: str, shapes: dict, R: int, device, dtype=torch.float16):
    """One layer's stacks of one group: A [S, n_seg, R, in] and B [S, out_total, R], adapter s in slot s, ranks below R and
    modules an adapter does not target zero."""
    mods = GROUPS[group]
    n_in = shapes[mods[0]][1]
    outs = [shapes[m][0] for m in mods]
    A = torch.zeros((len(adapters), len(mods), R, n_in), dtype=dtype)
    B = torch.zeros((len(adapters), sum(outs), R), dtype=dtype)
    for s, ad in enumerate(adapters):
        col = 0
        for g, m in enumerate(mods):
            w = ad.weights.get((layer, m))
            if w is not None:
                A[s, g, :ad.rank] = w[0].to(dtype)
                B[s, col:col + outs[g], :ad.rank] = w[1].to(dtype)
            col += outs[g]
    return A.to(device), B.to(device)


def seg_offsets(group: str, shapes: dict):
    offs = [0]
    for m in GROUPS[group]:
        offs.append(offs[-1] + shapes[m][0])
    return offs


class LoraState:
    """Every loaded adapter of a model, stacked: stacks[layer][group] = (A, B), scale fp32 [S], slot of each name."""

    def __init__(self, config, device):
        self.config, self.device = config, device
        self.shapes = module_shapes(config)
        self.names: dict = {}
        self.adapters: list = []
        self.stacks, self.scale, self.rank = None, None, 0
        self.segs = {g: seg_offsets(g, self.shapes) for g in GROUPS}

    def load(self, name: str, adapter: Adapter):
        if name in self.names:
            raise ValueError(f"adapter {name!r} is already loaded")
        self.names[name] = len(self.adapters)
        self.adapters.append(adapter)
        self.rank = padded_rank([a.rank for a in self.adapters])
        self.stacks = [{g: stack_group(self.adapters, i, g, self.shapes, self.rank, self.device) for g in GROUPS}
                       for i in range(self.config.num_hidden_layers)]
        self.scale = torch.tensor([a.scale for a in self.adapters], dtype=torch.float32, device=self.device)

    def slot(self, name) -> int:
        """The slot of adapter `name` (None: -1, no adapter); KeyError for a name that is not loaded."""
        if name is None:
            return -1
        if name not in self.names:
            raise KeyError(f"adapter {name!r} is not loaded (loaded: {sorted(self.names)})")
        return self.names[name]

    def add(self, layer: int, module: str, x, y, rows):
        """y += the LoRA delta of `module` in `layer` for each token, with the adapter slot rows[i] of token i (x [..., in],
        y [..., out] with N tokens, rows int [N] on y's device; a slot < 0 adds nothing).  The tokens are grouped by adapter
        and each group takes two torch matmuls; the intermediate t and the delta are fp32, as in the decode kernels, and y
        is rounded once."""
        group, seg = MODULE_GROUP[module]
        A, B = self.stacks[layer][group]
        lo, hi = self.segs[group][seg], self.segs[group][seg + 1]
        x2, y2 = x.reshape(-1, x.shape[-1]), y.view(-1, y.shape[-1])
        for a in rows.unique().tolist():
            if a < 0:
                continue
            sel = (rows == a).nonzero().squeeze(1)
            t = x2.index_select(0, sel).float() @ A[a, seg].float().t()
            d = (t @ B[a, lo:hi].float().t()) * self.scale[a]
            y2.index_copy_(0, sel, (y2.index_select(0, sel).float() + d).to(y2.dtype))
        return y

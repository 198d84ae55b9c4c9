"""PEFT LoRA adapters written the way peft's save_pretrained writes them (peft itself is not a dependency), and their
float64 merge into a transformers model (tests/test_lora_cpu.py, tests/test_lora_gpu.py)."""
import json

import torch

PREFIX = "base_model.model.model.layers.{}.{}.{}.lora_{}.weight"
BLOCK = {"q_proj": "self_attn", "k_proj": "self_attn", "v_proj": "self_attn", "o_proj": "self_attn",
         "gate_proj": "mlp", "up_proj": "mlp", "down_proj": "mlp"}


def shapes(cfg):
    D = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
    q, kv, hid, inter = cfg.num_attention_heads * D, cfg.num_key_value_heads * D, cfg.hidden_size, cfg.intermediate_size
    return {"q_proj": (q, hid), "k_proj": (kv, hid), "v_proj": (kv, hid), "o_proj": (hid, q), "gate_proj": (inter, hid),
            "up_proj": (inter, hid), "down_proj": (hid, inter)}


def adapter_state(cfg, r, targets, layers=None, seed=0, gain=1.0):
    """Random lora_A [r, in] / lora_B [out, r] fp16 for `targets` in `layers` (None: all), scaled so the delta of a
    projection is about `gain` times as large as a unit-variance input's."""
    g = torch.Generator().manual_seed(seed)
    state = {}
    for i in range(cfg.num_hidden_layers) if layers is None else layers:
        for m in targets:
            out, n_in = shapes(cfg)[m]
            state[PREFIX.format(i, BLOCK[m], m, "A")] = (torch.randn((r, n_in), generator=g) / n_in ** 0.5).half()
            state[PREFIX.format(i, BLOCK[m], m, "B")] = (torch.randn((out, r), generator=g) * gain / r ** 0.5).half()
    return state


def write_adapter(path, state, r, alpha, targets, safetensors=True, **extra):
    """adapter_config.json and adapter_model.safetensors (or .bin) in the directory `path` (pathlib)."""
    path.mkdir(parents=True, exist_ok=True)
    cfg = dict(peft_type="LORA", r=r, lora_alpha=alpha, target_modules=targets, bias="none", use_dora=False,
               use_rslora=False, fan_in_fan_out=False, modules_to_save=None, rank_pattern={}, alpha_pattern={},
               lora_dropout=0.0, task_type="CAUSAL_LM")
    cfg.update(extra)
    (path / "adapter_config.json").write_text(json.dumps(cfg))
    if safetensors:
        from safetensors.torch import save_file
        save_file({k: v.contiguous() for k, v in state.items()}, str(path / "adapter_model.safetensors"))
    else:
        torch.save(state, str(path / "adapter_model.bin"))
    return path


def merge_into(hf_model, state, scale):
    """W += scale * B @ A of every module in `state`, computed in float64 and stored in the model's dtype."""
    with torch.no_grad():
        for key, A in state.items():
            if ".lora_A." not in key:
                continue
            B = state[key.replace(".lora_A.", ".lora_B.")]
            i, block, m = key.split(".")[4], key.split(".")[5], key.split(".")[6]
            lin = getattr(getattr(hf_model.model.layers[int(i)], block), m)
            w = lin.weight.double() + scale * (B.double().to(lin.weight.device) @ A.double().to(lin.weight.device))
            lin.weight.copy_(w.to(lin.weight.dtype))

"""Tensor-parallel placement on the CPU (kivi_b200.tp): the shards of a state dict put back together in rank order are the
full tensors, shapes that do not split are refused, and from_pretrained(tensor_parallel=True) reads exactly its rank's shard
from a safetensors or .bin checkpoint."""
import json
from types import SimpleNamespace

import pytest
import torch

from kivi_b200 import tp
from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config

_CFG = dict(hidden_size=256, intermediate_size=768, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=4,
            vocab_size=320, rope_theta=10000.0, rms_norm_eps=1e-5)


def _state(seed=0):
    torch.manual_seed(seed)
    return {k: v.half() for k, v in LlamaForCausalLM_KIVI(default_config("tiny", **_CFG)).state_dict().items()}


@pytest.mark.parametrize("world", [1, 2, 4])
def test_shards_concatenate_to_the_full_tensors(world):
    cfg = default_config("tiny", **_CFG)
    full = _state()
    shards = [tp.shard_state_dict(full, cfg, r, world) for r in range(world)]
    for k, v in full.items():
        parts = [s[k] for s in shards]
        if k.endswith(("q_proj.weight", "k_proj.weight", "v_proj.weight", "gate_proj.weight", "up_proj.weight")):
            assert torch.equal(torch.cat(parts, 0), v), k
            assert parts[0].shape[0] == v.shape[0] // world
        elif k.endswith(("o_proj.weight", "down_proj.weight")):
            assert torch.equal(torch.cat(parts, 1), v), k
            assert parts[0].shape[1] == v.shape[1] // world
        else:                                                         # embedding, norms, lm_head: replicated
            assert all(torch.equal(p, v) for p in parts), k
    # a KV head and its query group stay together: rank r's q rows are the query heads of its KV heads
    hd = cfg.hidden_size // cfg.num_attention_heads
    q = shards[-1]["model.layers.0.self_attn.q_proj.weight"]
    lo = (world - 1) * cfg.num_attention_heads // world * hd
    assert torch.equal(q, full["model.layers.0.self_attn.q_proj.weight"][lo:lo + q.shape[0]])


@pytest.mark.parametrize("kw,world", [(dict(num_attention_heads=6, num_key_value_heads=6), 4),
                                      (dict(num_key_value_heads=2), 4),
                                      (dict(intermediate_size=770), 4),
                                      (dict(attention_bias=True), 2)])
def test_indivisible_shapes_raise(kw, world):
    cfg = default_config("tiny", **dict(_CFG, **kw))
    with pytest.raises(ValueError):
        tp.shard_state_dict({}, cfg, 0, world)
    with pytest.raises(ValueError):
        tp.check_divisible(cfg, world)


def test_tp_model_is_built_at_local_shapes(monkeypatch):
    import kivi_b200.dist as kdist
    monkeypatch.setattr(kdist, "init", lambda backend=None: (1, 4, 0))
    cfg = default_config("tiny", **_CFG)
    m = LlamaForCausalLM_KIVI(cfg, tensor_parallel=True)
    a, mlp = m.model.layers[0].self_attn, m.model.layers[0].mlp
    assert (m.tp_rank, m.tp_world, a.num_heads, a.num_key_value_heads, a.head_dim) == (1, 4, 2, 1, 32)
    assert a.q_proj.weight.shape == (64, 256) and a.o_proj.weight.shape == (256, 64)
    assert mlp.gate_proj.weight.shape == (192, 256) and mlp.down_proj.weight.shape == (256, 192)
    assert m.lm_head.weight.shape == (320, 256)
    with pytest.raises(NotImplementedError):
        m(torch.zeros((1, 3), dtype=torch.long))
    monkeypatch.setattr(kdist, "init", lambda backend=None: (0, 3, 0))
    with pytest.raises(ValueError):
        LlamaForCausalLM_KIVI(cfg, tensor_parallel=True)


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
def test_from_pretrained_reads_its_shard(tmp_path, monkeypatch, fmt):
    import kivi_b200.dist as kdist
    cfg = default_config("tiny", **_CFG)
    full = _state(1)
    if fmt == "safetensors":
        from safetensors.torch import save_file
        keys = sorted(full)
        save_file({k: full[k].contiguous() for k in keys[: len(keys) // 2]}, str(tmp_path / "model-00001.safetensors"))
        save_file({k: full[k].contiguous() for k in keys[len(keys) // 2:]}, str(tmp_path / "model-00002.safetensors"))
    else:
        torch.save(full, str(tmp_path / "pytorch_model.bin"))
    (tmp_path / "config.json").write_text(json.dumps(_CFG))
    world = 2
    for rank in range(world):
        monkeypatch.setattr(kdist, "init", lambda backend=None, r=rank: (r, world, 0))
        m = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path), tensor_parallel=True)
        assert (m.tp_rank, m.tp_world) == (rank, world)
        got = m.state_dict()
        exp = tp.shard_state_dict(full, SimpleNamespace(**_CFG), rank, world)
        assert set(got) == set(exp)
        for k in exp:
            assert got[k].dtype == torch.float16 and torch.equal(got[k], exp[k]), (rank, k)

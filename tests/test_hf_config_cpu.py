"""Configurations and RoPE tables of LlamaForCausalLM_KIVI against transformers, without a GPU.

* A checkpoint written by transformers' save_pretrained loads into the same model configuration from its config.json
  (config=None) and from the transformers config object carrying the KIVI attributes (the reference's usage).
* The model's fp16 cos / sin tables equal transformers' rotary embedding bit for bit, for the default, linear and llama3
  RoPE types, at positions up to 131071; the transformers 4.x spelling (top-level rope_theta + rope_scaling) gives the
  same tables as the 5.x rope_parameters.
* RoPE types the model does not implement and a head_dim other than hidden / heads = 128 are refused when the model is
  built, not at the first forward.
"""
import json

import pytest
import torch

from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, _rope_tables, rope_settings
from tests._hf import CASES, LLAMA3_SCALING, hf_config, kivi_config, write_checkpoint

SMALL = dict(vocab_size=512, num_hidden_layers=1)          # the configuration is what matters here, not the size
POSITIONS = [0, 1, 8191, 8192, 32767, 131071]


def _fields(cfg):
    names = ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "num_key_value_heads",
             "vocab_size", "rms_norm_eps", "max_position_embeddings", "tie_word_embeddings", "k_bits", "v_bits",
             "group_size", "residual_length")
    return {n: getattr(cfg, n, None) for n in names}, rope_settings(cfg)


@pytest.mark.parametrize("name", list(CASES))
def test_config_json_and_config_object_build_the_same_model(tmp_path, name):
    write_checkpoint(name, tmp_path, **SMALL)
    from_obj = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path), config=kivi_config(name, **SMALL))
    from_json = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))
    obj_fields, obj_rope = _fields(from_obj.config)
    json_fields, json_rope = _fields(from_json.config)
    kb, vb, g, R = CASES[name][2]
    assert (obj_fields["k_bits"], obj_fields["v_bits"], obj_fields["group_size"], obj_fields["residual_length"]) == \
        (kb, vb, g, R)
    json_fields.update(k_bits=kb, v_bits=vb, group_size=g, residual_length=R)     # config.json has no KIVI attributes
    assert obj_fields == json_fields and obj_rope == json_rope
    fields = CASES[name][1]
    assert obj_rope[0] == fields["rope_parameters"]["rope_theta"]
    assert (obj_rope[1] is None) == (fields["rope_parameters"]["rope_type"] == "default")
    sa, sb = from_obj.state_dict(), from_json.state_dict()
    assert set(sa) == set(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    if fields.get("tie_word_embeddings"):
        assert torch.equal(sa["lm_head.weight"], sa["model.embed_tokens.weight"])
    for m in (from_obj, from_json):                      # the tables are built from the config the model was given
        cos, sin = m._tables(torch.device("cpu"))
        exp_cos, exp_sin = _rope_tables(128, cos.shape[0], obj_rope[0], torch.device("cpu"), obj_rope[1])
        assert torch.equal(cos, exp_cos) and torch.equal(sin, exp_sin)


def _hf_tables(rope_parameters):
    """transformers' fp16 cos / sin at POSITIONS, from its own rotary embedding."""
    import transformers
    cfg = transformers.LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=4, num_hidden_layers=1,
                                   intermediate_size=256, vocab_size=64, max_position_embeddings=131072,
                                   rope_parameters=dict(rope_parameters))
    rot = transformers.models.llama.modeling_llama.LlamaRotaryEmbedding(cfg)
    cos, sin = rot(torch.zeros(1, dtype=torch.float16), torch.tensor([POSITIONS]))
    return cfg, cos[0], sin[0]


ROPES = {
    "default 1e4": dict(rope_type="default", rope_theta=1e4),
    "default 5e5": dict(rope_type="default", rope_theta=5e5),
    "linear 4": dict(rope_type="linear", factor=4.0, rope_theta=1e4),
    "llama3": dict(LLAMA3_SCALING, rope_theta=5e5),
    "llama3 orig 4096": dict(LLAMA3_SCALING, original_max_position_embeddings=4096, factor=16.0, rope_theta=5e5),
}


@pytest.mark.parametrize("rope", list(ROPES))
def test_rope_tables_equal_transformers_rotary_embedding(rope):
    cfg, hf_cos, hf_sin = _hf_tables(ROPES[rope])
    model = LlamaForCausalLM_KIVI(kivi_config("llama2", max_position_embeddings=131072, num_hidden_layers=1,
                                              vocab_size=64, rope_parameters=dict(ROPES[rope])))
    cos, sin = model._tables(torch.device("cpu"))
    assert cos.shape == (131072, 128) and cos.dtype == torch.float16
    idx = torch.tensor(POSITIONS)
    assert torch.equal(cos[idx], hf_cos) and torch.equal(sin[idx], hf_sin)
    if rope != "default 1e4":           # the test has teeth: the type's own parameters change the tables
        plain, _ = _rope_tables(128, 131072, 1e4, torch.device("cpu"))
        assert not torch.equal(plain[idx], hf_cos)


@pytest.mark.parametrize("rope", list(ROPES))
@pytest.mark.parametrize("key", ["type", "rope_type"])
def test_transformers_4_spelling_gives_the_same_tables(tmp_path, rope, key):
    """config.json as transformers 4.x wrote it: a top-level rope_theta, and rope_scaling null or a dict naming its type
    under "type" (before 4.43) or "rope_type"."""
    params = dict(ROPES[rope])
    theta, kind = params.pop("rope_theta"), params.pop("rope_type")
    scaling = None if kind == "default" else dict(params, **{key: kind})
    write_checkpoint("llama2", tmp_path, vocab_size=64, num_hidden_layers=1)
    raw = json.loads((tmp_path / "config.json").read_text())
    raw.pop("rope_parameters")
    raw.update(rope_theta=theta, rope_scaling=scaling, max_position_embeddings=131072)
    (tmp_path / "config.json").write_text(json.dumps(raw))
    old = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))
    _, hf_cos, hf_sin = _hf_tables(ROPES[rope])
    cos, sin = old._tables(torch.device("cpu"))
    idx = torch.tensor(POSITIONS)
    assert torch.equal(cos[idx], hf_cos) and torch.equal(sin[idx], hf_sin)
    assert rope_settings(raw) == rope_settings(hf_config("llama2", rope_parameters=dict(ROPES[rope])))


@pytest.mark.parametrize("kind", ["dynamic", "yarn", "longrope", "proportional", "su"])
def test_unsupported_rope_types_are_refused_at_load(tmp_path, kind):
    write_checkpoint("llama2", tmp_path, vocab_size=64, num_hidden_layers=1)
    raw = json.loads((tmp_path / "config.json").read_text())
    raw["rope_parameters"] = dict(rope_type=kind, rope_theta=1e4, factor=2.0)
    (tmp_path / "config.json").write_text(json.dumps(raw))
    with pytest.raises(NotImplementedError, match=kind):
        LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))
    raw.pop("rope_parameters")
    raw.update(rope_theta=1e4, rope_scaling=dict(type=kind, factor=2.0))        # 4.x spelling
    (tmp_path / "config.json").write_text(json.dumps(raw))
    with pytest.raises(NotImplementedError, match=kind):
        LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))
    cfg = kivi_config("llama2", vocab_size=64, num_hidden_layers=1)
    cfg.rope_parameters = dict(rope_type=kind, rope_theta=1e4, factor=2.0)
    with pytest.raises(NotImplementedError, match=kind):
        LlamaForCausalLM_KIVI(cfg)


def test_partial_rotary_factor_is_refused():
    cfg = kivi_config("llama2", vocab_size=64, num_hidden_layers=1)
    cfg.rope_parameters = dict(rope_type="default", rope_theta=1e4, partial_rotary_factor=0.5)
    with pytest.raises(NotImplementedError, match="partial_rotary_factor"):
        LlamaForCausalLM_KIVI(cfg)


@pytest.mark.parametrize("hidden,heads,head_dim", [(512, 4, 64), (512, 4, 256), (256, 4, 64), (1024, 4, 256)])
def test_unsupported_head_dim_is_refused_at_load(tmp_path, hidden, heads, head_dim):
    """An explicit head_dim must equal hidden / heads (the projections assume it) and be 128 (the fused cache's only
    head size)."""
    write_checkpoint("llama2", tmp_path, vocab_size=64, num_hidden_layers=1)
    raw = json.loads((tmp_path / "config.json").read_text())
    raw.update(hidden_size=hidden, num_attention_heads=heads, num_key_value_heads=heads, head_dim=head_dim)
    (tmp_path / "config.json").write_text(json.dumps(raw))
    with pytest.raises(NotImplementedError, match="head_dim"):
        LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))

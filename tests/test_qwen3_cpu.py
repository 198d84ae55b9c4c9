"""Qwen3 without a GPU: hub-style config.json files and transformers' Qwen3Config at the 0.6B and 4B shapes (head_dim 128
with hidden_size != heads x 128), the RoPE tables against transformers' Qwen3 rotary embedding, the tensor-parallel
shards, the refusal of Qwen3-MoE, the wrapper's refusal of a single norm weight, and the attention module's q / k / v
against Qwen3Attention's in float64."""
import json

import pytest
import torch

from kivi_b200 import tp
from kivi_b200.llama_kivi import LlamaFlashAttention_KIVI, LlamaForCausalLM_KIVI, default_config, head_dim, qk_norm

SMALL = dict(vocab_size=512, num_hidden_layers=2)

# The released configs' shapes (config.json of Qwen/Qwen3-0.6B and Qwen/Qwen3-4B), scaled down in layers and vocabulary.
HUB = {
    "0.6b": dict(hidden_size=1024, intermediate_size=3072, num_attention_heads=16, num_key_value_heads=8,
                 tie_word_embeddings=True),
    "4b": dict(hidden_size=2560, intermediate_size=9728, num_attention_heads=32, num_key_value_heads=8,
               tie_word_embeddings=True),
}
POSITIONS = [0, 1, 4095, 4096, 32767, 40959]


def _hub_config(shape):
    """config.json as the hub ships Qwen3 checkpoints: transformers 4.x spelling, an explicit head_dim, a window that is
    switched off."""
    return dict(architectures=["Qwen3ForCausalLM"], model_type="qwen3", attention_bias=False, attention_dropout=0.0,
                head_dim=128, hidden_act="silu", max_position_embeddings=40960, max_window_layers=28,
                rms_norm_eps=1e-6, rope_scaling=None, rope_theta=1000000, sliding_window=None, use_sliding_window=False,
                torch_dtype="bfloat16", **HUB[shape], **SMALL)


def _write(tmp_path, shape, seed=0):
    """A random-init Qwen3ForCausalLM of the shape saved with save_pretrained, its config.json replaced by the hub's."""
    import transformers
    raw = _hub_config(shape)
    cfg = transformers.Qwen3Config(**{k: v for k, v in raw.items() if k not in ("architectures", "torch_dtype")})
    torch.manual_seed(seed)
    model = transformers.Qwen3ForCausalLM(cfg)
    with torch.no_grad():
        for layer in model.model.layers:
            layer.self_attn.q_norm.weight.uniform_(2.0, 6.0)
            layer.self_attn.k_norm.weight.uniform_(2.0, 6.0)
    model.half().save_pretrained(str(tmp_path))
    (tmp_path / "config.json").write_text(json.dumps(raw))
    return model


@pytest.mark.parametrize("shape", list(HUB))
def test_hub_config_json_and_qwen3config_build_the_same_model(tmp_path, shape):
    """config.json (a SimpleNamespace of it) and Qwen3Config.from_pretrained give the same state dict, q_norm / k_norm
    included, head_dim 128 and the same tables."""
    import transformers
    hf = _write(tmp_path, shape)
    from_json = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))
    config = transformers.Qwen3Config.from_pretrained(str(tmp_path))
    config.k_bits, config.v_bits, config.group_size, config.residual_length = 2, 2, 32, 128
    from_obj = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path), config=config)
    hidden, heads = HUB[shape]["hidden_size"], HUB[shape]["num_attention_heads"]
    assert hidden != heads * 128
    for m in (from_json, from_obj):
        assert m.sliding_window is None
        a = m.model.layers[0].self_attn
        assert a.head_dim == 128 and head_dim(m.config) == 128
        assert a.q_proj.weight.shape == (heads * 128, hidden) and a.o_proj.weight.shape == (hidden, heads * 128)
        assert a.q_norm.weight.shape == (128,) and a.k_norm.weight.shape == (128,)
        assert a.q_proj.bias is None and a.o_proj.bias is None
        assert torch.equal(m.lm_head.weight, m.model.embed_tokens.weight)
    sa, sb = from_json.state_dict(), from_obj.state_dict()
    assert set(sa) == set(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    ref = hf.half().state_dict()
    assert torch.equal(sa["model.layers.1.self_attn.k_norm.weight"], ref["model.layers.1.self_attn.k_norm.weight"])
    ca, cb = from_json._tables(torch.device("cpu")), from_obj._tables(torch.device("cpu"))
    assert ca[0].shape == (40960, 128)
    assert all(torch.equal(x, y) for x, y in zip(ca, cb))


@pytest.mark.parametrize("shape", list(HUB))
def test_rope_tables_equal_transformers_qwen3_rotary_embedding(shape):
    """128-wide tables (hidden / heads would give 64 for 0.6B and 80 for 4B) equal to Qwen3RotaryEmbedding's."""
    import transformers
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RotaryEmbedding
    raw = _hub_config(shape)
    cfg = transformers.Qwen3Config(**{k: v for k, v in raw.items() if k not in ("architectures", "torch_dtype")})
    cfg.k_bits, cfg.v_bits, cfg.group_size, cfg.residual_length = 2, 2, 32, 128
    hf_cos, hf_sin = Qwen3RotaryEmbedding(cfg)(torch.zeros(1, dtype=torch.float16), torch.tensor([POSITIONS]))
    cos, sin = LlamaForCausalLM_KIVI(cfg)._tables(torch.device("cpu"))
    assert cos.shape == (40960, 128) and cos.dtype == torch.float16
    idx = torch.tensor(POSITIONS)
    assert torch.equal(cos[idx], hf_cos[0]) and torch.equal(sin[idx], hf_sin[0])


def test_head_dim_and_qk_norm_predicates():
    from types import SimpleNamespace
    assert head_dim(SimpleNamespace(hidden_size=2560, num_attention_heads=32, head_dim=128)) == 128
    assert head_dim(SimpleNamespace(hidden_size=2560, num_attention_heads=32, head_dim=None)) == 80
    assert head_dim(SimpleNamespace(hidden_size=4096, num_attention_heads=32)) == 128
    assert qk_norm(SimpleNamespace(model_type="qwen3"))
    assert not any(qk_norm(SimpleNamespace(model_type=t)) for t in ("llama", "mistral", "qwen2"))
    assert not qk_norm(SimpleNamespace())
    for name, hidden in (("qwen3-8b", 4096), ("qwen3-4b", 2560)):
        cfg = default_config(name)
        assert qk_norm(cfg) and head_dim(cfg) == 128 and cfg.hidden_size == hidden
        assert (cfg.num_attention_heads, cfg.num_key_value_heads) == (32, 8)
    m = LlamaForCausalLM_KIVI(default_config("qwen3-4b", num_hidden_layers=1, vocab_size=64))
    a = m.model.layers[0].self_attn
    assert a.q_proj.weight.shape == (32 * 128, 2560) and a.k_proj.weight.shape == (8 * 128, 2560)
    assert a.q_norm.variance_epsilon == 1e-6
    plain = LlamaForCausalLM_KIVI(default_config("qwen3-4b", model_type="llama", num_hidden_layers=1, vocab_size=64))
    assert plain.model.layers[0].self_attn.q_norm is None
    assert not any("_norm.weight" in k and "self_attn" in k for k in plain.state_dict())


_TP = dict(model_type="qwen3", hidden_size=256, intermediate_size=768, num_hidden_layers=2, num_attention_heads=4,
           num_key_value_heads=2, head_dim=128, vocab_size=320, rope_theta=1e6, rms_norm_eps=1e-6)


@pytest.mark.parametrize("world", [1, 2])
def test_shards_follow_head_dim_and_norms_are_replicated(world):
    """q / k / v rows and o_proj columns are sliced in whole 128-channel heads although hidden / heads = 64; q_norm and
    k_norm are whole on every rank."""
    cfg = default_config("tiny", **_TP)
    torch.manual_seed(0)
    full = {k: v.half() for k, v in LlamaForCausalLM_KIVI(cfg).state_dict().items()}
    shards = [tp.shard_state_dict(full, cfg, r, world) for r in range(world)]
    H, Hkv = 4 // world, 2 // world
    for r, s in enumerate(shards):
        q = s["model.layers.0.self_attn.q_proj.weight"]
        assert q.shape == (H * 128, 256)
        assert torch.equal(q, full["model.layers.0.self_attn.q_proj.weight"][r * H * 128:(r + 1) * H * 128])
        assert s["model.layers.0.self_attn.k_proj.weight"].shape == (Hkv * 128, 256)
        assert s["model.layers.0.self_attn.v_proj.weight"].shape == (Hkv * 128, 256)
        o = s["model.layers.1.self_attn.o_proj.weight"]
        assert o.shape == (256, H * 128)
        assert torch.equal(o, full["model.layers.1.self_attn.o_proj.weight"][:, r * H * 128:(r + 1) * H * 128])
        for k in ("model.layers.0.self_attn.q_norm.weight", "model.layers.1.self_attn.k_norm.weight"):
            assert tp.shard_of(k, cfg, r, world) is None and torch.equal(s[k], full[k])
    # a rank's modules take its shard
    a = LlamaFlashAttention_KIVI(cfg, 0, world)
    assert a.q_proj.weight.shape == (H * 128, 256) and a.q_norm.weight.shape == (128,)


def test_qwen3_moe_is_refused(tmp_path):
    raw = dict(_hub_config("0.6b"), model_type="qwen3_moe", architectures=["Qwen3MoeForCausalLM"], num_experts=8,
               num_experts_per_tok=2, moe_intermediate_size=256)
    with pytest.raises(NotImplementedError, match="qwen3_moe"):
        LlamaForCausalLM_KIVI(default_config("tiny", **{k: v for k, v in raw.items() if k != "architectures"}))
    (tmp_path / "config.json").write_text(json.dumps(raw))
    with pytest.raises(NotImplementedError, match="qwen3_moe"):
        LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))


def test_rope_split_rejects_a_single_norm_weight():
    from kivi_b200 import glue
    B, H, Hkv = 2, 4, 2
    qkv = torch.zeros(B, (H + 2 * Hkv) * 128, dtype=torch.float16)
    cos = sin = torch.zeros(16, 128, dtype=torch.float16)
    pos = torch.zeros(B, dtype=torch.int64)
    q, k, v = (torch.empty(B, n, 128, dtype=torch.float16) for n in (H, Hkv, Hkv))
    w = torch.ones(128, dtype=torch.float16)
    for qn, kn in ((w, None), (None, w)):
        with pytest.raises(ValueError, match="q_norm and k_norm"):
            glue.rope_split(qkv, cos, sin, pos, q, k, v, qn, kn, 1e-6)


@pytest.mark.parametrize("chunked", [False, True])
@pytest.mark.parametrize("shape", list(HUB))
def test_attention_qkv_equals_qwen3_attention(shape, chunked):
    """_qkv (the prompt pass, insert and forward()) and _qkv_rows (the chunked prompt pass) equal Qwen3Attention's q, k
    after q_norm / k_norm and RoPE, and v, in float64 on the CPU, with the weights of one Qwen3Attention."""
    import transformers
    from transformers.models.qwen3 import modeling_qwen3 as mq
    raw = _hub_config(shape)
    cfg = transformers.Qwen3Config(**{k: v for k, v in raw.items() if k not in ("architectures", "torch_dtype")})
    cfg.k_bits, cfg.v_bits, cfg.group_size, cfg.residual_length = 2, 2, 32, 128
    torch.manual_seed(1)
    hf = mq.Qwen3Attention(cfg, layer_idx=0).double().eval()
    with torch.no_grad():
        hf.q_norm.weight.uniform_(-3.0, 3.0)
        hf.k_norm.weight.uniform_(0.2, 6.0)
    ours = LlamaFlashAttention_KIVI(cfg, 0).double().eval()
    ours.load_state_dict(hf.state_dict(), strict=True)
    B, n = 2, 9
    x = torch.randn(B, n, cfg.hidden_size, dtype=torch.float64)
    pos = torch.tensor([[0, 1, 2, 3, 4, 5, 6, 7, 8], [4090, 4091, 4092, 4093, 4094, 4095, 4096, 30000, 40959]])
    cos, sin = mq.Qwen3RotaryEmbedding(cfg)(x, pos)                         # [B, n, 128] float64
    with torch.no_grad():
        shape_ = (B, n, -1, 128)
        eq = hf.q_norm(hf.q_proj(x).view(shape_)).transpose(1, 2)
        ek = hf.k_norm(hf.k_proj(x).view(shape_)).transpose(1, 2)
        ev = hf.v_proj(x).view(shape_).transpose(1, 2)
        eq, ek = mq.apply_rotary_pos_emb(eq, ek, cos, sin)
        if chunked:
            c, s = (t.reshape(B * n, 1, 128) for t in (cos, sin))
            q, k, v = ours._qkv_rows(x.reshape(B * n, -1), c, s)
            q, k, v = (t.view(B, n, -1, 128).transpose(1, 2) for t in (q, k, v))
        else:
            q, k, v = ours._qkv(x, cos[:, None], sin[:, None])
    for name, got, exp in (("q", q, eq), ("k", k, ek), ("v", v, ev)):
        assert got.shape == exp.shape, name
        torch.testing.assert_close(got, exp, rtol=1e-12, atol=1e-12, msg=name)
    with torch.no_grad():                                                   # the test has teeth: without q_norm, q differs
        plain_q = mq.apply_rotary_pos_emb(hf.q_proj(x).view(shape_).transpose(1, 2), ek, cos, sin)[0]
    assert not torch.allclose(q, plain_q)

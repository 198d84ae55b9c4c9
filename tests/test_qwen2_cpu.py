"""Qwen2 / Qwen2.5 without a GPU: configuration (biases, sliding window) from a hub-style config.json and from transformers'
Qwen2Config, the tensor-parallel shards of the q / k / v biases, and the work-unit geometry the decode attention picks for
GQA ratios 1 to 12."""
import ctypes
import json
from types import SimpleNamespace

import pytest
import torch

from kivi_b200 import tp
from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, attention_biases, default_config, sliding_window
from tests._qwen import QWEN_CASES, kivi_config, write_checkpoint

SMALL = dict(vocab_size=512, num_hidden_layers=2)


def _hub_config(fields, **extra):
    """config.json as the hub ships Qwen2.5 checkpoints: transformers 4.x spelling, a window that is switched off, no
    layer_types."""
    cfg = dict(architectures=["Qwen2ForCausalLM"], model_type="qwen2", hidden_act="silu", rms_norm_eps=1e-6,
               rope_theta=fields["rope_parameters"]["rope_theta"], rope_scaling=None, use_sliding_window=False,
               sliding_window=131072, max_window_layers=28, tie_word_embeddings=False, torch_dtype="bfloat16")
    cfg.update({k: v for k, v in fields.items() if k != "rope_parameters"})
    cfg.update(extra)
    return cfg


def test_hub_config_json_and_qwen2config_build_the_same_model(tmp_path):
    """A hand-written hub config.json (use_sliding_window false, sliding_window 131072, no layer_types) next to the weights
    of a Qwen2ForCausalLM checkpoint loads into the model that the Qwen2Config object builds: the same state dict (q / k /
    v biases, no o_proj bias), the same RoPE, no window."""
    name = "qwen-ratio7"
    write_checkpoint(name, tmp_path, **SMALL)
    fields = dict(QWEN_CASES[name][0], **SMALL)
    (tmp_path / "config.json").write_text(json.dumps(_hub_config(fields)))
    from_json = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))
    from_obj = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path), config=kivi_config(name, **SMALL))
    for m in (from_json, from_obj):
        assert m.sliding_window is None
        a = m.model.layers[0].self_attn
        assert a.q_proj.bias is not None and a.k_proj.bias is not None and a.v_proj.bias is not None
        assert a.o_proj.bias is None
    sa, sb = from_json.state_dict(), from_obj.state_dict()
    assert set(sa) == set(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    ca, cb = from_json._tables(torch.device("cpu")), from_obj._tables(torch.device("cpu"))
    assert all(torch.equal(x, y) for x, y in zip(ca, cb))


def test_tied_embeddings_load(tmp_path):
    write_checkpoint("qwen-tied", tmp_path, vocab_size=512, num_hidden_layers=1)
    m = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))
    assert torch.equal(m.lm_head.weight, m.model.embed_tokens.weight)


def test_sliding_window_rules():
    import transformers
    base = dict(num_hidden_layers=4, max_window_layers=28)
    # use_sliding_window false: no window, whatever sliding_window says (raw config.json and Qwen2Config alike)
    assert sliding_window(SimpleNamespace(use_sliding_window=False, sliding_window=131072, **base)) is None
    assert sliding_window(transformers.Qwen2Config(use_sliding_window=False, sliding_window=131072, **base)) is None
    # true with every layer below max_window_layers: transformers windows none of them
    assert sliding_window(SimpleNamespace(use_sliding_window=True, sliding_window=4096, **base)) is None
    assert sliding_window(transformers.Qwen2Config(use_sliding_window=True, sliding_window=4096, **base)) is None
    # true with max_window_layers 0: every layer is windowed, which the cache supports
    assert sliding_window(SimpleNamespace(use_sliding_window=True, sliding_window=4096, num_hidden_layers=4,
                                          max_window_layers=0)) == 4096
    # Llama / Mistral configs have no use_sliding_window: unchanged
    assert sliding_window(SimpleNamespace(sliding_window=4096)) == 4096
    assert sliding_window(SimpleNamespace(sliding_window=None)) is None


@pytest.mark.parametrize("obj", [False, True])
def test_windows_on_some_layers_are_refused(tmp_path, obj):
    """use_sliding_window true with max_window_layers < num_hidden_layers: windows on the upper layers only."""
    import transformers
    kw = dict(use_sliding_window=True, sliding_window=4096, num_hidden_layers=4, max_window_layers=2)
    cfg = transformers.Qwen2Config(**kw) if obj else SimpleNamespace(**kw)
    with pytest.raises(NotImplementedError):
        sliding_window(cfg)
    fields = dict(QWEN_CASES["qwen-ratio5"][0], vocab_size=512, num_hidden_layers=4)
    (tmp_path / "config.json").write_text(json.dumps(_hub_config(fields, use_sliding_window=True, max_window_layers=2)))
    with pytest.raises(NotImplementedError):
        LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))


def test_yarn_is_refused_at_load(tmp_path):
    fields = dict(QWEN_CASES["qwen-ratio7"][0], **SMALL)
    cfg = _hub_config(fields, rope_scaling=dict(type="yarn", factor=4.0, original_max_position_embeddings=32768))
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    with pytest.raises(NotImplementedError, match="yarn"):
        LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path))


def test_attention_biases():
    assert attention_biases(SimpleNamespace(model_type="qwen2")) == (True, False)
    assert attention_biases(SimpleNamespace(model_type="llama", attention_bias=True)) == (True, True)
    assert attention_biases(SimpleNamespace(model_type="llama")) == (False, False)
    assert attention_biases(default_config("qwen2.5-7b")) == (True, False)
    assert attention_biases(default_config("llama-3.2-3b")) == (False, False)


def test_bench_shapes():
    q, l3 = default_config("qwen2.5-7b"), default_config("llama-3.2-3b")
    assert (q.num_attention_heads, q.num_key_value_heads, q.vocab_size, q.rope_theta) == (28, 4, 152064, 1e6)
    assert q.hidden_size // q.num_attention_heads == 128
    assert (l3.num_attention_heads, l3.num_key_value_heads, l3.hidden_size // l3.num_attention_heads) == (24, 8, 128)


_TP = dict(model_type="qwen2", hidden_size=256, intermediate_size=768, num_hidden_layers=2, num_attention_heads=4,
           num_key_value_heads=2, vocab_size=320, rope_theta=1e6, rms_norm_eps=1e-6)


@pytest.mark.parametrize("world", [1, 2])
def test_qkv_biases_shard_with_their_rows(world):
    cfg = default_config("tiny", **_TP)
    torch.manual_seed(0)
    full = {k: v.half() for k, v in LlamaForCausalLM_KIVI(cfg).state_dict().items()}
    assert "model.layers.0.self_attn.q_proj.bias" in full and "model.layers.0.self_attn.o_proj.bias" not in full
    shards = [tp.shard_state_dict(full, cfg, r, world) for r in range(world)]
    for k, v in full.items():
        if k.endswith(("q_proj.bias", "k_proj.bias", "v_proj.bias")):
            parts = [s[k] for s in shards]
            assert torch.equal(torch.cat(parts, 0), v), k
            w = full[k.replace(".bias", ".weight")]
            for r, p in enumerate(parts):                 # the bias rows of the rank's weight rows
                wr = shards[r][k.replace(".bias", ".weight")]
                lo = r * wr.shape[0]
                assert p.shape[0] == wr.shape[0] and torch.equal(p, v[lo:lo + wr.shape[0]]) and wr.shape[1] == w.shape[1]
    tp.check_divisible(cfg, 2)
    with pytest.raises(ValueError):                       # an o_proj bias would be added once per rank
        tp.check_divisible(default_config("tiny", **dict(_TP, model_type="llama", attention_bias=True)), 2)
    with pytest.raises(ValueError):
        tp.check_divisible(default_config("tiny", **dict(_TP, mlp_bias=True)), 2)


def test_gqa_chunk_table():
    """The work unit of the decode attention per GQA ratio: the largest G in {1, 2, 4} dividing the ratio, except that odd
    ratios above 2 take G = 4 (ceil(ratio / 4) units instead of ratio); an explicit KIVI_CACHE_GQA_CHUNK G in {1, 2, 4}
    wins, whether or not it divides the ratio."""
    from kivi_b200 import _lib, build
    build.build()
    fn = _lib.bind("kivi_debug_gqa_chunk", ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int)])
    want = {1: 1, 2: 2, 3: 4, 4: 4, 5: 4, 6: 2, 7: 4, 8: 4, 9: 4, 10: 2, 12: 4}
    hc = ctypes.c_int()
    for ratio, G in want.items():
        assert fn(ratio, 0, ctypes.byref(hc)) == G, ratio
        assert hc.value == -(-ratio // G)
        for forced in (1, 2, 4):
            assert fn(ratio, forced << 4, ctypes.byref(hc)) == forced
            assert hc.value == -(-ratio // forced)
        assert fn(ratio, 1 | (3 << 4), ctypes.byref(hc)) == G      # 3 is not a chunk size: the geometry decides
    # even ratios keep the largest G that divides them
    for ratio in (1, 2, 4, 6, 8, 10, 16):
        old = 4 if ratio % 4 == 0 else 2 if ratio % 2 == 0 else 1
        assert fn(ratio, 0, ctypes.byref(hc)) == old

"""LoRA adapters without a GPU: PEFT config parsing, the scale rules and every refusal, key mapping and the padding of mixed
ranks into a stack, the C entries' argument checks (no launch happens when they fail), serve()'s validation of `adapter`
and the prefix cache's adapter namespaces."""
import math

import pytest
import torch

from tests._lora import adapter_state, write_adapter


def _cfg():
    from kivi_b200.llama_kivi import default_config
    return default_config("tiny", hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                          num_key_value_heads=1, vocab_size=128)


def test_config_scale_rules():
    from kivi_b200.lora import LINEARS, parse_config
    c = parse_config(dict(r=16, lora_alpha=32, target_modules=["q_proj", "v_proj"]))
    assert c.rank == 16 and c.scale == 2.0 and c.targets == {"q_proj", "v_proj"} and c.layers is None
    c = parse_config(dict(r=16, lora_alpha=32, use_rslora=True, target_modules="all-linear", layers_to_transform=[1]))
    assert c.scale == 32 / math.sqrt(16) and c.targets == set(LINEARS) and c.layers == {1}
    assert parse_config(dict(r=1, lora_alpha=1, target_modules=["down_proj"], layers_to_transform=0)).layers == {0}
    assert parse_config(dict(r=128, lora_alpha=16, target_modules=["o_proj"])).rank == 128


@pytest.mark.parametrize("field,value", [
    ("use_dora", True), ("rank_pattern", {"q_proj": 4}), ("alpha_pattern", {"q_proj": 4}), ("bias", "all"),
    ("bias", "lora_only"), ("fan_in_fan_out", True), ("modules_to_save", ["lm_head"]), ("target_modules", ["lm_head"]),
    ("target_modules", ["embed_tokens"]), ("target_modules", ".*q_proj"), ("r", 0), ("r", 129), ("r", 8.0),
    ("lora_alpha", "x"), ("peft_type", "IA3"), ("layers_to_transform", [-1]), ("lora_bias", True)])
def test_config_refusals_name_the_field(field, value):
    from kivi_b200.lora import parse_config
    cfg = dict(r=8, lora_alpha=16, target_modules=["q_proj"])
    cfg[field] = value
    with pytest.raises(ValueError, match=field):
        parse_config(cfg)


def test_read_and_stack_mixed_ranks(tmp_path):
    from kivi_b200 import lora
    cfg = _cfg()
    s1 = adapter_state(cfg, 4, ["q_proj", "v_proj", "down_proj"], layers=[1], seed=1)
    s2 = adapter_state(cfg, 12, list(lora.LINEARS), seed=2)
    a1 = lora.read_adapter(write_adapter(tmp_path / "a1", s1, 4, 8, ["q_proj", "v_proj", "down_proj"],
                                         layers_to_transform=[1]), cfg)
    a2 = lora.read_adapter(write_adapter(tmp_path / "a2", s2, 12, 24, "all-linear", safetensors=False), cfg)
    assert a1.rank == 4 and a1.scale == 2.0 and set(a1.weights) == {(1, "q_proj"), (1, "v_proj"), (1, "down_proj")}
    assert len(a2.weights) == 14
    R = lora.padded_rank([a1.rank, a2.rank])
    assert R == 16
    sh = lora.module_shapes(cfg)
    A, B = lora.stack_group([a1, a2], 1, "qkv", sh, R, "cpu")
    assert A.shape == (2, 3, 16, 256) and B.shape == (2, 256 + 128 + 128, 16)
    key = "base_model.model.model.layers.1.self_attn.{}.lora_{}.weight"
    assert torch.equal(A[0, 0, :4], s1[key.format("q_proj", "A")]) and (A[0, 0, 4:] == 0).all()
    assert (A[0, 1] == 0).all() and (B[0, 256:384] == 0).all()                       # k_proj not targeted: zeros
    assert torch.equal(B[0, 384:, :4], s1[key.format("v_proj", "B")]) and (B[0, :, 4:] == 0).all()
    assert torch.equal(A[1, 2, :12], s2[key.format("v_proj", "A")]) and (A[1, :, 12:] == 0).all()
    A0, B0 = lora.stack_group([a1, a2], 0, "down", sh, R, "cpu")
    assert (A0[0] == 0).all() and (B0[0] == 0).all()                                  # layer 0 not transformed
    assert lora.seg_offsets("gu", sh) == [0, 512, 1024]


def test_read_refuses_mismatches(tmp_path):
    from kivi_b200 import lora
    cfg = _cfg()
    s = adapter_state(cfg, 8, ["q_proj"])
    bad = dict(s)
    k = next(iter(bad))
    bad[k] = bad[k][:, :128].clone()
    with pytest.raises(ValueError, match="does not match"):
        lora.read_adapter(write_adapter(tmp_path / "shape", bad, 8, 16, ["q_proj"]), cfg)
    with pytest.raises(ValueError, match="target_modules"):
        lora.read_adapter(write_adapter(tmp_path / "target", s, 8, 16, ["k_proj"]), cfg)
    with pytest.raises(ValueError, match="layers_to_transform"):
        lora.read_adapter(write_adapter(tmp_path / "layers", s, 8, 16, ["q_proj"], layers_to_transform=[0]), cfg)
    emb = dict(s, **{"base_model.model.model.embed_tokens.lora_embedding_A": torch.zeros(8, 128)})
    with pytest.raises(ValueError, match="embedding"):
        lora.read_adapter(write_adapter(tmp_path / "emb", emb, 8, 16, ["q_proj"]), cfg)
    half = {k: v for k, v in s.items() if ".lora_B." not in k or ".layers.0." not in k}
    with pytest.raises(ValueError, match="without its pair"):
        lora.read_adapter(write_adapter(tmp_path / "pair", half, 8, 16, ["q_proj"]), cfg)
    with pytest.raises(FileNotFoundError):
        lora.read_adapter(tmp_path / "missing", cfg)


def test_entry_points_check_arguments():
    import ctypes
    from kivi_b200 import _lib, build, glue
    build.build()
    glue._bind()
    L = _lib.lib()
    n0 = _lib.launch_count()
    SHAPE, ALIGN, NULL = -2, -5, -6
    p = ctypes.c_void_p(256)                                              # never dereferenced: every call fails its checks
    segs = (ctypes.c_int * 4)(0, 64, 96, 128)
    sh, ex = L.kivi_lora_shrink_f16, L.kivi_lora_expand_f16
    assert sh(None, 4, 256, p, 2, 3, 16, p, p, None) == NULL
    assert sh(p, 4, 256, p, 2, 3, 16, None, p, None) == NULL
    for rows, n_in, S, n_seg, R in ((-1, 256, 2, 3, 16), (1025, 256, 2, 3, 16), (4, 250, 2, 3, 16), (4, 0, 2, 3, 16),
                                    (4, 256, 0, 3, 16), (4, 256, 65536, 3, 16), (4, 256, 2, 4, 16), (4, 256, 2, 0, 16),
                                    (4, 256, 2, 3, 4), (4, 256, 2, 3, 12), (4, 256, 2, 3, 136)):
        assert sh(p, rows, n_in, p, S, n_seg, R, p, p, None) == SHAPE, (rows, n_in, S, n_seg, R)
        assert ex(p, rows, n_in, p, p, S, n_seg, R, segs, p, p, 128, None) == SHAPE
        if S == 2:                                                        # the workspace does not depend on S
            assert L.kivi_lora_workspace_bytes(rows, n_in, n_seg, R) == SHAPE
    assert sh(ctypes.c_void_p(258), 4, 256, p, 2, 3, 16, p, p, None) == ALIGN
    assert ex(p, 4, 256, p, p, 2, 3, 16, None, p, p, 128, None) == NULL
    assert ex(p, 4, 256, p, p, 2, 3, 16, segs, p, p, 129, None) == SHAPE         # seg_off[n_seg] != out_total
    assert ex(p, 4, 256, p, p, 2, 3, 16, (ctypes.c_int * 4)(0, 64, 64, 128), p, p, 128, None) == SHAPE
    assert ex(p, 4, 256, p, p, 2, 3, 16, (ctypes.c_int * 4)(1, 64, 96, 128), p, p, 128, None) == SHAPE
    assert ex(p, 4, 256, ctypes.c_void_p(264), p, 2, 3, 16, segs, p, p, 128, None) == ALIGN
    assert sh(p, 0, 256, p, 2, 3, 16, p, p, None) == 0                    # no rows: nothing to do
    assert ex(p, 0, 256, p, p, 2, 3, 16, segs, p, p, 128, None) == 0
    assert L.kivi_lora_workspace_bytes(32, 4096, 3, 16) == 8 * 32 * 48 * 4
    assert L.kivi_lora_workspace_bytes(5, 600, 1, 8) == 2 * 5 * 8 * 4
    assert _lib.launch_count() == n0


def test_parse_requests_adapter():
    from kivi_b200.serve import parse_requests
    p = torch.arange(1, 5)
    _, params = parse_requests([(p, 3, dict(adapter="a")), (p, 3, dict(adapter="b", temperature=0.5)), (p, 3)],
                               adapters=["a", "b"])
    assert [x.adapter for x in params] == ["a", "b", None]
    assert params[0].sampling is None and params[0].processing is None     # adapter only: greedy
    assert params[1].sampling == dict(temperature=0.5) and params[1].processing is None
    for name in ("c", None, 3):
        with pytest.raises(ValueError, match="adapter"):
            parse_requests([(p, 3), (p, 3, dict(adapter=name))], adapters=["a", "b"])
    with pytest.raises(ValueError, match="adapter"):
        parse_requests([(p, 3, dict(adapter="a"))])                        # nothing loaded


def test_prefix_cache_adapter_namespaces():
    from kivi_b200.prefix import PrefixCache

    class Owner:
        pass
    owner = Owner()
    pc = PrefixCache(1 << 30)
    pc.bind(owner, 2, 1, "cpu")
    toks = list(range(100, 300))
    for adapter, fill in ((None, 1.0), ("a", 2.0), ("b", 3.0)):
        m = pc.match(toks, adapter)
        assert m.length == 0
        st = pc.reserve(m, len(toks))
        st.fill_(fill)
        pc.insert(toks, m, st, adapter)
    for adapter, fill in ((None, 1.0), ("a", 2.0), ("b", 3.0)):
        m = pc.match(toks + [7], adapter)
        assert m.length == len(toks)
        k = torch.empty((1, 200, 128), dtype=torch.float16)
        pc.copy_prefix(m, 200, 0, k, torch.empty_like(k))
        assert (k == fill).all()
    assert pc.match(toks, "c").length == 0 and len(pc) == 3
    m = pc.match(toks[:50] + [1], "a")                                     # a split inside adapter a's tree only
    st = pc.reserve(m, 1)
    pc.insert(toks[:50] + [1], m, st, "a")
    assert len(pc) == 5 and pc.match(toks, None).length == 200 and pc.match(toks, "a").length == 200
    from kivi_b200.prefix import charge
    small = PrefixCache(2 * charge(pc.span_bytes(200)))                   # room for two prompts: LRU over all trees
    small.bind(owner, 2, 1, "cpu")
    for adapter in ("a", "b", "c"):
        m = small.match(toks, adapter)
        small.insert(toks, m, small.reserve(m, len(toks)), adapter)
    assert small.evictions == 1 and small.match(toks, "a").length == 0 and small.match(toks, "c").length == 200

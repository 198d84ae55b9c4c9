"""Qwen3 checkpoints written by transformers' Qwen3ForCausalLM (and one MistralForCausalLM with an explicit head_dim), for
the CPU configuration tests (tests/test_qwen3_cpu.py) and the parity tests (tests/test_qwen3_hf_parity_gpu.py).  The
table mirrors tests/_qwen.py's; the Llama harness (Bar, Decoder, masks) is shared.  head_dim is 128 in every case, and
hidden_size differs from heads x 128 where the case name says "narrow"."""
import pytest
import torch

# name -> (config class name, config fields, KIVI (k_bits, v_bits, group_size, residual_length))
QWEN3_CASES = {
    # Qwen3-0.6B's shape (hidden 1024 < 16 x 128, ratio 2) at a smaller width, with its tied embeddings and vocabulary
    "qwen3-narrow-ratio2": ("Qwen3Config", dict(hidden_size=384, intermediate_size=1024, num_hidden_layers=2,
                                                num_attention_heads=4, num_key_value_heads=2, head_dim=128,
                                                vocab_size=151936, tie_word_embeddings=True,
                                                max_position_embeddings=40960,
                                                rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                            (2, 2, 32, 128)),
    # Qwen3-8B's ratio (32 / 8 heads) with hidden = heads x 128
    "qwen3-ratio4": ("Qwen3Config", dict(hidden_size=1024, intermediate_size=2048, num_hidden_layers=2,
                                         num_attention_heads=8, num_key_value_heads=2, head_dim=128, vocab_size=32000,
                                         max_position_embeddings=40960,
                                         rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                     (4, 4, 64, 64)),
    # Qwen3-32B's ratio (64 / 8 heads) with hidden < heads x 128
    "qwen3-narrow-ratio8": ("Qwen3Config", dict(hidden_size=640, intermediate_size=1536, num_hidden_layers=2,
                                                num_attention_heads=8, num_key_value_heads=1, head_dim=128,
                                                vocab_size=32000, max_position_embeddings=40960,
                                                rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                            (2, 4, 128, 128)),
    # Mistral-NeMo's shape: an explicit head_dim 128 with hidden / heads = 64, and no q / k norms
    "mistral-narrow": ("MistralConfig", dict(hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                                             num_attention_heads=8, num_key_value_heads=2, head_dim=128,
                                             vocab_size=32000, max_position_embeddings=8192, sliding_window=None,
                                             rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                       (2, 2, 32, 128)),
}

# q_norm / k_norm weights: E[w^2] ~ 4.3, so q.k / sqrt(128) has a standard deviation of about 4 -- the peaked attention
# tests/_hf.py's q / k gain gives, for which the bar is set -- and a dropped weight changes the logits' scale about 4-fold.
# U(2, 6) gives about 17, four times more peaked than any checkpoint the bar was set on.
NORM_LO, NORM_HI = 1.0, 3.0


def hf_config(name, **override):
    import transformers
    cls, fields, _ = QWEN3_CASES[name]
    return getattr(transformers, cls)(**dict(fields, rms_norm_eps=1e-6, **override))


def kivi_config(name, **override):
    cfg = hf_config(name, **override)
    cfg.k_bits, cfg.v_bits, cfg.group_size, cfg.residual_length = QWEN3_CASES[name][2]
    return cfg


def _model_class(name):
    import transformers
    return getattr(transformers, QWEN3_CASES[name][0].replace("Config", "ForCausalLM"))


def write_checkpoint(name, path, seed=0, **override):
    """A random-init model of case `name`, fp16, saved with save_pretrained into `path`.  Qwen3: q_norm / k_norm weights
    drawn from U(NORM_LO, NORM_HI), so attention is peaked and a dropped weight shows (scaling q_proj / k_proj, as
    tests/_hf.py does, would vanish in the norm).  Mistral: q_proj and k_proj scaled by 100 / sqrt(hidden) as tests/_hf.py does.  Returns
    the config."""
    cfg = hf_config(name, **override)
    torch.manual_seed(seed)
    model = _model_class(name)(cfg)
    with torch.no_grad():
        for layer in model.model.layers:
            a = layer.self_attn
            if hasattr(a, "q_norm"):
                a.q_norm.weight.uniform_(NORM_LO, NORM_HI)
                a.k_norm.weight.uniform_(NORM_LO, NORM_HI)
            else:
                gain = 100.0 / cfg.hidden_size ** 0.5
                a.q_proj.weight.mul_(gain)
                a.k_proj.weight.mul_(gain)
    model.half().save_pretrained(str(path))
    return cfg


@pytest.fixture(scope="module")
def qwen3_checkpoints(tmp_path_factory):
    made = {}

    def get(name):
        if name not in made:
            path = tmp_path_factory.mktemp(name)
            write_checkpoint(name, path)
            made[name] = path
        return made[name]
    return get


def reference_models(name, path):
    cls = _model_class(name)
    return [cls.from_pretrained(str(path), dtype=dt, attn_implementation="eager").cuda().eval()
            for dt in (torch.float64, torch.float16)]


def load_kivi(name, path, tensor_parallel=False):
    import transformers
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    config = getattr(transformers, QWEN3_CASES[name][0]).from_pretrained(str(path))
    config.k_bits, config.v_bits, config.group_size, config.residual_length = QWEN3_CASES[name][2]
    model = LlamaForCausalLM_KIVI.from_pretrained(str(path), config=config, device_map="cuda",
                                                  tensor_parallel=tensor_parallel)
    assert model.sliding_window is None
    return model

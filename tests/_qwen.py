"""Qwen2 / Qwen2.5 checkpoints written by transformers' Qwen2ForCausalLM, for the CPU configuration tests
(tests/test_qwen2_cpu.py) and the parity tests (tests/test_qwen2_hf_parity_gpu.py).  The table mirrors tests/_hf.py's
CASES and is looked up by the helpers below; the Llama harness (Bar, Decoder, masks) is shared.  head_dim is 128."""
import pytest
import torch

# name -> (config fields, KIVI (k_bits, v_bits, group_size, residual_length))
QWEN_CASES = {
    # Qwen2.5-7B's ratio (28 / 4 heads) at a tenth of its width
    "qwen-ratio7": (dict(hidden_size=896, intermediate_size=1792, num_hidden_layers=2, num_attention_heads=7,
                         num_key_value_heads=1, vocab_size=32000, max_position_embeddings=32768,
                         rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                    (2, 2, 32, 128)),
    # Qwen2.5-14B / 32B's ratio (40 / 8 heads)
    "qwen-ratio5": (dict(hidden_size=1280, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=10,
                         num_key_value_heads=2, vocab_size=32000, max_position_embeddings=32768,
                         rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                    (4, 4, 64, 64)),
    # the small sizes' tied embeddings, the Qwen vocabulary and ratio 3
    "qwen-tied": (dict(hidden_size=768, intermediate_size=1536, num_hidden_layers=2, num_attention_heads=6,
                       num_key_value_heads=2, vocab_size=151936, max_position_embeddings=32768, tie_word_embeddings=True,
                       rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                  (2, 4, 128, 128)),
}

BIAS_GAIN = 1.0                 # biases drawn from U(-1, 1): as large as the projections' outputs, so a dropped one shows


def hf_config(name, **override):
    import transformers
    fields, _ = QWEN_CASES[name]
    return transformers.Qwen2Config(**dict(fields, rms_norm_eps=1e-6, **override))


def kivi_config(name, **override):
    cfg = hf_config(name, **override)
    cfg.k_bits, cfg.v_bits, cfg.group_size, cfg.residual_length = QWEN_CASES[name][1]
    return cfg


def write_checkpoint(name, path, seed=0, **override):
    """A random-init Qwen2ForCausalLM of case `name`, fp16, saved with save_pretrained into `path`.  q_proj and k_proj are
    scaled by 100 / sqrt(hidden) (peaked attention, as tests/_hf.py does) and the q / k / v biases drawn from U(-1, 1).
    Returns the config."""
    import transformers
    cfg = hf_config(name, **override)
    torch.manual_seed(seed)
    model = transformers.Qwen2ForCausalLM(cfg)
    gain = 100.0 / cfg.hidden_size ** 0.5
    with torch.no_grad():
        for layer in model.model.layers:
            a = layer.self_attn
            a.q_proj.weight.mul_(gain)
            a.k_proj.weight.mul_(gain)
            for lin in (a.q_proj, a.k_proj, a.v_proj):
                lin.bias.uniform_(-BIAS_GAIN, BIAS_GAIN)
    model.half().save_pretrained(str(path))
    return cfg


@pytest.fixture(scope="module")
def qwen_checkpoints(tmp_path_factory):
    made = {}

    def get(name):
        if name not in made:
            path = tmp_path_factory.mktemp(name)
            write_checkpoint(name, path)
            made[name] = path
        return made[name]
    return get


def reference_models(path):
    import transformers
    return [transformers.Qwen2ForCausalLM.from_pretrained(str(path), dtype=dt, attn_implementation="eager").cuda().eval()
            for dt in (torch.float64, torch.float16)]


def load_kivi(name, path, tensor_parallel=False):
    import transformers
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    config = transformers.Qwen2Config.from_pretrained(str(path))
    config.k_bits, config.v_bits, config.group_size, config.residual_length = QWEN_CASES[name][1]
    model = LlamaForCausalLM_KIVI.from_pretrained(str(path), config=config, device_map="cuda",
                                                  tensor_parallel=tensor_parallel)
    assert model.sliding_window is None
    return model

"""Checkpoints written by transformers for the parity tests against its LlamaForCausalLM / MistralForCausalLM
(tests/test_hf_config_cpu.py, tests/test_hf_parity_gpu.py).  head_dim is 128 throughout."""
import torch

LLAMA3_SCALING = dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                      original_max_position_embeddings=8192)

# name -> (config class name, config fields, KIVI (k_bits, v_bits, group_size, residual_length), safetensors)
CASES = {
    "llama2": ("LlamaConfig", dict(hidden_size=512, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=4,
                                   num_key_value_heads=4, vocab_size=32000, max_position_embeddings=4096,
                                   rope_parameters=dict(rope_type="default", rope_theta=1e4)),
               (2, 2, 32, 32), False),
    "llama3": ("LlamaConfig", dict(hidden_size=1024, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=8,
                                   num_key_value_heads=2, vocab_size=128256, max_position_embeddings=8192,
                                   rope_parameters=dict(rope_type="default", rope_theta=5e5)),
               (2, 2, 32, 128), True),
    "llama3.1": ("LlamaConfig", dict(hidden_size=1024, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=8,
                                     num_key_value_heads=2, vocab_size=128256, max_position_embeddings=131072,
                                     rope_parameters=dict(LLAMA3_SCALING, rope_theta=5e5)),
                 (4, 2, 64, 64), True),
    "mistral": ("MistralConfig", dict(hidden_size=1024, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=8,
                                      num_key_value_heads=2, vocab_size=32000, max_position_embeddings=8192,
                                      sliding_window=None, rope_parameters=dict(rope_type="default", rope_theta=1e6)),
                (4, 4, 64, 64), True),
    "tied": ("LlamaConfig", dict(hidden_size=1024, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=8,
                                 num_key_value_heads=2, vocab_size=128256, max_position_embeddings=8192,
                                 tie_word_embeddings=True, rope_parameters=dict(rope_type="default", rope_theta=5e5)),
             (2, 4, 128, 128), True),
}


def hf_config(name, **override):
    """The case's transformers config (RMSNorm eps 1e-5, as the Llama checkpoints have), fields overridden by `override`."""
    import transformers
    cls, fields, _, _ = CASES[name]
    return getattr(transformers, cls)(**dict(fields, rms_norm_eps=1e-5, **override))


def kivi_config(name, **override):
    """hf_config with the case's KIVI attributes set on it: the reference's documented usage
    (config = LlamaConfig.from_pretrained(path); config.k_bits = ...; LlamaForCausalLM_KIVI.from_pretrained(path, config=config))."""
    cfg = hf_config(name, **override)
    cfg.k_bits, cfg.v_bits, cfg.group_size, cfg.residual_length = CASES[name][2]
    return cfg


def write_checkpoint(name, path, seed=0, qk_gain=None, head_gain=1.0, **override):
    """A random-init transformers model of case `name`, fp16, saved with save_pretrained into the pathlib directory `path`
    (a pytorch_model.bin where the case says so).  q_proj and k_proj are scaled by qk_gain (default 100 / sqrt(hidden): q.k / sqrt(128) then has a
    standard deviation of about 4 and attention is peaked, where transformers' std-0.02 init gives near-uniform
    attention); lm_head by head_gain.  Returns the config."""
    import transformers
    cfg = hf_config(name, **override)
    torch.manual_seed(seed)
    model = getattr(transformers, CASES[name][0].replace("Config", "ForCausalLM"))(cfg)
    gain = 100.0 / cfg.hidden_size ** 0.5 if qk_gain is None else qk_gain
    with torch.no_grad():
        for layer in model.model.layers:
            layer.self_attn.q_proj.weight.mul_(gain)
            layer.self_attn.k_proj.weight.mul_(gain)
        if not cfg.tie_word_embeddings:
            model.lm_head.weight.mul_(head_gain)
    model.half().save_pretrained(str(path))
    if not CASES[name][3]:          # transformers 5 writes safetensors only; 4.x wrote this with safe_serialization=False
        from safetensors.torch import load_file
        st = path / "model.safetensors"
        torch.save(load_file(str(st)), str(path / "pytorch_model.bin"))
        st.unlink()
    return cfg

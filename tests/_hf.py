"""Checkpoints written by transformers, and the harness that holds the model to its LlamaForCausalLM / MistralForCausalLM
(tests/test_hf_config_cpu.py; tests/test_hf_parity_gpu.py, whose docstring states the method and the bar;
tests/test_window_hf_parity_gpu.py).  The harness itself is tested without a GPU in tests/test_hf_harness_cpu.py.
head_dim is 128 throughout."""
import pytest
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

ALPHA, BETA = 4.0, 1e-3         # the bar (tests/test_hf_parity_gpu.py)


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


@pytest.fixture(scope="module")
def checkpoints(tmp_path_factory):
    """checkpoints(name, **override): the directory of write_checkpoint(name, path, **override), written once per module."""
    made = {}

    def get(name, **override):
        key = (name, tuple(sorted(override.items())))
        if key not in made:
            path = tmp_path_factory.mktemp(name.replace(".", "_"))
            write_checkpoint(name, path, **override)
            made[key] = path
        return made[key]
    return get


def reference_models(name, path):
    """ref64 and hf16: transformers' model of the checkpoint with eager attention, in float64 and in float16."""
    import transformers
    cls = getattr(transformers, CASES[name][0].replace("Config", "ForCausalLM"))
    return [cls.from_pretrained(str(path), dtype=dt, attn_implementation="eager").cuda().eval()
            for dt in (torch.float64, torch.float16)]


def load_kivi(name, path, tensor_parallel=False, **kivi):
    """The reference's documented usage: the transformers config of the checkpoint, the case's KIVI attributes set on it
    and overridden by `kivi` (e.g. residual_length=R)."""
    import transformers
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    config = getattr(transformers, CASES[name][0]).from_pretrained(str(path))
    config.k_bits, config.v_bits, config.group_size, config.residual_length = CASES[name][2]
    for attr, value in kivi.items():
        setattr(config, attr, value)
    model = LlamaForCausalLM_KIVI.from_pretrained(str(path), config=config, device_map="cuda",
                                                  tensor_parallel=tensor_parallel)
    assert model.sliding_window == getattr(config, "sliding_window", None)
    return model


class Bar:
    """The bar on logits tensors, and what it has seen: per check (its label up to " step"), the worst
    err / max|hf16 - ref64| and err / max|ref64|; the rows where the argmax check applied.  A test module holds one and
    prints its report at the end."""

    def __init__(self):
        self.worst = {}
        self.decided = [0, 0]       # rows where the argmax check applied, rows compared

    def check(self, what, ours, ref, hf):
        """ours, ref (ref64), hf (hf16): logits [..., vocab]."""
        ours, ref, hf = (t.reshape(-1, t.shape[-1]).double() for t in (ours, ref, hf))
        assert torch.isfinite(ours).all(), what
        err = (ours - ref).abs().max().item()
        hf_err = (hf - ref).abs().max().item()
        scale = ref.abs().max().item()
        bar = ALPHA * hf_err + BETA * scale
        w = self.worst.setdefault(what.split(" step")[0], [0.0, 0.0])
        w[0], w[1] = max(w[0], err / hf_err), max(w[1], err / scale)
        assert err <= bar, f"{what}: max|ours - ref64| = {err:.4g} > {bar:.4g} (hf16 {hf_err:.4g}, max|ref64| {scale:.4g})"
        self._argmax(what, ours.argmax(-1), ref, bar)

    def argmax_agrees(self, what, ids, ref, hf):
        """Token ids [...] that stand for logits, e.g. the first token serve() took: argmax(ref64) on every row whose ref64
        top-2 margin exceeds twice the bar of ref (ref64) and hf (hf16), logits [..., vocab]."""
        ref, hf = (t.reshape(-1, t.shape[-1]).double() for t in (ref, hf))
        self._argmax(what, ids.reshape(-1), ref, ALPHA * (hf - ref).abs().max().item() + BETA * ref.abs().max().item())

    def _argmax(self, what, ids, ref, bar):
        top2 = ref.topk(2, dim=-1).values
        decided = (top2[:, 0] - top2[:, 1]) > 2 * bar
        self.decided[0] += int(decided.sum())
        self.decided[1] += decided.numel()
        same = ids.to(ref.device) == ref.argmax(-1)
        assert same[decided].all(), f"{what}: argmax differs on rows {torch.nonzero(decided & ~same).flatten().tolist()}"

    def assert_decided(self, since, share=0.05):
        """The precondition of the argmax check: since `since` (a copy of self.decided) the logits spread enough that it
        applied to a fair share of the rows."""
        decided, rows = self.decided[0] - since[0], self.decided[1] - since[1]
        assert decided >= share * rows, f"the argmax check applied to only {decided} of {rows} rows"

    def report(self, title):
        print(f"\n[{title}] worst max|ours - ref64| / max|hf16 - ref64| per check:")
        for k, v in sorted(self.worst.items()):
            print(f"  {k:28s} {v[0]:.3f}   (err / max|ref64| {v[1]:.2e})")
        print(f"  argmax checked on {self.decided[0]} of {self.decided[1]} rows")


def pad_mask(pads, n, device="cuda"):
    """The 0 / 1 mask [B, n] of a left-padded prompt: pads[b] pad tokens in front of row b."""
    return (torch.arange(n, device=device)[None, :] >= torch.tensor(pads, device=device)[:, None]).long()


def hf_positions(mask):
    """What transformers' generate passes with a left-padded batch: cumsum - 1, pad positions 1."""
    pos = mask.long().cumsum(-1) - 1
    return pos.masked_fill(mask == 0, 1)


def hf_prompt_mask(mask, dtype, window=None):
    """The left-padding mask [B, n] as transformers' eager attention must be given it: 4-D additive, causal (and inside
    the sliding window: key j > query i - window), pad keys hidden, and each pad query seeing itself.  With the 2-D mask a
    pad query row is fully masked, transformers' eager softmax makes it NaN, and the NaN reaches the real rows of the next
    layer through 0 * NaN.  Real rows see exactly what the 2-D mask gives them."""
    n = mask.shape[1]
    i = torch.arange(n, device=mask.device)
    band = i[None, :] <= i[:, None]
    if window is not None:
        band &= i[None, :] > i[:, None] - window
    keep = (mask.bool()[:, None, None, :] & band) | torch.eye(n, dtype=torch.bool, device=mask.device)
    return torch.zeros(keep.shape, dtype=dtype, device=mask.device).masked_fill(~keep, torch.finfo(dtype).min)


def hf_kw(kw, dtype, window=None):
    """What transformers is given for a prompt for which the model is given `kw`: kw itself when it holds no mask (an
    unpadded prompt: transformers applies its own causal mask and window), else kw with hf_prompt_mask in place of the
    2-D mask."""
    if "attention_mask" not in kw:
        return kw
    return dict(kw, attention_mask=hf_prompt_mask(kw["attention_mask"], dtype, window))


def kv_fp64(tup, cfg):
    """Post-RoPE K, V [B, Hkv, T, 128] in fp64 from a 9-tuple: the codes dequantised exactly (c * s + z with
    cfg.k_bits / v_bits / group_size), then the fp16 windows."""
    from oracle import ref
    kc, kfull, ks, km, vc, vfull, vs, vm, _ = tup

    def dequant(code, s, z, bits):
        g = cfg.group_size
        c = torch.from_numpy(ref.unpack_codes_lastdim(code.cpu().numpy(), bits)).to(code.device).double()
        return c * s.double().repeat_interleave(g, -1) + z.double().repeat_interleave(g, -1)
    k = [dequant(kc, ks, km, cfg.k_bits).transpose(2, 3)] if kc is not None else []
    v = [dequant(vc, vs, vm, cfg.v_bits)] if vc is not None else []
    return torch.cat(k + ([kfull.double()] if kfull is not None else []), 2), torch.cat(v + [vfull.double()], 2)


def exports(model):
    """The 9-tuple of every layer of the model's cache.  A tensor-parallel model at world 1 holds every head on its one
    rank, so its cache exports like a whole model's."""
    cache = model.cache
    sharded = cache.tensor_parallel
    cache.tensor_parallel = sharded and model.tp_world > 1
    try:
        return [cache.export(layer) for layer in range(len(model.model.layers))]
    finally:
        cache.tensor_parallel = sharded


def reference_step(ref64, hf16, tuples, cfg, tok, pos, start):
    """ref64 / hf16 logits [B, vocab] of one decode step seeded with the K / V of `tuples` (one 9-tuple per layer, T
    positions, quantised as cfg says): token tok[b] at RoPE position pos[b] sees the timeline positions start[b] .. T - 1
    and itself; start[b] = None is a released slot, which sees its own token only."""
    from transformers import DynamicCache
    kv = [kv_fp64(t, cfg) for t in tuples]
    B, T = tok.shape[0], kv[0][0].shape[2]
    mask = torch.zeros(B, T + 1, dtype=torch.long, device=tok.device)
    for b, s in enumerate(start):
        mask[b, T if s is None else s:] = 1
    out = []
    for m in (ref64, hf16):
        cache = DynamicCache()
        for layer, (k, v) in enumerate(kv):
            cache.update(k.to(m.dtype), v.to(m.dtype), layer)
        out.append(m(input_ids=tok.view(B, 1), past_key_values=cache, attention_mask=mask,
                     position_ids=torch.tensor(pos, device=tok.device).view(B, 1)).logits[:, -1])
    return out


class Decoder:
    """Teacher-forced decode steps on the model, tokens drawn from `gen`, each checked step held to `bar` against
    reference_step on the model's cache.  The test keeps its own books: T (the shared length), pos[b] (row b's next
    position) and start[b] (row b's first visible timeline position; None = a released slot)."""

    def __init__(self, bar, model, ref64, hf16, T, pos, start, gen):
        self.bar, self.model, self.ref64, self.hf16, self.gen = bar, model, ref64, hf16, gen
        self.T, self.pos, self.start = T, list(pos), list(start)
        self.step_no, self.flushes, self.vpacks, self.flushed = 0, 0, 0, False

    def run(self, steps, label, every=7):
        """Checked: the first and last three steps, every `every`-th step of the decoder and each step after a K flush."""
        model, cache = self.model, self.model.cache
        B = len(self.pos)
        for s in range(steps):
            checked = s < 3 or s >= steps - 3 or self.step_no % every == 0 or self.flushed
            tok = torch.randint(0, model.config.vocab_size, (B,), device=self.gen.device, generator=self.gen)
            if checked:
                assert cache.kv_len == self.T
                ref, hf = reference_step(self.ref64, self.hf16, exports(model), model.config, tok, self.pos, self.start)
            tk, tv = cache.tk, cache.tv
            ours = model.decode_step(tok.view(B, 1), use_graph=self.step_no >= 2).clone()
            if checked:
                self.bar.check(f"{label} step {self.step_no}", ours, ref, hf)
            self.flushed = cache.tk > tk
            self.flushes += int(self.flushed)
            self.vpacks += cache.tv - tv
            self.T += 1
            self.pos = [p + 1 for p in self.pos]
            self.step_no += 1
        assert cache.kv_len == self.T

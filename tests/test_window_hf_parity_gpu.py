"""A windowed LlamaForCausalLM_KIVI (MistralForCausalLM_KIVI) against transformers' MistralForCausalLM with a small
config.sliding_window: prompt passes longer than the window, decode for several windows, forward() on the fused and the
9-tuple paths, serve() with shifts, and a rolling generate() several times longer than its cache.

The bar and method are those of tests/test_hf_parity_gpu.py: transformers' eager model in float64 (`ref64`) is the truth,
the same checkpoint in float16 (`hf16`) the yardstick, and every compared logits tensor must meet

    max|ours - ref64| <= ALPHA * max|hf16 - ref64| + BETA * max|ref64|

with argmax(ours) == argmax(ref64) on every row whose ref64 top-2 margin exceeds twice that bar.  Decode steps are checked
against transformers seeded with the model's own cache at that step (export(), codes dequantised exactly in fp64, then
the fp16 windows), so the window is applied by transformers' own mask (kv_idx > q_idx - sliding_window) to the positions
the cache holds; after a shift those are the last T positions, the RoPE positions stay absolute.
"""
import pytest
import torch

from tests._hf import CASES, write_checkpoint

pytestmark = pytest.mark.gpu

ALPHA, BETA = 4.0, 1e-3
NAME = "mistral"
WINDOWS = [(160, 64), (320, 128)]          # (sliding_window, residual_length R); K4V4 g64
DECIDED = [0, 0]


@pytest.fixture(scope="module")
def checkpoints(tmp_path_factory):
    made = {}

    def get(window):
        if window not in made:
            path = tmp_path_factory.mktemp(f"mistral_w{window}")
            write_checkpoint(NAME, path, sliding_window=window)
            made[window] = path
        return made[window]
    return get


def _models(path, R):
    import transformers
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    ref64 = transformers.MistralForCausalLM.from_pretrained(str(path), dtype=torch.float64,
                                                            attn_implementation="eager").cuda().eval()
    hf16 = transformers.MistralForCausalLM.from_pretrained(str(path), dtype=torch.float16,
                                                           attn_implementation="eager").cuda().eval()
    config = transformers.MistralConfig.from_pretrained(str(path))
    config.k_bits, config.v_bits, config.group_size, _ = CASES[NAME][2]
    config.residual_length = R
    model = LlamaForCausalLM_KIVI.from_pretrained(str(path), config=config, device_map="cuda")
    assert model.sliding_window == config.sliding_window
    return ref64, hf16, model


def check(what, ours, ref, hf):
    ours, ref, hf = (t.reshape(-1, t.shape[-1]).double() for t in (ours, ref, hf))
    assert torch.isfinite(ours).all(), what
    err = (ours - ref).abs().max().item()
    hf_err = (hf - ref).abs().max().item()
    scale = ref.abs().max().item()
    bar = ALPHA * hf_err + BETA * scale
    assert err <= bar, f"{what}: max|ours - ref64| = {err:.4g} > {bar:.4g} (hf16 {hf_err:.4g}, max|ref64| {scale:.4g})"
    top2 = ref.topk(2, dim=-1).values
    decided = (top2[:, 0] - top2[:, 1]) > 2 * bar
    DECIDED[0] += int(decided.sum())
    DECIDED[1] += decided.numel()
    same = ours.argmax(-1) == ref.argmax(-1)
    assert same[decided].all(), f"{what}: argmax differs on rows {torch.nonzero(decided & ~same).flatten().tolist()}"
    return decided


def _pad_mask(pads, n):
    return (torch.arange(n, device="cuda")[None, :] >= torch.tensor(pads, device="cuda")[:, None]).long()


def _hf_prompt_mask(mask, window, dtype):
    """The 4-D additive mask of a left-padded windowed prompt for transformers' eager attention: causal, inside the window,
    pad keys hidden, each pad query seeing itself (a fully masked row would turn into NaN there)."""
    n = mask.shape[1]
    i = torch.arange(n, device=mask.device)
    band = (i[None, :] <= i[:, None]) & (i[None, :] > i[:, None] - window)
    keep = (mask.bool()[:, None, None, :] & band) | torch.eye(n, dtype=torch.bool, device=mask.device)
    return torch.zeros(keep.shape, dtype=dtype, device=mask.device).masked_fill(~keep, torch.finfo(dtype).min)


def _kv_of(tup, cfg):
    """Post-RoPE K, V [B, Hkv, T, 128] in fp64 from a 9-tuple: codes dequantised exactly, then the windows."""
    from oracle import ref
    kc, kfull, ks, km, vc, vfull, vs, vm, _ = tup
    g = cfg.group_size
    ks_, vs_ = [], []
    if kc is not None:
        codes = torch.from_numpy(ref.unpack_codes_lastdim(kc.cpu().numpy(), cfg.k_bits)).cuda().double()
        ks_.append((codes * ks.double().repeat_interleave(g, -1) + km.double().repeat_interleave(g, -1)).transpose(2, 3))
    if kfull is not None:
        ks_.append(kfull.double())
    if vc is not None:
        codes = torch.from_numpy(ref.unpack_codes_lastdim(vc.cpu().numpy(), cfg.v_bits)).cuda().double()
        vs_.append(codes * vs.double().repeat_interleave(g, -1) + vm.double().repeat_interleave(g, -1))
    vs_.append(vfull.double())
    return torch.cat(ks_, 2), torch.cat(vs_, 2)


def _reference_step(ref64, hf16, tuples, cfg, tok, pos, start):
    """ref64 / hf16 logits of one decode step seeded with the K / V of `tuples` (one 9-tuple per layer).  start[b]: row b's
    first timeline position (padding); pos[b]: its RoPE position."""
    from transformers import DynamicCache
    kv = [_kv_of(t, cfg) for t in tuples]
    B, T = tok.shape[0], kv[0][0].shape[2]
    mask = torch.zeros(B, T + 1, dtype=torch.long, device="cuda")
    for b, s in enumerate(start):
        mask[b, s:] = 1
    out = []
    for m, dt in ((ref64, torch.float64), (hf16, torch.float16)):
        cache = DynamicCache()
        for layer, (k, v) in enumerate(kv):
            cache.update(k.to(dt), v.to(dt), layer)
        out.append(m(input_ids=tok.view(B, 1), past_key_values=cache, attention_mask=mask,
                     position_ids=torch.tensor(pos, device="cuda").view(B, 1)).logits[:, -1])
    return out


def _exports(model):
    return [model.cache.export(i) for i in range(len(model.model.layers))]


@pytest.mark.parametrize("window,R", WINDOWS)
def test_prompt_and_decode_match_transformers(checkpoints, window, R):
    """Prompts longer than the window, unpadded and left-padded: forward() on the 9-tuple path and prefill() against
    transformers; then 3W + 3 decode steps after the unpadded prefill and W after the padded one, across K flushes, V-ring
    wraps and a window start that moves through many packed blocks."""
    d0 = list(DECIDED)
    ref64, hf16, model = _models(checkpoints(window), R)
    cfg = model.config
    B, n = 3, window + 150
    gen = torch.Generator(device="cuda").manual_seed(window)
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda", generator=gen)
    for pads, steps in (([0] * B, 3 * window + 3), ([0, 17, n - 5], window)):
        padded = any(pads)
        mask = _pad_mask(pads, n)
        pos = mask.long().cumsum(-1) - 1
        pos.masked_fill_(mask == 0, 1)
        if padded:
            kw = dict(attention_mask=mask, position_ids=pos)
            ref = ref64(input_ids=ids, attention_mask=_hf_prompt_mask(mask, window, torch.float64), position_ids=pos).logits
            hf = hf16(input_ids=ids, attention_mask=_hf_prompt_mask(mask, window, torch.float16), position_ids=pos).logits
        else:
            kw = {}
            ref, hf = ref64(input_ids=ids).logits, hf16(input_ids=ids).logits
        real = mask.bool()
        model.fused_forward = False
        check(f"w{window} forward padded={padded}", model(input_ids=ids, **kw).logits[real], ref[real], hf[real])
        model.fused_forward = True
        model.init_cache(B, n + steps + 8)
        last = model.prefill(ids, attention_mask=mask if padded else None)
        check(f"w{window} prefill padded={padded}", last, ref[:, -1], hf[:, -1])
        nxt = [n - p for p in pads]
        tk0 = model.cache.tk
        for s in range(steps):
            tok = torch.randint(0, cfg.vocab_size, (B,), device="cuda", generator=gen)
            checked = s < 3 or s >= steps - 3 or s % 11 == 0
            if checked:
                r, h = _reference_step(ref64, hf16, _exports(model), cfg, tok, nxt, pads)
            ours = model.decode_step(tok.view(B, 1), use_graph=s >= 2).clone()
            if checked:
                check(f"w{window} decode padded={padded} step {s}", ours, r, h)
            nxt = [p + 1 for p in nxt]
        assert model.cache.tk > tk0 and model.cache.vhead != 0
    assert DECIDED[0] - d0[0] >= 0.05 * (DECIDED[1] - d0[1])


def test_forward_fused_and_tuple_paths_agree_with_transformers(checkpoints):
    """forward() decode steps past the window on the fused cache (KiviPast) and on the reference's 9-tuples (the window
    as an additive mask), each against transformers seeded with that path's own cache."""
    window, R = WINDOWS[0]
    ref64, hf16, model = _models(checkpoints(window), R)
    cfg = model.config
    B, n, steps = 2, window + 40, 2 * window
    gen = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda", generator=gen)
    model.fused_forward = True
    _, fused = model(input_ids=ids, return_dict=False)
    model.fused_forward = False
    _, tuples = model(input_ids=ids, return_dict=False)
    for s in range(steps):
        tok = torch.randint(0, cfg.vocab_size, (B, 1), device="cuda", generator=gen)
        checked = s < 2 or s >= steps - 2 or s % 13 == 0
        pos = [n + s] * B
        if checked:
            r_f, h_f = _reference_step(ref64, hf16, [tuple(p) for p in fused], cfg, tok, pos, [0] * B)
            r_t, h_t = _reference_step(ref64, hf16, tuples, cfg, tok, pos, [0] * B)
        model.fused_forward = True
        lf, fused = model(input_ids=tok, past_key_values=fused, return_dict=False)
        model.fused_forward = False
        lt, tuples = model(input_ids=tok, past_key_values=tuples, return_dict=False)
        if checked:
            check(f"fused forward step {s}", lf[:, -1], r_f, h_f)
            check(f"tuple forward step {s}", lt[:, -1], r_t, h_t)


def test_rolling_generate_matches_transformers_and_full_cache(checkpoints):
    """generate() of a windowed model holds about max(prompt, W) + 2 max(128, R) positions and runs for more than four
    times that.  The same steps driven by hand (prefill, decode_step, a shift whenever the cache is full) take generate()'s
    ids, and a twin model on a full-capacity cache (never shifted) is fed the same tokens: after several shifts both are
    checked against transformers at the same steps, so their argmax agrees wherever ref64's margin decides."""
    window, R = WINDOWS[0]
    path = checkpoints(window)
    ref64, hf16, model = _models(path, R)
    _, _, full = _models(path, R)
    cfg = model.config
    B, n = 2, 100
    gen = torch.Generator(device="cuda").manual_seed(5)
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda", generator=gen)
    cap = max(n, window) + 2 * max(128, R)
    new = 4 * cap + 50
    out = model.generate(ids, max_new_tokens=new)
    assert out.shape == (B, n + new) and model.cache.max_tokens == cap, model.cache.max_tokens
    model.init_cache(B, cap)
    full.init_cache(B, n + new + 8)
    tok = model.first_tokens(model.prefill(ids)).view(B, 1)
    full.prefill(ids)
    assert torch.equal(tok, out[:, n:n + 1])
    shifts, checks = 0, 0
    for s in range(new - 1):
        if model.cache.kv_len + 1 > model.cache.max_tokens:
            model._roll()
            shifts += 1
        checked = shifts >= 2 and (s % 37 == 0 or s >= new - 3)
        if checked:
            r, h = _reference_step(ref64, hf16, _exports(model), cfg, tok.view(B), [n + s] * B, [0] * B)
        lg = model.decode_step(tok).clone()
        lf = full.decode_step(tok).clone()
        if checked:
            check(f"rolling decode step {s} after {shifts} shifts", lg, r, h)
            check(f"full-capacity decode step {s}", lf, r, h)
            checks += 1
        tok = model.next_tokens.view(B, 1).clone()
        assert torch.equal(tok, out[:, n + s + 1:n + s + 2]), f"step {s}: generate() took another token"
    assert shifts >= 4 and checks >= 5 and model.cache.max_tokens == cap


def test_serve_shifts_positions_out_of_every_window(checkpoints):
    """serve() on a windowed model with a cache too short for its stream without shifts: positions that fell out of every
    live window are dropped (the admission shifts), every request completes, and each request's first token is
    transformers' argmax of its prompt wherever ref64's margin decides."""
    from kivi_b200.serve import serve
    window, R = WINDOWS[0]
    ref64, hf16, model = _models(checkpoints(window), R)
    cfg = model.config
    gen = torch.Generator(device="cuda").manual_seed(7)
    reqs = [(torch.randint(0, cfg.vocab_size, (int(n),), generator=gen, device="cuda").cpu(), int(m))
            for n, m in ((60, 300), (40, 200), (80, 260), (50, 300), (70, 150), (30, 280))]
    stats = {}
    got = dict(serve(model, reqs, batch=2, max_tokens=520, stats=stats))
    assert sorted(got) == list(range(len(reqs)))
    assert stats["shifts"] > 0, stats
    for i, (p, m) in enumerate(reqs):
        assert got[i].numel() == m
        ids = p.cuda().view(1, -1)
        ref, hf = ref64(input_ids=ids).logits[:, -1], hf16(input_ids=ids).logits[:, -1]
        top2 = ref.topk(2, dim=-1).values
        bar = ALPHA * (hf.double() - ref).abs().max().item() + BETA * ref.abs().max().item()
        if (top2[0, 0] - top2[0, 1]).item() > 2 * bar:
            assert int(got[i][0]) == int(ref.argmax(-1)), f"request {i}: first token"

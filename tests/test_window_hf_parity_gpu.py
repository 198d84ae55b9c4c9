"""A windowed LlamaForCausalLM_KIVI (MistralForCausalLM_KIVI) against transformers' MistralForCausalLM with a small
config.sliding_window: prompt passes longer than the window, decode for several windows, forward() on the fused and the
9-tuple paths, serve() with shifts, and a rolling generate() several times longer than its cache.

The bar and the method are those of tests/test_hf_parity_gpu.py, with the same harness (tests/_hf.py).  Decode steps are
checked against transformers seeded with the model's own cache at that step, so the window is applied by transformers'
own mask (kv_idx > q_idx - sliding_window) to the positions the cache holds; after a shift those are the last T
positions, the RoPE positions stay absolute.  The module prints its worst ratios at its end (DESIGN.md section 3); it
takes about 75 s on one H100.
"""
import pytest
import torch

from tests._hf import (Bar, Decoder, checkpoints, exports, hf_kw, hf_positions, load_kivi, pad_mask,  # noqa: F401
                       reference_models, reference_step)

pytestmark = pytest.mark.gpu

NAME = "mistral"
WINDOWS = [(160, 64), (320, 128)]          # (sliding_window, residual_length R); K4V4 g64

bar = Bar()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    bar.report("window hf parity")


def _models(checkpoints, window, R):
    path = checkpoints(NAME, sliding_window=window)
    return reference_models(NAME, path) + [load_kivi(NAME, path, residual_length=R)]


@pytest.mark.parametrize("window,R", WINDOWS)
def test_prompt_and_decode_match_transformers(checkpoints, window, R):
    """Prompts longer than the window, unpadded and left-padded: forward() on the 9-tuple path and prefill() against
    transformers; then 3W + 3 decode steps after the unpadded prefill and W after the padded one, across K flushes, V-ring
    wraps and a window start that moves through many packed blocks."""
    d0 = list(bar.decided)
    ref64, hf16, model = _models(checkpoints, window, R)
    cfg = model.config
    B, n = 3, window + 150
    gen = torch.Generator(device="cuda").manual_seed(window)
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda", generator=gen)
    for pads, steps in (([0] * B, 3 * window + 3), ([0, 17, n - 5], window)):
        padded = any(pads)
        mask = pad_mask(pads, n)
        kw = dict(attention_mask=mask, position_ids=hf_positions(mask)) if padded else {}
        ref = ref64(input_ids=ids, **hf_kw(kw, torch.float64, window)).logits
        hf = hf16(input_ids=ids, **hf_kw(kw, torch.float16, window)).logits
        real = mask.bool()
        model.fused_forward = False
        bar.check(f"w{window} forward padded={padded}", model(input_ids=ids, **kw).logits[real], ref[real], hf[real])
        model.fused_forward = True
        model.init_cache(B, n + steps + 8)
        last = model.prefill(ids, attention_mask=mask if padded else None)
        bar.check(f"w{window} prefill padded={padded}", last, ref[:, -1], hf[:, -1])
        tk0 = model.cache.tk
        Decoder(bar, model, ref64, hf16, T=n, pos=[n - p for p in pads], start=pads, gen=gen).run(
            steps, f"w{window} decode padded={padded}", every=11)
        assert model.cache.tk > tk0 and model.cache.vhead != 0
    bar.assert_decided(d0)


def test_forward_fused_and_tuple_paths_agree_with_transformers(checkpoints):
    """forward() decode steps past the window on the fused cache (KiviPast) and on the reference's 9-tuples (the window
    as an additive mask), each against transformers seeded with that path's own cache."""
    window, R = WINDOWS[0]
    ref64, hf16, model = _models(checkpoints, window, R)
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
            r_f, h_f = reference_step(ref64, hf16, [tuple(p) for p in fused], cfg, tok, pos, [0] * B)
            r_t, h_t = reference_step(ref64, hf16, tuples, cfg, tok, pos, [0] * B)
        model.fused_forward = True
        lf, fused = model(input_ids=tok, past_key_values=fused, return_dict=False)
        model.fused_forward = False
        lt, tuples = model(input_ids=tok, past_key_values=tuples, return_dict=False)
        if checked:
            bar.check(f"fused forward step {s}", lf[:, -1], r_f, h_f)
            bar.check(f"tuple forward step {s}", lt[:, -1], r_t, h_t)


def test_rolling_generate_matches_transformers_and_full_cache(checkpoints):
    """generate() of a windowed model holds about max(prompt, W) + 2 max(128, R) positions and runs for more than four
    times that.  The same steps driven by hand (prefill, decode_step, a shift whenever the cache is full) take generate()'s
    ids, and a twin model on a full-capacity cache (never shifted) is fed the same tokens: after several shifts both are
    checked against transformers at the same steps, so their argmax agrees wherever ref64's margin decides."""
    window, R = WINDOWS[0]
    ref64, hf16, model = _models(checkpoints, window, R)
    full = load_kivi(NAME, checkpoints(NAME, sliding_window=window), residual_length=R)
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
            r, h = reference_step(ref64, hf16, exports(model), cfg, tok.view(B), [n + s] * B, [0] * B)
        lg = model.decode_step(tok).clone()
        lf = full.decode_step(tok).clone()
        if checked:
            bar.check(f"rolling decode step {s} after {shifts} shifts", lg, r, h)
            bar.check(f"full-capacity decode step {s}", lf, r, h)
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
    ref64, hf16, model = _models(checkpoints, window, R)
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
        bar.argmax_agrees(f"request {i}: first token", got[i][:1], ref64(input_ids=ids).logits[:, -1],
                          hf16(input_ids=ids).logits[:, -1])

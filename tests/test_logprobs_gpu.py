"""Log-probabilities on the GPU: kivi_token_logprobs_f32 against the float64 reference of tests/_logprobs.py (top ids
exactly, values within the bar DESIGN.md derives), and the model's in-step logprobs, serve()'s per-request logprobs and
generate()'s scores and logits against eager restatements."""
import pytest
import torch

from tests._attn import left_padded, tiny_model
from tests._logits import reference_process, same_bits
from tests._logprobs import lse_of, reference_logprobs, within_bar
from tests._model import graphs, requests, small_cfg, world_one_pair  # noqa: F401

pytestmark = pytest.mark.gpu


def _run(logits, tokens, n):
    from kivi_b200 import glue
    B = logits.shape[0]
    x = logits.cuda().contiguous()
    lp = torch.full((B,), 12345.0, device="cuda")
    ids = torch.full((B, n), 777, dtype=torch.long, device="cuda") if n else None
    top = torch.full((B, n), 12345.0, device="cuda") if n else None
    glue.token_logprobs(x, tokens.cuda(), lp, ids, top)
    return lp, ids, top


def _rows(B, V, g, kind):
    if kind == "peaked":
        return torch.randn((B, V), generator=g) * 30
    if kind == "flat":
        return torch.randn((B, V), generator=g) * 1e-3
    if kind == "huge":
        return (torch.rand((B, V), generator=g) * 2 - 1) * 1e4
    if kind == "ties":                                                    # many equal values at and around the N-th place
        x = torch.randint(0, 6, (B, V), generator=g).float()
        x[:, ::3] = 5.0
        return x
    x = torch.randn((B, V), generator=g) * 4                              # special values
    for b in range(B):
        c = b % 4
        if c == 0:
            x[b, torch.randint(0, V, (max(1, V // 50),), generator=g)] = float("-inf")
        elif c == 1:
            x[b, V // 2] = float("nan")
            x[b, V - 1] = float("nan")
        elif c == 2:
            x[b, V // 3] = float("inf")
        else:
            x[b] = float("-inf")
    return x


def _check(logits, tokens, n):
    lp, ids, top = _run(logits, tokens, n)
    r_lp, r_ids, r_top = reference_logprobs(logits, tokens, n)
    lse = lse_of(logits)
    V = logits.shape[1]
    t = tokens.clamp(0, V - 1)
    ok, worst = within_bar(lp, r_lp, logits.gather(1, t.view(-1, 1)).view(-1), lse)
    assert ok, ("token logprob", worst)
    if n:
        assert torch.equal(ids.cpu(), r_ids), (ids.cpu()[:2], r_ids[:2])
        xs = torch.where(r_ids >= 0, logits.gather(1, r_ids.clamp(min=0)), torch.tensor(0.0))
        ok, worst = within_bar(top, r_top, xs, lse.view(-1, 1))
        assert ok, ("top logprobs", worst)
        hit = (ids == tokens.cuda().view(-1, 1))                          # the chosen token's value is its entry's bits
        for b, j in hit.nonzero().tolist():
            assert same_bits(lp[b], top[b, j])
    return lp, ids, top


@pytest.mark.parametrize("V", [1, 7, 20, 21, 32000, 32003, 128256])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_kernel_matches_reference(B, V):
    if B == 64 and V < 32000:
        pytest.skip("small vocabularies are covered at B 1 and 3")
    g = torch.Generator().manual_seed(B * 131 + V)
    for kind in ("peaked", "flat", "huge", "ties", "special"):
        logits = _rows(B, V, g, kind)
        tokens = torch.randint(0, V, (B,), generator=g)
        tokens[0] = logits[0].nan_to_num(nan=float("inf")).argmax()       # the chosen token in the list
        for n in (0, 1, 5, 20):
            _check(logits, tokens, n)


def test_tokens_outside_the_vocabulary_give_nan():
    g = torch.Generator().manual_seed(3)
    logits = torch.randn((4, 1000), generator=g)
    lp, _, _ = _check(logits, torch.tensor([-1, 1000, 5, 2 ** 40]), 3)
    assert torch.isnan(lp[[0, 1, 3]]).all() and torch.isfinite(lp[2])


def test_runs_are_bit_identical_and_rows_independent():
    g = torch.Generator().manual_seed(4)
    V, n = 128256, 20
    logits = torch.randn((9, V), generator=g) * 6
    tokens = torch.randint(0, V, (9,), generator=g)
    a = _run(logits, tokens, n)
    b = _run(logits, tokens, n)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y)
    other = torch.randn((5, V), generator=g) * 50                          # row 4 among other rows, at another index
    mixed = torch.cat([other[:2], logits[4:5], other[2:]])
    c = _run(mixed, torch.cat([tokens[:2], tokens[4:5], tokens[2:5]]), n)
    assert same_bits(c[0][2], a[0][4]) and torch.equal(c[1][2], a[1][4]) and same_bits(c[2][2], a[2][4])


def test_captured_call_replays_with_new_inputs():
    from kivi_b200 import glue
    g = torch.Generator().manual_seed(5)
    B, V, n = 3, 32003, 7
    x = torch.zeros((B, V), device="cuda")
    tok = torch.zeros(B, dtype=torch.long, device="cuda")
    lp, ids, top = (torch.empty(B, device="cuda"), torch.empty((B, n), dtype=torch.long, device="cuda"),
                    torch.empty((B, n), device="cuda"))
    glue.token_logprobs(x, tok, lp, ids, top)                             # loads the module before the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        glue.token_logprobs(x, tok, lp, ids, top)
    for _ in range(3):
        logits = torch.randn((B, V), generator=g) * 10
        tokens = torch.randint(0, V, (B,), generator=g)
        x.copy_(logits)
        tok.copy_(tokens)
        graph.replay()
        e = _run(logits, tokens, n)
        assert same_bits(lp, e[0]) and torch.equal(ids, e[1]) and same_bits(top, e[2])


# ------------------------------------------------------------------------------------------------ the model
def _step_matches_eager(model, n, what):
    """The step's in-graph logprobs are the kernel run eagerly on the step's logits and ids, bit for bit, and within the
    bar of the float64 log-softmax."""
    logits, tok = model._logits.clone(), model.next_tokens.clone()
    e = _run(logits, tok, n)
    assert same_bits(model.logprobs, e[0]), what
    if n:
        assert torch.equal(model.top_ids, e[1]) and same_bits(model.top_logprobs, e[2]), what
    r = reference_logprobs(logits.cpu(), tok.cpu(), n)
    ok, worst = within_bar(model.logprobs, r[0], logits.gather(1, tok.view(-1, 1)).view(-1), lse_of(logits))
    assert ok, (what, worst)


@pytest.mark.parametrize("mode", ["graph", "eager", "padded", "sampled", "processed", "window"])
def test_step_logprobs(mode):
    """generate() without logprobs, then the same decoding step by step with set_logprobs on: the same ids, one more
    launch, and every checked step's logprobs equal to the kernel run eagerly on the step's logits."""
    kw = dict(sliding_window=96, residual_length=32) if mode == "window" else {}
    model, cfg = tiny_model(11, **kw)
    B, n_top = 3, 5
    n, new = (150, 300) if mode == "window" else (40, 24)
    lengths = [40, 23, 31] if mode == "padded" else [n] * B
    ids, mask = left_padded(cfg, lengths, n, seed=2)
    graph = mode != "eager"
    gk = dict(max_new_tokens=new, attention_mask=mask, use_graph=graph)
    if mode == "sampled":
        gk.update(do_sample=True, temperature=1.2, top_k=30, top_p=0.9, seed=3)
    if mode == "processed":
        gk.update(repetition_penalty=1.3)
    plain = model.generate(ids, **gk)
    base = model.launches_per_step if graph else None
    model.set_logprobs(n_top)
    if mode == "sampled":
        model.set_sampling(1.2, 30, 0.9, 3)                                # draws from 0 again, as generate() starts
    first = model.prefill(ids, mask)
    tok = model.choose_first(first)
    e = _run(first, tok, n_top)
    assert same_bits(model.logprobs, e[0]) and torch.equal(model.top_ids, e[1])
    out = [tok.view(B, 1)]
    for s in range(1, new):
        if model.cache.kv_len + 1 > model.cache.max_tokens:
            model._roll()
        model.decode_step(out[-1], use_graph=graph)
        out.append(model.next_tokens.view(B, 1).clone())
        if s % 7 == 1 or s == new - 1:
            _step_matches_eager(model, n_top, f"{mode} step {s}")
    assert torch.equal(torch.cat([ids] + out, 1), plain), "logprobs changed the tokens"
    if graph:
        assert model.launches_per_step == base + 1


def test_logprobs_off_is_todays_step(graphs):
    model, cfg = tiny_model(12)
    twin, _ = tiny_model(12)
    ids = torch.randint(1, cfg.vocab_size, (3, 33), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    base = twin.generate(ids, max_new_tokens=20)
    logits_base = twin._logits.clone()
    model.generate(ids, max_new_tokens=4)
    model.set_logprobs(3)
    on = model.generate(ids, max_new_tokens=20)                            # a larger cache: the mode is kept
    assert model.top_ids.shape == (3, 3)
    assert torch.equal(on, base) and model.launches_per_step == twin.launches_per_step + 1
    made = graphs.made
    model.set_logprobs(3)                                                  # the same N: the same captured step
    assert model._graph is not None and graphs.made == made
    model.set_logprobs(4)                                                  # another N: recaptured
    assert model._graph is None
    model.set_logprobs(None)
    assert model.logprobs is None and model._graph is None
    off = model.generate(ids, max_new_tokens=20)
    assert torch.equal(off, base) and torch.equal(model._logits, logits_base)
    assert model.launches_per_step == twin.launches_per_step


def test_tensor_parallel_world_one_logprobs():
    cfg = small_cfg()
    plain, tpm = world_one_pair(cfg)
    ids, mask = left_padded(cfg, [40, 31], 40, seed=5)
    for m in (plain, tpm):
        m.generate(ids, max_new_tokens=2, attention_mask=mask)
        m.set_logprobs(4)
    a = plain.generate(ids, max_new_tokens=20, attention_mask=mask)
    b = tpm.generate(ids, max_new_tokens=20, attention_mask=mask)
    assert torch.equal(a, b)
    assert same_bits(plain.logprobs, tpm.logprobs) and torch.equal(plain.top_ids, tpm.top_ids)
    _step_matches_eager(tpm, 4, "tensor parallel")


# ------------------------------------------------------------------------------------------------ serve()
BUDGETS = [57, 17, 52, 39, 58, 64, 75, 83]


def _lp_params():
    return [dict(logprobs=3), None, dict(logprobs=0, temperature=1.1, top_p=0.9, seed=4), dict(logprobs=20), None,
            dict(temperature=1.2, top_k=30, seed=5), dict(logprobs=5, repetition_penalty=1.2), dict(logprobs=1)]


def test_serve_logprobs():
    from kivi_b200.serve import TokenLogprobs, serve
    model, cfg = tiny_model(2)
    par = _lp_params()
    plain_par = [None if p is None else {k: v for k, v in p.items() if k != "logprobs"} or None for p in par]
    eos = [cfg.vocab_size - 1]
    off = list(serve(model, requests(cfg, BUDGETS, params=plain_par), 3, 260, eos_token_id=eos))
    assert all(len(r) == 2 for r in off)
    off = dict(off)
    got = {}
    for r in serve(model, requests(cfg, BUDGETS, params=par), 3, 260, eos_token_id=eos):
        assert len(r) == 3
        got[r[0]] = r[1:]
    assert model.top_ids.shape[1] == 20
    for i in range(8):
        ids, lp = got[i]
        assert torch.equal(ids, off[i]), i                                # logprobs never change the tokens
        if par[i] is None or "logprobs" not in par[i]:
            assert lp is None, i
            continue
        n, k = par[i]["logprobs"], ids.numel()
        assert isinstance(lp, TokenLogprobs)
        assert lp.token.shape == (k,) and lp.top_ids.shape == (k, n) and lp.top.shape == (k, n)
        assert lp.token.dtype == torch.float32 and lp.top_ids.dtype == torch.int64 and not lp.token.is_cuda
        assert (lp.token <= 0).all() and torch.isfinite(lp.token).all()
        if n:
            assert (lp.top[:, :-1] >= lp.top[:, 1:]).all()
            hit = lp.top_ids == ids.view(-1, 1)
            assert torch.equal(lp.top[hit], lp.token[hit.any(1)])
        # the same request decoded alone
        alone = list(serve(tiny_model(2)[0], [requests(cfg, BUDGETS, params=par)[i]], 1, 260, eos_token_id=eos))
        (_, ids1, lp1), = alone
        assert torch.equal(ids1, ids), i
        # alone, the prompt is not left-padded and the batch has one row: the logits agree to the model-level bar
        assert torch.allclose(lp1.token, lp.token, atol=2e-2, rtol=0), i
        if n:
            assert torch.allclose(lp1.top, lp.top, atol=2e-2, rtol=0), i
            assert (lp1.top_ids == lp.top_ids).float().mean() > 0.9, i
    again = list(serve(model, requests(cfg, BUDGETS), 3, 260))            # without the key: 2-tuples, the mode off
    assert all(len(r) == 2 for r in again) and model.logprobs is None


# ------------------------------------------------------------------------------------------------ generate()
def _eager_loop(twin, ids, new, mask=None, proc=None):
    """An eager decode_step loop with processing as generate() sets it: the raw logits and the processed scores of every
    new token (the first from the prompt), and the tokens."""
    B = ids.shape[0]
    twin.init_cache(B, ids.shape[1] + new)
    twin._tables(twin.cache.device, ids.shape[1] + new)
    twin.set_sampling(None)
    if proc:
        twin.set_processing(**proc)
    else:
        twin.set_processing(None)
    first = twin.prefill(ids, mask)
    tok, sc = twin.choose_first(first, return_scores=True)
    logits, scores, toks = [first.clone()], [sc.clone()], [tok.view(B, 1)]
    for _ in range(1, new):
        lg = twin.decode_step(toks[-1], use_graph=False)
        logits.append(lg.clone())
        scores.append(twin._proc.scores.clone() if proc else lg.clone())
        toks.append(twin.next_tokens.view(B, 1).clone())
    return logits, scores, torch.cat(toks, 1)


@pytest.mark.parametrize("case", ["plain", "processed", "eos"])
def test_generate_scores_and_logits(case):
    model, cfg = tiny_model(13)
    twin, _ = tiny_model(13)
    B, n, new = 3, 37, 30
    ids, mask = left_padded(cfg, [37, 30, 22], n, seed=6)
    kw = {}
    if case != "plain":
        kw.update(repetition_penalty=1.3)
    if case == "eos":
        ref = twin.generate(ids, max_new_tokens=12, attention_mask=mask, repetition_penalty=1.3)
        kw.update(eos_token_id=sorted({int(x) for x in ref[:, n + 6]}))
    out = model.generate(ids, max_new_tokens=new, attention_mask=mask, return_dict_in_generate=True, output_logits=True,
                         output_scores=True, **kw)
    k = out.sequences.shape[1] - n
    assert len(out.logits) == k and len(out.scores) == k
    if case == "eos":
        assert k < new
    proc = None
    if kw:
        from kivi_b200.llama_kivi import _processing_args
        proc = _processing_args(n, kw["repetition_penalty"], None, None, kw.get("eos_token_id"), None)
    logits, scores, toks = _eager_loop(twin, ids, new, mask, proc)
    assert torch.equal(out.sequences[:, n:], toks[:, :k])
    for s in range(k):
        assert torch.equal(out.logits[s], logits[s]), s                    # raw logits: bit for bit
        assert same_bits(out.scores[s], scores[s]), s
        if proc is not None and s > 0:                                      # the restatement on unfinished rows
            p = twin._proc
            alive = ~torch.isin(out.sequences[:, n:n + s], torch.tensor(kw.get("eos_token_id", [-1]), device="cuda")).any(1)
            seen = torch.zeros((B, cfg.vocab_size), dtype=torch.bool)
            for b in range(B):
                seen[b, ids[b, mask[b].bool()].cpu()] = True
            counts = torch.zeros((B, cfg.vocab_size), dtype=torch.long)
            counts.scatter_add_(1, out.sequences[:, n:n + s].cpu(), torch.ones((B, s), dtype=torch.long))
            exp = reference_process(logits[s].cpu(), counts, seen, torch.full((B,), s, dtype=torch.int32),
                                    torch.zeros(B, dtype=torch.bool), torch.full((B,), 1.3), torch.zeros(B), torch.zeros(B),
                                    torch.zeros(B, dtype=torch.int32), [], 0)
            assert same_bits(out.scores[s][alive].cpu(), exp[alive.cpu()]), s
            del p
    ts = model.compute_transition_scores(out.sequences, out.logits, normalize_logits=True)
    assert ts.shape == (B, k) and (ts <= 0).all()
    plain = model.generate(ids, max_new_tokens=new, attention_mask=mask, **kw)
    assert torch.equal(plain, out.sequences)


def test_sampled_num_return_sequences_logits():
    model, cfg = tiny_model(14)
    ids = torch.randint(1, cfg.vocab_size, (2, 45), device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    kw = dict(max_new_tokens=16, do_sample=True, temperature=0.9, top_k=0, top_p=0.9, seed=3, num_return_sequences=3)
    out = model.generate(ids, return_dict_in_generate=True, output_logits=True, **kw)
    assert out.scores is None and len(out.logits) == 16 and out.logits[0].shape == (6, cfg.vocab_size)
    assert torch.equal(out.logits[0][0], out.logits[0][2]) and not torch.equal(out.logits[0][0], out.logits[0][3])
    again = model.generate(ids, **kw)
    assert torch.equal(again, out.sequences)
    # the logits are what the step computed from the chosen tokens: replay them eagerly
    twin, _ = tiny_model(14)
    twin.init_cache(6, 45 + 16)
    twin._tables(twin.cache.device, 45 + 16)
    first = twin.lm_head(twin._prompt_pass(ids, None, copies=3)[:, -1]).float().repeat_interleave(3, 0)
    assert torch.equal(first, out.logits[0])
    for s in range(1, 16):
        lg = twin.decode_step(out.sequences[:, 45 + s - 1:45 + s], use_graph=False)
        assert torch.equal(lg, out.logits[s]), s

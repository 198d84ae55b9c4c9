"""Logits processing on the GPU: kivi_logits_process_f32 and kivi_logits_record against the torch restatement of
tests/_logits.py bit for bit, and the model's fused processing (generate, serve) against a host loop that runs the
decode steps without processing and applies transformers' processors to the raw logits."""
import pytest
import torch

from tests._attn import left_padded, tiny_model
from tests._logits import pack_bits, reference_process, same_bits, special_logits, unpack_bits
from tests._model import graphs, requests, world_one_pair, small_cfg  # noqa: F401

pytestmark = pytest.mark.gpu


def _state(B, V, gen, eos):
    """Random per-row state and parameters (CPU): penalties below, at and above 1, counts in the thousands on a few
    tokens, random prompt bits, rows below and above their minimum length, and finished rows."""
    counts = torch.zeros((B, V), dtype=torch.int32)
    hot = torch.randint(0, V, (B, 64), generator=gen)
    counts.scatter_(1, hot, torch.randint(1, 5000, (B, 64), generator=gen, dtype=torch.int32))
    seen = torch.rand((B, V), generator=gen) < 0.01
    for b in range(B):
        seen[b, eos[b % len(eos)]] = True                                  # an EOS id in the prompt
    rep = torch.tensor([0.5, 1.0, 1.3, 1.0, 2.0])[torch.arange(B) % 5]
    pres = (torch.rand(B, generator=gen) * 4 - 2) * (torch.arange(B) % 4 != 1)
    freq = (torch.rand(B, generator=gen) * 4 - 2) * (torch.arange(B) % 3 != 1)
    n_new = torch.randint(0, 20, (B,), generator=gen, dtype=torch.int32)
    min_new = torch.randint(0, 20, (B,), generator=gen, dtype=torch.int32)
    finished = (torch.arange(B) % 7 == 3)
    return dict(counts=counts, seen=seen, repetition=rep, presence=pres.float(), frequency=freq.float(), n_new=n_new,
                min_new=min_new, finished=finished)


def _run_kernel(logits, st, eos, pad):
    from kivi_b200 import glue
    c = lambda t: t.cuda().contiguous()                                   # noqa: E731
    scores = torch.full_like(c(logits), 12345.0)
    e = torch.tensor(eos, dtype=torch.long, device="cuda") if eos else None
    glue.logits_process(c(logits), scores, c(st["counts"]), c(pack_bits(st["seen"])), c(st["n_new"]),
                        c(st["finished"].to(torch.uint8)), c(st["repetition"]), c(st["presence"]), c(st["frequency"]),
                        c(st["min_new"]), e, pad)
    return scores


@pytest.mark.parametrize("B,V", [(1, 32000), (3, 32001), (64, 128256)])
@pytest.mark.parametrize("n_eos", [1, 8])
def test_kernel_matches_restatement(B, V, n_eos):
    gen = torch.Generator().manual_seed(B * 7 + n_eos)
    for trial in range(3):
        eos = torch.randperm(V, generator=gen)[:n_eos].tolist()
        pad = int(torch.randint(0, V, (1,), generator=gen))
        logits = special_logits(B, V, gen)
        st = _state(B, V, gen, eos)
        if B == 1:                                                         # the one row: every step on, then finished
            st.update(repetition=torch.tensor([(0.7, 1.4, 1.0)[trial]]), presence=torch.tensor([0.75]),
                      frequency=torch.tensor([-1.5]), n_new=torch.tensor([0], dtype=torch.int32),
                      min_new=torch.tensor([3], dtype=torch.int32), finished=torch.tensor([trial == 2]))
        got = _run_kernel(logits, st, eos, pad)
        exp = reference_process(logits, st["counts"], st["seen"], st["n_new"], st["finished"], st["repetition"],
                                st["presence"], st["frequency"], st["min_new"], eos, pad)
        assert same_bits(got, exp), (trial, (got.cpu() != exp).nonzero()[:5])


@pytest.mark.parametrize("B,V", [(3, 32000), (2, 32001)])
def test_neutral_rows_are_the_logits(B, V):
    gen = torch.Generator().manual_seed(5)
    logits = special_logits(B, V, gen)
    st = _state(B, V, gen, [1])
    st.update(repetition=torch.ones(B), presence=torch.zeros(B), frequency=torch.zeros(B),
              min_new=torch.zeros(B, dtype=torch.int32), finished=torch.zeros(B, dtype=torch.bool))
    got = _run_kernel(logits, st, [1, 2], 0)
    assert torch.equal(got.cpu().view(torch.int32), logits.view(torch.int32))     # NaN payloads included


def test_record_counts_are_the_bincount():
    from kivi_b200 import glue
    B, V, calls = 5, 32001, 3000
    gen = torch.Generator(device="cuda").manual_seed(1)
    counts = torch.zeros((B, V), dtype=torch.int32, device="cuda")
    n_new = torch.zeros(B, dtype=torch.int32, device="cuda")
    finished = torch.zeros(B, dtype=torch.uint8, device="cuda")
    eos = torch.tensor([V - 1, 7], dtype=torch.long, device="cuda")
    toks = torch.randint(0, 40, (calls, B), device="cuda", generator=gen)   # many repeats: counts in the hundreds
    toks[100, 2] = V - 1                                                   # row 2 emits an EOS at call 100
    toks[:, 0] = toks[:, 0].clamp(min=8)                                   # row 0 never does
    toks[:, 3] = toks[:, 3].clamp(min=8)
    toks[:, 4] = toks[:, 4].clamp(min=8)
    toks[5, 4] = 7
    for t in toks:
        glue.logits_record(t.contiguous(), counts, n_new, finished, eos)
    for b in range(B):
        assert torch.equal(counts[b].long().cpu(), torch.bincount(toks[:, b].cpu(), minlength=V)), b
    assert n_new.tolist() == [calls] * B
    exp = [int(bool(((toks[:, b] == V - 1) | (toks[:, b] == 7)).any())) for b in range(B)]
    assert finished.tolist() == exp and exp[0] == 0 and exp[2] == 1 and exp[4] == 1


# ------------------------------------------------------------------------------------------------ the model
def _hf_processors(n, rep, min_length, min_new, eos):
    from transformers.generation.logits_process import (LogitsProcessorList, MinLengthLogitsProcessor,
                                                        MinNewTokensLengthLogitsProcessor, RepetitionPenaltyLogitsProcessor)
    procs = LogitsProcessorList()
    if rep is not None and rep != 1.0:
        procs.append(RepetitionPenaltyLogitsProcessor(rep))
    if eos is not None and min_length is not None:
        procs.append(MinLengthLogitsProcessor(min_length, eos))
    if eos is not None and min_new is not None:
        procs.append(MinNewTokensLengthLogitsProcessor(n, min_new, eos))
    return procs


def host_loop(twin, ids, new, mask=None, rep=None, min_length=None, min_new=None, eos=None, pad=None, sample=None,
              copies=1):
    """transformers' greedy / sampling loop over the twin's decode steps (processing off): its processors on the raw
    logits (on the CPU: IEEE division), the argmax or glue.sample with the rows' seeds and draws (sample = (temperature,
    top_k, top_p, seed)), pad after EOS, and the stop once every row has finished.  Left padding is replaced by the row's
    last token in the ids the processors see (the fused path does not penalise padding).  copies = K: K rows per prompt,
    the prompt run once for all of them, as generate(num_return_sequences=K)."""
    from kivi_b200 import glue
    from kivi_b200.choice import sampling_rows
    B, n = ids.shape
    rows = B * copies
    eos_l = None if eos is None else (eos if isinstance(eos, list) else [eos])
    pad = pad if pad is not None else (eos_l[0] if eos_l else 0)
    cap = n + new
    if twin.sliding_window is not None:
        cap = min(cap, max(n, twin.sliding_window) + 2 * max(128, twin.config.residual_length))
    twin.init_cache(rows, cap)
    twin._tables(twin.cache.device, n + new)
    twin.set_sampling(None)
    logits = twin.lm_head(twin._prompt_pass(ids, mask, copies=copies)[:, -1]).float().repeat_interleave(copies, 0)
    seen = ids.clone()
    if mask is not None:
        seen = torch.where(mask.bool(), seen, seen[:, -1:])
    seq = seen.repeat_interleave(copies, 0).cpu()
    out = ids.repeat_interleave(copies, 0)
    procs = _hf_processors(n, rep, min_length, min_new, eos_l)
    if sample is not None:
        t, k, p, sd = sampling_rows(rows, *sample)
        T, K, P = (torch.tensor(t, device="cuda"), torch.tensor(k, dtype=torch.int32, device="cuda"),
                   torch.tensor(p, device="cuda"))
        seed, draw = torch.tensor(sd, device="cuda"), torch.zeros(rows, dtype=torch.long, device="cuda")
    unfinished = torch.ones(rows, dtype=torch.long, device="cuda")
    for step in range(new):
        scores = procs(seq, logits.cpu().clone()).cuda().contiguous()
        if sample is None:
            tok = scores.argmax(-1)
        else:
            tok = torch.empty(rows, dtype=torch.long, device="cuda")
            glue.sample(scores, T, K, P, seed, draw, tok)
        tok = tok * unfinished + pad * (1 - unfinished)
        out = torch.cat([out, tok.view(rows, 1)], 1)
        seq = torch.cat([seq, tok.view(rows, 1).cpu()], 1)
        if eos_l is not None:
            unfinished = unfinished * (~torch.isin(tok, torch.tensor(eos_l, device="cuda"))).long()
            if int(unfinished.max()) == 0:
                break
        if step + 1 < new:
            if twin.cache.kv_len + 1 > twin.cache.max_tokens:
                twin._roll()
            logits = twin.decode_step(tok.view(rows, 1)).clone()
    return out


def _frequent(model, ids, new, mask=None, k=2):
    """The k most frequent generated ids of each row of a plain greedy run: EOS ids every row is likely to meet."""
    g = model.generate(ids, max_new_tokens=new, attention_mask=mask)[:, ids.shape[1]:]
    return sorted({int(x) for row in g for x in torch.bincount(row[2:]).topk(k).indices})[:8]


@pytest.mark.parametrize("mode", ["graph", "eager", "padded", "sampled"])
def test_generate_matches_host_loop(mode):
    model, cfg = tiny_model(4)
    twin, _ = tiny_model(4)
    B, n, new = 3, 40, 48
    if mode == "padded":
        ids, mask = left_padded(cfg, [40, 23, 31], n, seed=3)
    else:
        ids, mask = torch.randint(1, cfg.vocab_size, (B, n), device="cuda",
                                  generator=torch.Generator(device="cuda").manual_seed(3)), None
    eos = _frequent(twin, ids, new, mask, k=1)
    sample = (1.1, 40, 0.95, 9) if mode == "sampled" else None
    kw = dict(do_sample=True, temperature=1.1, top_k=40, top_p=0.95, seed=9) if sample else {}
    got = model.generate(ids, max_new_tokens=new, attention_mask=mask, repetition_penalty=1.3, min_new_tokens=4,
                         eos_token_id=eos, use_graph=mode != "eager", **kw)
    exp = host_loop(twin, ids, new, mask, rep=1.3, min_new=4, eos=eos, sample=sample)
    assert got.shape == exp.shape and torch.equal(got, exp)
    plain = model.generate(ids, max_new_tokens=new, attention_mask=mask, **kw)
    assert plain.shape == (B, n + new) and not torch.equal(got[:, :n + 8], plain[:, :n + 8])   # the penalty acts


def test_pred_long_bench_call_shape():
    """pred_long_bench.py's call: greedy, min_length = context + 1, eos_token_id = [eos, newline].  The ids have the shape
    transformers' greedy generate gives: cut at the step where the last row finished, pad after a row's EOS."""
    model, cfg = tiny_model(6)
    twin, _ = tiny_model(6)
    B, n, max_gen = 2, 57, 64
    ids = torch.randint(1, cfg.vocab_size, (B, n), device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    eos = _frequent(twin, ids, max_gen, k=1)[:2]
    got = model.generate(ids, max_new_tokens=max_gen, num_beams=1, do_sample=False, temperature=1.0, min_length=n + 1,
                         eos_token_id=eos)
    exp = host_loop(twin, ids, max_gen, min_length=n + 1, eos=eos)
    assert got.shape == exp.shape and torch.equal(got, exp)
    assert got.shape[1] < n + max_gen, "every row met an EOS"
    for b in range(B):
        row = got[b, n:].tolist()
        hits = [i for i, t in enumerate(row) if t in eos]
        assert hits, b
        assert all(t == eos[0] for t in row[hits[0] + 1:]), b              # pad (the first EOS id) after the EOS


def test_windowed_roll_matches_host_loop():
    model, cfg = tiny_model(7, sliding_window=96, residual_length=32)
    twin, _ = tiny_model(7, sliding_window=96, residual_length=32)
    ids = torch.randint(1, cfg.vocab_size, (2, 150), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    new = 300
    got = model.generate(ids, max_new_tokens=new, repetition_penalty=1.2, eos_token_id=[cfg.vocab_size - 1])
    assert model.cache.max_tokens < 150 + new, "the windowed cache rolled"
    exp = host_loop(twin, ids, new, rep=1.2, eos=[cfg.vocab_size - 1])
    assert torch.equal(got, exp)


def test_num_return_sequences_sampling_matches_host_loop():
    model, cfg = tiny_model(8)
    twin, _ = tiny_model(8)
    ids = torch.randint(1, cfg.vocab_size, (2, 45), device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    eos = _frequent(twin, ids, 40, k=1)
    got = model.generate(ids, max_new_tokens=40, do_sample=True, temperature=0.9, top_k=0, top_p=0.9, seed=3,
                         num_return_sequences=3, repetition_penalty=1.25, eos_token_id=eos, min_length=50)
    exp = host_loop(twin, ids, 40, rep=1.25, eos=eos, min_length=50, sample=(0.9, 0, 0.9, 3), copies=3)
    assert got.shape == exp.shape and torch.equal(got, exp)


def test_tensor_parallel_world_one_processes_like_the_model():
    cfg = small_cfg()
    plain, tpm = world_one_pair(cfg)
    ids, mask = left_padded(cfg, [40, 31], 40, seed=5)
    kw = dict(max_new_tokens=2 * cfg.residual_length + 5, attention_mask=mask, repetition_penalty=1.4,
              eos_token_id=[3, 9], min_new_tokens=5)
    a, b = plain.generate(ids, **kw), tpm.generate(ids, **kw)
    assert torch.equal(a, b) and plain.launches_per_step == tpm.launches_per_step
    exp = host_loop(plain, ids, kw["max_new_tokens"], mask, rep=1.4, eos=[3, 9], min_new=5)
    assert torch.equal(a, exp)


def test_counts_after_replays_are_the_fed_ids(graphs):
    """After generate() with k replayed steps, counts is the bincount of the ids it returned: the warm-up step before
    capture is undone, not counted twice.  Turning processing on and off recaptures, parameters alone do not, and the
    launch count grows by exactly the two processing kernels."""
    model, cfg = tiny_model(9)
    B, n, new = 3, 33, 20
    ids = torch.randint(1, cfg.vocab_size, (B, n), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    base = model.generate(ids, max_new_tokens=new)
    plain_launches = model.launches_per_step
    assert graphs.made == 1 and model._proc is None
    got = model.generate(ids, max_new_tokens=new, repetition_penalty=1.5)
    assert graphs.made == 2 and model.launches_per_step == plain_launches + 2
    p = model._proc
    for b in range(B):
        assert torch.equal(p.counts[b].long(), torch.bincount(got[b, n:], minlength=cfg.vocab_size)), b
        assert torch.equal(torch.nonzero(unpack_bits(p.seen[b:b + 1].cpu(), cfg.vocab_size)[0]).view(-1).cuda(),
                           torch.unique(ids[b]))
    assert p.n_new.tolist() == [new] * B and p.finished.tolist() == [0] * B
    model.generate(ids, max_new_tokens=new, repetition_penalty=1.1)        # other parameters: the same captured step
    assert graphs.made == 2
    again = model.generate(ids, max_new_tokens=new)                       # processing off: today's step, today's bits
    assert graphs.made == 3 and model._proc is None and model.launches_per_step == plain_launches
    assert torch.equal(again, base) and not torch.equal(got, base)
    neutral = model.generate(ids, max_new_tokens=new, repetition_penalty=1.0)     # asks for nothing: processing stays off
    assert torch.equal(neutral, base) and model._proc is None and graphs.made == 3


# ------------------------------------------------------------------------------------------------ serve()
BUDGETS = [57, 17, 52, 39, 58, 64, 75, 83]


def _params():
    pen = dict(repetition_penalty=1.3, presence_penalty=0.4, frequency_penalty=0.3, min_new_tokens=3)
    return [dict(pen), None, dict(pen, temperature=1.1, top_p=0.9, seed=4), dict(repetition_penalty=0.8), None,
            dict(temperature=1.2, top_k=30, seed=5), dict(frequency_penalty=1.5, seed=6, temperature=1.0), None]


def test_serve_requests_depend_on_their_own_parameters(graphs):
    """Mixed requests with penalties: the same tokens whichever slot a request gets (the first group permuted); requests
    without the new keys decode as with processing off; the step has exactly two more launches with processing."""
    from kivi_b200.serve import parse_requests, serve
    model, cfg = tiny_model(2)
    par = _params()
    split = parse_requests([([1], 1, p) for p in par])[1]
    reqs = requests(cfg, BUDGETS, params=par)
    eos = [cfg.vocab_size - 1, cfg.vocab_size - 2]
    off = dict(serve(model, requests(cfg, BUDGETS, params=[s.sampling for s in split]), 3, 260, eos_token_id=eos))
    off_launches = model.launches_per_step
    assert model.choice.proc is None
    a = dict(serve(model, reqs, 3, 260, eos_token_id=eos))
    assert model.launches_per_step == off_launches + 2 and model.choice.proc is not None
    order = [2, 0, 1] + list(range(3, 8))                                  # the first group's slots permuted
    b_perm = dict(serve(model, [reqs[i] for i in order], 3, 260, eos_token_id=eos))
    b = {order[j]: t for j, t in b_perm.items()}
    for i in range(8):
        assert torch.equal(a[i], b[i]), i
        if split[i].processing is None:
            assert torch.equal(a[i], off[i]), i                           # no processing keys: as without processing
    assert sum(not torch.equal(a[i], off[i]) for i in (0, 2, 3, 6)) >= 3
    # a neighbour's parameters do not reach a request
    other = list(par)
    other[1] = dict(repetition_penalty=2.0)
    c = dict(serve(model, requests(cfg, BUDGETS, params=other), 3, 260, eos_token_id=eos))
    for i in (0, 2, 3):
        assert torch.equal(c[i], a[i]), i
    again = dict(serve(model, requests(cfg, BUDGETS), 3, 260))
    assert model.choice.proc is None and model.launches_per_step == off_launches
    plain = dict(serve(tiny_model(2)[0], requests(cfg, BUDGETS), 3, 260))
    for i in range(8):
        assert torch.equal(again[i], plain[i]), i

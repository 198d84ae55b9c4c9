"""Sampling on the GPU.  Kernel level (kivi_sample_f32 through glue.sample) against the numpy reference of
tests/_sample.py: the uniform number bit for bit, greedy rows, the kept set, the chosen id, the distribution,
determinism across placements, argument errors.  Model level: generate(do_sample=True), serve() with per-request
parameters, tensor parallelism."""
import os

import numpy as np
import pytest
import torch

from tests._attn import tiny_model
from tests._model import (graphs, requests, same_logits, same_on_all_ranks, sharded_model, small_cfg,  # noqa: F401
                          spawn_ranks, world_one_pair)
from tests._sample import greedy_id, reference_pick, reference_row, uniform24

pytestmark = pytest.mark.gpu

VOCABS = [32000, 128256, 50257]              # staged in shared memory; re-read from L2; an odd size
BATCHES = [1, 3, 32, 64]
MODES = [(0, 1.0), (50, 1.0), (0, 0.9), (50, 0.9)]     # (top_k, top_p): both off, top-k alone, top-p alone, both
KIVI_ERR_SHAPE, KIVI_ERR_NULL = -2, -6


def _signed(x):
    return x - 2 ** 64 if x >= 2 ** 63 else x


def _run(logits, temperature, top_k, top_p, seed, draw):
    """One launch; per-row parameters as scalars or lists.  Returns (ids, n24 of dbg_u, dbg_kept, draw after) on the host."""
    from kivi_b200 import glue
    B = logits.shape[0]
    col = lambda v, dt: torch.tensor(v if isinstance(v, (list, tuple)) else [v] * B, dtype=dt, device="cuda")   # noqa: E731
    seed = [_signed(s) for s in (seed if isinstance(seed, (list, tuple)) else [seed] * B)]
    draw = [_signed(d) for d in (draw if isinstance(draw, (list, tuple)) else [draw] * B)]
    d = col(draw, torch.long)
    nxt = torch.full((B,), -1, dtype=torch.long, device="cuda")
    fb = torch.full((B,), -1, dtype=torch.long, device="cuda")
    u = torch.full((B,), -1.0, device="cuda")
    kept = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    glue.sample(logits, col(temperature, torch.float32), col(top_k, torch.int32), col(top_p, torch.float32),
                col(seed, torch.long), d, nxt, fb, u, kept)
    torch.cuda.synchronize()
    assert torch.equal(nxt, fb)
    n24 = (u.double() * 2 ** 24).round().long()
    assert torch.equal(n24.double() * 2.0 ** -24, u.double())             # u is a multiple of 2^-24 in [0, 1)
    return nxt.tolist(), n24.tolist(), kept.tolist(), [x % 2 ** 64 for x in d.tolist()]


def _rows(B, V, seed, scale=3.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((B, V), generator=g, device="cuda") * scale


@pytest.mark.parametrize("V", VOCABS)
def test_uniform_is_philox_and_draw_advances(V):
    B = 64
    logits = _rows(B, V, 1)
    seeds = [0, 1, 2 ** 32, 2 ** 63 + 5, 2 ** 64 - 1] + [12345 * (b + 1) ** 3 for b in range(B - 5)]
    draws = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 64 - 2] + [7 * b for b in range(B - 5)]
    temps = [0.0 if b % 4 == 3 else 1.0 for b in range(B)]
    ids, n24, kept, after = _run(logits, temps, 0, 1.0, seeds, draws)
    for b in range(B):
        if temps[b] == 0:
            assert after[b] == draws[b] and ids[b] == int(logits[b].argmax()) and kept[b] == 1, b
        else:
            assert n24[b] == uniform24(seeds[b], draws[b]), b
            assert after[b] == (draws[b] + 1) % 2 ** 64 and kept[b] == V, b


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("B", BATCHES)
def test_greedy_rows_equal_argmax(V, B):
    """temperature 0 is torch.argmax (first of equal maxima, a NaN wins), with ties, NaN and +-inf in the row; sampled rows
    with a +inf or without a finite logit take the same id and consume no draw, and a NaN is never sampled."""
    g = torch.Generator(device="cuda").manual_seed(B * 7 + V)
    logits = torch.randn((B, V), generator=g, device="cuda", dtype=torch.float16).float()   # fp16-rounded: ties exist
    logits[0, 5] = logits[0, 700 % V] = logits[0].max() + 1                                  # a tie for the maximum
    if B > 1:
        logits[1, V // 2] = logits[1, V - 1] = float("nan")
    if B > 2:
        logits[2, 17] = logits[2, 9] = float("inf")
        logits[2, 3] = float("-inf")
    host = logits.cpu().numpy()
    ids, _, kept, after = _run(logits, 0.0, 50, 0.9, 3, 11)
    assert ids == logits.argmax(-1).tolist() == [greedy_id(r) for r in host]
    assert after == [11] * B and kept == [1] * B
    if B >= 32:
        logits[3] = float("-inf")
        logits[4] = float("nan")
        logits[5, ::2] = float("nan")                                     # half NaN: the rest is sampled
        host = logits.cpu().numpy()
        ids, _, kept, after = _run(logits, 0.8, 0, 1.0, 3, 11)
        for b in (2, 3, 4):
            assert ids[b] == greedy_id(host[b]) and after[b] == 11 and kept[b] == 1, b
        assert ids[5] % 2 == 1 and kept[5] == V // 2 and after[5] == 12
        assert ids[1] not in (V // 2, V - 1) and kept[1] == V - 2


def _peaked_rows(B, V, seed):
    """Rows whose mass sits on 40 well-separated tokens scattered over the vocabulary; every other token is 40 units lower
    (kept when the thresholds are off, but e^-40 each)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn((B, V), generator=g, device="cuda") - 40.0
    at = torch.rand((B, V), generator=g, device="cuda").argsort(-1)[:, :40]
    logits.scatter_(1, at, torch.randn((B, 40), generator=g, device="cuda") * 2.0)
    return logits


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("rows_kind", ["peaked", "dense"])
def test_kept_set_and_chosen_id(V, rows_kind):
    """Rows without ties, B in {1, 3, 32, 64}, thresholds off / top-k / top-p / both.  Where the fp64 reference's top-p
    decision has a margin of 1e-5 of the mass, the number of kept tokens is the reference's and the id is a kept token.
    peaked (the mass on 40 tokens): the id is the reference's inverse-CDF id whenever u * S is further than 1e-5 * S from a
    CDF step, and at least 99 % of the rows of every mode are decidable so.
    dense (N(0, 2.5^2) over the whole vocabulary: with the thresholds off most tokens weigh less than any margin): the id's
    interval of the reference CDF holds u * S to within 2e-6 * S, and the id is the reference's beyond that margin."""
    EPS = 1e-5 if rows_kind == "peaked" else 2e-6
    rows = [0] * len(MODES)
    decidable = [0] * len(MODES)
    for B in BATCHES:
        for mode, (k, p) in enumerate(MODES):
            for temperature in (1.0, 0.6):
                seed = 100 * mode + B + int(temperature * 10)
                logits = _peaked_rows(B, V, seed) if rows_kind == "peaked" else _rows(B, V, seed, scale=2.5)
                host = logits.cpu().numpy()
                seeds = [1000 * mode + b for b in range(B)]
                ids, n24, kept, after = _run(logits, temperature, k, p, seeds, 4)
                assert after == [5] * B
                for b in range(B):
                    ctx = (B, mode, temperature, b)
                    assert n24[b] == uniform24(seeds[b], 4), ctx
                    w, margin = reference_row(host[b], temperature, k, p)
                    rows[mode] += 1
                    if margin <= 1e-5:
                        continue
                    assert kept[b] == int((w > 0).sum()), ctx
                    assert w[ids[b]] > 0, ctx
                    cdf = np.cumsum(w)
                    S, target = cdf[-1], n24[b] * 2.0 ** -24 * cdf[-1]
                    assert cdf[ids[b]] - w[ids[b]] - EPS * S <= target < cdf[ids[b]] + EPS * S, ctx
                    exp, margin = reference_pick(w, n24[b])
                    if margin > EPS:
                        assert ids[b] == exp, ctx
                        decidable[mode] += 1
    if rows_kind == "peaked":
        assert all(d >= 0.99 * r for d, r in zip(decidable, rows)), (decidable, rows)
    else:
        assert decidable[1] >= 0.99 * rows[1] and decidable[3] >= 0.99 * rows[3], (decidable, rows)


@pytest.mark.parametrize("V", VOCABS)
def test_ties_straddling_the_thresholds(V):
    """Equal logits stand or fall together: a tie at the k-th largest value is kept whole by top-k, a tie that the nucleus
    mass cuts through is kept whole by top-p."""
    row = torch.full((V,), -30.0)
    perm = torch.randperm(V, generator=torch.Generator().manual_seed(V))
    row[perm[:5]] = 3.0
    row[perm[5:15]] = 2.0
    row[perm[15:40]] = 1.0
    logits = row.cuda()[None].repeat(6, 1).contiguous()
    host = row.numpy()
    ks = [7, 15, 16, 0, 0, 7]
    ps = [1.0, 1.0, 1.0, 0.5, 0.75, 0.45]
    ids, n24, kept, _ = _run(logits, 1.0, ks, ps, list(range(6)), 0)
    for b in range(6):
        w, margin = reference_row(host, 1.0, ks[b], ps[b])
        assert margin > 1e-3
        assert kept[b] == int((w > 0).sum()), b
        assert ids[b] == reference_pick(w, n24[b])[0], b
    assert kept == [15, 15, 40, 15, 40, 5]                                # k = 7 and p = 0.5 fall inside the ten tokens at 2.0
    # fp16-rounded random rows: thousands of exact ties, thresholds wherever they fall
    g = torch.Generator(device="cuda").manual_seed(V)
    logits = torch.randn((8, V), generator=g, device="cuda", dtype=torch.float16).float()
    host = logits.cpu().numpy()
    for k, p in ((50, 1.0), (3000, 1.0), (0, 0.9), (500, 0.5)):
        ids, n24, kept, _ = _run(logits, 1.0, k, p, 9, 2)
        for b in range(8):
            w, margin = reference_row(host[b], 1.0, k, p)
            if margin > 1e-5:
                assert kept[b] == int((w > 0).sum()), (k, p, b)
                assert w[ids[b]] > 0


@pytest.mark.parametrize("shape", ["peaked", "flat"])
def test_distribution(shape):
    """200 000 draws under top-k 50 / top-p 0.9 against the reference probabilities (chi-square, fixed seeds)."""
    from scipy.stats import chisquare
    from kivi_b200 import glue
    V, B, launches = 32000, 500, 400
    row = _rows(1, V, 77, scale=4.0 if shape == "peaked" else 0.1)
    w, margin = reference_row(row[0].cpu().numpy(), 1.0, 50, 0.9)
    assert margin > 1e-5
    logits = row.repeat(B, 1).contiguous()
    t = torch.ones(B, device="cuda")
    k = torch.full((B,), 50, dtype=torch.int32, device="cuda")
    p = torch.full((B,), 0.9, device="cuda")
    seed = torch.arange(B, device="cuda") + 4242
    draw = torch.zeros(B, dtype=torch.long, device="cuda")
    out = torch.empty((launches, B), dtype=torch.long, device="cuda")
    for i in range(launches):
        glue.sample(logits, t, k, p, seed, draw, out[i])
    torch.cuda.synchronize()
    assert draw.tolist() == [launches] * B
    counts = np.bincount(out.flatten().cpu().numpy(), minlength=V).astype(np.float64)
    assert counts[w == 0].sum() == 0                                      # nothing outside the kept set
    n = launches * B
    exp = w / w.sum() * n
    big = exp >= 5                                                        # pool the cells too small for the chi-square law
    obs_cells, exp_cells = list(counts[big]), list(exp[big])
    if exp[~big & (w > 0)].sum() > 0:
        obs_cells.append(counts[~big].sum())
        exp_cells.append(exp[~big].sum())
    assert len(exp_cells) >= (3 if shape == "peaked" else 30)
    stat = chisquare(obs_cells, exp_cells)
    assert stat.pvalue > 1e-4, stat


@pytest.mark.parametrize("V", VOCABS)
def test_same_row_same_id_wherever_it_sits(V):
    """One row at different batch indices, in batches of different size, over repeated launches: the id is a function of
    (row, parameters, seed, draw) alone."""
    row = _rows(1, V, 5)[0]
    other = _rows(64, V, 6)
    want = {}
    for B in BATCHES:
        for at in sorted({0, B // 2, B - 1}):
            logits = other[:B].clone()
            logits[at] = row
            seeds = [50 + b for b in range(B)]
            seeds[at] = 999
            for k, p in MODES:
                for rep in range(2):
                    ids, n24, kept, _ = _run(logits, 0.9, k, p, seeds, 3)
                    got = (ids[at], n24[at], kept[at])
                    assert want.setdefault((k, p), got) == got, (B, at, k, p, rep)


def test_argument_errors_launch_nothing():
    from kivi_b200 import _lib, glue
    glue._bind()
    f = _lib.lib().kivi_sample_f32
    B, V = 4, 1000
    logits = _rows(B, V, 0)
    t, p = torch.ones(B, device="cuda"), torch.ones(B, device="cuda")
    k = torch.zeros(B, dtype=torch.int32, device="cuda")
    seed, draw, out = (torch.zeros(B, dtype=torch.long, device="cuda") for _ in range(3))
    ok = [logits.data_ptr(), B, V, t.data_ptr(), k.data_ptr(), p.data_ptr(), seed.data_ptr(), draw.data_ptr(),
          out.data_ptr(), None, None, None, None]
    n0 = _lib.launch_count()
    for i in (0, 3, 4, 5, 6, 7, 8):
        args = list(ok)
        args[i] = None
        assert f(*args) == KIVI_ERR_NULL, i
    for batch, vocab in ((-1, V), (B, 0), (B, -3)):
        args = list(ok)
        args[1], args[2] = batch, vocab
        assert f(*args) == KIVI_ERR_SHAPE
    assert _lib.launch_count() == n0
    with pytest.raises(ValueError):                                       # the wrapper's own checks
        glue.sample(logits, t[:3], k, p, seed, draw, out)
    with pytest.raises(ValueError):
        glue.sample(logits.half(), t, k, p, seed, draw, out)
    with pytest.raises(ValueError):
        glue.sample(logits, t, k.long(), p, seed, draw, out)
    with pytest.raises(RuntimeError):
        glue.sample(logits, t.cpu(), k, p, seed, draw, out)
    assert _lib.launch_count() == n0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------ model level
def _prompt(cfg, B, n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(1, cfg.vocab_size, (B, n), device="cuda", generator=g)


SAMPLED = dict(do_sample=True, temperature=1.3, top_k=40, top_p=0.95)


def test_generate_samples_reproducibly():
    model, cfg = tiny_model(1)
    ids = _prompt(cfg, 4, 37)
    a = model.generate(ids, max_new_tokens=24, seed=7, **SAMPLED)
    b = model.generate(ids, max_new_tokens=24, seed=7, **SAMPLED)
    c = model.generate(ids, max_new_tokens=24, seed=8, **SAMPLED)
    d = model.generate(ids, max_new_tokens=24, seed=7, use_graph=False, **SAMPLED)
    assert a.shape == (4, 37 + 24) and torch.equal(a[:, :37], ids)
    assert torch.equal(a, b) and torch.equal(a, d)
    assert not torch.equal(a, c)
    greedy = model.generate(ids, max_new_tokens=24)
    assert not torch.equal(a, greedy)
    cold = model.generate(ids, max_new_tokens=24, do_sample=True, temperature=0.0, seed=7)
    assert torch.equal(cold, greedy)                                      # temperature 0: the greedy ids exactly
    rows = model.generate(ids, max_new_tokens=24, do_sample=True, temperature=[0.0, 1.3, 0.0, 1.3], top_k=40, top_p=0.95,
                          seed=7)
    assert torch.equal(rows[0], greedy[0]) and torch.equal(rows[2], greedy[2])     # greedy and sampled rows share a batch
    assert torch.equal(rows[1], a[1]) and torch.equal(rows[3], a[3])


def test_in_graph_sampler_is_the_stand_alone_call():
    """The ids of a sampled generate() equal a replay that feeds the same tokens to a greedy-mode twin and calls glue.sample
    on the logits decode_step returned, with the same seeds and draw numbers."""
    from kivi_b200 import glue
    from kivi_b200.llama_kivi import sampling_rows
    model, cfg = tiny_model(2)
    twin, _ = tiny_model(2)
    B, n, new = 3, 29, 20
    ids = _prompt(cfg, B, n, seed=3)
    got = model.generate(ids, max_new_tokens=new, seed=11, **SAMPLED)
    t, k, p, sd = sampling_rows(B, 1.3, 40, 0.95, 11)
    dev = "cuda"
    T, K, P = (torch.tensor(t, device=dev), torch.tensor(k, dtype=torch.int32, device=dev), torch.tensor(p, device=dev))
    seed, draw = torch.tensor(sd, device=dev), torch.zeros(B, dtype=torch.long, device=dev)
    twin.init_cache(B, n + new)
    logits = twin.prefill(ids)
    tok = torch.empty(B, dtype=torch.long, device=dev)
    for step in range(new):
        glue.sample(logits.contiguous(), T, K, P, seed, draw, tok)
        assert torch.equal(tok, got[:, n + step]), step
        if step + 1 < new:
            logits = twin.decode_step(tok.view(B, 1)).clone()
    assert draw.tolist() == [new] * B


def test_mode_flip_keeps_launch_count_and_greedy_bits(graphs):
    """generate() sets the mode it needs and leaves it: the step is recaptured when do_sample changes and only then, the
    launch count is the same in both modes, and greedy decoding after sampling is bit for bit a fresh model's."""
    model, cfg = tiny_model(3)
    fresh, _ = tiny_model(3)
    ids = _prompt(cfg, 2, 33, seed=5)
    g0 = model.generate(ids, max_new_tokens=12)
    greedy_launches = model.launches_per_step
    assert graphs.made == 1 and not model._sampling
    model.generate(ids, max_new_tokens=12, seed=1, **SAMPLED)
    assert model.launches_per_step == greedy_launches
    assert graphs.made == 2 and model._sampling
    model.generate(ids, max_new_tokens=12, seed=2, **SAMPLED)              # other parameters, the same captured step
    assert graphs.made == 2
    g1 = model.generate(ids, max_new_tokens=12)
    assert graphs.made == 3 and not model._sampling
    assert torch.equal(g0, g1) and torch.equal(g1, fresh.generate(ids, max_new_tokens=12))
    model.generate(ids, max_new_tokens=12, seed=1, **SAMPLED)
    model.init_cache(2, 33 + 12)                                          # a new cache starts greedy
    fresh.init_cache(2, 33 + 12)
    a, b = model.prefill(ids), fresh.prefill(ids)
    assert torch.equal(a, b)
    same_logits(model, fresh, 11, a.argmax(-1).view(2, 1))
    with pytest.raises(RuntimeError):
        model.set_slot_sampling(0, temperature=1.0)                       # the step is greedy
    with pytest.raises(ValueError):
        model.set_sampling(temperature=-1.0)
    with pytest.raises(ValueError):
        model.set_sampling(top_p=[0.5, 0.5, 0.5])
    assert not model._sampling


def test_p2p_exchange_with_sampling_is_rejected():
    model, cfg = tiny_model(3)
    model.init_cache(2, 64)
    model._exchange = object()                                            # what enable_token_allgather(2, mode="p2p") sets
    with pytest.raises(NotImplementedError, match="greedy only"):
        model.set_sampling()
    model._exchange = None
    model.set_sampling()
    with pytest.raises(NotImplementedError, match="greedy only"):
        model.enable_token_allgather(2, mode="p2p")
    model.enable_token_allgather(2, mode="nccl", in_graph=False)          # gathers next_tokens, sampled or not
    assert model._sampling and model._dist_tokens is not None


BUDGETS = [57, 17, 52, 39, 58, 64, 75, 83]


def test_serve_mixes_greedy_and_sampled_requests():
    from kivi_b200.serve import serve
    model, cfg = tiny_model(2)
    par = lambda s: dict(temperature=1.2, top_k=30, top_p=0.9, seed=s)     # noqa: E731
    mixed = [None, par(1), None, par(2), par(3), None, par(4), None]
    all_greedy = dict(serve(model, requests(cfg, BUDGETS, params=[None] * 8), 3, 260))
    stats = {}
    a = dict(serve(model, requests(cfg, BUDGETS, params=mixed), 3, 260, stats=stats))
    assert model._sampling                                                # serve() leaves the mode its requests needed
    b = dict(serve(model, requests(cfg, BUDGETS, params=mixed), 3, 260))
    assert stats["inserts"] >= 1 and sorted(a) == list(range(8))
    for i in range(8):
        assert a[i].shape == (BUDGETS[i],) and torch.equal(a[i], b[i]), i
        if mixed[i] is None:
            assert torch.equal(a[i], all_greedy[i]), i                    # a greedy request next to sampled ones
    assert sum(not torch.equal(a[i], all_greedy[i]) for i in range(8) if mixed[i] is not None) >= 3
    others = [None if m is None else par(m["seed"] + 100) for m in mixed]
    others[3] = mixed[3]
    c = dict(serve(model, requests(cfg, BUDGETS, params=others), 3, 260))
    assert torch.equal(c[3], a[3])                                        # its own seed only
    assert sum(not torch.equal(c[i], a[i]) for i in (1, 4, 6)) >= 2
    # params {} is a sampled request with the defaults, not a greedy one
    empty, spelled = list(mixed), list(mixed)
    empty[1], spelled[1] = {}, dict(temperature=1.0, top_k=50, top_p=1.0, seed=0)
    d = dict(serve(model, requests(cfg, BUDGETS, params=empty), 3, 260))
    e = dict(serve(model, requests(cfg, BUDGETS, params=spelled), 3, 260))
    assert torch.equal(d[1], e[1]) and not torch.equal(d[1], all_greedy[1])
    again = dict(serve(model, requests(cfg, BUDGETS, params=[None] * 8), 3, 260))
    assert not model._sampling                                            # a list without params runs the greedy step
    for i in range(8):
        assert torch.equal(again[i], all_greedy[i]), i


def test_tensor_parallel_world_one_samples_like_the_model():
    cfg = small_cfg()
    plain, tpm = world_one_pair(cfg)
    ids = _prompt(cfg, 3, 40, seed=2)
    mask = torch.ones_like(ids)
    mask[1, :9] = 0
    a = plain.generate(ids, max_new_tokens=2 * cfg.residual_length + 5, attention_mask=mask, seed=5, **SAMPLED)
    b = tpm.generate(ids, max_new_tokens=2 * cfg.residual_length + 5, attention_mask=mask, seed=5, **SAMPLED)
    assert torch.equal(a, b)
    assert plain.launches_per_step == tpm.launches_per_step


def _tp_worker(rank, ws, out_dir):
    import torch.distributed as dist
    from kivi_b200.serve import serve
    cfg = small_cfg()
    model, _ = sharded_model(cfg, rank, ws)
    dev = torch.device("cuda", rank)
    prompt = torch.randint(0, cfg.vocab_size, (2, 48), generator=torch.Generator().manual_seed(2)).to(dev)
    out = model.generate(prompt, max_new_tokens=2 * cfg.residual_length + 5, seed=5, **SAMPLED)
    assert same_on_all_ranks(out)
    assert not torch.equal(out, model.generate(prompt, max_new_tokens=2 * cfg.residual_length + 5))
    gen = torch.Generator().manual_seed(3)
    reqs = [(torch.randint(0, cfg.vocab_size, (int(m),), generator=gen), int(k)) for m, k in
            ((30, 5), (45, 9), (12, 3), (40, 12), (25, 6))]
    reqs = [r + (dict(temperature=1.1, top_p=0.9, seed=i),) if i % 2 else r for i, r in enumerate(reqs)]
    got = dict(serve(model, reqs, 2, 200))
    for i in range(len(reqs)):
        assert same_on_all_ranks(got[i].to(dev)), i
    torch.cuda.synchronize()
    dist.barrier()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")
    dist.destroy_process_group()


def test_sharded_sampling_two_gpus(tmp_path):
    """Every rank of a sharded model samples the same ids with no collective: same logits bits, same seeds, same counters."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    spawn_ranks(_tp_worker, 2, tmp_path)

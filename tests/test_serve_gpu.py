"""Continuous batching on the fused cache: a slot refill is exactly a prefill of the right-aligned, pad-filled sequence, the
other slots do not change, decoding after it meets the oracle, a released slot sees only its new token, a timeline shift
drops positions bit for bit, the captured step survives both, and serve() at the model level."""
import numpy as np
import pytest
import torch

from oracle import ref
from tests._attn import assert_e2e, hidden_mask, left_padded, make_cache, rand16, tiny_model, tuple_equal
from tests._model import PROMPTS, TupleBar, graphs, packed_parts_equal, requests, same_logits, tuple_steps  # noqa: F401
from tests._util import to_np

pytestmark = pytest.mark.gpu

IDLE = 1 << 30

CASES = [  # kb, vb, g, R, H, Hkv  (G = 4 / 2 / 1 from H / Hkv): the geometries of the left-padded decode tests
    (2, 2, 32, 32, 4, 1),
    (2, 4, 64, 64, 2, 1),
    (4, 2, 128, 128, 2, 2),
    (4, 4, 32, 256, 8, 2),
    (2, 2, 128, 256, 2, 1),
    (4, 4, 64, 128, 3, 3),
    (2, 4, 32, 128, 4, 1),
    (4, 2, 64, 64, 8, 2),
    (4, 4, 128, 128, 4, 2),
]


def _h(rng, *shape, scale=1.0):
    return torch.from_numpy(rand16(rng, shape, scale)).cuda()


def _row(tup, b):
    """Sequence b's part of an exported 9-tuple (batch dim kept)."""
    return tuple(t[b:b + 1] if torch.is_tensor(t) else t for t in tup)


def _live(kb, vb, g, R, H, Hkv, seed, B=4, steps=None):
    """A B-sequence cache prefilled to r = R - 3 and stepped R + 2 times: the steps cross a K flush, the V ring wraps
    (vhead = 1) and the next step flushes again.  steps = R + 1: the ring has wrapped exactly once (vhead = 0)."""
    rng = np.random.default_rng(seed)
    n0 = max(3, -(-400 // R)) * R + R - 3
    cap = n0 + R + 64
    cache = make_cache(B, H, Hkv, kb, vb, g, R, cap)
    k, v = _h(rng, B, Hkv, n0, 128), _h(rng, B, Hkv, n0, 128)
    cache.prefill(0, k, v)
    steps = R + 2 if steps is None else steps
    for _ in range(steps):
        cache.decode_attention(0, _h(rng, B, H, 128, scale=0.7), _h(rng, B, Hkv, 128), _h(rng, B, Hkv, 128))
        cache.advance()
    assert cache.vhead == steps % (R + 1) and cache.tk > n0 - n0 % R
    return cache, rng, (k, v)


def _padded(src, s):
    """x[p] = src[max(p - s, 0)] along the token axis of [Hkv, n, 128]."""
    n = src.shape[1]
    idx = np.maximum(np.arange(n + s) - s, 0)
    return src[:, idx]


@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", CASES)
def test_refill_is_exact(kb, vb, g, R, H, Hkv):
    """Slot 2 of a live cache refilled with n tokens exports exactly what a B = 1 prefill of the pad-filled T-token
    sequence exports, and what the oracle's prefill split of it gives; slots 0, 1, 3 and `state` do not change."""
    cache, rng, _ = _live(kb, vb, g, R, H, Hkv, seed=kb * 100 + g + R)
    T = cache.kv_len
    before = [t.clone() if torch.is_tensor(t) else t for t in cache.export(0)]
    state = cache.read_state()
    for n in sorted({1, g - 1, R, R + 1, 133, T}):
        k, v = _h(rng, Hkv, n, 128), _h(rng, Hkv, n, 128)
        cache.refill(0, 2, k, v)
        got = cache.export(0)
        x_k, x_v = _padded(to_np(k), T - n)[None], _padded(to_np(v), T - n)[None]
        one = make_cache(1, H, Hkv, kb, vb, g, R, T + 8)
        one.prefill(0, torch.from_numpy(x_k).cuda(), torch.from_numpy(x_v).cuda())
        tuple_equal(_row(got, 2), one.export(0), f"n {n}: slot 2 vs a B = 1 prefill")
        tuple_equal(_row(got, 2), ref.prefill_cache(x_k, x_v, g, kb, vb, R), f"n {n}: slot 2 vs the oracle")
        for b in (0, 1, 3):
            tuple_equal(_row(got, b), _row(before, b), f"n {n}: slot {b}")
        assert cache.read_state() == state


@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", CASES)
def test_decode_after_refill(kb, vb, g, R, H, Hkv):
    """Six steps after refilling slot 2 (start s = T - n, across a K flush): slot 2 meets the oracle run with the
    finfo(fp16).min mask of s; a released slot returns its new token's V exactly; slots 0 and 3 are bit-identical to a twin
    cache that was not refilled."""
    seed = kb * 100 + g + R + 7
    cache, rng, _ = _live(kb, vb, g, R, H, Hkv, seed)
    twin, _, _ = _live(kb, vb, g, R, H, Hkv, seed)
    T = cache.kv_len
    n = R + 1
    s = T - n
    k, v = _h(rng, Hkv, n, 128), _h(rng, Hkv, n, 128)
    cache.refill(0, 2, k, v)
    for c in (cache, twin):
        c.set_kv_start(torch.tensor([0, 0, s, 0]))
        c.release(1)
    st = ref.prefill_cache(_padded(to_np(k), s)[None], _padded(to_np(v), s)[None], g, kb, vb, R)
    for step in range(6):
        q = _h(rng, 4, H, 128, scale=0.7)
        kn, vn = _h(rng, 4, Hkv, 128), _h(rng, 4, Hkv, 128)
        out = cache.decode_attention(0, q, kn, vn).clone()
        out_t = twin.decode_attention(0, q, kn, vn).clone()
        cache.advance()
        twin.advance()
        for b in (0, 3):
            assert torch.equal(out[b].view(torch.int16), out_t[b].view(torch.int16)), f"step {step}: slot {b}"
        idle = vn[1].repeat_interleave(H // Hkv, dim=0)
        assert torch.equal(out[1].view(torch.int16), idle.view(torch.int16)), f"step {step}: released slot"
        exp, _, st = ref.decode_step(st, to_np(q[2:3])[:, :, None], to_np(kn[2:3])[:, :, None], to_np(vn[2:3])[:, :, None],
                                     g, kb, vb, R, hidden_mask(1, st[8] + 1, [s]))
        assert_e2e(to_np(out[2:3])[:, :, None], exp, f"step {step}")
    assert cache.tk > T - T % R, "the steps crossed a K flush"
    tuple_equal(_row(cache.export(0), 2), st, "slot 2 after the steps")
    assert cache.read_state() == twin.read_state()


@pytest.mark.parametrize("blocks", ["one", "several"])
@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", [CASES[0], CASES[3], CASES[5], CASES[7]])
def test_shift(kb, vb, g, R, H, Hkv, blocks):
    """A shift by one quantum (max(128, R): one overlapping block for R <= 128) or by several drops exactly the first
    `shift` positions of the export, leaves the windows, lowers state and kv_start by `shift`; the next steps are
    bit-identical to a fresh cache imported from the shifted tuples with the same starts.  An import starts the V ring at
    slot 0 and the window part of p.V is summed in ring-slot items, so the cache is stepped until its ring head is back
    at slot 0 (vhead = 0 after a full wrap) for the bit-for-bit comparison."""
    cache, rng, _ = _live(kb, vb, g, R, H, Hkv, seed=kb * 10 + g + R + 3, steps=R + 1)
    q_ = max(128, R)
    shift = q_ if blocks == "one" else 2 * q_
    assert shift <= cache.tv
    T = cache.kv_len
    starts = [shift, shift + 1, min(shift + 200, T - 1), IDLE]
    cache.set_kv_start(torch.tensor(starts))
    before = [t.clone() if torch.is_tensor(t) else t for t in cache.export(0)]
    st0 = cache.read_state()
    with pytest.raises(ValueError):
        cache.shift(shift + q_ if shift + q_ <= cache.tv else 10 ** 6)   # would drop visible positions of slot 0
    cache.shift(shift)
    after = cache.export(0)
    kf, vf = 32 // kb, 32 // vb
    exp = (before[0][..., shift // kf:], before[1], before[2][..., shift // g:], before[3][..., shift // g:],
           before[4][:, :, shift:], before[5], before[6][:, :, shift:], before[7][:, :, shift:], before[8] - shift)
    tuple_equal(after, exp, "shifted export")
    assert cache.read_state()[:6] == [st0[0] - shift, st0[1], st0[2] - shift, st0[3], st0[4], st0[5] - shift]
    new_starts = [s - shift for s in starts]
    assert cache.kv_start.tolist() == new_starts and cache.kv_start_host == new_starts
    fresh = make_cache(4, H, Hkv, kb, vb, g, R, cache.max_tokens)
    fresh.import_tuple(0, after, kv_start=torch.tensor(new_starts))
    for step in range(6):
        q = _h(rng, 4, H, 128, scale=0.7)
        kn, vn = _h(rng, 4, Hkv, 128), _h(rng, 4, Hkv, 128)
        a = cache.decode_attention(0, q, kn, vn).clone()
        b = fresh.decode_attention(0, q, kn, vn).clone()
        cache.advance()
        fresh.advance()
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"step {step}"
    tuple_equal(cache.export(0), fresh.export(0), "after the steps")


# ------------------------------------------------------------------------------------------------------------ model level
GQA = dict(num_attention_heads=4, num_key_value_heads=1, hidden_size=512)


def test_graph_replays_after_refill_and_shift(graphs):
    """The step captured before an insert and a shift replays after them without a recapture, with logits bit-identical
    to the same model decoding without a graph."""
    model, cfg = tiny_model(5, **GQA)
    twin, _ = tiny_model(5, **GQA)
    twin.load_state_dict(model.state_dict())
    n = 300
    ids, mask = left_padded(cfg, [300, 170, 150], n, seed=1)
    for m in (model, twin):
        m.init_cache(3, 600)
        m.prefill(ids, attention_mask=mask)
    same_logits(model, twin, 3, graph_a=True, graph_b=False)
    assert graphs.made == 1
    prompt = torch.randint(1, cfg.vocab_size, (40,), device="cuda")
    for m in (model, twin):
        m.release(0)
        first = m.insert(0, prompt)
        m._ids[0] = first.argmax()
    assert model.cache.live_starts() == {0: model.cache.kv_len - 40, 1: 130, 2: 150}
    for m in (model, twin):
        m.cache.shift(128)
    assert model.cache.kv_len == n + 3 - 128
    same_logits(model, twin, 6, graph_a=True, graph_b=False)
    assert graphs.made == 1


BUDGETS = [157, 117, 152, 139, 158, 164, 175, 183]     # with PROMPTS, 3 slots and max_tokens = 360 need two shifts (R = 128)


@pytest.mark.parametrize("kw", [{}, GQA], ids=["tiny", "tiny-gqa"])
def test_serve(kw, graphs):
    """8 requests through 3 slots: each gets exactly its token budget (or stops at the chosen EOS, which it then ends
    with), the step graph is captured once, and max_tokens forces two shifts."""
    from kivi_b200.serve import serve
    model, cfg = tiny_model(2, **kw)
    reqs = requests(cfg, BUDGETS)
    stats = {}
    got = dict(serve(model, reqs, 3, 360, stats=stats))
    assert sorted(got) == list(range(len(reqs)))
    for i, (_, m) in enumerate(reqs):
        assert got[i].shape == (m,), i
    assert stats["shifts"] >= 2 and stats["inserts"] == 5 and stats["prefills"] == 1
    assert graphs.made == 1
    eos = int(torch.cat(list(got.values())).bincount().argmax())          # the most frequent token ends some requests
    got_e = dict(serve(model, reqs, 3, 360, eos_token_id=eos))
    assert sorted(got_e) == list(range(len(reqs)))
    stopped = 0
    for i, (_, m) in enumerate(reqs):
        t = got_e[i].tolist()
        assert 1 <= len(t) <= m and eos not in t[:-1], i
        assert len(t) == m or t[-1] == eos, i
        stopped += len(t) < m
    assert stopped > 0
    assert graphs.made == 1


def test_inserted_request_matches_tuple_path():
    """An inserted sequence continued two ways from the same cache contents: the fused batch (its slot) and the
    reference's tuple path on that slot's exported 9-tuples with its padding mask, fed the same tokens; the slot's packed
    cache parts equal the tuple path's after the steps."""
    model, cfg = tiny_model(3, **GQA)
    R = cfg.residual_length
    n = 2 * R + 100                                     # r = 105 after the prompt and 5 steps: the 40 steps flush K
    ids, mask = left_padded(cfg, [n, n - 50, 90], n, seed=4)
    model.init_cache(3, n + 80)
    model.prefill(ids, attention_mask=mask)
    for _ in range(5):
        model.decode_step()
    model.release(1)
    prompt = torch.randint(1, cfg.vocab_size, (70,), device="cuda")
    first = model.insert(1, prompt)
    T, p = model.cache.kv_len, prompt.numel()
    pasts = [_row(model.cache.export(i), 1) for i in range(cfg.num_hidden_layers)]
    pasts = [tuple(t.clone() if torch.is_tensor(t) else t for t in pk) for pk in pasts]
    pad = torch.zeros((1, T), dtype=torch.long, device="cuda")
    pad[:, T - p:] = 1
    model.fused_forward = False
    bar, steps = TupleBar("test_inserted_request_matches_tuple_path"), 40
    pasts = tuple_steps(model, pasts, first.argmax().view(1, 1), steps, bar, mask=pad, row=1)
    bar.done(steps)
    assert model.cache.tk > T - T % R, "the steps crossed a K flush"
    packed_parts_equal(_row(model.cache.export(0), 1), pasts[0], "slot 1, layer 0")


def test_inserted_prompt_does_not_reach_other_requests():
    """Replacing an inserted request's prompt (same length and budget) changes no token of any other request."""
    from kivi_b200.serve import serve
    model, cfg = tiny_model(4)
    reqs = requests(cfg, BUDGETS, seed=1)
    a = dict(serve(model, reqs, 3, 360))
    g = torch.Generator().manual_seed(99)
    swapped = list(reqs)
    swapped[5] = (torch.randint(1, cfg.vocab_size, (PROMPTS[5],), generator=g), BUDGETS[5])
    b = dict(serve(model, swapped, 3, 360))
    for i in range(len(reqs)):
        if i != 5:
            assert torch.equal(a[i], b[i]), i

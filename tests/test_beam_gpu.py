"""Beam search on the fused cache: the row reorder kernel against a torch gather of the raw buffers for every geometry and
map kind, decoding after a reorder, beam generate() against a torch-gather twin and the 9-tuple path, the prompt pass
run once for all beams or samples of a prompt, and the tensor-parallel model at world 1."""
import numpy as np
import pytest
import torch

from tests._attn import left_padded, make_cache, rand16, tiny_model
from tests._model import TupleBar, small_cfg, world_one_pair
from tests.test_serve_gpu import CASES

pytestmark = pytest.mark.gpu


def _h(rng, *shape, scale=1.0):
    return torch.from_numpy(rand16(rng, shape, scale)).cuda()


def torch_reorder(cache):
    """KiviCache._enqueue_reorder by torch: every buffer of every layer gathered by rows at full capacity, and kv_start."""
    src = cache.reorder_src.long()
    for bufs in cache._bufs:
        for buf in bufs:
            rows = buf.view(cache.batch, -1)
            rows.copy_(rows.index_select(0, src))
    if cache.ragged:
        cache.kv_start.copy_(cache.kv_start.index_select(0, src))


def maps(B, seed=0):
    """Identity, duplicates, a swap, a 3-cycle, a chain and a seeded random map with repeats, for B rows."""
    g = np.random.default_rng(seed)
    out = {"identity": list(range(B)), "duplicates": [0] * B,
           "swap": [1, 0] + list(range(2, B)), "chain": [0] + list(range(B - 1)),
           "random": [int(x) for x in g.integers(0, B, B)]}
    if B >= 3:
        out["3-cycle"] = [1, 2, 0] + list(range(3, B))
    return out


def _expected(cache, snap, src):
    """What the reorder must leave: live blocks and whole windows of rows with src[b] != b from the snapshot's row src[b],
    every other byte as it was."""
    B, Hkv = cache.batch, cache.num_kv_heads
    nkb, nvb = -(-cache.tk // 128), -(-cache.tv // 128)
    idx = torch.tensor(src, device=cache.device)
    exp = []
    for bufs in snap:
        ks = bufs[0].view(B, Hkv, cache.k_cap_blocks, -1).clone()
        vs = bufs[1].view(B, Hkv, cache.v_cap_blocks, -1).clone()
        ks[:, :, :nkb] = bufs[0].view(B, Hkv, cache.k_cap_blocks, -1)[idx, :, :nkb]
        vs[:, :, :nvb] = bufs[1].view(B, Hkv, cache.v_cap_blocks, -1)[idx, :, :nvb]
        exp.append([ks.view(-1), vs.view(-1), bufs[2].view(B, -1)[idx].view(-1), bufs[3].view(B, -1)[idx].view(-1)])
    return exp


def _check_reorder(cache, src, what):
    snap = [[b.clone() for b in bufs] for bufs in cache._bufs]
    state = cache.state.clone()
    starts = cache.kv_start.clone()
    cache.reorder(src)
    for layer, (got, exp) in enumerate(zip(cache._bufs, _expected(cache, snap, src))):
        for i, name in enumerate(("K store", "V store", "K window", "V ring")):
            assert torch.equal(got[i], exp[i]), f"{what}: layer {layer} {name}"
    assert torch.equal(cache.state, state), f"{what}: state"
    if cache.ragged:
        assert cache.kv_start.tolist() == [starts.tolist()[s] for s in src] == cache.kv_start_host, what
    cache.read_state()


def _states(kb, vb, g, R, H, Hkv, B, seed, window=None):
    """(name, cache) at the lengths the contract names: tk = 0, tv = 0 with tk > 0, tk % 128 != 0 and a wrapped V ring,
    after a shift; two layers, random contents.  window: a windowed cache."""
    rng = np.random.default_rng(seed)
    n_long = max(3, -(-400 // R)) * R + R - 3
    for name, n, steps in (("tk = 0", R - 3, 0), ("tv = 0", R, 0), ("wrapped ring", n_long, R + 2)):
        cache = make_cache(B, H, Hkv, kb, vb, g, R, n_long + 5 * R + 64, n_layers=2, sliding_window=window)
        for layer in range(2):
            cache.prefill(layer, _h(rng, B, Hkv, n, 128), _h(rng, B, Hkv, n, 128))
        for _ in range(steps):
            for layer in range(2):
                cache.decode_attention(layer, _h(rng, B, H, 128, scale=0.7), _h(rng, B, Hkv, 128), _h(rng, B, Hkv, 128))
            cache.advance()
        yield name, cache
    cache.set_kv_start(torch.full((B,), max(128, R)))               # no sequence sees the dropped positions
    cache.shift(max(128, R))
    yield "after a shift", cache


def _state(name, *geometry, **kw):
    return next(c for n, c in _states(*geometry, **kw) if n == name)


@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", CASES)
def test_reorder_is_a_row_gather(kb, vb, g, R, H, Hkv):
    for name, cache in _states(kb, vb, g, R, H, Hkv, B=5, seed=kb + vb + g + R):
        cache.set_kv_start(torch.tensor([0, 1, 2, 3, 4]) if name != "tk = 0" else None)
        for kind, src in maps(5, seed=R).items():
            _check_reorder(cache, src, f"{name}, {kind}")


def test_reorder_64_rows_and_a_window():
    kb, vb, g, R, H, Hkv = CASES[3]
    for name, cache in _states(kb, vb, g, R, H, Hkv, B=64, seed=1, window=200):
        for seed in range(3):
            _check_reorder(cache, maps(64, seed)["random"], f"{name}, random {seed}")


def test_out_of_range_row_writes_nothing():
    kb, vb, g, R, H, Hkv = CASES[0]
    cache = _state("wrapped ring", kb, vb, g, R, H, Hkv, B=4, seed=2)
    with pytest.raises(ValueError):
        cache.reorder([0, 1, 2, 4])
    snap = [[b.clone() for b in bufs] for bufs in cache._bufs]
    for bad in ([1, 0, 3, 4], [1, 0, -1, 2]):
        cache.reorder_src.copy_(torch.tensor(bad, dtype=torch.int32))       # past the host check: the device refuses
        cache._enqueue_reorder()
        for got, exp in zip(cache._bufs, snap):
            assert all(torch.equal(a, b) for a, b in zip(got, exp)), bad
        with pytest.raises(RuntimeError, match="row reorder"):
            cache.read_state()


def test_captured_reorder_follows_the_map_buffer():
    kb, vb, g, R, H, Hkv = CASES[2]
    cache, twin = [_state("wrapped ring", kb, vb, g, R, H, Hkv, B=6, seed=3) for _ in range(2)]
    cache.reorder_scratch()
    cache._enqueue_reorder()                                          # identity: loads the kernels, writes nothing
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cache._enqueue_reorder()
    for kind, src in maps(6, seed=5).items():
        cache.reorder_src.copy_(torch.tensor(src, dtype=torch.int32))
        graph.replay()
        twin.reorder(src)
        for a, b in zip(cache._bufs, twin._bufs):
            assert all(torch.equal(x, y) for x, y in zip(a, b)), kind
    cache.read_state()


@pytest.mark.parametrize("mode", ["unpadded", "ragged", "windowed"])
def test_decode_after_reorder(mode):
    """A cache reordered by the kernel and its twin reordered by the torch gather decode R + 2 steps (across a K flush and
    a ring wrap) with bit-equal outputs: stale bytes past the live blocks are never read."""
    kb, vb, g, R, H, Hkv = CASES[1]
    window = 150 if mode == "windowed" else None
    a, b = [_state("wrapped ring", kb, vb, g, R, H, Hkv, B=4, seed=4, window=window) for _ in range(2)]
    for c in (a, b):
        c.set_kv_start(torch.tensor([3, 0, 70, 9]) if mode == "ragged" else None)
    rng = np.random.default_rng(9)
    for src in ([2, 2, 0, 1], [3, 0, 0, 2], [1, 1, 1, 1]):
        a.reorder(src)
        b.reorder_src.copy_(torch.tensor(src, dtype=torch.int32))
        torch_reorder(b)
        b._mirror_reorder(src)
        for step in range(R + 2):
            q, kn, vn = _h(rng, 4, H, 128, scale=0.7), _h(rng, 4, Hkv, 128), _h(rng, 4, Hkv, 128)
            for layer in range(2):
                oa = a.decode_attention(layer, q, kn, vn).clone()
                ob = b.decode_attention(layer, q, kn, vn)
                assert torch.equal(oa.view(torch.int16), ob.view(torch.int16)), f"{src} step {step} layer {layer}"
            a.advance()
            b.advance()
    assert a.read_state() == b.read_state()


# ------------------------------------------------------------------------------------------------------------ model level
def _pair(seed=5, **kw):
    m, cfg = tiny_model(seed, **kw)
    twin, _ = tiny_model(seed, **kw)
    twin.load_state_dict(m.state_dict())
    return m, twin, cfg


@pytest.mark.parametrize("mode", ["unpadded", "padded", "windowed"])
def test_beam_generate_kernel_vs_torch_gather(mode, monkeypatch):
    from kivi_b200.cache import KiviCache
    kw = dict(sliding_window=96, residual_length=32) if mode == "windowed" else {}
    model, twin, cfg = _pair(**kw)
    new = 300 if mode == "windowed" else 40
    if mode == "padded":
        ids, mask = left_padded(cfg, [150, 97], 150, seed=2)
    else:
        ids, mask = torch.randint(1, cfg.vocab_size, (2, 150), device="cuda"), None
    args = dict(max_new_tokens=new, num_beams=4, num_return_sequences=2, return_dict_in_generate=True,
                attention_mask=mask, eos_token_id=-1)
    got = model.generate(ids, **args)
    assert model.launches_per_reorder == 2 * cfg.num_hidden_layers
    if mode == "windowed":
        assert model.cache.max_tokens < 150 + new, "the windowed cache rolled"
    monkeypatch.setattr(KiviCache, "_enqueue_reorder", torch_reorder)
    exp = twin.generate(ids, **args)
    assert got.sequences.shape == (4, 150 + new)
    assert torch.equal(got.sequences, exp.sequences) and torch.equal(got.sequences_scores, exp.sequences_scores)


def test_beams_teacher_forced_against_tuple_path():
    """forward() + _reorder_cache on the fused views, fed the beams chosen on the 9-tuple path's logits: per-step logits
    within TupleBar; a twin whose views are reordered by the torch gather stays bit-equal."""
    from kivi_b200.beam import BeamSearch
    model, twin, cfg = _pair(7)
    K, n, steps = 4, 140, cfg.residual_length + 4
    ids = torch.randint(1, cfg.vocab_size, (2, n), device="cuda").repeat_interleave(K, 0)
    bar = TupleBar("test_beams_teacher_forced_against_tuple_path")
    model.fused_forward = False
    lt, pt = model(ids)
    model.fused_forward = True
    lf, pf = model(ids)
    lw, pw = twin(ids)
    bar.prompt(lf[:, -1], lt[:, -1])
    search = BeamSearch(ids[::K], K, n + steps + 1)
    logits = lt[:, -1]
    for s in range(steps):
        beam_idx, tok, _ = search.step(logits)
        pt = model._reorder_cache(pt, beam_idx)
        pf = model._reorder_cache(pf, beam_idx)
        twin.cache.reorder_src.copy_(beam_idx)
        torch_reorder(twin.cache)
        pw = [type(p)(twin.cache, p.layer, twin.cache.kv_len) for p in pw]
        tok = tok.view(-1, 1)
        model.fused_forward = False
        lt, pt = model(tok, pt)
        model.fused_forward = True
        lf, pf = model(tok, pf)
        lw, pw = twin(tok, pw)
        bar.step(lf[:, -1], lt[:, -1], f"step {s}")
        assert torch.equal(lf, lw), f"step {s}: kernel vs torch-gather reorder"
        logits = lt[:, -1]
    bar.done(steps)


def test_prompt_once_fills_every_beam_row():
    model, one, cfg = _pair(8)
    K = 3
    ids, mask = left_padded(cfg, [130, 61], 130, seed=4)
    model.init_cache(2 * K, 200)
    one.init_cache(2, 200)
    model._prompt_pass(ids, mask, copies=K)
    one.prefill(ids, attention_mask=mask)
    for got, exp in zip(model.cache._bufs, one.cache._bufs):
        for a, b in zip(got, exp):
            assert torch.equal(a.view(2 * K, -1), b.view(2, -1).repeat_interleave(K, 0))
    assert torch.equal(model.cache.state, one.cache.state)
    assert model.cache.kv_start.tolist() == one.cache.kv_start.repeat_interleave(K).tolist()
    assert torch.equal(model._pos, one._pos.repeat_interleave(K, 0))


def test_sampled_sequences_per_prompt():
    from kivi_b200 import glue
    model, twin, cfg = _pair(9)
    one, _ = tiny_model(9)
    one.load_state_dict(model.state_dict())
    nrs, new, seed = 3, 12, 77
    ids = torch.randint(1, cfg.vocab_size, (2, 90), device="cuda")
    samp = dict(temperature=0.9, top_k=40, top_p=0.95)
    out = model.generate(ids, max_new_tokens=new, do_sample=True, num_return_sequences=nrs, seed=seed, **samp)
    assert out.shape == (2 * nrs, 90 + new) and torch.equal(out[:, :90], ids.repeat_interleave(nrs, 0))
    one.init_cache(2, 90 + new)
    lg = one.prefill(ids).repeat_interleave(nrs, 0).contiguous()
    rows = 2 * nrs
    first = torch.empty(rows, dtype=torch.long, device="cuda")
    glue.sample(lg, torch.full((rows,), samp["temperature"], device="cuda"),
                torch.full((rows,), samp["top_k"], dtype=torch.int32, device="cuda"),
                torch.full((rows,), samp["top_p"], device="cuda"), torch.arange(seed, seed + rows, device="cuda"),
                torch.zeros(rows, dtype=torch.long, device="cuda"), first)
    assert torch.equal(out[:, 90], first)
    twin.init_cache(rows, 90 + new)
    twin.set_sampling(seed=seed, **samp)
    twin.prefill(ids.repeat_interleave(nrs, 0))
    twin._samp.draw.fill_(1)                                        # the first draw went to the first token
    tok = first.view(-1, 1)
    for s in range(new - 1):
        twin.decode_step(tok)
        tok = twin.next_tokens.view(-1, 1).clone()
        assert torch.equal(out[:, 91 + s], tok[:, 0]), f"step {s}"


def test_tensor_parallel_world_one_beams():
    plain, tpm = world_one_pair(small_cfg())
    ids = torch.randint(1, 4096, (2, 70), device="cuda")
    args = dict(max_new_tokens=24, num_beams=4, num_return_sequences=2, return_dict_in_generate=True)
    a, b = plain.generate(ids, **args), tpm.generate(ids, **args)
    assert torch.equal(a.sequences, b.sequences) and torch.equal(a.sequences_scores, b.sequences_scores)

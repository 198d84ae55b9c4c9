"""Left-padded batches on the fused cache path (kivi_decode_attention_ragged_f16): per-sequence start offsets against the
additive-mask path they replace (bit for bit), padded blocks not read, the clamp, the captured step, and the model."""
import numpy as np
import pytest
import torch

from tests._attn import hidden_mask, left_padded, make_cache, tiny_model, tuple_equal
from tests._model import TupleBar, packed_parts_equal, same_logits, tuple_prompt, tuple_steps

pytestmark = pytest.mark.gpu


RAGGED_CASES = [  # kb, vb, g, R, H, Hkv  (G = 4 / 2 / 1 from H / Hkv)
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


@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", RAGGED_CASES)
def test_ragged_matches_mask_path(kb, vb, g, R, H, Hkv):
    """Two identically prefilled caches: per-sequence starts on one, the equivalent additive finfo.min mask on the other.
    out and dbg_probs bit-identical, dbg_logits equal at the visible positions, the 9-tuples bit-identical after every
    step, over steps that cross a K flush and a V-ring wrap."""
    dev = torch.device("cuda")
    rng = np.random.default_rng(kb * 1000 + g * 10 + R + H)
    n0 = max(3, -(-400 // R)) * R + R - 3                            # r = R - 3: the K window flushes at step 3
    steps = 6
    B = 10
    ragged, masked = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 64), make_cache(B, H, Hkv, kb, vb, g, R, n0 + 64)
    k = torch.from_numpy(rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)).to(dev)
    v = torch.from_numpy(rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)).to(dev)
    ragged.prefill(0, k, v)
    masked.prefill(0, k, v)
    tk, r, tv, L, kv = ragged.tk, ragged.r, ragged.tv, ragged.L, ragged.kv_len
    starts = [0, 1, 17, 127, 128, 129, tk, tk + r // 2, tv + L // 2, kv + 5]
    assert len(starts) == B
    ragged.set_kv_start(torch.tensor(starts))
    assert ragged.ragged and not masked.ragged
    Tmax = n0 + 64
    for step in range(steps):
        T = ragged.kv_len + 1
        q = torch.from_numpy((rng.standard_normal((B, H, 128)) * 0.7).astype(np.float16)).to(dev)
        kn = torch.from_numpy(rng.standard_normal((B, Hkv, 128)).astype(np.float16)).to(dev)
        vn = torch.from_numpy(rng.standard_normal((B, Hkv, 128)).astype(np.float16)).to(dev)
        dl_r, dp_r = (torch.zeros((B, H, Tmax), dtype=torch.float16, device=dev) for _ in range(2))
        dl_m, dp_m = (torch.zeros((B, H, Tmax), dtype=torch.float16, device=dev) for _ in range(2))
        # production epilogues first (no debug pointers: unpadded blocks take the fast epilogue), then instrumented
        out_fast = ragged.decode_attention(0, q, kn, vn).clone()
        out_r = ragged.decode_attention(0, q, kn, vn, dbg_logits=dl_r, dbg_probs=dp_r)
        mask = torch.from_numpy(hidden_mask(B, T, starts)).to(dev)
        out_m = masked.decode_attention(0, q, kn, vn, mask=mask, dbg_logits=dl_m, dbg_probs=dp_m)
        torch.cuda.synchronize()
        assert torch.equal(out_fast.view(torch.int16), out_r.view(torch.int16)), f"step {step}: fast / instrumented"
        assert torch.equal(out_r.view(torch.int16), out_m.view(torch.int16)), f"step {step}: out"
        assert torch.equal(dp_r.view(torch.int16), dp_m.view(torch.int16)), f"step {step}: dbg_probs"
        for b, s in enumerate(starts):
            s = min(max(s, 0), T - 1)
            assert torch.equal(dl_r[b, :, s:T].view(torch.int16), dl_m[b, :, s:T].view(torch.int16)), f"step {step}: logits {b}"
        ragged.advance()
        masked.advance()
        tuple_equal(ragged.export(0), masked.export(0), f"step {step}")
    assert ragged.read_state() == masked.read_state()


def test_padded_blocks_are_not_read():
    """NaN scales in the wholly padded 128-token blocks only: the ragged output is the clean cache's, bit for bit; the same
    poisoned cache through the mask path gives NaN (the poison landed)."""
    dev = torch.device("cuda")
    rng = np.random.default_rng(7)
    B, H, Hkv, kb, vb, g, R, n0 = 4, 4, 2, 2, 2, 32, 128, 700
    starts = [0, 300, 129, 512]
    clean = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8)
    k = torch.from_numpy(rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)).to(dev)
    v = torch.from_numpy(rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)).to(dev)
    clean.prefill(0, k, v, kv_start=torch.tensor(starts))
    tup = [t.clone() if torch.is_tensor(t) else t for t in clean.export(0)]
    poisoned_blocks = 0
    for b, s in enumerate(starts):
        nb = s // 128                                                # blocks wholly below the start
        poisoned_blocks += nb
        tup[2][b, :, :, :nb * 128 // g] = float("nan")               # K scales [B, Hkv, 128, tk / g]
        tup[6][b, :, :nb * 128, :] = float("nan")                    # V scales [B, Hkv, tv, 128 / g]
    assert poisoned_blocks > 0
    bad = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8)
    bad.import_tuple(0, tuple(tup), kv_start=torch.tensor(starts))
    q = torch.from_numpy((rng.standard_normal((B, H, 128)) * 0.7).astype(np.float16)).to(dev)
    kn = torch.from_numpy(rng.standard_normal((B, Hkv, 128)).astype(np.float16)).to(dev)
    vn = torch.from_numpy(rng.standard_normal((B, Hkv, 128)).astype(np.float16)).to(dev)
    out_clean = clean.decode_attention(0, q, kn, vn).clone()
    out_bad = bad.decode_attention(0, q, kn, vn).clone()
    torch.cuda.synchronize()
    assert not torch.isnan(out_clean).any()
    assert torch.equal(out_clean.view(torch.int16), out_bad.view(torch.int16))
    bad.set_kv_start(None)                                           # the same cache through the additive-mask path
    out_mask = bad.decode_attention(0, q, kn, vn, mask=torch.from_numpy(hidden_mask(B, bad.kv_len + 1, starts)).to(dev))
    torch.cuda.synchronize()
    for b in range(1, B):                                            # every sequence with a wholly padded block
        assert torch.isnan(out_mask[b]).any(), f"poison did not reach the mask path (sequence {b})"


@pytest.mark.parametrize("kb,vb,g,R,H,Hkv", [(2, 2, 32, 128, 4, 2), (4, 4, 64, 64, 8, 2), (4, 2, 32, 32, 3, 1)])
def test_start_at_or_beyond_kv_len_sees_only_the_new_token(kb, vb, g, R, H, Hkv):
    dev = torch.device("cuda")
    rng = np.random.default_rng(11)
    B, n0 = 3, 333
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + 8)
    k = torch.from_numpy(rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)).to(dev)
    v = torch.from_numpy(rng.standard_normal((B, Hkv, n0, 128)).astype(np.float16)).to(dev)
    cache.prefill(0, k, v, kv_start=torch.tensor([n0, n0 + 1, 1 << 30]))
    for _ in range(3):
        q = torch.from_numpy(rng.standard_normal((B, H, 128)).astype(np.float16)).to(dev)
        kn = torch.from_numpy(rng.standard_normal((B, Hkv, 128)).astype(np.float16)).to(dev)
        vn = torch.from_numpy(rng.standard_normal((B, Hkv, 128)).astype(np.float16)).to(dev)
        out = cache.decode_attention(0, q, kn, vn)
        exp = vn.repeat_interleave(H // Hkv, dim=1)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), exp.view(torch.int16))
        cache.advance()
        cache.set_kv_start(torch.full((B,), cache.kv_len, dtype=torch.int32))


def test_padded_decode_step_graph_matches_eager():
    model, cfg = tiny_model(5, num_attention_heads=4, num_key_value_heads=2, hidden_size=512)
    twin, _ = tiny_model(5, num_attention_heads=4, num_key_value_heads=2, hidden_size=512)
    twin.load_state_dict(model.state_dict())
    n = 200
    ids, mask = left_padded(cfg, [200, 130, 40], n, seed=1, low=0)
    for m in (model, twin):
        m.init_cache(3, n + 16)
    lg = model.prefill(ids, attention_mask=mask)
    lt = twin.prefill(ids, attention_mask=mask)
    assert torch.equal(lg, lt) and model.cache.ragged
    same_logits(model, twin, 10, lg.argmax(-1, keepdim=True), graph_a=True, graph_b=False)


@pytest.mark.parametrize("name,kw", [("tiny", {}), ("tiny", dict(num_attention_heads=4, num_key_value_heads=1, hidden_size=512,
                                                                k_bits=4, v_bits=4, group_size=64, residual_length=64))])
def test_padded_model_matches_tuple_model(name, kw, request):
    """B = 3 left-padded prompts (one shorter than R: its padding reaches the fp16 windows), 40 steps across a K flush:
    the fused padded decode against the tuple path with the 2-D padding mask, both fed the same tokens."""
    model, cfg = tiny_model(0, **kw)
    R = cfg.residual_length
    n, steps = 2 * R + R - 28 if R < 128 else R + 100, 40
    lengths = [n, n - 60, R // 2 - 5]
    ids, mask = left_padded(cfg, lengths, n, seed=3, low=0)
    bar = TupleBar(request.node.name)
    model.init_cache(len(lengths), n + steps + 4)
    pasts = tuple_steps(model, *tuple_prompt(model, ids, bar, mask), steps, bar, mask=mask)
    bar.done(steps)
    assert model.cache.tk > n - n % R, "the steps crossed a K flush"
    packed_parts_equal(model.cache.export(0), pasts[0], "layer 0")


def test_generate_with_masks():
    model, cfg = tiny_model(1)
    ids = torch.randint(0, cfg.vocab_size, (3, 140), device="cuda")
    plain = model.generate(ids, max_new_tokens=12)
    ones = model.generate(ids, max_new_tokens=12, attention_mask=torch.ones_like(ids))
    assert torch.equal(plain, ones)
    assert not model.cache.ragged
    pids, mask = left_padded(cfg, [140, 90, 20], 140, seed=2, low=0)
    out = model.generate(pids, max_new_tokens=12, attention_mask=mask)
    assert out.shape == (3, 152) and torch.equal(out[:, :140], pids) and model.cache.ragged
    again = model.generate(ids, max_new_tokens=12)                  # the unpadded step graph again
    assert torch.equal(again, plain)
    right = torch.ones_like(ids)
    right[1, -7:] = 0
    with pytest.raises(ValueError, match="left padding"):
        model.generate(ids, max_new_tokens=4, attention_mask=right)

"""Beam search without a GPU: kivi_b200.beam driven by a tiny fp32 transformers LlamaForCausalLM (the whole sequence
recomputed every step) returns the sequences and scores of that model's own generate(num_beams=K); the generate()
refusals of the fused model; and the C entry points of the row reorder, exported and rejecting bad arguments before any
launch."""
import ctypes
import itertools
import os
import re

import pytest
import torch

from kivi_b200.beam import BeamSearch

KIVI_ERR_SHAPE, KIVI_ERR_NULL = -2, -6
FAKE = 1 << 20                                       # never dereferenced: validation returns before any launch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOCAB, NEW = 48, 7


@pytest.fixture(scope="module")
def hf():
    transformers = pytest.importorskip("transformers")
    cfg = transformers.LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=2, vocab_size=VOCAB, max_position_embeddings=64,
                                   initializer_range=0.3, bos_token_id=None, eos_token_id=None, pad_token_id=None)
    torch.manual_seed(0)
    model = transformers.LlamaForCausalLM(cfg).float().eval()
    return model


def _positions(mask):
    return (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 0)


def _prompts(padded):
    g = torch.Generator().manual_seed(3)
    if not padded:
        ids = torch.randint(1, VOCAB, (1, 5), generator=g)
        return ids, torch.ones_like(ids)
    ids = torch.randint(1, VOCAB, (2, 6), generator=g)
    mask = torch.ones_like(ids)
    mask[1, :2] = 0
    ids[1, :2] = 0
    return ids, mask


@torch.no_grad()
def _ours(model, ids, mask, K, eos, **kw):
    """kivi_b200.beam over full recomputes of the running sequences; checks that each step's (beam_idx, tokens) describe
    the new running sequences: row r = the previous row beam_idx[r] + tokens[r]."""
    B, n = ids.shape
    bs = BeamSearch(ids, K, n + NEW, eos_token_id=eos, **kw)
    logits = model(ids, attention_mask=mask, position_ids=_positions(mask)).logits[:, -1].float()     # the prompts once
    rows = mask.repeat_interleave(K, 0)
    steps, early = 0, False
    while True:
        prev = bs.running[:, :, :bs.cur_len].reshape(B * K, -1).clone()
        beam_idx, tok, done = bs.step(logits)
        steps += 1
        cur = bs.running[:, :, :bs.cur_len].reshape(B * K, -1)
        assert torch.equal(cur[:, :-1], prev[beam_idx]) and torch.equal(cur[:, -1], tok)
        if bool(done):
            break
        early |= bool(bs.finished.any())                # before the last step only EOS finishes a hypothesis
        rows = torch.cat([rows, rows.new_ones((B * K, 1))], 1)
        logits = model(cur, attention_mask=rows, position_ids=_positions(rows)).logits[:, -1].float()
    assert steps <= NEW
    return bs.finalize() + (early,)


def _early_eos(model, ids, mask, K, **kw):
    """An EOS id with which a hypothesis finishes before max_length (joins the finished set at a step that does not reach
    it): the first such token among those the beams generate without an EOS.  Returns (eos, our sequences and scores)."""
    n = ids.shape[1]
    plain = model.generate(ids, attention_mask=mask, num_beams=K, max_new_tokens=NEW, do_sample=False)
    for eos in dict.fromkeys(plain[:, n:].reshape(-1).tolist()):
        seq, scores, early = _ours(model, ids, mask, K, eos, **kw)
        if early:
            return eos, seq, scores
    raise AssertionError("no generated token finishes a hypothesis early as the EOS id")


CASES = list(itertools.product([2, 4], ["one", "all"], [0.5, 1.0, 2.0], [True, False, "never"]))


@pytest.mark.parametrize("K,nrs,lp,es", CASES)
def test_matches_transformers_beam_search(hf, K, nrs, lp, es):
    _check(hf, K, K if nrs == "all" else 1, lp, es, padded=False)


@pytest.mark.parametrize("K,nrs", [(2, 2), (4, 1), (4, 4)])
def test_matches_transformers_on_a_left_padded_batch(hf, K, nrs):
    _check(hf, K, nrs, 1.0, False, padded=True)


def _check(model, K, nrs, lp, es, padded):
    ids, mask = _prompts(padded)
    kw = dict(num_return_sequences=nrs, length_penalty=lp, early_stopping=es)
    eos, seq, scores = _early_eos(model, ids, mask, K, **kw)
    ref = model.generate(ids, attention_mask=mask, num_beams=K, max_new_tokens=NEW, do_sample=False, eos_token_id=eos,
                         pad_token_id=eos, return_dict_in_generate=True, output_scores=True, **kw)
    assert torch.equal(seq, ref.sequences), (seq, ref.sequences)
    assert torch.allclose(scores, ref.sequences_scores, rtol=0, atol=1e-5), (scores, ref.sequences_scores)


def test_argument_errors():
    ids = torch.zeros((1, 3), dtype=torch.long)
    with pytest.raises(ValueError):
        BeamSearch(ids, 2, 8, num_return_sequences=3)
    with pytest.raises(ValueError):
        BeamSearch(ids, 2, 8, early_stopping="sometimes")
    with pytest.raises(ValueError):
        BeamSearch(ids, 2, 3)


# ------------------------------------------------------------------------------------------------ generate() refusals
def _model():
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    torch.manual_seed(0)
    return LlamaForCausalLM_KIVI(default_config("tiny")).half()


@pytest.mark.parametrize("kw,err", [
    (dict(num_beams=2, do_sample=True), NotImplementedError),                       # beam sampling
    (dict(num_beams=2, num_return_sequences=3), ValueError),                        # more sequences than beams
    (dict(num_return_sequences=2), ValueError),                                     # greedy decoding returns one
    (dict(num_beams=2, early_stopping="sometimes"), ValueError),
])
def test_generate_refusals(kw, err):
    m = _model()
    with pytest.raises(err):
        m.generate(torch.zeros(2, 3, dtype=torch.long), max_new_tokens=2, **kw)
    assert m.cache is None, "refused before any work"


def test_beams_refuse_token_allgather_replicas():
    m = _model()
    m._dist_tokens = torch.zeros(4, dtype=torch.long)                 # what enable_token_allgather(2) leaves
    with pytest.raises(NotImplementedError):
        m.generate(torch.zeros(2, 3, dtype=torch.long), max_new_tokens=2, num_beams=2)
    assert m.cache is None


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    from kivi_b200 import _lib, build
    build.build()
    from kivi_b200.cache import _bind
    _bind()
    return _lib.lib()


def _struct(**kw):
    from kivi_b200.cache import _CacheStruct
    f = dict(batch=4, num_heads=4, num_kv_heads=2, head_dim=128, k_bits=2, v_bits=2, group_size=32, residual_length=128,
             k_cap_blocks=4, v_cap_blocks=4, v_res_cap=129, flags=0)
    f.update(kw)
    return _CacheStruct(*[f[n] for n, _ in _CacheStruct._fields_[:12]], FAKE, FAKE, FAKE, FAKE, FAKE)


def test_reorder_entries_are_declared_and_bound():
    txt = open(os.path.join(ROOT, "include", "kivi_b200.h")).read()
    assert re.search(r"int64_t kivi_cache_reorder_scratch_bytes\(const kivi_cache_t\* cache\);", txt)
    assert re.search(r"int kivi_cache_reorder_f16\(const kivi_cache_t\* cache, const int32_t\* src, void\* scratch, "
                     r"int64_t scratch_bytes, void\* stream\);", txt)
    assert int(re.search(r"#define KIVI_STATE_ERR_ROWS\s+(\d+)", txt).group(1)) == 4
    import inspect
    from kivi_b200 import cache
    src = inspect.getsource(cache._bind)
    assert '"kivi_cache_reorder_scratch_bytes", i64, [P]' in src and '"kivi_cache_reorder_f16", i32, [P, vp, vp, i64, vp]' in src
    assert "st[6] & 4" in inspect.getsource(cache.KiviCache.read_state)


def test_reorder_scratch_is_one_layer_at_full_capacity(lib):
    st = _struct(k_bits=4, group_size=64)
    sizes = (ctypes.c_int64 * 8)()
    # 4 sequences of up to 384 tokens: 4 blocks of capacity
    assert lib.kivi_cache_sizes(4, 2, 4, 2, 64, 128, 384, sizes) == 0 and sizes[0] == 4 and sizes[2] == 129
    assert lib.kivi_cache_reorder_scratch_bytes(ctypes.byref(st)) == sum(sizes[3:7])
    assert lib.kivi_cache_reorder_scratch_bytes(None) == KIVI_ERR_NULL
    assert lib.kivi_cache_reorder_scratch_bytes(ctypes.byref(_struct(k_bits=3))) == -1


def test_reorder_validates_arguments(lib):
    st = _struct()
    need = lib.kivi_cache_reorder_scratch_bytes(ctypes.byref(st))
    assert need > 0
    call = lib.kivi_cache_reorder_f16
    assert call(None, FAKE, FAKE, need, None) == KIVI_ERR_NULL
    assert call(ctypes.byref(st), None, FAKE, need, None) == KIVI_ERR_NULL
    assert call(ctypes.byref(st), FAKE, None, need, None) == KIVI_ERR_NULL
    assert call(ctypes.byref(st), FAKE, FAKE, need - 1, None) == KIVI_ERR_SHAPE           # scratch too small
    assert call(ctypes.byref(_struct(group_size=48)), FAKE, FAKE, need, None) == -4        # the cache itself

"""The prefix store (kivi_b200.prefix) on CPU tensors, and kivi_prompt_attention_suffix_f16's argument checks without a
GPU.

Every stored value encodes what it stands for -- K = the token id, V = the position -- so a copied prefix shows whether
the tree returned the right tokens' K / V in the right places."""
import random

import pytest
import torch

from kivi_b200.prefix import MIN_REUSE, PrefixCache, reuse_length

LAYERS, HKV = 2, 1
TOKEN_BYTES = LAYERS * 2 * HKV * 128 * 2          # 1 KiB per stored token


class Owner:
    """Stands for a model: the cache keeps a weak reference to it."""


def cache(max_tokens, owner=None):
    pc = PrefixCache(max_tokens * TOKEN_BYTES)
    pc.bind(owner or OWNER, LAYERS, HKV, "cpu")
    return pc


OWNER = Owner()


def put(pc, tokens):
    """An insert of `tokens`: match, reserve the rest, fill it as the prompt pass would, record.  Returns the match."""
    m = pc.match(tokens)
    st = pc.reserve(m, len(tokens) - m.length)
    if st is not None:
        new = torch.tensor(tokens[m.length:], dtype=torch.float16)
        st[:, 0] = new.view(1, 1, -1, 1)
        st[:, 1] = torch.arange(m.length, len(tokens), dtype=torch.float16).view(1, 1, -1, 1)
    pc.insert(tokens, m, st)
    return m


def read(pc, tokens, r):
    """The stored K / V of the first r tokens of `tokens`, checked against the encoding in every layer."""
    m = pc.match(tokens)
    assert m.length >= r
    for layer in range(LAYERS):
        k = torch.full((HKV, r + 3, 128), -1.0, dtype=torch.float16)
        v = k.clone()
        pc.copy_prefix(m, r, layer, k, v)
        assert torch.equal(k[:, :r], torch.tensor(tokens[:r], dtype=torch.float16).view(1, -1, 1).expand(HKV, r, 128))
        assert torch.equal(v[:, :r], torch.arange(r, dtype=torch.float16).view(1, -1, 1).expand(HKV, r, 128))
        assert (k[:, r:] == -1).all() and (v[:, r:] == -1).all()          # nothing past r is written


def held_bytes(pc):
    """The bytes of the distinct allocations the tree's nodes still reference."""
    blocks = {id(nd.block): nd.block.nbytes for nd in pc._nodes()}
    return sum(blocks.values())


def seq(lo, hi):
    return list(range(lo, hi))


def test_longest_match_exact_and_inside_a_node():
    pc = cache(1000)
    a = seq(1, 101)
    assert put(pc, a).length == 0
    assert pc.match(a).length == 100
    assert pc.match(a + [7, 8]).length == 100
    assert pc.match(a[:50] + [999]).length == 50                     # diverges inside the one node
    assert pc.match(a[:50]).length == 50                             # a prompt shorter than the node
    assert pc.match([2, 3]).length == 0
    assert pc.match([]).length == 0
    read(pc, a + [5], 100)
    read(pc, a[:50] + [999], 50)


def test_divergence_splits_the_node_and_shares_its_block():
    pc = cache(1000)
    a, b = seq(1, 101), seq(1, 51) + seq(500, 561)
    put(pc, a)
    m = put(pc, b)
    assert m.length == 50 and len(m.path) == 1 and m.path[0][1] == 50
    assert len(pc) == 3                                              # head 1..50, tails 51..100 and 500..560
    assert pc.stored_bytes == (100 + 61) * TOKEN_BYTES               # the split keeps the first allocation whole
    assert pc.match(b).length == len(b) and pc.match(a).length == 100
    read(pc, a, 100)
    read(pc, b, len(b))
    c = seq(1, 21) + [7000] * 30                                     # diverges inside the new head
    put(pc, c)
    assert len(pc) == 5 and pc.match(c).length == len(c)
    read(pc, c, len(c))
    read(pc, a, 100)
    read(pc, b, len(b))
    assert pc.stored_bytes == held_bytes(pc) == (100 + 61 + 30) * TOKEN_BYTES


def test_split_halves_count_until_both_are_freed():
    pc = cache(170)
    a, b = seq(1, 101), seq(1, 51) + seq(500, 561)
    put(pc, a)
    put(pc, b)                                                       # 161 tokens held
    assert pc.stored_bytes == 161 * TOKEN_BYTES
    put(pc, seq(2000, 2009))                                         # 9 more: 170, fits
    assert pc.evictions == 0
    put(pc, seq(3000, 3050))                                         # 50 more: evict until it fits
    # LRU leaves: tail 51..100 (used at the first put), then 500..560.  Evicting the first tail frees nothing (its head
    # still holds the block); 500..560 frees 61, and 109 + 50 fit.  The head 1..50 still counts its whole 100 tokens.
    assert pc.match(a).length == 50 and pc.match(b).length == 50 and pc.evictions == 2
    assert pc.stored_bytes == held_bytes(pc) == (100 + 9 + 50) * TOKEN_BYTES
    read(pc, a, 50)
    put(pc, seq(4000, 4020))                                         # 20 more: the head is the LRU leaf, 100 freed
    assert pc.match(a).length == 0 and pc.evictions == 3
    assert pc.match(seq(2000, 2009)).length == 9
    assert pc.stored_bytes == held_bytes(pc) == (9 + 50 + 20) * TOKEN_BYTES


def test_reuse_length_caps_at_n_minus_1_and_needs_min_reuse():
    assert MIN_REUSE == 1024
    big = 4 * MIN_REUSE
    assert reuse_length(big, big) == big - 1                         # the last position is always computed
    assert reuse_length(big + 300, big) == big - 1
    assert reuse_length(MIN_REUSE - 1, big) == 0
    assert reuse_length(MIN_REUSE, big) == MIN_REUSE
    assert reuse_length(MIN_REUSE, MIN_REUSE) == 0                   # capped to MIN_REUSE - 1: below the threshold
    assert reuse_length(MIN_REUSE + 1, MIN_REUSE + 1) == MIN_REUSE
    assert reuse_length(200, 200) == 0 and reuse_length(0, 1) == 0


def test_lru_order_is_deterministic():
    def run():
        pc = cache(300)
        x, y, z = seq(1, 101), seq(1001, 1101), seq(2001, 2101)
        for t in (x, y, z):
            put(pc, t)
        put(pc, x + [9])                                             # a use of x; its one new token needs room
        return pc, x, y, z
    pc, x, y, z = run()
    # x + [9] needs one token: the least recently used leaf off its path, y, goes
    assert pc.match(y).length == 0 and pc.match(x + [9]).length == 101 and pc.match(z).length == 100
    assert pc.evictions == 1
    w = seq(3001, 3101)
    put(pc, w)                                                       # z is now the least recently used
    assert pc.match(z).length == 0 and pc.match(x).length == 100
    pc2, *_ = run()
    put(pc2, w)
    assert [nd.tokens[:1] for nd in pc._nodes()] == [nd.tokens[:1] for nd in pc2._nodes()]


def test_the_path_of_the_insert_is_never_evicted():
    pc = cache(150)
    p, q = seq(1, 101), seq(5001, 5041)
    put(pc, p)
    put(pc, q)                                                       # p is now older than q
    put(pc, p + seq(7001, 7031))                                     # 30 more: p is LRU but on the path, q goes
    assert pc.match(q).length == 0
    assert pc.match(p + seq(7001, 7031)).length == 130
    read(pc, p + seq(7001, 7031), 130)
    pc = cache(150)
    put(pc, p)
    before = pc.stored_bytes
    m = put(pc, p + seq(7001, 7061))                                 # 60 more: only the path could make room
    assert m.length == 100 and pc.stored_bytes == before and pc.evictions == 0
    assert pc.match(p + seq(7001, 7061)).length == 100 and len(pc) == 1


def test_a_span_over_the_budget_is_not_stored():
    pc = cache(10)
    m = put(pc, seq(1, 12))
    assert m.length == 0 and pc.stored_bytes == 0 and len(pc) == 0 and pc.match(seq(1, 12)).length == 0
    put(pc, seq(1, 11))
    assert pc.stored_bytes == 10 * TOKEN_BYTES
    put(pc, seq(100, 111))                                           # over the budget alone: nothing evicted for it
    assert pc.evictions == 0 and pc.match(seq(1, 11)).length == 10
    zero = PrefixCache(0)
    zero.bind(OWNER, LAYERS, HKV, "cpu")
    put(zero, [1, 2, 3])
    assert zero.stored_bytes == 0 and len(zero) == 0
    with pytest.raises(ValueError):
        PrefixCache(-1)


def test_byte_budget_holds_after_every_operation():
    """Random prompts built from a few shared heads (system prompts) and random tails; after every insert the bytes held
    equal the distinct allocations the tree references, never exceed the budget, and every stored prefix reads back."""
    rng = random.Random(0)
    heads = [[rng.randrange(1, 50) for _ in range(rng.randrange(20, 90))] for _ in range(4)]
    pc = cache(700)
    prompts = []
    for i in range(300):
        h = rng.choice(heads)
        cut = rng.randrange(0, len(h) + 1)
        prompt = h[:cut] + [rng.randrange(1, 50) for _ in range(rng.randrange(1, 60))]
        if prompts and rng.random() < 0.2:
            prompt = rng.choice(prompts) + [rng.randrange(1, 50) for _ in range(rng.randrange(1, 30))]   # a next turn
        prompts.append(prompt)
        m = pc.match(prompt)
        got = put(pc, prompt)
        assert got.length == m.length
        assert pc.stored_bytes == held_bytes(pc) <= pc.max_bytes, i
        assert pc.peak_bytes <= pc.max_bytes
        length = pc.match(prompt).length
        assert length in (got.length, len(prompt)), i                 # stored whole, or left as it was
        read(pc, prompt, length)
        for nd in pc._nodes():                                        # children are keyed by their first token
            assert all(c.tokens[0] == k for k, c in nd.children.items())
    assert pc.evictions > 0 and len(pc) > 4


def test_binding_to_a_model():
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    a = LlamaForCausalLM_KIVI(default_config("tiny", num_hidden_layers=2))
    b = LlamaForCausalLM_KIVI(default_config("tiny", num_hidden_layers=2))
    hkv = a.model.layers[0].self_attn.num_key_value_heads
    pc = PrefixCache(1 << 20)
    pc.bind(a, 2, hkv, "cpu")
    pc.bind(a, 2, hkv, torch.device("cpu"))                          # the same model again
    for args in ((b, 2, hkv, "cpu"), (a, 3, hkv, "cpu"), (a, 2, hkv + 1, "cpu"), (a, 2, hkv, "meta")):
        with pytest.raises(ValueError):
            pc.bind(*args)
    assert pc.span_bytes(1) == 2 * 2 * hkv * 128 * 2


# ------------------------------------------------------------------------------------------------ the C entry
KIVI_ERR_SHAPE, KIVI_ERR_GQA, KIVI_ERR_ALIGN, KIVI_ERR_NULL = -2, -3, -5, -6
FAKE = 1 << 20                                       # 16-byte aligned, never dereferenced: validation returns first


@pytest.fixture(scope="module")
def lib():
    from kivi_b200 import _lib, build, glue
    build.build()
    glue._bind()
    return _lib.lib()


def _call(lib, q=FAKE, k=FAKE, v=FAKE, out=FAKE, B=2, H=32, Hkv=8, m=40, n=100, q_strides=(40 * 4096, 128, 4096),
          kv_strides=(100 * 1024, 128, 1024), kv_start=None, window=0):
    return lib.kivi_prompt_attention_suffix_f16(q, k, v, out, B, H, Hkv, m, n, *q_strides, *kv_strides, kv_start, window,
                                                None)


def test_suffix_symbol_is_exported(lib):
    assert hasattr(lib, "kivi_prompt_attention_suffix_f16")


def test_suffix_rejects_every_invalid_argument(lib):
    for name in ("q", "k", "v", "out"):
        assert _call(lib, **{name: None}) == KIVI_ERR_NULL, name
    for kw in (dict(m=0), dict(m=-1), dict(m=101), dict(m=2, n=1), dict(B=0), dict(B=65536), dict(H=0), dict(n=0),
               dict(n=-3, m=-3), dict(window=-1), dict(H=65536 * 8, Hkv=65536)):
        assert _call(lib, **kw) == KIVI_ERR_SHAPE, kw
    for kw in (dict(Hkv=0), dict(Hkv=-8), dict(Hkv=5), dict(H=6, Hkv=4), dict(H=8, Hkv=65536 // 8)):
        assert _call(lib, **kw) == KIVI_ERR_GQA, kw
    for name in ("q", "k", "v", "out"):
        for off in (2, 8):
            assert _call(lib, **{name: FAKE + off}) == KIVI_ERR_ALIGN, (name, off)
    assert _call(lib, kv_start=FAKE + 2) == KIVI_ERR_ALIGN
    for i in range(3):
        qs, kvs = [40 * 4096, 128, 4096], [100 * 1024, 128, 1024]
        qs[i] += 4
        assert _call(lib, q_strides=tuple(qs)) == KIVI_ERR_ALIGN, ("q", i)
        kvs[i] -= 2
        assert _call(lib, kv_strides=tuple(kvs)) == KIVI_ERR_ALIGN, ("kv", i)
    assert _call(lib, q=FAKE + 2, m=0) == KIVI_ERR_SHAPE                  # shape errors come before alignment
    assert _call(lib, q=None, m=0) == KIVI_ERR_NULL
    assert _call(lib, out=FAKE + 2, H=32, Hkv=5) == KIVI_ERR_GQA


def test_full_entry_still_validates_as_before(lib):
    """The full entry now shares the suffix entry's checks (m = n): its documented codes are unchanged."""
    full = lambda **kw: lib.kivi_prompt_attention_f16(FAKE, FAKE, FAKE, FAKE, 2, 32, 8, kw.get("n", 100),   # noqa: E731
                                                      100 * 4096, 128, 4096, 100 * 1024, 128, 1024, None, 0, None)
    assert full(n=0) == KIVI_ERR_SHAPE and full(n=-1) == KIVI_ERR_SHAPE


def test_charge_is_the_allocators_worst_case_from_the_size_alone():
    """A block counts its size rounded up to 512 bytes, plus 1 MiB over 1 MiB (a large-pool block the caching allocator
    does not split); the charge, and so every eviction, depends on the size only."""
    from kivi_b200.prefix import charge
    assert charge(1) == 512 and charge(1024) == 1024 and charge(1025) == 1536
    assert charge(1 << 20) == 1 << 20
    assert charge((1 << 20) + 1) == (1 << 20) + 512 + (1 << 20)
    assert charge(512 << 20) == (513 << 20)
    pc = cache(3000)
    put(pc, seq(1, 1100))                                            # 1099 KiB: over 1 MiB, charged 1 MiB more
    assert pc.stored_bytes == held_bytes(pc) == 1099 * TOKEN_BYTES + (1 << 20)

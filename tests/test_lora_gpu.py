"""LoRA adapters on the GPU.  Kernels: kivi_lora_shrink_f16 + kivi_lora_expand_f16 against a float64 reference at the
header's bound over the group shapes of Llama-2-7B, Llama-3-8B and Qwen2.5-7B, ranks 1 .. 128 and mixed, rows, slots and
magnitudes; untouched rows, zero adapters, run-to-run and graph-replay bit-identity and row independence.  Model:
transformers parity with the adapter merged in float64 (llama3, Qwen2 with biases, Qwen3 with q/k norms), mixed-adapter
batches bit-equal to single-adapter ones, the launch count, generate(adapter=), serve() with mixed adapters and the prefix
cache's adapter namespaces."""
import pytest
import torch

from tests._hf import Bar, Decoder, checkpoints, load_kivi, reference_models  # noqa: F401 (fixture)
from tests._lora import adapter_state, merge_into, write_adapter
from tests._model import same_logits, small_cfg

pytestmark = pytest.mark.gpu

# (in, segment widths) of the four groups
SHAPES = {
    "llama-2-7b": dict(qkv=(4096, [4096, 4096, 4096]), o=(4096, [4096]), gu=(4096, [11008, 11008]), down=(11008, [4096])),
    "llama-3-8b": dict(qkv=(4096, [4096, 1024, 1024]), o=(4096, [4096]), gu=(4096, [14336, 14336]), down=(14336, [4096])),
    "qwen2.5-7b": dict(qkv=(3584, [3584, 512, 512]), o=(3584, [3584]), gu=(3584, [18944, 18944]), down=(18944, [3584])),
}


def _stack(S, n_seg, ranks, n_in, out, mag, gen):
    """A [S, n_seg, R, in], B [S, out, R] with adapter s of rank ranks[s] (zero-padded), scale [S]; deltas of about mag."""
    R = max(8, -(-max(ranks) // 8) * 8)
    A = torch.zeros((S, n_seg, R, n_in), dtype=torch.float16, device="cuda")
    B = torch.zeros((S, out, R), dtype=torch.float16, device="cuda")
    for s, r in enumerate(ranks):
        A[s, :, :r] = (torch.randn((n_seg, r, n_in), device="cuda", generator=gen) / n_in ** 0.5).half()
        B[s, :, :r] = (torch.randn((out, r), device="cuda", generator=gen) * mag / r ** 0.5).half()
    scale = torch.rand(S, device="cuda", generator=gen) + 0.5
    return A, B, scale


def _run(x, y, A, B, scale, segs, idx):
    from kivi_b200 import glue
    ws = torch.empty(glue.lora_workspace_bytes(x.shape[0], x.shape[1], A.shape[1], A.shape[2]) // 4, device="cuda")
    out = y.clone()
    glue.lora_apply(x, out, A, B, scale, segs, idx, ws)
    return out


def _check(x, y, A, B, scale, segs, idx, out):
    """out against the float64 value at the bound of include/kivi_b200.h; rows outside [0, S) bit-equal to y."""
    S, n_seg, R, n_in = A.shape
    live = (idx >= 0) & (idx < S)
    assert torch.equal(out[~live].view(torch.int16), y[~live].view(torch.int16))
    c = (n_in + R + 3) * 2.0 ** -24
    for s in idx[live].unique().tolist():
        rows = (idx == s).nonzero().squeeze(1)
        xd = x[rows].double()
        v, M = y[rows].double(), torch.zeros((rows.numel(), y.shape[1]), dtype=torch.float64, device="cuda")
        for g in range(n_seg):
            cols = slice(segs[g], segs[g + 1])
            Ad, Bd = A[s, g].double(), B[s, cols].double()
            v[:, cols] += float(scale[s]) * ((xd @ Ad.t()) @ Bd.t())
            M[:, cols] = abs(float(scale[s])) * ((xd.abs() @ Ad.abs().t()) @ Bd.abs().t())
        bound = 2.0 ** -11 * v.abs() + (1 + 2.0 ** -11) * c * (M + v.abs()) + 2.0 ** -25
        err = (out[rows].double() - v).abs()
        assert (err <= bound).all(), f"slot {s}: max err {err.max().item():.3g}, worst err / bound {(err / bound).max():.3g}"


RANKS = [[1], [8], [16], [64], [128], [1, 16, 64, 128, 8, 3]]


@pytest.mark.parametrize("model", list(SHAPES))
@pytest.mark.parametrize("group", ["qkv", "o", "gu", "down"])
def test_kernels_against_float64(model, group):
    import zlib
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"{model} {group}".encode()))
    n_in, widths = SHAPES[model][group]
    segs = [0]
    for w in widths:
        segs.append(segs[-1] + w)
    combos = [(rows, S) for rows in (1, 3, 32, 256) for S in (1, 4, 17)]
    for i, ranks in enumerate(RANKS):
        for j, mag in enumerate((1e-3, 1.0, 1e3)):
            rows, S = combos[(3 * i + j) % len(combos)]
            A, B, scale = _stack(S, len(widths), [ranks[s % len(ranks)] for s in range(S)], n_in, segs[-1], mag, gen)
            x = (torch.randn((rows, n_in), device="cuda", generator=gen)).half()
            y = (torch.randn((rows, segs[-1]), device="cuda", generator=gen) * mag).half()
            idx = torch.randint(-1, S + 1, (rows,), device="cuda", generator=gen, dtype=torch.int32)
            idx[0] = S - 1
            _check(x, y, A, B, scale, segs, idx, _run(x, y, A, B, scale, segs, idx))


def test_every_rows_and_slots():
    gen = torch.Generator(device="cuda").manual_seed(5)
    n_in, widths = SHAPES["llama-3-8b"]["qkv"]
    segs = [0, 4096, 5120, 6144]
    for rows in (1, 3, 32, 256, 1024):
        for S in (1, 4, 17):
            A, B, scale = _stack(S, 3, [16] * S, n_in, 6144, 1.0, gen)
            x = torch.randn((rows, n_in), device="cuda", generator=gen).half()
            y = torch.randn((rows, 6144), device="cuda", generator=gen).half()
            idx = torch.randint(0, S, (rows,), device="cuda", generator=gen, dtype=torch.int32)
            _check(x, y, A, B, scale, segs, idx, _run(x, y, A, B, scale, segs, idx))


def test_untouched_rows_zero_adapter_determinism_and_independence():
    from kivi_b200 import glue
    gen = torch.Generator(device="cuda").manual_seed(7)
    rows, S, n_in, segs = 64, 5, 4096, [0, 11008, 22016]
    A, B, scale = _stack(S, 2, [16, 8, 64, 16, 1], n_in, segs[-1], 1.0, gen)
    B[3].zero_()                                                          # slot 3: an adapter whose B is 0
    x = torch.randn((rows, n_in), device="cuda", generator=gen).half()
    y = torch.randn((rows, segs[-1]), device="cuda", generator=gen).half()
    y[::7] = -0.0
    idx = torch.randint(-3, S + 3, (rows,), device="cuda", generator=gen, dtype=torch.int32)
    idx[:6] = torch.tensor([-1, S, 3, 0, 2, 1], dtype=torch.int32)      # row 5 (slot 1) is the one followed below
    out = _run(x, y, A, B, scale, segs, idx)
    keep = (idx < 0) | (idx >= S) | (idx == 3)
    assert keep.sum() > 4 and (~keep).sum() > 4
    assert torch.equal(out[keep].view(torch.int16), y[keep].view(torch.int16))   # guard values and -0 stay
    assert not torch.equal(out[~keep], y[~keep])
    for _ in range(3):
        assert torch.equal(_run(x, y, A, B, scale, segs, idx), out)
    # graph replay
    ws = torch.empty(glue.lora_workspace_bytes(rows, n_in, 2, A.shape[2]) // 4, device="cuda")
    yy = y.clone()
    glue.lora_apply(x, yy, A, B, scale, segs, idx, ws)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        glue.lora_apply(x, yy, A, B, scale, segs, idx, ws)
    for _ in range(2):
        yy.copy_(y)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(yy, out)
    # row independence: other rows' adapters permuted, S grown -- row b stays bit-equal
    for trial in range(3):
        idx2 = idx[torch.randperm(rows, device="cuda", generator=gen)].clone()
        idx2[5] = idx[5]
        idx2[idx2 >= S] = -1                                              # slots the grown stack adds stay unused
        A2, B2, scale2 = (torch.cat([t, t[:2]]) for t in (A, B, scale))
        assert torch.equal(_run(x, y, A2, B2, scale2, segs, idx2)[5], out[5])


# ---------------------------------------------------------------------------------------------------- model
def _tiny(seed=0, **kw):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    torch.manual_seed(seed)
    return LlamaForCausalLM_KIVI(small_cfg(num_hidden_layers=2, **kw)).half().cuda().eval()


def _adapters(model, tmp_path, specs):
    """Load adapters name -> (rank, targets, seed) into model; returns their states."""
    states = {}
    for name, (r, targets, seed) in specs.items():
        st = adapter_state(model.config, r, targets, seed=seed, gain=2.0)
        model.load_adapter(write_adapter(tmp_path / name, st, r, 2 * r, targets), name)
        states[name] = st
    return states


SPECS = {"a": (16, "all-linear", 1), "b": (8, ["q_proj", "v_proj", "down_proj"], 2), "c": (64, "all-linear", 3)}


def _targets(t):
    from kivi_b200.lora import LINEARS
    return list(LINEARS) if t == "all-linear" else t


def test_no_adapter_unchanged_and_launch_count(tmp_path):
    B, n = 8, 40
    ids = torch.randint(0, 4096, (B, n), device="cuda")
    fresh, m = _tiny(), _tiny()
    for x in (fresh, m):
        x.init_cache(B, 256)
        x.prefill(ids)
    same_logits(fresh, m, 6, tok=ids[:, -1:])
    base = m.launches_per_step
    _adapters(m, tmp_path, {k: (r, _targets(t), s) for k, (r, t, s) in SPECS.items()})
    m.init_cache(B, 256)
    m.prefill(ids)
    m.decode_step(ids[:, -1:])
    assert m.launches_per_step == base + 8 * len(m.model.layers)
    m.init_cache(B, 256)
    m.prefill(ids)
    fresh.init_cache(B, 256)
    fresh.prefill(ids)
    same_logits(fresh, m, 6, tok=ids[:, -1:])                          # loaded but unused: rows bit-equal


def test_mixed_batch_rows_equal_single_adapter_batches(tmp_path):
    B, n = 6, 33
    m = _tiny()
    _adapters(m, tmp_path, {k: (r, _targets(t), s) for k, (r, t, s) in SPECS.items()})
    ids = torch.randint(0, 4096, (B, n), device="cuda")
    names = ["a", None, "b", "c", "a", "c"]

    def decode(sel):
        """The decode steps' logits from one cache state (prompt pass without adapters), rows on adapters `sel`."""
        m.init_cache(B, 256)
        m.set_adapters(None)
        tok = m.prefill(ids).argmax(-1, keepdim=True)
        m.set_adapters(sel)
        out = []
        for _ in range(6):
            out.append(m.decode_step(tok).clone())
            tok = m.next_tokens.view(-1, 1).clone()
        return out
    mixed = decode(names)
    for name in set(names):
        rows = [b for b in range(B) if names[b] == name]
        for s, got in enumerate(decode(name)):
            assert torch.equal(got[rows], mixed[s][rows]), (name, s)
    assert not torch.equal(mixed[-1][0], mixed[-1][1])


@pytest.mark.parametrize("case", ["llama3", "qwen2", "qwen3"])
def test_transformers_parity(tmp_path_factory, case):
    import importlib
    bar = Bar()
    tmp = tmp_path_factory.mktemp(f"lora_{case}")
    if case == "llama3":
        from tests._hf import write_checkpoint
        write_checkpoint("llama3", tmp / "ckpt")
        ref64, hf16 = reference_models("llama3", tmp / "ckpt")
        model = load_kivi("llama3", tmp / "ckpt")
    else:
        mod = importlib.import_module("tests._qwen" if case == "qwen2" else "tests._qwen3")
        name = "qwen-ratio7" if case == "qwen2" else "qwen3-ratio4"
        mod.write_checkpoint(name, tmp / "ckpt")
        ref64, hf16 = mod.reference_models(tmp / "ckpt") if case == "qwen2" else mod.reference_models(name, tmp / "ckpt")
        model = mod.load_kivi(name, tmp / "ckpt")
    cfg = model.config
    r, alpha = 16, 32
    st = adapter_state(cfg, r, _targets("all-linear"), seed=11, gain=1.0)
    model.load_adapter(write_adapter(tmp / "adapter", st, r, alpha, "all-linear"), "ft")
    B, n = 3, 150
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda")
    base = ref64(input_ids=ids).logits
    for hf in (ref64, hf16):
        merge_into(hf, st, alpha / r)
    ref, hf = ref64(input_ids=ids).logits, hf16(input_ids=ids).logits
    bar_value = 4.0 * (hf - ref).abs().max().item() + 1e-3 * ref.abs().max().item()
    assert (base - ref).abs().max().item() > 10 * bar_value                # the adapter moves the logits
    model.set_adapters("ft")
    model.fused_forward = False
    bar.check(f"{case} forward", model(input_ids=ids).logits, ref, hf)
    model.fused_forward = True
    model.init_cache(B, n + 80)
    model.set_adapters("ft")
    bar.check(f"{case} prefill", model.prefill(ids), ref[:, -1], hf[:, -1])
    Decoder(bar, model, ref64, hf16, T=n, pos=[n] * B, start=[0] * B,
            gen=torch.Generator(device="cuda").manual_seed(3)).run(40, f"{case} decode")
    bar.report(f"lora {case}")


def test_generate_with_adapters(tmp_path):
    m = _tiny()
    _adapters(m, tmp_path, {k: (r, _targets(t), s) for k, (r, t, s) in SPECS.items()})
    ids = torch.randint(0, 4096, (3, 24), device="cuda")
    mask = torch.ones_like(ids)
    mask[1, :5] = 0
    mask[2, :11] = 0
    names = ["a", "b", None]
    # greedy: a prompt's rows as with every prompt on its adapter.  Beam search and sampling choose among near-equal
    # scores of a random model, where the prompt pass's per-adapter grouping (the matmuls' row counts) can move a choice:
    # their rows are checked for reproducibility, for the prompt without an adapter and for taking the adapter.
    for kw in (dict(),):
        mixed = m.generate(ids, max_new_tokens=12, attention_mask=mask, adapter=names, **kw)
        K = mixed.shape[0] // 3
        for b, name in enumerate(names):
            alone = m.generate(ids, max_new_tokens=12, attention_mask=mask, adapter=name, **kw)
            assert torch.equal(alone[b * K:(b + 1) * K], mixed[b * K:(b + 1) * K]), (kw, name)
    for kw in (dict(num_beams=3, num_return_sequences=2), dict(do_sample=True, temperature=0.8, seed=3),
               dict(do_sample=True, num_return_sequences=2, seed=5)):
        mixed = m.generate(ids, max_new_tokens=12, attention_mask=mask, adapter=names, **kw)
        assert torch.equal(mixed, m.generate(ids, max_new_tokens=12, attention_mask=mask, adapter=names, **kw))
        base = m.generate(ids, max_new_tokens=12, attention_mask=mask, **kw)
        K = mixed.shape[0] // 3
        assert torch.equal(base[2 * K:], mixed[2 * K:]) and not torch.equal(base[:K], mixed[:K]), kw
    plain = m.generate(ids, max_new_tokens=12, attention_mask=mask)
    assert not torch.equal(plain[0], m.generate(ids, max_new_tokens=12, attention_mask=mask, adapter="a")[0])
    with pytest.raises(KeyError):
        m.generate(ids, max_new_tokens=4, adapter="nope")


def test_serve_mixed_adapters_and_prefix_namespaces(tmp_path):
    from kivi_b200.prefix import MIN_REUSE, PrefixCache
    from kivi_b200.serve import serve
    m = _tiny()
    _adapters(m, tmp_path, {k: (r, _targets(t), s) for k, (r, t, s) in SPECS.items()})
    gen = torch.Generator().manual_seed(0)
    prompts = [torch.randint(0, 4096, (int(n),), generator=gen) for n in (51, 41, 44, 49, 19, 43)]
    names = ["a", "b", None, "c", "a", "b"]
    samp = [dict(), dict(temperature=0.7, seed=9)]
    for extra in samp:
        reqs = [(p, 10, dict(extra, adapter=a) if a else (dict(extra) or None)) for p, a in zip(prompts, names)]
        reqs = [r if r[2] is not None else r[:2] for r in reqs]
        out = dict(serve(m, reqs, batch=3, max_tokens=256))
        again = dict(serve(m, reqs, batch=3, max_tokens=256))
        assert all(torch.equal(out[i], again[i]) for i in out)
        # the requests after the first group are inserts, one prompt pass each: their neighbours' adapters, swapped
        # around, do not change their tokens
        swapped = [(p, n, dict(par, adapter={"a": "c", "b": "a", "c": "b"}[par["adapter"]]))
                   if i < 3 and len(r) == 3 and par and "adapter" in par else r
                   for i, r in enumerate(reqs) for p, n, par in [(r[0], r[1], r[2] if len(r) == 3 else None)]]
        got = dict(serve(m, swapped, batch=3, max_tokens=256))
        for i in range(3, len(reqs)):
            assert torch.equal(got[i], out[i]), (extra, i)
        plain = dict(serve(m, [r[:2] for r in reqs], batch=3, max_tokens=256))
        assert not torch.equal(plain[0], out[0])
    # the same long prompt under two adapters: the filler keeps the timeline alive, so requests 2 and 3 are inserts
    long = torch.randint(0, 4096, (MIN_REUSE + 200,), generator=gen)
    pc, stats = PrefixCache(1 << 30), {}
    plain, hits = {}, []
    for a in ("a", "b"):
        req = (torch.cat([long, torch.tensor([1, 2, 3])]), 6, dict(adapter=a))
        stream = [(long[:300], 40), req, req, req]
        plain[a] = dict(serve(m, stream, batch=2, max_tokens=4096))
        got = dict(serve(m, stream, batch=2, max_tokens=4096, prefix_cache=pc, stats=stats))
        hits.append(stats["prefix_hits"])
        for i in range(4):
            assert torch.equal(got[i], plain[a][i]), (a, i)
    assert hits == [1, 2]                                                 # one hit per adapter, none across them
    assert not torch.equal(plain["a"][3], plain["b"][3])


def test_load_adapter_refused_under_tensor_parallel(tmp_path):
    from tests._model import world_one_pair
    _, tpm = world_one_pair(small_cfg(num_hidden_layers=2))
    st = adapter_state(tpm.config, 8, ["q_proj"])
    with pytest.raises(NotImplementedError, match="tensor parallel"):
        tpm.load_adapter(write_adapter(tmp_path / "a", st, 8, 16, ["q_proj"]), "a")

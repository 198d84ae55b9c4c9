"""Tensor-parallel decode on the GPU.

One GPU: kivi_allreduce_add_rmsnorm_f16 with N in {2, 4, 8} ranks emulated on one device -- the N rank buffers are regions of
one allocation with the layout of include/kivi_b200.h, the other ranks' arrival counters are pre-set to the call's number so
no call waits -- against add_rmsnorm of the fp32 rank-order sum, bit for bit; world 1 (no peers) against add_rmsnorm; argument
errors; and the tensor-parallel model at world 1 against the plain model.
Two or more GPUs (one process per GPU, NCCL on 127.0.0.1): the sharded model's decode steps against a one-GPU emulation of the
sharded step (bit for bit) and against the unsharded model (tolerance), identical tokens on every rank, left-padded generate
and serve()."""
import os
from types import SimpleNamespace

import pytest
import torch

from tests._model import same_logits, same_on_all_ranks, sharded_model, small_cfg, spawn_ranks, world_one_pair

pytestmark = pytest.mark.gpu

KIVI_ERR_SHAPE, KIVI_ERR_ALIGN, KIVI_ERR_NULL = -2, -5, -6


def _emulated_ranks(world, rows, hidden, epoch, call, partials, rank):
    """One device allocation holding `world` rank buffers; partial p in rank p's slot of `call`; the counters of `rank`'s
    buffer say every other rank has arrived at the call."""
    slot_words = rows * hidden * 2 // 8
    words = 2 * slot_words + world                                      # partial[2][rows][hidden] + arrived[world]
    buf = torch.zeros(world, words, dtype=torch.int64, device="cuda")
    for p in range(world):
        buf[p].view(torch.float16)[: 2 * rows * hidden].view(2, rows, hidden)[call & 1] = partials[p]
    e = epoch + call + 1
    buf[rank, 2 * slot_words:] = e
    buf[rank, 2 * slot_words + rank] = e - 1                            # the call itself announces this rank
    ptrs = torch.tensor([buf[p].data_ptr() for p in range(world)], dtype=torch.int64, device="cuda")
    ar = SimpleNamespace(peer_ptrs=ptrs, rank=rank, world=world, rows_max=rows, hidden=hidden,
                         epoch=torch.tensor([epoch], dtype=torch.int64, device="cuda"),
                         err=torch.zeros(1, dtype=torch.int32, device="cuda"))
    return buf, ar, 2 * slot_words


def _rank_order_sum(partials):
    acc = partials[0].float()
    for p in partials[1:]:
        acc = acc + p.float()
    return acc.half()


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("hidden", [4096, 5120, 8192])
def test_allreduce_add_rmsnorm_matches_add_rmsnorm(world, hidden):
    from kivi_b200 import glue
    gen = torch.Generator(device="cuda").manual_seed(world * 100 + hidden)
    for rows in (1, 3, 32, 64):
        for scale in (1e-3, 1.0, 300.0, 3e4):                            # 3e4: partial sums beyond the fp16 range
            partials = [(torch.randn((rows, hidden), generator=gen, device="cuda") * scale).clamp(-6e4, 6e4).half()
                        for _ in range(world)]                           # finite partials; their sums may not be
            res0 = (torch.randn((rows, hidden), generator=gen, device="cuda") * min(scale, 100.0)).half()
            w = (torch.rand(hidden, generator=gen, device="cuda") + 0.5).half()
            exp_res, exp_out = res0.clone(), torch.empty_like(res0)
            glue.add_rmsnorm(_rank_order_sum(partials), exp_res, w, exp_out, 1e-5)
            rank, call, epoch = rows % world, rows % 3, 2 * hidden
            for cluster in ((0, 1, 2, 4, 8) if scale == 1.0 else (0,)):
                buf, ar, cnt = _emulated_ranks(world, rows, hidden, epoch, call, partials, rank)
                res, out = res0.clone(), torch.full_like(res0, float("nan"))
                glue.allreduce_add_rmsnorm(res, w, out, 1e-5, ar, call=call, cluster=cluster)
                torch.cuda.synchronize()
                ctx = (world, hidden, rows, scale, cluster)
                assert int(ar.err.item()) == 0, ctx
                assert torch.equal(_bits(res), _bits(exp_res)), ctx
                assert torch.equal(_bits(out), _bits(exp_out)), ctx
                e = epoch + call + 1                                     # the arrival went to every rank's buffer
                assert all(int(buf[p, cnt + rank]) == e for p in range(world)), ctx


def test_world_one_without_peers_is_add_rmsnorm():
    from kivi_b200 import glue
    torch.manual_seed(0)
    for rows, hidden in ((1, 4096), (5, 8192), (64, 5120)):
        x = torch.randn((rows, hidden), device="cuda").half()
        res0 = torch.randn((rows, hidden), device="cuda").half()
        w = (torch.rand(hidden, device="cuda") + 0.5).half()
        r1, o1, r2, o2 = res0.clone(), torch.empty_like(x), res0.clone(), torch.empty_like(x)
        glue.add_rmsnorm(x, r1, w, o1, 1e-5)
        glue.allreduce_add_rmsnorm(r2, w, o2, 1e-5, None, x=x)
        assert torch.equal(_bits(r1), _bits(r2)) and torch.equal(_bits(o1), _bits(o2))


def test_argument_errors_launch_nothing():
    from kivi_b200 import _lib, glue
    glue._bind()
    f = _lib.lib().kivi_allreduce_add_rmsnorm_f16
    rows, hidden, world = 4, 4096, 2
    partials = [torch.zeros((rows, hidden), dtype=torch.float16, device="cuda")] * world
    buf, ar, _ = _emulated_ranks(world, rows, hidden, 0, 0, partials, 0)
    res = torch.zeros((rows, hidden), dtype=torch.float16, device="cuda")
    out, w = torch.empty_like(res), torch.ones(hidden, dtype=torch.float16, device="cuda")
    P, E, ERR = ar.peer_ptrs.data_ptr(), ar.epoch.data_ptr(), ar.err.data_ptr()
    R, W, O = res.data_ptr(), w.data_ptr(), out.data_ptr()
    cases = [
        ((None, None, W, O, rows, hidden, 1e-5, P, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_NULL),
        ((None, R, W, O, rows, 4100, 1e-5, P, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_SHAPE),      # hidden % 8
        ((None, R, W, O, rows, 16392, 1e-5, P, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_SHAPE),     # hidden > 16384
        ((None, R, W, O, -1, hidden, 1e-5, P, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_SHAPE),
        ((None, R, W, O, rows + 1, hidden, 1e-5, P, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_SHAPE),  # rows > rows_max
        ((None, R, W, O, rows, hidden, 1e-5, P, 0, 9, rows, 0, E, ERR, 0, None), KIVI_ERR_SHAPE),        # world > 8
        ((None, R, W, O, rows, hidden, 1e-5, P, 0, 0, rows, 0, E, ERR, 0, None), KIVI_ERR_SHAPE),        # world < 1
        ((None, R, W, O, rows, hidden, 1e-5, P, 2, world, rows, 0, E, ERR, 0, None), KIVI_ERR_SHAPE),    # rank >= world
        ((None, R, W, O, rows, hidden, 1e-5, P, 0, world, rows, 0, E, ERR, 3, None), KIVI_ERR_SHAPE),    # cluster width
        ((None, R, W, O, rows, hidden, 1e-5, None, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_NULL),  # world 2, no peers
        ((None, R, W, O, rows, hidden, 1e-5, P, 0, world, rows, 0, None, ERR, 0, None), KIVI_ERR_NULL),
        ((None, R + 2, W, O, rows, hidden, 1e-5, P, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_ALIGN),
        ((None, R, W, O + 8, rows, hidden, 1e-5, P, 0, world, rows, 0, E, ERR, 0, None), KIVI_ERR_ALIGN),
    ]
    n0 = _lib.launch_count()
    for args, code in cases:
        assert f(*args) == code, (args, code)
    assert _lib.launch_count() == n0
    with pytest.raises(ValueError):                                       # the wrapper's own checks
        glue.allreduce_add_rmsnorm(torch.zeros((rows + 1, hidden), dtype=torch.float16, device="cuda"), w,
                                   torch.empty((rows + 1, hidden), dtype=torch.float16, device="cuda"), 1e-5, ar)
    torch.cuda.synchronize()


def _fill_cache(model, heads, n, seed, rank=0, world=1):
    """The same n random K/V tokens for every rank (this rank's KV heads of them), packed by the real prefill kernels."""
    c = model.cache
    gen = torch.Generator(device=c.device).manual_seed(seed)
    lo, hi = rank * heads // world, (rank + 1) * heads // world
    for layer in range(c.n_layers):
        k = torch.randn((c.batch, heads, n, 128), generator=gen, device=c.device, dtype=torch.float16)
        v = torch.randn((c.batch, heads, n, 128), generator=gen, device=c.device, dtype=torch.float16)
        c.prefill(layer, k[:, lo:hi].contiguous(), v[:, lo:hi].contiguous())
    model._pos.fill_(n)


def test_tensor_parallel_model_at_world_one_matches_the_model():
    """tensor_parallel=True on one GPU runs the sharded decode step (partials in the PeerAllReduce slots, the all-reduce
    kernel, the in-graph call counter) with one rank: its logits and tokens equal the plain model's bit for bit."""
    cfg = small_cfg()
    plain, tpm = world_one_pair(cfg)
    B, n = 3, 70
    for m in (plain, tpm):
        m.init_cache(B, n + 2 * cfg.residual_length + 8)
        _fill_cache(m, cfg.num_key_value_heads, n, seed=5)
    ids = torch.randint(0, cfg.vocab_size, (B, 1), device="cuda")
    graph = lambda s: s >= 1                                              # noqa: E731
    same_logits(plain, tpm, 2 * cfg.residual_length + 3, ids, graph, graph)     # crosses a K flush and a V-ring wrap
    assert int(tpm._allreduce.epoch.item()) == (2 * cfg.residual_length + 3 + 1) * 2 * cfg.num_hidden_layers  # + warm-up
    # prompt pass, left padding and generate on the same path
    prompt = torch.randint(0, cfg.vocab_size, (2, 40), device="cuda")
    mask = torch.ones_like(prompt)
    mask[1, :9] = 0
    a = plain.generate(prompt, max_new_tokens=12, attention_mask=mask)
    b = tpm.generate(prompt, max_new_tokens=12, attention_mask=mask)
    assert torch.equal(a, b)
    with pytest.raises(NotImplementedError):
        tpm(prompt)
    with pytest.raises(NotImplementedError):
        tpm.cache.export(0)
    with pytest.raises(NotImplementedError):
        tpm.enable_token_allgather(2)


# ------------------------------------------------------------------------------------------------ two or more GPUs
class _Emulation:
    """The sharded decode step of `world` ranks run on one GPU: one KiviCache per rank, the per-rank GEMMs of the same
    shapes as the ranks run, the partials added in fp32 in rank order, then add_rmsnorm."""

    def __init__(self, cfg, shards, B, max_tokens, n, seed):
        from kivi_b200.cache import KiviCache
        from kivi_b200.llama_kivi import _rope_tables
        self.cfg, self.world, self.B = cfg, len(shards), B
        dev = torch.device("cuda", 0)
        g = lambda s, k: s[k].to(dev)                                        # noqa: E731
        self.ranks = []
        for r, s in enumerate(shards):
            layers = []
            for i in range(cfg.num_hidden_layers):
                p = f"model.layers.{i}."
                layers.append(SimpleNamespace(
                    wqkv=torch.cat([g(s, p + "self_attn.q_proj.weight"), g(s, p + "self_attn.k_proj.weight"),
                                    g(s, p + "self_attn.v_proj.weight")], 0).t().contiguous(),
                    wo=g(s, p + "self_attn.o_proj.weight").t().contiguous(),
                    wgu=torch.cat([g(s, p + "mlp.gate_proj.weight"), g(s, p + "mlp.up_proj.weight")], 0).t().contiguous(),
                    wd=g(s, p + "mlp.down_proj.weight")))
            H, Hkv = cfg.num_attention_heads // self.world, cfg.num_key_value_heads // self.world
            cache = KiviCache(cfg.num_hidden_layers, B, H, Hkv, 128, cfg.k_bits, cfg.v_bits, cfg.group_size,
                              cfg.residual_length, max_tokens, device=dev, overlap_prologue=True)
            holder = SimpleNamespace(cache=cache, _pos=torch.zeros((B, 1), dtype=torch.long, device=dev))
            _fill_cache(holder, cfg.num_key_value_heads, n, seed, r, self.world)
            self.ranks.append(SimpleNamespace(layers=layers, cache=cache, H=H, Hkv=Hkv))
        s = shards[0]
        self.embed, self.norm, self.lm_head = g(s, "model.embed_tokens.weight"), g(s, "model.norm.weight"), g(s, "lm_head.weight")
        self.ln = [(g(s, f"model.layers.{i}.input_layernorm.weight"), g(s, f"model.layers.{i}.post_attention_layernorm.weight"))
                   for i in range(cfg.num_hidden_layers)]
        self.pos = torch.full((B, 1), n, dtype=torch.long, device=dev)
        self.cos, self.sin = _rope_tables(128, max_tokens + 1, cfg.rope_theta, dev)

    def step(self, ids):
        from kivi_b200 import glue
        cfg, B, eps = self.cfg, self.B, self.cfg.rms_norm_eps
        res = self.embed[ids.view(-1)].contiguous()
        h = torch.empty_like(res)
        glue.add_rmsnorm(None, res, self.ln[0][0], h, eps)
        for i in range(cfg.num_hidden_layers):
            parts = []
            for r in self.ranks:
                L = r.layers[i]
                qkv = torch.mm(h, L.wqkv)
                q, k, v = (torch.empty((B, n_, 128), dtype=torch.float16, device=h.device) for n_ in (r.H, r.Hkv, r.Hkv))
                glue.rope_split(qkv, self.cos, self.sin, self.pos, q, k, v)
                attn = r.cache.decode_attention(i, q, k, v)
                parts.append(torch.mm(attn.view(B, -1), L.wo))
            glue.add_rmsnorm(_rank_order_sum(parts), res, self.ln[i][1], h, eps)
            parts = []
            for r in self.ranks:
                L = r.layers[i]
                gu = torch.mm(h, L.wgu)
                act = torch.empty((B, gu.shape[1] // 2), dtype=torch.float16, device=h.device)
                glue.silu_mul(gu, act)
                parts.append(torch.mm(act, L.wd.t()))
            nxt = self.ln[i + 1][0] if i + 1 < cfg.num_hidden_layers else self.norm
            glue.add_rmsnorm(_rank_order_sum(parts), res, nxt, h, eps)
        for r in self.ranks:
            r.cache.advance()
        self.pos += 1
        return torch.mm(h, self.lm_head.t()).float()


def _tp_worker(rank, ws, out_dir):
    import torch.distributed as dist
    from kivi_b200 import tp
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    from kivi_b200.serve import serve
    cfg = small_cfg()
    model, full = sharded_model(cfg, rank, ws)
    dev = torch.device("cuda", rank)
    B, n, R = 4, 70, cfg.residual_length
    steps = 2 * R + 3                                                     # crosses a K flush and a V-ring wrap
    model.init_cache(B, n + steps + 8)
    _fill_cache(model, cfg.num_key_value_heads, n, seed=9, rank=rank, world=ws)
    if rank == 0:
        emu = _Emulation(cfg, [tp.shard_state_dict(full, cfg, r, ws) for r in range(ws)], B, n + steps + 8, n, seed=9)
        ref = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
        ref.load_state_dict(full)
        ref.init_cache(B, n + steps + 8)
        _fill_cache(ref, cfg.num_key_value_heads, n, seed=9)
        worst = 0.0
    ids = torch.randint(0, cfg.vocab_size, (B, 1), generator=torch.Generator().manual_seed(1)).to(dev)
    for step in range(steps):
        logits = model.decode_step(ids).clone()
        assert same_on_all_ranks(model.next_tokens), step
        assert same_on_all_ranks(logits), step
        if rank == 0:
            le = emu.step(ids)
            assert torch.equal(logits, le), (step, (logits - le).abs().max().item())
            lr = ref.decode_step(ids)
            d = (logits - lr).abs().max().item()
            worst = max(worst, d / (lr.abs().max().item() + 1e-6))
            assert d <= 2e-2 * lr.abs().max().item() + 2e-2, (step, d)
        ids = model.next_tokens.view(B, 1).clone()
    # left-padded generate and a short serve() stream: every rank returns the same tokens
    prompt = torch.randint(0, cfg.vocab_size, (2, 48), generator=torch.Generator().manual_seed(2)).to(dev)
    mask = torch.ones_like(prompt)
    mask[1, :11] = 0
    out = model.generate(prompt, max_new_tokens=10, attention_mask=mask)
    assert same_on_all_ranks(out)
    gen = torch.Generator().manual_seed(3)
    reqs = [(torch.randint(0, cfg.vocab_size, (int(m),), generator=gen), int(k)) for m, k in
            ((30, 5), (45, 9), (12, 3), (40, 12), (25, 6))]
    got = dict(serve(model, reqs, 2, 200))
    assert sorted(got) == list(range(len(reqs)))
    for i in range(len(reqs)):
        assert same_on_all_ranks(got[i].to(dev)), i
    torch.cuda.synchronize()
    dist.barrier()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write(f"{worst:.3e}" if rank == 0 else "ok")
    dist.destroy_process_group()


@pytest.mark.parametrize("ws", [2, 4])
def test_sharded_decode_multi_gpu(tmp_path, ws):
    if torch.cuda.device_count() < ws:
        pytest.skip(f"needs {ws} GPUs")
    worst = spawn_ranks(_tp_worker, ws, tmp_path)
    print(f"[tp] world {ws}: max |logits - unsharded| / max|logits| = {worst}")

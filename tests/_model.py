"""The model-level checks of LlamaForCausalLM_KIVI, shared by the model, padding, serving, sampling and tensor-parallel
tests: the fused cache against the reference's 9-tuple path (TupleBar, packed_parts_equal, tuple_prompt, tuple_steps),
two models that must give the same bits (same_logits), the counting CUDA graph, the small config and request lists, and
the harness that runs one process per rank.  The checks are tested without a GPU in tests/test_model_check_cpu.py,
spawn_ranks by the gloo run of tests/test_dist_cpu.py.

This module imports without CUDA: kivi_b200 is imported inside the functions."""
import os
import socket

import pytest
import torch

from tests._hf import hf_positions

PROMPT_RTOL, PROMPT_ATOL = 2e-2, 2e-2   # prompt logits: allclose(rtol, atol)
STEP_REL, STEP_ABS = 3e-2, 3e-2         # a decode step: max|got - ref| <= STEP_REL * max|ref| + STEP_ABS
FLIPS = 3                               # steps in which the argmax may differ
PACKED = (0, 2, 3, 4, 6, 7)             # the packed fields of a 9-tuple: K and V codes, scales and zero points


class TupleBar:
    """The fused path held to the 9-tuple path at one call site (`site`), and what it has seen: the worst d / bar of the
    prompt and of the steps, and the number of steps whose argmax agreed on every compared row."""

    def __init__(self, site):
        self.site, self.worst, self.agree = site, {}, 0

    def prompt(self, got, ref, what="prompt"):
        ratio = ((got - ref).abs() / (PROMPT_ATOL + PROMPT_RTOL * ref.abs())).max().item()
        self.worst["prompt"] = max(self.worst.get("prompt", 0.0), ratio)
        assert torch.allclose(got, ref, rtol=PROMPT_RTOL, atol=PROMPT_ATOL), f"{what}: worst |got - ref| / bar {ratio:.4g}"

    def step(self, got, ref, what):
        d = (got - ref).abs().max().item()
        bar = STEP_REL * ref.abs().max().item() + STEP_ABS
        self.worst["step"] = max(self.worst.get("step", 0.0), d / bar)
        assert d <= bar, f"{what}: max|got - ref| = {d:.4g} > {bar:.4g}"     # False for a NaN or inf d
        self.agree += int((got.argmax(-1) == ref.argmax(-1)).all())

    def report(self):
        worst = ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.worst.items()))
        print(f"\n[{self.site}] worst d / bar: {worst}; argmax agreed in {self.agree} steps")

    def done(self, steps):
        self.report()
        assert self.agree >= steps - FLIPS, f"{self.site}: argmax agreed in {self.agree} of {steps} steps"


def packed_parts_equal(fused, ref, what):
    """The packed fields of two 9-tuples equal (torch.equal, ref's read through view_as of fused's), or both None, and
    kv_seq_len (field 8) equal."""
    for i in PACKED:
        a, b = fused[i], ref[i]
        assert (a is None) == (b is None), f"{what}: tuple[{i}] is None on one side only"
        assert a is None or torch.equal(a, b.view_as(a)), f"{what}: tuple[{i}]"
    assert fused[8] == ref[8], f"{what}: kv_seq_len {fused[8]} != {ref[8]}"


def tuple_prompt(model, ids, bar, mask=None):
    """The prompt through forward() on the 9-tuple path (fused_forward = False; with the left-padding `mask`, transformers'
    positions of it) and through prefill() on the model's cache: last-position logits held to bar.prompt.  Returns the
    9-tuples and the tuple path's first token [B, 1]."""
    model.fused_forward = False
    kw = {} if mask is None else dict(attention_mask=mask, position_ids=hf_positions(mask))
    logits, pasts = model(ids, **kw)
    bar.prompt(model.prefill(ids, attention_mask=mask), logits[:, -1])
    return pasts, logits[:, -1].argmax(-1, keepdim=True)


def tuple_steps(model, pasts, tok, steps, bar, mask=None, row=None):
    """`steps` teacher-forced decode steps: both paths are fed the tuple path's token, and each step's logits are held to
    bar.step.  row None: the whole batch through decode_step(tok), eager in the first two steps; row b: the token goes
    to model._ids[b] and only row b of the fused logits is compared (an inserted request; the other rows continue from
    the step's own feedback).  mask: the tuple path's padding mask, one column appended per step, the positions
    transformers gives it.  Returns the tuple path's 9-tuples."""
    for s in range(steps):
        kw = {}
        if mask is not None:
            mask = torch.cat([mask, mask.new_ones((mask.shape[0], 1))], 1)
            kw = dict(attention_mask=mask, position_ids=hf_positions(mask)[:, -1:])
        lt, pasts = model(tok, pasts, **kw)
        lt = lt[:, -1]
        if row is None:
            lf = model.decode_step(tok, use_graph=s >= 2)
        else:
            model._ids[row] = tok[0, 0]
            lf = model.decode_step(use_graph=s >= 2)[row:row + 1]
        bar.step(lf, lt, f"{bar.site} step {s}")
        tok = lt.argmax(-1, keepdim=True)
    return pasts


def same_logits(a, b, steps, tok=None, graph_a=True, graph_b=True):
    """Twin models decoding the same tokens: logits and next_tokens bit-equal at every step.  tok [B, 1]: the first
    token, then b's next_tokens; None: both models continue from their in-step feedback.  graph_a / graph_b: whether the
    model replays its CUDA graph, a bool or a function of the step number."""
    for s in range(steps):
        la = a.decode_step(tok, use_graph=graph_a(s) if callable(graph_a) else graph_a).clone()
        lb = b.decode_step(tok, use_graph=graph_b(s) if callable(graph_b) else graph_b)
        assert torch.equal(la, lb), f"step {s}: logits"
        assert torch.equal(a.next_tokens, b.next_tokens), f"step {s}: next_tokens"
        if tok is not None:
            tok = b.next_tokens.view(-1, 1).clone()


def world_one_pair(cfg, seed=0):
    """The plain model and the tensor-parallel model at world 1 with the same (seeded) weights."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    torch.manual_seed(seed)
    plain = LlamaForCausalLM_KIVI(cfg).half().cuda().eval()
    tpm = LlamaForCausalLM_KIVI(cfg, tensor_parallel=True).half().cuda().eval()
    tpm.load_state_dict(plain.state_dict())
    assert tpm.tp_world == 1
    return plain, tpm


@pytest.fixture
def graphs(monkeypatch):
    """torch.cuda.CUDAGraph replaced by a subclass that counts the graphs made; returns the subclass (`graphs.made`)."""
    class Counting(torch.cuda.CUDAGraph):
        made = 0

        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            type(self).made += 1
    monkeypatch.setattr(torch.cuda, "CUDAGraph", Counting)
    return Counting


def small_cfg(**kw):
    """The tensor-parallel tests' model: 8 query and 4 KV heads (so 2 and 4 ranks split both), R = g = 32."""
    from kivi_b200.llama_kivi import default_config
    return default_config("tiny", **dict(dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=4,
                                              num_attention_heads=8, num_key_value_heads=4, vocab_size=4096,
                                              residual_length=32, group_size=32), **kw))


PROMPTS = [51, 41, 44, 49, 19, 43, 42, 23]     # with the serving tests' budgets, 3 slots need inserts and shifts


def requests(cfg, budgets, seed=0, params=None, prompts=PROMPTS):
    """serve() requests: (prompt ids, budget) with prompts of the given lengths drawn in order from one seeded generator,
    and params[i] appended where it is not None."""
    g = torch.Generator().manual_seed(seed)
    reqs = [(torch.randint(1, cfg.vocab_size, (n,), generator=g), m) for n, m in zip(prompts, budgets)]
    return reqs if params is None else [r if p is None else r + (p,) for r, p in zip(reqs, params)]


# ------------------------------------------------------------------------------------------------ one process per rank
def _rank_entry(rank, worker, ws, port, out_dir, args):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(ws), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    worker(rank, ws, out_dir, *args)


def spawn_ranks(worker, ws, out_dir, *args):
    """worker(rank, ws, out_dir, *args) in `ws` processes that rendezvous on a free port of 127.0.0.1; each must write
    out_dir/ok{rank}.  Returns rank 0's text."""
    import torch.multiprocessing as mp
    ok = [os.path.join(out_dir, f"ok{r}") for r in range(ws)]
    for path in ok:
        if os.path.exists(path):
            os.remove(path)                                     # left by an earlier run into the same directory
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_rank_entry, args=(worker, ws, port, str(out_dir), args), nprocs=ws, join=True)
    assert all(os.path.exists(path) for path in ok), [os.path.exists(path) for path in ok]
    with open(ok[0]) as f:
        return f.read()


def sharded_model(cfg, rank, ws):
    """In a rank's process: the process group, the rank's GPU, and the tensor-parallel model holding the rank's shard of
    the weights seeded with 0 (the same on every rank).  Returns the model and the full fp16 state dict."""
    from kivi_b200 import dist as kdist, tp
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI
    kdist.init()
    torch.cuda.set_device(torch.device("cuda", rank))
    torch.manual_seed(0)
    full = {k: v.half() for k, v in LlamaForCausalLM_KIVI(cfg).state_dict().items()}
    model = LlamaForCausalLM_KIVI(cfg, tensor_parallel=True)
    model.load_state_dict(tp.shard_state_dict(full, cfg, rank, ws))
    return model.half().cuda().eval(), full


def same_on_all_ranks(t):
    import torch.distributed as dist
    got = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(got, t.contiguous())
    return all(torch.equal(got[0], x) for x in got)

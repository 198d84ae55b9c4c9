"""Greedy sampling kernel (kivi_greedy_sample_exchange_f32): argmax parity with torch on one GPU; with two or more GPUs the
fused argmax + peer-store exchange against an NCCL all-gather of the same ids (one process per GPU, NCCL rendezvous on
127.0.0.1)."""
import os

import pytest
import torch

from tests._model import spawn_ranks

pytestmark = pytest.mark.gpu


def test_greedy_sample_matches_torch_argmax():
    from kivi_b200 import glue
    gen = torch.Generator(device="cuda").manual_seed(0)
    for B, V in ((32, 32000), (3, 128256), (5, 777)):
        logits = torch.randn((B, V), generator=gen, device="cuda", dtype=torch.float16).float()   # fp16-rounded: ties exist
        logits[0, 5] = logits[0, 700 % V] = logits[0].max() + 1                                    # a tie for the maximum
        nxt = torch.full((B,), -1, dtype=torch.long, device="cuda")
        fb = torch.full((B, 1), -1, dtype=torch.long, device="cuda")
        glue.greedy_sample(logits, nxt, fb.view(-1))
        torch.cuda.synchronize()
        assert torch.equal(nxt, fb.view(-1))
        assert int(nxt[0]) == 5                                                                   # first index among equal maxima
        assert torch.equal(logits.gather(1, nxt[:, None]), logits.max(-1, keepdim=True)[0])        # a maximal element
        first = (logits == logits.max(-1, keepdim=True)[0]).float().argmax(-1)                     # index of the first maximum
        assert torch.equal(nxt, first)


def _worker(rank, ws, out_dir):
    import torch.distributed as dist
    from kivi_b200 import dist as kdist, glue
    kdist.init()
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    B, V = 8, 4096
    ex = kdist.PeerTokenExchange(B, dev)
    nxt = torch.zeros(B, dtype=torch.long, device=dev)
    fb = torch.zeros(B, dtype=torch.long, device=dev)
    gen = torch.Generator(device=dev).manual_seed(100 + rank)
    logits = torch.randn((B, V), generator=gen, device=dev)
    g = torch.cuda.CUDAGraph()                       # the exchange lives inside a CUDA graph, like the decode step
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ex.step.add_(1)
        glue.greedy_sample(logits, nxt, fb, ex)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        ex.step.add_(1)
        glue.greedy_sample(logits, nxt, fb, ex)
    for it in range(6):
        logits.copy_(torch.randn((B, V), generator=gen, device=dev))
        g.replay()
        got = ex.tokens().clone()
        ref = kdist.gather_tokens(logits.argmax(-1))
        assert torch.equal(got, ref), (rank, it, got, ref)
        assert torch.equal(nxt, logits.argmax(-1)) and torch.equal(fb, nxt)
    torch.cuda.synchronize()
    dist.barrier()
    open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_peer_token_exchange_two_gpus(tmp_path):
    spawn_ranks(_worker, 2, tmp_path)

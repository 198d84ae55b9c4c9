"""N > 1 host logic on CPU: world_size-2 gloo run of the batch sharding + logits all-gather + identical
greedy sampling (the only collective of the design, SURVEY 8e)."""
import os

import torch
import torch.distributed as dist

from tests._model import spawn_ranks


def _worker(rank, ws, out_dir, gb):
    from kivi_b200 import dist as kdist
    r, w, _ = kdist.init(backend="gloo")
    assert (r, w) == (rank, ws)
    lo, hi = kdist.shard_range(gb, rank, ws)
    torch.manual_seed(0)
    full = torch.randn(gb, 37)                                   # what a single process would compute
    local = full[lo:hi].clone()
    toks, mine = kdist.greedy_next_tokens(local, rank, ws, gb)
    assert torch.equal(toks, full.argmax(-1)) and torch.equal(mine, full.argmax(-1)[lo:hi])
    g = kdist.gather_logits(local, gb)
    assert torch.equal(g, full)
    if gb % ws == 0:                                             # the greedy path: only the sampled ids travel
        allt = kdist.gather_tokens(local.argmax(-1))
        assert torch.equal(allt, full.argmax(-1))
        buf = torch.empty(gb, dtype=torch.long)
        assert kdist.gather_tokens(local.argmax(-1), out=buf) is buf and torch.equal(buf, full.argmax(-1))
    m = kdist.max_over_ranks(float(rank + 1))
    assert m == float(ws)
    kdist.barrier()
    torch.save(toks, os.path.join(out_dir, f"toks{rank}.pt"))
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")


def test_dp_sharding_and_logits_allgather_gloo(tmp_path):
    for gb in (8, 7):                                            # even and ragged global batch
        spawn_ranks(_worker, 2, tmp_path, gb)
        a, b = torch.load(tmp_path / "toks0.pt"), torch.load(tmp_path / "toks1.pt")
        assert torch.equal(a, b) and a.numel() == gb


def test_shard_range_partition():
    from kivi_b200.dist import shard_range
    for gb in (1, 7, 32, 256):
        for ws in (1, 2, 4, 8):
            rs = [shard_range(gb, r, ws) for r in range(ws)]
            assert rs[0][0] == 0 and rs[-1][1] == gb
            assert all(rs[i][1] == rs[i + 1][0] for i in range(ws - 1))
            assert max(h - l for l, h in rs) - min(h - l for l, h in rs) <= 1

"""Multi-GPU decode: data-parallel replicas over the batch, one all-gather per step at the sampling point.

Every (b, kv-head) unit of the KIVI hot path is independent (SURVEY 8e), so the batch is sharded in
contiguous ranges, each rank runs the whole model on its shard with NO per-layer collective, and the
only exchange is one all-gather of the final logits [B/N, vocab] at the sampling step (NCCL over
NVLink 5 / NVSwitch on GPUs, gloo on CPU for the tests), followed by identical sampling on every rank.
The reference has nothing here (device_map="auto" layer placement only).
Tensor parallelism (kivi_b200.tp) adds one collective per sharded projection: `PeerAllReduce` below.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def world():
    """(rank, world_size, local_rank) from the torchrun environment (1 process per GPU)."""
    return (int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0)))


def init(backend: str | None = None):
    rank, ws, local = world()
    if ws > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl":
            torch.cuda.set_device(local)
            kw["device_id"] = torch.device("cuda", local)
        dist.init_process_group(backend=backend, rank=rank, world_size=ws, **kw)
    return rank, ws, local


def shard_range(global_batch: int, rank: int, world_size: int):
    """Contiguous batch range [lo, hi) of `rank`; sizes differ by at most one."""
    base, rem = divmod(global_batch, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_logits(local_logits: torch.Tensor, global_batch: int | None = None) -> torch.Tensor:
    """All-gather [B_local, vocab] -> [B_global, vocab] (rank order = batch order)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local_logits
    ws = dist.get_world_size()
    if global_batch is None or global_batch % ws == 0:
        out = torch.empty((ws * local_logits.shape[0],) + local_logits.shape[1:], dtype=local_logits.dtype,
                          device=local_logits.device)
        dist.all_gather_into_tensor(out, local_logits.contiguous())
        return out
    # ragged shards: pad every shard to the largest one, gather, drop the padding
    sizes = [hi - lo for lo, hi in (shard_range(global_batch, r, ws) for r in range(ws))]
    mx = max(sizes)
    padded = torch.zeros((mx,) + local_logits.shape[1:], dtype=local_logits.dtype, device=local_logits.device)
    padded[: local_logits.shape[0]] = local_logits
    out = torch.empty((ws * mx,) + local_logits.shape[1:], dtype=local_logits.dtype, device=local_logits.device)
    dist.all_gather_into_tensor(out, padded)
    return torch.cat([out[r * mx: r * mx + n] for r, n in enumerate(sizes)], 0)


def greedy_next_tokens(local_logits: torch.Tensor, rank: int, world_size: int, global_batch: int):
    """The sampling step: gather the logits of all shards, take the argmax on every rank (identical result),
    return (all tokens [B_global], this rank's tokens [B_local])."""
    full = gather_logits(local_logits, global_batch)
    toks = full.argmax(-1)
    lo, hi = shard_range(global_batch, rank, world_size)
    return toks, toks[lo:hi]


def gather_tokens(local_tokens: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """Greedy sampling needs no logits from the other shards: argmax is local to a sequence, so the exchange shrinks to
    the sampled ids themselves, 8 bytes per sequence (`gather_logits` stays the general path, e.g. for samplers that
    need the whole distribution on one rank).  local_tokens [B_local] int64 -> [B_global] (rank order = batch order,
    equal shards).  `out` may be a preallocated [world_size * B_local] buffer: the call is then allocation-free and
    capturable in a CUDA graph (NCCL all-gathers are)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        if out is not None:
            out.copy_(local_tokens)
            return out
        return local_tokens
    ws = dist.get_world_size()
    if out is None:
        out = torch.empty(ws * local_tokens.numel(), dtype=local_tokens.dtype, device=local_tokens.device)
    dist.all_gather_into_tensor(out, local_tokens.contiguous().view(-1))
    return out


def _symmetric_buffer(words: int, device):
    """This rank's `words` int64 of one symmetric allocation (torch.distributed._symmetric_memory: peer-mapped over NVLink /
    NVSwitch), zeroed on every rank before any returns, so no rank's kernel signals into a buffer that is still being zeroed.
    Returns (buffer, rendezvous handle, int64 device tensor of every rank's buffer address in rank order)."""
    import torch.distributed._symmetric_memory as symm
    buf = symm.empty(words, dtype=torch.int64, device=device)
    buf.zero_()
    handle = symm.rendezvous(buf, dist.group.WORLD)
    ptrs = torch.tensor([int(p) for p in handle.buffer_ptrs], dtype=torch.int64, device=device)
    torch.cuda.synchronize(device)
    dist.barrier()
    return buf, handle, ptrs


class PeerTokenExchange:
    """The token exchange of greedy data-parallel decoding WITHOUT a library collective: every rank owns one symmetric buffer
    (torch.distributed._symmetric_memory: peer-mapped over NVLink / NVSwitch), and the sampling kernel
    (kivi_greedy_sample_exchange_f32) stores its ids straight into every peer's buffer and signals arrival counters -- the
    compute step (argmax) and its collective (all-gather of the ids) are ONE kernel, capturable in the step's CUDA graph.
    Layout per rank: int64 tokens[2][world * B] (double-buffered by step parity) + uint64 arrived[world]."""

    def __init__(self, batch: int, device):
        self.world, self.rank, self.batch = dist.get_world_size(), dist.get_rank(), batch
        self.buf, self.handle, self.peer_ptrs = _symmetric_buffer(2 * self.world * batch + self.world, device)
        self.step = torch.zeros(1, dtype=torch.int32, device=device)      # incremented inside the step, before the kernel
        self.err = torch.zeros(1, dtype=torch.int32, device=device)

    def tokens(self) -> torch.Tensor:
        """[world * B] ids of the last completed step (synchronises: reads the device step counter)."""
        if int(self.err.item()) != 0:
            raise RuntimeError("kivi_b200: the peer token exchange timed out waiting for another rank")
        par = int(self.step.item()) & 1
        return self.buf[par * self.world * self.batch: (par + 1) * self.world * self.batch]


class PeerAllReduce:
    """The per-layer all-reduce of tensor-parallel decoding (kivi_allreduce_add_rmsnorm_f16) WITHOUT a library collective:
    every rank owns one symmetric buffer that its o_proj / down_proj GEMMs write their partial sums into, and the
    residual-add + RMSNorm kernel reads all ranks' partials straight from the peers' buffers over NVLink.
    Layout per rank (include/kivi_b200.h): half partial[2][rows_max][hidden] (call c uses slot c & 1) + uint64 arrived[world].
    `epoch` is the device call counter (advanced by the calls of a step, inside the step's CUDA graph), `err` the time-out
    word of the arrival waits.  With one rank the buffer is ordinary device memory and the kernel reads only it."""

    def __init__(self, rows_max: int, hidden: int, device):
        multi = dist.is_initialized() and dist.get_world_size() > 1
        self.world, self.rank = (dist.get_world_size(), dist.get_rank()) if multi else (1, 0)
        self.rows_max, self.hidden = rows_max, hidden
        slot = rows_max * hidden                                          # halves per slot
        n = (2 * slot * 2 + 8 * self.world + 7) // 8                      # int64 words
        if multi:
            self.buf, self.handle, self.peer_ptrs = _symmetric_buffer(n, device)
        else:
            self.buf = torch.zeros(n, dtype=torch.int64, device=device)
            self.peer_ptrs = torch.tensor([self.buf.data_ptr()], dtype=torch.int64, device=device)
        self._slots = self.buf.view(torch.float16)[: 2 * slot].view(2, rows_max, hidden)
        self.epoch = torch.zeros(1, dtype=torch.int64, device=device)     # call number = epoch + call + 1
        self.err = torch.zeros(1, dtype=torch.int32, device=device)

    def slot(self, call: int, rows: int) -> torch.Tensor:
        """[rows, hidden] fp16 view of this rank's partial-sum slot of call number `call` (what the GEMM writes)."""
        return self._slots[call & 1, :rows]

    def check(self):
        """Raise if a reduction timed out waiting for another rank (synchronises: reads the device error word)."""
        if int(self.err.item()) != 0:
            raise RuntimeError("kivi_b200: the tensor-parallel all-reduce timed out waiting for another rank")


def barrier():
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()


def max_over_ranks(x: float, device=None) -> float:
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=device if device is not None else "cpu")
    if dist.get_backend() == "nccl":
        t = t.to(torch.device("cuda", torch.cuda.current_device()))
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())

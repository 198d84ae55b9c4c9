"""Pre-allocated KIVI cache (all layers of a model) + the fused decode-attention call.

Host-side mirror of the cache policy of LlamaFlashAttention_KIVI.forward (models/llama_kivi.py:314-455):
the reference keeps a per-layer 9-tuple that it regrows with torch.cat every step; here the buffers are
allocated once (sizes from the C ABI), the lengths live in a device int32[8] shared by all layers, and
one CUDA launch per layer does attention + cache update.  `export(layer)` returns the reference's 9-tuple.
A left-padded batch keeps one length for all sequences; `set_kv_start` names each sequence's first real token, and the
attention then skips the padding on the device (kivi_decode_attention_ragged_f16).  The same offsets let one batch row
("slot") take a new sequence while the others decode: `refill` writes a prompt right-aligned to the shared length,
`release` idles a slot, and `shift` drops timeline positions that no live sequence sees any more.
`reorder` makes batch rows copies of other rows on the device (beam search: each beam continues the row it extends).
A cache built with `sliding_window` = W attends, like transformers' Mistral, to the last W positions only
(kivi_decode_attention_window_f16): the packed blocks below the window are not read, and `shift` may drop them.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib


class _CacheStruct(ctypes.Structure):
    """kivi_cache_t of include/kivi_b200.h"""
    _fields_ = [(n, ctypes.c_int32) for n in
                ("batch", "num_heads", "num_kv_heads", "head_dim", "k_bits", "v_bits", "group_size",
                 "residual_length", "k_cap_blocks", "v_cap_blocks", "v_res_cap", "flags")] + \
               [(n, ctypes.c_void_p) for n in ("k_store", "v_store", "k_res", "v_res", "state")]


_BOUND = False


def kv_start_from_mask(attention_mask) -> torch.Tensor:
    """HF padding mask [B, n] (1 = real token) of a LEFT-padded batch -> int32 [B] number of pad tokens in front of each
    sequence (the first visible position), on the mask's device.  Raises ValueError for right padding, holes in the
    middle of a sequence, or a sequence without any real token."""
    m = torch.as_tensor(attention_mask)
    if m.dim() != 2:
        raise ValueError(f"attention_mask must be 2-D [batch, tokens], got shape {tuple(m.shape)}")
    keep = m != 0
    pad = (~keep).sum(1)
    left = torch.arange(m.shape[1], device=m.device)[None, :] >= pad[:, None]
    if not torch.equal(keep, left):
        raise ValueError("attention_mask: left padding is required (zeros only before each sequence's first real token); "
                         "right padding and holes in the middle are not supported")
    if bool((pad == m.shape[1]).any()):
        raise ValueError("attention_mask: every sequence needs at least one real token")
    return pad.to(torch.int32)


def _bind():
    global _BOUND
    if _BOUND:
        return
    P = ctypes.POINTER(_CacheStruct)
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    _lib.bind("kivi_cache_sizes", i32, [i32] * 7 + [ctypes.POINTER(i64)])
    _lib.bind("kivi_cache_prefill_f16", i32, [P, vp, vp, i32, vp])
    _lib.bind("kivi_decode_workspace_bytes", i64, [P, i32])
    _lib.bind("kivi_decode_attention_f16", i32, [P, vp, vp, vp, vp, vp, vp, i64, vp, vp, i64, i32, vp])
    _lib.bind("kivi_decode_attention_ragged_f16", i32, [P, vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, i64, i32, vp])
    _lib.bind("kivi_decode_attention_window_f16", i32, [P, vp, vp, vp, vp, i32, vp, vp, vp, i64, vp, vp, i64, i32, vp])
    _lib.bind("kivi_cache_advance", i32, [P, vp])
    _lib.bind("kivi_cache_export_f16", i32, [P, i32, i32, i32, i32, i32] + [vp] * 9)
    _lib.bind("kivi_cache_import_f16", i32, [P, i32, i32, i32, i32] + [vp] * 9)
    _lib.bind("kivi_cache_read_state", i32, [P, ctypes.POINTER(ctypes.c_int32), vp])
    _lib.bind("kivi_cache_refill_f16", i32, [P, i32, vp, vp] + [i32] * 6 + [vp])
    _lib.bind("kivi_cache_shift_f16", i32, [P, i32, i32, i32, vp])
    _lib.bind("kivi_cache_shift_state", i32, [P, i32, vp, vp])
    _lib.bind("kivi_cache_reorder_scratch_bytes", i64, [P])
    _lib.bind("kivi_cache_reorder_f16", i32, [P, vp, vp, i64, vp])
    _BOUND = True


IDLE_START = 1 << 30        # kv_start of a released slot: beyond any length, so it attends to its new token only


class KiviCache:
    """KV cache of `n_layers` attention layers: packed K/V stores + fp16 windows, fixed capacity."""

    def __init__(self, n_layers: int, batch: int, num_heads: int, num_kv_heads: int, head_dim: int = 128,
                 k_bits: int = 2, v_bits: int = 2, group_size: int = 32, residual_length: int = 128,
                 max_tokens: int = 4096, device="cuda", overlap_prologue: bool = False, gqa_chunk: int = 0,
                 sliding_window: int | None = None):
        """sliding_window = W: every step attends to the positions max(kv_start, T - W) .. T - 1 only (T = the length
        including the new token; transformers' kv_idx > q_idx - W); None = the whole cache.
        overlap_prologue = KIVI_CACHE_OVERLAP_PROLOGUE of include/kivi_b200.h: promise that the kernel enqueued directly
        before every decode_attention() call never writes this cache (true inside a decoder layer, where it produces
        q / k_new / v_new), so the q.K^T launch may overlap its tail.
        gqa_chunk = KIVI_CACHE_GQA_CHUNK: query heads of a KV head that share one work unit (0 = from the geometry)."""
        _bind()
        if head_dim != 128:
            raise NotImplementedError("kivi_b200 fused decode supports head_dim 128 (all models the reference ships)")
        assert residual_length % group_size == 0                     # models/llama_kivi.py:344
        if sliding_window is not None and int(sliding_window) < 1:
            raise ValueError(f"sliding_window must be a positive number of tokens or None, got {sliding_window}")
        self.sliding_window = None if sliding_window is None else int(sliding_window)
        self.device = torch.device(device)
        _lib.require_cuda(torch.empty(0, device=self.device))
        self.n_layers, self.batch, self.num_heads, self.num_kv_heads = n_layers, batch, num_heads, num_kv_heads
        self.head_dim, self.k_bits, self.v_bits = head_dim, k_bits, v_bits
        self.group_size, self.residual_length, self.max_tokens = group_size, residual_length, max_tokens
        self.tensor_parallel = False      # set by a tensor-parallel model: the heads are one rank's share of the model's heads
        sizes = (ctypes.c_int64 * 8)()
        _lib.check(_lib.lib().kivi_cache_sizes(batch, num_kv_heads, k_bits, v_bits, group_size, residual_length,
                                               max_tokens, sizes), "kivi_cache_sizes")
        self.k_cap_blocks, self.v_cap_blocks, self.v_res_cap = int(sizes[0]), int(sizes[1]), int(sizes[2])
        self._bytes = [int(s) for s in sizes[3:7]]                    # k_store, v_store, k_res, v_res
        self.state = torch.zeros(8, dtype=torch.int32, device=self.device)
        self._bufs, self._structs = [], []
        for _ in range(n_layers):
            bufs = [torch.zeros(nb, dtype=torch.uint8, device=self.device) for nb in self._bytes]
            st = _CacheStruct(batch, num_heads, num_kv_heads, head_dim, k_bits, v_bits, group_size, residual_length,
                              self.k_cap_blocks, self.v_cap_blocks, self.v_res_cap,
                              (1 if overlap_prologue else 0) | (int(gqa_chunk) << 4),
                              *[b.data_ptr() for b in bufs], self.state.data_ptr())
            self._bufs.append(bufs)
            self._structs.append(st)
        # scratch of the decode attention (logits rows, softmax statistics, partial records, arrival counters):
        # one zero-initialised buffer shared by all layers (they run one after the other on the stream)
        nws = int(_lib.lib().kivi_decode_workspace_bytes(ctypes.byref(self._structs[0]), max_tokens))
        if nws < 0:
            _lib.check(nws, "kivi_decode_workspace_bytes")
        self._ws = torch.zeros(nws, dtype=torch.uint8, device=self.device)
        # left padding: first visible position of every sequence (device-resident, so a captured step reads the current
        # values); used only while `ragged` is set, otherwise the unpadded entry runs
        self.kv_start = torch.zeros(batch, dtype=torch.int32, device=self.device)
        self.kv_start_host = [0] * batch                             # host mirror of kv_start (valid while `ragged`)
        self.ragged = False
        # reorder(): the row map, device-resident so that a captured reorder reads the map written before each replay, and
        # the staging scratch (allocated on the first reorder)
        self.reorder_src = torch.arange(batch, dtype=torch.int32, device=self.device)
        self._reorder_scratch = None
        self.adapter_idx = None         # a model's per-row LoRA adapter slots (int32 [batch]), gathered by reorder()
        # host mirror of `state` (its evolution is deterministic)
        self.tk = self.r = self.tv = self.L = self.vhead = self.kv_len = 0

    # ------------------------------------------------------------------ bookkeeping
    def nbytes(self) -> int:
        return self.n_layers * sum(self._bytes)

    def _mirror_prefill(self, n: int):
        R = self.residual_length
        nqk = (0 if n < R else n - n % R) if n % R != 0 else n       # models/llama_kivi.py:425-434
        nqv = 0 if n <= R else n - R                                 # :442-449
        self.tk, self.r, self.tv, self.L, self.vhead, self.kv_len = nqk, n - nqk, nqv, n - nqv, 0, n

    def _mirror_advance(self):
        R = self.residual_length
        self.r += 1
        if self.r == R:                                              # :343-356
            self.tk += R
            self.r = 0
        self.L += 1
        if self.L > R:                                               # :386-399
            self.tv += 1
            self.vhead = (self.vhead + 1) % self.v_res_cap
            self.L = R
        self.kv_len += 1

    def set_kv_start(self, kv_start):
        """Mark the batch as left-padded: kv_start [B] = each sequence's first visible position (its number of pad tokens);
        positions before it are excluded from attention.  None = no padding.  The values are copied into the cache's own
        device buffer, so they may change between replays of a captured step."""
        if kv_start is None:
            self.ragged = False                                      # the buffer is not read while the flag is clear
            return
        t = torch.as_tensor(kv_start).reshape(-1)
        if t.numel() != self.batch:
            raise ValueError(f"kv_start needs {self.batch} entries, got {t.numel()}")
        t = t.to(torch.int32)
        self.kv_start.copy_(t)
        self.kv_start_host = [int(x) for x in t.tolist()]
        self.ragged = True

    # ------------------------------------------------------------------ slots (continuous batching)
    def set_seq_start(self, seq: int, start: int):
        """kv_start[seq] = start (one sequence's first visible position) and turn the ragged entry on; the other
        sequences keep their starts (0 if the batch was not padded)."""
        if not 0 <= seq < self.batch:
            raise ValueError(f"sequence {seq} outside the batch of {self.batch}")
        if not self.ragged:
            self.kv_start.zero_()
            self.kv_start_host = [0] * self.batch
            self.ragged = True
        self.kv_start[seq] = int(start)
        self.kv_start_host[seq] = int(start)

    def release(self, seq: int):
        """Make slot `seq` idle: its start lies beyond every length, so its attention reads no cached byte and returns
        its own new token's V.  Its cache contents stay until a refill overwrites them."""
        self.set_seq_start(seq, IDLE_START)

    def live_starts(self):
        """{seq: start} of the sequences that see part of the cache (start < kv_len).  With a sliding window W the start
        is the effective one of the next step, max(kv_start, kv_len + 1 - W): positions below it are seen by no one."""
        starts = self.kv_start_host if self.ragged else [0] * self.batch
        if self.sliding_window is not None:
            starts = [max(s, self.kv_len + 1 - self.sliding_window) for s in starts]
        return {b: s for b, s in enumerate(starts) if s < self.kv_len}

    def refill(self, layer: int, seq: int, k: torch.Tensor, v: torch.Tensor):
        """Write a new prompt's k, v [Hkv, n, 128] (or [1, Hkv, n, 128]) fp16, K post-RoPE at positions 0 .. n-1, into
        slot `seq` of `layer`, right-aligned to the shared length T (positions T - n .. T - 1; the positions before repeat
        its first token).  The slot then holds what prefill() writes for that T-token sequence; the other slots and the
        lengths do not change.  Call set_seq_start(seq, T - n) once all layers are refilled."""
        _lib.require_cuda(k, v)
        if k.dim() == 4:
            assert k.shape[0] == 1 and v.shape[0] == 1, "refill takes one sequence"
            k, v = k.reshape(k.shape[1:]), v.reshape(v.shape[1:])
        Hkv, n, D = k.shape
        assert (Hkv, D) == (self.num_kv_heads, self.head_dim) and v.shape == k.shape
        assert k.dtype == torch.float16 and v.dtype == torch.float16
        if not 1 <= n <= self.kv_len:
            raise ValueError(f"a prompt of {n} tokens does not fit the shared length {self.kv_len} (1 <= n <= length)")
        k, v = k.contiguous(), v.contiguous()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().kivi_cache_refill_f16(
                ctypes.byref(self._structs[layer]), seq, k.data_ptr(), v.data_ptr(), n, self.tk, self.r, self.tv, self.L,
                self.vhead, _lib.stream_ptr(self.device)), "kivi_cache_refill_f16")

    def shift(self, tokens: int):
        """Drop the first `tokens` positions of the shared timeline in every layer (packed blocks move down; windows stay)
        and lower the lengths and every kv_start by as much.  tokens: a positive multiple of max(128, R), at most tk and tv.
        Raises ValueError if a live sequence would lose a visible position (effective start < tokens, live_starts)."""
        q = max(128, self.residual_length)
        if tokens <= 0 or tokens % q != 0:
            raise ValueError(f"shift must be a positive multiple of {q}, got {tokens}")
        if tokens > self.tk or tokens > self.tv:
            raise ValueError(f"shift {tokens} exceeds the packed lengths (tk {self.tk}, tv {self.tv})")
        low = {b: s for b, s in self.live_starts().items() if s < tokens}
        if low:
            raise ValueError(f"shift {tokens} would drop visible positions of live sequences (starts {low})")
        with torch.cuda.device(self.device):
            stream = _lib.stream_ptr(self.device)
            for layer in range(self.n_layers):
                _lib.check(_lib.lib().kivi_cache_shift_f16(ctypes.byref(self._structs[layer]), tokens, self.tk, self.tv,
                                                           stream), "kivi_cache_shift_f16")
            _lib.check(_lib.lib().kivi_cache_shift_state(ctypes.byref(self._structs[0]), tokens,
                                                         self.kv_start.data_ptr() if self.ragged else None, stream),
                       "kivi_cache_shift_state")
        self.tk, self.tv, self.kv_len = self.tk - tokens, self.tv - tokens, self.kv_len - tokens
        if self.ragged:
            self.kv_start_host = [s - tokens for s in self.kv_start_host]

    # ------------------------------------------------------------------ beam search
    def reorder(self, src):
        """Batch row b of every layer becomes a copy of row src[b] as it was before the call (any map: duplicates, swaps,
        cycles), and so does kv_start[b] while the batch is left-padded.  The lengths do not change.  src: batch ints in
        [0, batch) (a list or a tensor; ValueError otherwise).  The first call allocates a staging scratch of one layer's
        rows at full capacity, i.e. 1 / n_layers of nbytes(), kept for later calls."""
        t = torch.as_tensor(src).reshape(-1)
        if t.numel() != self.batch:
            raise ValueError(f"reorder needs {self.batch} source rows, got {t.numel()}")
        if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
            raise ValueError(f"reorder: source rows must be integers, got {t.dtype}")
        rows = [int(x) for x in t.tolist()]
        bad = [x for x in rows if not 0 <= x < self.batch]
        if bad:
            raise ValueError(f"reorder: source rows {bad} lie outside the batch of {self.batch}")
        self.reorder_src.copy_(torch.tensor(rows, dtype=torch.int32))
        self._enqueue_reorder()
        self._mirror_reorder(rows)

    def reorder_scratch(self) -> torch.Tensor:
        """The staging scratch of reorder(), allocated on first use (before capturing _enqueue_reorder, call this)."""
        if self._reorder_scratch is None:
            nb = int(_lib.lib().kivi_cache_reorder_scratch_bytes(ctypes.byref(self._structs[0])))
            if nb < 0:
                _lib.check(nb, "kivi_cache_reorder_scratch_bytes")
            self._reorder_scratch = torch.empty(nb, dtype=torch.uint8, device=self.device)
        return self._reorder_scratch

    def _enqueue_reorder(self):
        """The device half of reorder(), reading the map in `reorder_src`: two launches per layer and, while `ragged`, the
        kv_start gather.  Capturable in a CUDA graph whose every replay is followed by _mirror_reorder(map)."""
        scratch = self.reorder_scratch()
        with torch.cuda.device(self.device):
            stream = _lib.stream_ptr(self.device)
            for layer in range(self.n_layers):
                _lib.check(_lib.lib().kivi_cache_reorder_f16(ctypes.byref(self._structs[layer]), self.reorder_src.data_ptr(),
                                                             scratch.data_ptr(), scratch.numel(), stream),
                           "kivi_cache_reorder_f16")
            if self.ragged:
                self.kv_start.copy_(self.kv_start.index_select(0, self.reorder_src))
            if self.adapter_idx is not None:
                self.adapter_idx.copy_(self.adapter_idx.index_select(0, self.reorder_src))

    def _mirror_reorder(self, rows):
        if self.ragged:
            self.kv_start_host = [self.kv_start_host[s] for s in rows]

    # ------------------------------------------------------------------ operations
    def prefill(self, layer: int, k: torch.Tensor, v: torch.Tensor, kv_start=None):
        """k, v [B, Hkv, n, 128] fp16 (K post-RoPE): models/llama_kivi.py:425-452 in three launches.  kv_start: see
        set_kv_start (None: the batch is not padded)."""
        _lib.require_cuda(k, v)
        B, Hkv, n, D = k.shape
        assert (B, Hkv, D) == (self.batch, self.num_kv_heads, self.head_dim) and v.shape == k.shape
        assert k.dtype == torch.float16 and v.dtype == torch.float16
        if n > self.max_tokens:
            raise ValueError(f"prompt of {n} tokens exceeds the cache capacity {self.max_tokens}")
        k, v = k.contiguous(), v.contiguous()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().kivi_cache_prefill_f16(ctypes.byref(self._structs[layer]), k.data_ptr(), v.data_ptr(),
                                                         n, _lib.stream_ptr(self.device)), "kivi_cache_prefill_f16")
        self._mirror_prefill(n)
        self.set_kv_start(kv_start)

    def decode_attention(self, layer: int, q: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor,
                         mask: torch.Tensor | None = None, out: torch.Tensor | None = None,
                         dbg_logits: torch.Tensor | None = None, dbg_probs: torch.Tensor | None = None,
                         ):
        """Attention of q [B,H,128] over the cache + k_new/v_new [B,Hkv,128], then the cache update for this
        layer (two launches: q.K^T + statistics, then p.V + output + update).  Call advance() once after the last
        layer of the step."""
        _lib.require_cuda(q, k_new, v_new)
        assert q.shape == (self.batch, self.num_heads, self.head_dim) and q.dtype == torch.float16
        assert k_new.shape == (self.batch, self.num_kv_heads, self.head_dim) and v_new.shape == k_new.shape
        assert q.is_contiguous() and k_new.is_contiguous() and v_new.is_contiguous()
        if self.kv_len + 1 > self.max_tokens:
            raise ValueError("KIVI cache capacity exceeded")
        if out is None:
            out = torch.empty_like(q)
        if mask is not None:
            mask = mask.reshape(self.batch, -1).to(torch.float16).contiguous()
            assert mask.shape[1] == self.kv_len + 1
        stride = 0
        for d in (dbg_logits, dbg_probs):
            if d is not None:
                assert d.dtype == torch.float16 and d.is_contiguous() and d.shape[:2] == (self.batch, self.num_heads)
                stride = d.shape[-1]
        args = (mask.data_ptr() if mask is not None else None, out.data_ptr(), self._ws.data_ptr(), self._ws.numel(),
                dbg_logits.data_ptr() if dbg_logits is not None else None,
                dbg_probs.data_ptr() if dbg_probs is not None else None, stride, self.max_tokens, _lib.stream_ptr(self.device))
        with torch.cuda.device(self.device):
            if self.sliding_window is not None:                      # the blocks below the window are skipped
                _lib.check(_lib.lib().kivi_decode_attention_window_f16(
                    ctypes.byref(self._structs[layer]), q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                    self.kv_start.data_ptr() if self.ragged else None, self.sliding_window, *args),
                    "kivi_decode_attention_window_f16")
            elif self.ragged:                                        # left-padded batch: padded blocks are skipped
                _lib.check(_lib.lib().kivi_decode_attention_ragged_f16(
                    ctypes.byref(self._structs[layer]), q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                    self.kv_start.data_ptr(), *args), "kivi_decode_attention_ragged_f16")
            else:
                _lib.check(_lib.lib().kivi_decode_attention_f16(
                    ctypes.byref(self._structs[layer]), q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(), *args),
                    "kivi_decode_attention_f16")
        return out

    def advance(self):
        self._enqueue_advance()
        self._mirror_advance()

    def _enqueue_advance(self):
        """The device half of advance(): one launch, capturable in a CUDA graph whose every replay is followed by
        _mirror_advance()."""
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().kivi_cache_advance(ctypes.byref(self._structs[0]), _lib.stream_ptr(self.device)),
                       "kivi_cache_advance")

    def read_state(self):
        """The device-side `state` words (synchronises the stream); raises if a decode kernel flagged a capacity
        violation (KIVI_STATE_ERR_CAPACITY in state[6]) and checks the host mirror."""
        host = (ctypes.c_int32 * 8)()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().kivi_cache_read_state(ctypes.byref(self._structs[0]), host, _lib.stream_ptr(self.device)),
                       "kivi_cache_read_state")
        st = list(host)
        if st[6] & 4:                                                # KIVI_STATE_ERR_ROWS
            raise RuntimeError(f"kivi_b200: a row reorder refused to run (state error word {st[6]}): a source row lies "
                               f"outside the batch of {self.batch}")
        if st[6] & 2:                                                # KIVI_STATE_ERR_LENGTHS
            raise RuntimeError(f"kivi_b200: a refill or shift refused to run (state error word {st[6]}): the device-side "
                               f"lengths {st[:6]} are not the ones the host passed")
        if st[6] != 0:
            raise RuntimeError(f"kivi_b200: the decode kernels refused to run (state error word {st[6]}): the device-side "
                               f"lengths {st[:6]} exceed the capacity the cache was created with")
        return st

    def _whole_model_only(self, what: str):
        if self.tensor_parallel:
            raise NotImplementedError(f"KiviCache.{what}: the reference's 9-tuples hold every head of a layer; this cache "
                                      "holds one tensor-parallel rank's heads")

    def import_tuple(self, layer: int, past, kv_start=None):
        """Load `layer` from the reference's per-layer 9-tuple (models/llama_kivi.py:454-455), the inverse of
        export(): a cache that was built by the reference's own hook (or by kivi_prefill_tuple /
        kivi_decode_attention_tuple) continues on the fused path.  All layers of a model share one `state`, so every
        layer must be imported from tuples of the same lengths.  kv_start: see set_kv_start."""
        self._whole_model_only("import_tuple")
        kc, kfull, ks, km, vc, vfull, vs, vm, seen = past
        B, Hkv, D, g = self.batch, self.num_kv_heads, self.head_dim, self.group_size
        kf, vf = 32 // self.k_bits, 32 // self.v_bits
        tk = 0 if kc is None else kc.shape[-1] * kf
        r = 0 if kfull is None else kfull.shape[-2]
        tv = 0 if vc is None else vc.shape[-2]
        L = 0 if vfull is None else vfull.shape[-2]
        if tk + r != seen or tv + L != seen:
            raise ValueError(f"inconsistent KIVI cache tuple: tk {tk} + r {r}, tv {tv} + L {L}, kv_seq_len {seen}")
        if seen > self.max_tokens:
            raise ValueError(f"cache tuple of {seen} tokens exceeds the capacity {self.max_tokens}")

        def prep(t, shape, dtype):
            if t is None:
                return None
            _lib.require_cuda(t)
            assert tuple(t.shape) == shape and t.dtype == dtype, (tuple(t.shape), shape, t.dtype)
            return t.contiguous()
        kc = prep(kc, (B, Hkv, D, tk // kf), torch.int32)
        ks, km = prep(ks, (B, Hkv, D, tk // g), torch.float16), prep(km, (B, Hkv, D, tk // g), torch.float16)
        kfull = prep(kfull, (B, Hkv, r, D), torch.float16)
        vc = prep(vc, (B, Hkv, tv, D // vf), torch.int32)
        vs, vm = prep(vs, (B, Hkv, tv, D // g), torch.float16), prep(vm, (B, Hkv, tv, D // g), torch.float16)
        vfull = prep(vfull, (B, Hkv, L, D), torch.float16)
        ptr = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()   # noqa: E731
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().kivi_cache_import_f16(
                ctypes.byref(self._structs[layer]), tk, r, tv, L, ptr(kc), ptr(ks), ptr(km), ptr(kfull),
                ptr(vc), ptr(vs), ptr(vm), ptr(vfull), _lib.stream_ptr(self.device)), "kivi_cache_import_f16")
        self.tk, self.r, self.tv, self.L, self.vhead, self.kv_len = tk, r, tv, L, 0, seen
        self.set_kv_start(kv_start)

    def export(self, layer: int):
        """The reference's per-layer 9-tuple (models/llama_kivi.py:454-455):
        (Kq_code [B,Hkv,128,tk/fpi] | None, K_full [B,Hkv,r,128] | None, K_scale, K_mn,
         Vq_code [B,Hkv,tv,128/fpi] | None, V_full [B,Hkv,L,128], V_scale, V_mn, kv_seq_len)"""
        self._whole_model_only("export")
        B, Hkv, D, g = self.batch, self.num_kv_heads, self.head_dim, self.group_size
        dev = self.device
        kf, vf = 32 // self.k_bits, 32 // self.v_bits
        kc = torch.empty((B, Hkv, D, self.tk // kf), dtype=torch.int32, device=dev)
        ks = torch.empty((B, Hkv, D, self.tk // g), dtype=torch.float16, device=dev)
        km = torch.empty_like(ks)
        kfull = torch.empty((B, Hkv, self.r, D), dtype=torch.float16, device=dev)
        vc = torch.empty((B, Hkv, self.tv, D // vf), dtype=torch.int32, device=dev)
        vs = torch.empty((B, Hkv, self.tv, D // g), dtype=torch.float16, device=dev)
        vm = torch.empty_like(vs)
        vfull = torch.empty((B, Hkv, self.L, D), dtype=torch.float16, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().kivi_cache_export_f16(
                ctypes.byref(self._structs[layer]), self.tk, self.r, self.tv, self.L, self.vhead,
                kc.data_ptr(), ks.data_ptr(), km.data_ptr(), kfull.data_ptr(),
                vc.data_ptr(), vs.data_ptr(), vm.data_ptr(), vfull.data_ptr(), _lib.stream_ptr(dev)),
                "kivi_cache_export_f16")
        return (kc if self.tk > 0 else None, kfull if self.r > 0 else None, ks if self.tk > 0 else None,
                km if self.tk > 0 else None, vc if self.tv > 0 else None, vfull, vs if self.tv > 0 else None,
                vm if self.tv > 0 else None, self.kv_len)

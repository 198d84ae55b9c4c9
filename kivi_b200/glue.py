"""ctypes wrappers of the decode-step glue kernels (csrc/kivi_model.cu): residual-add + RMSNorm,
RoPE + q/k/v split, SiLU*mul (fp16 CUDA tensors), logits processing, greedy and sampled next-token selection and the
log-probabilities of chosen tokens (fp32 logits), and of the prompt
pass's attention (csrc/kivi_prompt.cu); each wrapper checks device, dtype, contiguity and shapes
before the call (ValueError, or RuntimeError for a CPU tensor)."""
from __future__ import annotations

import ctypes
import math

import torch

from . import _lib

_B = False


def _bind():
    global _B
    if _B:
        return
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    _lib.bind("kivi_add_rmsnorm_f16", i32, [vp, vp, vp, vp, i32, i32, ctypes.c_float, vp])
    _lib.bind("kivi_rope_split_f16", i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp])
    _lib.bind("kivi_qk_norm_rope_split_f16", i32,
              [vp, vp, vp, vp, vp, vp, ctypes.c_float, vp, vp, vp, i32, i32, i32, i32, vp])
    _lib.bind("kivi_silu_mul_f16", i32, [vp, vp, i32, i32, vp])
    _lib.bind("kivi_greedy_sample_exchange_f32", i32, [vp, i32, i32, vp, vp, vp, i32, i32, vp, vp, vp])
    _lib.bind("kivi_sample_f32", i32, [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])
    _lib.bind("kivi_allreduce_add_rmsnorm_f16", i32,
              [vp, vp, vp, vp, i32, i32, ctypes.c_float, vp, i32, i32, i32, i32, vp, vp, i32, vp])
    i64 = ctypes.c_int64
    _lib.bind("kivi_logits_process_f32", i32, [vp, vp, i32, i32] + [vp] * 9 + [i32, i64, vp])
    _lib.bind("kivi_logits_record", i32, [vp, i32, i32, vp, vp, vp, vp, i32, vp])
    _lib.bind("kivi_token_logprobs_f32", i32, [vp, i32, i32, vp, i32, vp, vp, vp, vp])
    _lib.bind("kivi_prompt_attention_f16", i32, [vp, vp, vp, vp, i32, i32, i32, i32] + [i64] * 6 + [vp, i32, vp])
    _lib.bind("kivi_prompt_attention_suffix_f16", i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32] + [i64] * 6 +
              [vp, i32, vp])
    _lib.bind("kivi_lora_workspace_bytes", i64, [i32, i32, i32, i32])
    _lib.bind("kivi_lora_shrink_f16", i32, [vp, i32, i32, vp, i32, i32, i32, vp, vp, vp])
    _lib.bind("kivi_lora_expand_f16", i32, [vp, i32, i32, vp, vp, i32, i32, i32, vp, vp, vp, i32, vp])
    _B = True


def _check(name, t, dtype, shape):
    """t is a contiguous CUDA tensor of `dtype` and `shape`; a kernel would otherwise read or write the wrong bytes."""
    _lib.require_cuda(t)
    if t.dtype != dtype:
        raise ValueError(f"{name}: expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: expected a contiguous tensor")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}")


def _check_norm(residual, weight, out, x):
    """The operands of a residual-add + RMSNorm (x may be None); returns (rows, hidden)."""
    if residual.dim() != 2:
        raise ValueError(f"residual: expected [rows, hidden], got shape {tuple(residual.shape)}")
    rows, hidden = residual.shape
    for name, t, shape in (("residual", residual, (rows, hidden)), ("weight", weight, (hidden,)), ("out", out, (rows, hidden)),
                           ("x", x, (rows, hidden))):
        if t is not None:
            _check(name, t, torch.float16, shape)
    return rows, hidden


def add_rmsnorm(x, residual, weight, out, eps: float):
    """residual += x (x may be None); out = weight * fp16(residual * rsqrt(mean(residual^2) + eps))."""
    _bind()
    rows, hidden = _check_norm(residual, weight, out, x)
    _lib.check(_lib.lib().kivi_add_rmsnorm_f16(x.data_ptr() if x is not None else None, residual.data_ptr(),
                                               weight.data_ptr(), out.data_ptr(), rows, hidden, eps,
                                               _lib.stream_ptr(residual.device)), "kivi_add_rmsnorm_f16")
    return out


def allreduce_add_rmsnorm(residual, weight, out, eps: float, ar, call: int = 0, x=None, cluster: int = 0):
    """Tensor-parallel add_rmsnorm: residual += fp16(sum over ranks of fp32 partials, in rank order); out = RMSNorm(residual).
    ar: kivi_b200.dist.PeerAllReduce (or an object with its fields); this rank's partial of call number `call` must already be
    in ar.slot(call, rows).  ar None: one rank, `x` is the whole sum (exactly add_rmsnorm).  cluster: CTAs per row (1, 2, 4,
    8; 0 = the library's default, one) -- the result does not depend on it."""
    _bind()
    rows, hidden = _check_norm(residual, weight, out, x)
    if ar is not None:
        if ar.hidden != hidden or rows > ar.rows_max:
            raise ValueError(f"the all-reduce buffer holds [{ar.rows_max}, {ar.hidden}] rows, got [{rows}, {hidden}]")
        _lib.require_cuda(ar.peer_ptrs, ar.epoch, ar.err)
    _lib.check(_lib.lib().kivi_allreduce_add_rmsnorm_f16(
        x.data_ptr() if x is not None else None, residual.data_ptr(), weight.data_ptr(), out.data_ptr(), rows, hidden, eps,
        ar.peer_ptrs.data_ptr() if ar is not None else None, ar.rank if ar is not None else 0,
        ar.world if ar is not None else 1, ar.rows_max if ar is not None else rows, call,
        ar.epoch.data_ptr() if ar is not None else None, ar.err.data_ptr() if ar is not None else None, cluster,
        _lib.stream_ptr(residual.device)), "kivi_allreduce_add_rmsnorm_f16")
    return out


def rope_split(qkv, cos_table, sin_table, pos, q, k, v, q_norm=None, k_norm=None, eps=None):
    """qkv [B,(H+2Hkv)*128] -> q [B,H,128], k [B,Hkv,128] rotated at position pos[b] (int64), v [B,Hkv,128].
    With q_norm and k_norm (fp16 [128] each, Qwen3's per-head RMSNorm weights) every q and k head is first normalised
    over its 128 channels with epsilon `eps`, as LlamaRMSNorm rounds (kivi_qk_norm_rope_split_f16); one weight alone is a
    ValueError."""
    if (q_norm is None) != (k_norm is None):
        raise ValueError("q_norm and k_norm: expected both or neither")
    _bind()
    if q.dim() != 3 or k.dim() != 3:
        raise ValueError(f"q, k: expected [B, heads, 128], got shapes {tuple(q.shape)}, {tuple(k.shape)}")
    B, H, Hkv = q.shape[0], q.shape[1], k.shape[1]
    f16 = torch.float16
    _check("qkv", qkv, f16, (B, (H + 2 * Hkv) * 128))
    _check("q", q, f16, (B, H, 128))
    _check("k", k, f16, (B, Hkv, 128))
    _check("v", v, f16, (B, Hkv, 128))
    if cos_table.dim() != 2 or cos_table.shape[1] != 128:              # the kernel's rows are 128 wide (head_dim 128)
        raise ValueError(f"cos_table: expected [rows, 128], got shape {tuple(cos_table.shape)}")
    _check("cos_table", cos_table, f16, cos_table.shape)
    _check("sin_table", sin_table, f16, cos_table.shape)
    _lib.require_cuda(pos)
    if pos.dtype != torch.int64 or pos.numel() != B or not pos.is_contiguous():
        raise ValueError(f"pos: expected {B} contiguous int64 positions, got {pos.dtype} of shape {tuple(pos.shape)}")
    if q_norm is None:
        _lib.check(_lib.lib().kivi_rope_split_f16(qkv.data_ptr(), cos_table.data_ptr(), sin_table.data_ptr(),
                                                  pos.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), B, H, Hkv,
                                                  cos_table.shape[0], _lib.stream_ptr(qkv.device)), "kivi_rope_split_f16")
        return
    _check("q_norm", q_norm, f16, (128,))
    _check("k_norm", k_norm, f16, (128,))
    for name, t in (("q_norm", q_norm), ("k_norm", k_norm)):
        if t.device != qkv.device:
            raise ValueError(f"{name}: on {t.device}, qkv on {qkv.device}")
    if eps is None or not math.isfinite(eps) or eps < 0:
        raise ValueError(f"eps: expected a finite number >= 0, got {eps!r}")
    _lib.check(_lib.lib().kivi_qk_norm_rope_split_f16(
        qkv.data_ptr(), cos_table.data_ptr(), sin_table.data_ptr(), pos.data_ptr(), q_norm.data_ptr(), k_norm.data_ptr(),
        float(eps), q.data_ptr(), k.data_ptr(), v.data_ptr(), B, H, Hkv, cos_table.shape[0], _lib.stream_ptr(qkv.device)),
        "kivi_qk_norm_rope_split_f16")


def silu_mul(gate_up, out):
    _bind()
    if out.dim() != 2:
        raise ValueError(f"out: expected [rows, I], got shape {tuple(out.shape)}")
    rows, inter = out.shape
    _check("out", out, torch.float16, (rows, inter))
    _check("gate_up", gate_up, torch.float16, (rows, 2 * inter))
    _lib.check(_lib.lib().kivi_silu_mul_f16(gate_up.data_ptr(), out.data_ptr(), rows, inter,
                                            _lib.stream_ptr(out.device)), "kivi_silu_mul_f16")
    return out


def greedy_sample(logits, next_local, ids_feedback=None, exchange=None):
    """next_local[b] = argmax(logits[b]) (+ copy into ids_feedback); with `exchange` (kivi_b200.dist.PeerTokenExchange) the
    same kernel also stores the ids into every rank's token buffer over NVLink and waits for the other ranks' ids."""
    _bind()
    B, V = logits.shape
    assert logits.dtype == torch.float32 and logits.is_contiguous() and next_local.dtype == torch.int64
    ex = exchange
    _lib.check(_lib.lib().kivi_greedy_sample_exchange_f32(
        logits.data_ptr(), B, V, next_local.data_ptr(), ids_feedback.data_ptr() if ids_feedback is not None else None,
        ex.peer_ptrs.data_ptr() if ex is not None else None, ex.rank if ex is not None else 0, ex.world if ex is not None else 1,
        ex.step.data_ptr() if ex is not None else None, ex.err.data_ptr() if ex is not None else None,
        _lib.stream_ptr(logits.device)), "kivi_greedy_sample_exchange_f32")
    return next_local


def sample(logits, temperature, top_k, top_p, seed, draw, next_local, ids_feedback=None, dbg_u=None, dbg_kept=None):
    """next_local[b] = one draw from logits[b] (fp32 [B, vocab]) after temperature[b] (fp32), top_k[b] (int32) and top_p[b]
    (fp32), with the uniform number Philox4x32-10(seed[b], draw[b]) (int64 tensors holding the uint64 bits); draw[b] += 1.
    temperature[b] == 0 is the greedy id and leaves draw[b] alone.  All operands are device tensors of B elements: the kernel
    reads them, so a captured call follows later changes.  include/kivi_b200.h (kivi_sample_f32) has the exact rules.
    The parameter VALUES are not checked here (that would read the device and break a capture): callers validate them on the
    host before uploading, as choice.sampling_rows does; the kernel takes a row whose temperature is not > 0 as greedy.
    dbg_u (fp32) / dbg_kept (int32): optional outputs, the uniform number and the size of the kept set."""
    _bind()
    if logits.dim() != 2:
        raise ValueError(f"logits: expected [B, vocab], got shape {tuple(logits.shape)}")
    B, V = logits.shape
    _check("logits", logits, torch.float32, (B, V))
    for name, t, dtype in (("temperature", temperature, torch.float32), ("top_k", top_k, torch.int32),
                           ("top_p", top_p, torch.float32), ("seed", seed, torch.int64), ("draw", draw, torch.int64),
                           ("next_local", next_local, torch.int64), ("ids_feedback", ids_feedback, torch.int64),
                           ("dbg_u", dbg_u, torch.float32), ("dbg_kept", dbg_kept, torch.int32)):
        if t is not None:
            _check(name, t, dtype, (B,))
            if t.device != logits.device:
                raise ValueError(f"{name}: on {t.device}, logits on {logits.device}")
    ptr = lambda t: t.data_ptr() if t is not None else None             # noqa: E731
    _lib.check(_lib.lib().kivi_sample_f32(
        logits.data_ptr(), B, V, temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), seed.data_ptr(), draw.data_ptr(),
        next_local.data_ptr(), ptr(ids_feedback), ptr(dbg_u), ptr(dbg_kept), _lib.stream_ptr(logits.device)),
        "kivi_sample_f32")
    return next_local


def _check_state(B, V, device, counts, n_new, finished, eos, seen=None):
    """The per-row processing state of B rows of a vocabulary of V tokens, on `device`; returns the number of EOS ids."""
    for name, t, dtype, shape in (("counts", counts, torch.int32, (B, V)), ("n_new", n_new, torch.int32, (B,)),
                                  ("finished", finished, torch.uint8, (B,)),
                                  ("seen", seen, torch.int32, (B, (V + 31) // 32))):
        if t is not None:
            _check(name, t, dtype, shape)
            if t.device != device:
                raise ValueError(f"{name}: on {t.device}, expected {device}")
    if eos is None:
        return 0
    if eos.dim() != 1 or eos.numel() > 8:
        raise ValueError(f"eos: expected at most 8 ids in a 1-D tensor, got shape {tuple(eos.shape)}")
    _check("eos", eos, torch.int64, eos.shape)
    if eos.device != device:
        raise ValueError(f"eos: on {eos.device}, expected {device}")
    return eos.numel()


def logits_process(logits, scores, counts, seen, n_new, finished, repetition, presence, frequency, min_new, eos, pad_id: int):
    """scores = logits (fp32 [B, vocab]) after the repetition penalty over the prompt bits `seen` (int32 [B, ceil(vocab / 32)]
    holding the uint32 words) and the generated `counts` (int32 [B, vocab]), the frequency and presence penalties, EOS
    suppression while n_new[b] < min_new[b], and the masking of `finished` rows to pad_id; include/kivi_b200.h
    (kivi_logits_process_f32) has the exact rules.  repetition / presence / frequency fp32 [B], min_new / n_new int32 [B],
    finished uint8 [B], eos int64 [<= 8] or None.  The kernel reads every state and parameter on the device, so a captured
    call follows later changes; the parameter VALUES are checked on the host by choice.processing_rows."""
    _bind()
    if logits.dim() != 2:
        raise ValueError(f"logits: expected [B, vocab], got shape {tuple(logits.shape)}")
    B, V = logits.shape
    _check("logits", logits, torch.float32, (B, V))
    _check("scores", scores, torch.float32, (B, V))
    if scores.data_ptr() == logits.data_ptr():
        raise ValueError("scores: expected a buffer distinct from logits")
    n_eos = _check_state(B, V, logits.device, counts, n_new, finished, eos, seen)
    for name, t, dtype in (("repetition", repetition, torch.float32), ("presence", presence, torch.float32),
                           ("frequency", frequency, torch.float32), ("min_new", min_new, torch.int32)):
        _check(name, t, dtype, (B,))
        if t.device != logits.device:
            raise ValueError(f"{name}: on {t.device}, logits on {logits.device}")
    if not 0 <= int(pad_id) < V:
        raise ValueError(f"pad_id {pad_id} outside the vocabulary of {V}")
    _lib.check(_lib.lib().kivi_logits_process_f32(
        logits.data_ptr(), scores.data_ptr(), B, V, counts.data_ptr(), seen.data_ptr(), n_new.data_ptr(), finished.data_ptr(),
        repetition.data_ptr(), presence.data_ptr(), frequency.data_ptr(), min_new.data_ptr(),
        eos.data_ptr() if n_eos else None, n_eos, int(pad_id), _lib.stream_ptr(logits.device)), "kivi_logits_process_f32")
    return scores


def logits_record(tokens, counts, n_new, finished, eos):
    """After the token choice: counts[b, tokens[b]] += 1, n_new[b] += 1, finished[b] = 1 when tokens[b] is one of `eos`
    (int64 [<= 8] or None).  tokens int64 [B]; the state as in logits_process (kivi_logits_record)."""
    _bind()
    if counts.dim() != 2:
        raise ValueError(f"counts: expected [B, vocab], got shape {tuple(counts.shape)}")
    B, V = counts.shape
    _check("tokens", tokens, torch.int64, (B,))
    n_eos = _check_state(B, V, tokens.device, counts, n_new, finished, eos)
    _lib.check(_lib.lib().kivi_logits_record(
        tokens.data_ptr(), B, V, counts.data_ptr(), n_new.data_ptr(), finished.data_ptr(), eos.data_ptr() if n_eos else None,
        n_eos, _lib.stream_ptr(tokens.device)), "kivi_logits_record")


MAX_TOP_LOGPROBS = 20


def token_logprobs(logits, tokens, logprob, top_ids=None, top_logprobs=None):
    """logprob[b] = log_softmax(logits[b])[tokens[b]] (NaN for an id outside the vocabulary) and, with N = top_ids.shape[1]
    (0 <= N <= 20), the row's N most likely ids in top_ids[b] (descending, ties by ascending id) and their log-probabilities
    in top_logprobs[b].  logits fp32 [B, vocab], tokens int64 [B], logprob fp32 [B], top_ids int64 [B, N], top_logprobs fp32
    [B, N] (both None for N = 0); include/kivi_b200.h (kivi_token_logprobs_f32) has the rules for NaN and infinities and
    the error bound.  One launch, nothing allocated: a captured call reads new logits and tokens on every replay."""
    _bind()
    if logits.dim() != 2:
        raise ValueError(f"logits: expected [B, vocab], got shape {tuple(logits.shape)}")
    B, V = logits.shape
    _check("logits", logits, torch.float32, (B, V))
    if (top_ids is None) != (top_logprobs is None):
        raise ValueError("top_ids and top_logprobs: expected both or neither")
    N = 0
    if top_ids is not None:
        if top_ids.dim() != 2:
            raise ValueError(f"top_ids: expected [B, N], got shape {tuple(top_ids.shape)}")
        N = top_ids.shape[1]
        if not 0 <= N <= MAX_TOP_LOGPROBS:
            raise ValueError(f"top_ids: expected at most {MAX_TOP_LOGPROBS} columns, got {N}")
    for name, t, dtype, shape in (("tokens", tokens, torch.int64, (B,)), ("logprob", logprob, torch.float32, (B,)),
                                  ("top_ids", top_ids, torch.int64, (B, N)),
                                  ("top_logprobs", top_logprobs, torch.float32, (B, N))):
        if t is not None:
            _check(name, t, dtype, shape)
            if t.device != logits.device:
                raise ValueError(f"{name}: on {t.device}, logits on {logits.device}")
    ptr = lambda t: t.data_ptr() if t is not None else None             # noqa: E731
    _lib.check(_lib.lib().kivi_token_logprobs_f32(
        logits.data_ptr(), B, V, tokens.data_ptr(), N, logprob.data_ptr(), ptr(top_ids), ptr(top_logprobs),
        _lib.stream_ptr(logits.device)), "kivi_token_logprobs_f32")
    return logprob


def lora_workspace_bytes(rows: int, in_features: int, n_seg: int, rank: int) -> int:
    """The fp32 workspace of lora_apply (kivi_lora_workspace_bytes); ValueError for shapes the kernels refuse."""
    _bind()
    n = int(_lib.lib().kivi_lora_workspace_bytes(rows, in_features, n_seg, rank))
    if n < 0:
        raise ValueError(f"LoRA kernels: unsupported shape rows={rows} in={in_features} n_seg={n_seg} rank={rank}")
    return n


def lora_apply(x, y, A, B, scale, seg_off, idx, ws):
    """y[b] += the LoRA delta of row b's adapter idx[b] (kivi_lora_shrink_f16 then kivi_lora_expand_f16, two launches):
    x fp16 [rows, in], y fp16 [rows, out] (in place), A fp16 [S, n_seg, R, in], B fp16 [S, out, R], scale fp32 [S],
    seg_off the segments' first columns (a host sequence of n_seg + 1 ints, read now), idx int32 [rows] (a row with
    idx < 0 or >= S is not written), ws fp32 of at least lora_workspace_bytes.  include/kivi_b200.h has the arithmetic
    and the error bound.  Nothing allocated: a captured call reads new x, idx and weights on every replay."""
    _bind()
    if x.dim() != 2 or y.dim() != 2 or A.dim() != 4 or B.dim() != 3:
        raise ValueError(f"lora_apply: expected x [rows, in], y [rows, out], A [S, n_seg, R, in], B [S, out, R]; got "
                         f"{tuple(x.shape)}, {tuple(y.shape)}, {tuple(A.shape)}, {tuple(B.shape)}")
    rows, n_in = x.shape
    S, n_seg, R, _ = A.shape
    out = y.shape[1]
    for name, t, dtype, shape in (("x", x, torch.float16, (rows, n_in)), ("y", y, torch.float16, (rows, out)),
                                  ("A", A, torch.float16, (S, n_seg, R, n_in)), ("B", B, torch.float16, (S, out, R)),
                                  ("scale", scale, torch.float32, (S,)), ("idx", idx, torch.int32, (rows,))):
        _check(name, t, dtype, shape)
        if t.device != x.device:
            raise ValueError(f"{name}: on {t.device}, x on {x.device}")
    _check("ws", ws, torch.float32, ws.shape)
    if ws.numel() * 4 < lora_workspace_bytes(rows, n_in, n_seg, R) or ws.device != x.device:
        raise ValueError("ws: smaller than lora_workspace_bytes or on another device")
    if len(seg_off) != n_seg + 1:
        raise ValueError(f"seg_off: expected {n_seg + 1} offsets, got {len(seg_off)}")
    segs = (ctypes.c_int * (n_seg + 1))(*[int(v) for v in seg_off])
    stream = _lib.stream_ptr(x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().kivi_lora_shrink_f16(x.data_ptr(), rows, n_in, A.data_ptr(), S, n_seg, R, idx.data_ptr(),
                                                   ws.data_ptr(), stream), "kivi_lora_shrink_f16")
        _lib.check(_lib.lib().kivi_lora_expand_f16(ws.data_ptr(), rows, n_in, B.data_ptr(), scale.data_ptr(), S, n_seg, R,
                                                   segs, idx.data_ptr(), y.data_ptr(), out, stream), "kivi_lora_expand_f16")
    return y


def _prompt_operands(q, k, v, out, kv_start):
    """The checks and strides shared by the prompt-attention entries -> (B, H, Hkv, m, n, q strides, k / v strides)."""
    _bind()
    _lib.require_cuda(q, k, v, out, kv_start)
    for name, t in (("q", q), ("k", k), ("v", v)):
        if t.dtype != torch.float16:
            raise ValueError(f"{name}: expected torch.float16, got {t.dtype}")
        if t.dim() != 4 or t.shape[-1] != 128 or t.stride(-1) != 1:
            raise ValueError(f"{name}: expected [B, heads, n, 128] with a contiguous last dimension, got shape "
                             f"{tuple(t.shape)}, strides {t.stride()}")
    B, H, m, _ = q.shape
    Hkv, n = k.shape[1], k.shape[2]
    if k.shape != (B, Hkv, n, 128) or v.shape != k.shape:
        raise ValueError(f"k, v: expected [{B}, Hkv, n, 128] each, got {tuple(k.shape)}, {tuple(v.shape)}")
    # the stride of a dimension of size 1 is never used (its index is 0): 0, so that views differing there agree
    q_str, k_str, v_str = ([0 if t.shape[i] == 1 else t.stride(i) for i in range(3)] for t in (q, k, v))
    if v_str != k_str:
        raise ValueError(f"k, v: expected equal strides, got {k.stride()}, {v.stride()}")
    _check("out", out, torch.float16, (B, m, H, 128))
    if kv_start is not None:
        _check("kv_start", kv_start, torch.int32, (B,))
    for name, t in (("k", k), ("v", v), ("out", out), ("kv_start", kv_start)):
        if t is not None and t.device != q.device:
            raise ValueError(f"{name}: on {t.device}, q on {q.device}")
    return B, H, Hkv, m, n, q_str, k_str


def prompt_attention(q, k, v, out, kv_start=None, window=None):
    """Attention of a prompt over itself (kivi_prompt_attention_f16): q [B, H, n, 128], k / v [B, Hkv, n, 128] fp16 with
    a contiguous head dimension -- the strided [B, heads, n, 128] views of the q / k / v projections -- and k, v of equal
    strides; out [B, n, H, 128] fp16 contiguous.  Query i of sequence b sees the keys max(s_b, i - window + 1) <= j <= i
    with s_b = kv_start[b] (int32 [B] on the device, clamped into [0, n]; None = 0) and window None or 0 = no window.
    A query with no visible key gets zeros.  Returns out."""
    B, H, Hkv, m, n, q_str, k_str = _prompt_operands(q, k, v, out, kv_start)
    if m != n:
        raise ValueError(f"q: expected {n} tokens, as k and v, got {m} (prompt_attention_suffix takes fewer)")
    _lib.check(_lib.lib().kivi_prompt_attention_f16(
        q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, Hkv, n, *q_str, *k_str,
        kv_start.data_ptr() if kv_start is not None else None, int(window or 0), _lib.stream_ptr(q.device)),
        "kivi_prompt_attention_f16")
    return out


def prompt_attention_suffix(q, k, v, out, kv_start=None, window=None):
    """The last m tokens of a prompt over the whole prompt (kivi_prompt_attention_suffix_f16): q [B, H, m, 128] holds the
    queries at positions n - m .. n - 1 of k / v [B, Hkv, n, 128]; out [B, m, H, 128].  Layouts, kv_start and window as
    prompt_attention, whose rows n - m .. n - 1 this returns bit for bit.  1 <= m <= n.  Returns out."""
    B, H, Hkv, m, n, q_str, k_str = _prompt_operands(q, k, v, out, kv_start)
    if not 1 <= m <= n:
        raise ValueError(f"q: expected 1 <= m <= n = {n} tokens, got {m}")
    _lib.check(_lib.lib().kivi_prompt_attention_suffix_f16(
        q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, Hkv, m, n, *q_str, *k_str,
        kv_start.data_ptr() if kv_start is not None else None, int(window or 0), _lib.stream_ptr(q.device)),
        "kivi_prompt_attention_suffix_f16")
    return out

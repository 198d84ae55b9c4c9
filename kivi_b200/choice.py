"""The token choice between lm_head and the next ids, per batch row: logits processing, the greedy or sampled choice and
the log-probabilities of the chosen ids, for the decode step and for its first token alike (TokenChoice.choose)."""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch

from . import glue

SAMPLING_KEYS = ("temperature", "top_k", "top_p", "seed")
PROCESSING_KEYS = ("repetition_penalty", "presence_penalty", "frequency_penalty", "min_new_tokens")
GREEDY = dict(temperature=0.0, top_k=0, top_p=1.0, seed=0)            # a greedy row of a sampling step
NEUTRAL = dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0, min_new_tokens=0)   # no processing


def _sequence(v) -> bool:
    return isinstance(v, (list, tuple)) or (torch.is_tensor(v) and v.dim() > 0)


def _rows(name, v, conv, n=None):
    """v as a list of values converted by conv: a sequence (list, tuple, tensor of dim >= 1) gives its own, which must be n
    (None: any number); a scalar gives n copies (None: one).  A value conv refuses is a ValueError naming `name`."""
    vals = list(v) if _sequence(v) else [v] * (1 if n is None else n)
    if n is not None and len(vals) != n:
        raise ValueError(f"{name}: expected a scalar or {n} values, got {len(vals)}")
    try:
        return [conv(x) for x in vals]
    except (TypeError, OverflowError, ValueError) as e:
        raise ValueError(f"{name}: {e}") from None


def _integer(x):
    if isinstance(x, bool) or int(x) != x:
        raise ValueError(f"expected an integer, got {x!r}")
    return int(x)


def sampling_rows(n: int, temperature=1.0, top_k=50, top_p=1.0, seed=0):
    """The sampling parameters of n batch rows as four lists (temperature, top_k, top_p, seed), from scalars or length-n
    sequences.  An int seed gives row b the Philox key seed + b (mod 2^64); a sequence gives row b its own key.
    temperature >= 0 (0 = greedy), top_k an int (<= 0 = off), 0 <= top_p <= 1; anything else is a ValueError."""
    t, p = _rows("temperature", temperature, float, n), _rows("top_p", top_p, float, n)
    k, sd = _rows("top_k", top_k, _integer, n), _rows("seed", seed, _integer, n)
    if not _sequence(seed):
        sd = [s + b for b, s in enumerate(sd)]
    for b in range(n):
        if not (math.isfinite(t[b]) and t[b] >= 0.0):
            raise ValueError(f"temperature: expected a finite value >= 0 (0 = greedy), got {t[b]}")
        if not 0.0 <= p[b] <= 1.0:
            raise ValueError(f"top_p: expected a value in [0, 1], got {p[b]}")
        if not -2 ** 31 <= k[b] < 2 ** 31:
            raise ValueError(f"top_k: {k[b]} is not an int32")
        if sd[b] < 0:
            raise ValueError(f"seed: expected a non-negative integer, got {sd[b]}")
        sd[b] %= 2 ** 64
    return t, k, p, sd


def processing_rows(n: int, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0, min_new_tokens=0,
                    eos_token_id=None, vocab: int | None = None):
    """The logits-processing parameters of n batch rows as four lists (repetition, presence, frequency, min_new), from
    scalars or length-n sequences, and the EOS ids as a list (an int, a sequence of at most 8, or None = []).
    repetition_penalty > 0 and finite (1 = off), presence_penalty and frequency_penalty in [-2, 2] (0 = off),
    min_new_tokens an int >= 0, EOS ids integers inside [0, vocab) (vocab None: >= 0); anything else is a ValueError."""
    rep, pres = _rows("repetition_penalty", repetition_penalty, float, n), _rows("presence_penalty", presence_penalty, float, n)
    freq, mn = _rows("frequency_penalty", frequency_penalty, float, n), _rows("min_new_tokens", min_new_tokens, _integer, n)
    for b in range(n):
        if not (math.isfinite(rep[b]) and rep[b] > 0.0):
            raise ValueError(f"repetition_penalty: expected a finite value > 0 (1 = off), got {rep[b]}")
        for name, v in (("presence_penalty", pres[b]), ("frequency_penalty", freq[b])):
            if not -2.0 <= v <= 2.0:
                raise ValueError(f"{name}: expected a value in [-2, 2], got {v}")
        if not 0 <= mn[b] < 2 ** 31:
            raise ValueError(f"min_new_tokens: expected an int32 >= 0, got {mn[b]}")
    eos = _rows("eos_token_id", [] if eos_token_id is None else eos_token_id, _integer)
    if len(eos) > 8:
        raise ValueError(f"eos_token_id: at most 8 ids, got {len(eos)}")
    for e in eos:
        if e < 0 or (vocab is not None and e >= vocab):
            raise ValueError(f"eos_token_id: {e} is outside the vocabulary" + (f" [0, {vocab})" if vocab else ""))
    return rep, pres, freq, mn, eos


class TokenChoice:
    """The token choice of the `batch` rows of one cache.  samp: each row's sampling parameters (seed / draw: uint64 bits),
    None when the step takes the argmax; proc: the logits-processing state, None when off; n_top: the top
    log-probabilities (None: off) written into `logprobs`, `top_ids` and `top_logprobs`.  The setters of a mode return
    whether the step's launch sequence changed: the caller drops its captured step then."""

    def __init__(self, batch: int, vocab: int, device):
        self.batch, self.vocab, self.device = batch, vocab, device
        self.samp = self.proc = self.n_top = self.logprobs = self.top_ids = self.top_logprobs = None

    sampling = property(lambda self: self.samp is not None)

    # ------------------------------------------------------------------ sampling
    def set_sampling(self, temperature=1.0, top_k=50, top_p=1.0, seed=0) -> bool:
        was = self.sampling
        if temperature is None:
            self.samp = None
            return was
        rows = sampling_rows(self.batch, temperature, top_k, top_p, seed)
        if not was:                                         # every row is written below
            e = lambda dtype: torch.empty(self.batch, dtype=dtype, device=self.device)    # noqa: E731
            self.samp = SimpleNamespace(temperature=e(torch.float32), top_k=e(torch.int32), top_p=e(torch.float32),
                                        seed=e(torch.long), draw=e(torch.long))
        self._write_sampling(slice(None), *rows)
        return not was

    def set_slot_sampling(self, seq: int, temperature=1.0, top_k=50, top_p=1.0, seed=0):
        if not self.sampling:
            raise RuntimeError("set_slot_sampling: the step is greedy; call set_sampling() first")
        self._write_sampling(self._slot(seq), *sampling_rows(1, temperature, top_k, top_p, seed))

    def _write_sampling(self, rows, t, k, p, sd):
        s, dev = self.samp, self.device
        s.temperature[rows] = torch.tensor(t, dtype=torch.float32).to(dev)
        s.top_k[rows] = torch.tensor(k, dtype=torch.int32).to(dev)
        s.top_p[rows] = torch.tensor(p, dtype=torch.float32).to(dev)
        s.seed[rows] = torch.tensor([x - 2 ** 64 if x >= 2 ** 63 else x for x in sd], dtype=torch.long).to(dev)
        s.draw[rows] = 0

    def sample(self, scores, rows, out, feedback=None):
        """One draw per row of `rows` (a slice) from scores [r, vocab] fp32 with the rows' parameters into out [r] (and
        feedback), consuming the rows' next draw."""
        s = self.samp
        return glue.sample(scores, s.temperature[rows], s.top_k[rows], s.top_p[rows], s.seed[rows], s.draw[rows], out,
                           feedback)

    # ------------------------------------------------------------------ logits processing
    def set_processing(self, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0, min_new_tokens=0,
                       eos_token_id=None, pad_token_id=None) -> bool:
        if repetition_penalty is None:
            changed, self.proc = self.proc is not None, None
            return changed
        B, V, dev = self.batch, self.vocab, self.device
        rep, pres, freq, mn, eos = processing_rows(B, repetition_penalty, presence_penalty, frequency_penalty,
                                                   min_new_tokens, eos_token_id, V)
        pad = pad_token_id if pad_token_id is not None else (eos[0] if eos else 0)
        if isinstance(pad, bool) or int(pad) != pad or not 0 <= int(pad) < V:
            raise ValueError(f"pad_token_id: expected an id inside the vocabulary [0, {V}), got {pad!r}")
        p = self.proc
        if p is None:
            i32 = dict(dtype=torch.int32, device=dev)
            p = self.proc = SimpleNamespace(
                counts=torch.zeros((B, V), **i32), seen=torch.zeros((B, (V + 31) // 32), **i32),
                n_new=torch.zeros(B, **i32), finished=torch.zeros(B, dtype=torch.uint8, device=dev),
                repetition=torch.ones(B, dtype=torch.float32, device=dev),
                presence=torch.zeros(B, dtype=torch.float32, device=dev),
                frequency=torch.zeros(B, dtype=torch.float32, device=dev), min_new=torch.zeros(B, **i32),
                eos=torch.full((8,), -1, dtype=torch.long, device=dev),   # -1 matches no token: a fixed-size list
                scores=torch.empty((B, V), dtype=torch.float32, device=dev), pad=None, stops=False)
        self._write_processing(slice(None), rep, pres, freq, mn)
        p.eos.copy_(torch.tensor(eos + [-1] * (8 - len(eos)), dtype=torch.long).to(dev))
        p.stops = bool(eos)
        changed, p.pad = p.pad != int(pad), int(pad)
        return changed

    def set_slot_processing(self, seq: int, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0,
                            min_new_tokens=0):
        if self.proc is None:
            raise RuntimeError("set_slot_processing: processing is off; call set_processing() first")
        self._write_processing(self._slot(seq), *processing_rows(1, repetition_penalty, presence_penalty,
                                                                frequency_penalty, min_new_tokens)[:4])

    def _write_processing(self, rows, rep, pres, freq, mn):
        p, dev = self.proc, self.device
        p.repetition[rows] = torch.tensor(rep, dtype=torch.float32).to(dev)
        p.presence[rows] = torch.tensor(pres, dtype=torch.float32).to(dev)
        p.frequency[rows] = torch.tensor(freq, dtype=torch.float32).to(dev)
        p.min_new[rows] = torch.tensor(mn, dtype=torch.int32).to(dev)

    def _slot(self, seq: int):
        if not 0 <= seq < self.batch:
            raise ValueError(f"seq {seq} outside the batch of {self.batch}")
        return slice(seq, seq + 1)

    def set_slot(self, seq: int, sampling=None, processing=None):
        """Row `seq` for a new request: its sampling / processing keywords (None: GREEDY / NEUTRAL) for the modes on."""
        if self.sampling:
            self.set_slot_sampling(seq, **(GREEDY if sampling is None else sampling))
        if self.proc is not None:
            self.set_slot_processing(seq, **(NEUTRAL if processing is None else processing))

    def mark_prompt(self, ids, starts, rows, copies: int = 1):
        """Logits processing (nothing when it is off): the prompt ids [r, n] become the prompt bits of the batch rows `rows`
        (a slice of r * copies rows; row j gets prompt j // copies), counting position i of prompt j only when
        i >= starts[j] (None: 0), so left padding is not penalised.  The rows' generated counts, n_new and finished flags
        start from 0."""
        p = self.proc
        if p is None:
            return
        r, n = ids.shape
        words = p.seen.shape[1]
        live = ids.clamp(0, self.vocab - 1)
        if starts is not None:
            pos = torch.arange(n, device=ids.device).view(1, n)
            live = torch.where(pos >= starts.to(ids.device).view(r, 1), live, words * 32)    # a column past the bits
        hit = torch.zeros((r, words * 32 + 1), dtype=torch.bool, device=ids.device)
        hit.scatter_(1, live, True)
        w = (hit[:, :-1].view(r, words, 32).long() << torch.arange(32, device=ids.device)).sum(-1)
        w = torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)                    # the uint32 words' bits
        p.seen[rows] = w.repeat_interleave(copies, 0)
        for t in (p.counts, p.n_new, p.finished):
            t[rows].zero_()

    def release(self, seq: int):
        """Row `seq` made idle: its processing state (prompt bits, counts, length, flag) back to 0."""
        p = self.proc
        if p is not None:
            for t in (p.seen, p.counts, p.n_new, p.finished):
                t[seq].zero_()

    # ------------------------------------------------------------------ log-probabilities
    def set_logprobs(self, n_top=0) -> bool:
        if n_top is not None and (isinstance(n_top, bool) or int(n_top) != n_top or
                                  not 0 <= int(n_top) <= glue.MAX_TOP_LOGPROBS):
            raise ValueError(f"n_top: expected an int in [0, {glue.MAX_TOP_LOGPROBS}], got {n_top!r}")
        n_top = None if n_top is None else int(n_top)
        if n_top == self.n_top:
            return False
        self.n_top = n_top
        if n_top is None:
            self.logprobs = self.top_ids = self.top_logprobs = None
        else:
            B, dev = self.batch, self.device
            self.logprobs = torch.zeros(B, dtype=torch.float32, device=dev)
            self.top_ids = torch.zeros((B, n_top), dtype=torch.long, device=dev)
            self.top_logprobs = torch.zeros((B, n_top), dtype=torch.float32, device=dev)
        return True

    # ------------------------------------------------------------------ the choice
    def choose(self, logits, rows, pick):
        """The ids of the rows `rows` (a slice; None: the decode step's every row, into its static buffers) from their raw
        logits [r, vocab] fp32: processed (proc), chosen by pick(scores), their logprobs (n_top), recorded (proc).
        Returns (what pick returned, the processed scores or None when processing is off)."""
        p, at = self.proc, slice(None) if rows is None else rows
        scores = logits
        if p is not None:
            scores = p.scores if rows is None else torch.empty_like(logits)
            glue.logits_process(logits, scores, p.counts[at], p.seen[at], p.n_new[at], p.finished[at], p.repetition[at],
                                p.presence[at], p.frequency[at], p.min_new[at], p.eos, p.pad)
        chosen = pick(scores)
        tok = chosen.reshape(-1)
        if self.n_top is not None:
            top = self.n_top > 0
            glue.token_logprobs(logits, tok, self.logprobs[at], self.top_ids[at] if top else None,
                                self.top_logprobs[at] if top else None)
        if p is not None:
            glue.logits_record(tok, p.counts[at], p.n_new[at], p.finished[at], p.eos)
        return chosen, None if p is None else scores

    def snapshot(self, *tensors):
        """Copies of `tensors` and of every tensor of the choice a decode step changes: the draw counters when the step
        samples, the counts, lengths and finished flags when it processes."""
        p = self.proc
        live = ([self.samp.draw] if self.sampling else []) + ([p.counts, p.n_new, p.finished] if p is not None else [])
        return [(t, t.clone()) for t in list(tensors) + live]

    @staticmethod
    def restore(saved):
        """Undo the steps run since snapshot() returned `saved`."""
        for t, copy in saved:
            t.copy_(copy)

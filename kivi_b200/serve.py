"""Continuous batching on the fused cache path: a finished sequence's batch row ("slot") takes the next request while the
other sequences keep decoding.

All sequences share one length T (one `state` for the whole batch).  A new prompt of n <= T tokens goes into a free slot
right-aligned, at positions [T - n, T), with kv_start = T - n (LlamaForCausalLM_KIVI.insert -> KiviCache.refill); a
finished slot is released (kv_start beyond every length: it reads no cached byte).  T grows by one per step; positions
that no live sequence sees any more are dropped from the front in multiples of max(128, R) (KiviCache.shift), so the
timeline stays inside the cache.  A request decodes greedily, or samples with its own temperature / top-k / top-p / seed:
the sampling kernel of the step reads each slot's parameters on the device, so both kinds share a batch and one step graph.
A request may also carry a repetition, presence and frequency penalty and a minimum number of new tokens (logits processing
inside the step, LlamaForCausalLM_KIVI.set_processing), read per slot on the device in the same way, and ask for the
log-probabilities of its tokens (`logprobs`, LlamaForCausalLM_KIVI.set_logprobs), computed inside the step as well.
With a PrefixCache (kivi_b200.prefix), an insert whose prompt starts with a stored prefix computes only the rest.
A request may name a loaded LoRA adapter (`adapter`, LlamaForCausalLM_KIVI.load_adapter): its slot's row takes that
adapter's deltas in the step, so requests with different adapters share a batch.
"""
from __future__ import annotations

from collections import deque
from typing import NamedTuple

from types import SimpleNamespace

import torch

from .cache import kv_start_from_mask
from .llama_kivi import PROCESSING_KEYS, processing_rows, sampling_rows

GREEDY = dict(temperature=0.0, top_k=0, top_p=1.0, seed=0)            # the slot parameters of a request without params
SAMPLING_KEYS = ("temperature", "top_k", "top_p", "seed")
NEUTRAL = dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0, min_new_tokens=0)   # no processing
MAX_LOGPROBS = 20


class TokenLogprobs(NamedTuple):
    """The raw log-probabilities of a request's k new tokens, on the host: `token` fp32 [k] of each chosen token, and the
    request's N most likely tokens at each position, `top_ids` int64 [k, N] (descending, ties by ascending id) with their
    log-probabilities `top` fp32 [k, N]."""
    token: torch.Tensor
    top_ids: torch.Tensor
    top: torch.Tensor


def logprobs_param(par):
    """The number of top log-probabilities a request's params ask for (0: the chosen token's only), or None."""
    return None if par is None else par.get("logprobs")


def adapter_param(par):
    """The LoRA adapter a request's params name, or None."""
    return None if par is None else par.get("adapter")


def decoding_params(par):
    """A request's params without `logprobs` and `adapter`, which are not decoding parameters: None (greedy) when those
    were its only keys."""
    if par is None or ("logprobs" not in par and "adapter" not in par):
        return par
    rest = {k: v for k, v in par.items() if k not in ("logprobs", "adapter")}
    return rest or None


def sampling_params(par):
    """The sampling parameters of a request's params: None (greedy) for a request without params or whose params hold
    processing keys only, else its sampling keys (the missing ones take generate(do_sample=True)'s defaults)."""
    if par is None or (not any(k in par for k in SAMPLING_KEYS) and any(k in par for k in PROCESSING_KEYS)):
        return None
    return {k: v for k, v in par.items() if k in SAMPLING_KEYS}


def processing_params(par):
    """The logits-processing parameters of a request's params (None when it has none of the keys)."""
    if par is None or not any(k in par for k in PROCESSING_KEYS):
        return None
    return {k: v for k, v in par.items() if k in PROCESSING_KEYS}


def parse_requests(requests, adapters=()):
    """requests: (prompt ids, max_new_tokens) or (prompt ids, max_new_tokens, params) with params a dict of temperature,
    top_k, top_p, seed (missing keys: 1.0, 50, 1.0, 0, as generate(do_sample=True); the seed is the request's Philox key)
    and of repetition_penalty, presence_penalty, frequency_penalty, min_new_tokens (missing keys: 1.0, 0.0, 0.0, 0;
    processing_rows), and `logprobs`: an int N, 0 <= N <= 20, the number of top log-probabilities wanted with each token.
    `adapter`: the name of a LoRA adapter, one of `adapters` (the model's loaded adapters; None: any string).
    A request whose params hold processing keys, `logprobs` or `adapter` only is greedy.
    Returns ([(prompt int64 1-D on the host, max_new_tokens)], [params or None]); ValueError for an empty prompt, a budget
    below 1, an unknown key or a value outside its range."""
    reqs, params = [], []
    for i, r in enumerate(requests):
        if len(r) not in (2, 3):
            raise ValueError(f"request {i}: expected (prompt, max_new_tokens) or (prompt, max_new_tokens, params)")
        p = torch.as_tensor(r[0]).reshape(-1).to(torch.long).cpu()
        if p.numel() < 1 or int(r[1]) < 1:
            raise ValueError("every request needs at least one prompt token and max_new_tokens >= 1")
        reqs.append((p, int(r[1])))
        par = r[2] if len(r) == 3 else None
        if par is not None:
            unknown = set(par) - set(SAMPLING_KEYS) - set(PROCESSING_KEYS) - {"logprobs", "adapter"}
            if unknown:
                raise ValueError(f"request {i}: unknown sampling parameters {sorted(unknown)}")
            n = par.get("logprobs", 0)
            if isinstance(n, bool) or not isinstance(n, int) or not 0 <= n <= MAX_LOGPROBS:
                raise ValueError(f"request {i}: logprobs: expected an int in [0, {MAX_LOGPROBS}], got {n!r}")
            if "adapter" in par and (not isinstance(par["adapter"], str) or
                                     (adapters is not None and par["adapter"] not in adapters)):
                raise ValueError(f"request {i}: adapter {par['adapter']!r} is not loaded (loaded: {sorted(adapters)})")
            sampling_rows(1, **{k: v for k, v in par.items() if k in SAMPLING_KEYS})   # ValueError outside its range
            processing_rows(1, **{k: v for k, v in par.items() if k in PROCESSING_KEYS})
            par = dict(par)
        params.append(par)
    return reqs, params


def plan_admission(T: int, tv: int, max_tokens: int, quantum: int, live_starts, prompt_len: int, new_tokens: int,
                   longest_pending: int):
    """Whether the next queued request (prompt_len tokens, new_tokens to generate) may enter a running batch whose shared
    length is T (tv of it in the packed V store), and after which shift.  A request fits when prompt_len <= T and
    T + new_tokens <= max_tokens.  If it does not, the timeline may shift by the largest multiple of `quantum` that is at
    most the smallest start of any live sequence (it loses no visible position), at most tv, and leaves T at least the
    longest pending prompt (every later insert still fits under T).
    Returns None when no sequence is live (start the next group with a fresh prefill), else (shift, admit):
    (0, True) fits now, (s, True) fits after shifting s positions, (0, False) wait for a later step."""
    live_starts = list(live_starts)
    if not live_starts:
        return None
    if prompt_len <= T and T + new_tokens <= max_tokens:
        return 0, True
    room = min(min(live_starts), tv, T - longest_pending)
    s = max(room, 0) // quantum * quantum
    if s > 0 and prompt_len <= T - s and T - s + new_tokens <= max_tokens:
        return s, True
    return 0, False


@torch.no_grad()
def serve(model, requests, batch: int, max_tokens: int, eos_token_id=None, use_graph: bool = True,
          stats: dict | None = None, prefix_cache=None):
    """Decoding of a stream of requests with `batch` slots on one cache of `max_tokens` positions.
    requests: a list of (prompt ids 1-D, max_new_tokens), greedy, or (prompt ids, max_new_tokens, params), sampled on the
    device with params = a dict of temperature, top_k, top_p, seed, and of the logits-processing keys repetition_penalty,
    presence_penalty, frequency_penalty, min_new_tokens (parse_requests; min_new_tokens suppresses eos_token_id).  A
    request's tokens depend on its own prompt, parameters and seed only, not on its slot or on the other requests.  When no
    request has sampling parameters the step is the greedy one throughout, and when none has processing keys the step has
    no processing.  serve() sets the model's modes (set_sampling, set_processing) for its requests and leaves them so.
    Yields (index into requests, new token ids [k] int64 on the host) as each request finishes: after max_new_tokens
    tokens, or after an id of eos_token_id (an int or a list; included, as in HF).  When a request of the call has a
    `logprobs` key, every yield is (index, ids, lp) instead: lp is None for a request without the key, else a
    TokenLogprobs of its k tokens with its own N columns -- the raw log-probabilities (before processing, temperature,
    top-k and top-p) that the step computes at the largest N asked for (set_logprobs) and returns under the step's one
    device-to-host read.  `logprobs` never changes a request's tokens.
    The first `batch` requests start with one left-padded prefill, padded to the longest prompt of the whole list, so every
    later prompt fits under the shared length.  Each step is one decode_step (its CUDA graph is captured once: the batch
    is ragged from the start) and one device-to-host read of the sampled ids; finished slots are released and refilled
    from the queue in order.  stats: an optional dict that receives counters (steps, slot_steps = live slots summed over
    the steps, inserts, shifts, shifted_tokens, prefills, prefix_hits, prefix_tokens).
    prefix_cache: a kivi_b200.prefix.PrefixCache, or None.  Every insert reuses the longest prefix of its prompt stored
    there (of at least prefix.MIN_REUSE tokens) and stores the rest of its prompt; stats counts the inserts that reused
    one (prefix_hits) and their reused tokens (prefix_tokens).  The caller owns the cache, so it may outlive the call
    (the next turn of a conversation starts with the previous prompt).  The first group's left-padded prefill neither
    uses nor fills it.
    A request's `adapter` names a LoRA adapter loaded into the model; its prompt pass and its slot's decode steps apply it,
    and a stored prefix is reused only by requests with the same adapter.  An unknown name is a ValueError before any work."""
    reqs, params = parse_requests(requests, adapters=None)
    if not reqs:
        return
    lora = [adapter_param(par) for par in params]
    if any(a is not None for a in lora):                                  # the names, before any work
        parse_requests(requests, model.adapters)
    lp_n = [logprobs_param(par) for par in params]
    params = [decoding_params(par) for par in params]
    samp = [sampling_params(par) for par in params]
    proc = [processing_params(par) for par in params]
    want_lp = any(n is not None for n in lp_n)
    sampling, processing = any(s is not None for s in samp), any(p is not None for p in proc)
    eos = set() if eos_token_id is None else set(torch.as_tensor(eos_token_id).reshape(-1).tolist())
    longest = max(p.numel() for p, _ in reqs)
    for i, (p, m) in enumerate(reqs):
        if longest + m > max_tokens:
            raise ValueError(f"request {i}: the longest prompt ({longest}) + max_new_tokens ({m}) exceeds max_tokens "
                             f"({max_tokens})")
    if stats is None:
        stats = {}
    for key in ("steps", "slot_steps", "inserts", "shifts", "shifted_tokens", "prefills", "prefix_hits", "prefix_tokens"):
        stats.setdefault(key, 0)
    cache = model.cache
    if cache is None or cache.batch != batch or cache.max_tokens != max_tokens:
        cache = model.init_cache(batch, max_tokens)
    loaded = bool(model.adapters)                                         # LoRA: every slot's adapter is set below
    quantum = max(128, cache.residual_length)
    dev = cache.device
    # serve() owns the step's mode: sampling with every slot greedy until a sampled request takes it, or the greedy step
    if sampling:
        model.set_sampling(**GREEDY)
    else:
        model.set_sampling(None)
    # the same for processing: neutral in every slot until a request with processing keys takes it (its scores are then
    # its logits, bit for bit); EOS ends a request on the host (emit), and its slot's state is reset when it is released
    if processing:
        model.set_processing(**NEUTRAL, eos_token_id=eos_token_id)
    else:
        model.set_processing(None)
    if want_lp:
        n_top = max(n for n in lp_n if n is not None)
        model.set_logprobs(n_top)
        host = SimpleNamespace(ids=torch.empty(batch, dtype=torch.long, pin_memory=True),
                               lp=torch.empty(batch, dtype=torch.float32, pin_memory=True),
                               top_ids=torch.empty((batch, n_top), dtype=torch.long, pin_memory=True),
                               top=torch.empty((batch, n_top), dtype=torch.float32, pin_memory=True),
                               done=torch.cuda.Event())
    else:
        model.set_logprobs(None)

    def read(ids):
        """The ids [batch] (device) to the host, with the logprobs buffers when they are on: one synchronisation."""
        if not want_lp:
            return ids.tolist()
        for dst, src in ((host.ids, ids), (host.lp, model.logprobs), (host.top_ids, model.top_ids),
                         (host.top, model.top_logprobs)):
            dst.copy_(src, non_blocking=True)
        host.done.record()
        host.done.synchronize()
        return host.ids.tolist()

    def first_token(logits, slot=None, rows=None):
        """The first token(s) from prompt logits: of slot `slot` (insert) or of the whole batch, whose row b holds request
        rows[b] (prefill); a slot gets its request's parameters and a fresh draw counter here."""
        for b, i in enumerate(rows) if slot is None else [(slot, rows)]:
            if sampling:
                model.set_slot_sampling(b, **(GREEDY if samp[i] is None else samp[i]))
            if processing:
                model.set_slot_processing(b, **(NEUTRAL if proc[i] is None else proc[i]))
        return model.choose_first(logits, slot)

    queue = deque(range(len(reqs)))
    owner = [None] * batch                  # request index decoding in each slot
    outs = [[] for _ in range(batch)]
    lps = [[] for _ in range(batch)]        # the slot's rows of the host logprobs buffers, one per token
    done = []

    def emit(slot, tok):
        """Append a token to the slot's output; finish (release) the slot on EOS or on its token budget."""
        outs[slot].append(tok)
        i = owner[slot]
        if want_lp and lp_n[i] is not None:
            n = lp_n[i]
            lps[slot].append((host.lp[slot].clone(), host.top_ids[slot, :n].clone(), host.top[slot, :n].clone()))
        if tok in eos or len(outs[slot]) >= reqs[i][1]:
            ids = torch.tensor(outs[slot], dtype=torch.long)
            if not want_lp:
                done.append((i, ids))
            elif lp_n[i] is None:
                done.append((i, ids, None))
            else:
                t, top_ids, top = zip(*lps[slot])
                done.append((i, ids, TokenLogprobs(torch.stack(t), torch.stack(top_ids), torch.stack(top))))
            owner[slot], outs[slot], lps[slot] = None, [], []
            model.release(slot)

    def start_group():
        rows = [queue.popleft() for _ in range(min(batch, len(queue)))]
        P = max([reqs[i][0].numel() for i in rows] + [reqs[j][0].numel() for j in queue])
        ids = torch.zeros((batch, P), dtype=torch.long)
        mask = torch.zeros((batch, P), dtype=torch.long)
        mask[:, -1] = 1                                                   # rows without a request: one pad token
        for b, i in enumerate(rows):
            n = reqs[i][0].numel()
            ids[b, P - n:] = reqs[i][0]
            mask[b, P - n:] = 1
        if loaded:
            model.set_adapters([lora[i] for i in rows] + [None] * (batch - len(rows)))
        ids, mask = ids.to(dev), mask.to(dev)
        logits = model.prefill(ids, attention_mask=mask)
        cache.set_kv_start(kv_start_from_mask(mask))                      # ragged from the start: one step graph
        first = first_token(logits, rows=rows)
        model._ids.copy_(first.view(batch, 1))
        first = read(first)
        stats["prefills"] += 1
        for b in range(batch):
            if b < len(rows):
                owner[b] = rows[b]
                emit(b, first[b])
            else:
                model.release(b)

    while queue or any(o is not None for o in owner):
        if all(o is None for o in owner):
            start_group()
        else:
            for slot in range(batch):
                while owner[slot] is None and queue:                      # a slot may finish on its first token
                    p, m = reqs[queue[0]]
                    plan = plan_admission(cache.kv_len, cache.tv, max_tokens, quantum, cache.live_starts().values(),
                                          p.numel(), m, max(reqs[j][0].numel() for j in queue))
                    if plan is None or not plan[1]:
                        break
                    if plan[0]:
                        cache.shift(plan[0])
                        stats["shifts"] += 1
                        stats["shifted_tokens"] += plan[0]
                    i = queue.popleft()
                    if prefix_cache is not None:
                        hits, reused = prefix_cache.hits, prefix_cache.reused_tokens
                    tok = first_token(model.insert(slot, p.to(dev), prefix_cache, adapter=lora[i]), slot, i)
                    if prefix_cache is not None:
                        stats["prefix_hits"] += prefix_cache.hits - hits
                        stats["prefix_tokens"] += prefix_cache.reused_tokens - reused
                    tok = read(tok.view(1).expand(batch))[0] if want_lp else int(tok)
                    model._ids[slot] = tok
                    owner[slot] = i
                    stats["inserts"] += 1
                    emit(slot, tok)
                if not queue:
                    break
        yield from done
        done.clear()
        live = [b for b in range(batch) if owner[b] is not None]
        if not live:
            continue
        model.decode_step(use_graph=use_graph)
        toks = read(model.next_tokens)                                    # the step's one device-to-host read
        stats["steps"] += 1
        stats["slot_steps"] += len(live)
        for b in live:
            emit(b, toks[b])
        yield from done
        done.clear()

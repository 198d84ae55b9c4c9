"""Beam-search bookkeeping: which beams continue and with which tokens, step by step, with the semantics of transformers'
GenerationMixin._beam_search (5.5): log-softmax of fp32 logits added to the running beam scores, the top
max(2, 1 + n_eos) * K candidates over the K * vocab continuations of every prompt, finished hypotheses scored
sum_logprobs / generated_length ** length_penalty, early_stopping True / False / "never", num_return_sequences <= K, and
finished sequences padded with pad_token_id (default: the first EOS id).

A few torch ops on [B, K * vocab] tensors per step, the same on CPU and GPU; the model runs them between its decode-step
and cache-reorder graphs.  Beam sampling, group / diverse beam search, constraints and logits processors are not
supported.
"""
from __future__ import annotations

import torch


def _gather(t, idx):
    """t [B, n, ...] -> t[b, idx[b, j], ...] (transformers' _gather_beams)."""
    while idx.dim() < t.dim():
        idx = idx.unsqueeze(-1)
    return torch.take_along_dim(t, idx, dim=1)


class BeamSearch:
    """The beams of `batch` prompts of `prompt_len` tokens (prompt_ids [batch, prompt_len]), num_beams each, up to
    max_length tokens in all.  step() takes the logits of every beam row b * K + j and returns the rows the next step
    continues; finalize() returns the best num_return_sequences hypotheses of every prompt."""

    def __init__(self, prompt_ids, num_beams: int, max_length: int, eos_token_id=None, pad_token_id=None,
                 length_penalty: float = 1.0, early_stopping=False, num_return_sequences: int = 1):
        B, n = prompt_ids.shape
        K = int(num_beams)
        if K < 1:
            raise ValueError(f"num_beams must be >= 1, got {num_beams}")
        if not 1 <= num_return_sequences <= K:
            raise ValueError(f"num_return_sequences ({num_return_sequences}) must be between 1 and num_beams ({K})")
        if early_stopping not in (True, False, "never"):
            raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
        if max_length <= n:
            raise ValueError(f"max_length ({max_length}) leaves no room after the {n}-token prompt")
        dev = prompt_ids.device
        if eos_token_id is not None:
            eos = torch.as_tensor(eos_token_id, dtype=torch.long).reshape(-1).to(dev)
        else:
            eos = None
        self.B, self.K, self.prompt_len, self.max_length = B, K, n, int(max_length)
        self.eos, self.length_penalty, self.early_stopping = eos, float(length_penalty), early_stopping
        self.num_return_sequences = int(num_return_sequences)
        self.keep = max(2, 1 + (0 if eos is None else eos.numel())) * K
        self.top_mask = torch.arange(self.keep, device=dev) < K
        # transformers: `pad_token_id or eos_token_id[0] if eos_token_id is not None else -1`
        fill = (pad_token_id or int(eos[0])) if eos is not None else -1
        self.running = torch.full((B, K, self.max_length), fill, dtype=torch.long, device=dev)
        self.running[:, :, :n] = prompt_ids[:, None, :]
        self.sequences = self.running.clone()
        self.running_scores = torch.zeros((B, K), dtype=torch.float32, device=dev)
        self.running_scores[:, 1:] = -1e9                    # the first step selects among the continuations of beam 0
        self.scores = torch.full((B, K), -1e9, dtype=torch.float32, device=dev)
        self.finished = torch.zeros((B, K), dtype=torch.bool, device=dev)
        self.improvable = torch.ones((B, 1), dtype=torch.bool, device=dev)
        self.running_idx = torch.full((B, K, self.max_length - n), -1, dtype=torch.int32, device=dev)
        self.beam_indices = self.running_idx.clone()
        self.cur_len = n

    def step(self, logits):
        """logits: fp32 [B * K, vocab] of the rows of the beams, or [B, vocab] of the prompts (the first step: every beam
        of a prompt holds the same prefix).  Returns (beam_idx [B * K] long, tokens [B * K] long, done: a 0-d bool tensor),
        all on the logits' device: row r continues row beam_idx[r] with tokens[r].  After done, call finalize()."""
        B, K, cur = self.B, self.K, self.cur_len
        if logits.shape[0] == B and K > 1:
            logits = logits.repeat_interleave(K, dim=0)
        vocab = logits.shape[-1]
        log_probs = torch.nn.functional.log_softmax(logits.float(), dim=-1).view(B, K, vocab)
        log_probs = (log_probs + self.running_scores[:, :, None]).reshape(B, K * vocab)
        # c. the top `keep` continuations over all beams
        top_lp, top_i = torch.topk(log_probs, k=self.keep)
        top_beam = top_i // vocab
        top_idx = _gather(self.running_idx, top_beam)
        top_seq = _gather(self.running, top_beam)
        top_ids = top_i % vocab
        top_seq[:, :, cur] = top_ids
        top_idx[:, :, cur - self.prompt_len] = (top_beam + torch.arange(B, device=top_i.device).view(-1, 1) * K).to(torch.int32)
        # d. which continuations stop: EOS, or max_length reached
        hits = torch.full_like(top_ids, cur + 1 >= self.max_length, dtype=torch.bool)
        if self.eos is not None:
            hits = hits | torch.isin(top_ids, self.eos)
        # e. the best K unfinished continuations run on
        run_lp = top_lp + hits.to(torch.float32) * -1.0e9
        nxt = torch.topk(run_lp, k=K)[1]
        self.running = _gather(top_seq, nxt)
        self.running_scores = _gather(run_lp, nxt)
        self.running_idx = _gather(top_idx, nxt)
        # f. finished hypotheses among the top K join the finished set if they beat it
        just = hits & self.top_mask[None, :]
        fin_lp = top_lp / ((cur + 1 - self.prompt_len) ** self.length_penalty)
        full = torch.all(self.finished, dim=-1, keepdim=True) & (self.early_stopping is True)
        fin_lp = fin_lp + full.to(torch.float32) * -1.0e9
        fin_lp = fin_lp + (~self.improvable).to(torch.float32) * -1.0e9
        fin_lp = fin_lp + (~just) * -1.0e9
        m_seq = torch.cat((self.sequences, top_seq), 1)
        m_sc = torch.cat((self.scores, fin_lp), 1)
        m_idx = torch.cat((self.beam_indices, top_idx), 1)
        m_fin = torch.cat((self.finished, just), 1)
        best = torch.topk(m_sc, k=K)[1]
        self.sequences, self.scores = _gather(m_seq, best), _gather(m_sc, best)
        self.beam_indices, self.finished = _gather(m_idx, best), _gather(m_fin, best)
        # g. the rows the next step continues, and whether the search is over
        beam_idx = self.running_idx[..., cur - self.prompt_len].reshape(-1).to(torch.long)
        tokens = self.running[:, :, cur].reshape(-1)
        self.cur_len = cur = cur + 1
        if self.early_stopping == "never" and self.length_penalty > 0.0:
            best_len = self.max_length - self.prompt_len
        else:
            best_len = cur - self.prompt_len
        best_running = self.running_scores[:, :1] / (best_len ** self.length_penalty)
        worst_fin = torch.where(self.finished, torch.min(self.scores, dim=1, keepdim=True)[0], -1.0e9)
        self.improvable = self.improvable & torch.any(best_running > worst_fin, dim=-1, keepdim=True)
        open_beam = ~(torch.all(self.finished) & (self.early_stopping is True))
        done = ~(torch.any(self.improvable) & open_beam & ~torch.all(hits))
        return beam_idx, tokens, done

    def finalize(self):
        """(sequences [B * num_return_sequences, length], sequences_scores [B * num_return_sequences]): the best finished
        hypotheses of every prompt, in descending score, cut to the longest one."""
        n = self.num_return_sequences
        seq = self.sequences[:, :n].reshape(self.B * n, -1)
        sc = self.scores[:, :n].reshape(-1)
        idx = self.beam_indices[:, :n].reshape(self.B * n, -1)
        gen = int((idx + 1).bool().sum(dim=1).max())
        return seq[:, :self.prompt_len + gen], sc

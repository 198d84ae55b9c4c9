"""The float64 reference of kivi_token_logprobs_f32 (include/kivi_b200.h) and the bar its values are held to, shared by the
kernel and model tests; the reference's ranking is checked against torch.topk in tests/test_logprobs_cpu.py."""
import torch


def reference_logprobs(logits, tokens, n):
    """(logprob [B], top_ids [B, n], top [B, n]) of fp32 logits [B, V] on the CPU, in float64: torch.log_softmax, the
    tokens' values (NaN outside [0, V)) and a stable sort by (value descending, id ascending) with every NaN first and
    -0 equal to +0; ids past V are -1 with -inf."""
    x = logits.double().cpu()
    B, V = x.shape
    lp = torch.log_softmax(x, -1)
    t = tokens.long().cpu()
    inside = (t >= 0) & (t < V)
    tok = torch.where(inside, lp.gather(1, t.clamp(0, V - 1).view(B, 1)).view(B), torch.tensor(float("nan"), dtype=x.dtype))
    key = torch.where(torch.isnan(x), torch.tensor(float("inf"), dtype=x.dtype), x)
    rank = torch.isnan(x).long()                                            # NaN above +inf: sort by (NaN, value) desc
    order = torch.argsort(key, dim=-1, descending=True, stable=True)
    order = order.gather(1, torch.argsort(rank.gather(1, order), dim=-1, descending=True, stable=True))
    k = min(n, V)
    ids = torch.full((B, n), -1, dtype=torch.long)
    top = torch.full((B, n), float("-inf"), dtype=x.dtype)
    ids[:, :k] = order[:, :k]
    top[:, :k] = lp.gather(1, order[:, :k])
    return tok, ids, top


def lse_of(logits):
    return torch.logsumexp(logits.double().cpu(), -1)


def within_bar(got, ref, x, lse):
    """|got - ref| <= 1e-5 + 2^-23 (|x| + |lse|) elementwise (x: the logits the values came from, lse: their row's), with
    NaN, +-inf at the same places as the reference.  Returns (ok, worst |got - ref| / bar)."""
    got, ref = got.double().cpu(), ref.double().cpu()
    x, lse = x.double().cpu(), lse.double().cpu().expand_as(ref)
    same_special = torch.equal(torch.isnan(got), torch.isnan(ref)) and torch.equal(torch.isinf(got), torch.isinf(ref))
    if not same_special:
        return False, float("inf")
    fin = torch.isfinite(ref)
    if not fin.any():
        return bool(torch.equal(got[~fin].nan_to_num(), ref[~fin].nan_to_num())), 0.0
    bar = 1e-5 + 2.0 ** -23 * (x[fin].abs() + lse[fin].abs())
    r = ((got[fin] - ref[fin]).abs() / bar).max().item()
    inf_ok = torch.equal(got[torch.isinf(ref)], ref[torch.isinf(ref)])
    return r <= 1.0 and inf_ok, r

"""The torch restatement of the logits processing (kivi_logits_process_f32 / kivi_logits_record, include/kivi_b200.h),
the reference of the kernel tests, and the helpers around it.  It is checked against transformers' processors in
tests/test_logits_process_cpu.py.  Every step is one fp32 torch operation on the CPU (IEEE, round to nearest, no
contraction), in the kernel's order, so the kernel must give the same bits."""
import torch


def pack_bits(mask):
    """bool [B, V] -> int32 [B, ceil(V / 32)]: bit v & 31 of word v >> 5 (the uint32 words of `seen`)."""
    B, V = mask.shape
    W = (V + 31) // 32
    full = torch.zeros((B, W * 32), dtype=torch.long)
    full[:, :V] = mask.long()
    w = (full.view(B, W, 32) << torch.arange(32)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def unpack_bits(words, V):
    """The inverse of pack_bits: int32 [B, W] -> bool [B, V]."""
    w = words.long() & 0xffffffff
    return ((w.unsqueeze(-1) >> torch.arange(32)) & 1).view(words.shape[0], -1)[:, :V].bool()


def reference_process(logits, counts, seen, n_new, finished, repetition, presence, frequency, min_new, eos, pad):
    """scores of kivi_logits_process_f32, on the CPU.  logits fp32 [B, V]; counts int [B, V]; seen bool [B, V]; n_new,
    min_new int [B]; finished bool [B]; repetition / presence / frequency fp32 [B]; eos a list of ids; pad an id."""
    x = logits.float().clone()
    B, V = x.shape
    c = counts.long()
    p = repetition.float().view(B, 1)
    hit = seen.bool() | (c > 0)
    x = torch.where(hit, torch.where(x < 0, x * p, x / p), x)                       # 1. repetition
    x = x - frequency.float().view(B, 1) * c.float()                                 # 2. frequency ...
    x = torch.where(c > 0, x - presence.float().view(B, 1), x)                       # ... then presence
    ids = torch.tensor([e for e in eos if 0 <= e < V], dtype=torch.long)
    if ids.numel():
        sup = (n_new.long() < min_new.long()).view(B, 1) & torch.isin(torch.arange(V), ids).view(1, V)
        x = torch.where(sup, torch.tensor(float("-inf")), x)                         # 3. EOS below the minimum
    fin = torch.full((V,), float("-inf"))
    fin[pad] = 0.0
    return torch.where(finished.bool().view(B, 1), fin.view(1, V), x)              # 4. finished rows: pad only


def same_bits(a, b):
    """Two fp32 tensors equal bit for bit, every NaN equal to every NaN (a NaN's payload is not part of the contract)."""
    a, b = a.float().cpu(), b.float().cpu()
    nan = torch.isnan(a)
    return bool(torch.equal(nan, torch.isnan(b)) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32)))


def special_logits(B, V, gen):
    """Random fp32 logits [B, V] with +-0, +-inf, NaN and denormals sprinkled in (each in about 1 % of the entries)."""
    x = torch.randn((B, V), generator=gen) * 8
    specials = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -1e-40, 1.4e-45])
    pick = torch.randint(0, 100 * len(specials), (B, V), generator=gen)
    hit = pick < len(specials)
    x[hit] = specials[pick[hit]]
    return x

"""The numpy reference of kivi_sample_f32 (tests/test_sample_gpu.py compares the kernel with it; tests/test_sample_cpu.py
checks it on known answers and hand-made rows): Philox4x32-10 and the row semantics in fp64."""
import numpy as np

M32 = 0xFFFFFFFF


def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., SC11): counter = 4 words, key = 2 words -> 4 words."""
    c0, c1, c2, c3 = counter
    k0, k1 = key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & M32, (p0 >> 32) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
    return c0, c1, c2, c3


def uniform24(seed: int, draw: int) -> int:
    """The 24-bit integer n of the kernel's uniform number u = n * 2^-24 for (seed, draw), both uint64."""
    return philox4x32_10((draw & M32, draw >> 32, 0, 0), (seed & M32, seed >> 32))[0] >> 8


def greedy_id(row) -> int:
    """torch.argmax's rule: the first NaN, else the first maximum."""
    row = np.asarray(row)
    nan = np.isnan(row)
    return int(nan.argmax()) if nan.any() else int(row.argmax())


def reference_row(row, temperature, top_k, top_p):
    """Row semantics in fp64.  Returns None for a row that takes the greedy id (temperature 0, a +inf, no finite logit), else
    (w, margin): w [vocab] fp64 the kept tokens' masses exp(x - max) (0 = not kept), margin the distance of the top-p
    decision from its nearest alternative as a fraction of the mass (inf when top-p is off)."""
    row = np.asarray(row, dtype=np.float32)
    if temperature == 0:
        return None
    with np.errstate(all="ignore"):
        x = (row / np.float32(temperature)).astype(np.float64)          # the fp32 quotient, as the kernel forms it
    x[np.isnan(x)] = -np.inf
    V, mx = x.size, x.max()
    if not np.isfinite(mx):
        return None
    kept = x > -np.inf
    if 0 < top_k < V:
        kept &= x >= np.partition(x, V - top_k)[V - top_k]
    w = np.where(kept, np.exp(x - mx), 0.0)
    margin = np.inf
    if top_p < 1:
        if top_p <= 0:
            thr = mx
        else:
            vals, inv = np.unique(x[kept], return_inverse=True)         # ascending distinct values; ties share a class
            mass = np.bincount(inv, weights=w[kept])[::-1]
            cum, target = np.cumsum(mass), top_p * w.sum()
            j = int(np.argmax(cum >= target)) if (cum >= target).any() else len(cum) - 1
            thr = vals[::-1][j]
            margin = np.abs(cum - target).min() / w.sum()
        w = np.where(x >= thr, w, 0.0)
    return w, margin


def reference_pick(w, n24: int):
    """The inverse CDF in token-id order: (first id whose cumulative mass exceeds u * S, distance of u * S from the nearest
    CDF step as a fraction of S)."""
    cdf = np.cumsum(w)
    S = cdf[-1]
    target = n24 * 2.0 ** -24 * S
    return int(np.argmax(cdf > target)), np.abs(cdf[w > 0] - target).min() / S

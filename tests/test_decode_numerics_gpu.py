"""The fused decode attention against the C oracle away from standard-normal inputs.

Magnitude sweep: the packed blocks are contracted on mma.sync with the B operand x*s split into hi = fp16(x*s) and
lo = fma(x, s, -hi), where x is q (q.K^T) or a scaled probability (p.V) and s a K or V scale.  The split is exact only
while the residual stays clear of the fp16 denormal range, so the kernel's error depends on the magnitudes of q, K, V and
the context length; the reference computes fma(fma(s, c, z), x, acc) in fp32 and does not.  Named regimes, each on its own
seed, at the kernels of the benchmark's configurations and one g = 128 kernel, at about 600, 4096 and 32768 tokens.

Edge values: the cache has three quantisers of its own (the prompt's block prefill, the K flush of the p.V kernel, the V
token pack), each with its own min / max, scale and code assembly.  They get the edge rows of test_pack_edge_values."""
import numpy as np
import pytest
import torch

from oracle import ref
from tests._attn import OUTLIER_CHANNELS, _put_k_edges, _put_v_edges, checked_step, make_cache, rand16, tuple_equal

pytestmark = pytest.mark.gpu

KERNELS = {   # name: k_bits, v_bits, g, R, G, Hkv  (B = 1, H = G * Hkv: the oracle checks every unit)
    "cfg2-k2v2-g32-G1": (2, 2, 32, 128, 1, 2),
    "cfg3-k2v2-g32-G4": (2, 2, 32, 128, 4, 2),
    "cfg4-k4v4-g64-G4": (4, 4, 64, 64, 4, 2),
    "k4v2-g128-G2": (4, 2, 128, 128, 2, 2),
}

REGIMES = {   # name: seed, q std, K std, V std, extras
    "unit": (1, 1.0, 1.0, 1.0, {}),
    "q-2^-6": (2, 2.0 ** -6, 1.0, 1.0, {}),
    "q-2^-3": (3, 2.0 ** -3, 1.0, 1.0, {}),
    "q-8": (4, 8.0, 1.0, 1.0, {}),
    "k-2^-6": (5, 1.0, 2.0 ** -6, 1.0, {}),
    "k-16": (6, 1.0, 16.0, 1.0, {}),
    "k-outliers-x32": (7, 1.0, 1.0, 1.0, {"outliers": 32.0}),
    "v-2^-6": (8, 1.0, 1.0, 2.0 ** -6, {}),
    "v-2^-3": (9, 1.0, 1.0, 2.0 ** -3, {}),
    "v-0.02": (10, 1.0, 1.0, 0.02, {}),
    "qk-1e-2": (11, 1e-2, 1e-2, 1.0, {}),
    "q-zero": (12, 0.0, 1.0, 1.0, {}),                    # every probability is fp16(1 / T)
    "peaked": (13, 1.0, 1.0, 1.0, {"peaked": 4.0}),      # q = 4 k_j: the output is token j's dequantised V row
    "k-64-q-2-finite-logits": (14, 2.0, 64.0, 1.0, {}),  # |logits| in the thousands, still finite in fp16
}
LONG_REGIMES = ["unit", "q-2^-6", "k-2^-6", "v-2^-6", "v-2^-3", "v-0.02", "q-zero", "peaked"]


def _sweep_cases():
    cases = []
    for T in (600, 4096, 32768):
        for kname in KERNELS:
            for rname in (LONG_REGIMES if T == 32768 else REGIMES):
                cases.append(pytest.param(kname, rname, T, id=f"{kname}-{rname}-T{T}"))
    return cases


@pytest.mark.parametrize("kname,rname,T", _sweep_cases())
def test_magnitude_sweep_matches_oracle(kname, rname, T):
    """Prefill T - 1 tokens of the regime, then two decode steps, each fully checked (checked_step: fast == instrumented,
    every stage against the oracle at the suite's bars, end to end, the exported cache bit for bit)."""
    kb, vb, g, R, G, Hkv = KERNELS[kname]
    seed, qs, ks, vs, extra = REGIMES[rname]
    B, H, n0 = 1, G * Hkv, T - 1
    rng = np.random.default_rng(seed * 100003 + T)

    def kv(n):
        k = rng.standard_normal((B, Hkv, n, 128)) * ks
        if "outliers" in extra:
            k[..., OUTLIER_CHANNELS] *= extra["outliers"]
        return k.astype(np.float16), (rng.standard_normal((B, Hkv, n, 128)) * vs).astype(np.float16)

    k, v = kv(n0)
    cache = make_cache(B, H, Hkv, kb, vb, g, R, T + 16, gqa_chunk=G)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    for step in range(2):
        if "peaked" in extra:                        # aligned with a token of the packed K store
            j = (n0 // 3) + step
            q = np.repeat(k[:, :, j:j + 1, :].astype(np.float32) * extra["peaked"], H // Hkv, axis=1).astype(np.float16)
        else:
            q = (rng.standard_normal((B, H, 1, 128)) * qs).astype(np.float16)
        k_new, v_new = kv(1)
        st = checked_step(cache, st, q, k_new, v_new, (g, kb, vb, R))


# ---------------------------------------------------------------------------------------------------
# edge values through the cache's own quantisers
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kb,vb,g,R,n0", [(2, 2, 32, 32, 3 * 128 + 5), (4, 4, 64, 64, 4 * 64 + 5),
                                          (2, 4, 32, 64, 2 * 128 + 5), (4, 2, 128, 128, 3 * 128 + 5)])
def test_edge_values_through_cache_quantisers(kb, vb, g, R, n0):
    """Edge rows in chosen K channels and V tokens of the prompt (block prefill), then again through k_new / v_new over one
    or two K flush periods (the K flush, the V-token pack).  The exported cache equals the oracle's 9-tuple bit for bit
    after every step.  A sequence whose oracle output is finite (finite edge rows only) gets every check of the suite; where
    the oracle's output is not finite (the rows whose scale overflows), the kernel's must be non-finite at exactly the same
    positions, and equal within the end-to-end bar where it is finite."""
    B, H, Hkv = 2, 4, 2
    cfg = (g, kb, vb, R)
    rng = np.random.default_rng(kb * 31 + vb * 7 + g + R)
    k, v = rand16(rng, (B, Hkv, n0, 128)), rand16(rng, (B, Hkv, n0, 128))
    _put_k_edges(k, 0, kb)
    _put_v_edges(v, 0, vb)
    steps = 2 * R - 4 if R <= 64 else R - 4                          # r = 5 -> flushes at r = R - 1
    cache = make_cache(B, H, Hkv, kb, vb, g, R, n0 + steps + 8)
    cache.prefill(0, torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
    st = ref.prefill_cache(k, v, *cfg)
    tuple_equal(cache.export(0), st, "prefill")
    flushes = 0
    for step in range(steps):
        pos = cache.kv_len
        q, k_new, v_new = rand16(rng, (B, H, 1, 128), 0.7), rand16(rng, (B, Hkv, 1, 128)), rand16(rng, (B, Hkv, 1, 128))
        _put_k_edges(k_new, pos, kb)
        _put_v_edges(v_new, pos, vb)
        tk0 = cache.tk
        fin = np.isfinite(ref.decode_step(st, q, k_new, v_new, *cfg)[0])
        assert fin[0].all(), "the finite edge rows must give a finite oracle output"
        assert (~fin[1]).any(), "the overflowing edge rows must reach the output"
        # sequence 0 (finite) through every check of the suite; sequence 1 held to the oracle's non-finite positions
        st = checked_step(cache, st, q, k_new, v_new, cfg, bad=(1,))
        flushes += cache.tk != tk0
    assert flushes == (2 if R <= 64 else 1)

"""The decode step's glue kernels (csrc/kivi_model.cu) against exact references, at the shipped shapes and across value
magnitudes: residual-add + RMSNorm, RoPE + q/k/v split, SiLU*mul and the greedy argmax.  Every logit of
LlamaForCausalLM_KIVI.decode_step passes through them.

References and bars.  The references are numpy, in fp64 or in fp16 arithmetic (numpy rounds every fp16 op correctly);
none uses torch's kernels.  Each kernel is also compared with the HF op chain run by torch on the same device.
* RMSNorm: r64 = f * (mean(f^2) + float32(eps))^-1/2 in fp64, from the fp16 residual the kernel wrote.  With a <= r64 <= b
  the adjacent fp16 values, every finite output equals fp16(w*a) or fp16(w*b): the fp32 statistics may round the inner
  value either way, the weight product must be rounded correctly.  Non-finite positions equal the torch chain's.
* RoPE: bit-identical to x*cos + rotate_half(x)*sin in fp16 arithmetic on the rows cos[clamp(pos)], at every position
  that is not NaN (NaN positions must match); v is an exact copy.
* SiLU*mul: out = fp16(a*u) with a one of the fp16 neighbours of the fp64 silu(g) = g / (1 + e^-g) (NaN for g = -inf,
  as the formula gives in any precision), NaN where that is NaN, and bit-identical to F.silu(gate) * up: both evaluate
  x / (1 + expf(-x)) in fp32 with IEEE division and round once.
* Greedy argmax: the first index of the maximum, a NaN counting as the maximum and the first NaN winning (torch.argmax).

Production wiring: a one-layer model with Llama-3-8B layer shapes decodes a left-padded batch through its CUDA graph, and
each glue stage is checked from the static buffers the graph wrote."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests._util import to_np

pytestmark = pytest.mark.gpu

EPS = 1e-5
TABLE_ROWS = 32768 + 1024                 # default_config's max_position_embeddings


# ---------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------
def f16_neighbours(x):
    """fp16 values a <= x <= b adjacent to the fp64 x (a == b where x is representable; NaN stays NaN)."""
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        r = x.astype(np.float16)
        r64 = r.astype(np.float64)
        a = np.where(r64 > x, np.nextafter(r, np.float16(-np.inf)), r)
        b = np.where(r64 < x, np.nextafter(r, np.float16(np.inf)), r)
    return a, b


def check_rounded_product(got, w, inner64, what):
    """got equals fp16(w*a) or fp16(w*b) (an infinity included) for the fp16 neighbours a, b of inner64, and is NaN
    exactly where w*inner64 is NaN."""
    got = np.asarray(got, np.float16).astype(np.float64)
    a, b = f16_neighbours(inner64)
    w = np.asarray(w, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        ea = (w * a.astype(np.float64)).astype(np.float16).astype(np.float64)   # fp16 x fp16 is exact in fp64: one rounding
        eb = (w * b.astype(np.float64)).astype(np.float16).astype(np.float64)
        ref_nan = np.isnan(w * inner64)
    ok = (got == ea) | (got == eb) | (np.isnan(got) & ref_nan)
    if not ok.all():
        i = np.argwhere(~ok)[0]
        raise AssertionError(f"{what}: {(~ok).sum()} / {ok.size} outputs are neither rounding; first at {tuple(i)}: got "
                             f"{got[tuple(i)]!r}, allowed {ea[tuple(i)]!r} / {eb[tuple(i)]!r} (exact {inner64[tuple(i)]!r})")


def rmsnorm_inner64(res16):
    f = np.asarray(res16, np.float16).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        ms = (f * f).mean(-1, keepdims=True)
        return f / np.sqrt(ms + float(np.float32(EPS)))


def hf_rmsnorm(x, w):
    """transformers' LlamaRMSNorm.forward (the module the reference star-imports), written out."""
    h = x.float()
    h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + EPS)
    return w * h.to(x.dtype)


def check_rmsnorm(out, res16, w16, what):
    """The RMSNorm bar, and the kernel's non-finite positions equal those of the torch chain."""
    out_np = to_np(out)
    check_rounded_product(out_np, to_np(w16), rmsnorm_inner64(to_np(res16)), what)
    with torch.no_grad():
        hf_nf = ~torch.isfinite(hf_rmsnorm(res16, w16)).cpu().numpy()
    got_nf = ~np.isfinite(out_np.astype(np.float64))
    assert (got_nf == hf_nf).all(), f"{what}: non-finite at {got_nf.sum()} positions, torch chain at {hf_nf.sum()}"


def rope_ref(qkv, cos, sin, pos, H, Hkv):
    """apply_rotary_pos_emb in fp16 arithmetic: qkv [B, (H+2Hkv)*128] -> (q, k, v); rows cos[clamp(pos)]."""
    B = qkv.shape[0]
    x = qkv.reshape(B, H + 2 * Hkv, 128)
    p = np.clip(np.asarray(pos, np.int64).reshape(B), 0, cos.shape[0] - 1)
    c, s = cos[p][:, None, :], sin[p][:, None, :]
    qk = x[:, :H + Hkv]
    rot = np.concatenate([-qk[..., 64:], qk[..., :64]], -1)
    with np.errstate(over="ignore", invalid="ignore"):
        out = qk * c + rot * s                                               # every op on float16 arrays rounds to fp16
    return out[:, :H], out[:, H:], x[:, H + Hkv:]


def assert_bits(got, exp, what):
    """Bit-identical fp16 except that NaN (any payload) only has to be NaN at the same positions."""
    got, exp = np.asarray(got, np.float16), np.asarray(exp, np.float16)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    gn, en = np.isnan(got), np.isnan(exp)
    same = (got.view(np.uint16) == exp.view(np.uint16)) | (gn & en)
    assert (gn == en).all(), f"{what}: NaN at {gn.sum()} positions, expected {en.sum()}"
    if not same.all():
        i = tuple(np.argwhere(~same)[0])
        raise AssertionError(f"{what}: {(~same).sum()} / {same.size} differ; first at {i}: got {got[i]!r}, expected {exp[i]!r}")


def silu64(g):
    g = np.asarray(g, np.float16).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        return g / (1.0 + np.exp(-g))


def argmax_ref(x):
    """First index of the row maximum; a NaN counts as the maximum and the first NaN wins."""
    x = np.asarray(x)
    nan = np.isnan(x)
    return np.where(nan.any(-1), nan.argmax(-1), np.where(nan, -np.inf, x).argmax(-1))


# ---------------------------------------------------------------------------------------------------
# residual-add + RMSNorm
# ---------------------------------------------------------------------------------------------------
def _norm_weight(rng, hidden, regime):
    if regime == "weights":                       # 0.01 ... 8 in magnitude, both signs, some zeros
        w = np.exp(rng.uniform(np.log(0.01), np.log(8.0), hidden)) * rng.choice([-1.0, 1.0], hidden)
        w[rng.choice(hidden, max(1, hidden // 64), replace=False)] = 0.0
        return w.astype(np.float16)
    return rng.uniform(0.3, 2.0, hidden).astype(np.float16)


def _norm_inputs(rng, B, hidden, regime):
    """(residual, x) fp16 such that residual + x has the regime's distribution."""
    std = {"unit": 1.0, "tiny": 2.0 ** -20, "zero_row": 1.0, "std300": 300.0, "outlier": 1.0, "overflow": 1.0,
           "weights": 1.0}[regime]
    r = rng.standard_normal((B, hidden)) * std / np.sqrt(2)
    x = rng.standard_normal((B, hidden)) * std / np.sqrt(2)
    if regime == "zero_row":
        r[B // 2], x[B // 2] = 0.0, 0.0
    if regime == "outlier":                       # a "massive activation" channel per row, 2000 ... 60000
        ch = rng.integers(0, hidden, B)
        r[np.arange(B), ch] = np.exp(rng.uniform(np.log(2000.0), np.log(60000.0), B)) * rng.choice([-1.0, 1.0], B)
    if regime == "overflow":                      # one residual + x per row overflows to +-inf
        ch = rng.integers(0, hidden, B)
        sgn = rng.choice([-1.0, 1.0], B)
        r[np.arange(B), ch], x[np.arange(B), ch] = 40000.0 * sgn, 30000.0 * sgn
    return r.astype(np.float16), x.astype(np.float16)


def _run_add_rmsnorm(res16, x16, w16, add):
    from kivi_b200 import glue
    res = torch.from_numpy(res16 if add else (res16 + x16)).cuda()
    x = torch.from_numpy(x16).cuda() if add else None
    w = torch.from_numpy(w16).cuda()
    out = torch.full_like(res, float("nan"))
    glue.add_rmsnorm(x, res, w, out, EPS)
    return res, w, out


def _check_add_rmsnorm(B, hidden, regime, add, seed):
    rng = np.random.default_rng(seed)
    res16, x16 = _norm_inputs(rng, B, hidden, regime)
    w16 = _norm_weight(rng, hidden, regime)
    with np.errstate(over="ignore"):
        exp_res = res16 + x16                                                # fp16 add, correctly rounded
    res, w, out = _run_add_rmsnorm(res16, x16, w16, add)
    what = f"add_rmsnorm<{add}> B={B} hidden={hidden} {regime}"
    assert_bits(to_np(res), exp_res, what + ": residual")
    assert not np.isnan(exp_res).any()
    check_rmsnorm(out, res, w, what)
    return to_np(out), exp_res


NORM_SHAPES = [(1, 4096), (32, 4096), (64, 4096), (3, 8), (3, 4088), (3, 4104), (3, 5120), (3, 8192), (3, 16384)]


@pytest.mark.parametrize("add", [True, False], ids=["add", "noadd"])
@pytest.mark.parametrize("B,hidden", NORM_SHAPES)
def test_add_rmsnorm_shapes(B, hidden, add):
    """Every register slice (hidden > 4096 uses slices 1..3 of the 512 threads), partial slices and the shipped width."""
    _check_add_rmsnorm(B, hidden, "unit", add, seed=hidden * 131 + B * 2 + add)


NORM_REGIMES = ["unit", "tiny", "zero_row", "std300", "outlier", "overflow", "weights"]


@pytest.mark.parametrize("add", [True, False], ids=["add", "noadd"])
@pytest.mark.parametrize("hidden", [4096, 16384])
@pytest.mark.parametrize("regime", NORM_REGIMES)
def test_add_rmsnorm_magnitudes(regime, hidden, add):
    out, res = _check_add_rmsnorm(8, hidden, regime, add, seed=1000 + NORM_REGIMES.index(regime) * 7 + hidden + add)
    if regime == "zero_row":
        assert (out[4] == 0).all()
    if regime == "overflow":                      # rsqrt(inf) = 0: NaN at the inf element, +-0 everywhere else
        inf = np.isinf(res)
        assert inf.sum(-1).tolist() == [1] * 8
        assert np.isnan(out[inf]).all() and (out[~inf] == 0).all()


def test_rmsnorm_module_matches_hf_chain():
    """LlamaRMSNorm (the prefill / insert / tuple-forward path) rounds like HF's chain and like the decode kernel:
    the normalised value is rounded to fp16 before the weight product."""
    from kivi_b200.llama_kivi import LlamaRMSNorm
    rng = np.random.default_rng(7)
    norm = LlamaRMSNorm(4096, EPS).half().cuda()
    with torch.no_grad():
        norm.weight.copy_(torch.from_numpy(_norm_weight(rng, 4096, "weights")))
    for regime in ("unit", "outlier", "std300", "tiny"):
        r, x = _norm_inputs(rng, 24, 4096, regime)
        h = torch.from_numpy(r + x).cuda().view(2, 12, 4096)
        with torch.no_grad():
            got = norm(h)
        exp = hf_rmsnorm(h, norm.weight)
        assert_bits(to_np(got), to_np(exp), f"LlamaRMSNorm {regime}")
        check_rmsnorm(got.view(24, 4096), h.view(24, 4096), norm.weight.detach(), f"LlamaRMSNorm {regime}")


# ---------------------------------------------------------------------------------------------------
# RoPE + split
# ---------------------------------------------------------------------------------------------------
_TABLES = {}


def _tables(theta):
    """The model's tables (llama_kivi._rope_tables, max_position_embeddings rows) on the device and as numpy."""
    if theta not in _TABLES:
        from kivi_b200.llama_kivi import _rope_tables
        c, s = _rope_tables(128, TABLE_ROWS, theta, torch.device("cuda"))
        _TABLES[theta] = (c, s, to_np(c), to_np(s))
    return _TABLES[theta]


EDGE_POS = [0, 1, 4095, 4096, 32767, 33791]


def _positions(rng, B):
    """B different-ish positions per row, the edge positions among them (B = 1: the last table row)."""
    p = rng.integers(0, TABLE_ROWS, B)
    e = min(B, len(EDGE_POS))
    p[:e] = EDGE_POS[len(EDGE_POS) - e:]
    return rng.permutation(p)


def _rope_qkv(rng, B, H, Hkv, regime):
    n = (H + 2 * Hkv) * 128
    if regime == "near_max":                      # |x| near 65504: x*cos + rot*sin overflows
        x = rng.uniform(60000.0, 65504.0, (B, n)) * rng.choice([-1.0, 1.0], (B, n))
    else:
        x = rng.standard_normal((B, n)) * {"unit": 1.0, "tiny": 1e-4, "std300": 300.0, "nan": 1.0}[regime]
    x = x.astype(np.float16)
    if regime == "nan":                           # one NaN channel in every head
        x.reshape(B, H + 2 * Hkv, 128)[:, :, rng.integers(0, 128)] = np.nan
    return x


def _run_rope(qkv16, cos, sin, pos, H, Hkv):
    from kivi_b200 import glue
    B = qkv16.shape[0]
    qkv = torch.from_numpy(qkv16).cuda()
    p = torch.as_tensor(pos, dtype=torch.int64).cuda().view(B, 1)
    q = torch.full((B, H, 128), float("nan"), device="cuda", dtype=torch.float16)
    k = torch.full((B, Hkv, 128), float("nan"), device="cuda", dtype=torch.float16)
    v = torch.full_like(k, float("nan"))
    glue.rope_split(qkv, cos, sin, p, q, k, v)
    return qkv, p, q, k, v


def _torch_rope(qkv, cos, sin, pos, H, Hkv):
    from kivi_b200.llama_kivi import _rotate_half
    B = qkv.shape[0]
    x = qkv.view(B, H + 2 * Hkv, 128)
    rows = pos.view(B).clamp(0, cos.shape[0] - 1)
    c, s = cos[rows][:, None], sin[rows][:, None]
    qk = x[:, :H + Hkv]
    out = qk * c + _rotate_half(qk) * s
    return out[:, :H], out[:, H:]


def _check_rope(B, H, Hkv, cos, sin, cos_np, sin_np, pos, regime, seed):
    rng = np.random.default_rng(seed)
    qkv16 = _rope_qkv(rng, B, H, Hkv, regime)
    qkv, p, q, k, v = _run_rope(qkv16, cos, sin, pos, H, Hkv)
    eq, ek, ev = rope_ref(qkv16, cos_np, sin_np, pos, H, Hkv)
    what = f"rope B={B} H={H}/{Hkv} {regime}"
    assert_bits(to_np(q), eq, what + ": q")
    assert_bits(to_np(k), ek, what + ": k")
    assert_bits(to_np(v), ev, what + ": v")
    assert np.array_equal(to_np(v).view(np.uint16), ev.view(np.uint16)), what + ": v is not an exact copy"
    tq, tk = _torch_rope(qkv, cos, sin, p, H, Hkv)
    assert_bits(to_np(q), to_np(tq), what + ": q vs torch")
    assert_bits(to_np(k), to_np(tk), what + ": k vs torch")
    return to_np(q), eq


@pytest.mark.parametrize("theta", [1e4, 5e5, 1e6])
@pytest.mark.parametrize("B", [1, 32, 64])
@pytest.mark.parametrize("H,Hkv", [(32, 32), (32, 8)])
def test_rope_split_shapes(H, Hkv, B, theta):
    """Per-row positions, among them the first and last table rows and the 4096 / 32768 boundaries."""
    rng = np.random.default_rng(int(theta) % 9973 + B * 5 + Hkv)
    cos, sin, cn, sn = _tables(theta)
    _check_rope(B, H, Hkv, cos, sin, cn, sn, _positions(rng, B), "unit", seed=int(rng.integers(1 << 30)))


@pytest.mark.parametrize("H,Hkv", [(32, 32), (32, 8)])
@pytest.mark.parametrize("regime", ["unit", "tiny", "std300", "near_max", "nan"])
def test_rope_split_magnitudes(regime, H, Hkv):
    rng = np.random.default_rng(["unit", "tiny", "std300", "near_max", "nan"].index(regime) * 17 + Hkv)
    cos, sin, cn, sn = _tables(5e5)
    q, eq = _check_rope(64, H, Hkv, cos, sin, cn, sn, _positions(rng, 64), regime, seed=int(rng.integers(1 << 30)))
    if regime == "near_max":
        assert np.isinf(eq).any() and np.isfinite(eq).any()
    if regime == "tiny":
        assert (np.abs(eq[eq != 0]) < 2.0 ** -14).any()                      # products in the fp16 subnormals


def test_rope_split_arbitrary_tables():
    """The kernel's contract is the elementwise x*cos + rotate_half(x)*sin on 128-wide rows.  The model's tables repeat
    their first half, so they cannot tell the halves apart; random tables can."""
    rng = np.random.default_rng(11)
    rows = 300
    cn = rng.uniform(-1, 1, (rows, 128)).astype(np.float16)
    sn = rng.uniform(-1, 1, (rows, 128)).astype(np.float16)
    cos, sin = torch.from_numpy(cn).cuda(), torch.from_numpy(sn).cuda()
    _check_rope(64, 32, 8, cos, sin, cn, sn, rng.integers(0, rows, 64), "unit", seed=12)


def test_rope_split_clamps_positions():
    """Out-of-table positions read the nearest row: below 0 -> row 0, at or past table_rows -> row table_rows - 1."""
    rng = np.random.default_rng(13)
    cos, sin, cn, sn = _tables(1e4)
    pos = np.array([-1, TABLE_ROWS, 10 ** 9, -(10 ** 12), TABLE_ROWS - 1, 0, TABLE_ROWS + 1, 2 ** 62], np.int64)
    q, _ = _check_rope(len(pos), 32, 8, cos, sin, cn, sn, pos, "unit", seed=14)
    # the clamp is the kernel's: the rows it must have read, spelled out
    qkv16 = _rope_qkv(np.random.default_rng(14), len(pos), 32, 8, "unit")
    rows = np.array([0, TABLE_ROWS - 1, TABLE_ROWS - 1, 0, TABLE_ROWS - 1, 0, TABLE_ROWS - 1, TABLE_ROWS - 1])
    eq, _, _ = rope_ref(qkv16, cn, sn, rows, 32, 8)
    assert_bits(q, eq, "clamped rows")
    assert not np.array_equal(cn[TABLE_ROWS - 1], cn[TABLE_ROWS - 2])          # the last row is distinguishable


# ---------------------------------------------------------------------------------------------------
# SiLU * mul
# ---------------------------------------------------------------------------------------------------
_ALL16 = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
_SPECIAL = np.array([np.inf, -np.inf, np.nan, -0.0, 0.0, -88.0, -88.75, -89.0, -90.0, -100.0, -65504.0, 65504.0,
                     -17.0, 11.1], np.float16)


def _gates(rng, n):
    """All 65536 fp16 patterns (shuffled, repeated to fill n) when n >= 65536, else the special values and a random draw."""
    if n >= _ALL16.size:
        return np.resize(rng.permutation(_ALL16), n)
    return np.concatenate([_SPECIAL, rng.choice(_ALL16, n)])[:n]


SILU_SHAPES = [(1, 2), (64, 2), (1, 514), (32, 514), (64, 1408), (32, 11008), (1, 14336), (64, 14336)]


@pytest.mark.parametrize("up", ["ones", "std1", "std1e3"])
@pytest.mark.parametrize("rows,inter", SILU_SHAPES)
def test_silu_mul(rows, inter, up):
    from kivi_b200 import glue
    rng = np.random.default_rng(rows * 7 + inter + len(up))
    g = _gates(rng, rows * inter).reshape(rows, inter)
    u = {"ones": np.ones((rows, inter)), "std1": rng.standard_normal((rows, inter)),
         "std1e3": rng.standard_normal((rows, inter)) * 1e3}[up].astype(np.float16)
    gu = torch.from_numpy(np.concatenate([g, u], 1)).cuda()
    out = torch.full((rows, inter), float("nan"), device="cuda", dtype=torch.float16)
    glue.silu_mul(gu, out)
    got = to_np(out)
    what = f"silu_mul rows={rows} I={inter} up={up}"
    s = silu64(g)
    check_rounded_product(got, u, s, what)
    assert (np.isnan(got) == np.isnan(s)).all(), f"{what}: NaN positions differ from the NaN (and -inf) gates"
    exp_t = F.silu(gu[:, :inter]) * gu[:, inter:]
    assert_bits(got, to_np(exp_t), what + ": vs F.silu(gate) * up")
    if rows * inter >= _ALL16.size:
        assert np.unique(g.view(np.uint16)).size == 1 << 16                  # exhaustive over the gate patterns
    if up == "std1e3" and rows * inter >= _ALL16.size:
        assert np.isinf(got).any()                                           # products past 65504 overflow


# ---------------------------------------------------------------------------------------------------
# greedy argmax
# ---------------------------------------------------------------------------------------------------
PATTERNS = ["plain", "tie_thread", "tie_lanes", "tie_warps", "tie_ends", "signed_zero", "all_neginf", "posinf", "nan1",
            "nans"]


def _logit_row(rng, V, pattern, rounded):
    x = rng.standard_normal(V).astype(np.float32)
    if rounded:
        x = x.astype(np.float16).astype(np.float32)
    top = np.float32(x.max() + 1.0 if V > 1 else 0.0)
    j = int(rng.integers(0, V))
    if pattern == "tie_thread":                   # j and j + 256k: the same thread's strided loop
        j %= 256
        x[j::256 * int(rng.integers(1, 4))] = top
    elif pattern == "tie_lanes":                  # neighbouring lanes of one warp
        x[[j, min(V - 1, j + int(rng.integers(1, 32)))]] = top
    elif pattern == "tie_warps":                  # different warps
        x[[j, (j + 32 * int(rng.integers(1, 8))) % V]] = top
    elif pattern == "tie_ends":
        x[[0, V - 1]] = top
    elif pattern == "signed_zero":                # -0 and +0 are equal: the first one wins
        x = -np.abs(x) - 1.0
        x[j], x[(j + int(rng.integers(1, 300))) % V] = (-0.0, 0.0) if rng.random() < 0.5 else (0.0, -0.0)
    elif pattern == "all_neginf":
        x[:] = -np.inf
    elif pattern == "posinf":
        x[j] = np.inf
        if rng.random() < 0.5:
            x[int(rng.integers(0, V))] = np.inf
    elif pattern == "nan1":
        x[j] = np.nan
    elif pattern == "nans":
        x[int(rng.integers(0, V))] = np.inf
        x[rng.integers(0, V, 4)] = np.nan
    return x


def _run_argmax(x):
    from kivi_b200 import glue
    B = x.shape[0]
    logits = torch.from_numpy(x).cuda()
    nxt = torch.full((B,), -7, dtype=torch.int64, device="cuda")
    fb = torch.full((B, 1), -9, dtype=torch.int64, device="cuda")
    glue.greedy_sample(logits, nxt, fb.view(-1))
    exp = argmax_ref(x)
    got = to_np(nxt)
    bad = np.flatnonzero(got != exp)
    assert bad.size == 0, f"argmax differs at rows {bad[:8].tolist()}: got {got[bad[:8]].tolist()}, expected {exp[bad[:8]].tolist()}"
    assert np.array_equal(to_np(fb).ravel(), got), "ids_feedback != next_local"
    assert np.array_equal(to_np(logits.argmax(-1)), got), "differs from torch.argmax"


@pytest.mark.parametrize("rounded", [False, True], ids=["fp32", "fp16rounded"])
@pytest.mark.parametrize("B", [1, 32, 64])
@pytest.mark.parametrize("V", [1, 7, 255, 256, 257, 32000, 128256])
def test_greedy_argmax(V, B, rounded):
    """Rows cycle through every pattern (ties inside a thread, across lanes and warps, at both ends, signed zeros,
    all -inf, +inf, one and several NaNs)."""
    rng = np.random.default_rng(V * 3 + B + rounded)
    off = int(rng.integers(0, len(PATTERNS)))
    x = np.stack([_logit_row(rng, V, PATTERNS[(b + off) % len(PATTERNS)], rounded) for b in range(B)])
    _run_argmax(x)


@pytest.mark.parametrize("V", [257, 128256])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_greedy_argmax_patterns(pattern, V):
    rng = np.random.default_rng(PATTERNS.index(pattern) * 101 + V)
    _run_argmax(np.stack([_logit_row(rng, V, pattern, rounded=bool(b & 1)) for b in range(64)]))


# ---------------------------------------------------------------------------------------------------
# wrapper validation
# ---------------------------------------------------------------------------------------------------
def test_glue_wrappers_reject_bad_arguments():
    """The Python wrappers refuse what the kernels would misread, before anything is enqueued."""
    from kivi_b200 import glue
    dev, h = "cuda", torch.float16
    B, H, Hkv, hid, inter = 4, 4, 2, 512, 1408
    res, w, out = torch.zeros(B, hid, device=dev, dtype=h), torch.ones(hid, device=dev, dtype=h), torch.empty(B, hid, device=dev, dtype=h)
    x = torch.zeros(B, hid, device=dev, dtype=h)
    for bad in (dict(x=x.cpu()), dict(residual=res.cpu()), dict(weight=w.float()), dict(out=out.float()),
                dict(x=torch.zeros(B, 2 * hid, device=dev, dtype=h)[:, ::2]), dict(residual=torch.zeros(hid, B, device=dev, dtype=h).t()),
                dict(weight=torch.ones(hid + 8, device=dev, dtype=h)), dict(out=torch.empty(B + 1, hid, device=dev, dtype=h)),
                dict(x=torch.zeros(B, hid + 8, device=dev, dtype=h)), dict(residual=torch.zeros(B, 1, hid, device=dev, dtype=h))):
        a = dict(x=x, residual=res, weight=w, out=out)
        a.update(bad)
        with pytest.raises((ValueError, RuntimeError)):
            glue.add_rmsnorm(a["x"], a["residual"], a["weight"], a["out"], EPS)
    cos, sin = torch.ones(64, 128, device=dev, dtype=h), torch.zeros(64, 128, device=dev, dtype=h)
    qkv = torch.zeros(B, (H + 2 * Hkv) * 128, device=dev, dtype=h)
    q, k, v = (torch.empty(B, n, 128, device=dev, dtype=h) for n in (H, Hkv, Hkv))
    pos = torch.zeros(B, 1, dtype=torch.int64, device=dev)
    for bad in (dict(qkv=qkv.cpu()), dict(qkv=qkv.float()), dict(qkv=torch.zeros(B, (H + 2 * Hkv) * 128 + 128, device=dev, dtype=h)),
                dict(cos=torch.ones(128, 64, device=dev, dtype=h)), dict(sin=torch.zeros(128, 64, device=dev, dtype=h)),
                dict(cos=cos.float()), dict(sin=torch.zeros(32, 128, device=dev, dtype=h)), dict(cos=cos.cpu()),
                dict(cos=torch.ones(128, 64, device=dev, dtype=h).t()), dict(pos=pos.int()), dict(pos=pos[:B - 1]),
                dict(pos=pos.cpu()), dict(q=torch.empty(B, H, 64, device=dev, dtype=h)),
                dict(k=torch.empty(B + 1, Hkv, 128, device=dev, dtype=h)), dict(v=torch.empty(B, H, 128, device=dev, dtype=h)),
                dict(q=torch.empty(B, 128, H, device=dev, dtype=h).transpose(1, 2))):
        a = dict(qkv=qkv, cos=cos, sin=sin, pos=pos, q=q, k=k, v=v)
        a.update(bad)
        with pytest.raises((ValueError, RuntimeError)):
            glue.rope_split(a["qkv"], a["cos"], a["sin"], a["pos"], a["q"], a["k"], a["v"])
    gu, act = torch.zeros(B, 2 * inter, device=dev, dtype=h), torch.empty(B, inter, device=dev, dtype=h)
    for bad in (dict(gu=gu.cpu()), dict(gu=gu.float()), dict(out=act.float()), dict(gu=gu[:, 1:inter * 2 - 1]),
                dict(gu=torch.zeros(B, 2 * inter + 2, device=dev, dtype=h)), dict(out=torch.empty(B + 1, inter, device=dev, dtype=h)),
                dict(gu=torch.zeros(2 * inter, B, device=dev, dtype=h).t())):
        a = dict(gu=gu, out=act)
        a.update(bad)
        with pytest.raises((ValueError, RuntimeError)):
            glue.silu_mul(a["gu"], a["out"])
    torch.cuda.synchronize()
    # the valid calls still run
    glue.add_rmsnorm(x, res, w, out, EPS)
    glue.rope_split(qkv, cos, sin, pos, q, k, v)
    glue.silu_mul(gu, act)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------
# production wiring
# ---------------------------------------------------------------------------------------------------
def test_decode_step_glue_wiring():
    """One layer with Llama-3-8B layer shapes (H 32, Hkv 8, hidden 4096, I 14336, vocab 128256): a left-padded batch of 8
    (per-row positions) is prefilled, then decoded through the CUDA graph; each glue stage of the step is checked from
    the static buffers against its own inputs, and the prefill's final norm against the same bar."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, _rope_tables, default_config
    cfg = default_config("llama-3-8b", num_hidden_layers=1)
    torch.manual_seed(5)
    with torch.device("cuda"):
        model = LlamaForCausalLM_KIVI(cfg)
    model = model.half().eval()
    with torch.no_grad():
        for nrm in (model.model.layers[0].input_layernorm, model.model.layers[0].post_attention_layernorm, model.model.norm):
            nrm.weight.uniform_(0.2, 3.0)
    B, n = 8, 180
    starts = torch.tensor([0, 3, 17, 64, 100, 127, 128, 179])
    mask = (torch.arange(n)[None, :] >= starts[:, None]).long().cuda()
    ids = torch.randint(0, cfg.vocab_size, (B, n), device="cuda")
    model.init_cache(B, n + 8)
    seen = {}
    hook = model.model.norm.register_forward_hook(lambda m, i, o: seen.update(inp=i[0].detach().clone(), out=o.detach().clone()))
    try:
        logits = model.prefill(ids, attention_mask=mask)
    finally:
        hook.remove()
    # the prefill's model.norm (LlamaRMSNorm) against the bar and the HF chain, on its own input
    w_final = model.model.norm.weight.detach()
    pin, pout = seen["inp"].reshape(-1, cfg.hidden_size), seen["out"].reshape(-1, cfg.hidden_size)
    check_rmsnorm(pout, pin, w_final, "prefill model.norm")
    assert_bits(to_np(pout), to_np(hf_rmsnorm(pin, w_final)), "prefill model.norm vs HF chain")
    cos_t, sin_t = _rope_tables(128, cfg.max_position_embeddings, cfg.rope_theta, torch.device("cuda"))
    cn, sn = to_np(cos_t), to_np(sin_t)
    tok = logits.argmax(-1, keepdim=True)
    exp_pos = (n - starts).numpy()
    H, Hkv, inter = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.intermediate_size
    for step in range(3):
        model.decode_step(tok)                                               # graph captured at step 0, replayed after
        torch.cuda.synchronize()
        f = model._fast
        pos = to_np(model._pos).ravel() - 1                                  # the step advanced _pos after its RoPE
        assert np.array_equal(pos, exp_pos + step), (step, pos)
        eq, ek, ev = rope_ref(to_np(f.qkv), cn, sn, pos, H, Hkv)
        assert_bits(to_np(f.q), eq, f"step {step}: q")
        assert_bits(to_np(f.k), ek, f"step {step}: k")
        assert_bits(to_np(f.v), ev, f"step {step}: v")
        gu = to_np(f.gu)
        check_rounded_product(to_np(f.act), gu[:, inter:], silu64(gu[:, :inter]), f"step {step}: act")
        assert_bits(to_np(f.act), to_np(F.silu(f.gu[:, :inter]) * f.gu[:, inter:]), f"step {step}: act vs torch")
        check_rmsnorm(f.h, f.res, w_final, f"step {step}: final add_rmsnorm")
        with torch.no_grad():
            mod = model.model.norm(f.res)
        check_rmsnorm(mod, f.res, w_final, f"step {step}: model.norm on the step's residual")
        lg = to_np(model._logits)
        assert np.array_equal(to_np(model.next_tokens), argmax_ref(lg)), f"step {step}: next_tokens"
        assert np.array_equal(to_np(model._ids).ravel(), to_np(model.next_tokens)), f"step {step}: fed-back ids"
        tok = model.next_tokens.view(B, 1).clone()

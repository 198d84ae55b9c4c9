"""The oracle check of the fused decode attention (tests/_attn.py) on the oracle's own values: it accepts them, and it
rejects each single defect a kernel could make.  The only checks of the harness that run without a GPU."""
import numpy as np
import pytest
import torch

from oracle import ref
from tests._attn import NEG16, check_stages, hidden_mask, rand16, tuple_equal

CFG = (32, 2, 4, 128)                                               # g, k_bits, v_bits, R
B, H, HKV, N0 = 3, 4, 2, 300                                        # tk 256, r 44, tv 172, L 128
T = N0 + 1
STATES = ["unpadded", "padded", "window-user", "inf-scale"]


def _call(name):
    """check_stages' arguments for one call, the oracle's scaled logits, probabilities and output standing for the kernel's."""
    g, kb, vb, R = CFG
    rng = np.random.default_rng(STATES.index(name))
    k, v = rand16(rng, (B, HKV, N0, 128)), rand16(rng, (B, HKV, N0, 128))
    if name == "inf-scale":                                          # sequence 1: a packed V group of scale inf
        v[1, :, 40, 0], v[1, :, 40, 1] = -60000.0, 60000.0
    st = ref.prefill_cache(k, v, g, kb, vb, R)
    q, kn, vn = rand16(rng, (B, H, 1, 128), 0.7), rand16(rng, (B, HKV, 1, 128)), rand16(rng, (B, HKV, 1, 128))
    user = np.zeros((B, T), np.float16)
    user[:, 5:T - 1:7] = NEG16
    mask = {"padded": hidden_mask(B, T, [0, 70, 200]),
            "window-user": hidden_mask(B, T, [0, 70, 200], window=150, user=user)}.get(name)
    out, p, _ = ref.decode_step(st, q, kn, vn, *CFG, mask)
    logits = np.concatenate([ref.bmm_fA_qB_outer(g, q, st[0], st[2], st[3], kb),
                             ref.residual_qk(q, np.concatenate([st[1], kn], axis=2))], -1)
    s = (logits.astype(np.float32) * (np.float32(1.0) / np.float32(11.313708))).astype(np.float16)
    return [st, q, kn, vn, CFG, out, s, p, mask, (1,) if name == "inf-scale" else ()]


def test_hidden_mask():
    user = np.zeros((3, 10), np.float16)
    user[:, 7] = NEG16
    m = hidden_mask(3, 10, [3, 20, -4], window=5, user=user)
    assert ((m[:, 0, 0] == NEG16).sum(-1) == [6, 9, 6]).all() and (m[:, ..., 7] == NEG16).all()
    assert hidden_mask(3, 10) is None


@pytest.mark.parametrize("name", STATES)
def test_accepts_the_oracle(name):
    args = _call(name)
    assert np.isfinite(args[5][0]).all() and np.isfinite(args[5][1]).all() == (name != "inf-scale"), "precondition"
    check_stages(*args)


def _rejects(args, i, edit, match):
    bad = list(args)
    bad[i] = args[i].copy()
    edit(bad[i])
    with pytest.raises(AssertionError, match=match):
        check_stages(*bad)


def test_rejects_each_defect():
    args = _call("window-user")
    visible = np.broadcast_to(args[8] != NEG16, args[6].shape)
    j = np.unravel_index(np.argmax(np.where(visible, np.abs(args[6].astype(np.float64)), -1)), visible.shape)
    _rejects(args, 6, lambda s: s.view(np.uint16).__setitem__(j, s.view(np.uint16)[j] + 2), "scaled logits")  # 2 steps out
    _rejects(args, 7, lambda p: p.__setitem__(np.unravel_index(p.argmax(), p.shape), p.max() * np.float16(1.01)),
             "softmax stage")
    _rejects(args, 7, lambda p: p.__setitem__((1, 2, 0, 100), 1e-3), "hidden positions")
    inf = _call("inf-scale")
    nonfinite = np.argwhere(~np.isfinite(inf[5]))[0]
    assert nonfinite[0] == 1
    _rejects(inf, 5, lambda o: o.__setitem__((1, 0, 0, 100), o[1, 0, 0, 100] + 1.0), "end-to-end")
    _rejects(inf, 5, lambda o: o.__setitem__(tuple(nonfinite), 0.0), "non-finite positions")


def test_tuple_equal():
    st = _call("unpadded")[0]
    tuple_equal(tuple(torch.from_numpy(t) if isinstance(t, np.ndarray) else t for t in st), st, "torch against numpy")
    tuple_equal(st[:1] + (np.zeros((B, HKV, 0, 128), np.float16),) + st[2:], st[:1] + (None,) + st[2:], "empty as None")
    for i in (0, 2, 5):                                              # K codes, K scale, V window
        flipped = list(st)
        flipped[i] = st[i].copy()
        flipped[i].view(np.uint16 if st[i].dtype == np.float16 else np.int32).flat[7] ^= 1
        with pytest.raises(AssertionError, match=rf"tuple\[{i}\]"):
            tuple_equal(flipped, st, "flipped bit")

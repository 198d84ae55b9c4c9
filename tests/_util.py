"""Shared helpers for the parity tests."""
import hashlib

import numpy as np
import torch


def to_np(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().numpy()


def rand_quantised(rng, shape_rows_T, g, bits):
    """Random fp16 data -> oracle pack (codes/scale/mn as numpy)."""
    from oracle import ref
    x = rng.standard_normal(shape_rows_T).astype(np.float16)
    return (x,) + ref.pack_lastdim(x, g, bits)


def input_digest(*arrays):
    return hashlib.sha256(b"".join(np.ascontiguousarray(a).tobytes() for a in arrays)).digest()

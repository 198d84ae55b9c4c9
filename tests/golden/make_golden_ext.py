"""Store the outputs of the UNMODIFIED reference CUDA extension for tests/test_bgemv_gpu.py.

Usage (on a CUDA device, after oracle/build_ref.py has built oracle/_ref/kivi_gemv.so from the reference sources):
    python tests/golden/make_golden_ext.py [OUT_DIR]      # default OUT_DIR: tests/golden

Runs gemv_forward_cuda_outer_dim of the reference extension on the seeded inputs of
test_against_reference_cuda_extension and writes, per bit width and case, the fp16 output and a digest of the
inputs into OUT_DIR/reference_ext_gemv.npz.  Nothing here is imported at test time.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests._gemv import reference_extension_inputs  # noqa: E402
from tests._util import input_digest  # noqa: E402


def main(out_dir):
    refmod = build_ref.load()
    assert refmod is not None, "oracle/_ref/kivi_gemv.so is not built"
    out = {}
    for bits in (2, 4):
        for i, ((B, nh, nh_kv, IC, OC, GS), inp, (code, scale, mn), (qw_t, sc_t, mn_t)) in \
                enumerate(reference_extension_inputs(bits)):
            args = [torch.from_numpy(a).cuda() for a in (inp, qw_t, sc_t, mn_t)]
            res = refmod.gemv_forward_cuda_outer_dim(*args, bits, GS, nh, nh_kv)
            torch.cuda.synchronize()
            out[f"out_b{bits}_{i}"] = res.cpu().numpy()
            out[f"digest_b{bits}_{i}"] = np.frombuffer(input_digest(inp, code, scale, mn), np.uint8)
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "reference_ext_gemv.npz"), **out)
    print("reference_ext_gemv.npz", len(out), "arrays on", torch.cuda.get_device_name(0))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.dirname(os.path.abspath(__file__)))

"""The block word layout of kivi_decode.cuh, checked on the host: lay_word_off / lay_bit_pos, its two parts lay_word_inner +
lay_word_row, its inverse lay_word_pos and the meta pair offset must agree with the layout the header comment states, for
every element of a block (tests/layout_check.cu, compiled by nvcc as host code; no GPU needed)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_word_layout_helpers_match_the_documented_layout(tmp_path):
    from kivi_b200 import build
    exe = str(tmp_path / "layout_check")
    subprocess.check_call([build._nvcc(), "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, os.path.join(ROOT, "tests", "layout_check.cu")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.strip() == "0", out.stdout + out.stderr

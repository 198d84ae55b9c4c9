"""Build tuning variants of libkivi_b200.so (extra -D flags) into tools/variants/ and print a sweep command.

    python tools/build_variants.py NAME "-DKIVI_UNROLL=4 -DKIVI_SHIFT_IMAD=1" [NAME2 "flags2" ...]

The variants are loaded through KIVI_B200_LIB (kivi_b200/_lib.py); they are git-ignored build artefacts."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kivi_b200 import build as kb  # noqa: E402

out_dir = os.path.join(ROOT, "tools", "variants")
os.makedirs(out_dir, exist_ok=True)
args = sys.argv[1:]
for name, flags in zip(args[0::2], args[1::2]):
    objs, procs = [], []
    for s in kb._sources():
        obj = os.path.join(out_dir, f"{name}_{s.replace('.cu', '.o')}")
        cmd = [kb._nvcc(), "-c", os.path.join(kb.CSRC, s), "-o", obj] + kb.NVCC_FLAGS + flags.split()
        procs.append(subprocess.Popen(cmd))
        objs.append(obj)
    assert all(p.wait() == 0 for p in procs), name
    so = os.path.join(out_dir, f"libkivi_{name}.so")
    subprocess.check_call([kb._nvcc(), "-shared", "-o", so] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-lcudart"])
    for o in objs:
        os.remove(o)
    print(so)

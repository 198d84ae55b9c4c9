"""Build the UNMODIFIED reference CUDA extension `kivi_gemv` into oracle/_ref/.

TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is imported by the product
package `kivi_b200`; only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may use it.

The sources are compiled *where they lie* under KIVI_REFERENCE_ROOT
(quant/csrc/pybind.cpp + quant/csrc/gemv_cuda.cu, the two files that
quant/setup.py:37-40 lists) with the nvcc flags of quant/setup.py:5-29 plus an
explicit sm_90a -gencode (the reference passes none and relies on
TORCH_CUDA_ARCH_LIST).  No reference source is copied into this repository:
only the resulting shared object lands in oracle/_ref/ (git-ignored).

Where the reference sources are absent this script is a no-op and the
prebuilt oracle/_ref/kivi_gemv.so (if any) is used as is.  The tests do not
need it: tests/golden/reference_ext_gemv.npz holds its outputs.
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("KIVI_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref")
SO = os.path.join(OUT, "kivi_gemv.so")


def _run(cmd):
    print("[oracle/_ref]", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)


def build(force: bool = False) -> str | None:
    src_cu = os.path.join(REF, "quant", "csrc", "gemv_cuda.cu")
    src_cpp = os.path.join(REF, "quant", "csrc", "pybind.cpp")
    if not (os.path.exists(src_cu) and os.path.exists(src_cpp)):
        return SO if os.path.exists(SO) else None
    if os.path.exists(SO) and not force:
        newest = max(os.path.getmtime(src_cu), os.path.getmtime(src_cpp))
        if os.path.getmtime(SO) >= newest:
            return SO
    import torch
    from torch.utils import cpp_extension as ce

    os.makedirs(OUT, exist_ok=True)
    incs = []
    for p in ce.include_paths() + [sysconfig.get_paths()["include"], os.path.join(REF, "quant", "csrc")]:
        incs += ["-I", p]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    defs = ["-DTORCH_EXTENSION_NAME=kivi_gemv", "-DTORCH_API_INCLUDE_EXTENSION_H",
            f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DENABLE_BF16"]
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    obj_cu = os.path.join(OUT, "gemv_cuda.o")
    obj_cpp = os.path.join(OUT, "pybind.o")
    _run([nvcc, "-c", src_cu, "-o", obj_cu, "-O3", "-std=c++17",
          "-gencode", "arch=compute_90a,code=sm_90a",
          "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
          "-U__CUDA_NO_BFLOAT16_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
          "-U__CUDA_NO_BFLOAT162_OPERATORS__", "-U__CUDA_NO_BFLOAT162_CONVERSIONS__",
          "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math",
          "-Xcompiler", "-fPIC"] + defs + incs)
    _run(["g++", "-c", src_cpp, "-o", obj_cpp, "-O3", "-std=c++17", "-fPIC"] + defs + incs)
    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    _run(["g++", "-shared", "-o", SO, obj_cu, obj_cpp,
          "-L", tlib, "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
          "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{tlib}"])
    for o in (obj_cu, obj_cpp):
        os.remove(o)
    return SO


def load():
    """Import the prebuilt reference extension (needs `import torch` first). None if absent."""
    if not os.path.exists(SO):
        return None
    import importlib.util
    import torch  # noqa: F401  (registers libtorch symbols)
    spec = importlib.util.spec_from_file_location("kivi_gemv", SO)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))

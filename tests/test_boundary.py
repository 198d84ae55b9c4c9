"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol that
include/kivi_b200.h declares, argument validation returns the documented codes without touching a
GPU, the Python surface mirrors the reference's names/signatures, and the product never reaches
into oracle/."""
import inspect
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    names = []
    for fn in os.listdir(os.path.join(ROOT, "include")):
        if fn.endswith(".h"):
            txt = open(os.path.join(ROOT, "include", fn)).read()
            txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
            names += re.findall(r"\b(kivi_[a-z0-9_]+)\s*\(", txt)
    return sorted(set(names))


@pytest.fixture(scope="module")
def L():
    from kivi_b200 import build, _lib
    build.build()                                                     # nvcc cross-compiles without a GPU
    return _lib.lib()


def test_library_exports_every_declared_symbol(L):
    syms = _declared_symbols()
    assert len(syms) >= 7
    for s in syms:
        assert hasattr(L, s), f"libkivi_b200.so does not export {s} declared in include/kivi_b200.h"
    assert L.kivi_version() >= 100


def test_argument_validation_without_gpu(L):
    """Every check happens before the first CUDA call, so the codes are observable on a CPU box."""
    one = 16                                                          # a non-NULL dummy address, never dereferenced
    assert L.kivi_pack_lastdim_f16(one, 4, 128, 32, 3, one, one, one, None) == -1          # bits
    assert L.kivi_pack_lastdim_f16(one, 4, 100, 32, 2, one, one, one, None) == -2          # T % g   (new_pack.py:222)
    assert L.kivi_pack_lastdim_f16(None, 4, 128, 32, 2, one, one, one, None) == -6         # NULL
    assert L.kivi_pack_lastdim_f16(None, 0, 128, 32, 2, None, None, None, None) == 0       # empty is fine
    assert L.kivi_bgemv_outer_f16(one, 128, one, 1, 1, one, one, 1, 1, one, 1, 3, 2, 128, 128, 2, 32, 0, None) == -3   # GQA
    assert L.kivi_bgemv_outer_f16(one, 128, one, 1, 1, one, one, 1, 1, one, 1, 2, 2, 128, 128, 3, 32, 0, None) == -1   # bits
    assert L.kivi_bgemv_outer_f16(one, 128, one, 1, 1, one, one, 1, 1, one, 1, 2, 2, 128, 100, 2, 32, 0, None) == -2   # N % g
    assert L.kivi_bgemv_outer_f16(one, 128, one, 1, 1, one, one, 1, 1, one, 1, 2, 2, 128, 128, 8, 32, 1, None) == -1   # 8-bit only on ref layout
    assert L.kivi_gemv_inner_f16(one, one, one, one, one, 1, 100, 8, 4, 64, 2, None) == -2                            # IC % fpi
    assert L.kivi_error_string(-4).decode() == "unsupported group_size"


def test_surface_mirrors_reference_names():
    """Same function names and positional parameters as quant/new_pack.py, quant/matmul.py, quant/gemv.py
    and the kivi_gemv extension (SURVEY 8b)."""
    from kivi_b200 import gemv, kivi_gemv, matmul, new_pack
    expect = {
        (new_pack, "triton_quantize_and_pack_along_last_dim"): ["data", "group_size", "bit"],
        (new_pack, "quant_and_pack_kcache"): ["k", "group_size", "bits"],
        (new_pack, "quant_and_pack_vcache"): ["v", "group_size", "bits"],
        (new_pack, "unpack_and_dequant_kcache"): ["k_code", "scale", "mn", "group_size", "bits"],
        (new_pack, "unpack_and_dequant_vcache"): ["v_code", "scale", "mn", "group_size", "bits"],
        (new_pack, "pack_tensor"): ["data", "bits", "pack_dim"],
        (new_pack, "unpack_tensor"): ["v_code", "bits", "pack_dim"],
        (matmul, "cuda_bmm_fA_qB_outer"): ["group_size", "fA", "qB", "scales", "zeros", "bits"],
        (matmul, "triton_bmm_fA_qB_outer"): ["group_size", "fA", "qB", "scales", "zeros", "bits"],
        (gemv, "gemv_fwd"): ["bit", "group_size", "inp", "qweight", "mn", "scale"],
        (gemv, "dequant_weight"): ["w", "scale", "mn", "gs"],
        (gemv, "dequant_weight_outer"): ["w", "scale", "mn", "gs"],
        (kivi_gemv, "gemv_forward_cuda"): ["_in_feats", "_kernel", "_scaling_factors", "_zeros", "bit", "group_size"],
        (kivi_gemv, "gemv_forward_cuda_outer_dim"): ["_in_feats", "_kernel", "_scaling_factors", "_zeros", "bit",
                                                     "group_size", "nh", "nh_kv"],
    }
    for (mod, name), params in expect.items():
        fn = getattr(mod, name)
        assert list(inspect.signature(fn).parameters) == params, name


def test_product_never_touches_the_oracle():
    """The oracle is test infrastructure: no file of the product package (or the include dir) may import,
    load or execute anything under oracle/."""
    pat = re.compile(r"(^\s*(from|import)\s+oracle\b)|(oracle[/\\._])|(kivi_oracle)", re.M)
    for base in ("kivi_b200", "include", "quant", "models"):
        d = os.path.join(ROOT, base)
        if not os.path.isdir(d):
            continue
        for dp, _, files in os.walk(d):
            for fn in files:
                if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".c")):
                    txt = open(os.path.join(dp, fn), errors="ignore").read()
                    m = pat.search(txt)
                    assert m is None or "never imports oracle" in txt.lower() or "Nothing in this package imports oracle" in txt, \
                        f"{os.path.join(dp, fn)} references the oracle: {m.group(0)!r}"


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from kivi_b200 import _lib
    monkeypatch.setattr(_lib, "_LIB", None)
    monkeypatch.setattr(_lib, "SO_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU or PyTorch fallback"):
        _lib.lib()


def test_cpu_tensors_are_rejected():
    import torch
    from kivi_b200 import matmul, new_pack
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        new_pack.triton_quantize_and_pack_along_last_dim(torch.zeros((1, 1, 2, 64), dtype=torch.float16), 32, 2)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        matmul.cuda_bmm_fA_qB_outer(32, torch.zeros((1, 1, 1, 8), dtype=torch.float16),
                                    torch.zeros((1, 1, 8, 2), dtype=torch.int32),
                                    torch.zeros((1, 1, 8, 1), dtype=torch.float16),
                                    torch.zeros((1, 1, 8, 1), dtype=torch.float16), 2)


def test_cache_struct_mirrors_the_header():
    """kivi_b200.cache._CacheStruct (ctypes) has the fields of kivi_cache_t in include/kivi_b200.h, in order, and the
    overlap flag the Python side sets is the header's KIVI_CACHE_OVERLAP_PROLOGUE."""
    import ctypes
    from kivi_b200 import cache
    txt = open(os.path.join(ROOT, "include", "kivi_b200.h")).read()
    body = re.search(r"typedef struct kivi_cache \{(.*?)\} kivi_cache_t;", txt, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        ctype, names = ("ptr", decl.replace("void*", "")) if decl.startswith("void*") else ("i32", decl.replace("int32_t", ""))
        fields += [(n.strip(), ctype) for n in names.split(",")]
    mirror = [(n, "ptr" if t is ctypes.c_void_p else "i32") for n, t in cache._CacheStruct._fields_]
    assert mirror == fields
    assert ctypes.sizeof(cache._CacheStruct) == 12 * 4 + 5 * 8
    flag = int(re.search(r"#define KIVI_CACHE_OVERLAP_PROLOGUE\s+(\d+)", txt).group(1))
    assert flag == 1                                                  # KiviCache(overlap_prologue=True) stores 1 in `flags`
    src = inspect.getsource(cache.KiviCache.__init__)
    assert "1 if overlap_prologue else 0" in src
    shift = int(re.search(r"#define KIVI_CACHE_GQA_CHUNK_SHIFT\s+(\d+)", txt).group(1))
    assert shift == 4 and "int(gqa_chunk) << 4" in src


def test_reference_import_paths_resolve_here():
    """models/llama_kivi.py:9-10 does `from quant.new_pack import triton_quantize_and_pack_along_last_dim` and
    `from quant.matmul import cuda_bmm_fA_qB_outer`; quant/matmul.py:6 does `import kivi_gemv`; example.py:4 /
    mem_spd_test.py:4 do `from models.llama_kivi import LlamaForCausalLM_KIVI`.  The same statements work in this
    repository and land on kivi_b200."""
    import kivi_gemv
    from models.llama_kivi import LlamaForCausalLM_KIVI
    from models.mistral_kivi import MistralForCausalLM_KIVI
    from quant.gemv import dequant_weight_outer, gemv_fwd
    from quant.matmul import cuda_bmm_fA_qB_outer, triton_bmm_fA_qB_outer
    from quant.new_pack import triton_quantize_and_pack_along_last_dim, unpack_and_dequant_vcache
    import kivi_b200.kivi_gemv
    import kivi_b200.llama_kivi
    import kivi_b200.matmul
    import kivi_b200.new_pack
    assert triton_quantize_and_pack_along_last_dim is kivi_b200.new_pack.triton_quantize_and_pack_along_last_dim
    assert cuda_bmm_fA_qB_outer is kivi_b200.matmul.cuda_bmm_fA_qB_outer
    assert triton_bmm_fA_qB_outer is kivi_b200.matmul.triton_bmm_fA_qB_outer
    assert kivi_gemv.gemv_forward_cuda_outer_dim is kivi_b200.kivi_gemv.gemv_forward_cuda_outer_dim
    assert LlamaForCausalLM_KIVI is kivi_b200.llama_kivi.LlamaForCausalLM_KIVI is MistralForCausalLM_KIVI
    assert callable(unpack_and_dequant_vcache) and callable(gemv_fwd) and callable(dequant_weight_outer)


def test_model_class_contract_on_cpu(tmp_path):
    """LlamaForCausalLM_KIVI keeps the reference's class contract (models/llama_kivi.py:785-957) where no GPU is
    needed: from_pretrained on a local checkpoint directory, HF parameter names, prepare_inputs_for_generation
    (:908-948) and _reorder_cache (:950-957) on 9-tuples."""
    import json
    import torch
    from safetensors.torch import save_file
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    cfg = default_config("tiny")
    torch.manual_seed(0)
    src = LlamaForCausalLM_KIVI(cfg)
    save_file({k: v.contiguous() for k, v in src.state_dict().items()}, str(tmp_path / "model.safetensors"))
    with open(tmp_path / "config.json", "w") as f:
        json.dump({k: v for k, v in vars(cfg).items() if k not in ("k_bits", "v_bits", "group_size", "residual_length")}, f)
    m = LlamaForCausalLM_KIVI.from_pretrained(str(tmp_path), torch_dtype=torch.float16)
    assert (m.config.k_bits, m.config.v_bits, m.config.group_size, m.config.residual_length) == (2, 2, 32, 128)
    assert m.lm_head.weight.dtype == torch.float16
    for k, v in src.state_dict().items():
        assert torch.equal(m.state_dict()[k], v.half()), k
    assert "model.layers.0.self_attn.q_proj.weight" in m.state_dict() and "model.norm.weight" in m.state_dict()
    with pytest.raises(FileNotFoundError):
        LlamaForCausalLM_KIVI.from_pretrained("meta-llama/Llama-2-7b-hf")          # no network: local directories only
    # generation plumbing on the reference's 9-tuple (Kq, K_full, K_scale, K_mn, Vq, V_full, V_scale, V_mn, kv_seq_len)
    B = 3
    past = tuple((torch.zeros(B, 2, 128, 8, dtype=torch.int32), None, torch.zeros(B, 2, 128, 4), torch.zeros(B, 2, 128, 4),
                  None, torch.arange(B * 2 * 5 * 128, dtype=torch.float32).view(B, 2, 5, 128), None, None, 133)
                 for _ in range(2))
    ids = torch.arange(B * 134).view(B, 134)
    mask = torch.ones(B, 134, dtype=torch.long)
    mask[1, :4] = 0                                                                # a left-padded row
    inp = m.prepare_inputs_for_generation(ids, past_key_values=past, attention_mask=mask)
    assert inp["input_ids"].shape == (B, 1) and torch.equal(inp["input_ids"][:, 0], ids[:, -1])
    assert inp["position_ids"].tolist() == [[133], [129], [133]] and inp["past_key_values"] is past
    first = m.prepare_inputs_for_generation(ids, past_key_values=None, attention_mask=mask)
    assert first["input_ids"].shape == (B, 134) and first["position_ids"][1, :6].tolist() == [1, 1, 1, 1, 0, 1]
    re_ = LlamaForCausalLM_KIVI._reorder_cache(past, torch.tensor([2, 0, 0]))
    assert len(re_) == 2 and re_[0][8] == 133 and re_[0][1] is None
    assert torch.equal(re_[1][5], past[1][5][[2, 0, 0]])


def test_fused_cache_needs_fp16_weights():
    """The fused cache path runs fp16 weights only: init_cache, and generate() through it, refuse any other dtype with a
    ValueError that names it, before anything is allocated."""
    import torch
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    m = LlamaForCausalLM_KIVI(default_config("tiny"))
    with pytest.raises(ValueError, match="float32"):
        m.init_cache(2, 16)
    with pytest.raises(ValueError, match="float32"):
        m.generate(torch.zeros(2, 3, dtype=torch.long), max_new_tokens=2)
    assert m.cache is None

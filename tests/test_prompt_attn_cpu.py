"""kivi_prompt_attention_f16 without a GPU: every invalid argument is rejected by return code before any CUDA call.  Every
call here is invalid in at least one argument, so none of them launches.  And the model's choice of mask for a prompt
on the 9-tuple path: the kernel only for masks its rule states exactly (decided on the host, nothing runs)."""
import pytest
import torch

KIVI_ERR_SHAPE, KIVI_ERR_GQA, KIVI_ERR_ALIGN, KIVI_ERR_NULL = -2, -3, -5, -6
FAKE = 1 << 20                                       # 16-byte aligned, never dereferenced: validation returns first


@pytest.fixture(scope="module")
def lib():
    from kivi_b200 import _lib, build, glue
    build.build()
    glue._bind()
    return _lib.lib()


def _call(lib, q=FAKE, k=FAKE, v=FAKE, out=FAKE, B=2, H=32, Hkv=8, n=100, q_strides=(100 * 4096, 128, 4096),
          kv_strides=(100 * 1024, 128, 1024), kv_start=None, window=0):
    return lib.kivi_prompt_attention_f16(q, k, v, out, B, H, Hkv, n, *q_strides, *kv_strides, kv_start, window, None)


def test_symbol_is_exported(lib):
    assert hasattr(lib, "kivi_prompt_attention_f16")


def test_null_pointers(lib):
    for name in ("q", "k", "v", "out"):
        assert _call(lib, **{name: None}) == KIVI_ERR_NULL, name


def test_shapes(lib):
    assert _call(lib, B=0) == KIVI_ERR_SHAPE
    assert _call(lib, B=-1) == KIVI_ERR_SHAPE
    assert _call(lib, B=65536) == KIVI_ERR_SHAPE                           # grid.z
    assert _call(lib, H=0) == KIVI_ERR_SHAPE
    assert _call(lib, n=0) == KIVI_ERR_SHAPE
    assert _call(lib, n=-3) == KIVI_ERR_SHAPE
    assert _call(lib, window=-1) == KIVI_ERR_SHAPE
    assert _call(lib, H=8, Hkv=65536 // 8) == KIVI_ERR_GQA                 # H % Hkv
    assert _call(lib, H=65536 * 8, Hkv=65536) == KIVI_ERR_SHAPE            # grid.y: one CTA row per KV head


def test_gqa(lib):
    assert _call(lib, H=32, Hkv=0) == KIVI_ERR_GQA
    assert _call(lib, H=32, Hkv=-8) == KIVI_ERR_GQA
    assert _call(lib, H=32, Hkv=5) == KIVI_ERR_GQA
    assert _call(lib, H=6, Hkv=4) == KIVI_ERR_GQA


def test_alignment(lib):
    for name in ("q", "k", "v", "out"):
        for off in (2, 8):
            assert _call(lib, **{name: FAKE + off}) == KIVI_ERR_ALIGN, (name, off)
    assert _call(lib, kv_start=FAKE + 2) == KIVI_ERR_ALIGN                  # int32 starts
    for i in range(3):                                                     # every row of 128 halves on 16 bytes
        qs, kvs = [100 * 4096, 128, 4096], [100 * 1024, 128, 1024]
        qs[i] += 4
        assert _call(lib, q_strides=tuple(qs)) == KIVI_ERR_ALIGN, ("q", i)
        kvs[i] -= 2
        assert _call(lib, kv_strides=tuple(kvs)) == KIVI_ERR_ALIGN, ("kv", i)


def test_shape_errors_come_before_alignment(lib):
    assert _call(lib, q=FAKE + 2, n=0) == KIVI_ERR_SHAPE
    assert _call(lib, q=None, n=0) == KIVI_ERR_NULL
    assert _call(lib, out=FAKE + 2, H=32, Hkv=5) == KIVI_ERR_GQA


def _windowed_model(**kw):
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    return LlamaForCausalLM_KIVI(default_config("tiny", sliding_window=16, **kw)).half()


def test_tuple_prompt_keeps_masks_the_kernel_does_not_state():
    """A windowed fp16 model, n > W: a right-padded, holed or empty-row [B, n] mask, a mask of another shape and a 4-D
    mask keep the additive mask (None); no mask and an all-ones mask take the kernel with the window alone."""
    m, B, n, cuda = _windowed_model(), 2, 40, torch.device("cuda")
    ones = torch.ones((B, n), dtype=torch.long)
    right, holes, empty = ones.clone(), ones.clone(), ones.clone()
    right[1, -5:] = 0
    holes[0, 10:12] = 0
    empty[1] = 0
    for what, mask in (("right", right), ("holes", holes), ("empty row", empty), ("longer", torch.ones((B, n + 3))),
                       ("4-D", torch.zeros((B, 1, n, n), dtype=torch.float16))):
        assert m._tuple_prompt_mask(mask, B, n, cuda) is None, what
    for mask in (None, ones):
        assert m._tuple_prompt_mask(mask, B, n, cuda) == (None, 16)
    assert m._tuple_prompt_mask(ones, B, 16, cuda) is None                  # the window does not cut: causal SDPA
    assert m._tuple_prompt_mask(ones, B, n, torch.device("cpu")) is None


def test_kernel_mask_needs_fp16_and_head_dim_128():
    n, cuda = 40, torch.device("cuda")
    assert _windowed_model()._kernel_mask(None, n, cuda) == (None, 16)
    assert _windowed_model().float()._kernel_mask(None, n, cuda) is None
    assert _windowed_model(hidden_size=512, num_attention_heads=8, num_key_value_heads=8)._kernel_mask(None, n, cuda) is None

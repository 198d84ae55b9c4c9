"""Logits processing without a GPU: the torch restatement of tests/_logits.py against transformers' processors, the host
validation of the parameters (processing_rows, parse_requests, generate's arguments) and the C entry points' argument
checks (no launch happens when they fail)."""
import pytest
import torch

from tests._logits import pack_bits, reference_process, same_bits, special_logits, unpack_bits

V = 1000


def _neutral(B):
    return dict(presence=torch.zeros(B), frequency=torch.zeros(B), min_new=torch.zeros(B, dtype=torch.int32),
                n_new=torch.zeros(B, dtype=torch.int32), finished=torch.zeros(B, dtype=torch.bool))


def test_pack_bits_round_trip():
    g = torch.Generator().manual_seed(0)
    for v in (1, 31, 32, 33, 1000, 32001):
        m = torch.rand((3, v), generator=g) < 0.3
        w = pack_bits(m)
        assert w.shape == (3, (v + 31) // 32) and w.dtype == torch.int32
        assert torch.equal(unpack_bits(w, v), m)
    assert pack_bits(torch.tensor([[False] * 31 + [True]])).item() == -2 ** 31


@pytest.mark.parametrize("penalty", [0.5, 1.0, 1.2, 3.0])
def test_repetition_matches_transformers(penalty):
    """Prompt tokens (seen) and generated tokens (counts) together are transformers' input_ids."""
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor
    g = torch.Generator().manual_seed(1)
    B, n, k = 4, 30, 12
    prompt = torch.randint(0, V, (B, n), generator=g)
    gen = torch.randint(0, V, (B, k), generator=g)
    gen[:, :3] = prompt[:, :3]                                            # tokens both in the prompt and generated
    logits = special_logits(B, V, g)
    ref = RepetitionPenaltyLogitsProcessor(penalty)(torch.cat([prompt, gen], 1), logits.clone())
    seen = torch.zeros((B, V), dtype=torch.bool).scatter_(1, prompt, True)
    counts = torch.zeros((B, V), dtype=torch.long).scatter_add_(1, gen, torch.ones_like(gen))
    got = reference_process(logits, counts, seen, repetition=torch.full((B,), penalty), eos=[], pad=0, **_neutral(B))
    assert same_bits(got, ref)


@pytest.mark.parametrize("eos", [[7], [7, 0, 999, 500, 3, 4, 5, 6]])
def test_min_length_matches_transformers(eos):
    from transformers.generation.logits_process import MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor
    g = torch.Generator().manual_seed(2)
    B, n = 3, 20
    logits = special_logits(B, V, g)
    for k in range(0, 8):                                                 # k tokens generated so far
        ids = torch.randint(0, V, (B, n + k), generator=g)
        for min_length, min_new in ((n + 5, None), (n, None), (None, 5), (None, 0)):
            if min_length is not None:
                ref = MinLengthLogitsProcessor(min_length, eos)(ids, logits.clone())
                floor = min_length - n
            else:
                ref = MinNewTokensLengthLogitsProcessor(n, min_new, eos)(ids, logits.clone())
                floor = min_new
            kw = _neutral(B)
            kw.update(n_new=torch.full((B,), k, dtype=torch.int32), min_new=torch.full((B,), floor, dtype=torch.int32))
            got = reference_process(logits, torch.zeros((B, V), dtype=torch.long), torch.zeros((B, V), dtype=torch.bool),
                                    repetition=torch.ones(B), eos=eos, pad=0, **kw)
            assert same_bits(got, ref), (k, min_length, min_new)


def test_presence_frequency_and_finished_rows():
    """vLLM's order: x - f * count, then - presence where count > 0; a finished row keeps only the pad id."""
    g = torch.Generator().manual_seed(3)
    B = 3
    logits = torch.randn((B, V), generator=g)
    counts = torch.randint(0, 4, (B, V), generator=g)
    kw = _neutral(B)
    kw.update(presence=torch.tensor([0.5, -1.0, 2.0]), frequency=torch.tensor([0.25, 2.0, -2.0]),
              finished=torch.tensor([False, True, False]))
    got = reference_process(logits, counts, torch.zeros((B, V), dtype=torch.bool), repetition=torch.ones(B), eos=[5],
                            pad=9, **kw)
    for b in (0, 2):
        exp = logits[b] - kw["frequency"][b] * counts[b].float()
        exp = torch.where(counts[b] > 0, exp - kw["presence"][b], exp)
        assert same_bits(got[b], exp)
    assert got[1, 9].item() == 0.0 and torch.isinf(got[1]).sum().item() == V - 1 and (got[1] <= 0).all()


def test_processing_rows_rejects_out_of_range():
    from kivi_b200.llama_kivi import processing_rows
    rep, pres, freq, mn, eos = processing_rows(2, [1.2, 0.8], 0.5, -0.5, 3, [2, 3], vocab=10)
    assert rep == [1.2, 0.8] and pres == [0.5, 0.5] and freq == [-0.5, -0.5] and mn == [3, 3] and eos == [2, 3]
    assert processing_rows(1, eos_token_id=4)[4] == [4] and processing_rows(1)[4] == []
    bad = [dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=float("inf")),
           dict(repetition_penalty=float("nan")), dict(presence_penalty=2.5), dict(frequency_penalty=-2.01),
           dict(presence_penalty=float("nan")), dict(min_new_tokens=-1), dict(min_new_tokens=1.5),
           dict(eos_token_id=10), dict(eos_token_id=-1), dict(eos_token_id=list(range(9))), dict(eos_token_id=1.5),
           dict(repetition_penalty=[1.0, 1.0, 1.0])]
    for kw in bad:
        with pytest.raises(ValueError):
            processing_rows(2, vocab=10, **kw)


def test_parse_requests_validates_processing_keys():
    from kivi_b200.serve import parse_requests, processing_params, sampling_params
    p = torch.arange(1, 5)
    _, params = parse_requests([(p, 3, dict(repetition_penalty=1.3, presence_penalty=0.5, frequency_penalty=0.2,
                                            min_new_tokens=2, temperature=0.7))])
    assert sampling_params(params[0]) == dict(temperature=0.7)
    assert processing_params(params[0]) == dict(repetition_penalty=1.3, presence_penalty=0.5, frequency_penalty=0.2,
                                                min_new_tokens=2)
    _, params = parse_requests([(p, 3, dict(repetition_penalty=1.3)), (p, 3, {}), (p, 3)])
    assert sampling_params(params[0]) is None                             # processing keys only: greedy
    assert sampling_params(params[1]) == {} and processing_params(params[1]) is None     # {}: sampled, the defaults
    assert sampling_params(params[2]) is None and processing_params(params[2]) is None
    for par in (dict(repetition_penalty=0.0), dict(presence_penalty=3.0), dict(frequency_penalty=-2.5),
                dict(min_new_tokens=-2), dict(repetition_penalty=1.1, top_p=2.0), dict(no_repeat_ngram_size=2)):
        with pytest.raises(ValueError):
            parse_requests([(p, 3, par)])


def test_generate_refuses_before_any_work():
    """Beam search with a processor, and min_length without eos_token_id, raise before the model is touched: the model
    here has no weights on a GPU and no cache."""
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    model = LlamaForCausalLM_KIVI(default_config("tiny", num_hidden_layers=1))
    ids = torch.ones((1, 4), dtype=torch.long)
    with pytest.raises(NotImplementedError, match="beam search"):
        model.generate(ids, max_new_tokens=4, num_beams=2, repetition_penalty=1.2)
    with pytest.raises(NotImplementedError, match="beam search"):
        model.generate(ids, max_new_tokens=4, num_beams=2, min_new_tokens=2, eos_token_id=3)
    with pytest.raises(ValueError, match="eos_token_id"):
        model.generate(ids, max_new_tokens=4, min_length=6)
    with pytest.raises(ValueError, match="repetition_penalty"):
        model.generate(ids, max_new_tokens=4, repetition_penalty=0.0)
    with pytest.raises(ValueError, match="eos_token_id"):
        model.generate(ids, max_new_tokens=4, eos_token_id=10 ** 9)
    assert model.cache is None


def test_entry_points_check_arguments():
    """Both entry points return KIVI_ERR_* for bad arguments before touching a pointer (no device needed)."""
    import ctypes
    from kivi_b200 import _lib, build, glue
    build.build()
    glue._bind()
    L = _lib.lib()
    n0 = _lib.launch_count()
    SHAPE, NULL = -2, -6
    p = ctypes.c_void_p(16)                                               # never dereferenced: every call fails its checks
    args = lambda **kw: [kw.get(k, d) for k, d in (("logits", p), ("scores", p), ("B", 2), ("V", 100))] + \
        [p] * 9 + [kw.get("n_eos", 1), kw.get("pad", 0), None]                             # noqa: E731
    assert L.kivi_logits_process_f32(*args(logits=None)) == NULL
    assert L.kivi_logits_process_f32(*args(V=0)) == SHAPE
    assert L.kivi_logits_process_f32(*args(B=-1)) == SHAPE
    assert L.kivi_logits_process_f32(*args(n_eos=9)) == SHAPE
    assert L.kivi_logits_process_f32(*args(pad=100)) == SHAPE
    assert L.kivi_logits_process_f32(*args(pad=-1)) == SHAPE
    assert L.kivi_logits_record(None, 2, 100, p, p, p, p, 1, None) == NULL
    assert L.kivi_logits_record(p, 2, 100, p, p, p, None, 1, None) == NULL
    assert L.kivi_logits_record(p, 2, 100, p, p, p, p, 9, None) == SHAPE
    assert L.kivi_logits_record(p, 2, 0, p, p, p, p, 1, None) == SHAPE
    assert L.kivi_logits_record(p, 0, 100, p, p, p, p, 1, None) == 0                 # an empty batch is fine
    assert _lib.launch_count() == n0

"""Log-probabilities without a GPU: the C entry point's argument checks (no launch happens when they fail), the float64
reference's ranking against torch.topk, serve()'s validation of `logprobs`, generate()'s refusals before any work, and
compute_transition_scores against transformers' own."""
import pytest
import torch

from tests._logprobs import reference_logprobs


def test_entry_point_checks_arguments():
    import ctypes
    from kivi_b200 import _lib, build, glue
    build.build()
    glue._bind()
    L = _lib.lib()
    assert hasattr(L, "kivi_token_logprobs_f32")
    n0 = _lib.launch_count()
    SHAPE, NULL = -2, -6
    p = ctypes.c_void_p(16)                                               # never dereferenced: every call fails its checks
    f = L.kivi_token_logprobs_f32
    assert f(None, 2, 100, p, 5, p, p, p, None) == NULL
    assert f(p, 2, 100, None, 5, p, p, p, None) == NULL
    assert f(p, 2, 100, p, 5, None, p, p, None) == NULL
    assert f(p, 2, 100, p, 5, p, None, p, None) == NULL
    assert f(p, 2, 100, p, 5, p, p, None, None) == NULL
    assert f(p, 2, 100, p, 21, p, p, p, None) == SHAPE
    assert f(p, 2, 100, p, -1, p, p, p, None) == SHAPE
    assert f(p, 2, 0, p, 5, p, p, p, None) == SHAPE
    assert f(p, 2, 2 ** 22 + 1, p, 5, p, p, p, None) == SHAPE
    assert f(p, -1, 100, p, 5, p, p, p, None) == SHAPE
    assert f(p, 0, 2 ** 22, p, 20, p, p, p, None) == 0                    # an empty batch is fine
    assert f(p, 0, 100, p, 0, p, None, None, None) == 0                   # N = 0 needs no top buffers
    assert _lib.launch_count() == n0


def test_reference_ranks_like_topk():
    g = torch.Generator().manual_seed(0)
    x = torch.randn((4, 300), generator=g) * 5
    x[1, 7] = x[1, 9] = float("nan")
    x[2, 3] = float("inf")
    tok, ids, top = reference_logprobs(x, torch.tensor([0, 5, 299, 300]), 10)
    ref = torch.topk(x.double(), 10, -1)
    assert torch.equal(ids[[0, 3]], ref.indices[[0, 3]])                  # no ties: topk's order
    assert ids[1, :2].tolist() == [7, 9]                                  # NaN first, by id
    assert ids[2, 0].item() == 3 and torch.isnan(top[2]).all() and torch.isnan(tok[1:3]).all()
    assert torch.isnan(tok[3]) and torch.isfinite(tok[0])                 # 300 is outside the vocabulary
    tie = torch.zeros((1, 40))
    tie[0, 5] = 1.0
    tie[0, 30] = -0.0
    _, ids, _ = reference_logprobs(tie, torch.tensor([0]), 5)
    assert ids.tolist() == [[5, 0, 1, 2, 3]]                              # the tie by ascending id, -0 equal to +0
    _, ids, top = reference_logprobs(torch.randn((2, 7), generator=g), torch.tensor([0, 1]), 9)
    assert (ids[:, 7:] == -1).all() and torch.isneginf(top[:, 7:]).all()


def test_parse_requests_validates_logprobs():
    from kivi_b200.serve import decoding_params, logprobs_param, parse_requests, sampling_params
    p = torch.arange(1, 5)
    _, params = parse_requests([(p, 3, dict(logprobs=0)), (p, 3, dict(logprobs=20, temperature=0.5)), (p, 3)])
    assert [logprobs_param(x) for x in params] == [0, 20, None]
    assert decoding_params(params[0]) is None                              # logprobs only: greedy, as without params
    assert sampling_params(decoding_params(params[1])) == dict(temperature=0.5)
    for n in (-1, 21, 2.0, True, "3", None):
        with pytest.raises(ValueError, match="logprobs"):
            parse_requests([(p, 3, dict(logprobs=n))])


def test_generate_refuses_before_any_work():
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    model = LlamaForCausalLM_KIVI(default_config("tiny", num_hidden_layers=1))
    ids = torch.ones((1, 4), dtype=torch.long)
    with pytest.raises(NotImplementedError, match="do_sample"):
        model.generate(ids, max_new_tokens=4, do_sample=True, output_scores=True)
    with pytest.raises(NotImplementedError, match="do_sample"):
        model.generate(ids, max_new_tokens=4, do_sample=True, num_return_sequences=2, output_scores=True)
    for kw in (dict(output_scores=True), dict(output_logits=True), dict(output_scores=True, output_logits=True)):
        with pytest.raises(NotImplementedError, match="beam search"):
            model.generate(ids, max_new_tokens=4, num_beams=2, return_dict_in_generate=True, **kw)
    with pytest.raises(NotImplementedError, match="beam_indices"):
        model.compute_transition_scores(ids, (torch.zeros(1, 10),), beam_indices=torch.zeros((1, 1), dtype=torch.long))
    assert model.cache is None


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_transition_scores_match_transformers(normalize, dtype):
    from types import SimpleNamespace
    from transformers.generation.utils import GenerationMixin
    from kivi_b200.llama_kivi import LlamaForCausalLM_KIVI, default_config
    V = 97
    model = LlamaForCausalLM_KIVI(default_config("tiny", num_hidden_layers=1, vocab_size=V))
    g = torch.Generator().manual_seed(1)
    rows, n, steps = 3, 5, 6
    seq = torch.randint(0, V, (rows, n + steps), generator=g)
    scores = tuple((torch.randn((rows, V), generator=g) * 4).to(dtype) for _ in range(steps))
    scores[2][1, :] = float("-inf")
    scores[2][1, 3] = 0.0                                                 # a finished row's pad-only scores
    got = model.compute_transition_scores(seq, scores, normalize_logits=normalize)
    text = SimpleNamespace(vocab_size=V)
    text.get_text_config = lambda: text
    ref = GenerationMixin.compute_transition_scores(SimpleNamespace(config=text), seq, scores, normalize_logits=normalize)
    assert got.shape == (rows, steps) and got.dtype == ref.dtype
    assert torch.equal(got.isnan(), ref.isnan()) and torch.equal(got.nan_to_num(), ref.nan_to_num())

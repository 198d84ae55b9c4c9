"""kivi_b200.choice.TokenChoice on the host: the state a decode step changes round-trips through snapshot / restore, the
setters report when the step's launch sequence changes, and the per-row setters write one row and refuse what
sampling_rows / processing_rows refuse."""
import pytest
import torch

from kivi_b200.choice import TokenChoice, processing_rows, sampling_rows

B, V = 3, 70


def _choice():
    c = TokenChoice(B, V, "cpu")
    assert c.set_sampling(0.7, 20, 0.9, 5) and c.set_processing(1.2, 0.1, 0.2, 2, eos_token_id=[4, 9])
    return c


def test_snapshot_restore_round_trips_what_a_step_changes():
    c = _choice()
    p = c.proc
    changed = [c.samp.draw, p.counts, p.n_new, p.finished]
    g = torch.Generator().manual_seed(0)
    for t in changed:                                                      # a state that is not all zeros
        t.copy_(torch.randint(0, 100, t.shape, generator=g).to(t.dtype))
    before = [t.clone() for t in changed]
    saved = c.snapshot()
    assert {id(t) for t, _ in saved} == {id(t) for t in changed}
    for t in changed:                                                      # what a step does: counts, lengths, flags
        t.add_(1)
    c.restore(saved)
    for t, exp in zip(changed, before):
        assert torch.equal(t, exp)
    c.set_sampling(None)
    c.set_processing(None)
    assert c.snapshot() == []                                              # a greedy step without processing changes none


def test_setters_report_launch_sequence_changes():
    c = TokenChoice(B, V, "cpu")
    assert not c.set_sampling(None) and c.set_sampling(1.0) and not c.set_sampling(0.5, seed=[1, 2, 3])
    assert c.set_sampling(None) and not c.sampling
    assert c.set_processing(1.1) and not c.set_processing(1.3)                 # parameters alone: the same step
    assert c.set_processing(1.3, pad_token_id=7) and not c.set_processing(1.0, pad_token_id=7)   # the pad is an argument
    assert c.set_processing(None) and c.proc is None and not c.set_processing(None)
    assert c.set_logprobs(0) and not c.set_logprobs(0) and c.set_logprobs(5) and c.top_ids.shape == (B, 5)
    assert c.set_logprobs(None) and c.logprobs is None
    for n in (-1, 21, 2.5, True):
        with pytest.raises(ValueError):
            c.set_logprobs(n)


def test_slot_setters_write_one_row():
    c = _choice()
    s, p = c.samp, c.proc
    s.draw.fill_(4)
    before = [t.clone() for t in (s.temperature, s.top_k, s.top_p, s.seed, p.repetition, p.presence, p.frequency, p.min_new)]
    c.set_slot_sampling(1, temperature=1.5, top_k=3, top_p=0.5, seed=2 ** 64 - 1)
    c.set_slot_processing(1, repetition_penalty=0.8, presence_penalty=-1.0, frequency_penalty=2.0, min_new_tokens=9)
    after = (s.temperature, s.top_k, s.top_p, s.seed, p.repetition, p.presence, p.frequency, p.min_new)
    for t, old, row1 in zip(after, before, (1.5, 3, 0.5, -1, 0.8, -1.0, 2.0, 9)):
        assert t[0] == old[0] and t[2] == old[2] and t[1].item() == pytest.approx(row1)
    assert s.draw.tolist() == [4, 0, 4]
    c.set_slot(2)                                                          # a request without params: greedy, neutral
    assert (s.temperature[2].item(), s.top_k[2].item(), s.seed[2].item(), s.draw[2].item()) == (0.0, 0, 0, 0)
    assert (p.repetition[2].item(), p.presence[2].item(), p.frequency[2].item(), p.min_new[2].item()) == (1.0, 0.0, 0.0, 0)


@pytest.mark.parametrize("kind", ["sampling", "processing"])
def test_slot_setters_refuse_what_the_row_parsers_refuse(kind):
    c = _choice()
    state = [t.clone() for t in vars(c.samp).values()] + [t.clone() for t in (c.proc.repetition, c.proc.min_new)]
    if kind == "sampling":
        bad = [dict(temperature=-0.1), dict(temperature=float("nan")), dict(top_p=1.5), dict(top_k=2.5),
               dict(top_k=2 ** 31), dict(top_k="many"), dict(seed=-1), dict(seed=1.5), dict(temperature=[1.0, 1.0])]
        parse, slot = sampling_rows, c.set_slot_sampling
    else:
        bad = [dict(repetition_penalty=0.0), dict(repetition_penalty=float("inf")), dict(presence_penalty=2.5),
               dict(frequency_penalty=-2.01), dict(min_new_tokens=-1), dict(min_new_tokens=1.5),
               dict(repetition_penalty=[1.0, 1.0])]
        parse, slot = processing_rows, c.set_slot_processing
    for kw in bad:
        with pytest.raises(ValueError):
            parse(1, **kw)
        with pytest.raises(ValueError):
            slot(0, **kw)
    for seq in (-1, B):
        with pytest.raises(ValueError):
            slot(seq)
    now = [t for t in vars(c.samp).values()] + [c.proc.repetition, c.proc.min_new]
    assert all(torch.equal(a, b) for a, b in zip(now, state))              # nothing written
    off = TokenChoice(B, V, "cpu")
    with pytest.raises(RuntimeError):
        (off.set_slot_sampling if kind == "sampling" else off.set_slot_processing)(0)

"""The greedy-id contract itself (tests/parity.py) on hand-made logits: what it accepts and what it must reject."""
import pytest
import torch

from parity import check_greedy_ids

V = 10


def _logits(seq):
    out = torch.zeros(len(seq), 1, V)
    for i, t in enumerate(seq):
        out[i, 0, t] = 1.0
    return out


def _teacher(ids):
    out = torch.zeros(1, ids.shape[1] + 1, V)
    for s, t in enumerate(ids[0].tolist()):
        out[0, s, t] = 1.0
    return out


def test_equal_ids_need_no_oracle_pass():
    ref = torch.tensor([[1, 2, 3, 4]])
    assert check_greedy_ids(ref.clone(), ref, _logits([1, 2, 3, 4]), 0.05, None) == {"flips": 0, "resynced": 0}


def test_flip_at_a_clear_margin_is_rejected():
    ref, got = torch.tensor([[1, 2, 3, 4]]), torch.tensor([[1, 5, 3, 4]])
    with pytest.raises(AssertionError, match="oracle margin"):
        check_greedy_ids(got, ref, _logits([1, 2, 3, 4]), 0.05, _teacher)


def test_tolerated_flip_resyncs_and_keeps_checking():
    ref, got = torch.tensor([[1, 2, 3, 4]]), torch.tensor([[1, 5, 3, 4]])
    rl = _logits([1, 2, 3, 4])
    rl[1, 0, 5] = 0.99                                  # top-2 margin 0.01 at the flipped step
    assert check_greedy_ids(got, ref, rl, 0.05, _teacher) == {"flips": 1, "resynced": 3}

    def corrupted(ids):                                 # the oracle disagrees with the engine's suffix -> must fail
        out = _teacher(ids)
        out[0, 3, 7] = 2.0
        return out

    with pytest.raises(AssertionError, match="after the flip"):
        check_greedy_ids(got, ref, rl, 0.05, corrupted)


def test_shorter_output_without_a_flip_is_rejected():
    ref = torch.tensor([[1, 2, 3, 4]])
    with pytest.raises(AssertionError):
        check_greedy_ids(ref[:, :3].clone(), ref, _logits([1, 2, 3, 4]), 0.05, _teacher)


def test_repetition_penalty_is_applied_to_the_resync_logits():
    ref, got = torch.tensor([[1, 2, 3]]), torch.tensor([[1, 5, 6]])
    rl = _logits([1, 2, 3])
    rl[1, 0, 5] = 0.99

    def teacher(ids):
        out = torch.zeros(1, 4, V)
        out[0, 1, 5] = 1.0
        out[0, 2, 5] = 1.0                              # raw argmax repeats token 5 ...
        out[0, 2, 6] = 0.6                              # ... but 5 was generated: 1.0 / 2 = 0.5 < 0.6
        return out

    assert check_greedy_ids(got, ref, rl, 0.05, teacher, repetition_penalty=2.0)["resynced"] == 2


def test_repetition_penalty_is_applied_to_the_flip_margin():
    ref, got = torch.tensor([[1, 2, 3]]), torch.tensor([[1, 5, 3]])
    rl = _logits([1, 2, 3])
    rl[1, 0, 1] = 1.5                                   # raw top-1 is token 1, 0.5 above the rest ...
    rl[1, 0, 5] = 1.0                                   # ... but 1 was generated: 1.5 / 3 = 0.5, so 2 and 5 tie at 1.0
    assert check_greedy_ids(got, ref, rl, 0.05, _teacher, repetition_penalty=3.0)["flips"] == 1
    with pytest.raises(AssertionError, match="oracle margin"):
        check_greedy_ids(got, ref, rl, 0.05, _teacher, repetition_penalty=1.2)   # 1.5 / 1.2 = 1.25: a clear margin

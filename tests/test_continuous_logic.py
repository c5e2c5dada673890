"""The continuous-batching scheduler (starvector_b200/continuous.py) driven by a stand-in engine, and the session entry
points of the built library.  No GPU needed."""
import ctypes
import os
import types

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200.continuous import ContinuousScheduler
from starvector_b200.engine import GenerationParams


class FakeEngine:
    """Mimics the session calls: slot s decodes one token per step; request `tag` (the first pixel value of its image)
    finishes after `lengths[tag]` tokens or at its cap, and its tokens are [tag * 1000 + seed % 1000, ...]."""

    def __init__(self, slots, lengths):
        self.dims = types.SimpleNamespace(max_batch=slots)
        self.lengths = lengths
        self.log = []
        self.open = False

    def session_begin(self, params, slots):
        assert not self.open
        self.open, self.S, self.cap = True, slots, params.max_new_tokens
        self.rows = {}

    def session_admit(self, pixels, prompt_ids, slots, *, max_new_tokens, seeds, src):
        assert self.open and len(slots) == len(max_new_tokens) == len(seeds) == len(src)
        for j, s in enumerate(slots):
            assert s not in self.rows, f"slot {s} admitted while busy"
            tag = int(pixels[src[j]].flatten()[0])
            n = min(self.lengths[tag], max_new_tokens[j])
            self.rows[s] = {"tag": tag, "seed": seeds[j], "n": n, "done": 0}
        self.log.append(("admit", list(slots), [int(pixels[i].flatten()[0]) for i in src]))

    def session_run(self, max_steps):
        steps = 0
        while steps < max_steps and self.rows and not any(r["done"] >= r["n"] for r in self.rows.values()):
            for r in self.rows.values():
                r["done"] += 1
            steps += 1
        fin = [s in self.rows and self.rows[s]["done"] >= self.rows[s]["n"] for s in range(self.S)]
        self.finished = [s for s in range(self.S) if fin[s]]
        return steps, fin, [self.rows[s]["done"] if s in self.rows else 0 for s in range(self.S)]

    def session_read(self, slot):
        r = self.rows.pop(slot)
        return torch.arange(r["n"], dtype=torch.int32) + r["tag"] * 1000 + r["seed"] % 1000

    def session_end(self):
        self.open = False


def _images(n):
    return torch.arange(n, dtype=torch.float32).view(n, 1, 1, 1).expand(n, 3, 2, 2).contiguous()


def test_fifo_admission_and_slot_reuse():
    eng = FakeEngine(3, lengths=[5, 2, 9, 1, 4, 3])
    out = ContinuousScheduler(eng).run(_images(6), torch.tensor([1, 2]), GenerationParams(max_new_tokens=20))
    assert eng.log[0] == ("admit", [0, 1, 2], [0, 1, 2])          # the first three requests fill the slots in order
    admitted = [tag for _, _, tags in eng.log for tag in tags]
    assert admitted == list(range(6)), "requests are admitted in FIFO order"
    assert eng.log[1] == ("admit", [1], [3])                        # request 1 (2 tokens) finished first: its slot is reused
    assert [len(o) for o in out] == [5, 2, 9, 1, 4, 3]
    assert not eng.open


def test_admit_steps_are_recorded():
    eng = FakeEngine(2, lengths=[6, 2, 3, 4])
    sch = ContinuousScheduler(eng)
    sch.run(_images(4), torch.tensor([1]), GenerationParams(max_new_tokens=10))
    # request 1 finishes after 2 steps -> request 2 joins at step 2; it finishes at 5 while request 0 is done at 6
    assert sch.stats["admit_step"] == [0, 0, 2, 5]
    assert sch.stats["steps"] == 9 and sch.stats["admissions"] == 3


def test_results_in_request_order_whatever_the_completion_order():
    eng = FakeEngine(4, lengths=[30, 3, 20, 1, 7, 2, 9])
    done = []
    out = ContinuousScheduler(eng).run(_images(7), torch.tensor([1]), GenerationParams(max_new_tokens=40),
                                       on_finish=lambda k, ids: done.append(k))
    assert done != sorted(done) and sorted(done) == list(range(7))
    for k, ids in enumerate(out):
        assert int(ids[0]) // 1000 == k


def test_n_completions_wait_for_n_free_slots():
    eng = FakeEngine(4, lengths=[6, 2, 8])
    out = ContinuousScheduler(eng).run(_images(3), torch.tensor([1]), GenerationParams(max_new_tokens=10, seed=100), n=3)
    assert eng.log[0] == ("admit", [0, 1, 2], [0, 0, 0])           # image 0 takes 3 slots; image 1 needs 3, only 1 free
    assert all(len(slots) % 3 == 0 for _, slots, _ in eng.log)
    assert len(eng.log) == 3
    assert len(out) == 9
    for k, ids in enumerate(out):
        assert int(ids[0]) // 1000 == k // 3                        # completion j of image i at index i * n + j
        assert int(ids[0]) % 1000 == 100 + k                        # seed + k


def test_seed_assignment_and_explicit_seeds():
    eng = FakeEngine(2, lengths=[3, 3, 3])
    out = ContinuousScheduler(eng).run(_images(3), torch.tensor([1]), GenerationParams(max_new_tokens=5, seed=40))
    assert [int(o[0]) % 1000 for o in out] == [40, 41, 42]
    out = ContinuousScheduler(eng).run(_images(3), torch.tensor([1]), GenerationParams(max_new_tokens=5), seeds=[7, 8, 9])
    assert [int(o[0]) % 1000 for o in out] == [7, 8, 9]


def test_per_request_caps():
    eng = FakeEngine(2, lengths=[50, 50, 50])
    out = ContinuousScheduler(eng).run(_images(3), torch.tensor([1]), GenerationParams(max_new_tokens=10),
                                       max_new_tokens=[10, 4, 7])
    assert [len(o) for o in out] == [10, 4, 7]
    with pytest.raises(ValueError, match="session cap"):
        ContinuousScheduler(eng).run(_images(3), torch.tensor([1]), GenerationParams(max_new_tokens=10),
                                     max_new_tokens=[10, 11, 7])
    with pytest.raises(ValueError):
        ContinuousScheduler(eng).run(_images(3), torch.tensor([1]), GenerationParams(max_new_tokens=10), max_new_tokens=[0, 1, 1])
    with pytest.raises(ValueError):
        ContinuousScheduler(eng).run(_images(3), torch.tensor([1]), GenerationParams(max_new_tokens=10), n=3)   # 2 slots
    assert not eng.open


def test_session_symbols_in_the_library():
    assert _lib.ABI_VERSION == 7
    for name in ("sv_session_begin", "sv_session_admit", "sv_session_run", "sv_session_read", "sv_session_end"):
        assert name in _lib.SIGNATURES
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert lib.sv_abi_version() == 7
    for name in ("sv_session_begin", "sv_session_admit", "sv_session_run", "sv_session_read", "sv_session_end"):
        assert hasattr(lib, name), name

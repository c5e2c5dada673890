"""CPU tests of beam sessions: the scheduler's group bookkeeping with a stand-in engine, and the ABI surface."""
import os
import re
import subprocess
from types import SimpleNamespace

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200.continuous import ContinuousScheduler
from starvector_b200.engine import BeamSearchParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class StandInBeamEngine:
    """Mimics sv_beam_session_*: a group runs for its cap steps (or `stop_at[image]` if smaller) and returns
    [image, seed, its first slot] as its ids."""

    def __init__(self, max_batch, stop_at=None):
        self.dims = SimpleNamespace(max_batch=max_batch)
        self.stop_at = stop_at or {}
        self.admits, self.slots_used = [], set()

    def beam_session_begin(self, params, slots):
        self.nb, self.S, self.live, self.done = params.num_beams, slots, {}, {}

    def beam_session_admit(self, pixels, prompt_ids, groups, *, max_new_tokens, seeds):
        assert pixels.shape[0] == prompt_ids.shape[0] == len(groups) == len(max_new_tokens) == len(seeds)
        for j, g in enumerate(groups):
            assert 0 <= g < self.S // self.nb and g not in self.live
            img = int(pixels[j, 0, 0, 0])
            self.live[g] = [min(max_new_tokens[j], self.stop_at.get(img, 10 ** 9)), img, int(seeds[j])]
            self.admits.append((img, g))
            self.slots_used.update(range(g * self.nb, (g + 1) * self.nb))

    def session_run(self, max_steps):
        fin = [False] * self.S
        if not self.live:
            return 0, fin, [0] * self.S
        n = min(v[0] for v in self.live.values())
        for g in list(self.live):
            self.live[g][0] -= n
            if self.live[g][0] == 0:
                _, img, seed = self.live.pop(g)
                fin[g * self.nb] = True
                self.done[g * self.nb] = torch.tensor([img, seed, g * self.nb], dtype=torch.int32)
        return n, fin, [0] * self.S

    def session_read(self, slot):
        return self.done.pop(slot)

    def session_end(self):
        self.ended = True


def _pixels(n):
    return torch.arange(n, dtype=torch.float32).view(n, 1, 1, 1).expand(n, 3, 4, 4).contiguous()


@pytest.mark.parametrize("nb,slots", [(2, 8), (3, 6), (4, 8)])
def test_groups_fifo_seeds_and_reuse(nb, slots):
    eng = StandInBeamEngine(8)
    caps = [7, 3, 9, 1, 4, 4, 8, 2, 5, 6, 3]
    order = []
    sch = ContinuousScheduler(eng, slots, num_beams=nb)
    got = sch.run(_pixels(11), torch.tensor([5, 6]), BeamSearchParams(nb, 9, seed=40), max_new_tokens=caps,
                  on_finish=lambda k, ids: order.append(k))
    assert eng.ended
    assert [int(g[0]) for g in got] == list(range(11))                      # request order
    assert [int(g[1]) for g in got] == [40 + k for k in range(11)]          # seeds seed + k
    assert all(int(g[2]) % nb == 0 for g in got)                            # a group's first slot
    assert [a[0] for a in eng.admits] == list(range(11))                    # FIFO
    assert eng.slots_used == set(range(slots))                              # every slot reused
    assert sorted(order) == list(range(11)) and order != list(range(11))
    assert sch.stats["admissions"] > 1 and len(sch.stats["admit_step"]) == 11


def test_explicit_seeds_and_early_finish():
    eng = StandInBeamEngine(4, stop_at={2: 1})
    got = ContinuousScheduler(eng, 4, num_beams=2).run(_pixels(5), torch.tensor([[5, 6]] * 5), BeamSearchParams(2, 6),
                                                       seeds=[9, 8, 7, 6, 5])
    assert [int(g[1]) for g in got] == [9, 8, 7, 6, 5]


def test_validation():
    eng = StandInBeamEngine(8)
    with pytest.raises(ValueError, match="multiple of num_beams"):
        ContinuousScheduler(eng, 7, num_beams=2)
    sch = ContinuousScheduler(eng, 8, num_beams=2)
    with pytest.raises(ValueError, match="outside"):
        sch.run(_pixels(3), torch.tensor([5]), BeamSearchParams(2, 6), max_new_tokens=[3, 7, 2])
    with pytest.raises(ValueError, match="num_beams"):
        sch.run(_pixels(3), torch.tensor([5]), BeamSearchParams(4, 6))
    with pytest.raises(ValueError, match="one request per image"):
        sch.run(_pixels(3), torch.tensor([5]), BeamSearchParams(2, 6), n=2)


def test_beam_params_to_c():
    bp = BeamSearchParams(3, 20, do_sample=True, early_stopping="never", eos_token_id=None, pad_token_id=-1,
                          stop_ids=[4, 5], seed=-1).to_c()
    assert (bp.num_beams, bp.max_new_tokens, bp.do_sample, bp.early_stopping) == (3, 20, 1, 2)
    assert (bp.eos_token_id, bp.pad_token_id, bp.n_stop_ids, list(bp.stop_ids)[:2]) == (-1, -1, 2, [4, 5])
    assert bp.seed == 2 ** 64 - 1
    assert BeamSearchParams(2, 5, early_stopping=False).to_c().early_stopping == 0
    with pytest.raises(ValueError):
        BeamSearchParams(2, 5, stop_ids=list(range(9))).to_c()


def test_beam_session_symbols_declared_exported_and_bound():
    assert _lib.ABI_VERSION == 7
    text = open(os.path.join(ROOT, "include", "starvector_b200.h")).read()
    declared = set(re.findall(r"SV_API\s+[\w\s\*]+?\b(sv_\w+)\s*\(", text))
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (sv_\w+)", out))
    for name in ("sv_beam_session_begin", "sv_beam_session_admit"):
        assert name in declared and name in exported and name in _lib.SIGNATURES
    assert _lib.load().sv_abi_version() == 7

"""Speculative sessions without a GPU: the column allocation and the per-row accept walk through their host replays
(sv_spec_session_plan_host / sv_spec_session_tail_host, the code the tail kernel runs), and the scheduler's hint rule
against a stand-in engine."""
import ctypes as C
import random
import types

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200.continuous import ContinuousScheduler, spec_session_k
from starvector_b200.engine import GenerationParams

NEW = ["sv_session_begin_speculative", "sv_session_spec_stats", "sv_spec_session_plan_host", "sv_spec_session_tail_host",
       "sv_op_spec_session_select"]


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_symbols_exported(lib):
    for name in NEW:
        assert name in _lib.SIGNATURES and hasattr(lib, name), name


def _plan_py(S, active, want, budget):
    """DESIGN.md §7i, stated plainly: one column per live row, then one draft per pass, slot order, while columns last."""
    g = [0] * S
    spare = min(budget, S) - sum(1 for a in active if a)
    while spare > 0:
        gave = False
        for r in range(S):
            if spare > 0 and active[r] and g[r] < want[r]:
                g[r] += 1
                spare -= 1
                gave = True
        if not gave:
            break
    first, c = [], 0
    for r in range(S):
        first.append(c if active[r] else -1)
        c += (1 + g[r]) if active[r] else 0
    return g, first, c


def _plan_host(lib, S, active, want, budget):
    A = C.c_int32 * S
    g, first = A(), A()
    n = lib.sv_spec_session_plan_host(S, A(*active), A(*want), budget, g, first)
    return list(g), list(first), n


def test_allocation_matches_the_rule_and_its_invariants(lib):
    rng = random.Random(7)
    for _ in range(3000):
        S = rng.randint(1, 16)
        active = [int(rng.random() < rng.choice([0.2, 0.5, 0.9, 1.0])) for _ in range(S)]
        k = rng.randint(1, 15)
        want = [min(k, rng.randint(0, 16)) if a else rng.randint(0, 3) for a in active]
        budget = rng.choice([S, S, rng.randint(sum(active), 16) if sum(active) else S])
        g, first, n = _plan_host(lib, S, active, want, budget)
        assert (g, first, n) == _plan_py(S, active, want, budget)
        live = [r for r in range(S) if active[r]]
        assert n == sum(1 + g[r] for r in live) <= S
        assert n <= max(budget, len(live))
        c = 0
        for r in range(S):
            if active[r]:
                assert first[r] == c and 0 <= g[r] <= want[r]     # contiguous rows in slot order, no more than wanted
                c += 1 + g[r]
            else:
                assert first[r] == -1 and g[r] == 0
        # round-robin: nobody got two drafts more than a row that still wanted one
        for a in live:
            for b in live:
                if g[a] >= g[b] + 2:
                    assert g[b] == want[b]


def test_full_session_gets_no_drafts(lib):
    g, first, n = _plan_host(lib, 8, [1] * 8, [5] * 8, 8)
    assert g == [0] * 8 and first == list(range(8)) and n == 8


# ---- the accept walk: many verify steps of the host tail against a plain per-row loop --------------------------------
def _plain(seq, cap, eos, stop):
    """What a plain session emits for a row whose model always continues with seq: session_append_token per token."""
    out = []
    for t in seq:
        out.append(t)
        if (eos >= 0 and t == eos) or (stop and out[-len(stop):] == list(stop)) or len(out) >= cap:
            break
    return out


def _run_tail(lib, seqs, caps, params, k, ngram, stride=128, prefix=20, tcap=4096):
    S = len(seqs)
    rows = _lib.SessionRows()
    out = (C.c_int32 * (S * stride))(*([params.pad_token_id] * (S * stride)))
    for r in range(S):            # admission: token 0 selected, row_step 1, finished when it is a stop already
        out[r * stride] = seqs[r][0]
        rows.row_len[r], rows.row_step[r], rows.row_max_new[r] = prefix, 1, caps[r]
        done = _plain(seqs[r][:1], caps[r], params.eos_token_id, params.stop_ids)
        rows.row_active[r] = int(not (len(done) == 1 and (caps[r] == 1 or seqs[r][0] == params.eos_token_id)))
    ss = _lib.SpecSessionState(ncols=S, k=k, max_ngram=ngram)
    cp = params.to_c()
    assert lib.sv_spec_session_tail_host(C.byref(cp), C.byref(rows), out, stride, C.byref(ss), 0, tcap) >= 0
    for _ in range(400):
        if not any(rows.row_active[r] for r in range(S)):
            break
        for c in range(ss.n_live):     # the column's token: the model's continuation after the row's tokens + drafts
            r, j = ss.row[c], ss.off[c]
            ss.sel[c] = seqs[r][rows.row_step[r] + j]
        n = lib.sv_spec_session_tail_host(C.byref(cp), C.byref(rows), out, stride, C.byref(ss), 1, tcap)
        assert 0 <= n <= S
        for c in range(n):           # the map: live rows in slot order, contiguous, at consecutive positions
            r, j = ss.row[c], ss.off[c]
            assert rows.row_active[r] and ss.pos[c] == rows.row_len[r] + j
            assert (j == 0 and ss.tok[c] == out[r * stride + rows.row_step[r] - 1]) or (j > 0 and ss.off[c - 1] == j - 1)
            assert j <= k and rows.row_step[r] + j < rows.row_max_new[r]
    got = [[out[r * stride + i] for i in range(rows.row_step[r])] for r in range(S)]
    return got, rows, ss


@pytest.mark.parametrize("k", [1, 3, 7])
def test_accept_walk_equals_the_plain_loop(lib, k):
    rng = random.Random(k)
    eos, stop = 0, (5, 6)
    params = GenerationParams(max_new_tokens=100, eos_token_id=eos, pad_token_id=1, stop_ids=stop)
    accepted = 0
    for trial in range(40):
        S = rng.randint(2, 8)
        seqs, caps = [], []
        for r in range(S):
            period = [rng.randint(7, 12) for _ in range(rng.randint(2, 5))]
            seq = [period[i % len(period)] if rng.random() < 0.85 else rng.randint(7, 30) for i in range(120)]
            kind = rng.random()
            if kind < 0.3:                              # EOS somewhere in the run (often inside an accepted draft)
                seq[rng.randint(1, 60)] = eos
            elif kind < 0.6:                            # the stop sequence, possibly straddling two verify steps
                at = rng.randint(2, 60)
                seq[at - 1], seq[at] = stop
            seqs.append(seq)
            caps.append(rng.randint(1, 100))
        got, rows, ss = _run_tail(lib, seqs, caps, params, k, ngram=rng.choice([1, 2, 3]))
        for r in range(S):
            assert got[r] == _plain(seqs[r], caps[r], eos, stop), (trial, r)
            assert not rows.row_active[r]
        assert ss.drafted >= ss.accepted
        accepted += ss.accepted
    assert accepted > 0


def test_no_drafts_without_spare_columns(lib):
    params = GenerationParams(max_new_tokens=60, eos_token_id=0, pad_token_id=1)
    S = 4
    rows = _lib.SessionRows()
    out = (C.c_int32 * (S * 64))(*([7, 8] * (S * 32)))
    for r in range(S):
        rows.row_len[r], rows.row_step[r], rows.row_max_new[r], rows.row_active[r] = 30, 20, 60, 1
    ss = _lib.SpecSessionState(ncols=S, k=3, max_ngram=2)
    cp = params.to_c()
    assert lib.sv_spec_session_tail_host(C.byref(cp), C.byref(rows), out, 64, C.byref(ss), 0, 4096) == S
    assert list(ss.off)[:S] == [0] * S and ss.drafted == 0      # every slot busy: no drafts


def test_column_budget_keeps_the_first_rows_prefetch_inside_its_cache_row(lib):
    params = GenerationParams(max_new_tokens=60, eos_token_id=0, pad_token_id=1)
    rows = _lib.SessionRows()
    out = (C.c_int32 * (4 * 64))(*([7, 8] * 128))
    rows.row_len[0], rows.row_step[0], rows.row_max_new[0], rows.row_active[0] = 98, 20, 60, 1
    ss = _lib.SpecSessionState(ncols=4, k=3, max_ngram=2)
    cp = params.to_c()
    n = lib.sv_spec_session_tail_host(C.byref(cp), C.byref(rows), out, 64, C.byref(ss), 0, 100)
    assert n == 2 and ss.pos[0] + n <= 100                     # tcap 100: two columns, not four


# ---- the scheduler's hint rule ----------------------------------------------------------------------------------
class SpecFakeEngine:
    """One slot finishes per step after `length` tokens; records what session_begin was asked."""

    def __init__(self, slots, variant=0, fused=True):
        self.dims = types.SimpleNamespace(max_batch=slots, variant=variant)
        self.fused_decode = fused
        self.begun = []
        self.stats_calls = 0

    def session_begin(self, params, slots):
        self.begun.append((params.prompt_lookup_num_tokens, spec_session_k(params, slots, self)))
        self.S, self.rows = slots, {}

    def session_admit(self, pixels, prompt_ids, slots, *, max_new_tokens, seeds, src):
        for j, s in enumerate(slots):
            self.rows[s] = max_new_tokens[j]

    def session_run(self, max_steps):
        fin = [s in self.rows for s in range(self.S)]
        lens = [self.rows.get(s, 0) for s in range(self.S)]
        return 1, fin, lens

    def session_read(self, slot):
        return torch.zeros(self.rows.pop(slot), dtype=torch.int32)

    def session_spec_stats(self):
        self.stats_calls += 1
        return {"steps": 1, "drafted": 2, "accepted": 1}

    def session_end(self):
        pass


def _px(n):
    return torch.zeros(n, 3, 2, 2)


@pytest.mark.parametrize("slots,variant,fused,k,expect", [
    (8, 0, True, 3, 3), (8, 0, True, 20, 7), (2, 0, True, 5, 1), (1, 0, True, 3, 0),
    (8, 1, True, 3, 0), (8, 0, False, 3, 0), (8, 0, True, 0, 0)])
def test_hint_rule(slots, variant, fused, k, expect):
    eng = SpecFakeEngine(slots, variant, fused)
    params = GenerationParams(max_new_tokens=4, prompt_lookup_num_tokens=k)
    sched = ContinuousScheduler(eng)
    out = sched.run(_px(3), torch.tensor([1]), params)
    assert [len(o) for o in out] == [4, 4, 4]
    assert eng.begun == [(k, expect)]
    assert (eng.stats_calls == 1) == (expect > 0)
    assert ("spec" in sched.stats) == (expect > 0)


def test_plain_params_need_no_engine_attributes():
    """Without the hint the rule reads nothing from the engine (stand-ins without dims.variant keep working)."""
    assert spec_session_k(GenerationParams(max_new_tokens=4), 8, object()) == 0

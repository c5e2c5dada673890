"""CPU checks of prompt-lookup speculative decoding (`sv_generate_speculative`, DESIGN.md §7g) through the host replays of
the device rules: the draft rule against transformers' `PromptLookupCandidateGenerator.get_candidates`, and the accept
walk against a plain one-token-per-step loop over a symbolic next-token function."""
import ctypes as C
import os
import random
import re
import subprocess

import pytest
import torch
from transformers.generation.candidate_generator import PromptLookupCandidateGenerator

from starvector_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPEC_SYMBOLS = ("sv_generate_speculative", "sv_last_spec_stats", "sv_spec_verify_step", "sv_spec_draft_host",
                "sv_spec_accept_host")


def test_spec_symbols_exported():
    header = open(os.path.join(ROOT, "include", "starvector_b200.h")).read()
    declared = set(re.findall(r"SV_API\s+[\w\s\*]+?\b(sv_\w+)\s*\(", header))
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    for name in SPEC_SYMBOLS:
        assert name in declared and name in exported and name in _lib.SIGNATURES, name
    assert C.sizeof(_lib.SpecParams) == 8
    assert _lib.load().sv_abi_version() == _lib.ABI_VERSION == 7     # new entry points only: no existing one changed


def draft(hist, k, g, eos=-1, budget=1 << 30):
    lib = _lib.load()
    arr = (C.c_int32 * max(len(hist), 1))(*hist)
    out = (C.c_int32 * max(k, 1))()
    m = lib.sv_spec_draft_host(arr, len(hist), k, g, eos, budget, out)
    assert 0 <= m <= k
    return list(out[:m])


def hf_draft(hist, k, g, eos):
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor([eos]), num_output_tokens=k, max_matching_ngram_size=g,
                                         max_length=1 << 30)
    ids, _ = gen.get_candidates(torch.tensor([hist], dtype=torch.long))
    return ids[0, len(hist):].tolist()


def _histories():
    rng = random.Random(7)
    hs = [[5], [5, 5], [1, 2, 3, 4, 5, 6], list(range(40))]                  # too short, self-match only, no match
    for _ in range(150):                                                      # seeded random over small alphabets
        n, a = rng.randint(2, 60), rng.randint(2, 6)
        hs.append([rng.randrange(a) for _ in range(n)])
    for _ in range(60):                                                       # highly repetitive: noisy periodic text
        period = [rng.randrange(50) for _ in range(rng.randint(1, 9))]
        h = [period[i % len(period)] for i in range(rng.randint(3, 90))]
        for _ in range(rng.randint(0, 3)):
            h[rng.randrange(len(h))] = rng.randrange(50)
        hs.append(h)
    return hs


@pytest.mark.parametrize("g", [1, 2, 3])
def test_draft_rule_matches_transformers(g):
    rng = random.Random(g)
    n_drafts = 0
    for h in _histories():
        k = rng.randint(1, 15)
        eos = rng.choice([0, 1, 3, 99])                                       # 99 never occurs: no EOS crop
        ref = hf_draft(h, k, g, eos)
        assert draft(h, k, g, eos) == ref, (h, k, g, eos)
        n_drafts += bool(ref)
    assert n_drafts > 50


def test_draft_rule_cases():
    assert draft([7, 8, 9, 7, 8], 4, 2) == [9, 7, 8]                          # continuation shorter than k
    assert draft([7, 8, 9, 7, 8], 1, 2) == [9]
    assert draft([1, 2, 3, 4], 3, 2) == []                                     # no match
    assert draft([4, 1, 2, 0, 6, 4, 1, 2], 5, 3, eos=0) == []                  # EOS first: HF keeps no candidate
    assert draft([4, 1, 2, 5, 0, 6, 4, 1, 2], 5, 3, eos=0) == [5]              # cropped at the first EOS
    assert hf_draft([4, 1, 2, 5, 0, 6, 4, 1, 2], 5, 3, 0) == [5]
    # the larger n-gram wins even when a smaller one matches earlier
    assert draft([2, 9, 5, 1, 2, 7, 1, 2], 3, 2) == [7, 1, 2] == hf_draft([2, 9, 5, 1, 2, 7, 1, 2], 3, 2, 99)
    h = [3, 1, 4, 1, 5, 9, 2, 6] * 4
    full = draft(h, 15, 2)
    assert len(full) == 15
    for b in range(0, 16):                                                     # the remaining-budget clamp
        assert draft(h, 15, 2, budget=b) == full[:b]


# ---- accept walk: symbolic next-token functions, plain loop vs draft + accept replays ---------------------------------
def next_token_fn(seed, period, noise):
    """A deterministic 'model': mostly a periodic text, with hash noise that depends on the whole history and the step
    (the counter a sampled token depends on), so drafts get accepted and rejected."""
    rng = random.Random(seed)
    text = [rng.randrange(2, 40) for _ in range(period)]

    def f(hist):
        n = len(hist)
        if hash((seed, tuple(hist[-4:]), n)) % 100 < noise:
            return 2 + hash((seed, n, tuple(hist[-2:]))) % 38
        return text[n % period]
    return f


def plain_run(f, max_new, eos, stop):
    out = []
    while True:
        t = f(out)
        out.append(t)
        if (eos >= 0 and t == eos) or (stop and out[-len(stop):] == stop) or len(out) >= max_new:
            return out


def spec_run(f, max_new, eos, stop, k, g=2, prefix=30):
    lib = _lib.load()
    p = _lib.GenParams(max_new_tokens=max_new, eos_token_id=eos, pad_token_id=1, n_stop_ids=len(stop), stop_row0_only=1)
    for i, s in enumerate(stop):
        p.stop_ids[i] = s
    state = (C.c_int32 * 3)(prefix, 0, 0)                                      # cur_len, step, done
    out = (C.c_int32 * max_new)()
    steps, accepted, straddle = 0, 0, False
    hist = []
    while not state[2]:
        step0 = state[1]
        drafts = draft(hist, k, g, eos, budget=max_new - step0 - 1) if hist else []
        cols = ([hist[-1]] if hist else [0]) + drafts
        sel = [f(hist + drafts[:c]) for c in range(len(cols))]
        m = lib.sv_spec_accept_host(C.byref(p), state, out, max_new, (C.c_int32 * 16)(*sel), (C.c_int32 * 16)(*cols),
                                    len(cols))
        assert 1 <= m <= len(cols) and state[1] == step0 + m and state[0] == prefix + state[1]
        hist = list(out[:state[1]])
        steps += 1
        accepted += m - 1
        if stop and hist[-len(stop):] == stop and state[1] - len(stop) < step0 < state[1]:
            straddle = True
    return hist, steps, accepted, straddle


@pytest.mark.parametrize("k", list(range(1, 16)))
def test_accept_walk_equals_plain_decoding(k):
    straddles = 0
    for seed in range(12):
        f = next_token_fn(seed, period=3 + seed % 5, noise=[0, 5, 20, 50][seed % 4])
        toks = plain_run(f, 400, -1, [])
        eos = toks[len(toks) // 3]                                             # an EOS in the middle of the run
        stop = toks[150:153] if seed % 2 else toks[90:92]                      # stop pairs / triples that occur
        for max_new, e, st in ((400, -1, []), (400, eos, []), (400, -1, stop), (97 + seed, -1, []), (1, -1, []),
                               (2, -1, [])):
            ref = plain_run(f, max_new, e, st)
            got, steps, accepted, straddle = spec_run(f, max_new, e, st, k)
            assert got == ref, (seed, max_new, e, st)
            straddles += straddle
            if e < 0 and not st and max_new == 400 and seed % 4 == 0:          # noiseless text: most drafts are taken
                assert accepted > 0 and steps < len(ref) // (k + 1) + 16
    if k > 1:
        assert straddles > 0                                                   # a stop sequence crossed a step boundary


def test_accept_host_rejects_bad_arguments():
    lib = _lib.load()
    p = _lib.GenParams(max_new_tokens=8)
    st, out, z = (C.c_int32 * 3)(), (C.c_int32 * 8)(), (C.c_int32 * 16)()
    assert lib.sv_spec_accept_host(C.byref(p), st, out, 8, z, z, 17) == _lib.SV_ERR_INVALID
    assert lib.sv_spec_accept_host(C.byref(p), st, out, 7, z, z, 1) == _lib.SV_ERR_INVALID
    assert lib.sv_spec_draft_host(z, 4, 3, 0, -1, 4, z) == _lib.SV_ERR_INVALID

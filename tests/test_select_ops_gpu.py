"""The token-selection kernels one launch at a time (sv_op_select, sv_op_beam_candidates), at the shipped vocabularies
(49156, 49157) and at sizes where the sampler's per-thread id ranges degenerate (500, 1000, 1024, 1025).

References, all in this file:
  * a NumPy Philox4x32-10 (Random123 definition, checked against its known-answer vector) gives the uniform `u` every
    (seed, row, step) must draw: rectangle batches use the counter (row, step), session rows (0, row_step) under the
    row's own seed;
  * transformers' RepetitionPenaltyLogitsProcessor / TemperatureLogitsWarper on `logits.float()` and a softmax in fp64
    give the distribution; the nucleus is the kernel's documented rule "kept iff the mass of strictly more probable
    tokens is < top_p" (all members of a tie share their fate), cross-checked against TopPLogitsWarper, whose sort keeps
    only some members of a tie at the cut;
  * the HF `_sample` loop body with EosTokenCriteria / MaxLengthCriteria and the reference's row-0 stop rule, restated in
    Python, steps alongside the kernels.

The draw check: the emitted token's fp64 CDF interval (ids in ascending order over the kept set), widened by DELTA_CDF, must
contain `u`.  Ids whose strictly-greater mass is within DELTA_G of top_p, or whose probability is less than BISECT below
the cut (the kernel bisects the threshold 30 times: 2^-30), may or may not be kept: every threshold set in that band is
tried.  Calibrated on an H100 SXM 80 GB (700 W): over about 1.1 million draws the worst distance was 2.9e-7 (DELTA_CDF = 2e-6); the beam
log-probs were within 9.5e-7 of fp64 (tolerance 2e-5).  The CALIB lines printed with -s give the worst case of every test.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                    TopPLogitsWarper)
from transformers.generation.stopping_criteria import EosTokenCriteria, MaxLengthCriteria

from starvector_b200 import _lib
from starvector_b200 import engine as E
from starvector_b200.engine import GenerationParams

pytestmark = pytest.mark.gpu
DEV = "cuda"
GREEDY, SAMPLE, FUSED = _lib.SV_SELECT_GREEDY, _lib.SV_SELECT_SAMPLE, _lib.SV_SELECT_FUSED
DELTA_G = 2e-6          # fp32 slack of a 49k-term mass sum against top_p
BISECT = 2.0 ** -29     # the 2^-30 bisection floor, with one bit to spare
DELTA_CDF = 2e-6        # distance of u outside the token's fp64 CDF interval (fp32 scan, __expf)
VOCABS = [49156, 49157, 500, 1000, 1024, 1025]
SAMPLE_PARAMS = [(1.0, 1.0), (0.25, 0.9), (0.9, 0.8), (1.5, 0.95), (1.0, 0.5)]     # (temperature, top_p)


def _calib(name, worst, tol):
    print(f"CALIB {name}: worst = {worst:.3e} (tolerance {tol:.1e}, ratio {worst / tol:.3f})")


# ---- Philox4x32-10 (Random123) ---------------------------------------------------------------------------------------
def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (or ints), key: two ints -> four uint32 arrays."""
    m32 = np.uint64(0xFFFFFFFF)
    x = [np.asarray(c, dtype=np.uint64) & m32 for c in np.broadcast_arrays(*ctr)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * x[0], np.uint64(0xCD9E8D57) * x[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & m32, p1 >> np.uint64(32), p1 & m32
        x = [hi1 ^ x[1] ^ np.uint64(k0), lo1, hi0 ^ x[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return x


def _u01(x0):
    """The engine's mapping of the first output word to (0, 1], in fp32."""
    return (((x0 >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def sampler_u(seed, c0, c1):
    return _u01(philox4x32_10((c0, c1, 0x5356, 0x42323030), (seed & 0xFFFFFFFF, seed >> 32))[0])


def beam_gumbel(seed, step, row, token):
    u = _u01(philox4x32_10((np.asarray(token) + ((row >> 3) << 24), step * 8 + (row & 7), 0x4245414D, 0x53563032),
                           (seed & 0xFFFFFFFF, seed >> 32))[0])
    return -np.log(-np.log(u.astype(np.float64)))


def test_philox_known_answers():
    assert [int(v) for v in philox4x32_10((0, 0, 0, 0), (0, 0))] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    ff = 0xFFFFFFFF
    assert [int(v) for v in philox4x32_10((ff, ff, ff, ff), (ff, ff))] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    u = sampler_u(7, np.arange(4), 3)
    assert u.dtype == np.float32 and len(set(u.tolist())) == 4 and (u > 0).all() and (u <= 1).all()


# ---- logit families ----------------------------------------------------------------------------------------------------
def _last_range(V):
    """First id of the last non-empty per-thread range of the sampler (1024 threads, ceil(V / 1024) ids each)."""
    per = (V + 1023) // 1024
    return ((V + per - 1) // per - 1) * per


def _with_mass(tail, ids, masses):
    """Set logits[ids[j]] so that token j holds about masses[j] of the row (the tail shares the remainder)."""
    row = tail.clone()
    mask = torch.ones_like(row, dtype=torch.bool)
    mask[ids] = False
    lse = torch.logsumexp(row[mask & torch.isfinite(row)], 0)
    rest = 1.0 - float(sum(masses))
    for i, m in zip(ids, masses):
        row[i] = lse + math.log(m / rest)
    return row


def make_rows(V, seed):
    """16 fp32 logit rows, one to four of each family (see FAMILIES); values are bf16-representable."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda s=1.0: torch.randn(V, generator=g, dtype=torch.float64) * s
    pick = lambda n: torch.randperm(V, generator=g)[:n].tolist()
    last0 = _last_range(V)
    rows = []
    for k in range(4):                                  # peaked: a few tokens hold most of the mass, long tail
        rows.append(_with_mass(rn(2.0), pick(6), [0.4, 0.2, 0.1, 0.05, 0.03, 0.02]))
    for k in range(2):                                  # flat: |logit| < 0.05
        rows.append((torch.rand(V, generator=g, dtype=torch.float64) - 0.5) * 0.098)
    for k in range(2):                                  # exact 48-way tie astride every top_p cut in SAMPLE_PARAMS at T = 1
        ids = [0, V - 1, 31, 32, 1023 % V, 1024 % V] + pick(60)
        ids = list(dict.fromkeys(ids))[:49]
        rows.append(_with_mass(rn(0.5), ids, [0.3] + [0.6 / 48] * 48))
    for k in range(2):                                  # the top token alone exceeds every top_p < 1
        rows.append(_with_mass(rn(1.0), pick(1), [0.97]))
    rows.append(_with_mass(rn(1.0), [V - 1], [0.999]))    # the mass at the last id
    r = rn(1.0) - 30.0                                  # the mass inside the last thread's short range
    r[last0:] += 38.0
    rows.append(r)
    for k in range(2):                                  # -inf entries, among them id 0, id V - 1 and a would-be winner
        r = _with_mass(rn(2.0), pick(4), [0.3, 0.25, 0.2, 0.1])
        r[torch.rand(V, generator=g) < 0.3] = -math.inf
        r[0] = r[V - 1] = -math.inf
        r[pick(1)] = 9.0
        rows.append(r)
    for k in range(2):                                  # +-60: exp() of the raw logits over / underflows
        rows.append((torch.rand(V, generator=g, dtype=torch.float64) - 0.5) * 120.0)
    return torch.stack(rows).bfloat16().float()


FAMILIES = ["peaked"] * 4 + ["flat"] * 2 + ["tie"] * 2 + ["dominant"] * 2 + ["last_id", "last_range"] + ["neg_inf"] * 2 + ["large"] * 2


# ---- the fp64 reference of the HF chain ------------------------------------------------------------------------------------
def hf_scores(logits_f32, seen_ids, T, rp):
    """transformers' processors on one fp32 row, in the order `_sample` applies them."""
    s = logits_f32[None].clone()
    ids = seen_ids[None].long()
    if rp != 1.0:
        s = RepetitionPenaltyLogitsProcessor(rp)(ids, s)
    if T != 1.0:
        s = TemperatureLogitsWarper(T)(ids, s)
    return s[0]


class RowRef:
    """fp64 distribution of one row and the threshold sets the kernel may keep (one, unless ids fall in the band)."""

    def __init__(self, scores_f32, top_p):
        P = torch.softmax(scores_f32.double(), 0)
        self.P = P
        if top_p >= 1.0:
            self.definite, self.ambiguous = P > 0, torch.zeros_like(P, dtype=torch.bool)
            self.sets = [self.definite]
            return
        vals, inv = torch.unique(P, return_inverse=True)                       # ascending
        mass = torch.zeros_like(vals).index_add_(0, inv, P)
        G = (torch.flip(torch.cumsum(torch.flip(mass, [0]), 0), [0]) - mass)[inv]   # mass of strictly more probable ids
        self.G = G
        self.definite = G < top_p - DELTA_G
        p_cut = P[G <= top_p + DELTA_G].min()
        self.ambiguous = ~self.definite & ((G <= top_p + DELTA_G) | (P > p_cut - BISECT)) & (P > 0)
        levels = torch.unique(P[self.ambiguous]).flip(0)
        assert len(levels) <= 64, "too many distinct probabilities inside the tolerance band for an exact check"
        self.sets = [self.definite] + [self.definite | (self.ambiguous & (P >= c)) for c in levels]

    def excess(self, toks, us):
        """Per draw: how far u lies outside the token's CDF interval, for the best admissible kept set (inf: never kept)."""
        best = torch.full((len(toks),), math.inf, dtype=torch.float64, device=self.P.device)
        u = torch.as_tensor(us, dtype=torch.float64, device=self.P.device)
        for S in self.sets:
            pS = torch.where(S, self.P, torch.zeros_like(self.P))
            Z = pS.sum()
            cdf = torch.cumsum(pS, 0) / Z
            hi = cdf[toks]
            lo = hi - pS[toks] / Z
            ex = torch.clamp(torch.maximum(lo - u, u - hi), min=0.0)
            ex[~S[toks]] = math.inf
            best = torch.minimum(best, ex)
        return best

    def check_against_transformers(self, scores_f32, top_p):
        """TopPLogitsWarper keeps a subset of definite + ambiguous; what it drops from `definite` ties with its smallest kept."""
        if top_p >= 1.0:
            return
        hf = torch.isfinite(TopPLogitsWarper(top_p)(None, scores_f32[None].clone())[0])
        loose_hi, loose_lo = self.G <= top_p + 2e-5, self.G < top_p - 2e-5       # HF's own cumsum is fp32
        assert not (hf & ~loose_hi & ~self.ambiguous).any()
        dropped = loose_lo & ~hf
        assert (scores_f32[dropped] == scores_f32[hf].min()).all()


# ---- running the op --------------------------------------------------------------------------------------------------------
def _plain_state(B, step=0, cur_len=5, done=0, unfinished=None):
    return dict(step=step, cur_len=cur_len, done=done, unfinished=list(unfinished or [1] * B))


def _row_state(B, row_len=None, row_step=None, active=None, max_new=None, seeds=None, mask=0xFFFF, event=0):
    return dict(row_len=list(row_len or [5] * B), row_step=list(row_step or [0] * B), row_active=list(active or [1] * B),
                row_max_new=list(max_new or [1 << 20] * B), row_seed=list(seeds or [0] * B), row_mask=mask, event=event)


def run_sampler(logits, T, top_p, rp, nsteps, per_row, seed=1234, step0=3, seen=None, row_steps=None, seeds=None):
    """nsteps draws per row -> (tokens [B, nsteps] on the CPU, u [B, nsteps] from the NumPy Philox, seen after)."""
    B, V = logits.shape
    row_steps = row_steps or [step0 + 2 * b for b in range(B)]
    seeds = seeds or [seed + 1000003 * b for b in range(B)]
    stride = (max(row_steps) if per_row else step0) + nsteps
    out = torch.full((B, stride), -7, dtype=torch.int32, device=DEV)
    nxt = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    seen = torch.zeros(B, V, dtype=torch.uint8, device=DEV) if seen is None else seen.clone()
    p = GenerationParams(max_new_tokens=stride, do_sample=True, temperature=T, top_p=top_p, repetition_penalty=rp,
                         eos_token_id=None, pad_token_id=0, seed=seed)
    s = np.arange(nsteps)
    if per_row:
        st = _row_state(B, row_step=row_steps, seeds=seeds)
        E.op_select(SAMPLE, logits, p, seen, out, nxt, st, per_row=True, nsteps=nsteps)
        toks = torch.stack([out[b, row_steps[b]:row_steps[b] + nsteps] for b in range(B)])
        us = np.stack([sampler_u(seeds[b], 0, row_steps[b] + s) for b in range(B)])
        assert st["row_step"] == [r + nsteps for r in row_steps] and st["row_active"] == [1] * B
    else:
        st = _plain_state(B, step=step0)
        E.op_select(SAMPLE, logits, p, seen, out, nxt, st, nsteps=nsteps)
        toks = out[:, step0:step0 + nsteps]
        us = np.stack([sampler_u(seed, b, step0 + s) for b in range(B)])
        assert st["step"] == step0 + nsteps
    assert torch.equal(nxt, toks[:, -1])
    return toks.long(), us, seen


def check_static(rows_f32, toks, us, T, top_p, name):
    """Draw check when the distribution does not change between draws (no repetition penalty)."""
    worst = 0.0
    none = torch.zeros(0, dtype=torch.long, device=DEV)
    for b in range(rows_f32.shape[0]):
        sc = hf_scores(rows_f32[b], none, T, 1.0)
        ref = RowRef(sc, top_p)
        ref.check_against_transformers(sc, top_p)
        ex = ref.excess(toks[b], us[b])
        bad = (ex > DELTA_CDF).nonzero().flatten()
        assert len(bad) == 0, (f"{name} row {b} ({FAMILIES[b % 16]}): {len(bad)} of {len(ex)} draws outside their CDF interval; first: "
                               f"draw {int(bad[0])} token {int(toks[b, bad[0]])} u {us[b, bad[0]]:.8f} excess {float(ex[bad[0]]):.3e}")
        worst = max(worst, float(ex.max()))
    return worst


# ---- sampling ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_row", [False, True], ids=["plain", "rows"])
@pytest.mark.parametrize("T,top_p", SAMPLE_PARAMS, ids=str)
@pytest.mark.parametrize("V", [49156, 49157])
def test_sampler_draws_follow_philox_and_fp64_cdf(V, T, top_p, per_row):
    """16 rows (every family) x 2048 draws: each token's CDF interval contains the u of its (seed, row, step)."""
    rows = make_rows(V, seed=V).to(DEV)
    toks, us, _ = run_sampler(rows.bfloat16(), T, top_p, 1.0, 2048, per_row)
    worst = check_static(rows, toks, us, T, top_p, f"V={V} T={T} top_p={top_p}")
    _calib(f"sampler V={V} T={T} top_p={top_p} {'rows' if per_row else 'plain'} ({toks.numel()} draws)", worst, DELTA_CDF)


@pytest.mark.parametrize("V", [500, 1000, 1024, 1025])
def test_sampler_draws_small_vocabularies(V):
    """per = 1 (threads >= V own nothing), V = 1024 exactly, and per = 2 where id 1024 sits alone in thread 512."""
    rows = make_rows(V, seed=V).to(DEV)
    worst = 0.0
    for T, top_p in SAMPLE_PARAMS:
        for per_row in (False, True):
            toks, us, _ = run_sampler(rows.bfloat16(), T, top_p, 1.0, 512, per_row)
            worst = max(worst, check_static(rows, toks, us, T, top_p, f"V={V} T={T} top_p={top_p}"))
    _calib(f"sampler V={V}", worst, DELTA_CDF)


@pytest.mark.parametrize("per_row", [False, True], ids=["plain", "rows"])
@pytest.mark.parametrize("V,T,top_p", [(49156, 0.9, 0.8), (49157, 1.0, 1.0), (1025, 1.5, 0.95)], ids=str)
def test_sampler_with_repetition_penalty_replays_seen(V, T, top_p, per_row):
    """rp = 1.3: every drawn token changes the row's distribution; the reference replays `seen` draw by draw."""
    rp, n = 1.3, 96
    rows = make_rows(V, seed=V + 1).to(DEV)
    g = torch.Generator().manual_seed(V)
    seen0 = (torch.rand(16, V, generator=g) < 0.05).to(torch.uint8).to(DEV)
    seen0[torch.arange(16), rows.argmax(1)] = 1                       # the favourite is penalised from the start
    toks, us, seen1 = run_sampler(rows.bfloat16(), T, top_p, rp, n, per_row, seen=seen0)
    worst = 0.0
    for b in range(16):
        seen, ref = seen0[b].bool().clone(), None
        for s in range(n):
            if ref is None:
                ref = RowRef(hf_scores(rows[b], seen.nonzero().flatten(), T, rp), top_p)
            t = toks[b, s:s + 1]
            ex = float(ref.excess(t, us[b, s:s + 1])[0])
            assert ex <= DELTA_CDF, f"row {b} ({FAMILIES[b]}) draw {s}: token {int(t)} u {us[b, s]:.8f} excess {ex:.3e}"
            worst = max(worst, ex)
            if not seen[t]:
                seen[t], ref = True, None
        assert torch.equal(seen.to(torch.uint8), seen1[b])
    _calib(f"sampler rp=1.3 V={V} T={T} top_p={top_p}", worst, DELTA_CDF)


def test_sampler_streams_are_per_row_per_step_and_batch_independent():
    V = 49157
    flat = make_rows(V, seed=5)[4:5].repeat(16, 1).bfloat16().to(DEV)          # 16 copies of one flat row
    t16, us, _ = run_sampler(flat, 1.0, 1.0, 1.0, 64, False)
    assert len(set(us.flatten().tolist())) == us.size                        # no (row, step) shares a draw
    assert len(set(t16[:, 0].tolist())) > 12 and len(set(t16[0].tolist())) > 48
    t8, _, _ = run_sampler(flat[:8], 1.0, 1.0, 1.0, 64, False)
    assert torch.equal(t8, t16[:8])
    # a session row at slot 11 with seed s and step r = row 0 of a one-row generate with seed s at step r
    seeds, steps = [100 + b for b in range(16)], [0] * 11 + [9] + [0] * 4
    trow, _, _ = run_sampler(flat, 0.9, 0.95, 1.0, 64, True, row_steps=steps, seeds=seeds)
    tone, _, _ = run_sampler(flat[:1], 0.9, 0.95, 1.0, 64, False, seed=seeds[11], step0=9)
    assert torch.equal(trow[11], tone[0])


def test_sampler_exact_edges():
    for V in (49156, 1025, 500):
        rows = make_rows(V, seed=V + 2).to(DEV)
        lg = rows.bfloat16()
        # top_p = 1 keeps everything with p > 0: -inf logits are never drawn
        toks, _, _ = run_sampler(lg, 1.0, 1.0, 1.0, 1024, False)
        assert torch.isfinite(rows.gather(1, toks)).all()
        # a top token above top_p is always returned (dominant rows and the last id)
        toks, _, _ = run_sampler(lg, 1.0, 0.9, 1.0, 256, True)
        for b in (8, 9, 10):
            assert (toks[b] == rows[b].argmax()).all(), (V, b)
        # the only kept mass inside the last thread's range
        assert (toks[11] >= _last_range(V)).all()
        # the tie at the cut: every tied member is drawable and nothing below the tie is drawn
        toks, _, _ = run_sampler(lg, 1.0, 0.5, 1.0, 2048, False)
        for b in (6, 7):
            top = rows[b].argmax()
            tied = (rows[b] == rows[b][rows[b] < rows[b].max()].max()).nonzero().flatten()
            assert len(tied) == 48
            drawn = set(toks[b].tolist())
            assert drawn == set(tied.tolist()) | {int(top)}, (V, b, len(drawn))


def test_sampler_frequencies_match_fp64_distribution():
    """Independent of the Philox reference: 32768 draws of one peaked row against its fp64 nucleus distribution."""
    V, T, top_p = 49156, 0.9, 0.95
    row = make_rows(V, seed=11)[0].to(DEV)
    toks, _, _ = run_sampler(row[None].repeat(16, 1).bfloat16(), T, top_p, 1.0, 2048, False)
    ref = RowRef(hf_scores(row, torch.zeros(0, dtype=torch.long, device=DEV), T, 1.0), top_p)
    q = torch.where(ref.sets[0], ref.P, torch.zeros_like(ref.P))
    q = q / q.sum()
    emp = torch.bincount(toks.flatten(), minlength=V).double() / toks.numel()
    top = torch.topk(q, 12).indices
    tv = 0.5 * ((emp[top] - q[top]).abs().sum() + abs((1 - emp[top].sum()) - (1 - q[top].sum())))
    assert (emp[~(ref.sets[-1])] == 0).all()
    _calib("sampler frequencies, total variation over the 12 top ids + rest", float(tv), 0.015)
    assert tv < 0.015


# ---- greedy ------------------------------------------------------------------------------------------------------------------
def _first_max(v):
    return int((v == v.max()).nonzero()[0])


def greedy_rows(V, seed):
    """16 rows with planted exact ties -> (bf16 logits, seen, rp); the answer comes from the fp32 reference below."""
    g = torch.Generator().manual_seed(seed)
    lg = (torch.randn(16, V, generator=g) * 2).bfloat16().float().clamp(-7, 7)
    seen = (torch.rand(16, V, generator=g) < 0.1).to(torch.uint8)
    far = min(V - 1, 1024 + 37)
    plants = [([0, V - 1], 9.0), ([V - 1], 9.0), ([37, 37 + 32], 9.0), ([37 + 64, 37], 9.0), ([far, 37], 9.0),
              ([V - 1, V - 2, 5], 9.0), ([3, 4], -0.5), ([V // 2, V // 2 + 1], 9.0)]
    for b, (ids, val) in enumerate(plants):
        if val < 0:
            lg[b] = lg[b].clamp(max=-1.0)
        lg[b, ids] = val
        seen[b, ids] = 0
    # rows 8-15: the would-be winner is marked seen, for both signs of its logit; 12-13: the penalty creates a tie
    for b in range(8, 12):
        lg[b] = lg[b].clamp(-7, 6) if b % 2 == 0 else lg[b].clamp(-7, -2)
        w = 11 * b
        lg[b, w] = 6.5 if b % 2 == 0 else -1.5
        lg[b, w + 40] = 6.0 if b % 2 == 0 else -1.75
        seen[b, w], seen[b, w + 40] = 1, 0
    for b in (12, 13):                                    # 8 / 2 == 4 (seen) ties with an unseen 4 at a lower / higher id
        lg[b] = lg[b].clamp(-7, 3)
        a, c = (70, 200) if b == 12 else (200, 70)
        lg[b, a], lg[b, c] = 8.0, 4.0
        seen[b, a], seen[b, c] = 1, 0
    for b in (14, 15):                                    # -1 * 2 (seen) ties with an unseen -2
        lg[b] = lg[b].clamp(-7, -3)
        a, c = (90, 300) if b == 14 else (300, 90)
        lg[b, a], lg[b, c] = -1.0, -2.0
        seen[b, a], seen[b, c] = 1, 0
    return lg.bfloat16(), seen


def greedy_reference(lg_bf16, seen, rp):
    v = lg_bf16.float()
    pen = torch.where(v < 0, v * rp, v / rp)
    v = torch.where(seen.bool(), pen, v) if rp != 1.0 else v
    return [_first_max(v[b]) for b in range(v.shape[0])]


def _select_once(impl, per_row, lg, seen, rp, wte=None, wpe=None, amax=None, cur_len=5, n_positions=64):
    B, V = lg.shape
    out = torch.full((B, 4), -7, dtype=torch.int32, device=DEV)
    nxt = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    seen = seen.clone()
    p = GenerationParams(max_new_tokens=4, repetition_penalty=rp, eos_token_id=None, pad_token_id=0)
    st = _row_state(B, row_len=[cur_len + b for b in range(B)], max_new=[4] * B) if per_row else _plain_state(B, cur_len=cur_len)
    x = torch.full((B, wte.shape[1]), 7.0, dtype=torch.bfloat16, device=DEV) if wte is not None else None
    E.op_select(impl, lg, p, seen, out, nxt, st, per_row=per_row, wte=wte, wpe=wpe, x=x, amax=amax, n_positions=n_positions)
    assert torch.equal(out[:, 0], nxt) and (out[:, 1:] == -7).all()
    return nxt.tolist(), seen, x, st


@pytest.mark.parametrize("rp", [1.0, 2.0, 1.3])
@pytest.mark.parametrize("V", VOCABS)
def test_greedy_first_maximum_of_penalised_logits(V, rp):
    lg, seen = greedy_rows(V, seed=V)
    want = greedy_reference(lg, seen, rp)
    if rp == 2.0:
        assert want[12] == 70 and want[13] == 70 and want[14] == 90 and want[15] == 90      # the penalty-made ties
        assert want[8] != 88 and want[9] == 99 + 40
    lg, seen = lg.to(DEV), seen.to(DEV)
    h = 64
    wte = torch.randn(V, h, device=DEV).bfloat16()
    for B in (1, 8, 9, 16):
        for impl in (GREEDY, FUSED):
            for per_row in (False, True):
                rows = slice(16 - B, 16) if B < 16 else slice(0, 16)
                got, seen_after, _, _ = _select_once(impl, per_row, lg[rows].contiguous(), seen[rows].contiguous(), rp,
                                                     wte=wte if impl == FUSED else None)
                assert got == want[rows], (V, rp, B, impl, per_row)
                exp_seen = seen[rows].clone()
                exp_seen[torch.arange(B), torch.tensor(got)] = 1
                assert torch.equal(seen_after, exp_seen)
    if rp == 1.0:                                                      # rows 0-7 on their own (ties, no penalty)
        got, _, _, _ = _select_once(GREEDY, False, lg[:8].contiguous(), seen[:8].contiguous(), rp)
        assert got == want[:8]


@pytest.mark.parametrize("B", [1, 8, 9, 16])
def test_fused_reads_partials_only_without_penalty(B):
    """Partials in the lm_head's layout [ntiles][row stride]: ties go to the lower id; with a penalty the logits row decides."""
    V, h = 49156, 64
    lib = _lib.load()
    nt, stride = lib.sv_op_ring_ntiles(V), lib.sv_op_ring_row_stride(B)
    assert stride == (8 if B <= 8 else 16) and nt >= 1
    g = torch.Generator().manual_seed(B)
    lg = (torch.randn(B, V, generator=g)).bfloat16().to(DEV)
    seen = torch.zeros(B, V, dtype=torch.uint8, device=DEV)
    val = torch.full((nt, stride), -1e30, dtype=torch.float32)
    idx = torch.randint(0, V, (nt, stride), generator=g, dtype=torch.int32)
    want = []
    for b in range(B):
        tiles = torch.randperm(nt, generator=g)[:3].tolist()
        ids = sorted(torch.randperm(V, generator=g)[:3].tolist())
        val[tiles[0], b], idx[tiles[0], b] = 50.0, ids[2]
        val[tiles[1], b], idx[tiles[1], b] = 50.0, ids[0]               # the same value at a lower id, in another tile
        val[tiles[2], b], idx[tiles[2], b] = 49.75, ids[1]
        want.append(ids[0])
    wte = torch.randn(V, h, device=DEV).bfloat16()
    amax = (val.to(DEV), idx.to(DEV))
    for per_row in (False, True):
        got, _, _, _ = _select_once(FUSED, per_row, lg, seen, 1.0, wte=wte, amax=amax)
        assert got == want                                             # disagrees with the logits row: the partials were read
        assert got != greedy_reference(lg.cpu(), seen.cpu(), 1.0)
        got, _, _, _ = _select_once(FUSED, per_row, lg, seen, 1.3, wte=wte, amax=amax)
        assert got == greedy_reference(lg.cpu(), seen.cpu(), 1.3)


@pytest.mark.parametrize("use_wpe", [True, False], ids=["wpe", "rope"])
def test_fused_embedding_bitwise(use_wpe):
    V, h, npos, B = 1000, 256, 12, 16
    g = torch.Generator().manual_seed(3)
    lg = torch.randn(B, V, generator=g).bfloat16().to(DEV)
    seen = torch.zeros(B, V, dtype=torch.uint8, device=DEV)
    wte = torch.randn(V, h, generator=g).bfloat16().to(DEV)
    wpe = torch.randn(npos, h, generator=g).bfloat16().to(DEV) if use_wpe else None
    emb = lambda tok, pos: (wte[tok].float() + wpe[min(pos, npos - 1)].float()).bfloat16() if use_wpe else wte[tok]
    for cur in (0, 5, 10, 11, 40):                                   # the position after the advance, clamped to npos - 1
        got, _, x, st = _select_once(FUSED, False, lg, seen, 1.0, wte=wte, wpe=wpe, cur_len=cur, n_positions=npos)
        assert st["cur_len"] == cur + 1
        for b in range(B):
            assert torch.equal(x[b], emb(got[b], cur + 1)), (cur, b)
    # session rows: each at its own length; rows that do not select keep x, out_ids, seen and their state
    cur = 3
    out = torch.full((B, 4), -7, dtype=torch.int32, device=DEV)
    nxt = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    x = torch.full((B, h), 7.0, dtype=torch.bfloat16, device=DEV)
    seen2 = torch.full((B, V), 3, dtype=torch.uint8, device=DEV)
    active = [1] * B
    active[2] = active[9] = 0
    mask = 0xFFFF & ~(1 << 5) & ~(1 << 12)
    st = _row_state(B, row_len=[cur + b for b in range(B)], active=active, max_new=[4] * B, mask=mask)
    before = {k: list(v) if isinstance(v, list) else v for k, v in st.items()}
    p = GenerationParams(max_new_tokens=4, eos_token_id=None, pad_token_id=0)
    E.op_select(FUSED, lg, p, seen2, out, nxt, st, per_row=True, wte=wte, wpe=wpe, x=x, n_positions=npos)
    want = greedy_reference(lg.cpu(), seen.cpu(), 1.0)
    for b in range(B):
        if b in (2, 9, 5, 12):
            assert (x[b] == 7.0).all() and (out[b] == -7).all() and nxt[b] == -7 and (seen2[b] == 3).all()
            assert st["row_len"][b] == before["row_len"][b] and st["row_step"][b] == 0 and st["row_active"][b] == before["row_active"][b]
        else:
            assert nxt[b] == want[b] and st["row_len"][b] == cur + b + 1 and st["row_step"][b] == 1
            assert torch.equal(x[b], emb(want[b], cur + b + 1)), b
    assert st["event"] == 0


# ---- bookkeeping -------------------------------------------------------------------------------------------------------------
class HFLoop:
    """`GenerationMixin._sample`'s loop body after the token choice, for a rectangle batch: the pad rule, the append,
    `unfinished &= ~stopping_criteria(input_ids)` with EosTokenCriteria, MaxLengthCriteria and the reference's
    StoppingCriteriaSub (the stop ids at the end of ROW 0 end every row; per-row mode: each row's own end), and
    `this_peer_finished = unfinished.max() == 0`."""

    def __init__(self, B, V, stride, p, st, seen, out):
        self.p, self.B, self.V = p, B, V
        self.step, self.cur_len, self.done, self.unfinished = st["step"], st["cur_len"], st["done"], torch.tensor(st["unfinished"])
        self.seen, self.out, self.next = seen.clone().cpu(), out.clone().cpu(), torch.full((B,), -7, dtype=torch.int32)
        self.ids = torch.zeros(B, 0, dtype=torch.long)

    def advance(self, toks, advance_len):
        if self.done:
            return
        p = self.p
        nt = torch.tensor(toks)
        if p.eos_token_id is not None:
            nt = nt * self.unfinished + p.pad_token_id * (1 - self.unfinished)
        self.ids = torch.cat([self.ids, nt[:, None]], 1)
        self.out[:, self.step] = nt.int()
        self.next = nt.int()
        self.seen[torch.arange(self.B), nt] = 1
        stop = torch.zeros(self.B, dtype=torch.bool)
        if p.eos_token_id is not None:
            stop = stop | EosTokenCriteria(p.eos_token_id)(self.ids, None)
        n = len(p.stop_ids)
        if n and self.ids.shape[1] >= n:
            tail = (self.ids[:, -n:] == torch.tensor(list(p.stop_ids))).all(1)
            stop = stop | (tail[0].expand(self.B) if p.stop_row0_only else tail)
        self.unfinished = self.unfinished & ~stop
        self.step += 1
        self.cur_len += advance_len
        # MaxLengthCriteria ends the loop through `done`; the kernels leave `unfinished` as it is then
        self.done = int(self.unfinished.max() == 0 or bool(MaxLengthCriteria(p.max_new_tokens)(self.ids, None).all()))

    def state(self):
        return dict(step=self.step, cur_len=self.cur_len, done=self.done, unfinished=self.unfinished.tolist())


class RowLoop:
    """The session rule: a row with its mask bit and row_active set appends at its own step; EOS, the stop ids at the end
    of its own tokens, or its own cap finish it and raise `event`.  No pad rule (a finished row no longer selects)."""

    def __init__(self, B, V, stride, p, st, seen, out):
        self.p, self.B, self.st = p, B, {k: list(v) if isinstance(v, list) else v for k, v in st.items()}
        self.seen, self.out, self.next = seen.clone().cpu(), out.clone().cpu(), torch.full((B,), -7, dtype=torch.int32)

    def advance(self, toks, advance_len):
        p, st = self.p, self.st
        for b in range(self.B):
            if not ((st["row_mask"] >> b) & 1 and st["row_active"][b]):
                continue
            s = st["row_step"][b]
            self.out[b, s] = self.next[b] = toks[b]
            self.seen[b, toks[b]] = 1
            n = len(p.stop_ids)
            fin = p.eos_token_id is not None and toks[b] == p.eos_token_id
            fin = fin or (n > 0 and s + 1 >= n and self.out[b, s + 1 - n:s + 1].tolist() == list(p.stop_ids))
            st["row_step"][b] += 1
            st["row_len"][b] += advance_len
            if fin or s + 1 >= st["row_max_new"][b]:
                st["row_active"][b], st["event"] = 0, 1

    def state(self):
        return self.st


A, Bk, Ck = 7, 8, 9      # script tokens; EOS = 0, pad = 499
SCRIPTS = {
    # name: (params, tokens per step [steps][B], extra state)
    "eos_row3_then_pad": (dict(eos_token_id=0, max_new_tokens=6), [[5, 6, 7, 8, 9], [5, 6, 7, 8, 9], [5, 6, 7, 0, 9], [1, 2, 3, 4, 5],
                                                                  [1, 2, 3, 4, 5], [1, 2, 3, 4, 5], [1, 2, 3, 4, 5]], {}),
    "all_rows_eos": (dict(eos_token_id=0, max_new_tokens=8), [[5, 0, 7], [0, 6, 7], [5, 6, 0], [1, 2, 3]], {}),
    "stop1_at_first_step": (dict(eos_token_id=0, max_new_tokens=6, stop_ids=[A]), [[A, 1, 2], [3, 4, 5]], {}),
    "stop3_at_step_n_minus_1": (dict(eos_token_id=0, max_new_tokens=8, stop_ids=[A, Bk, Ck]), [[A, 1, 2], [Bk, 1, 2], [Ck, 1, 2], [3, 3, 3]], {}),
    "stop8_at_step_n_minus_1": (dict(eos_token_id=0, max_new_tokens=12, stop_ids=[11, 12, 13, 14, 15, 16, 17, 18]),
                                [[t, 1] for t in range(11, 19)] + [[3, 3]], {}),
    "stop3_late_after_near_miss": (dict(eos_token_id=0, max_new_tokens=12, stop_ids=[A, Bk, Ck]),
                                   [[A, 1], [Bk, 1], [A, 1], [Bk, 1], [Ck, 1], [3, 3]], {}),
    "stop_on_row2_only": (dict(eos_token_id=0, max_new_tokens=8, stop_ids=[A, Bk]), [[1, 1, A], [1, 1, Bk], [2, 2, 2], [A, 2, 2], [Bk, 2, 2], [3, 3, 3]], {}),
    "stop_overlaps_itself": (dict(eos_token_id=0, max_new_tokens=8, stop_ids=[A, A, Bk]), [[A, 1], [A, 1], [A, 1], [Bk, 1], [3, 3]], {}),
    "max_new_reached": (dict(eos_token_id=0, max_new_tokens=3), [[1, 2]] * 5, {}),
    "no_eos_id": (dict(eos_token_id=None, max_new_tokens=4), [[0, 1], [0, 0], [2, 0], [1, 1], [1, 1]], {}),
    "done_on_entry": (dict(eos_token_id=0, max_new_tokens=4), [[1, 2]] * 2, dict(done=1)),
    "row_caps_differ": (dict(eos_token_id=0, max_new_tokens=8), [[1, 2, 3, 4]] * 6, dict(max_new=[1, 3, 5, 2])),
    "masked_and_inactive_rows": (dict(eos_token_id=0, max_new_tokens=8, stop_ids=[A]), [[1, 2, 3, 4], [1, 0, 3, A], [A, 2, 3, 4], [1, 2, 3, 4]],
                                 dict(mask=0b1011, active=[1, 1, 1, 0])),
}


def _one_hot_logits(toks, V, sample):
    lg = torch.zeros(len(toks), V)
    lg[torch.arange(len(toks)), torch.tensor(toks)] = 60.0 if sample else 5.0
    return lg.bfloat16().to(DEV)


def run_script(impl, per_row, row0_only, name):
    kw, script, extra = SCRIPTS[name]
    B, V, h, npos, stride = len(script[0]), 500, 64, 12, 16
    p = GenerationParams(pad_token_id=499, stop_row0_only=row0_only, do_sample=impl == SAMPLE, top_p=0.5, seed=3, **kw)
    g = torch.Generator().manual_seed(1)
    wte, wpe = torch.randn(V, h, generator=g).bfloat16().to(DEV), torch.randn(npos, h, generator=g).bfloat16().to(DEV)
    out = torch.full((B, stride), -7, dtype=torch.int32, device=DEV)
    nxt = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    seen = torch.zeros(B, V, dtype=torch.uint8, device=DEV)
    x = torch.full((B, h), 7.0, dtype=torch.bfloat16, device=DEV)
    if per_row:
        st = _row_state(B, row_len=[8 + b for b in range(B)], max_new=extra.get("max_new", [kw["max_new_tokens"]] * B),
                        active=extra.get("active"), mask=extra.get("mask", 0xFFFF))
        model = RowLoop(B, V, stride, p, st, seen, out)
    else:
        st = _plain_state(B, cur_len=8, done=extra.get("done", 0))
        model = HFLoop(B, V, stride, p, st, seen, out)
    trace = []
    for s, toks in enumerate(script):
        fused_kw = dict(wte=wte, wpe=wpe, x=x, n_positions=npos) if impl == FUSED else {}
        E.op_select(impl, _one_hot_logits(toks, V, impl == SAMPLE), p, seen, out, nxt, st, per_row=per_row, advance_len=1, **fused_kw)
        was_done = (not per_row) and model.done
        model.advance(toks, 1)
        want = model.state()
        for k, v in want.items():
            assert st[k] == v, (name, s, k, st[k], v)
        assert torch.equal(out.cpu(), model.out) and torch.equal(seen.cpu(), model.seen), (name, s)
        sel = [b for b in range(B) if (per_row and torch.ne(model.next, -7)[b]) or (not per_row and model.step > 0)]
        assert torch.equal(nxt.cpu()[sel], model.next[sel]), (name, s)
        if impl == FUSED and not was_done and not per_row:
            for b in range(B):
                pos = min(want["cur_len"], npos - 1)
                assert torch.equal(x[b], (wte[int(model.next[b])].float() + wpe[pos].float()).bfloat16()), (name, s, b)
        trace.append((out.cpu().clone(), nxt.cpu().clone(), {k: (list(v) if isinstance(v, list) else v) for k, v in st.items()}))
    return trace


@pytest.mark.parametrize("name", list(SCRIPTS))
def test_bookkeeping_follows_the_hf_loop(name):
    """Every impl, rectangle (row-0 stop and per-row stop) and session kernels, against the Python loop after every step."""
    extra = SCRIPTS[name][2]
    traces = {}
    for impl in (GREEDY, FUSED, SAMPLE):
        if not ({"max_new", "mask", "active"} & set(extra)):
            for row0 in (True, False):
                traces[(impl, "plain", row0)] = run_script(impl, False, row0, name)
        if "done" not in extra:
            traces[(impl, "rows")] = run_script(impl, True, False, name)
    for key, tr in traces.items():                      # greedy, fused and sample agree bitwise on every script
        ref = traces[(GREEDY,) + key[1:]]
        for (o1, n1, s1), (o2, n2, s2) in zip(tr, ref):
            assert torch.equal(o1, o2) and torch.equal(n1, n2) and s1 == s2, (name, key)


@pytest.mark.parametrize("name", ["eos_row3_then_pad", "stop3_at_step_n_minus_1", "stop_overlaps_itself", "max_new_reached", "no_eos_id"])
def test_session_row_equals_one_row_generate(name):
    """With one row the session kernels do what the rectangle kernels do, up to and including the row's last token."""
    kw, script, _ = SCRIPTS[name]
    one = {**SCRIPTS}
    SCRIPTS["_one"] = (kw, [[t[0] if name != "eos_row3_then_pad" else t[3]] for t in script], {})
    try:
        for impl in (GREEDY, FUSED, SAMPLE):
            plain = run_script(impl, False, True, "_one")
            rows = run_script(impl, True, False, "_one")
            done_at = next((i for i, t in enumerate(plain) if t[2]["done"]), len(plain) - 1)
            for i in range(done_at + 1):
                assert torch.equal(plain[i][0], rows[i][0]) and torch.equal(plain[i][1], rows[i][1]), (name, impl, i)
                assert plain[i][2]["step"] == rows[i][2]["row_step"][0] and plain[i][2]["cur_len"] == rows[i][2]["row_len"][0]
                assert plain[i][2]["done"] == 1 - rows[i][2]["row_active"][0] == rows[i][2]["event"]
    finally:
        del SCRIPTS["_one"]
        assert one.keys() == SCRIPTS.keys()


# ---- beam candidates ---------------------------------------------------------------------------------------------------------
def _beam_params(nb, do_sample=0, T=1.0, top_p=1.0, rp=1.0, seed=0, eos=0):
    return _lib.BeamParams(num_beams=nb, max_new_tokens=64, do_sample=do_sample, early_stopping=1, temperature=T, top_p=top_p,
                           repetition_penalty=rp, length_penalty=1.0, eos_token_id=eos, pad_token_id=0, seed=seed)


def _beam_inputs(R, V, seed, cur_len):
    g = torch.Generator().manual_seed(seed)
    rows = torch.stack([_with_mass(torch.randn(V, generator=g, dtype=torch.float64) * 2, torch.randperm(V, generator=g)[:6].tolist(),
                                   [0.3, 0.2, 0.12, 0.08, 0.05, 0.03]) for _ in range(R)]).bfloat16()
    for r in range(R):                                  # exact ties across lanes and at both ends of the row
        top = rows[r].float().max()
        ids = [[0, V - 1], [33, 64 + 33], [V - 1, V - 2]][r % 3]
        rows[r, ids] = (top + 1.0).bfloat16()
    seq = torch.randint(0, V, (R, 64), generator=g, dtype=torch.int32)
    seq[:, 0] = torch.tensor([int(rows[r].float().argmax()) for r in range(R)])     # a favourite is penalised
    seq[:, 1], seq[:, 2] = V + 5, -3                                              # ids outside the vocabulary are ignored
    scores = (-torch.rand(R, generator=g) * 5).tolist()
    return rows, seq, scores


def _beam_fp64(rows, seq, scores, cur_len, rp):
    V = rows.shape[1]
    lp = torch.log_softmax(rows.float().double(), 1)
    for r in range(rows.shape[0]):
        if rp != 1.0 and cur_len > 0:
            ids = seq[r, :cur_len].long()
            ids = torch.unique(ids[(ids >= 0) & (ids < V)])
            lp[r, ids] = torch.where(lp[r, ids] < 0, lp[r, ids] * rp, lp[r, ids] / rp)
    return lp + torch.tensor(scores, dtype=torch.float64)[:, None]


@pytest.mark.parametrize("cur_len,rp", [(0, 1.3), (7, 1.3), (7, 1.0)], ids=str)
@pytest.mark.parametrize("R,nb", [(2, 2), (8, 4), (16, 8), (16, 2)], ids=str)
@pytest.mark.parametrize("V", [49156, 49157, 500])
def test_beam_candidates_greedy_against_fp64(V, R, nb, cur_len, rp):
    TOL = 2e-5
    rows, seq, scores = _beam_inputs(R, V, seed=V + R + nb, cur_len=cur_len)
    key, val, tok = E.op_beam_candidates(rows.to(DEV), _beam_params(nb, rp=rp), R // nb, cur_len, scores, seq.to(DEV))
    ref = _beam_fp64(rows, seq, scores, cur_len, rp)
    key, val, tok = key.cpu().double(), val.cpu().double(), tok.cpu().long()
    K, worst = 2 * nb, 0.0
    assert torch.equal(key, val)
    for r in range(R):
        order = sorted(range(V), key=lambda i: (-float(ref[r, i]), i))[:K + 1]
        assert len(set(tok[r].tolist())) == K
        for k in range(K):
            t = int(tok[r, k])
            worst = max(worst, abs(float(val[r, k] - ref[r, t])))
            assert abs(val[r, k] - ref[r, t]) <= TOL and abs(ref[r, t] - ref[r, order[k]]) <= TOL, (r, k)
            lone = (k == 0 or ref[r, order[k - 1]] - ref[r, order[k]] > TOL) and ref[r, order[k]] - ref[r, order[k + 1]] > TOL
            tie_prev = k > 0 and ref[r, order[k - 1]] == ref[r, order[k]]
            if lone or tie_prev or ref[r, order[k]] == ref[r, order[k + 1]]:
                assert t == order[k], (r, k, t, order[k])                     # exact ties: ascending id
    _calib(f"beam log-probs V={V} R={R} nb={nb}", worst, TOL)


def _host_candidates(bp, row_f32, seq, cur_len, score, row):
    K = 2 * bp.num_beams
    lib = _lib.load()
    lg = row_f32.contiguous().numpy()
    sq = seq.contiguous().numpy()
    k, v, t = (C.c_float * K)(), (C.c_float * K)(), (C.c_int32 * K)()
    assert lib.sv_beam_row_candidates_host(C.byref(bp), lg.ctypes.data_as(C.POINTER(C.c_float)), len(lg),
                                           sq.ctypes.data_as(C.POINTER(C.c_int32)), cur_len, score, cur_len, row, k, v, t) == 0
    return list(k), list(v), list(t)


def _permuted_rows(R, V, seed, masses):
    """R rows with one sorted distribution (so one nucleus cut fits all), the ids permuted per row."""
    g = torch.Generator().manual_seed(seed)
    base = _with_mass(torch.randn(V, generator=g, dtype=torch.float64) * 1.5, list(range(len(masses))), masses).bfloat16()
    return torch.stack([base[torch.randperm(V, generator=g)] for _ in range(R)])


@pytest.mark.parametrize("R,nb", [(2, 2), (16, 4), (16, 8)], ids=str)
@pytest.mark.parametrize("V", [49156, 49157, 500])
def test_beam_sample_equals_host_mirror_and_hf_nucleus(V, R, nb):
    masses = [0.22, 0.17, 0.13, 0.1, 0.08, 0.06, 0.05, 0.04, 0.03, 0.02]
    rows = _permuted_rows(R, V, seed=V + R, masses=masses)
    P = torch.softmax(rows[0].float().double() / 0.9, 0).sort(descending=True).values
    cum = torch.cumsum(P, 0)
    top_p = float((cum[7] + cum[8]) / 2)                                   # the cut sits between the 9th and 10th id
    assert min(float(top_p - cum[7]), float(cum[8] - top_p)) > 1e-3
    g = torch.Generator().manual_seed(7)
    seq = torch.stack([rows[r].float().argsort()[:64].int()[torch.randperm(64, generator=g)] for r in range(R)])  # tail ids only
    scores = (-torch.rand(R, generator=g) * 3).tolist()
    cur_len = 5
    bp = _beam_params(nb, do_sample=1, T=0.9, top_p=top_p, rp=1.2, seed=99)
    key, val, tok = (t.cpu() for t in E.op_beam_candidates(rows.to(DEV), bp, R // nb, cur_len, scores, seq.to(DEV)))
    K = 2 * nb
    for r in range(R):
        hk, hv, ht = _host_candidates(bp, rows[r].float(), seq[r], cur_len, scores[r], r)
        for k in range(K):
            assert abs(float(key[r, k]) - hk[k]) <= 1e-5 or (math.isinf(hk[k]) and key[r, k] == hk[k]), (r, k)
            close = any(abs(hk[k] - hk[j]) <= 1e-5 for j in (k - 1, k + 1) if 0 <= j < K and math.isfinite(hk[j]))
            if math.isfinite(hk[k]):
                assert int(tok[r, k]) == ht[k] or close, (r, k)
                if int(tok[r, k]) == ht[k]:
                    assert abs(float(val[r, k]) - hv[k]) <= 1e-5
            else:
                assert val[r, k] == -math.inf
        # every finite candidate lies inside transformers' nucleus (9 ids), and the noise is the Philox Gumbel draw
        sc = hf_scores(rows[r].float().log_softmax(0), torch.unique(seq[r, :cur_len].long()), 0.9, 1.2)
        keep = torch.isfinite(TopPLogitsWarper(top_p, min_tokens_to_keep=2)(None, sc[None])[0])
        assert int(keep.sum()) == 9
        fin = torch.isfinite(key[r])
        assert int(fin.sum()) == min(K, 9) and keep[tok[r][fin].long()].all()
        noise = (key[r][fin] - val[r][fin]).double().numpy()
        want = beam_gumbel(99, cur_len, r, tok[r][fin].numpy().astype(np.int64))
        assert np.abs(noise - want).max() <= 2e-5 * (1 + np.abs(want).max()), r


def test_beam_sample_nucleus_edges_and_noise_streams():
    V, nb = 49157, 8
    R, K = 16, 16
    # row A: the top token alone exceeds top_p -> min_tokens_to_keep = 2 keeps the runner-up; row B: a 6-way tie at the cut
    g = torch.Generator().manual_seed(5)
    a = _with_mass(torch.randn(V, generator=g, dtype=torch.float64), [V - 1, 77], [0.9, 0.05]).bfloat16()
    b = _with_mass(torch.randn(V, generator=g, dtype=torch.float64), [5, 0, V - 1, 1024, 2048, 4000, 9000], [0.4] + [0.09] * 6).bfloat16()
    rows = torch.stack([a, b] * 8)
    seq = torch.zeros(R, 8, dtype=torch.int32)
    bp = _beam_params(nb, do_sample=1, top_p=0.6, seed=4)
    key, val, tok = (t.cpu() for t in E.op_beam_candidates(rows.to(DEV), bp, 2, 0, [0.0] * R, seq.to(DEV)))
    for r in range(0, R, 2):
        assert set(tok[r][torch.isfinite(key[r])].tolist()) == {V - 1, 77}
        assert (val[r][~torch.isfinite(key[r])] == -math.inf).all() and int(torch.isfinite(val[r]).sum()) == 2
        assert set(tok[r + 1][torch.isfinite(key[r + 1])].tolist()) == {5, 0, V - 1, 1024, 2048, 4000, 9000}
    hf = torch.isfinite(TopPLogitsWarper(0.6, min_tokens_to_keep=2)(None, a.float().log_softmax(0)[None])[0])
    assert set(hf.nonzero().flatten().tolist()) == {V - 1, 77}
    # the same logits at another row, seed or step draw other noise; rows >= 8 differ from rows < 8
    noise = lambda k, v, t, r, token: float((k[r] - v[r])[t[r] == token][0])
    base = noise(key, val, tok, 0, 77)
    assert all(abs(noise(key, val, tok, r, 77) - base) > 1e-6 for r in range(2, R, 2))
    assert abs(noise(key, val, tok, 8, 77) - noise(key, val, tok, 0, 77)) > 1e-6
    for kw, cur in ((dict(seed=5), 0), (dict(seed=4), 1)):
        k2, v2, t2 = (t.cpu() for t in E.op_beam_candidates(rows.to(DEV), _beam_params(nb, do_sample=1, top_p=0.6, **kw), 2, cur,
                                                           [0.0] * R, seq.to(DEV)))
        assert abs(noise(k2, v2, t2, 0, 77) - base) > 1e-6
    for r in (0, 8, 14):
        got = noise(key, val, tok, r, 77)
        assert abs(got - float(beam_gumbel(4, 0, r, np.asarray([77]))[0])) <= 2e-5 * (1 + abs(got))


def test_beam_candidates_fewer_finite_logits_than_candidates():
    V, nb, R = 500, 4, 4
    rows = torch.full((R, V), -math.inf)
    rows[:, 3], rows[:, 499] = 1.0, 1.0
    rows[:, 250] = 0.5
    key, val, tok = (t.cpu() for t in E.op_beam_candidates(rows.bfloat16().to(DEV), _beam_params(nb), 1, 0, [0.0, -1.0, -2.0, -3.0],
                                                           torch.zeros(R, 8, dtype=torch.int32, device=DEV)))
    assert tok[:, :3].tolist() == [[3, 499, 250]] * R
    assert torch.isinf(val[:, 3:]).all() and (val[:, 3:] < 0).all() and torch.isfinite(val[:, :3]).all()

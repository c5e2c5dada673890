"""The selection kernels of a speculative verify step one launch at a time (sv_op_spec_select), at the StarVector-1B
widths (hidden 2048, vocabulary 49156 / 49157).

References:
  * column b's token: greedy_reference / the fp64 CDF of test_select_ops_gpu on column b's logits, penalised by the row's
    seen set plus drafts 1..b, with the Philox counter (0, step + b) for sampling;
  * the accept walk: test_select_ops_gpu.HFLoop (the HF `_sample` loop body) per emitted token, stopping at the finish or
    at the first selected token that differs from the next draft;
  * the next drafts: sv_spec_draft_host (test_speculative_logic.draft, pinned there to transformers'
    PromptLookupCandidateGenerator), the column map svspec::set_map, the embeddings bf16(wte[tok] + wpe[pos]).
Every output of the op is compared exactly: the history, seen, next_ids, the counters, the column map, the drafts and all
ncols embedding rows.  The draft search runs across the CTA with a 1024 stride, so the planted histories put the deciding
match in the second and third stride, in neighbouring lanes, at the history's start and at its end.  `CALIB` lines (-s)
give each family's count and worst case.
"""
import numpy as np
import pytest
import torch

from starvector_b200 import _lib
from starvector_b200 import engine as E
from starvector_b200.engine import GenerationParams
from test_decode_ops_gpu import _nsm, _plant_ties, _weights
from test_select_ops_gpu import DELTA_CDF, HFLoop, RowRef, greedy_reference, hf_scores, make_rows, sampler_u
from test_speculative_logic import draft

pytestmark = pytest.mark.gpu
DEV = "cuda"
V0, H, NPOS = 49156, 2048, 4200
GREEDY, SAMPLE, ACCEPT = _lib.SV_SPEC_GREEDY, _lib.SV_SPEC_SAMPLE, _lib.SV_SPEC_ACCEPT


def _calib(name, n, worst=None, tol=None):
    extra = f", worst = {worst:.3e} (tolerance {tol:.1e}, ratio {worst / tol:.3f})" if tol else ", every output exact"
    print(f"CALIB spec {name}: {n} calls{extra}")


@pytest.fixture(scope="module")
def emb():
    g = torch.Generator(device=DEV).manual_seed(11)
    wte = torch.randn(V0 + 1, H, generator=g, device=DEV).bfloat16()
    wpe = (0.1 * torch.randn(NPOS, H, generator=g, device=DEV)).bfloat16()
    return wte, wpe


def set_map(ncols, n_live, cur_len):
    """svspec::set_map: live columns at cur_len + c, inert ones at the last live position."""
    last = max(cur_len + n_live - 1, 0)
    return [cur_len + c if c < n_live else last for c in range(ncols)]


def make_spec(k, g, tok, n_live, cur_len, sel=None, counters=(3, 20, 9)):
    s = _lib.SpecState(n_live=n_live, ncols=k + 1, k=k, max_ngram=g, steps=counters[0], drafted=counters[1],
                       accepted=counters[2])
    for c in range(16):
        s.row[c], s.pos[c], s.tok[c], s.sel[c] = 0, 0, -3, -5
    for c, p in enumerate(set_map(k + 1, n_live, cur_len)):
        s.pos[c] = min(p, NPOS - 1)
    for c, t in enumerate(tok):
        s.tok[c] = t
    for c, t in enumerate(sel or []):
        s.sel[c] = t
    return s


def snap(s):
    return {f: (list(getattr(s, f)) if f in ("row", "pos", "tok", "sel") else int(getattr(s, f))) for f, _ in s._fields_}


def params(max_new, eos=None, stop=(), rp=1.0, T=1.0, top_p=1.0, seed=0):
    return GenerationParams(max_new_tokens=max_new, eos_token_id=eos, pad_token_id=V0 - 4, stop_ids=tuple(stop),
                            repetition_penalty=rp, temperature=T, top_p=top_p, seed=seed)


def run_op(impl, p, hist, stride, gen, spec, seen, emb, V=V0, logits=None, amax=None):
    """One sv_op_spec_select call on fresh device copies; returns every output."""
    wte, wpe = emb
    out = torch.full((stride,), -7, dtype=torch.int32, device=DEV)
    out[:len(hist)] = torch.tensor(hist, dtype=torch.int32)
    sd = seen.to(DEV).clone()
    nxt = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    x = torch.full((spec.ncols, H), 7.0, dtype=torch.bfloat16, device=DEV)
    st = dict(gen)
    E.op_spec_select(impl, p, sd, out, nxt, st, spec, wte[:V], wpe, x, NPOS, logits=logits, amax=amax)
    return dict(out=out.cpu(), seen=sd.cpu(), next=int(nxt[0]), x=x, gen=st, spec=snap(spec))


def expect(p, hist, stride, gen, spec_in, seen, sel, emb, V=V0):
    """The Python restatement of the accept walk and spec_tail for the selected tokens `sel`."""
    wte, wpe = emb
    sp = snap(spec_in)
    out = torch.full((stride,), -7, dtype=torch.int32)
    out[:len(hist)] = torch.tensor(hist, dtype=torch.int32)
    res = dict(out=out, seen=seen.cpu().clone(), next=-7, x=None, gen=dict(gen), spec=sp)
    if gen["done"]:                                       # nothing runs: every output keeps its value (x too)
        return res
    ncols, n_live, tok = sp["ncols"], sp["n_live"], sp["tok"]
    loop = HFLoop(1, V, stride, p, dict(gen, unfinished=[gen["unfinished"]]), seen.cpu()[None], out[None])
    loop.ids = out[None, :gen["step"]].long()
    m = 0
    for c in range(n_live):
        loop.advance([sel[c]], 1)
        m += 1
        if loop.done or c + 1 >= n_live or sel[c] != tok[c + 1]:
            break
    if n_live > 0:
        sp["steps"] += 1
        sp["drafted"] += n_live - 1
        sp["accepted"] += m - 1
    n, done = loop.step, bool(loop.done)
    h2 = loop.out[0, :n].tolist()
    eos = -1 if p.eos_token_id is None else p.eos_token_id
    d = [] if done else draft(h2, sp["k"], sp["max_ngram"], eos, p.max_new_tokens - n - 1)
    nl = 0 if done else 1 + len(d)
    new_tok = [h2[-1]] + d + [h2[-1]] * (ncols - 1 - len(d))
    pos = set_map(ncols, nl, loop.cur_len)
    sp["n_live"] = nl
    sp["tok"][:ncols] = new_tok
    sp["pos"][:ncols] = pos
    sp["row"][:ncols] = [0] * ncols
    t = torch.tensor(new_tok, device=DEV)
    pp = torch.tensor([min(q, NPOS - 1) for q in pos], device=DEV)
    res.update(out=loop.out[0], seen=loop.seen[0], gen=dict(step=n, cur_len=loop.cur_len, done=int(done),
                                                             unfinished=int(loop.unfinished[0])),
               x=(wte[t].float() + wpe[pp].float()).bfloat16(), next=int(loop.next[0]) if m else -7, drafts=d)
    return res


def compare(got, want, name):
    assert torch.equal(got["out"], want["out"]), (name, "out_ids")
    assert torch.equal(got["seen"], want["seen"]), (name, "seen", (got["seen"] != want["seen"]).nonzero().flatten()[:8].tolist())
    assert got["next"] == want["next"], (name, "next_ids", got["next"], want["next"])
    assert got["gen"] == want["gen"], (name, got["gen"], want["gen"])
    assert got["spec"] == want["spec"], (name, {k: (got["spec"][k], want["spec"][k]) for k in want["spec"]
                                                if got["spec"][k] != want["spec"][k]})
    if want["x"] is None:
        assert (got["x"] == 7.0).all(), (name, "x written")
    else:
        assert torch.equal(got["x"], want["x"]), (name, "x")


def one_hot(sel, ncols, V, val, g):
    lg = torch.zeros(ncols, V)
    ids = list(sel) + torch.randint(0, V, (ncols - len(sel),), generator=g).tolist()
    lg[torch.arange(ncols), torch.tensor(ids)] = val
    return lg.bfloat16().to(DEV)


# ---- e. the accept walk and the next step ----------------------------------------------------------------------------------
WALKS = ["reject_mid", "accept_all", "eos_mid", "stop_completed", "max_new_cap", "no_eos", "done_on_entry", "pos_clamp"]


def walk_case(k, kind, seed):
    """A periodic history (so the drafts are long), the entry state the previous step left, and the selected tokens."""
    g = torch.Generator().manual_seed(seed)
    period = (torch.randperm(40, generator=g)[:5] + 10).tolist()
    n0 = 40 + int(torch.randint(0, 5, (1,), generator=g))
    hist = [period[i % 5] for i in range(n0)]
    hist[7] = 77                                           # one irregularity, so that not every match is the same
    eos = None if kind == "no_eos" else 3
    max_new, stride, stop = 200, 256, ()
    if kind == "max_new_cap":                                  # the budget lets every draft in; accepting them reaches the cap
        max_new = n0 + 1 + min(k, 2)
    d = draft(hist, k, 2, -1 if eos is None else eos, max_new - n0 - 1)
    assert d, "the periodic history gives drafts"
    j = {"accept_all": len(d), "max_new_cap": len(d)}.get(kind, len(d) // 2)
    sel = [d[c] for c in range(j)] + [90 + c for c in range(j, k + 1)]     # 90.. never equal a draft
    if kind == "eos_mid":
        sel[j] = eos
    if kind == "stop_completed" and len(d) >= 2:            # an accepted draft completes the stop sequence
        stop = (d[0], d[1])
        sel[:2] = d[:2]
    cur_len = NPOS - 3 if kind == "pos_clamp" else 300 + n0
    gen = dict(step=n0, cur_len=cur_len, done=int(kind == "done_on_entry"), unfinished=1)
    seen = (torch.rand(V0, generator=g) < 0.03).to(torch.uint8)
    seen[torch.tensor(hist)] = 0                           # so that a rejected draft entering seen would show
    return hist, stride, gen, seen, params(max_new, eos, stop), [hist[-1]] + d, 1 + len(d), sel


@pytest.mark.parametrize("impl", [ACCEPT, GREEDY, SAMPLE], ids=["accept", "greedy", "sample"])
@pytest.mark.parametrize("k", [1, 7, 15])
def test_accept_walk_and_next_step(emb, k, impl):
    """EOS at a middle column, a stop completed by an accepted draft, the max_new cap, no EOS id, done on entry, and
    positions past the position table; the column tokens come in as `sel` (ACCEPT) or as one-hot logits (GREEDY with a
    repetition penalty, SAMPLE)."""
    g = torch.Generator().manual_seed(k)
    for i, kind in enumerate(WALKS):
        hist, stride, gen, seen, p, tok, n_live, sel = walk_case(k, kind, seed=k * 100 + i)
        if impl == GREEDY:
            p.repetition_penalty = 1.3
        spec = make_spec(k, 2, tok + [tok[0]] * (k + 1 - len(tok)), n_live, gen["cur_len"],
                         sel=sel if impl == ACCEPT else None)
        want = expect(p, hist, stride, gen, spec, seen, sel, emb)
        lg = None if impl == ACCEPT else one_hot(sel, k + 1, V0, 5.0 if impl == GREEDY else 60.0, g)
        got = run_op(impl, p, hist, stride, gen, spec, seen, emb, logits=lg)
        if impl == SAMPLE and not gen["done"]:       # the sampler wrote the live columns' tokens, nothing else
            want["spec"]["sel"] = sel[:n_live] + [-5] * (16 - n_live)
        compare(got, want, f"{kind} k={k}")
        if kind in ("eos_mid", "max_new_cap") or (kind == "stop_completed" and p.stop_ids):   # the finish inside the walk
            assert got["spec"]["n_live"] == 0 and got["gen"]["done"] == 1, kind
        if kind == "stop_completed" and p.stop_ids:
            assert got["gen"]["step"] == gen["step"] + 2
    _calib(f"accept walk impl={impl} k={k}", len(WALKS))


# ---- f. the draft search ---------------------------------------------------------------------------------------------------
def _unique(n):
    return [100 + i for i in range(n)]


def _plant(h, e, seq):
    h[e - len(seq):e] = list(seq)


def draft_cases():
    """(name, history, k, max_ngram, eos, max_new - n - 1 + (n + 1) = max_new)."""
    cs = []
    for n, g in ((1, 2), (2, 2), (3, 2)):
        cs.append((f"n={n}", [7, 7, 8][:n] if n < 3 else [7, 8, 7], 15, g, -1, None))
    for n in (1023, 1024, 1025, 2049, 4095):             # a 3-gram match in the middle, 1-grams early
        h = _unique(n)
        _plant(h, n // 2 + 5, h[n - 3:])
        _plant(h, 9, h[n - 1:])
        cs.append((f"n={n} middle", h, 15, 3, -1, None))
    h = _unique(2049)                                      # the longest match only at e > 1024
    _plant(h, 1500, h[-3:]); _plant(h, 10, h[-1:]); _plant(h, 600, h[-2:])
    cs.append(("longest past 1024", h, 15, 3, -1, None))
    h = _unique(4095)                                      # ... only at e > 2048
    _plant(h, 3000, h[-3:]); _plant(h, 1200, h[-2:]); _plant(h, 5, h[-1:])
    cs.append(("longest past 2048", h, 15, 3, -1, None))
    h = _unique(3000)                                      # equal lengths at e and e + 1024: the earlier wins
    _plant(h, 700, h[-3:]); _plant(h, 1724, h[-3:])
    cs.append(("lanes e and e+1024", h, 7, 3, -1, None))
    h = _unique(1500)                                      # equal lengths at e and e + 1 (neighbouring lanes)
    h[-2] = h[-1] = 55
    _plant(h, 801, [55, 55, 55])
    cs.append(("lanes e and e+1", h, 7, 2, -1, None))
    h = _unique(1100)                                      # a 5-gram and a 2-gram match, both capped at 2: the earlier
    _plant(h, 900, h[-5:]); _plant(h, 400, h[-2:])
    cs.append(("capped by max_ngram", h, 15, 2, -1, None))
    h = _unique(1200)                                      # a match capped by e at e = 2, and a later one of equal length
    h[0:2] = h[-2:]
    _plant(h, 800, h[-2:])
    cs.append(("capped by e", h, 15, 3, -1, None))
    h = _unique(1300)                                      # the longest match continues with EOS: no draft, no fallback
    _plant(h, 1000, h[-3:]); h[1000] = 3; _plant(h, 200, h[-1:])
    cs.append(("continuation is EOS", h, 15, 3, 3, None))
    for n in (1024, 1025, 2049):                           # the last token repeated, no other match: e = n - 1
        h = _unique(n)
        h[-2] = h[-1]
        cs.append((f"ends repeated n={n}", h, 15, 3, -1, None))
    h = _unique(1500)                                      # a continuation running off the end of the history
    _plant(h, 1495, h[-3:])
    cs.append(("runs off the end", h, 15, 3, -1, None))
    for budget in (0, 1, 2):
        h = _unique(1100)
        _plant(h, 500, h[-3:])
        cs.append((f"budget {budget}", h, 15, 3, -1, len(h) + 1 + budget))
    h = [int(t) for t in np.random.default_rng(3).integers(10, 14, 4095)]   # a small alphabet: matches everywhere
    cs.append(("random n=4095", h, 15, 4, -1, None))
    return cs


def test_draft_search_planted_histories(emb):
    """ACCEPT with no live column (the first drafts of a generation): the drafts, the column map and the embeddings of
    every column, for every planted history."""
    cases = draft_cases()
    for name, hist, k, gng, eos, max_new in cases:
        n = len(hist)
        stride = n + 40
        max_new = max_new or stride
        p = params(max_new, None if eos < 0 else eos)
        gen = dict(step=n, cur_len=n + 30, done=0, unfinished=1)
        seen = torch.zeros(V0, dtype=torch.uint8)
        seen[torch.tensor(hist)] = 1
        spec = make_spec(k, gng, [hist[-1]] * (k + 1), 0, gen["cur_len"])
        want = expect(p, hist, stride, gen, spec, seen, [], emb)
        got = run_op(ACCEPT, p, hist, stride, gen, spec, seen, emb)
        compare(got, want, name)
        if name == "continuation is EOS":
            assert want["drafts"] == []
        elif name.startswith("budget"):
            assert len(want["drafts"]) == max_new - n - 1
        elif n >= 3:
            assert want["drafts"], name
    _calib("draft search", len(cases))


# ---- c. greedy selection -----------------------------------------------------------------------------------------------------
def test_greedy_partials_with_ties(emb):
    """rp = 1: the lm_head GEMV's argmax partials at B = ncols, exact ties planted within a tile, across two tiles and in the
    last partial tile (the lowest id wins); inert columns carry poisoned logits and partials."""
    N, K = V0, H
    g = torch.Generator(device=DEV).manual_seed(21)
    w, _ = _weights(N, K, g, bias=False)
    ln = (torch.ones(K, device=DEV).bfloat16(), torch.zeros(K, device=DEV).bfloat16())
    rpc = (N + _nsm() - 1) // _nsm()
    tpc = (rpc + 15) // 16
    R = (rpc + tpc - 1) // tpc
    calls = 0
    for ncols, n_live in ((16, 16), (16, 11), (9, 9), (8, 5), (2, 2), (1, 1)):
        x = torch.randn(ncols, K, generator=g, device=DEV).bfloat16()
        rows = list(dict.fromkeys(r for r in (0, ncols - 1, n_live // 2) if r < n_live))
        pairs = _plant_ties(w, x, N, R, rows)
        y, (val, idx) = E.op_gemv_ring(x, w, None, None, ln, epi=2)
        want = [int(torch.argmax(y[c].float())) for c in range(n_live)]    # the first maximum
        for i, r in enumerate(rows):
            assert want[r] == pairs[i % 3][0]
        y, val, idx = y.clone(), val.clone(), idx.clone()
        y[n_live:] = 0.0
        y[n_live:, 5] = 100.0
        val[:, n_live:] = 1e30
        idx[:, n_live:] = 5
        k = ncols - 1
        hist = [40, 41, 42, 43]
        tok = [hist[-1]] + want[:n_live - 1] + [hist[-1]] * (ncols - n_live)
        gen = dict(step=len(hist), cur_len=500, done=0, unfinished=1)
        seen = torch.zeros(V0, dtype=torch.uint8)
        p = params(100)
        spec = make_spec(k, 2, tok, n_live, gen["cur_len"])
        exp = expect(p, hist, 128, gen, spec, seen, want, emb)
        got = run_op(GREEDY, p, hist, 128, gen, spec, seen, emb, logits=y, amax=(val, idx))
        compare(got, exp, f"partials ncols={ncols} n_live={n_live}")
        assert got["out"][len(hist):len(hist) + n_live].tolist() == want            # every live column's token was emitted
        calls += 1
    _calib("greedy partials", calls)


def greedy_plan(rp, ncols, n_live, seed, tok0_seen, V=V0):
    """Column logits whose argmax each boundary of the penalty set decides, and drafts equal to the columns' expected
    tokens (so the walk emits every live column's selection); returns (logits, seen, tok, want)."""
    g = torch.Generator().manual_seed(seed)
    lg = (torch.randn(ncols, V, generator=g) * 1.5).clamp(-7, 3)
    seen = (torch.rand(V, generator=g) < 0.1).to(torch.uint8)
    tok0 = 1000 + seed % 100
    seen[tok0] = int(tok0_seen)
    tok, want = [tok0], []
    fresh = iter(range(20000, 21000))
    for b in range(ncols):
        kind = KINDS[(b + seed) % len(KINDS)]
        r = lg[b]
        if b >= n_live:                                   # inert: poisoned, never read
            r[:] = 50.0
            continue
        u = next(fresh)
        seen[u] = 0
        if kind == "draft_b_penalised" and b >= 1:        # draft b at 9 (/ rp < 8) against an unseen 8
            r[tok[b]], r[u] = 9.0, 8.0
        elif kind == "tok0":                              # tok[0] at 9 against an unseen 8: penalised only if seen
            r[tok0], r[u] = 9.0, 8.0
        elif kind == "negative_max" and b >= 1:           # all negative; draft b at -1 (x rp) against an unseen -1.25
            r.clamp_(max=-2.0)
            r[tok[b]], r[u] = -1.0, -1.25
        elif kind == "penalty_tie" and b >= 1 and rp == 2.0:   # draft b at 8 / 2 ties an unseen 4 at a lower / higher id
            u = 50 if b % 2 else V - 50
            seen[u] = 0
            r[tok[b]], r[u] = 8.0, 4.0
        else:                                             # an unseen winner just above an unseen runner-up: the next
            v = next(fresh)                               # draft is the winner and must not be penalised here
            seen[v] = 0
            r[u], r[v] = 8.0, 7.0
        pen = seen.clone()
        pen[torch.tensor(tok[1:b + 1], dtype=torch.long)] = 1
        want.append(greedy_reference(r.bfloat16()[None], pen[None], rp)[0])
        if b + 1 < ncols:
            tok.append(want[-1] if b + 1 < n_live else tok0)
    return lg.bfloat16(), seen, tok, want


KINDS = ["draft_b_penalised", "tok0", "negative_max", "penalty_tie", "plain"]


@pytest.mark.parametrize("rp", [1.3, 2.0, 3.1])
def test_greedy_scan_penalty_set_boundaries(emb, rp):
    """rp != 1 (the logits rows are scanned): column b's penalty set is seen + drafts 1..b.  Planted: draft b penalised in
    column b, draft b + 1 not, tok[0] only when seen, a negative maximum multiplied, and (rp = 2) a tie the penalty makes,
    won by the lower id."""
    calls = 0
    for seed, (ncols, n_live) in enumerate(((16, 16), (16, 12), (9, 9), (8, 8), (8, 3), (2, 2))):
        for tok0_seen in (False, True):
            lg, seen, tok, want = greedy_plan(rp, ncols, n_live, seed * 7 + int(tok0_seen), tok0_seen)
            hist = [30, 31, tok[0]]
            gen = dict(step=len(hist), cur_len=700, done=0, unfinished=1)
            p = params(200, rp=rp)
            spec = make_spec(ncols - 1, 2, tok, n_live, gen["cur_len"])
            exp = expect(p, hist, 256, gen, spec, seen, want, emb)
            got = run_op(GREEDY, p, hist, 256, gen, spec, seen, emb, logits=lg.to(DEV))
            compare(got, exp, f"scan rp={rp} ncols={ncols} n_live={n_live} tok0_seen={tok0_seen}")
            assert got["out"][len(hist):len(hist) + n_live].tolist() == want      # every live column's token was emitted
            calls += 1
    _calib(f"greedy scan rp={rp}", calls)


# ---- d. sampled selection ------------------------------------------------------------------------------------------------------
SPEC_SAMPLE_PARAMS = [(1.0, 1.0, 1.3), (0.9, 0.9, 1.0), (0.7, 0.95, 3.1), (1.5, 0.8, 1.3)]    # (T, top_p, rp)


@pytest.mark.parametrize("V", [49156, 49157])
def test_sampled_columns_follow_philox_and_fp64_cdf(emb, V):
    """128 calls x up to 16 columns per vocabulary: column b draws u = Philox(seed, (0, step + b)) from the distribution
    penalised by seen + drafts 1..b (within the select tests' 2e-6 CDF band); columns >= n_live keep sel; the walk,
    drafts and embeddings follow; a call with done set changes nothing."""
    base = [make_rows(V, seed=V + s).to(DEV) for s in range(2)]
    worst, calls = 0.0, 0
    g = torch.Generator().manual_seed(V)
    for call in range(128):
        T, top_p, rp = SPEC_SAMPLE_PARAMS[call % len(SPEC_SAMPLE_PARAMS)]
        rows = torch.roll(base[call % 2], shifts=call // 2, dims=0)
        ncols = 16 if call % 8 else 9
        n_live = ncols if call % 3 else max(1, ncols - 1 - call % 7)
        step = 3 + 37 * call % 1500
        seed = 1000 + call
        top = [int(torch.argmax(rows[b])) for b in range(ncols)]
        tok0 = int(torch.randint(0, V, (1,), generator=g))
        drafts = [top[b] if (b + call) % 3 else int(torch.randint(0, V, (1,), generator=g)) for b in range(ncols - 1)]
        tok = [tok0] + drafts
        seen = (torch.rand(V, generator=g) < 0.05).to(torch.uint8)
        hist = torch.randint(0, V, (step,), generator=g).tolist()
        hist[-1] = tok0
        seen[torch.tensor(hist)] = 1
        p = params(step + 100, eos=None, rp=rp, T=T, top_p=top_p, seed=seed)
        gen = dict(step=step, cur_len=step + 50, done=0, unfinished=1)
        spec = make_spec(ncols - 1, 2, tok, n_live, gen["cur_len"])
        lg = rows[:ncols].bfloat16()
        got = run_op(SAMPLE, p, hist, step + 128, gen, spec, seen, emb, V=V, logits=lg)
        sel = got["spec"]["sel"]
        assert sel[n_live:] == [-5] * (16 - n_live), "an inert column selected"
        seen_ids = seen.nonzero().flatten().to(DEV)
        for b in range(n_live):
            ids = torch.cat([seen_ids, torch.tensor(tok[1:b + 1], dtype=torch.long, device=DEV)])
            sc = hf_scores(lg[b].float(), ids, T, rp)
            u = sampler_u(seed, 0, step + b)
            ex = float(RowRef(sc, top_p).excess(torch.tensor([sel[b]], device=DEV), np.array([u]))[0])
            assert ex <= DELTA_CDF, f"call {call} column {b}: token {sel[b]} u {float(u):.8f} excess {ex:.3e}"
            worst = max(worst, ex)
        spec_in = make_spec(ncols - 1, 2, tok, n_live, gen["cur_len"])
        want = expect(p, hist, step + 128, gen, spec_in, seen, sel, emb, V=V)
        want["spec"]["sel"] = sel
        compare(got, want, f"sample call {call}")
        calls += 1
    # done on entry: nothing is selected or written
    spec = make_spec(ncols - 1, 2, tok, n_live, gen["cur_len"])
    done = dict(gen, done=1)
    got = run_op(SAMPLE, p, hist, step + 128, done, spec, seen, emb, V=V, logits=lg)
    compare(got, expect(p, hist, step + 128, done, make_spec(ncols - 1, 2, tok, n_live, gen["cur_len"]), seen, [], emb, V=V),
            "done on entry")
    _calib(f"sampled columns V={V}", calls, worst, DELTA_CDF)

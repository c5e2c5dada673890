"""The beam-search bookkeeping and KV-cache movement kernels one launch at a time (sv_op_beam_step, sv_op_beam_kv_copy,
sv_op_kv_gather, sv_op_session_admit), at the StarVector-1B and -8B cache shapes.

References, all exact:
  * beam_step_kernel: the host replay sv_beam_step_host, the same sv_beam_core.h code that tests/test_beam_core.py holds to
    HF generate(num_beams > 1).  Both start from identical inputs; after every step the whole state, both halves of the
    sequence buffers, next_ids, the counters and the plan are compared, and the next tokens' embeddings bitwise against
    bf16(float(wte[clamp(tok)]) + float(wpe[min(pos, n_positions - 1)])).  Rows >= R of x and next_ids keep sentinels.
  * beam_kv_copy_kernel: HF's whole-row `_reorder_cache`, `ref[:, :, :cache_hi + 1] = ref[run_parent]`, applied by torch to
    a copy of the caches; the suffix copies must leave every layer and row bit-equal to it.  The plans come from a chain of
    device beam steps, so rows 8-15 of the divergence matrix are checked here.
  * kv_gather_kernel: the source rows copied by torch.  K positions [0, len) and V^T positions [0, round_up(len, 8)) are
    copied (the V^T rows go in 16-byte vectors: the round-up to 8 is part of the contract, pinned here); past that, and in
    rows >= rows, the destination keeps its sentinel.
  * session_admit_kernel: the documented reset of the admitted slots; every other slot's bytes and fields unchanged.
The copy kernels stride their grids (4 CTAs x 256 threads per row and layer; beam_step's 1024 threads), so the suffixes,
sequence moves and fin_len boundaries are chosen to cross those strides.  `CALIB` lines (-s) count the calls per family.
"""
import ctypes as C

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200 import engine as E

pytestmark = pytest.mark.gpu
DEV = "cuda"
V0, PAD, EOS = 49156, 49152, 7
H1, H8 = 2048, 4608                       # hidden widths of StarVector-1B (learned positions) and -8B (RoPE: no wpe)
SHAPES = {"1b": dict(n_kv=1, tcap=8224, n_layer=3), "8b": dict(n_kv=4, tcap=16416, n_layer=2)}   # max_len 8192 / 16384
PREFIX = 259                              # the 1B visual prefix + prompt
SENT_BF16 = -777.0

_CALLS = {}


def _count(family, n=1):
    _CALLS[family] = _CALLS.get(family, 0) + n


@pytest.fixture(scope="module", autouse=True)
def _print_calib():
    yield
    for k in sorted(_CALLS):
        print(f"CALIB beam ops {k}: {_CALLS[k]} calls, every output exact")


@pytest.fixture(scope="module")
def emb():
    g = torch.Generator(device=DEV).manual_seed(5)
    wte1 = torch.randn(V0, H1, generator=g, device=DEV).bfloat16()
    wpe1 = (0.1 * torch.randn(8192, H1, generator=g, device=DEV)).bfloat16()
    wte8 = torch.randn(V0, H8, generator=g, device=DEV).bfloat16()
    return {"1b": (wte1, wpe1, 8192), "8b": (wte8, None, 16384)}


def _fp(t):
    return C.cast(t.data_ptr(), C.POINTER(C.c_float))


def _ip(t):
    return C.cast(t.data_ptr(), C.POINTER(C.c_int32)) if t is not None else None


def _copy(s):
    t = type(s)()
    C.memmove(C.addressof(t), C.addressof(s), C.sizeof(s))
    return t


def _bytes(s):
    return C.string_at(C.addressof(s), C.sizeof(s))


def beam_params(nb, max_new, es=1, lp=1.0, eos=-1, stop=()):
    bp = _lib.BeamParams(num_beams=nb, max_new_tokens=max_new, do_sample=0, early_stopping=es, temperature=1.0, top_p=1.0,
                         repetition_penalty=1.0, length_penalty=lp, eos_token_id=eos, pad_token_id=PAD, n_stop_ids=len(stop))
    for i, s in enumerate(stop):
        bp.stop_ids[i] = s
    return bp


def init_state(bp, B, first_cache_pos):
    s = _lib.BeamState()
    assert _lib.load().sv_beam_state_init_host(C.byref(bp), B, first_cache_pos, C.addressof(s)) == 0
    return s


PLAN_ROWS = ("run_parent", "run_tok", "fin_old", "fin_parent", "fin_tok", "copy_src", "copy_lo")


class Pair:
    """One search stepped by the device op and by the host replay from identical inputs; every step compares all outputs."""

    def __init__(self, bp, B, V, state, run_seq, fin_seq, cur_len, emb_set):
        self.bp, self.B, self.V = bp, B, V
        self.R, self.K, self.stride = B * bp.num_beams, 2 * bp.num_beams, run_seq.shape[-1]
        self.hstate, self.dstate = _copy(state), _copy(state)
        self.hrun, self.hfin = run_seq.clone().contiguous(), fin_seq.clone().contiguous()
        self.drun, self.dfin = run_seq.to(DEV), fin_seq.to(DEV)
        self.gen = [cur_len, 0]
        self.wte, self.wpe, self.npos = emb_set
        self.x = torch.full((16, self.wte.shape[1]), SENT_BF16, dtype=torch.bfloat16, device=DEV)
        self.next_ids = torch.full((16,), -7, dtype=torch.int32, device=DEV)
        self.plan = _lib.BeamPlan()
        C.memset(C.addressof(self.plan), 0xF7, C.sizeof(self.plan))
        self.steps = 0

    def running(self):
        return list(self.dstate.running_scores)[: self.R]

    def step(self, key, val, tok, advance):
        """key / val / tok: [R, K] (any device).  Returns (cont, cache_hi, plan)."""
        R, lib = self.R, _lib.load()
        key, val, tok = key.float().contiguous(), val.float().contiguous(), tok.to(torch.int32).contiguous()
        cache_hi = self.gen[0] - 1 + advance
        hk, hv, ht = key.cpu(), val.cpu(), tok.cpu()
        nxt = torch.full((R,), -1, dtype=torch.int32)
        src = torch.full((R,), -1, dtype=torch.int32)
        plan_out = torch.full((64,), -11, dtype=torch.int32) if R <= 8 else None
        cont = lib.sv_beam_step_host(C.byref(self.bp), self.B, self.V, self.stride, C.addressof(self.hstate), _fp(hk), _fp(hv),
                                     _ip(ht), _ip(self.hrun), _ip(self.hfin), cache_hi, _ip(nxt), _ip(src), _ip(plan_out))
        assert cont in (0, 1)
        gen0, x0, ids0 = list(self.gen), self.x.clone(), self.next_ids.clone()
        E.op_beam_step(self.bp, self.B, self.V, self.dstate, (key.to(DEV), val.to(DEV), tok.to(DEV)), self.drun, self.dfin,
                       self.gen, advance, self.wte, self.wpe, self.x, self.npos, self.next_ids, self.plan)
        _count("beam_step")
        self.steps += 1
        p = self.plan
        assert _bytes(self.dstate) == _bytes(self.hstate), f"step {self.steps}: state differs"
        assert torch.equal(self.drun.cpu(), self.hrun) and torch.equal(self.dfin.cpu(), self.hfin), f"step {self.steps}: sequences"
        assert p.cont == cont and list(p.run_parent)[:R] == src.tolist() and list(p.run_tok)[:R] == nxt.tolist()
        if plan_out is not None:
            po = plan_out.tolist()
            for a, name in enumerate(PLAN_ROWS):
                assert list(getattr(p, name))[:R] == po[8 * a: 8 * a + R], (self.steps, name)
            assert (p.copy_hi, p.cont, p.old_len) == tuple(po[56:59])
        assert self.gen == [gen0[0] + (advance if cont else 0), 0 if cont else 1]
        if cont:
            ids = torch.tensor(list(p.run_tok)[:R], device=DEV).clamp(0, self.V - 1).long()
            pos = min(self.gen[0], self.npos - 1)
            ref = self.wte[ids].float() + (self.wpe[pos].float()[None] if self.wpe is not None else 0.0)
            assert torch.equal(self.x[:R].view(torch.int16), ref.bfloat16().view(torch.int16)), f"step {self.steps}: embeddings"
            assert torch.equal(self.x[R:], x0[R:])
            assert self.next_ids[:R].tolist() == nxt.tolist() and torch.equal(self.next_ids[R:], ids0[R:])
        else:                        # the search ended: the next step's inputs and cur_len stay as they were
            assert torch.equal(self.x, x0) and torch.equal(self.next_ids, ids0)
        return cont, cache_hi, p


def random_candidates(pair, g, eos_rate=0.0, scale=3.0):
    """beam_candidates_kernel on random bf16 logits at V = 49156 (EOS planted as a row's best at rate eos_rate)."""
    R, V = pair.R, pair.V
    logits = torch.randn(R, V, generator=g, device=DEV) * scale
    if eos_rate > 0:
        hit = torch.rand(R, generator=g, device=DEV) < eos_rate
        logits[:, EOS] = torch.where(hit, logits.max(1).values + 1.0, logits[:, EOS])
    run = pair.drun[pair.dstate.parity]
    _count("beam_candidates (inputs)")
    return E.op_beam_candidates(logits.bfloat16(), pair.bp, pair.B, pair.dstate.cur_len, pair.running(), run)


def hand_candidates(pair, g, eos=None, plant=None):
    """Hand-built lists, each row best-first: running score + nonzero multiples of -0.25, so equal keys across beams and within
    a row are common.  plant: {row: token} becomes that row's best candidate, 0.5 above the rest."""
    R, K = pair.R, pair.K
    rs = torch.tensor(pair.running(), dtype=torch.float32)
    q = -(torch.randint(1, 6, (R, K), generator=g).float() * 0.25)     # < 0: running scores fall, the searches run long
    val = q.sort(1, descending=True).values + rs[:, None]
    tok = torch.stack([torch.randperm(pair.V, generator=g)[:K] for _ in range(R)]).to(torch.int32)
    if eos is not None:
        for r in range(R):
            if torch.rand(1, generator=g).item() < 0.2:
                tok[r, int(torch.randint(0, K // 2, (1,), generator=g))] = eos
    for r, t in (plant or {}).items():        # above every other candidate of the row's image (row 0 leads its image)
        tok[r, 0], val[r, 0] = t, rs[r] + 0.5
    return val, val.clone(), tok


SHAPES_BNB = [(1, 2), (2, 2), (1, 8), (2, 4), (4, 4), (8, 2), (2, 8)]
PARAM_SETS = {"es1-lp1-noeos": dict(es=1, lp=1.0, eos=False), "es1-lp1-eos": dict(es=1, lp=1.0, eos=True),
              "es0-lpm1-eos": dict(es=0, lp=-1.0, eos=True), "esnever-lp2-eos": dict(es=2, lp=2.0, eos=True)}


def _fresh_pair(B, nb, max_new, emb_set, es=1, lp=1.0, eos=-1, stop=(), V=V0, stride=None):
    bp = beam_params(nb, max_new, es=es, lp=lp, eos=eos, stop=stop)
    R, stride = B * nb, stride or max_new
    seq = torch.full((2, R, stride), PAD, dtype=torch.int32)
    return Pair(bp, B, V, init_state(bp, B, PREFIX), seq, seq.clone(), PREFIX, emb_set)


@pytest.mark.parametrize("pset", list(PARAM_SETS))
@pytest.mark.parametrize("B,nb", SHAPES_BNB, ids=str)
def test_beam_step_chain_from_the_candidates_kernel(emb, B, nb, pset):
    """48-step searches fed by beam_candidates_kernel: every step of the device op equals the host replay."""
    ps = PARAM_SETS[pset]
    pair = _fresh_pair(B, nb, 48, emb["1b"], es=ps["es"], lp=ps["lp"], eos=EOS if ps["eos"] else -1)
    g = torch.Generator(device=DEV).manual_seed(100 * B + nb)
    cont, advance = 1, 0
    while cont:
        cont, _, _ = pair.step(*random_candidates(pair, g, eos_rate=0.03 if ps["eos"] else 0.0), advance)
        advance = 1
    if not ps["eos"]:
        assert pair.steps == 48                       # ends at the step where cur + 1 == max_length


@pytest.mark.parametrize("B,nb", SHAPES_BNB, ids=str)
@pytest.mark.parametrize("stop", [False, True])
def test_beam_step_chain_with_planted_ties(emb, B, nb, stop):
    """40+ steps of hand-built lists with exact ties and EOS among the top candidates; with `stop`, row 0's best candidates
    spell the stop sequence at steps 30-31 and end the search there."""
    stop_ids = (4242, 4343) if stop else ()
    pair = _fresh_pair(B, nb, 64, emb["1b"], es=2, lp=1.0, eos=EOS, stop=stop_ids)
    g = torch.Generator().manual_seed(7 * B + nb)
    cont, advance = 1, 0
    while cont:
        plant = {0: stop_ids[pair.steps - 30]} if stop and pair.steps in (30, 31) else None
        cont, _, _ = pair.step(*hand_candidates(pair, g, eos=EOS if pair.steps < 30 or not stop else None, plant=plant), advance)
        advance = 1
    assert (pair.steps == 32) if stop else (pair.steps >= 40), pair.steps


def test_beam_step_tie_rules(emb):
    """Equal keys across beams go to the lower beam (merge), equal running scores to the lower k."""
    pair = _fresh_pair(1, 2, 16, emb["1b"])
    pair.dstate.running_scores[1] = pair.hstate.running_scores[1] = 0.0         # both beams alive with equal scores
    val = torch.tensor([[-1.0, -1.0, -2.0, -3.0]] * 2)
    tok = torch.tensor([[11, 12, 13, 14]] * 2, dtype=torch.int32)
    cont, _, p = pair.step(val, val.clone(), tok, 1)
    assert cont and list(p.run_parent)[:2] == [0, 0] and list(p.run_tok)[:2] == [11, 12]


def _long_state(bp, B, cur, seed):
    """A state deep into a search: cur_len near 3000, finished hypotheses of 1023-1025 tokens kept in permuted order,
    divergence entries between the prefix and cache_hi + 1."""
    g = torch.Generator().manual_seed(seed)
    nb, R = bp.num_beams, B * bp.num_beams
    s = init_state(bp, B, PREFIX)
    s.cur_len, s.parity = cur, seed % 2
    lens = [1023, 1024, 1025, 700, cur, 1, 1024, 1025]
    for r in range(R):
        j = r % nb
        s.running_scores[r] = -1.0 - 0.5 * j
        s.beam_scores[r] = -5.0 + 0.5 * j                  # ascending: the merge reverses the finished slots
        s.is_finished[r] = 1
        s.fin_len[r] = lens[(r + seed) % len(lens)]
    hi = PREFIX + cur
    for r in range(R):
        for q in range(R):
            s.div[r][q] = int(torch.randint(PREFIX, hi + 1, (1,), generator=g)) if r // nb == q // nb else PREFIX
    return s


@pytest.mark.parametrize("B,nb", [(2, 4), (4, 4), (2, 8)], ids=str)
@pytest.mark.parametrize("cur", [2990, 3071])
def test_beam_step_long_histories(emb, B, nb, cur):
    """Sequence moves of ~3000 tokens and fin_len 1023 / 1024 / 1025 across the kernel's 1024-thread strides."""
    bp = beam_params(nb, 4000, es=0, lp=1.0, eos=EOS)
    R, stride = B * nb, 4096
    g = torch.Generator().manual_seed(cur + R)
    run = torch.randint(0, V0, (2, R, stride), generator=g, dtype=torch.int32)
    fin = torch.randint(0, V0, (2, R, stride), generator=g, dtype=torch.int32)
    pair = Pair(bp, B, V0, _long_state(bp, B, cur, B + nb), run, fin, PREFIX + cur, emb["1b"])
    boundary_kept = 0
    for s in range(6):
        cont, _, p = pair.step(*hand_candidates(pair, g, eos=EOS if s >= 3 else None), 1)
        assert cont
        boundary_kept += sum(p.fin_old[r] >= 0 and pair.dstate.fin_len[r] in (1023, 1024, 1025) for r in range(R))
    assert boundary_kept >= 3            # finished rows at the stride edges really were moved


@pytest.mark.parametrize("width", ["1b", "8b"])
@pytest.mark.parametrize("B,nb", [(2, 2), (2, 8)], ids=str)
def test_beam_step_embeddings_at_the_position_limit(emb, width, B, nb):
    """Positions n_positions - 2 .. n_positions + 2 (the last two clamped to n_positions - 1), advance 0 then 1, and token
    ids outside the vocabulary (clamped) among the selected ones."""
    wte, wpe, _ = emb[width]
    npos = 300
    pair = _fresh_pair(B, nb, 16, (wte, wpe, npos))
    pair.gen[0] = npos - 2
    g = torch.Generator().manual_seed(B * nb)
    advance = 0
    for s in range(5):
        plant = {0: V0 + 3, pair.R - 1: -2} if s in (1, 3) else None
        cont, _, _ = pair.step(*hand_candidates(pair, g, plant=plant), advance)
        assert cont and pair.gen[0] == npos - 2 + s
        advance = 1


def test_beam_step_is_a_no_op_once_done(emb):
    """The captured graph keeps replaying after the search ends: with `done` set nothing may change, the plan included."""
    B, nb = 2, 4
    bp = beam_params(nb, 64, eos=EOS)
    R, stride = B * nb, 64
    g = torch.Generator().manual_seed(3)
    s = init_state(bp, B, PREFIX)
    s.cur_len, s.done, s.parity = 40, 1, 1
    for r in range(R):
        s.running_scores[r], s.fin_len[r], s.is_finished[r] = -0.5 * r, r, r % 2
    run = torch.randint(0, V0, (2, R, stride), generator=g, dtype=torch.int32).to(DEV)
    fin = torch.randint(0, V0, (2, R, stride), generator=g, dtype=torch.int32).to(DEV)
    run0, fin0, s0 = run.clone(), fin.clone(), _bytes(s)
    wte, wpe, npos = emb["1b"]
    x = torch.full((16, H1), SENT_BF16, dtype=torch.bfloat16, device=DEV)
    ids = torch.full((16,), -7, dtype=torch.int32, device=DEV)
    plan = _lib.BeamPlan()
    C.memset(C.addressof(plan), 0xF7, C.sizeof(plan))
    p0 = _bytes(plan)
    val = torch.zeros(R, 2 * nb, device=DEV)
    tok = torch.full((R, 2 * nb), EOS, dtype=torch.int32, device=DEV)
    gen = [PREFIX + 40, 0]
    E.op_beam_step(bp, B, V0, s, (val, val, tok), run, fin, gen, 1, wte, wpe, x, npos, ids, plan)
    _count("beam_step")
    assert _bytes(s) == s0 and _bytes(plan) == p0 and gen == [PREFIX + 40, 0]
    assert torch.equal(run, run0) and torch.equal(fin, fin0)
    assert bool((x == SENT_BF16).all()) and bool((ids == -7).all())


# ---- KV suffix copies ---------------------------------------------------------------------------------------------------
def _caches(shape, fill=None, seed=0):
    n_layer, n_kv, tcap = shape["n_layer"], shape["n_kv"], shape["tcap"]
    k = torch.empty(n_layer, 16, n_kv, tcap, 128, dtype=torch.bfloat16, device=DEV)
    v = torch.empty(n_layer, 16, n_kv, 128, tcap, dtype=torch.bfloat16, device=DEV)
    if fill is None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        k.normal_(generator=g)
        v.normal_(generator=g)
    else:
        k.fill_(fill)
        v.fill_(fill)
    return k, v


@pytest.mark.parametrize("shape,B,nb", [("1b", 2, 2), ("1b", 4, 4), ("1b", 2, 8), ("8b", 4, 4), ("8b", 1, 8)], ids=str)
def test_beam_kv_copy_chain_equals_whole_row_reorder(emb, shape, B, nb):
    """44-step searches: a simulated forward writes a fresh K/V column at cache_hi for every row and layer, the device step
    plans the copies, and after them every cache row equals HF's whole-row reorder of the same history."""
    sh = SHAPES[shape]
    pair = _fresh_pair(B, nb, 44, emb["1b"])
    R = pair.R
    k, v = _caches(sh, fill=SENT_BF16)
    g = torch.Generator(device=DEV).manual_seed(17 * B + nb)
    for b in range(B):                                  # the beams of an image share the prefill
        k[:, b * nb:(b + 1) * nb, :, :PREFIX] = torch.randn(sh["n_layer"], 1, sh["n_kv"], PREFIX, 128, generator=g, device=DEV).bfloat16()
        v[:, b * nb:(b + 1) * nb, :, :, :PREFIX] = torch.randn(sh["n_layer"], 1, sh["n_kv"], 128, PREFIX, generator=g, device=DEV).bfloat16()
    rk, rv = k.clone(), v.clone()
    cont, advance, far = 1, 0, 0
    while cont:
        if advance:                                     # the forward of the tokens fed last step writes column cur_len
            pos = pair.gen[0]
            ck = torch.randn(sh["n_layer"], R, sh["n_kv"], 128, generator=g, device=DEV).bfloat16()
            cv = torch.randn(sh["n_layer"], R, sh["n_kv"], 128, generator=g, device=DEV).bfloat16()
            k[:, :R, :, pos], rk[:, :R, :, pos] = ck, ck
            v[:, :R, :, :, pos], rv[:, :R, :, :, pos] = cv, cv
        cont, cache_hi, p = pair.step(*random_candidates(pair, g, scale=2.0), advance)
        advance = 1
        if not cont:
            break
        E.op_beam_kv_copy(k, v, R, p)
        _count(f"beam_kv_copy {shape}")
        parent = torch.tensor(list(p.run_parent)[:R], device=DEV)
        rk[:, :R], rv[:, :R] = rk[:, parent], rv[:, parent]
        assert p.copy_hi == cache_hi
        assert torch.equal(k, rk) and torch.equal(v, rv), f"step {pair.steps}: the cache differs from the whole-row reorder"
        far = max([far] + [cache_hi - p.copy_lo[r] for r in range(8, R) if p.copy_src[r] >= 0])
    assert pair.steps == 44
    if R > 8:
        assert far >= 2, "rows 8-15 never copied a suffix of more than two positions: the check lost its power"


def _plan(copy_hi, rows, cont=1):
    p = _lib.BeamPlan(copy_hi=copy_hi, cont=cont)
    for r in range(16):
        p.copy_src[r], p.copy_lo[r] = -1, 0
    for r, (src, lo) in rows.items():
        p.copy_src[r], p.copy_lo[r] = src, lo
    return p


HAND_PLANS = {
    # a swap (0 <- 1, 1 <- 0) and a 3-cycle (2 <- 3 <- 4 <- 2): correct only through the staging phase
    "cycles": (600, {0: (1, 259), 1: (0, 300), 2: (3, 0), 3: (4, 580), 4: (2, 599), 9: (15, 311), 15: (9, 259)}),
    # one-token (lo == hi), empty (lo > hi), lo = 0, and a long suffix over several grid strides
    "edges": (8000, {0: (1, 8000), 1: (2, 8001), 2: (3, 0), 3: (0, 259), 8: (12, 4000), 12: (8, 7999), 5: (5, 100)}),
    "last-slot": (None, {0: (3, 0), 3: (0, 8192), 7: (6, 9000)}),
    "no-op": (500, {0: (1, 0), 1: (0, 0)}),
}


@pytest.mark.parametrize("name", list(HAND_PLANS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_beam_kv_copy_hand_built_plans(shape, name):
    sh = SHAPES[shape]
    hi, rows = HAND_PLANS[name]
    hi = sh["tcap"] - 1 if hi is None else hi
    p = _plan(hi, rows, cont=0 if name == "no-op" else 1)
    R = 16
    k, v = _caches(sh, seed=len(name))
    rk, rv = k.clone(), v.clone()
    if p.cont:
        for r in range(R):
            src, lo = p.copy_src[r], p.copy_lo[r]
            if src >= 0 and lo <= hi:
                rk[:, r, :, lo:hi + 1] = k[:, src, :, lo:hi + 1]
                rv[:, r, :, :, lo:hi + 1] = v[:, src, :, :, lo:hi + 1]
    E.op_beam_kv_copy(k, v, R, p)
    _count(f"beam_kv_copy {shape}")
    assert torch.equal(k, rk) and torch.equal(v, rv)


# ---- kv_gather ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gather_src():
    out = {}
    for name, sh in SHAPES.items():
        one = dict(sh, n_layer=1)
        k, v = _caches(one, seed=31)
        out[name] = (k[0], v[0])
    return out


IDX = {"perm": (16, lambda g: torch.randperm(16, generator=g)), "dup": (13, lambda g: torch.arange(16) // 4), "null": (11, None)}


def _round8(n):
    return (n + 7) // 8 * 8


def _len(length, tcap):
    return {"tcap-1": tcap - 1, "tcap": tcap}.get(length, length)


@pytest.mark.parametrize("length", [1, 7, 8, 9, 259, 580, "tcap-1", "tcap"])
@pytest.mark.parametrize("kind", list(IDX))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_kv_gather_rows(gather_src, shape, kind, length):
    ks, vs = gather_src[shape]
    tcap = ks.shape[2]
    n = _len(length, tcap)
    rows, make = IDX[kind]
    idx = make(torch.Generator().manual_seed(n)) if make else None
    kd, vd = torch.full_like(ks, SENT_BF16), torch.full_like(vs, SENT_BF16)
    ek, ev = kd.clone(), vd.clone()
    sel = (idx if idx is not None else torch.arange(16))[:rows].to(DEV)
    ek[:rows, :, :n] = ks[sel, :, :n]
    ev[:rows, :, :, :_round8(n)] = vs[sel, :, :, :_round8(n)]       # V^T goes in 8-key vectors: round_up(len, 8)
    E.op_kv_gather(ks, vs, kd, vd, idx.to(torch.int32).to(DEV) if idx is not None else None, rows, n)
    _count(f"kv_gather {shape}")
    assert torch.equal(kd, ek) and torch.equal(vd, ev)


@pytest.mark.parametrize("length", [580, "tcap-1"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_kv_gather_in_place_reorder(gather_src, shape, length):
    """sv_reorder_cache's form: gather into a one-layer scratch, copy back with identity; = index_select on rows."""
    ks, vs = gather_src[shape]
    n = _len(length, ks.shape[2])
    k, v = ks.clone(), vs.clone()
    sk, sv = torch.full_like(k, SENT_BF16), torch.full_like(v, SENT_BF16)
    idx = torch.tensor([3, 3, 0, 1, 15, 14, 2, 2, 9, 8, 8, 7, 6, 5, 4, 0], dtype=torch.int32, device=DEV)
    ek, ev = k.clone(), v.clone()
    ek[:, :, :n] = torch.index_select(k, 0, idx.long())[:, :, :n]
    ev[..., :_round8(n)] = torch.index_select(v, 0, idx.long())[..., :_round8(n)]
    E.op_kv_gather(k, v, sk, sv, idx, 16, n)
    E.op_kv_gather(sk, sv, k, v, None, 16, n)
    _count(f"kv_gather {shape}", 2)
    assert torch.equal(k, ek) and torch.equal(v, ev)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_kv_gather_session_slot_copy(gather_src, shape):
    """sv_session_admit's n-completions copy: slot-offset pointers, rows = 1, len = the prefix."""
    ks, vs = gather_src[shape]
    k, v = ks.clone(), vs.clone()
    for first, slot, n in ((3, 9, PREFIX), (0, 15, 580), (15, 1, 583)):
        ek, ev = k.clone(), v.clone()
        ek[slot, :, :n] = k[first, :, :n]
        ev[slot, :, :, :_round8(n)] = v[first, :, :, :_round8(n)]
        E.op_kv_gather(k[first:first + 1], v[first:first + 1], k[slot:slot + 1], v[slot:slot + 1], None, 1, n)
        _count(f"kv_gather {shape}")
        assert torch.equal(k, ek) and torch.equal(v, ev)


# ---- session admission ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 3, 16])
@pytest.mark.parametrize("V", [49156, 49157])
def test_session_admit_resets_only_the_admitted_slots(V, k):
    S, stride = 16, 8192
    g = torch.Generator().manual_seed(V + k)
    seen = torch.randint(1, 256, (S, V), generator=g, dtype=torch.uint8).to(DEV)
    out = torch.randint(0, V, (S, stride), generator=g, dtype=torch.int32).to(DEV)
    rnd = lambda: torch.randint(0, 1 << 20, (S,), generator=g).tolist()
    state = dict(row_len=rnd(), row_step=rnd(), row_active=[int(a) for a in torch.randint(0, 2, (S,), generator=g)],
                 row_max_new=rnd(), row_seed=[(a << 40) | b for a, b in zip(rnd(), rnd())], event=5)
    slots = torch.randperm(S, generator=g)[:k].tolist()
    lens = [PREFIX + j for j in range(k)]
    max_new = [100 + 3 * j for j in range(k)]
    seeds = [(1 << 63) + 977 * j for j in range(k)]
    exp_seen, exp_out = seen.clone(), out.clone()
    exp = {key: list(val) if isinstance(val, list) else val for key, val in state.items()}
    for j, s in enumerate(slots):
        exp_seen[s], exp_out[s] = 0, PAD
        exp["row_len"][s], exp["row_step"][s], exp["row_active"][s] = lens[j], 0, 1
        exp["row_max_new"][s], exp["row_seed"][s] = max_new[j], seeds[j]
    E.op_session_admit(slots, lens, max_new, seeds, seen, out, PAD, state)
    _count("session_admit")
    assert torch.equal(seen, exp_seen) and torch.equal(out, exp_out)
    assert state == exp

"""The teacher-forced scoring kernels one launch at a time, against fp64 references at the 1B and 8B shapes
(sv_op_attention_score, sv_op_lm_logprob, sv_op_logits_logprob), and the chunk bookkeeping of sv_score_tokens through
Engine.score at full widths.

Tolerances (the worst error / tolerance of every family is printed as one `CALIB` line at the end, with -s):
  chunk attention:        1 ulp(ref) + 0.02 rms(ref of that row and head); bitwise independent of the poison in unread
                          slots, bitwise repeatable, bitwise equal to the same queries split over two calls; the
                          scattered K / V bit-exact and every other slot untouched
  lm log-prob, exact:     1e-5 + 1 fp32 ulp(ref) of the fp64 log-softmax (every logit is exact in bf16, asserted)
  lm log-prob, random:    ulp(l_t) + sum_i p_i ulp(l_i) + 1e-5 against fp64 logits rounded to bf16: a logit one bf16 ulp
                          off moves logZ by at most p_i ulp(l_i)
  epilogue vs resident:   EPI_TOL + 1 fp32 ulp(ref), both paths against the fp64 log-softmax of the bf16 logits
                          sv_op_lm_logits writes (the same values: only the fp32 reductions differ)
  resident logits:        1e-5 + 1 fp32 ulp(ref); a target outside [0, vocab) gives NaN
  ragged calls:           1e-5 between one Engine.score call and the same tokens over ragged calls; the decode step
                          after them gives bitwise equal logits (the appended KV rows and their positions)
"""
import functools
import math

import pytest
import torch

from starvector_b200 import engine as E
from starvector_b200.config import dims_1b, dims_8b
from starvector_b200.engine import Engine
from starvector_b200.weights import synthetic_state_dict
from test_ops_gpu import _close_attn, plant_strong_keys, ref_causal_attention

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
D = 128
EPI_TOL = 4e-6

_WORST = {}


def _calib(family, ratio):
    _WORST[family] = max(_WORST.get(family, 0.0), float(ratio))
    assert ratio <= 1.0, f"{family}: worst error / tolerance = {ratio:.3f}"


@pytest.fixture(scope="module", autouse=True)
def _print_calib():
    yield
    for k in sorted(_WORST):
        print(f"CALIB {k}: worst error / tolerance = {_WORST[k]:.3f}")


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _round32(x):
    return (x + 31) // 32 * 32


def _ulp32(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -126))) - 23)


def _ulp_bf16(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -126))) - 7)


# ---- chunk attention over caller-owned caches ---------------------------------------------------------------------------
def _strong_positions(pos0, C, window):
    """Keys every head of a group scores at 20: pos0 - 1, pos0, the tile edge after pos0 (and 31/32/33), the last position,
    and with a window the window starts (first visible key and the one before it) of the first and last query of the
    first, middle and last CTA (8 queries) and of CTAs whose queries' window starts straddle a 32-key tile edge."""
    L = pos0 + C
    e = _round32(pos0 + 1)
    pos = {pos0 - 1, pos0, L - 1, 31, 32, 33, e - 1, e, e + 1}
    if window:
        nct = (C + 7) // 8
        last = [pos0 + min(C, 8 * c + 8) - 1 for c in range(nct)]
        straddle = [c for c in range(nct) if max(0, pos0 + 8 * c + 1 - window) // 32 != max(0, last[c] + 1 - window) // 32]
        for c in {0, nct // 2, nct - 1} | set(straddle[:1] + straddle[-1:]):
            for q in (pos0 + 8 * c, last[c]):
                pos |= {q - window, q - window + 1}
    return sorted(p for p in pos if 0 <= p < L)


def _split(t_list, C):
    return sorted({t for t in t_list if 0 < t < C})


def _check_attention_score(B, C, pos0, nh, nkv, window, seed):
    grp, cols, L = nh // nkv, (nh + 2 * nkv) * D, pos0 + C
    tcap = _round32(L + 1)                           # as the engine: round32(max_len + 1)
    x = torch.randn(B * L, cols, generator=torch.Generator().manual_seed(seed)).to(BF)
    groups = [([(k * grp + j) * D for j in range(grp)], (nh + k) * D, (nh + nkv + k) * D) for k in range(nkv)]
    plant_strong_keys(x, B, L, groups, D, _strong_positions(pos0, C, window), seed=seed)
    x = x.to(DEV).view(B, L, nh + 2 * nkv, D)
    chunk = x[:, pos0:].reshape(B * C, cols).contiguous()
    strong_k = x[:, L - 1, nh:nh + nkv]               # [B, nkv, D]: scores 20 for every head of its group

    def fresh(kscale, vval):
        """The prefix K / V in slots [0, pos0) of images < B; a finite poison in every other slot and in image B's row."""
        pk = (strong_k.float() * kscale).to(BF)
        kc = torch.empty(B + 1, nkv, tcap, D, dtype=BF, device=DEV)
        kc[:B] = pk[:, :, None, :]
        kc[B] = pk[0, :, None, :]
        vc = torch.full((B + 1, nkv, D, tcap), vval, dtype=BF, device=DEV)
        kc[:B, :, :pos0] = x[:, :pos0, nh:nh + nkv].transpose(1, 2)
        vc[:B, :, :, :pos0] = x[:, :pos0, nh + nkv:].permute(0, 2, 3, 1)
        return kc, vc

    kc, vc = fresh(1.5, 500.0)
    kc0, vc0 = kc.clone(), vc.clone()
    out = E.op_attention_score(chunk, kc, vc, C, pos0, nh, nkv, window)
    kc2, vc2 = fresh(-1.0, -300.0)
    assert torch.equal(out, E.op_attention_score(chunk, kc2, vc2, C, pos0, nh, nkv, window)), \
        "the output depends on cache slots the attention must not read"
    kc3, vc3 = fresh(1.5, 500.0)
    assert torch.equal(out, E.op_attention_score(chunk, kc3, vc3, C, pos0, nh, nkv, window)), "not bitwise repeatable"
    # the scatter: slots [pos0, pos0 + C) of images < B are the chunk's K / V columns bit for bit; nothing else changed
    assert torch.equal(kc[:B, :, pos0:L], x[:, pos0:, nh:nh + nkv].transpose(1, 2))
    assert torch.equal(vc[:B, :, :, pos0:L], x[:, pos0:, nh + nkv:].permute(0, 2, 3, 1))
    assert torch.equal(kc[:, :, :pos0], kc0[:, :, :pos0]) and torch.equal(kc[:, :, L:], kc0[:, :, L:])
    assert torch.equal(vc[:, :, :, :pos0], vc0[:, :, :, :pos0]) and torch.equal(vc[:, :, :, L:], vc0[:, :, :, L:])
    assert torch.equal(kc[B], kc0[B]) and torch.equal(vc[B], vc0[B])
    # the same queries over two calls split at t (the second reads the first's K / V from the cache): the same bits
    xc = chunk.view(B, C, cols)
    for t in _split((1, 7, 8, 9, 31, C // 2, C - 1), C):
        kc4, vc4 = fresh(1.5, 500.0)
        a = E.op_attention_score(xc[:, :t].reshape(B * t, cols).contiguous(), kc4, vc4, t, pos0, nh, nkv, window)
        b = E.op_attention_score(xc[:, t:].reshape(B * (C - t), cols).contiguous(), kc4, vc4, C - t, pos0 + t, nh, nkv,
                                 window)
        both = torch.cat([a.view(B, t, -1), b.view(B, C - t, -1)], 1).view(B * C, -1)
        assert torch.equal(both, out), f"split at t = {t} changes the output"
    ref = ref_causal_attention(x.view(B * L, cols), B, L, nh, nkv, window, chunk=256, q0=pos0)
    _calib("chunk attention", _close_attn(out, ref, D))


P1B = 259                  # the 1B visual prefix (257 + "<svg")
SCORE_ATTN_CASES = [       # (B, C, pos0, n_head, n_kv, window): C = 4096 / B at the 1B grouping
    (1, 4096, P1B, 16, 1, 0), (1, 4096, P1B + 4096, 16, 1, 0), (3, 1365, P1B, 16, 1, 0), (3, 1365, P1B + 2 * 1365, 16, 1, 0),
    (8, 512, P1B, 16, 1, 0), (8, 512, P1B + 3 * 512, 16, 1, 0), (16, 256, P1B, 16, 1, 0), (16, 256, P1B + 7 * 256, 16, 1, 0),
    (3, 1365, 1023, 16, 1, 0), (3, 1365, 1024, 16, 1, 0), (3, 1365, 1025, 16, 1, 0), (2, 100, 0, 16, 1, 0),
    # 8B: 36 heads over 4 KV heads, window 4096 below, across and far past
    (2, 1024, 4000, 36, 4, 4096), (2, 2048, 4090, 36, 4, 4096), (1, 1024, 9000, 36, 4, 4096), (1, 2048, 9000, 36, 4, 4096),
    # the tiny groupings with window 24
    (2, 45, 300, 4, 2, 24), (3, 100, 40, 18, 2, 24), (2, 64, 0, 4, 2, 24), (2, 333, 77, 18, 2, 24),
] + [(2, c, P1B, 16, 1, 0) for c in (1, 7, 8, 9, 17)] + [(2, c, 300, 4, 2, 24) for c in (1, 7, 8, 9, 17)]


@pytest.mark.parametrize("B,C,pos0,nh,nkv,window", SCORE_ATTN_CASES, ids=lambda v: str(v))
def test_attention_score(B, C, pos0, nh, nkv, window):
    """sv_op_attention_score as run_score_chunk calls it: the chunk's B x C qkv rows, the prefix already in the cache,
    tcap = round32(pos0 + C + 1), a finite poison in every slot past the chunk and in the next image's row."""
    _check_attention_score(B, C, pos0, nh, nkv, window, seed=C * 7 + pos0 + nh)


# ---- the fused lm_head log-likelihood -----------------------------------------------------------------------------------
LM_SHAPES = [(2048, 49156), (2048, 49157), (4608, 49156), (4608, 49157)]        # (K, N): 1B / 8B hidden, both vocabularies
LM_M = [1, 8, 64, 127, 128, 129, 1365 * 3, 4096]
TIE, HOT, HOT_COL = 63, 64, 484         # x columns of the planted rows; HOT_COL lies in warp 3 of N-tile 3


@functools.lru_cache(maxsize=1)
def _exact_w(K, N):
    """w in quarter steps of [-2, 2].  Column TIE: maximum 3 at rows 5 and N - 2 (the last, partial N-tile).  Column HOT:
    -60 over N-tile 3 except +60 at HOT_COL."""
    g = _gen(K + N)
    w = torch.randint(-8, 9, (N, K), generator=g, device=DEV).float() * 0.25
    w[:, TIE] = w[:, TIE].clamp(max=2.0)
    w[5, TIE] = w[N - 2, TIE] = 3.0
    w[384:512, HOT] = -60.0
    w[HOT_COL, HOT] = 60.0
    return w.to(BF)


def _exact_rows(M, K, N, seed):
    """Sparse +-1 rows of x (nonzeros at 64-element stage edges and at K - 1, never at TIE / HOT) with targets, and the
    planted rows at the front (and again at the end when M >= 32): a tied maximum as target, the tie in the last partial
    tile, +60 / -60 in a tile of the opposite sign, a flat row, the last column, the row maximum."""
    g = _gen(seed)
    edges = sorted({0, K - 1} | {64 * j - 1 for j in range(2, K // 64)} | {64 * j for j in range(2, K // 64)})
    edges = torch.tensor(edges, device=DEV)
    x = torch.zeros(M, K, device=DEV)
    idx = edges[torch.randint(len(edges), (M, 6), generator=g, device=DEV)]
    x.scatter_(1, idx, (torch.randint(0, 2, (M, 6), generator=g, device=DEV) * 2 - 1).float())
    tg = torch.randint(0, N, (M,), generator=g, device=DEV)
    plant = [(TIE, 1.0, 5), (TIE, 1.0, N - 2), (HOT, 1.0, HOT_COL), (HOT, -1.0, HOT_COL), (None, 0.0, 17),
             (-1, 0.0, N - 1), (-1, 0.0, "max")]
    rows = list(range(min(M, len(plant))))
    if M >= 32:
        rows += [M - 1 - i for i in range(len(plant))]
    for r in rows:
        col, sign, t = plant[r if r < len(plant) else M - 1 - r]
        if col is not None and col >= 0:
            x[r] = 0.0
            x[r, col] = sign
        elif col is None:
            x[r] = 0.0
        tg[r] = -1 if t == "max" else t
    return x, tg


def _exact_logits(x, w, tg):
    logits = x.double() @ w.double().T
    assert torch.equal(logits, logits.to(BF).double()), "the planted inputs must give logits exact in bf16"
    tg = torch.where(tg < 0, logits.argmax(-1), tg)
    return logits, tg


def _lp(logits, tg):
    return torch.log_softmax(logits, dim=-1).gather(-1, tg.long()[:, None]).squeeze(-1)


@pytest.mark.parametrize("M", LM_M)
@pytest.mark.parametrize("K,N", LM_SHAPES, ids=lambda v: str(v))
def test_lm_logprob_exact(K, N, M):
    """Exact inputs: the fused epilogue and, over the same bf16 logits, the resident-logits path must match the fp64
    log-softmax to fp32 precision.  The +60 among -60 row would overflow a tile sum whose maximum missed a warp."""
    w = _exact_w(K, N)
    x, tg = _exact_rows(M, K, N, seed=M + K + N)
    logits, tg = _exact_logits(x, w, tg)
    ref = _lp(logits, tg)
    tol = 1e-5 + _ulp32(ref)
    got = E.op_lm_logprob(x.to(BF), w, tg).double()
    _calib("lm log-prob exact", ((got - ref).abs() / tol).max().item())
    res = E.op_logits_logprob(logits.to(BF), tg).double()
    _calib("resident logits", ((res - ref).abs() / tol).max().item())
    if M >= 7:
        assert logits[0, 5] == logits[0].max() and logits[1, N - 2] == logits[1].max() and logits[2, HOT_COL] == 60.0
        assert ref[4].item() == pytest.approx(-math.log(N), abs=1e-12)


@functools.lru_cache(maxsize=1)
def _random_w(K, N):
    return (torch.randn(N, K, generator=_gen(K * 3 + N), device=DEV) * (2.0 / math.sqrt(K))).to(BF)


@pytest.mark.parametrize("M", [1, 127, 129, 4096])
@pytest.mark.parametrize("K,N", LM_SHAPES, ids=lambda v: str(v))
def test_lm_logprob_random(K, N, M):
    w = _random_w(K, N)
    g = _gen(M * 5 + K)
    x = torch.randn(M, K, generator=g, device=DEV).to(BF)
    tg = torch.randint(0, N, (M,), generator=g, device=DEV)
    tg[-1] = N - 1
    lb = (x.double() @ w.double().T).to(BF).double()
    ref = _lp(lb, tg)
    lt = lb.gather(-1, tg[:, None]).squeeze(-1)
    tol = _ulp_bf16(lt) + (torch.softmax(lb, dim=-1) * _ulp_bf16(lb)).sum(-1) + 1e-5
    got = E.op_lm_logprob(x, w, tg).double()
    _calib("lm log-prob random", ((got - ref).abs() / tol).max().item())


@pytest.mark.parametrize("M", [1, 129, 4096])
@pytest.mark.parametrize("K,N", [(2048, 49156), (4608, 49157)], ids=lambda v: str(v))
def test_epilogue_and_resident_logits_agree(K, N, M):
    """run_score_chunk leaves resident logits from sv_op_lm_logits' tiling so that position 0 of the next call sees the
    bf16 values the fused epilogue saw: both paths must be within fp32 reduction error of log_softmax(those logits)."""
    w = _random_w(K, N)
    g = _gen(M * 11 + K)
    x = torch.randn(M, K, generator=g, device=DEV).to(BF)
    tg = torch.randint(0, N, (M,), generator=g, device=DEV)
    logits = E.op_lm_logits(x, w)
    ref = _lp(logits.double(), tg)
    tol = EPI_TOL + _ulp32(ref)
    fused = E.op_lm_logprob(x, w, tg).double()
    res = E.op_logits_logprob(logits, tg).double()
    _calib("epilogue vs resident", max(((fused - ref).abs() / tol).max().item(), ((res - ref).abs() / tol).max().item()))


# ---- the resident-logits path -----------------------------------------------------------------------------------------------
def _resident_rows(M, V, seed):
    """bf16 logits ~ 3 N(0, 1) with planted rows: a tied maximum (target on it, and on its copy in the last tile), -60 with
    +60 in warp 3 of a tile, a flat row, the last column, the row maximum, and two targets outside [0, V)."""
    g = _gen(seed)
    lg = (torch.randn(M, V, generator=g, device=DEV) * 3).to(BF).double()
    tg = torch.randint(0, V, (M,), generator=g, device=DEV)
    hot = 128 * min(3, (V - 1) // 128) + 100
    hot = hot if hot < V else V - 1
    plant = ["tie", "tie_last", "hot", "flat", "last", "max", "below", "above"]
    rows = list(range(min(M, len(plant))))
    if M >= 32:
        rows += [M - 1 - i for i in range(len(plant))]
    for r in rows:
        kind = plant[r if r < len(plant) else M - 1 - r]
        if kind in ("tie", "tie_last"):
            lg[r, 5] = lg[r, V - 2] = 20.0
            tg[r] = 5 if kind == "tie" else V - 2
        elif kind == "hot":
            lg[r] = -60.0
            lg[r, hot] = 60.0
            tg[r] = hot
        elif kind == "flat":
            lg[r] = 0.0
        elif kind == "last":
            tg[r] = V - 1
        elif kind == "max":
            tg[r] = lg[r].argmax()
        else:
            tg[r] = -1 if kind == "below" else V
    return lg, tg


@pytest.mark.parametrize("V", [500, 49156, 49157])
def test_logits_logprob(V):
    for M in list(range(1, 17)) + [4096]:
        lg, tg = _resident_rows(M, V, seed=M * 3 + V)
        bad = (tg < 0) | (tg >= V)
        got = E.op_logits_logprob(lg.to(BF), tg).double()
        assert bool(got[bad].isnan().all()), "a target outside [0, vocab) must give NaN"
        ref = _lp(lg[~bad], tg[~bad])
        tol = 1e-5 + _ulp32(ref)
        _calib("resident logits", ((got[~bad] - ref).abs() / tol).max().item())


def test_lm_logprob_unmatched_targets_are_nan():
    """The target-logit scratch starts as NaN: a target no column matches cannot return leftover memory."""
    K, N = 2048, 49157
    w = _random_w(K, N)
    x = torch.randn(6, K, generator=_gen(9), device=DEV).to(BF)
    tg = torch.tensor([-1, N, N + 5, 3, N - 1, -100], device=DEV)
    for _ in range(2):
        got = E.op_lm_logprob(x, w, tg)
        assert bool(got[[0, 1, 2, 5]].isnan().all()) and bool(got[[3, 4]].isfinite().all())


# ---- chunk bookkeeping through Engine.score -------------------------------------------------------------------------------
def _dims(case):
    if case == "1b-16x1024":
        d, B, T = dims_1b(max_batch=16, max_len=1100), 16, 1024             # four chunks of 256 rows
    elif case == "1b-3x2800":
        d, B, T = dims_1b(max_batch=16, max_len=3200), 3, 2800              # chunks of 1365, the last one ragged
    else:
        d, B, T = dims_8b(max_batch=2, max_len=4480), 2, 4400               # chunks of 2048; the window is crossed
    d.n_layer = 2
    return d, B, T


@pytest.mark.parametrize("case", ["1b-16x1024", "1b-3x2800", "8b-2x4400"])
def test_score_ragged_calls_match_one_call(case):
    """One Engine.score call against the same tokens over ragged calls split at every chunk edge and edge +- 1 (so one-token
    calls sit on both sides of every edge), behind a 40-row embedding prefix: log-probs within 1e-5, and the decode step
    after them bitwise equal (the KV rows the score path appended, at their positions)."""
    d, B, T = _dims(case)
    sd = synthetic_state_dict(d, seed=21, device=DEV)
    eng = Engine(d, 0)
    eng.load_state_dict(sd)
    del sd
    g = torch.Generator().manual_seed(T + B)
    emb = (torch.randn(B, 40, d.hidden, generator=g) * 0.5).to(BF).to(DEV)
    ids = torch.randint(0, d.vocab, (B, T + 1), generator=g).to(DEV)
    C = max(1, 4096 // B)
    eng.prefill_embeds(emb)
    whole = eng.score(ids[:, :T].contiguous())
    after_whole = eng.decode_step(ids[:, T].contiguous())
    cuts = sorted({c for e in range(C, T, C) for c in (e - 1, e, e + 1) if 0 < c < T})
    eng.prefill_embeds(emb)
    parts = [eng.score(ids[:, a:b].contiguous()) for a, b in zip([0] + cuts, cuts + [T])]
    after_ragged = eng.decode_step(ids[:, T].contiguous())
    eng.close()
    assert bool(whole.isfinite().all())
    _calib("ragged calls", (torch.cat(parts, 1) - whole).abs().max().item() / 1e-5)
    assert torch.equal(after_whole, after_ragged), "the KV rows appended by ragged calls differ from one call's"

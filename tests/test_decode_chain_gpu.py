"""The decode step as the engine chains it (sv_op_decode_chain: the host code of sv_decode_step over caller-owned weights,
caches and buffers), at the full 1B and 8B widths with 2 layers.

Stage by stage, every layer: each stage's output is checked against fp64 computed from the chain's OWN previous-stage
output, under the single-launch tests' rules (test_decode_ops_gpu: ring GEMV, decode attention; test_prefill_ops_gpu:
rowgroup linear, LayerNorm), and replayed alone through the single-launch op on the same inputs, which must give the same
bits.  The K/V append changes the caches at the appended slot only, with the qkv row's bits; slots no row may read hold a
finite poison.

Bitwise invariants: the chain with PDL = without PDL = its CUDA-graph replay (and the PDL capture must be accepted on an
sm_90 part); one buffer per activation (the engine's aliasing, residual stream in place) = a slot per layer; slab-tiled =
row-major weights (FUSED); the first layer alone = the first layer of two; an Engine's decode_step logits = the chain's
for the same weights, tokens and prefilled history (1B default and SV_PDL=0, 8B).

Composed error: the whole 2-layer step against an fp64 forward from the same inputs (not stage-fed), relative to the
rms of the fp64 logits (~49 at 1B, ~73 at 8B with these weights).  Measured on an H100 SXM 80 GB (700 W): max 0.066 / mean
0.0038 (1B, FUSED and PER_OP alike), max 0.087 / mean 0.0038 (8B PER_OP); bounded by COMPOSED_MAX = 0.15 and
COMPOSED_MEAN = 0.008, and printed as `CALIB` lines.
"""
import dataclasses
import math
import os

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200 import engine as E
from starvector_b200.config import dims_1b, dims_8b
from starvector_b200.weights import synthetic_state_dict
from test_decode_ops_gpu import ATTN_C, ATTN_ULPS, _key_lo, _ncta_for, _nsplit_for, _ring_check, _ring_ref, _ulp
import test_prefill_ops_gpu as PF

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 128
BF = torch.bfloat16
FUSED, PER_OP = _lib.SV_CHAIN_FUSED, _lib.SV_CHAIN_PER_OP
GELU = _lib.SV_ACT_GELU_TANH
ROWGROUP = _lib.SV_LINEAR_ROWGROUP
COMPOSED_MAX, COMPOSED_MEAN = 0.15, 0.008   # |logit - fp64|: max and mean, over rms(fp64 logits)
POISON_K, POISON_V = 30.0, 500.0

SHAPES = {
    "1b": dict(H=2048, nh=16, nkv=1, I=8192, V=49156, npos=8192, tcap=8224, window=0, rope=False),
    "8b": dict(H=4608, nh=36, nkv=4, I=18432, V=49157, npos=16384, tcap=4128, window=4096, rope=True),
}
_WORST = {}


def _calib(family, ratio):
    _WORST[family] = max(_WORST.get(family, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _print_calib():
    yield
    for family, ratio in sorted(_WORST.items()):
        print(f"CALIB {family}: worst error / tolerance = {ratio:.3f}")


# ---- a 2-layer model at the full widths, drawn on the GPU --------------------------------------------------------------
class Model:
    def __init__(self, shape, seed=0, n_layer=2, wpe=True):
        s = SHAPES[shape]
        self.shape, self.s = shape, s
        H, I, nh, nkv, V = s["H"], s["I"], s["nh"], s["nkv"], s["V"]
        g = torch.Generator(device=DEV).manual_seed(seed)
        rn = lambda *sh, scale=1.0, mean=0.0: (torch.randn(*sh, generator=g, device=DEV) * scale + mean).to(BF)
        qkv = (nh + 2 * nkv) * D
        self.layers = []
        for _ in range(n_layer):
            self.layers.append(dict(
                ln1_w=rn(H, scale=0.3, mean=1.0), ln1_b=rn(H, scale=0.2), attn_w=rn(qkv, H, scale=1 / math.sqrt(H)),
                attn_b=rn(qkv, scale=0.1), proj_w=rn(H, H, scale=1 / math.sqrt(H)), proj_b=rn(H, scale=0.1),
                ln2_w=rn(H, scale=0.3, mean=1.0), ln2_b=rn(H, scale=0.2), fc_w=rn(I, H, scale=1 / math.sqrt(H)),
                fc_b=rn(I, scale=0.1), fc2_w=rn(H, I, scale=1 / math.sqrt(I)), fc2_b=rn(H, scale=0.1)))
        self.wte = rn(V, H)
        self.wpe = rn(s["npos"], H, scale=0.3) if (wpe and not s["rope"]) else None
        self.lnf = (rn(H, scale=0.3, mean=1.0), rn(H, scale=0.2))
        self.lm_head = self.wte
        self.rope = _rope_tables(s["npos"]) if s["rope"] else None


def _rope_tables(npos, theta=1.0e6):
    """The tables Engine._load_rope_tables gives the engine (fp32 outer product, cast to bf16)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
    freqs = torch.outer(torch.arange(npos, dtype=torch.float32), inv_freq)
    return freqs.cos().to(BF).to(DEV), freqs.sin().to(BF).to(DEV)


def _caches(m, B, pos, seed):
    """kcache / vtcache [n_layer, B, n_kv, tcap, D] with N(0, 1) history in the slots row b reads (its window below pos[b]),
    finite poison everywhere else (the appended slot pos[b] included: the chain overwrites it)."""
    s = m.s
    g = torch.Generator(device=DEV).manual_seed(seed)
    n = len(m.layers)
    kc = torch.randn(n, B, s["nkv"], s["tcap"], D, generator=g, device=DEV).to(BF)
    vc = torch.randn(n, B, s["nkv"], D, s["tcap"], generator=g, device=DEV).to(BF)
    for b, p in enumerate(pos):
        lo = _key_lo(p + 1, s["window"])
        for sl in (slice(0, lo), slice(p, s["tcap"])):
            kc[:, b, :, sl] = POISON_K
            vc[:, b, :, :, sl] = POISON_V
    return kc, vc


def _run(m, mode, kc, vc, pos, ids, n_layer=None, tail=True, **kw):
    layers = m.layers[:n_layer] if n_layer else m.layers
    s = m.s
    return E.op_decode_chain(mode, layers, kc[:len(layers)], vc[:len(layers)], pos, s["nh"], s["nkv"], s["npos"], ids=ids,
                             wte=m.wte, wpe=m.wpe, lnf=m.lnf if tail else None, lm_head=m.lm_head if tail else None,
                             rope=m.rope, window=s["window"], **kw)


def _ids(B, V, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, V, (B,), generator=g, device=DEV, dtype=torch.int32)


# ---- stage-fed fp64 checks and single-launch replays ---------------------------------------------------------------------
def _lin_check(y, x, w, b, r, act, family):
    """check_linear's random-input rule (test_prefill_ops_gpu) on the chain's own input x."""
    xd, wd = x.double(), w.double()
    ref, pre = PF._chain(xd @ wd.T, b, r, act)
    tol = _ulp(ref) + 2.0 ** -18 * (xd.abs() @ wd.abs().T) * PF.SLOPE[act]
    if act or r is not None:
        tol = tol + _ulp(pre) * PF.SLOPE[act]
    err = (y.double() - ref).abs()
    ratio = (err / tol).max().item()
    _calib(family, ratio)
    assert ratio <= 1.0, f"{family}: worst err/tol {ratio:.2f}"
    eq = (y.double() == ref).double().mean().item()
    assert eq >= (0.99 if x.shape[1] <= 8192 else 0.98), f"{family}: only {100 * eq:.2f} % bit-equal"


def _ln_check(y, x, ln, family):
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    ref = ((xd - mu) / torch.sqrt((xd - mu).pow(2).mean(-1, keepdim=True) + 1e-5) * ln[0].double() + ln[1].double())
    PF._check_ln(family, y.double(), ref, PF._ln_tol(xd, -1, 1e-5, ln[0], ln[1], ref), 0.995)
    _calib(family, PF._WORST[family])


def _attn_check(out, qkv, kc, vc, pos, s, family):
    """fp64 decode attention of the chain's qkv rows over the chain's caches (after the append), keys [lo, pos]."""
    nh, nkv = s["nh"], s["nkv"]
    grp = nh // nkv
    B = qkv.shape[0]
    ref = torch.empty(B, nh, D, dtype=torch.float64, device=DEV)
    for b, p in enumerate(pos):
        lo = _key_lo(p + 1, s["window"])
        q = qkv[b, :nh * D].view(nh, D).double()
        for h in range(nkv):
            hs = slice(h * grp, (h + 1) * grp)
            w = torch.softmax(q[hs] @ kc[b, h, lo:p + 1].double().T / math.sqrt(D), dim=-1)
            ref[b, hs] = w @ vc[b, h, :, lo:p + 1].double().T
    tol = ATTN_ULPS * _ulp(ref) + ATTN_C * ref.pow(2).mean(-1, keepdim=True).sqrt()
    o = out.view(B, nh, D).double()
    ratio = ((o - ref).abs() / tol).max().item()
    _calib(family, ratio)
    assert bool(torch.isfinite(o).all()) and ratio <= 1.0, f"{family}: worst err/tol {ratio:.2f}"


def _check_append(kc0, vc0, kc1, vc1, qkv, pos, s, l):
    """The chain's append: slot pos[b] of row b holds qkv row b's K / V bits; every other cache byte is unchanged."""
    nh, nkv = s["nh"], s["nkv"]
    kexp, vexp = kc0.clone(), vc0.clone()
    for b, p in enumerate(pos):
        kexp[l, b, :, p] = qkv[b, nh * D:(nh + nkv) * D].view(nkv, D)
        vexp[l, b, :, :, p] = qkv[b, (nh + nkv) * D:].view(nkv, D)
    assert torch.equal(kc1[l], kexp[l]) and torch.equal(vc1[l], vexp[l]), f"layer {l}: KV append"


def _amax_equal(a, b, B):
    """The lm_head argmax partials of rows < B (the columns of the other rows of a row group are not written)."""
    return all(torch.equal(u[:, :B], v[:, :B]) for u, v in zip(a, b))


def _check_embedding(m, x0, ids, pos):
    rows = m.wte[ids.long()].float()
    if m.wpe is not None:
        rows = rows + m.wpe[torch.tensor(pos, device=DEV).clamp(max=m.s["npos"] - 1)].float()
    assert torch.equal(x0, rows.to(BF)), "embedding"


def _stages(m, mode, pos, per_row, seed):
    """One keep-every-slot chain run, every stage checked against fp64 on its own inputs and replayed alone."""
    s = m.s
    B = len(pos)
    ids = _ids(B, s["V"], seed)
    kc0, vc0 = _caches(m, B, pos, seed)
    kc, vc = kc0.clone(), vc0.clone()
    r = _run(m, mode, kc, vc, pos, ids, per_row=per_row, keep=True, pdl=True)
    x, ln, qkv, attn, h = r["x"], r["ln"], r["qkv"], r["attn"], r["h"]
    tag = f"{m.shape} {'fused' if mode == FUSED else 'per-op'}"
    _check_embedding(m, x[0], ids, pos)
    parts = r["parts_used"]
    assert parts == (_ncta_for if mode == FUSED else _nsplit_for)(max(pos) + 1)
    impl = _lib.SV_ATTN_DECODE_CLUSTER if mode == FUSED else _lib.SV_ATTN_DECODE_SPLIT
    for l, L in enumerate(m.layers):
        ln1, ln2 = (L["ln1_w"], L["ln1_b"]), (L["ln2_w"], L["ln2_b"])
        x0, x1, x2 = x[2 * l], x[2 * l + 1], x[2 * l + 2]
        # LayerNorm + c_attn (+ RoPE) + the append
        if mode == FUSED:
            k1, v1 = kc0[l].clone(), vc0[l].clone()
            y = E.op_gemv_ring(x0, L["attn_w"], L["attn_b"], None, ln1, epi=1, kcache=k1, vtcache=v1, n_head=s["nh"],
                               n_kv=s["nkv"], pos=pos, per_row=per_row)
            assert torch.equal(y, qkv[l]) and torch.equal(k1, kc[l]) and torch.equal(v1, vc[l]), f"layer {l}: c_attn replay"
            ref, floor, _ = _ring_ref(x0, L["attn_w"], L["attn_b"], None, ln1)
            _ring_check(qkv[l], ref, floor, f"chain {tag} c_attn layer {l} B={B}")
        else:
            assert torch.equal(E.op_layernorm(x0, *ln1), ln[2 * l]), f"layer {l}: ln_1 replay"
            _ln_check(ln[2 * l], x0, ln1, f"chain {tag} ln_1")
            y = E.op_linear(ln[2 * l], L["attn_w"], L["attn_b"], None, 0, ROWGROUP)
            _lin_check(y, ln[2 * l], L["attn_w"], L["attn_b"], None, 0, f"chain {tag} c_attn")
            if m.rope:
                E.op_rope(y, m.rope[0], m.rope[1], s["nh"], s["nkv"], pos=pos, per_row=per_row)
            assert torch.equal(y, qkv[l]), f"layer {l}: c_attn (+ RoPE) replay"
        _check_append(kc0, vc0, kc, vc, qkv[l], pos, s, l)
        # attention over the caches as the chain left them
        one = E.op_attention_decode(qkv[l], kc[l], vc[l], [p + 1 for p in pos], s["nh"], s["nkv"], parts, s["window"], impl,
                                    per_row)
        assert torch.equal(one, attn[l]), f"layer {l}: attention replay"
        _attn_check(attn[l], qkv[l], kc[l], vc[l], pos, s, f"chain {tag} attention")
        # c_proj + residual, LayerNorm + c_fc + GELU, c_fc2 + residual
        if mode == FUSED:
            assert torch.equal(E.op_gemv_ring(attn[l], L["proj_w"], L["proj_b"], x0), x1), f"layer {l}: c_proj replay"
            ref, floor, _ = _ring_ref(attn[l], L["proj_w"], L["proj_b"], x0)
            _ring_check(x1, ref, floor, f"chain {tag} c_proj layer {l} B={B}")
            assert torch.equal(E.op_gemv_ring(x1, L["fc_w"], L["fc_b"], None, ln2, GELU), h[l]), f"layer {l}: c_fc replay"
            ref, floor, _ = _ring_ref(x1, L["fc_w"], L["fc_b"], None, ln2, GELU)
            _ring_check(h[l], ref, floor, f"chain {tag} c_fc layer {l} B={B}")
            assert torch.equal(E.op_gemv_ring(h[l], L["fc2_w"], L["fc2_b"], x1), x2), f"layer {l}: c_fc2 replay"
            ref, floor, _ = _ring_ref(h[l], L["fc2_w"], L["fc2_b"], x1)
            _ring_check(x2, ref, floor, f"chain {tag} c_fc2 layer {l} B={B}")
        else:
            assert torch.equal(E.op_linear(attn[l], L["proj_w"], L["proj_b"], x0, 0, ROWGROUP), x1), f"layer {l}: c_proj replay"
            _lin_check(x1, attn[l], L["proj_w"], L["proj_b"], x0, 0, f"chain {tag} c_proj")
            assert torch.equal(E.op_layernorm(x1, *ln2), ln[2 * l + 1]), f"layer {l}: ln_2 replay"
            _ln_check(ln[2 * l + 1], x1, ln2, f"chain {tag} ln_2")
            assert torch.equal(E.op_linear(ln[2 * l + 1], L["fc_w"], L["fc_b"], None, GELU, ROWGROUP), h[l]), f"layer {l}: c_fc"
            _lin_check(h[l], ln[2 * l + 1], L["fc_w"], L["fc_b"], None, GELU, f"chain {tag} c_fc")
            assert torch.equal(E.op_linear(h[l], L["fc2_w"], L["fc2_b"], x1, 0, ROWGROUP), x2), f"layer {l}: c_fc2 replay"
            _lin_check(x2, h[l], L["fc2_w"], L["fc2_b"], x1, 0, f"chain {tag} c_fc2")
    xn = x[2 * len(m.layers)]
    if mode == FUSED:
        y, amax = E.op_gemv_ring(xn, m.lm_head, None, None, m.lnf, epi=2)
        assert torch.equal(y, r["logits"]) and _amax_equal(amax, r["amax"], B), "lm_head replay"
        ref, floor, _ = _ring_ref(xn, m.lm_head, None, None, m.lnf)
        _ring_check(r["logits"], ref, floor, f"chain {tag} lm_head B={B}")
    else:
        lnf = ln[2 * len(m.layers)]
        assert torch.equal(E.op_layernorm(xn, *m.lnf), lnf), "ln_f replay"
        _ln_check(lnf, xn, m.lnf, f"chain {tag} ln_f")
        assert torch.equal(E.op_linear(lnf, m.lm_head, None, None, 0, ROWGROUP), r["logits"]), "lm_head replay"
        _lin_check(r["logits"], lnf, m.lm_head, None, None, 0, f"chain {tag} lm_head")
    return ids, kc0, vc0, r, kc, vc


def _invariants(m, mode, pos, per_row, ids, kc0, vc0, keep_run, kc_keep, vc_keep):
    """PDL = plain = graph replay; stride 0 = a slot per layer; tiled = row-major (FUSED); one layer = the first of two."""
    n = len(m.layers)
    outs = []
    for kw in (dict(pdl=True), dict(pdl=False), dict(pdl=True, graph=True)) + ((dict(pdl=True, tiled=True),) if mode == FUSED else ()):
        kc, vc = kc0.clone(), vc0.clone()
        r = _run(m, mode, kc, vc, pos, ids, per_row=per_row, **kw)
        if mode == FUSED:
            assert r["pdl_used"] == kw["pdl"], f"{kw}: the chain ran with pdl_used={r['pdl_used']} (a refused PDL capture?)"
        assert torch.equal(r["logits"], keep_run["logits"]), f"{kw}: logits differ from the per-layer-slot run"
        assert torch.equal(r["x"][0], keep_run["x"][2 * n]), f"{kw}: final residual stream differs"
        assert torch.equal(kc, kc_keep) and torch.equal(vc, vc_keep), f"{kw}: caches differ"
        if mode == FUSED:
            assert _amax_equal(r["amax"], keep_run["amax"], len(pos)), f"{kw}: argmax partials differ"
        outs.append(r)
    kc, vc = kc0.clone(), vc0.clone()
    one = _run(m, mode, kc, vc, pos, ids, n_layer=1, tail=False, per_row=per_row, keep=True)
    assert torch.equal(one["x"], keep_run["x"][:3]), "the first layer alone differs from the first of two"


# ---- 1B FUSED: every cluster size the engine picks, 259 + a few, tcap - 1; rows 1..16 -------------------------------------
FUSED_1B = [(1, 0), (2, 255), (3, 256), (8, 511), (9, 512), (16, 767), (1, 768), (2, 1024), (3, 1280), (8, 1536),
            (9, 1792), (16, 1793), (1, 261), (16, 262), (8, 8222)]


@pytest.fixture(scope="module")
def m1b():
    return Model("1b", seed=1)


@pytest.mark.parametrize("B,p", FUSED_1B, ids=[f"B{b}-pos{p}" for b, p in FUSED_1B])
def test_chain_1b_fused(m1b, B, p):
    pos = [p] * B
    ids, kc0, vc0, r, kc, vc = _stages(m1b, FUSED, pos, False, seed=B * 10000 + p)
    _invariants(m1b, FUSED, pos, False, ids, kc0, vc0, r, kc, vc)


# ---- per-op chains: the GenState append at 31/32/33 and tcap - 1, the embedding at n_positions - 1 and past it -----------
PER_OP_1B = [(1, 31), (8, 32), (1, 33), (8, 8191), (1, 8192), (8, 8223)]


@pytest.mark.parametrize("B,p", PER_OP_1B, ids=[f"B{b}-pos{p}" for b, p in PER_OP_1B])
def test_chain_1b_per_op(m1b, B, p):
    pos = [p] * B
    ids, kc0, vc0, r, kc, vc = _stages(m1b, PER_OP, pos, False, seed=B * 10000 + p)
    _invariants(m1b, PER_OP, pos, False, ids, kc0, vc0, r, kc, vc)


def test_chain_1b_per_op_without_wpe():
    m = Model("1b", seed=2, wpe=False)
    pos = [40, 40]
    ids, kc0, vc0, r, kc, vc = _stages(m, PER_OP, pos, False, seed=7)
    _invariants(m, PER_OP, pos, False, ids, kc0, vc0, r, kc, vc)


@pytest.fixture(scope="module")
def m8b():
    return Model("8b", seed=3)


PER_OP_8B = [(1, 577), (4, 4094), (9, 4095), (16, 4096)]


@pytest.mark.parametrize("B,p", PER_OP_8B, ids=[f"B{b}-pos{p}" for b, p in PER_OP_8B])
def test_chain_8b_per_op(m8b, B, p):
    pos = [p] * B
    ids, kc0, vc0, r, kc, vc = _stages(m8b, PER_OP, pos, False, seed=B * 10000 + p)
    _invariants(m8b, PER_OP, pos, False, ids, kc0, vc0, r, kc, vc)


# ---- sessions: ragged per-row positions (RowState) -----------------------------------------------------------------------
SESSIONS = [("1b", FUSED, [0, 31, 32, 33, 256, 257, 1793, 8222, 5]), ("1b", PER_OP, [31, 32, 33, 0, 8191, 8192, 100, 8223]),
            ("8b", PER_OP, [0, 4095, 4096, 4097])]


@pytest.mark.parametrize("shape,mode,pos", SESSIONS, ids=["1b-fused", "1b-per-op", "8b-per-op"])
def test_chain_session_rows(m1b, m8b, shape, mode, pos):
    m = m1b if shape == "1b" else m8b
    ids, kc0, vc0, r, kc, vc = _stages(m, mode, pos, True, seed=len(pos))
    _invariants(m, mode, pos, True, ids, kc0, vc0, r, kc, vc)


# ---- rowgroup GEMVs at the 8B decoder shapes, decode row counts ---------------------------------------------------------
@pytest.mark.parametrize("M", [1, 2, 4, 8, 9, 16])
@pytest.mark.parametrize("name,N,K,act,res", [("qkv", 5632, 4608, 0, None), ("o_proj", 4608, 4608, 0, "inplace"),
                                               ("c_fc", 18432, 4608, GELU, None), ("c_proj", 4608, 18432, 0, "inplace")],
                         ids=["qkv", "o_proj", "c_fc", "c_proj"])
def test_rowgroup_8b_decoder_shapes(name, N, K, act, res, M):
    family = f"rowgroup 8b {name}"
    PF.check_linear(ROWGROUP, M, N, K, True, act, res, seed=N + K + M, family=family)
    _calib(family, PF._WORST[family])


# ---- composed error: the whole 2-layer step against fp64 ----------------------------------------------------------------
def _fp64_step(m, x, kc, vc, pos):
    """fp64 forward of one step from the embedding x [B, H] over the history in kc / vc (slots < pos[b])."""
    s = m.s
    nh, nkv = s["nh"], s["nkv"]
    grp = nh // nkv
    xd = x.double()

    def ln(v, p):
        mu = v.mean(-1, keepdim=True)
        return (v - mu) / torch.sqrt((v - mu).pow(2).mean(-1, keepdim=True) + 1e-5) * p[0].double() + p[1].double()

    def rope(t, p):        # t [heads, D] at position p
        c = torch.cat([m.rope[0][p], m.rope[0][p]]).double()
        sn = torch.cat([m.rope[1][p], m.rope[1][p]]).double()
        return t * c + torch.cat([-t[:, D // 2:], t[:, :D // 2]], -1) * sn

    for l, L in enumerate(m.layers):
        qkv = ln(xd, (L["ln1_w"], L["ln1_b"])) @ L["attn_w"].double().T + L["attn_b"].double()
        att = torch.empty(len(pos), nh * D, dtype=torch.float64, device=DEV)
        for b, p in enumerate(pos):
            q = qkv[b, :nh * D].view(nh, D)
            k = qkv[b, nh * D:(nh + nkv) * D].view(nkv, D)
            v = qkv[b, (nh + nkv) * D:].view(nkv, D)
            if m.rope:
                q, k = rope(q, min(p, s["npos"] - 1)), rope(k, min(p, s["npos"] - 1))
            lo = _key_lo(p + 1, s["window"])
            for h in range(nkv):
                K = torch.cat([kc[l, b, h, lo:p].double(), k[h:h + 1]])
                V = torch.cat([vc[l, b, h, :, lo:p].double().T, v[h:h + 1]])
                w = torch.softmax(q[h * grp:(h + 1) * grp] @ K.T / math.sqrt(D), dim=-1)
                att[b, h * grp * D:(h + 1) * grp * D] = (w @ V).reshape(-1)
        xd = xd + att @ L["proj_w"].double().T + L["proj_b"].double()
        hh = torch.nn.functional.gelu(ln(xd, (L["ln2_w"], L["ln2_b"])) @ L["fc_w"].double().T + L["fc_b"].double(),
                                      approximate="tanh")
        xd = xd + hh @ L["fc2_w"].double().T + L["fc2_b"].double()
    return ln(xd, m.lnf) @ m.lm_head.double().T


@pytest.mark.parametrize("shape,mode,B,p", [("1b", FUSED, 8, 700), ("1b", PER_OP, 8, 700), ("8b", PER_OP, 4, 4096)],
                         ids=["1b-fused", "1b-per-op", "8b-per-op"])
def test_chain_composed_error(m1b, m8b, shape, mode, B, p):
    m = m1b if shape == "1b" else m8b
    pos = [p] * B
    ids = _ids(B, m.s["V"], seed=99)
    kc, vc = _caches(m, B, pos, seed=99)
    hist_k, hist_v = kc.clone(), vc.clone()
    r = _run(m, mode, kc, vc, pos, ids, keep=True)
    ref = _fp64_step(m, r["x"][0], hist_k, hist_v, pos)
    rms = ref.pow(2).mean().sqrt().item()
    err = (r["logits"].double() - ref).abs() / rms
    e_max, e_mean = err.max().item(), err.mean().item()
    print(f"CALIB composed {shape} mode={mode} B={B} pos={p}: max |err| / rms {e_max:.4f}, mean {e_mean:.5f} (rms {rms:.2f})")
    _calib(f"composed {shape} mode={mode} max", e_max / COMPOSED_MAX)
    _calib(f"composed {shape} mode={mode} mean", e_mean / COMPOSED_MEAN)
    assert e_max <= COMPOSED_MAX and e_mean <= COMPOSED_MEAN, (e_max, e_mean)


# ---- the engine's decode_step is the chain ------------------------------------------------------------------------------
def _engine_identity(dims, shape, B, T, env=None):
    d = dataclasses.replace(dims, n_layer=2, max_batch=B)
    sd = synthetic_state_dict(d, seed=5, init="randomized", device=DEV)
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        eng = E.Engine(d)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    eng.load_state_dict(sd)
    s = SHAPES[shape]
    g = torch.Generator(device=DEV).manual_seed(T)
    emb = torch.randn(B, T, d.hidden, generator=g, device=DEV).to(BF)
    ids = _ids(B, d.vocab, seed=T)
    eng.prefill_embeds(emb)
    logits = eng.decode_step(ids)
    describe = eng.describe() if hasattr(eng, "describe") else ""
    eng.close()
    # the same weights, and the same history through the prefill kernels run_prefill issues
    if shape == "1b":
        pre = "model.svg_transformer.transformer.transformer."
        names = dict(ln1_w="ln_1.weight", ln1_b="ln_1.bias", attn_w="attn.c_attn.weight", attn_b="attn.c_attn.bias",
                     proj_w="attn.c_proj.weight", proj_b="attn.c_proj.bias", ln2_w="ln_2.weight", ln2_b="ln_2.bias",
                     fc_w="mlp.c_fc.weight", fc_b="mlp.c_fc.bias", fc2_w="mlp.c_proj.weight", fc2_b="mlp.c_proj.bias")
        layers = [{k: sd[f"{pre}h.{i}.{v}"].to(DEV) for k, v in names.items()} for i in range(2)]
        wte, wpe, lnf = sd[pre + "wte.weight"].to(DEV), sd[pre + "wpe.weight"].to(DEV), (sd[pre + "ln_f.weight"], sd[pre + "ln_f.bias"])
    else:
        pre = "model.svg_transformer.transformer.model."
        layers = []
        for i in range(2):
            p = f"{pre}layers.{i}."
            a = lambda n: sd[p + n].to(DEV)
            layers.append(dict(
                ln1_w=a("input_layernorm.weight"), ln1_b=a("input_layernorm.bias"),
                attn_w=torch.cat([a("self_attn.q_proj.weight"), a("self_attn.k_proj.weight"), a("self_attn.v_proj.weight")]),
                attn_b=torch.cat([a("self_attn.q_proj.bias"), a("self_attn.k_proj.bias"), a("self_attn.v_proj.bias")]),
                proj_w=a("self_attn.o_proj.weight"), proj_b=a("self_attn.o_proj.bias"),
                ln2_w=a("post_attention_layernorm.weight"), ln2_b=a("post_attention_layernorm.bias"),
                fc_w=a("mlp.c_fc.weight"), fc_b=a("mlp.c_fc.bias"), fc2_w=a("mlp.c_proj.weight"), fc2_b=a("mlp.c_proj.bias")))
        wte, wpe, lnf = sd[pre + "embed_tokens.weight"].to(DEV), None, (sd[pre + "norm.weight"], sd[pre + "norm.bias"])
    lnf = (lnf[0].to(DEV), lnf[1].to(DEV))
    rope = _rope_tables(d.n_positions, d.rope_theta) if shape == "8b" else None
    tcap = (min(d.max_len, d.n_positions) + 1 + 31) // 32 * 32
    kc = torch.zeros(2, B, d.n_kv_head, tcap, D, dtype=BF, device=DEV)
    vc = torch.zeros(2, B, d.n_kv_head, D, tcap, dtype=BF, device=DEV)
    x = E.op_embed_prefix(emb.view(B * T, -1), None, wte, wpe, B, T, 0)
    auto = _lib.SV_LINEAR_AUTO
    for l, L in enumerate(layers):
        qkv = E.op_linear(E.op_layernorm(x, L["ln1_w"], L["ln1_b"], d.ln_eps), L["attn_w"], L["attn_b"], None, 0, auto)
        if rope is not None:
            E.op_rope(qkv, rope[0], rope[1], d.n_head, d.n_kv_head, seq=T)
        att = E.op_attention_prefill(qkv, kc[l], vc[l], T, d.n_head, d.n_kv_head, d.sliding_window if shape == "8b" else 0)
        x = PF._run_linear(auto, att, L["proj_w"], L["proj_b"], x, 0, True)
        hh = E.op_linear(E.op_layernorm(x, L["ln2_w"], L["ln2_b"], d.ln_eps), L["fc_w"], L["fc_b"], None, GELU, auto)
        x = PF._run_linear(auto, hh, L["fc2_w"], L["fc2_b"], x, 0, True)
    mode = FUSED if shape == "1b" else PER_OP
    r = E.op_decode_chain(mode, layers, kc, vc, [T] * B, d.n_head, d.n_kv_head, d.n_positions, ids=ids, wte=wte, wpe=wpe,
                          lnf=lnf, lm_head=wte, rope=rope, window=d.sliding_window if shape == "8b" else 0, ln_eps=d.ln_eps,
                          pdl=(env or {}).get("SV_PDL") != "0")
    assert torch.equal(logits, r["logits"].float()), \
        f"engine decode_step differs from the chain: max |diff| {(logits - r['logits'].float()).abs().max().item()}"
    return describe


def test_engine_decode_step_is_the_chain_1b():
    desc = _engine_identity(dims_1b(max_len=2048), "1b", 3, 300)
    assert "decode=ring-gemv-graph" in desc and "pdl=1" in desc, desc
    desc = _engine_identity(dims_1b(max_len=2048), "1b", 3, 300, env={"SV_PDL": "0"})
    assert "pdl=0" in desc, desc


def test_engine_decode_step_is_the_chain_8b():
    desc = _engine_identity(dims_8b(max_len=4608), "8b", 2, 600)
    assert "decode=legacy-kernels" in desc, desc

"""The dataflow decode kernel (decode_flow_kernel, SV_FLOW=1) one launch at a time through sv_op_decode_flow, at the 1B
widths (hidden 2048, c_fc 8192, 16 heads over 1 KV head, vocab 49156 and 49157) and the tiny GQA widths (hidden 512, 4 heads
over 2 KV heads: the only shape where an attention item loops over more than one KV head).

Each phase of the last layer is read back from the exchange buffers (the flagged words, decoded by test_flow_layout) and
checked against fp64 computed from the kernel's OWN previous-phase output, under the single-launch tests' rules
(test_decode_ops_gpu: ring GEMV, decode attention): c_attn(LN1(x_in)), attention over the poisoned cache plus the new k/v,
x_in + c_proj, gelu_tanh(c_fc(LN2)), + c_fc2, then the logits and the lm_head's argmax partials.  Every word carries the tag
of the last phase that wrote it, and the cache changes at slot cur_len only, with the qkv row's K/V bits.

The attention at its item boundaries (256 keys per item; longer rows go through the fp32 partial merge): B in {1, 3, 5, 8},
contexts from 1 to 8192 keys; every cached key is solved for its logit in each of the kernel's own query heads, so that
the probe keys at every item's first and last key together, and the new token, each hold >= 20 % of the softmax mass in
every (row, head).

Bitwise: one launch of N tokens = N one-token launches = launches split anywhere (out_ids, seen, state, caches, logits);
a launch whose phase tags wrap past 0x7fff = the same launch from epoch 0; the plain variant = the register-reallocating
one; l2_ahead = 8 = 0.  Greedy selection after every one-token launch = the first maximum of the kernel's own bf16 logits
after the repetition penalty (planted exact ties within a tile, across tiles and in the ragged last tile), and the HF
bookkeeping step by step (test_select_ops_gpu.HFLoop).  An SV_FLOW=1 Engine's decode_step logits and a greedy generate
over three launches (the tags wrap inside the third) = the op's.
"""
import dataclasses
import math
import os

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200 import engine as E
from starvector_b200.config import dims_1b
from starvector_b200.engine import GenerationParams
from starvector_b200.weights import synthetic_state_dict
from test_decode_chain_gpu import _attn_check, _check_append
import test_decode_chain_gpu as CH
from test_decode_ops_gpu import _ring_check, _ring_ref, _ulp
from test_flow_layout import attn_items, decode_amax, decode_partial, decode_rows, plan, tag16, tag32
from test_select_ops_gpu import HFLoop, greedy_reference
import test_prefill_ops_gpu as PF

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 128
BF = torch.bfloat16
GELU = _lib.SV_ACT_GELU_TANH
POISON_K, POISON_V = 30.0, 500.0
TCAP = 8224
SHAPES = {
    "1b": dict(H=2048, nh=16, nkv=1, I=8192, V=49156, npos=8192, window=0),
    "1b_v49157": dict(H=2048, nh=16, nkv=1, I=8192, V=49157, npos=8192, window=0),
    "gqa": dict(H=512, nh=4, nkv=2, I=1024, V=500, npos=8192, window=0),
}
_WORST = {}


def _calib(family, ratio):
    _WORST[family] = max(_WORST.get(family, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _print_calib():
    yield
    for family, ratio in sorted(_WORST.items()):
        print(f"CALIB flow {family}: worst error / tolerance = {ratio:.3f}")


class Model:
    def __init__(self, shape, seed=0, n_layer=2):
        s = SHAPES[shape]
        self.shape, self.s = shape, s
        H, I, nh, nkv, V = s["H"], s["I"], s["nh"], s["nkv"], s["V"]
        g = torch.Generator(device=DEV).manual_seed(seed)
        rn = lambda *sh, scale=1.0, mean=0.0: (torch.randn(*sh, generator=g, device=DEV) * scale + mean).to(BF)
        qkv = (nh + 2 * nkv) * D
        self.layers = [dict(
            ln1_w=rn(H, scale=0.3, mean=1.0), ln1_b=rn(H, scale=0.2), attn_w=rn(qkv, H, scale=1 / math.sqrt(H)),
            attn_b=rn(qkv, scale=0.1), proj_w=rn(H, H, scale=1 / math.sqrt(H)), proj_b=rn(H, scale=0.1),
            ln2_w=rn(H, scale=0.3, mean=1.0), ln2_b=rn(H, scale=0.2), fc_w=rn(I, H, scale=1 / math.sqrt(H)),
            fc_b=rn(I, scale=0.1), fc2_w=rn(H, I, scale=1 / math.sqrt(I)), fc2_b=rn(H, scale=0.1)) for _ in range(n_layer)]
        self.wte = rn(V, H)
        self.wpe = rn(s["npos"], H, scale=0.3)
        self.lnf = (rn(H, scale=0.3, mean=1.0), rn(H, scale=0.2))
        self.lm_head = self.wte


_MODELS = {}


def _model(shape, n_layer=2):
    if (shape, n_layer) not in _MODELS:
        _MODELS[(shape, n_layer)] = Model(shape, seed=3, n_layer=n_layer)
    return _MODELS[(shape, n_layer)]


def _caches(m, B, cur_len, seed, n_layer=None):
    """[n_layer, B, n_kv, TCAP, D] / [.., D, TCAP]: N(0, 1) history below cur_len, finite poison from cur_len on
    (the new token's slot included: the kernel takes the new k/v from its own qkv vector)."""
    s = m.s
    n = n_layer or len(m.layers)
    g = torch.Generator(device=DEV).manual_seed(seed)
    kc = torch.randn(n, B, s["nkv"], TCAP, D, generator=g, device=DEV).to(BF)
    vc = torch.randn(n, B, s["nkv"], D, TCAP, generator=g, device=DEV).to(BF)
    kc[:, :, :, cur_len:] = POISON_K
    vc[:, :, :, :, cur_len:] = POISON_V
    return kc, vc


def _embed(m, ids, pos):
    return (m.wte[ids.long()].float() + m.wpe[min(pos, m.s["npos"] - 1)].float()).to(BF)


def _run(m, kc, vc, x_plain, cur_len, n_layer=None, bufs=None, **kw):
    s = m.s
    layers = m.layers[:n_layer] if n_layer else m.layers
    B = x_plain.shape[0]
    if bufs is None:
        bufs = E.flow_buffers(B, s["H"], s["I"], s["nkv"], s["V"], DEV)
    kw.setdefault("clear", kw.get("first_plain", True))
    r = E.op_decode_flow(layers, kc, vc, s["nh"], s["nkv"], s["npos"], wte=m.wte, wpe=m.wpe, lnf=m.lnf,
                         lm_head=kw.pop("lm_head", m.lm_head), x_plain=x_plain, bufs=bufs, cur_len0=cur_len, **kw)
    r["bufs"] = bufs
    return r


def _attn(out, qkv, kc, vc, pos, s, family):
    """test_decode_chain_gpu._attn_check (fp64 over the cache after the append, ATTN_ULPS / ATTN_C), its ratio recorded here."""
    _attn_check(out, qkv, kc, vc, pos, s, family)
    _calib(family, CH._WORST[family])


def _check_gemv(y, ref, floor, family):
    """test_decode_ops_gpu._ring_check (fp64 with the kernel's rounding points, ulp + fp32-accumulation floor, >= 99 %
    bit-equal), its ratio recorded here.  A LayerNorm-fed phase's reference input is the ring kernel's bf16 LayerNorm
    output (_ring_ref): the flow kernel's own staged LayerNorm is not observable, so it is checked through the GEMV it
    feeds, and against fp64 through the ring LayerNorm's own test (test_gemv_ring_layernorm)."""
    _calib(family, ((y.double() - ref).abs() / (_ulp(ref) + floor)).max().item())
    _ring_check(y, ref, floor, f"flow {family}")


def _words(r, name, B, n, tag, what):
    vals, tags = decode_rows(r["bufs"][name], B, n)
    assert bool((tags == tag).all()), f"{what}: {int((tags != tag).sum())} words without the tag {tag:#x}"
    return vals.to(DEV)


def _phases(m, r, x_in, n_layer, B, cur_len, step0, kc0, vc0, kc, vc, tag):
    """Every phase of layer n_layer - 1 from the buffers against fp64 on the kernel's own previous-phase output."""
    s = m.s
    L = m.layers[n_layer - 1]
    l = n_layer - 1
    gp = step0 * (n_layer + 1) + l
    qkv_cols = (s["nh"] + 2 * s["nkv"]) * D
    qkv = _words(r, "qkv", B, qkv_cols, tag16(gp), f"{tag} qkv")
    att = _words(r, "att", B, s["H"], tag16(gp), f"{tag} att")
    xb = _words(r, "xb", B, s["H"], tag16(gp), f"{tag} xb")
    hb = _words(r, "hb", B, s["I"], tag16(gp), f"{tag} hb")
    xa = _words(r, "xa", B, s["H"], tag16(gp + 1), f"{tag} xa")
    ref, floor, _ = _ring_ref(x_in, L["attn_w"], L["attn_b"], None, (L["ln1_w"], L["ln1_b"]))
    _check_gemv(qkv, ref, floor, f"{m.shape} c_attn(LN1)")
    _check_append(kc0, vc0, kc, vc, qkv, [cur_len] * B, s, l)
    _attn(att, qkv, kc[l], vc[l], [cur_len] * B, s, f"{m.shape} attention")
    ref, floor, _ = _ring_ref(att, L["proj_w"], L["proj_b"], x_in)
    _check_gemv(xb, ref, floor, f"{m.shape} c_proj + residual")
    ref, floor, _ = _ring_ref(xb, L["fc_w"], L["fc_b"], None, (L["ln2_w"], L["ln2_b"]), GELU)
    _check_gemv(hb, ref, floor, f"{m.shape} gelu(c_fc(LN2))")
    ref, floor, _ = _ring_ref(hb, L["fc2_w"], L["fc2_b"], xb)
    _check_gemv(xa, ref, floor, f"{m.shape} c_fc2 + residual")
    lg = r["logits"]
    ref, floor, _ = _ring_ref(xa, m.lm_head, None, None, m.lnf)
    _check_gemv(lg, ref, floor, f"{m.shape} lm_head(LN_f)")
    # the argmax partials: per tile and row, the tile's maximum bf16 logit and its FIRST index
    R, nt = plan(s["V"], r["ncta"])
    tags, vals, idx = decode_amax(r["bufs"]["amax"], nt, B)
    assert bool((tags == tag16(step0 * (n_layer + 1) + n_layer)).all()), f"{tag}: argmax partial tags"
    pad = torch.full((B, nt * R), -math.inf, device=DEV)
    pad[:, :s["V"]] = lg.float()
    tiles = pad.view(B, nt, R)
    mx = tiles.max(-1).values
    first = (tiles == mx[..., None]).int().argmax(-1) + torch.arange(nt, device=DEV) * R
    assert torch.equal(vals.float().to(DEV), mx.T) and torch.equal(idx.to(DEV), first.T), f"{tag}: argmax partials"
    return xa


PHASE_CASES = [("1b", 2, 300), ("1b", 1, 0), ("1b_v49157", 8, 40), ("1b_v49157", 3, 256), ("gqa", 3, 70), ("gqa", 5, 600),
               ("gqa", 1, 31)]


@pytest.mark.parametrize("shape,B,cur_len", PHASE_CASES, ids=str)
def test_flow_phases(shape, B, cur_len):
    """Layer 1 alone, then two layers on the same inputs: layer 2's phases are fed by the 1-layer launch's xa, and the
    2-layer launch's layer 1 (its cache append) is bit-equal to the 1-layer launch's."""
    m = _model(shape)
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + cur_len)
    ids = torch.randint(0, m.s["V"], (B,), generator=g, device=DEV, dtype=torch.int32)
    x0 = _embed(m, ids, cur_len)
    kc0, vc0 = _caches(m, B, cur_len, seed=cur_len + B)
    step0 = 5
    kc1, vc1 = kc0.clone(), vc0.clone()
    r1 = _run(m, kc1, vc1, x0.clone(), cur_len, n_layer=1, step0=step0)
    assert r1["ncta"] == torch.cuda.get_device_properties(0).multi_processor_count
    x1 = _phases(m, r1, x0, 1, B, cur_len, step0, kc0, vc0, kc1, vc1, f"{shape} 1 layer")
    nact, _ = attn_items(cur_len + 1)
    if nact > 1:                                       # the fp32 partials of every item carry the attention's tag
        for b in range(B):
            for h in range(m.s["nkv"]):
                for c in range(nact):
                    _, t = decode_partial(r1["bufs"]["part"], b, h, c, m.s["nkv"])
                    assert bool((t == tag32(step0 * 2)).all()), ("partial tags", b, h, c)
    kc2, vc2 = kc0.clone(), vc0.clone()
    r2 = _run(m, kc2, vc2, x0.clone(), cur_len, step0=step0)
    assert torch.equal(kc2[0], kc1[0]) and torch.equal(vc2[0], vc1[0]), "layer 1 alone differs from layer 1 of two"
    _phases(m, r2, x1, 2, B, cur_len, step0, kc1, vc1, kc2, vc2, f"{shape} 2 layers")


# ---- the attention at its item boundaries ----------------------------------------------------------------------------------
CONTEXTS = [1, 31, 32, 33, 255, 256, 257, 288, 289, 512, 513, 2048, 2049, 8192]


@pytest.mark.parametrize("B", [1, 3, 5, 8])
@pytest.mark.parametrize("nkeys", CONTEXTS)
def test_flow_attention_boundaries(B, nkeys):
    """Keys [0, nkeys - 1) from the cache, key nkeys - 1 the new token.  A first launch gives the queries q_h and the new
    token's key; the cache is then rebuilt around them, every key solved (minimum norm) for a chosen logit in EACH of the
    16 query heads of the KV head: probe keys at the first and last key of every attention item (attn_split) share the
    new token's logit minus log(#probes), the other history keys sit log(2 * #history) below it (+ N(0, 0.1^2) noise),
    poison keys past the new token score 20.  So in every (row, head) the probes together and the new token each hold
    ~40 % of the softmax mass (asserted >= 20 % from the fp64 weights), and a probe's value rows are 4x the others'.
    The second launch has the same queries (layer 1: they do not depend on the cache)."""
    m = _model("1b", 2)
    s = m.s
    nh, H = s["nh"], s["H"]
    cur = nkeys - 1
    g = torch.Generator(device=DEV).manual_seed(nkeys * 10 + B)
    ids = torch.randint(0, s["V"], (B,), generator=g, device=DEV, dtype=torch.int32)
    x0 = _embed(m, ids, cur)
    kc0, vc0 = _caches(m, B, cur, seed=nkeys, n_layer=1)
    r = _run(m, kc0.clone(), vc0.clone(), x0.clone(), cur, n_layer=1)
    qkv1 = decode_rows(r["bufs"]["qkv"], B, (nh + 2 * s["nkv"]) * D)[0]
    q = qkv1[:, :H]
    nact, per = attn_items(nkeys)
    edges = sorted({k for c in range(nact) for k in (c * per * 32, min(nkeys, (c + 1) * per * 32) - 1) if k < cur})
    hist = [k for k in range(cur) if k not in set(edges)]
    for b in range(B):
        Q = q[b].double().view(nh, D).to(DEV)
        s_new = Q @ qkv1[b, H:H + D].double().to(DEV) / math.sqrt(D)        # the new token's logit per head
        P = torch.linalg.pinv(Q)                                                # [D, nh]: Q @ P = I
        solve = lambda t: ((t * math.sqrt(D)) @ P.T).to(BF)                    # keys with logits t [.., nh]
        if hist:
            eps = 0.1 * torch.randn(len(hist), nh, generator=g, device=DEV, dtype=torch.float64)
            kc0[0, b, 0, hist] = solve(s_new - math.log(2 * len(hist)) + eps)
        if edges:
            kc0[0, b, 0, edges] = solve(s_new - math.log(len(edges)))
            vc0[0, b, 0, :, edges] = (4 * vc0[0, b, 0, :, edges].float()).to(BF)
        kc0[0, b, 0, cur + 1:] = solve(torch.full((nh,), 20.0, device=DEV, dtype=torch.float64))
    kc, vc = kc0.clone(), vc0.clone()
    r = _run(m, kc, vc, x0.clone(), cur, n_layer=1)
    qkv = _words(r, "qkv", B, (nh + 2 * s["nkv"]) * D, tag16(0), "qkv")
    att = _words(r, "att", B, H, tag16(0), "att")
    assert torch.equal(qkv.cpu(), qkv1), "the qkv row changed between the two launches"
    _check_append(kc0, vc0, kc, vc, qkv, [cur] * B, s, 0)
    # the softmax mass the probes and the new token hold, in fp64 over the cache as the kernel read it
    w = torch.softmax(qkv[:, :H].double().view(B, nh, D) @ kc[0, :, 0, :cur + 1].double().transpose(1, 2) / math.sqrt(D), -1)
    new_mass = w[:, :, cur].min().item()
    probe_mass = w[:, :, edges].sum(-1).min().item() if edges else 1.0
    _calib("1b attention boundaries: 0.2 / least new-token mass", 0.2 / max(new_mass, 1e-9))
    _calib("1b attention boundaries: 0.2 / least probe mass", 0.2 / max(probe_mass, 1e-9))
    assert new_mass >= 0.2 and probe_mass >= 0.2, (new_mass, probe_mass)
    _attn(att, qkv, kc[0], vc[0], [cur] * B, s, "1b attention boundaries")


# ---- launch segmentation, tag wrap, variants ---------------------------------------------------------------------------------
def _gen_state(B, cur_len, step=0):
    return dict(step=step, cur_len=cur_len, done=0, unfinished=[1] * B)


def _sequence(m, kc0, vc0, x0, cur0, segments, step0=0, stride=64, params=None, seen0=None, **kw):
    """Launches of `segments` tokens one after the other (the first from x_plain with the buffers cleared, the others from
    the xa words the previous selection left) -> every observable."""
    B = x0.shape[0]
    kc, vc, x = kc0.clone(), vc0.clone(), x0.clone()
    st = _gen_state(B, cur0)
    seen = seen0.clone() if seen0 is not None else torch.zeros(B, m.s["V"], dtype=torch.uint8, device=DEV)
    out = torch.full((B, stride), -1, dtype=torch.int32, device=DEV)
    nxt = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    bufs = E.flow_buffers(B, m.s["H"], m.s["I"], m.s["nkv"], m.s["V"], DEV)
    done = 0
    r = None
    for i, n in enumerate(segments):
        r = _run(m, kc, vc, x, cur0 + done, bufs=bufs, nsteps=n, step0=step0 + done, first_plain=i == 0, do_select=True,
                 params=params, state=st, seen=seen, out_ids=out, next_ids=nxt, **kw)
        done += n
    return dict(kc=kc, vc=vc, x=x, state=st, seen=seen, out=out, next=nxt, logits=r["logits"], realloc=r["realloc"])


def _same(a, b, what):
    for k in ("out", "next", "seen", "kc", "vc", "logits", "x"):
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs"
    assert a["state"] == b["state"], (what, a["state"], b["state"])


def test_flow_launch_segmentation_is_bitwise():
    m = _model("1b", 2)
    B, cur0, N = 8, 50, 24
    g = torch.Generator(device=DEV).manual_seed(7)
    ids = torch.randint(0, m.s["V"], (B,), generator=g, device=DEV, dtype=torch.int32)
    x0 = _embed(m, ids, cur0)
    kc0, vc0 = _caches(m, B, cur0, seed=11)
    base = _sequence(m, kc0, vc0, x0, cur0, [N])
    assert base["realloc"] and base["state"]["step"] == N and base["state"]["cur_len"] == cur0 + N
    assert bool((base["out"][:, :N] >= 0).all()) and bool((base["out"][:, N:] == -1).all())
    _same(base, _sequence(m, kc0, vc0, x0, cur0, [1] * N), "N one-token launches")
    _same(base, _sequence(m, kc0, vc0, x0, cur0, [5, 11, 1, 7]), "launches split at 5, 16, 17")
    wrap = 0x8000 // 3 - 10                       # gp = step * 3 + layer crosses 0x7fff at the launch's 11th step
    _same(base, _sequence(m, kc0, vc0, x0, cur0, [N], step0=wrap), "tags wrapping inside the launch")
    _same(base, _sequence(m, kc0, vc0, x0, cur0, [9, 15], step0=wrap), "tags wrapping inside the second launch")
    plain = _sequence(m, kc0, vc0, x0, cur0, [N], realloc=False)
    assert not plain["realloc"]
    _same(base, plain, "the plain variant")
    _same(base, _sequence(m, kc0, vc0, x0, cur0, [N], l2_ahead=8), "l2_ahead = 8")


def test_flow_first_plain_0_needs_the_tagged_input():
    """A relaunch from xa words that do not carry the first step's tag would spin until the watchdog: refused on the host."""
    m = _model("gqa", 2)
    B, cur0 = 2, 10
    x0 = _embed(m, torch.tensor([3, 4], dtype=torch.int32, device=DEV), cur0)
    kc, vc = _caches(m, B, cur0, seed=1)
    bufs = E.flow_buffers(B, m.s["H"], m.s["I"], m.s["nkv"], m.s["V"], DEV)
    _run(m, kc, vc, x0.clone(), cur0, bufs=bufs, step0=0)          # no selection: xa holds the lm_head phase's tag
    with pytest.raises(ValueError, match="does not carry the tag"):
        _run(m, kc, vc, x0.clone(), cur0 + 1, bufs=bufs, step0=1, first_plain=False)


# ---- selection and bookkeeping ----------------------------------------------------------------------------------------------
def _tied_lm_head(m, B, x0, kc0, vc0, cur0):
    """lm_head = wte with exact ties planted at the first step's winners: row 0's winner also at a lower id in another
    tile (which must win), row 1's at its tile neighbour, row 2's moved to the two last ids (the ragged last tile)."""
    r = _run(m, kc0.clone(), vc0.clone(), x0.clone(), cur0)
    win = r["logits"].float().argmax(-1).tolist()
    V = m.s["V"]
    R, _ = plan(V, r["ncta"])
    lm = m.wte.clone()
    lower = (win[0] // R - 3) * R + 2 if win[0] >= 4 * R else win[0] + 2 * R      # (V > 6 R: in range)
    lm[lower] = lm[win[0]]
    nb = win[1] + 1 if (win[1] + 1) % R and win[1] + 1 < V else win[1] - 1
    lm[nb] = lm[win[1]]
    lm[V - 2] = lm[V - 1] = lm[win[2]]
    lm[win[2]] = -lm[win[2]]
    return lm, [min(lower, win[0]), min(nb, win[1]), V - 2], win[:3] + [lower, nb, V - 2, V - 1]


@pytest.mark.parametrize("rp", [1.0, 1.3])
def test_flow_selection_is_the_first_max_of_the_penalised_logits(rp):
    m = _model("1b_v49157", 2)
    B, cur0, N = 4, 30, 12
    g = torch.Generator(device=DEV).manual_seed(int(rp * 10))
    x0 = _embed(m, torch.randint(0, m.s["V"], (B,), generator=g, device=DEV, dtype=torch.int32), cur0)
    kc0, vc0 = _caches(m, B, cur0, seed=3)
    lm, tied, planted = _tied_lm_head(m, B, x0, kc0, vc0, cur0)
    seen0 = (torch.rand(B, m.s["V"], generator=g, device=DEV) < 0.05).to(torch.uint8)
    seen0[:, planted] = 0
    kc, vc, x = kc0.clone(), vc0.clone(), x0.clone()
    st = _gen_state(B, cur0)
    seen = seen0.clone()
    out = torch.full((B, 64), -1, dtype=torch.int32, device=DEV)
    nxt = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    bufs = E.flow_buffers(B, m.s["H"], m.s["I"], m.s["nkv"], m.s["V"], DEV)
    params = GenerationParams(max_new_tokens=1 << 20, repetition_penalty=rp, eos_token_id=None)
    for s in range(N):
        before = seen.clone()
        r = _run(m, kc, vc, x, cur0 + s, bufs=bufs, step0=s, first_plain=s == 0, do_select=True, params=params, state=st,
                 seen=seen, out_ids=out, next_ids=nxt, lm_head=lm)
        want = greedy_reference(r["logits"].cpu(), before.cpu(), rp)
        assert out[:, s].tolist() == want, (s, out[:, s].tolist(), want)
        if s == 0:
            assert want[:3] == tied, (want, tied)
        assert torch.equal(x, (m.wte[out[:, s].long()].float() + m.wpe[cur0 + s + 1].float()).to(BF)), "next embedding"


SCRIPTS = {"eos": dict(eos_row=1, eos_step=3), "row0_stop": dict(stop_row=0, stop_step=4, row0_only=True),
           "row_stop": dict(stop_row=2, stop_step=2, row0_only=False, eos_row=0, eos_step=5)}


@pytest.mark.parametrize("name", list(SCRIPTS))
def test_flow_bookkeeping_follows_the_hf_loop(name):
    """EOS -> pad, per-row stop and row-0 stop, one-token launches checked step by step against HFLoop on the kernel's own
    logits; then the same generation as ONE launch (a row finishes mid-launch while the launch keeps stepping) = those."""
    sc = SCRIPTS[name]
    m = _model("gqa", 2)
    B, cur0, N = 4, 20, 12
    g = torch.Generator(device=DEV).manual_seed(5)
    x0 = _embed(m, torch.randint(0, m.s["V"], (B,), generator=g, device=DEV, dtype=torch.int32), cur0)
    kc0, vc0 = _caches(m, B, cur0, seed=9)
    free = _sequence(m, kc0, vc0, x0, cur0, [N], params=GenerationParams(max_new_tokens=1 << 20, eos_token_id=None))
    toks = free["out"].cpu()
    eos = int(toks[sc["eos_row"], sc["eos_step"]]) if "eos_row" in sc else None
    stop = [int(t) for t in toks[sc["stop_row"], sc["stop_step"] - 1:sc["stop_step"] + 1]] if "stop_row" in sc else []
    params = GenerationParams(max_new_tokens=N + 4, eos_token_id=eos, pad_token_id=m.s["V"] - 1, stop_ids=stop,
                              stop_row0_only=sc.get("row0_only", True))
    kc, vc, x = kc0.clone(), vc0.clone(), x0.clone()
    st = _gen_state(B, cur0)
    seen = torch.zeros(B, m.s["V"], dtype=torch.uint8, device=DEV)
    out = torch.full((B, 64), -1, dtype=torch.int32, device=DEV)
    nxt = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    hf = HFLoop(B, m.s["V"], 64, params, dict(st), seen, out)
    bufs = E.flow_buffers(B, m.s["H"], m.s["I"], m.s["nkv"], m.s["V"], DEV)
    for s in range(N):
        r = _run(m, kc, vc, x, cur0 + s, bufs=bufs, step0=s, first_plain=s == 0, do_select=True, params=params, state=st,
                 seen=seen, out_ids=out, next_ids=nxt)
        hf.advance(greedy_reference(r["logits"].cpu(), seen.cpu(), 1.0), 1)
        assert st == hf.state(), (s, st, hf.state())
        assert torch.equal(out.cpu(), hf.out) and torch.equal(seen.cpu(), hf.seen), s
        if not hf.done:
            assert torch.equal(nxt.cpu(), hf.next), s
    assert 0 in st["unfinished"] and (st["done"] == 1) == (name == "row0_stop"), st
    one = _sequence(m, kc0, vc0, x0, cur0, [N], params=params)
    assert torch.equal(one["out"], out) and torch.equal(one["seen"], seen) and one["state"] == st, name
    assert torch.equal(one["kc"], kc) and torch.equal(one["vc"], vc) and torch.equal(one["logits"], r["logits"]), name


# ---- the op is the engine -----------------------------------------------------------------------------------------------------
def _engine(d, sd, env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        eng = E.Engine(d)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    if sd is not None:
        eng.load_state_dict(sd)
    return eng


def _history(d, sd, emb):
    """The engine's weights as op tensors and its caches after prefill_embeds(emb) (the prefill kernels run_prefill
    issues, as test_decode_chain_gpu._engine_identity rebuilds them)."""
    pre = "model.svg_transformer.transformer.transformer."
    names = dict(ln1_w="ln_1.weight", ln1_b="ln_1.bias", attn_w="attn.c_attn.weight", attn_b="attn.c_attn.bias",
                 proj_w="attn.c_proj.weight", proj_b="attn.c_proj.bias", ln2_w="ln_2.weight", ln2_b="ln_2.bias",
                 fc_w="mlp.c_fc.weight", fc_b="mlp.c_fc.bias", fc2_w="mlp.c_proj.weight", fc2_b="mlp.c_proj.bias")
    n = d.n_layer
    layers = [{k: sd[f"{pre}h.{i}.{v}"].to(DEV) for k, v in names.items()} for i in range(n)]
    wte, wpe = sd[pre + "wte.weight"].to(DEV), sd[pre + "wpe.weight"].to(DEV)
    lnf = (sd[pre + "ln_f.weight"].to(DEV), sd[pre + "ln_f.bias"].to(DEV))
    B, T, _ = emb.shape
    tcap = (min(d.max_len, d.n_positions) + 1 + 31) // 32 * 32
    kc = torch.zeros(n, B, d.n_kv_head, tcap, D, dtype=BF, device=DEV)
    vc = torch.zeros(n, B, d.n_kv_head, D, tcap, dtype=BF, device=DEV)
    x = E.op_embed_prefix(emb.view(B * T, -1), None, wte, wpe, B, T, 0)
    auto = _lib.SV_LINEAR_AUTO
    for l, L in enumerate(layers):
        qkv = E.op_linear(E.op_layernorm(x, L["ln1_w"], L["ln1_b"], d.ln_eps), L["attn_w"], L["attn_b"], None, 0, auto)
        att = E.op_attention_prefill(qkv, kc[l], vc[l], T, d.n_head, d.n_kv_head, 0)
        x = PF._run_linear(auto, att, L["proj_w"], L["proj_b"], x, 0, True)
        hh = E.op_linear(E.op_layernorm(x, L["ln2_w"], L["ln2_b"], d.ln_eps), L["fc_w"], L["fc_b"], None, GELU, auto)
        x = PF._run_linear(auto, hh, L["fc2_w"], L["fc2_b"], x, 0, True)
    return layers, wte, wpe, lnf, kc, vc


def _op(d, layers, wte, wpe, lnf, kc, vc, x, cur0, bufs, **kw):
    return E.op_decode_flow(layers, kc, vc, d.n_head, d.n_kv_head, d.n_positions, wte=wte, wpe=wpe, lnf=lnf, lm_head=wte,
                            x_plain=x, bufs=bufs, cur_len0=cur0, ln_eps=d.ln_eps, **kw)


@pytest.mark.parametrize("B", [1, 8])
def test_engine_decode_step_is_the_op(B):
    d = dataclasses.replace(dims_1b(max_len=2048), n_layer=2, max_batch=B)
    sd = synthetic_state_dict(d, seed=5, init="randomized", device=DEV)
    eng = _engine(d, sd, {"SV_FLOW": "1"})
    T = 300
    g = torch.Generator(device=DEV).manual_seed(T + B)
    emb = torch.randn(B, T, d.hidden, generator=g, device=DEV).to(BF)
    ids = torch.randint(0, d.vocab, (B,), generator=g, device=DEV, dtype=torch.int32)
    try:
        assert "decode=dataflow-kernel-setmaxnreg" in eng.describe(), eng.describe()
        eng.prefill_embeds(emb)
        want = [eng.decode_step(ids), eng.decode_step(ids.flip(0))]
    finally:
        eng.close()
    layers, wte, wpe, lnf, kc, vc = _history(d, sd, emb)
    bufs = E.flow_buffers(B, d.hidden, d.n_inner, d.n_kv_head, d.vocab, DEV)
    for s, t in enumerate((ids, ids.flip(0))):
        x = (wte[t.long()].float() + wpe[T + s].float()).to(BF)
        r = _op(d, layers, wte, wpe, lnf, kc, vc, x, T + s, bufs, step0=s, clear=s == 0)
        assert torch.equal(r["logits"].float(), want[s]), f"step {s}: max |diff| {(r['logits'].float() - want[s]).abs().max()}"


def test_engine_generate_is_the_op_across_launches_and_the_tag_wrap():
    """24 layers (the most the kernel holds): 1400 greedy tokens are three launches of 512, 512 and 375 steps, and
    gp = step * 25 + layer passes 0x7fff at step 1311, inside the third."""
    d = dataclasses.replace(dims_1b(max_len=1536), n_layer=24, max_batch=1)
    sd = synthetic_state_dict(d, seed=6, init="randomized", device=DEV)
    T, n_new = 40, 1400
    emb = torch.randn(1, T, d.hidden, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV).to(BF)
    eng = _engine(d, sd, {"SV_FLOW": "1"})
    try:
        eng.prefill_embeds(emb)
        want = eng.generate(GenerationParams(max_new_tokens=n_new, eos_token_id=None))
    finally:
        eng.close()
    assert want.shape == (1, n_new)
    layers, wte, wpe, lnf, kc, vc = _history(d, sd, emb)
    bufs = E.flow_buffers(1, d.hidden, d.n_inner, d.n_kv_head, d.vocab, DEV)
    tok0 = want[:, 0]
    st = dict(step=1, cur_len=T, done=0, unfinished=[1])
    seen = torch.zeros(1, d.vocab, dtype=torch.uint8, device=DEV)
    seen[0, tok0.long()] = 1
    out = torch.full((1, d.max_len), 0, dtype=torch.int32, device=DEV)
    out[:, 0] = tok0
    nxt = torch.zeros(1, dtype=torch.int32, device=DEV)
    x = (wte[tok0.long()].float() + wpe[T].float()).to(BF)
    params = GenerationParams(max_new_tokens=n_new, eos_token_id=None)
    done = 0
    for i, n in enumerate((512, 512, n_new - 1 - 1024)):
        _op(d, layers, wte, wpe, lnf, kc, vc, x, T + done, bufs, nsteps=n, step0=done, first_plain=i == 0, clear=i == 0,
            do_select=True, params=params, state=st, seen=seen, out_ids=out, next_ids=nxt)
        done += n
    assert (done + 1) * 25 > 0x8000
    assert st["step"] == n_new and st["done"] == 1, st
    assert torch.equal(out[:, :n_new], want), f"first difference at {int((out[:, :n_new] != want).int().argmax())}"


def test_sv_flow_3_selects_the_plain_variant():
    d = dataclasses.replace(dims_1b(max_len=1024), n_layer=1, max_batch=2)
    sd = synthetic_state_dict(d, seed=1, init="randomized", device=DEV)
    for env, want in (({"SV_FLOW": "3"}, "decode=dataflow-kernel "), ({"SV_FLOW": "1"}, "decode=dataflow-kernel-setmaxnreg ")):
        eng = _engine(d, sd, env)
        try:
            assert want in eng.describe(), (env, eng.describe())
        finally:
            eng.close()


@pytest.mark.parametrize("case", ["max_len 16416", "hidden 768"])
def test_sv_flow_falls_back_to_the_graph_path_outside_the_kernels_range(case):
    """Rows longer than the attention's item split covers (16384 keys), and a hidden vector that is not 2^k fragments
    (the staged LayerNorm), decode on the graph path although SV_FLOW=1 is set."""
    if case == "max_len 16416":
        d = dataclasses.replace(dims_1b(max_len=16416), n_positions=16448, n_layer=1, max_batch=1)
    else:
        d = dataclasses.replace(dims_1b(max_len=1024), hidden=768, n_head=6, n_inner=3072, n_layer=1, max_batch=1)
    eng = _engine(d, None, {"SV_FLOW": "1"})
    try:
        assert "dataflow" not in eng.describe().split(" flow[")[0], eng.describe()
    finally:
        eng.close()
    ok = dataclasses.replace(d, max_len=16384, n_positions=16384) if case == "max_len 16416" else None
    if ok is not None:                                  # the longest rows the kernel takes still run it
        eng = _engine(ok, None, {"SV_FLOW": "1"})
        try:
            assert "decode=dataflow-kernel" in eng.describe(), eng.describe()
        finally:
            eng.close()

"""The image-encoder, adapter and prefill kernels one launch at a time, against fp64 references at the 1B and 8B shapes
(sv_op_linear, sv_op_lm_logits, sv_op_layernorm, sv_op_im2col, sv_op_vit_assemble, sv_op_adapter_norm, sv_op_embed_prefix,
sv_op_attention_prefill).

Linear layers are checked twice.  EXACT inputs: x, w and bias on dyadic grids (x in {-2..2}/4, w in {-3..3}/8, bias in
{-4..4}/8), so every fp32 partial sum is exact whatever the accumulation order; the output must then equal the reference's
rounding chain bf16(acc + bias) [-> bf16(act)] [-> bf16(+ residual)] bit for bit (within 1 ulp and >= 99 % bit-equal with
an activation: the kernels' __expf / tanhf are not torch's).  A wrong K block, tile position, mask or rounding point
cannot hide there.  RANDOM inputs at realistic scale: within the rule below and >= 99 % bit-equal (98 % at K > 8192, where the fp32 sum's
rounding reaches a bf16 rounding boundary more often).

Tolerances (the worst error / tolerance of every kernel family is printed as one `CALIB` line at the end, with -s):
  linear:          |y - ref| <= 1 ulp(ref) + 2^-18 sum_k |x_k w_nk| (times the activation's slope) + 1 ulp of the
                   pre-activation / pre-residual value when there is one
  LayerNorm:       1 ulp(ref) + 2^-20 |mean| rstd |w| (the fp32 cancellation floor of large-mean rows) + 2^-22 (|x_hat w|
                   + |b|) (fp32 arithmetic, visible where the affine output cancels to near zero); >= 99.5 % bit-equal
  adapter slab LN: the same rule over the [Q, H] slab; >= 99 % bit-equal
  token BatchNorm: 1 ulp(ref) + 2^-21 (|x_hat w| + |b|); >= 99 % bit-equal
  attention:       1 ulp(ref) + 0.02 rms(ref of that row and head), bitwise independent of the poison in unread slots
  im2col, vit_assemble, embed_prefix, lm_logits on exact inputs, the KV scatter: bit-exact
"""
import math

import pytest
import torch
import torch.nn.functional as F

from starvector_b200 import _lib
from starvector_b200 import engine as E
from test_decode_ops_gpu import _ulp
from test_ops_gpu import _close_attn, plant_strong_keys, ref_causal_attention

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
NONE, QGELU, GELU, SILU = _lib.SV_ACT_NONE, _lib.SV_ACT_QUICKGELU, _lib.SV_ACT_GELU_TANH, _lib.SV_ACT_SILU
RG, WG, AUTO = _lib.SV_LINEAR_ROWGROUP, _lib.SV_LINEAR_TCGEN05, _lib.SV_LINEAR_AUTO
P = 2                       # prompt tokens after the visual prefix ("<svg")
SLOPE = {NONE: 1.0, QGELU: 1.15, GELU: 1.15, SILU: 1.15}   # max |act'| over the range the inputs reach

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


def _randn(*shape, g, scale=1.0, mean=0.0):
    return (torch.randn(*shape, generator=g, device=DEV) * scale + mean).to(BF)


def _grid(*shape, g, lo, hi, div):
    return (torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float() / div).to(BF)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wide_tile(M, N, sms):
    """launch_linear_wgmma's tile rule: BN = 128 when N % 128 == 0 and the BN = 64 tiles would not fit one wave of two
    CTAs per SM."""
    return N % 128 == 0 and ((M + 127) // 128) * ((N + 63) // 64) > 2 * sms


def _resolve_m(M, N, sms):
    """'narrow' / 'wide': the largest M that still gets BN = 64 at this N and SM count, and the smallest that gets 128."""
    if isinstance(M, int):
        return M
    mt = 2 * sms // ((N + 63) // 64)            # most 128-row tiles that still fit the BN = 64 wave
    return mt * 128 if M == "narrow" else mt * 128 + 1


# ---- linear ------------------------------------------------------------------------------------------------------------
def _act_ref(v, act):
    """The reference's activation on bf16-rounded fp32 values, result rounded to bf16 (sv_common.cuh epilogue_elem)."""
    r = lambda t: t.to(BF).float()
    if act == QGELU:
        return r(v * r(torch.sigmoid(r(1.702 * v))))
    if act == SILU:
        return r(v * r(torch.sigmoid(v)))
    if act == GELU:
        return r(F.gelu(v, approximate="tanh"))
    return v


def _chain(acc, bias, res, act):
    """bf16(acc + bias) -> bf16(act) -> bf16(+ residual) from the fp64 accumulator; returns (output, pre-residual value)."""
    v = acc + bias.double() if bias is not None else acc
    r1 = v.float().to(BF).float()
    r2 = _act_ref(r1, act)
    out = (r2 + res.float()).to(BF).float() if res is not None else r2
    return out.double(), r1.double()


def _run_linear(impl, x, w, bias, res, act, inplace):
    M, K = x.shape
    N = w.shape[0]
    if inplace:                                  # y aliases the residual, as the engine's x += f(x) layers run
        y = res.clone()
        lib = _lib.load()
        _lib.check(lib, lib.sv_op_linear(impl, E._p(x), E._p(w), E._p(bias), E._p(y), E._p(y), M, N, K, act,
                                         E._stream_ptr(x.device)))
        torch.cuda.synchronize()
        return y
    y = E.op_linear(x, w, bias, res, act, impl)
    torch.cuda.synchronize()
    return y


def check_linear(impl, M, N, K, bias, act, res, seed, family):
    """res: None, "add" (separate residual) or "inplace".  Exact-input then random-input check."""
    g = _gen(seed)
    # exact inputs
    x = _grid(M, K, g=g, lo=-2, hi=2, div=4)
    w = _grid(N, K, g=g, lo=-3, hi=3, div=8)
    b = _grid(N, g=g, lo=-4, hi=4, div=8) if bias else None
    r = _randn(M, N, g=g) if res else None
    y = _run_linear(impl, x, w, b, r, act, res == "inplace").double()
    ref, _ = _chain(x.double() @ w.double().T, b, r, act)
    if act == NONE:
        bad = (y != ref).nonzero()
        assert bad.numel() == 0, f"exact inputs: {bad.shape[0]} of {y.numel()} outputs differ, first at {bad[0].tolist()}: " \
                                 f"{y[tuple(bad[0])].item()} vs {ref[tuple(bad[0])].item()}"
    else:
        assert ((y - ref).abs() <= _ulp(ref)).all(), "exact inputs: more than 1 ulp off with an activation"
        assert (y == ref).double().mean().item() >= 0.99
    # random inputs at realistic scale
    x = _randn(M, K, g=g)
    w = _randn(N, K, g=g, scale=1 / math.sqrt(K))
    b = _randn(N, g=g, scale=0.1) if bias else None
    r = _randn(M, N, g=g) if res else None
    y = _run_linear(impl, x, w, b, r, act, res == "inplace").double()
    xd, wd = x.double(), w.double()
    ref, pre = _chain(xd @ wd.T, b, r, act)
    s = xd.abs() @ wd.abs().T
    tol = _ulp(ref) + 2.0 ** -18 * s * SLOPE[act]
    if act != NONE or res:
        tol = tol + _ulp(pre) * SLOPE[act]
    err = (y - ref).abs()
    _calib(family, (err / tol).max().item())
    eq = (y == ref).double().mean().item()
    assert eq >= (0.99 if K <= 8192 else 0.98), f"random inputs, impl {impl}: only {100 * eq:.2f} % bit-equal"


def _engine_gemms():
    """Every GEMM of run_encode and run_prefill: (id, M, N, K, bias, act, res) at the 1B and 8B widths."""
    out = []
    for name, W, H, qkv, inner, Q, NP, Kp, conv_bias, vit_act, Bs in (
            ("v1", 1024, 2048, 2304, 8192, 257, 256, 640, False, QGELU, (1, 2, 8, 16)),
            ("v2", 1024, 4608, 5632, 18432, 576, 576, 768, True, GELU, (1, 2, 4))):
        for B in Bs:
            Me, Mp = B * Q, B * (Q + P)
            for lay, M, N, K, bias, act, res in (
                    ("patch", B * NP, W, Kp, conv_bias, NONE, None), ("vit_qkv", Me, 3 * W, W, True, NONE, None),
                    ("vit_out", Me, W, W, True, NONE, "inplace"), ("vit_fc", Me, 4 * W, W, True, vit_act, None),
                    ("vit_proj", Me, W, 4 * W, True, NONE, "inplace"), ("adapter_fc", Me, 2 * W, W, True, SILU, None),
                    ("adapter_proj", Me, H, 2 * W, True, NONE, None), ("dec_qkv", Mp, qkv, H, True, NONE, None),
                    ("dec_proj", Mp, H, H, True, NONE, "inplace"), ("dec_fc", Mp, inner, H, True, GELU, None),
                    ("dec_fc2", Mp, H, inner, True, NONE, "inplace")):
                out.append(pytest.param(M, N, K, bias, act, res, id=f"{name}-B{B}-{lay}-{M}x{N}x{K}"))
    return out


ENGINE_GEMMS = _engine_gemms()

# (M, N, K, bias, act, res): M at the 128-row tile edges, N below / at the tile widths, K over the 3- and 4-stage ring
# wraps (nk = 1..5) and the largest K; "narrow" / "wide" sit on either side of the BN = 128 rule at this GPU's SM count
EDGE_GEMMS = [
    (1, 128, 64, True, NONE, None), (2, 8, 64, False, NONE, None), (127, 72, 128, True, NONE, None),
    (128, 192, 192, True, NONE, "add"), (129, 320, 256, False, NONE, "inplace"), (255, 1024, 320, True, NONE, None),
    (256, 2112, 320, True, NONE, None), (129, 8, 320, True, NONE, None), (257, 72, 128, True, NONE, "inplace"),
    (127, 320, 128, True, GELU, None), (129, 192, 256, True, QGELU, None), (129, 256, 18432, False, NONE, None),
    ("narrow", 1024, 64, True, NONE, None), ("narrow", 1024, 320, True, NONE, "inplace"),
    ("wide", 1024, 64, True, NONE, None), ("wide", 1024, 128, False, NONE, None), ("wide", 1024, 192, True, SILU, None),
    ("wide", 1024, 256, True, NONE, "inplace"), ("wide", 1024, 320, False, NONE, "inplace"),
    ("wide", 1024, 18432, True, NONE, None),
]


@pytest.mark.parametrize("M,N,K,bias,act,res", ENGINE_GEMMS)
def test_linear_engine_shapes(M, N, K, bias, act, res):
    check_linear(WG, M, N, K, bias, act, res, seed=M * 7 + N + K, family="linear wgmma")


@pytest.mark.parametrize("M,N,K,bias,act,res", EDGE_GEMMS, ids=lambda v: str(v))
def test_linear_edges(M, N, K, bias, act, res):
    M = _resolve_m(M, N, _sms())
    check_linear(WG, M, N, K, bias, act, res, seed=M + 3 * N + K, family="linear wgmma")
    if M <= 300:         # the rowgroup kernel's > 8-row loop (its correctness fallback) at the same shapes
        check_linear(RG, M, N, K, bias, act, res, seed=M + 3 * N + K + 1, family="linear rowgroup")


def test_linear_tiles_reach_both_widths():
    """The parametrisation runs the wgmma kernel on both tiles, BN = 128 in place and not in place."""
    sms = _sms()
    seen = set()
    for p in ENGINE_GEMMS + [pytest.param(*e) for e in EDGE_GEMMS]:
        M, N, K, bias, act, res = p.values
        seen.add((_wide_tile(_resolve_m(M, N, sms), N, sms), res == "inplace"))
    assert seen == {(False, False), (False, True), (True, False), (True, True)}, seen
    assert not _wide_tile(_resolve_m("narrow", 1024, sms), 1024, sms) and _wide_tile(_resolve_m("wide", 1024, sms), 1024, sms)


@pytest.mark.parametrize("M", [1, 8, 16, 32, 33, 64, 257])
def test_linear_auto_picks_the_engine_kernel(M):
    """AUTO (the engine's default) equals the kernel it picks bit for bit: rowgroup for M <= 32, wgmma above."""
    g = _gen(M)
    x, w, b = _randn(M, 2048, g=g), _randn(2304, 2048, g=g, scale=2048 ** -0.5), _randn(2304, g=g, scale=0.1)
    auto = E.op_linear(x, w, b, None, GELU, AUTO)
    pick = E.op_linear(x, w, b, None, GELU, RG if M <= 32 else WG)
    assert torch.equal(auto, pick)


LM_HEADS = [(49156, 2048), (49157, 4608)]


@pytest.mark.parametrize("N,K", LM_HEADS, ids=["v1", "v2"])
@pytest.mark.parametrize("M", [1, 5, 8, 9, 16])
def test_linear_rowgroup_lm_head(M, N, K):
    """The prefill / per-op decode lm_head on the rowgroup kernel: 1..16 rows (the > 8-row group loop) and the ragged
    last 16-row block of the vocabulary (rows clamped to N - 1)."""
    check_linear(RG, M, N, K, False, NONE, None, seed=M + K, family="linear rowgroup")


@pytest.mark.parametrize("N,K", LM_HEADS, ids=["v1", "v2"])
@pytest.mark.parametrize("M", [1, 9, 16, 129])
def test_lm_logits_exact(M, N, K):
    """The kEpiLogits launch (the bf16 logits left resident after sv_score_tokens): bit-equal to bf16 of the exact-input
    product at the ragged vocabulary, and nothing written past element M * N."""
    g = _gen(N + M)
    x = _grid(M, K, g=g, lo=-2, hi=2, div=4)
    w = _grid(N, K, g=g, lo=-3, hi=3, div=8)
    canary = torch.tensor(-12345.0, dtype=BF, device=DEV)
    buf = torch.full((M * N + 4096,), float(canary), dtype=BF, device=DEV)
    E.op_lm_logits(x, w, buf)
    ref = (x.double() @ w.double().T).float().to(BF)
    assert torch.equal(buf[:M * N].view(M, N), ref)
    assert (buf[M * N:] == canary).all(), "lm_logits wrote past its M * N outputs"
    _calib("lm_logits (bit-exact)", 0.0)


# ---- LayerNorm ---------------------------------------------------------------------------------------------------------
def _ln_tol(xd, dims, eps, w, b, ref):
    """1 ulp + the fp32 floors: x - mean cancels on rows with a large mean, leaving ~2^-20 |mean| of error (times rstd and
    w); and the affine output carries ~2^-22 of the magnitude of its terms, which shows where they cancel."""
    mean = xd.mean(dims, keepdim=True)
    rstd = 1.0 / (xd.var(dims, unbiased=False, keepdim=True) + eps).sqrt()
    wd, bd = w.double(), b.double()
    return _ulp(ref) + 2.0 ** -20 * mean.abs() * rstd * wd.abs() + 2.0 ** -22 * (((xd - mean) * rstd * wd).abs() + bd.abs())


def _check_ln(family, y, ref, tol, min_eq):
    err = (y - ref).abs()
    eq = (y == ref.to(BF).double()).double().mean().item()
    ulps = (err / _ulp(ref)).max().item()
    assert eq >= min_eq, f"{family}: only {100 * eq:.3f} % bit-equal (worst {ulps:.1f} ulp)"
    _calib(family, (err / tol).max().item())


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("cols,rows", [(1024, 16 * 257), (1024, 16 * 576), (2048, 16 * (257 + P)), (4608, 16 * (576 + P))])
def test_layernorm(cols, rows, eps):
    g = _gen(cols + rows)
    x = torch.randn(rows, cols, generator=g, device=DEV) * 2.0
    x[: rows // 4] = torch.randn(rows // 4, cols, generator=g, device=DEV) + 50.0       # mean 50, std 1
    x[rows // 4: rows // 4 + 8] = torch.randn(8, 1, generator=g, device=DEV) * 10.0    # constant rows: var = 0
    x = x.to(BF)
    w, b = _randn(cols, g=g, scale=0.3, mean=1.0), _randn(cols, g=g, scale=0.2)
    y = E.op_layernorm(x, w, b, eps).double()
    xd = x.double()
    ref = F.layer_norm(xd, (cols,), w.double(), b.double(), eps)
    _check_ln("layernorm", y, ref, _ln_tol(xd, -1, eps, w, b, ref), 0.995)
    const = slice(rows // 4, rows // 4 + 8)
    assert torch.equal(y[const], b.double().expand(8, cols)), "a constant row must give exactly b"


# ---- ViT front -----------------------------------------------------------------------------------------------------------
VIT_FRONTS = [(224, 14, 640), (384, 16, 768), (56, 14, 640), (64, 16, 768)]


def _unfold_ref(px, patch, kpad):
    B = px.shape[0]
    cols = F.unfold(px.float(), kernel_size=patch, stride=patch)            # [B, 3 p p, L], (c, iy, ix) x (py, px)
    ref = cols.transpose(1, 2).reshape(-1, cols.shape[1])
    return F.pad(ref, (0, kpad - ref.shape[1])).to(BF).view(B * cols.shape[2], kpad)


@pytest.mark.parametrize("image,patch,kpad", VIT_FRONTS, ids=lambda v: str(v))
def test_im2col_bit_exact(image, patch, kpad):
    g = _gen(image)
    px = _randn(3, 3, image, image, g=g)
    got = E.op_im2col(px, patch, kpad)
    assert torch.equal(got, _unfold_ref(px, patch, kpad))
    _calib("im2col (bit-exact)", 0.0)


@pytest.mark.parametrize("bias", [False, True], ids=["no_bias", "bias"])
@pytest.mark.parametrize("image,patch,kpad", VIT_FRONTS[:2], ids=["224-14", "384-16"])
def test_patch_embedding_against_conv2d(image, patch, kpad, bias):
    """im2col + the wgmma GEMM over the zero-padded conv weight == fp64 F.conv2d (CLIP without, SigLIP with a bias)."""
    g = _gen(image + bias)
    B, W = 2, 1024
    px = _randn(B, 3, image, image, g=g)
    cw = _randn(W, 3, patch, patch, g=g, scale=(3 * patch * patch) ** -0.5)
    cb = _randn(W, g=g, scale=0.1) if bias else None
    wpad = F.pad(cw.reshape(W, -1), (0, kpad - 3 * patch * patch))
    pe = E.op_linear(E.op_im2col(px, patch, kpad), wpad, cb, None, NONE, WG).double()
    conv = F.conv2d(px.double(), cw.double(), None, stride=patch)                  # [B, W, g, g]
    acc = conv.flatten(2).transpose(1, 2).reshape(-1, W)
    ref, _ = _chain(acc, cb, None, NONE)
    s = F.conv2d(px.double().abs(), cw.double().abs(), None, stride=patch).flatten(2).transpose(1, 2).reshape(-1, W)
    _calib("patch conv (im2col + wgmma)", ((pe - ref).abs() / (_ulp(ref) + 2.0 ** -18 * s)).max().item())


@pytest.mark.parametrize("B,np_,cls", [(3, 256, True), (2, 576, False), (1, 16, True)], ids=["clip", "siglip", "tiny"])
def test_vit_assemble_bit_exact(B, np_, cls):
    g = _gen(np_)
    W = 1024
    q = np_ + cls
    pe, pos = _randn(B * np_, W, g=g), _randn(q, W, g=g, scale=0.5)
    c = _randn(W, g=g) if cls else None
    got = E.op_vit_assemble(pe, c, pos, B)
    src = pe.float().view(B, np_, W)
    if cls:
        src = torch.cat([c.float().expand(B, 1, W), src], 1)
    assert torch.equal(got, (src + pos.float()).to(BF).view(B * q, W))
    _calib("vit_assemble (bit-exact)", 0.0)


# ---- adapter norm ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 8, 16])
@pytest.mark.parametrize("Q,H", [(257, 2048), (576, 4608), (17, 256), (3, 8)], ids=["v1", "v2", "tiny", "24"])
def test_adapter_slab_layernorm(Q, H, B):
    """LayerNorm([Q, H]) per image, large-mean slabs (mean 20, std 0.5) included, against fp64 F.layer_norm; the tiny
    model's slab and a 24-element one, where the variance's divisor shows."""
    g = _gen(Q * B)
    z = torch.randn(B, Q, H, generator=g, device=DEV) * 1.5
    z[B // 2] = torch.randn(Q, H, generator=g, device=DEV) * 0.5 + 20.0
    if B > 2:
        z[-1] = torch.randn(Q, H, generator=g, device=DEV) * 0.5 - 20.0
    z = z.to(BF)
    w, b = _randn(Q, H, g=g, scale=0.2, mean=1.0), _randn(Q, H, g=g, scale=0.1)
    y = E.op_adapter_norm(_lib.SV_ADAPTER_NORM_SLAB, z, w, b).double()
    zd = z.double()
    ref = F.layer_norm(zd, (Q, H), w.double(), b.double(), 1e-5)
    _check_ln("adapter slab LayerNorm", y, ref, _ln_tol(zd, (1, 2), 1e-5, w, b, ref), 0.99)


@pytest.mark.parametrize("B", [2, 16])
@pytest.mark.parametrize("Q,H", [(257, 2048), (576, 4608)], ids=["v1", "v2"])
def test_adapter_token_batchnorm(Q, H, B):
    """Eval BatchNorm1d(Q) with bf16 running statistics (channel = token): a token with running var 0, one with a large
    mean, against fp64 F.batch_norm."""
    g = _gen(Q + B)
    rm = _randn(Q, g=g, scale=0.5)
    rv = torch.exp(torch.randn(Q, generator=g, device=DEV)).to(BF)
    w, b = _randn(Q, g=g, scale=0.3, mean=1.0), _randn(Q, g=g, scale=0.2)
    rm[3], rv[5], rv[6] = 40.0, 0.0, 1e-7
    z = torch.randn(B, Q, H, generator=g, device=DEV) * rv.float().sqrt()[:, None] + rm.float()[:, None]
    z = z.to(BF)
    y = E.op_adapter_norm(_lib.SV_ADAPTER_NORM_TOKENS, z, w, b, rm, rv).double()
    ref = F.batch_norm(z.double(), rm.double(), rv.double(), w.double(), b.double(), False, 0.0, 1e-5)
    xhat = (z.double() - rm.double()[:, None]) / (rv.double()[:, None] + 1e-5).sqrt()
    tol = _ulp(ref) + 2.0 ** -21 * ((xhat * w.double()[:, None]).abs() + b.double().abs()[:, None])
    _calib("adapter token BatchNorm", ((y - ref).abs() / tol).max().item())
    assert (y == ref.to(BF).double()).double().mean().item() >= 0.99


# ---- prefix embedding ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", ["v1", "v2_no_wpe", "scoring"])
def test_embed_prefix_bit_exact(form):
    """bf16(visual or wte[clamp(id)] + wpe[pos0 + t]): ids -1, vocab and vocab + 5 clamp to 0 / vocab - 1; the scoring
    form has no visual rows, starts at pos0 > 0 and reads its ids with a row stride != p; v2 has no wpe."""
    g = _gen(len(form))
    if form == "v1":
        B, q, p, H, vocab, pos0, stride, npos = 3, 257, 6, 2048, 49156, 0, 6, 8192
    elif form == "v2_no_wpe":
        B, q, p, H, vocab, pos0, stride, npos = 2, 576, 6, 4608, 49157, 0, 6, 0
    else:
        B, q, p, H, vocab, pos0, stride, npos = 4, 0, 16, 2048, 49156, 300, 40, 8192     # ids [B][40], chunk at 8
    wte = _randn(vocab, H, g=g)
    wpe = _randn(npos, H, g=g, scale=0.3) if npos else None
    vis = _randn(B, q, H, g=g) if q else None
    c0 = 8 if form == "scoring" else 0                       # the chunk's ids start c0 into each row of `stride` ids
    ids = torch.randint(0, vocab, (B, stride), generator=g, device=DEV, dtype=torch.int32)
    ids[0, c0:c0 + 3] = torch.tensor([-1, vocab, vocab + 5], dtype=torch.int32)
    ids[B - 1, c0 + p - 1] = -7
    got = E.op_embed_prefix(vis, ids.view(-1)[c0:], wte, wpe, B, q, p, pos0, stride)
    take = ids[:, c0:c0 + p].long().clamp(0, vocab - 1)
    rows = wte[take].float()                                  # [B, p, H]
    if q:
        rows = torch.cat([vis.float(), rows], 1)
    if wpe is not None:
        rows = rows + wpe[pos0: pos0 + q + p].float()
    assert torch.equal(got, rows.to(BF).view(B * (q + p), H))
    _calib("embed_prefix (bit-exact)", 0.0)


# ---- prefill attention -----------------------------------------------------------------------------------------------------
D = 128
PREFILL_CASES = [   # (B, seq, n_head, n_kv, window)
    (2, 259, 16, 1, 0), (2, 300, 36, 4, 0), (2, 100, 4, 2, 24), (3, 70, 18, 2, 0), (1, 700, 36, 4, 512),
    (4, 47, 36, 4, 24), (1, 4150, 36, 4, 4096),
]


def _strong_positions(seq, window):
    pos = {0, 31, 32, 33, seq - 1}
    if window:
        pos |= {seq - window, max(0, seq - window - 1), window - 1}
    return sorted(p for p in pos if 0 <= p < seq)


@pytest.mark.parametrize("B,seq,nh,nkv,window", PREFILL_CASES, ids=lambda v: str(v))
def test_attention_prefill(B, seq, nh, nkv, window):
    """sv_op_attention_prefill over caller-owned caches: strong keys at 0, 31/32/33, window starts and seq - 1; slots
    seq .. tcap - 1 and the cache row of an image past the batch hold a finite poison key.  The output is within 1 ulp +
    0.02 rms of fp64, bitwise independent of the poison, and the scattered K / V equal the qkv columns bit for bit."""
    grp = nh // nkv
    tcap = (seq + 31) // 32 * 32 + 32
    qkv = _randn(B * seq, (nh + 2 * nkv) * D, g=_gen(seq + nh)).cpu()
    groups = [([(k * grp + j) * D for j in range(grp)], (nh + k) * D, (nh + nkv + k) * D) for k in range(nkv)]
    plant_strong_keys(qkv, B, seq, groups, D, _strong_positions(seq, window), seed=seq)
    qkv = qkv.to(DEV)
    x = qkv.view(B, seq, nh + 2 * nkv, D)
    strong_k = x[:, seq - 1, nh:nh + nkv]                    # [B, nkv, D]: scores 20 for every head of its group

    def run(kscale, vval):
        kc = torch.empty(B + 1, nkv, tcap, D, dtype=BF, device=DEV)
        vc = torch.full((B + 1, nkv, D, tcap), vval, dtype=BF, device=DEV)
        pk = (strong_k.float() * kscale).to(BF)
        kc[:B] = pk[:, :, None, :]
        kc[B] = pk[0, :, None, :]
        out = E.op_attention_prefill(qkv, kc, vc, seq, nh, nkv, window)       # batch B: image B's row is not read
        return out, kc, vc, pk

    out, kc, vc, pk = run(1.5, 500.0)
    out2, _, _, _ = run(-1.0, -300.0)
    assert torch.equal(out, out2), "the output depends on cache slots the attention must not read"
    # the scatter: K rows and V^T columns of slots [0, seq) are the qkv columns; slots >= seq and image B untouched
    assert torch.equal(kc[:B, :, :seq], x[:, :, nh:nh + nkv].transpose(1, 2))
    assert torch.equal(vc[:B, :, :, :seq], x[:, :, nh + nkv:].permute(0, 2, 3, 1))
    assert torch.equal(kc[:B, :, seq:], pk[:, :, None, :].expand(B, nkv, tcap - seq, D))
    assert (vc[:B, :, :, seq:] == 500.0).all() and (vc[B] == 500.0).all()
    ref = ref_causal_attention(qkv, B, seq, nh, nkv, window)
    _calib("attention_prefill", _close_attn(out, ref, D))

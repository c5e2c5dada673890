"""Single-kernel parity through the C-ABI (sv_op_*) against plain PyTorch fp32 references."""
import math

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200 import engine as E

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bf(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _r(x):  # bf16 rounding point
    return x.to(torch.bfloat16).float()


def _ref_linear(x, w, b, res, act):
    y = x.float() @ w.float().t()
    if b is not None:
        y = y + b.float()
    y = _r(y)
    if act == _lib.SV_ACT_QUICKGELU:
        y = _r(y * _r(torch.sigmoid(_r(1.702 * y))))
    elif act == _lib.SV_ACT_SILU:
        y = _r(y * _r(torch.sigmoid(y)))
    elif act == _lib.SV_ACT_GELU_TANH:
        y = _r(torch.nn.functional.gelu(y, approximate="tanh"))
    if res is not None:
        y = _r(y + res.float())
    return y


def _close(got, ref, ulps=2.0, atol=2e-2):
    got, ref = got.float(), ref.float()
    tol = ulps * 2.0 ** -8 * ref.abs() + atol
    bad = (got - ref).abs() > tol
    assert not bool(bad.any()), f"{int(bad.sum())} / {bad.numel()} mismatches, max err {(got - ref).abs().max().item():.4f}"


def test_layernorm():
    for rows, cols in ((5, 128), (259, 2048), (3, 8192)):
        x, w, b = _bf(rows, cols, seed=1), _bf(cols, scale=0.5, seed=2) + 1, _bf(cols, scale=0.1, seed=3)
        y = E.op_layernorm(x, w, b, 1e-5)
        ref = torch.nn.functional.layer_norm(x.float(), (cols,), w.float(), b.float(), 1e-5)
        _close(y, _r(ref), ulps=1.5, atol=1e-2)


@pytest.mark.parametrize("impl", [_lib.SV_LINEAR_ROWGROUP, _lib.SV_LINEAR_TCGEN05], ids=["rowgroup", "tcgen05"])
@pytest.mark.parametrize("M,N,K", [(1, 256, 256), (8, 2304, 2048), (5, 500, 256), (259, 2304, 2048), (514, 1024, 640),
                                   (257, 4096, 1024), (130, 128, 8192), (64, 64, 64)])
def test_linear_shapes(impl, M, N, K):
    if impl == _lib.SV_LINEAR_TCGEN05 and (N % 8 or K % 64):
        pytest.skip("shape not taken by the wgmma kernel")
    if impl == _lib.SV_LINEAR_ROWGROUP and M > 300:
        pytest.skip("fallback path: covered at smaller M")
    x, w, b = _bf(M, K, seed=4), _bf(N, K, scale=1 / math.sqrt(K), seed=5), _bf(N, scale=0.1, seed=6)
    y = E.op_linear(x, w, b, None, _lib.SV_ACT_NONE, impl)
    _close(y, _ref_linear(x, w, b, None, 0))


@pytest.mark.parametrize("impl", [_lib.SV_LINEAR_ROWGROUP, _lib.SV_LINEAR_TCGEN05], ids=["rowgroup", "tcgen05"])
@pytest.mark.parametrize("act", [_lib.SV_ACT_NONE, _lib.SV_ACT_QUICKGELU, _lib.SV_ACT_GELU_TANH, _lib.SV_ACT_SILU])
def test_linear_epilogues(impl, act):
    M, N, K = 70, 384, 512
    x, w, b, res = _bf(M, K, seed=7), _bf(N, K, scale=1 / math.sqrt(K), seed=8), _bf(N, scale=0.2, seed=9), _bf(M, N, seed=10)
    _close(E.op_linear(x, w, b, None, act, impl), _ref_linear(x, w, b, None, act))
    _close(E.op_linear(x, w, None, res, act, impl), _ref_linear(x, w, None, res, act))
    # in-place residual (how the engine uses it): y aliases the residual
    buf = res.clone()
    lib = _lib.load()
    _lib.check(lib, lib.sv_op_linear(impl, E._p(x), E._p(w), E._p(b), E._p(buf), E._p(buf), M, N, K, act,
                                     E._stream_ptr(x.device)))
    _close(buf, _ref_linear(x, w, b, res, act))


def test_linear_tcgen05_agrees_with_rowgroup():
    """The two kernels accumulate in different orders; they must agree to <= 1 bf16 ulp."""
    x, w, b = _bf(200, 1024, seed=11), _bf(512, 1024, scale=1 / 32, seed=12), _bf(512, scale=0.1, seed=13)
    a = E.op_linear(x, w, b, None, 0, _lib.SV_LINEAR_ROWGROUP).float()
    c = E.op_linear(x, w, b, None, 0, _lib.SV_LINEAR_TCGEN05).float()
    assert ((a - c).abs() <= 2.0 ** -7 * a.abs() + 1e-3).all()
    assert (a == c).float().mean() > 0.98


@pytest.mark.parametrize("B,L,H", [(1, 17, 2), (2, 257, 16), (3, 40, 4)])
def test_attention_vit(B, L, H):
    W = H * 64
    qkv = _bf(B * L, 3 * W, seed=14)
    out = E.op_attention_vit(qkv, B, L, H)
    q, k, v = qkv.float().view(B, L, 3, H, 64).permute(2, 0, 3, 1, 4)
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(B * L, W)
    _close(out, ref, ulps=2, atol=1.5e-2)


@pytest.mark.parametrize("B,T,H", [(1, 19, 2), (2, 259, 16), (1, 70, 9)])
def test_attention_mqa_causal(B, T, H):
    D = 128
    qkv = _bf(B * T, H * D + 2 * D, seed=15)
    out = E.op_attention_mqa(qkv, B, T, H)
    x = qkv.float().view(B, T, H * D + 2 * D)
    q = x[..., : H * D].view(B, T, H, D).transpose(1, 2)
    k = x[..., H * D: H * D + D].unsqueeze(1).expand(B, H, T, D)
    v = x[..., H * D + D:].unsqueeze(1).expand(B, H, T, D)
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B * T, H * D)
    _close(out, ref, ulps=2, atol=1.5e-2)

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


def _close_attn(got, ref, dim, ulps=1.0, c=0.02):
    """Scale-aware attention tolerance: 1 bf16 ulp + 2 % of the rms of that (row, head) output.  Attention outputs shrink
    as the context grows, so a fixed atol would end up larger than the output itself and pass a key range off by one."""
    got, ref = got.double().reshape(-1, dim), ref.double().reshape(-1, dim)
    rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp(min=2.0 ** -126))) - 7)
    err = (got - ref).abs()
    tol = ulps * ulp + c * rms
    bad = err > tol
    assert not bool(bad.any()), f"{int(bad.sum())} / {bad.numel()} mismatches, worst err/rms {(err / rms).max().item():.4f}"
    return (err / tol).max().item()


def ref_causal_attention(qkv, B, T, n_head, n_kv, window=0, chunk=512, q0=0):
    """fp64 causal attention of packed qkv rows [B*T, (n_head + 2 n_kv) * 128] (query head h reads KV head h // group;
    keys > t - window when window > 0) -> [B*(T - q0), n_head * 128] for the queries of positions [q0, T), over chunks of
    queries."""
    D, grp = 128, n_head // n_kv
    x = qkv.double().view(B, T, n_head + 2 * n_kv, D)
    q = x[:, :, :n_head].reshape(B, T, n_kv, grp, D)
    k, v = x[:, :, n_head:n_head + n_kv], x[:, :, n_head + n_kv:]
    out = torch.empty(B, T - q0, n_kv, grp, D, dtype=torch.float64, device=qkv.device)
    ks = torch.arange(T, device=qkv.device)
    for t0 in range(q0, T, chunk):
        t1 = min(T, t0 + chunk)
        s = torch.einsum("btkgd,bskd->bkgts", q[:, t0:t1], k) / math.sqrt(D)
        tq = torch.arange(t0, t1, device=qkv.device)[:, None]
        mask = ks[None, :] <= tq
        if window > 0:
            mask &= ks[None, :] > tq - window
        p = torch.softmax(s.masked_fill(~mask, float("-inf")), dim=-1)
        out[:, t0 - q0:t1 - q0] = torch.einsum("bkgts,bskd->btkgd", p, v)
    return out.reshape(B * (T - q0), n_head * D)


def plant_strong_keys(x, B, L, groups, dim, positions, seed):
    """In packed rows x [B*L, cols] (CPU): aim every query of each group's heads along its own direction u_h (orthonormal in
    the group) and make the keys at `positions` score 20 for all of them, with V = 4 N(0,1).  Where such a key is visible it
    dominates the output; where it is masked, reading it would.  groups: [(q column offsets, k offset, v offset)]."""
    g = torch.Generator().manual_seed(seed)
    x = x.view(B, L, -1)
    for qo, ko, vo in groups:
        u = torch.linalg.qr(torch.randn(dim, len(qo), generator=g, dtype=torch.float64)).Q.T
        for j, o in enumerate(qo):
            x[:, :, o:o + dim] = (u[j] * math.sqrt(dim) + 0.3 * torch.randn(B, L, dim, generator=g, dtype=torch.float64)).to(x.dtype)
        for p in positions:
            x[:, p, ko:ko + dim] = (20.0 * u.sum(0)).to(x.dtype)
            x[:, p, vo:vo + dim] = (4.0 * torch.randn(B, dim, generator=g)).to(x.dtype)


@pytest.mark.parametrize("B,L,H,strong", [(1, 17, 2, False), (2, 257, 16, False), (3, 40, 4, False), (2, 257, 4, True),
                                           (8, 257, 16, True), (16, 257, 16, True), (1, 576, 16, True), (4, 576, 16, True)],
                         ids=["1-17-2", "2-257-16", "3-40-4", "2-257-4-strong", "8-257-16-strong", "16-257-16-strong",
                              "1-576-16-strong", "4-576-16-strong"])
def test_attention_vit(B, L, H, strong):
    """strong: keys at 0, 31, 32, 33, 255, 256 and L - 1 that every query of a head scores at 20 (CLIP: L = 257 at up to
    16 images; SigLIP: L = 576)."""
    W = H * 64
    qkv = _bf(B * L, 3 * W, seed=14)
    if strong:
        x = qkv.cpu()
        pos = sorted({p for p in (0, 31, 32, 33, 255, 256) if p < L} | {L - 1})
        plant_strong_keys(x, B, L, [([h * 64], W + h * 64, 2 * W + h * 64) for h in range(H)], 64, pos, seed=1)
        qkv = x.to(DEV)
    out = E.op_attention_vit(qkv, B, L, H)
    q, k, v = qkv.double().view(B, L, 3, H, 64).permute(2, 0, 3, 1, 4)
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(B * L, W)
    print(f"CALIB attention_vit B={B} L={L} H={H}: worst error / tolerance = {_close_attn(out, ref, 64):.3f}")


@pytest.mark.parametrize("B,T,H,strong", [(1, 19, 2, False), (2, 259, 16, False), (1, 70, 9, False), (2, 259, 16, True)],
                         ids=["1-19-2", "2-259-16", "1-70-9", "2-259-16-strong"])
def test_attention_mqa_causal(B, T, H, strong):
    """strong: keys at 0, 31, 32, 33 and T - 1 that every head scores at 20; each query must see exactly the ones <= it."""
    D = 128
    qkv = _bf(B * T, H * D + 2 * D, seed=15)
    if strong:
        x = qkv.cpu()
        plant_strong_keys(x, B, T, [([h * D for h in range(H)], H * D, H * D + D)], D, [0, 31, 32, 33, T - 1], seed=2)
        qkv = x.to(DEV)
    out = E.op_attention_mqa(qkv, B, T, H)
    _close_attn(out, ref_causal_attention(qkv, B, T, H, 1), D)

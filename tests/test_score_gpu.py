"""Teacher-forced scoring on the device (`sv_score_tokens`, `Engine.score`, `StarVectorForCausalLM.score`, the im2svg loss):
the two new kernels against fp64 / fp32 torch, the whole path against the CPU oracle, and its agreement with the per-token
decode path at the 1B and 8B widths."""
import math

import pytest
import torch

from oracle.pipeline import OracleStarVector, OracleStarVectorV2
from starvector_b200 import engine as E
from starvector_b200.config import dims_1b, dims_8b, dims_tiny, dims_tiny_v2
from starvector_b200.engine import Engine, GenerationParams
from starvector_b200.modeling import StarVectorForCausalLM
from starvector_b200.weights import synthetic_images, synthetic_state_dict
from test_ops_gpu import _close_attn, plant_strong_keys
from test_score_logic import oracle_im2svg_loss

pytestmark = pytest.mark.gpu


def _close(got, ref, ulps=2.0, atol=2e-2):
    got, ref = got.float(), ref.float()
    tol = ulps * 2.0 ** -8 * ref.abs() + atol
    bad = (got - ref).abs() > tol
    assert not bool(bad.any()), f"{int(bad.sum())} / {bad.numel()} mismatches, max err {(got - ref).abs().max().item():.4f}"


def _err(a, ref):
    d = (a.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), d.mean().item()


def _as_accurate_as_bf16(engine_out, oracle_bf16, oracle_fp32, slack=2.0, floor=2e-2):
    e_max, e_mean = _err(engine_out, oracle_fp32)
    o_max, o_mean = _err(oracle_bf16, oracle_fp32)
    assert e_max <= slack * o_max + floor, f"max err {e_max:.4f} vs bf16-oracle {o_max:.4f}"
    assert e_mean <= slack * o_mean + floor / 10, f"mean err {e_mean:.5f} vs bf16-oracle {o_mean:.5f}"


def _gather_lp(logits, ids):
    return torch.log_softmax(logits.float(), dim=-1).gather(-1, ids.long().unsqueeze(-1)).squeeze(-1)


# ---- sv_op_lm_logprob --------------------------------------------------------------------------
@pytest.mark.parametrize("N", [500, 49156])
def test_lm_logprob_exact_inputs(N):
    """x in {-1,0,1}, w in quarter steps: every dot product and every bf16 logit is exact, whatever the summation order."""
    g = torch.Generator().manual_seed(N)
    M, K = 37, 128
    x = torch.randint(-1, 2, (M, K), generator=g).to(torch.bfloat16)
    w = (torch.randint(-2, 3, (N, K), generator=g) * 0.25).to(torch.bfloat16)
    w[N - 3] = w[N - 7]                                     # two tied maxima candidates
    x[0] = w[N - 3].float().sign().to(torch.bfloat16)       # row 0: its maximum sits on the tied pair
    tg = torch.randint(0, N, (M,), generator=g)
    tg[0], tg[1], tg[2] = N - 3, N - 7, N - 1               # a tied maximum and the last (partial) tile
    got = E.op_lm_logprob(x.cuda(), w.cuda(), tg.cuda()).cpu().double()
    logits = x.double() @ w.double().T
    assert torch.equal(logits, logits.to(torch.bfloat16).double())
    ref = torch.log_softmax(logits, dim=-1).gather(-1, tg.unsqueeze(-1)).squeeze(-1)
    assert (got - ref).abs().max().item() < 1e-5
    assert logits[0, N - 3] == logits[0].max() and logits[0, N - 7] == logits[0].max()


def test_lm_logprob_random_within_one_ulp():
    g = torch.Generator().manual_seed(7)
    M, N, K = 300, 1003, 256
    x = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.2).to(torch.bfloat16)
    tg = torch.randint(0, N, (M,), generator=g)
    got = E.op_lm_logprob(x.cuda(), w.cuda(), tg.cuda()).cpu().double()
    logits = (x.float() @ w.float().T).to(torch.bfloat16).double()
    ref = torch.log_softmax(logits, dim=-1).gather(-1, tg.unsqueeze(-1)).squeeze(-1)
    lt = logits.gather(-1, tg.unsqueeze(-1)).squeeze(-1).abs().clamp(min=1e-30)
    ulp = torch.exp2(torch.floor(torch.log2(lt)) - 7)
    assert bool(((got - ref).abs() <= ulp + 1e-4).all()), (got - ref).abs().max().item()


# ---- sv_op_attention_chunk ---------------------------------------------------------------------
def _attention_ref(qkv, B, seq, q0, nh, nkv, window):
    D = 128
    x = qkv.double().view(B, seq, (nh + 2 * nkv), D)
    q, k, v = x[:, :, :nh], x[:, :, nh:nh + nkv], x[:, :, nh + nkv:]
    grp = nh // nkv
    out = torch.empty(B, seq - q0, nh, D, dtype=torch.float64)
    for p in range(q0, seq):
        lo = max(0, p + 1 - window) if window > 0 else 0
        for h in range(nh):
            s = torch.einsum("bd,bkd->bk", q[:, p, h], k[:, lo:p + 1, h // grp])
            pr = torch.softmax(s / math.sqrt(D), dim=-1)
            out[:, p - q0, h] = torch.einsum("bk,bkd->bd", pr, v[:, lo:p + 1, h // grp])
    return out.reshape(B * (seq - q0), nh * D)


@pytest.mark.parametrize("q0,nh,nkv,window,strong", [(0, 16, 1, 0, False), (17, 16, 1, 0, False), (300, 16, 1, 0, False),
                                                     (17, 4, 2, 0, False), (300, 4, 2, 24, False), (40, 18, 2, 24, False),
                                                     (300, 4, 2, 24, True)],
                         ids=["0-16-1-0", "17-16-1-0", "300-16-1-0", "17-4-2-0", "300-4-2-24", "40-18-2-24", "300-4-2-24-strong"])
def test_attention_chunk(q0, nh, nkv, window, strong):
    """strong: keys every head scores at 20 at the window edges of the chunk's queries (and 31/32/33, the last position):
    each must count exactly for the queries whose window holds it."""
    B, seq = 2, q0 + 45
    g = torch.Generator().manual_seed(q0 * 7 + nh)
    qkv = torch.randn(B * seq, (nh + 2 * nkv) * 128, generator=g).to(torch.bfloat16)
    if strong:
        grp, D = nh // nkv, 128
        groups = [([(k * grp + j) * D for j in range(grp)], (nh + k) * D, (nh + nkv + k) * D) for k in range(nkv)]
        plant_strong_keys(qkv, B, seq, groups, D, [q0 - window, q0 - window + 1, q0 + 10 - window, 31, 32, 33, seq - 1], seed=3)
    got = E.op_attention_chunk(qkv.cuda(), B, seq, q0, nh, nkv, window).cpu()
    _close_attn(got, _attention_ref(qkv, B, seq, q0, nh, nkv, window), 128)


# ---- Engine.score against the oracle -----------------------------------------------------------
def _tiny(variant):
    if variant == "v2":
        d = dims_tiny_v2()
        sd = synthetic_state_dict(d, seed=0, init="randomized")
        return d, sd, OracleStarVectorV2(d, sd, dtype=torch.bfloat16), OracleStarVectorV2(d, sd, dtype=torch.float32)
    d = dims_tiny(adapter_norm=1 if variant == "v1_bn" else 0)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    pad = d.vocab - 4
    return (d, sd, OracleStarVector(d, sd, dtype=torch.bfloat16, pad_token_id=pad),
            OracleStarVector(d, sd, dtype=torch.float32, pad_token_id=pad))


PROMPT = [44, 78]


@pytest.mark.parametrize("variant", ["v1_ln", "v1_bn", "v2"])
def test_engine_score_matches_oracle(variant):
    d, sd, o16, o32 = _tiny(variant)
    B, T = 3, 40                                    # v2: the 24-token window is crossed inside the scored span
    eng = Engine(d, 0)
    eng.load_state_dict(sd)
    img = synthetic_images(d, B, seed=2)
    ids = torch.randint(0, d.vocab - 5, (B, T), generator=torch.Generator().manual_seed(3))
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT] * B))
    whole = eng.score(ids).cpu()
    ref32 = _gather_lp(o32.teacher_forced_logits(img.float(), PROMPT, ids)[:, :T], ids)
    ref16 = _gather_lp(o16.teacher_forced_logits(img, PROMPT, ids)[:, :T], ids)
    _as_accurate_as_bf16(whole, ref16, ref32)
    eng.encode_images(img)                          # the same T split over three ragged calls
    eng.prefill(torch.tensor([PROMPT] * B))
    parts = [eng.score(ids[:, a:b]).cpu() for a, b in ((0, 7), (7, 8), (8, T))]
    assert (torch.cat(parts, dim=1) - whole).abs().max().item() <= 1e-5
    eng.close()


def test_score_leaves_decode_state():
    d, sd, o16, o32 = _tiny("v1_ln")
    B, T = 3, 20
    eng = Engine(d, 0)
    eng.load_state_dict(sd)
    img = synthetic_images(d, B, seed=4)
    ids = torch.randint(0, d.vocab - 5, (B, T + 1), generator=torch.Generator().manual_seed(5))
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT] * B))
    eng.score(ids[:, :T])
    got = eng.decode_step(ids[:, T]).cpu()
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT] * B))
    for j in range(T + 1):
        stepped = eng.decode_step(ids[:, j]).cpu()
    ref32 = o32.teacher_forced_logits(img.float(), PROMPT, ids)[:, T + 1]
    ref16 = o16.teacher_forced_logits(img, PROMPT, ids)[:, T + 1]
    _as_accurate_as_bf16(got, ref16, ref32)
    _as_accurate_as_bf16(stepped, ref16, ref32)
    # the scored tokens extend the prefix: a generation continues from them
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT] * B))
    eng.score(ids[:, :T])
    out = eng.generate(GenerationParams(max_new_tokens=6, eos_token_id=None, pad_token_id=d.vocab - 4))
    assert out.shape == (B, 6)
    with pytest.raises(ValueError):
        eng.score(ids[:1])                           # batch != the current batch
    eng.close()


def test_facade_score_agrees_with_forward():
    d = dims_tiny()
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    m = StarVectorForCausalLM.from_config(dims=d, state_dict=sd)
    b, G, T = 2, 2, 12
    emb, _ = m.model.engine.encode_images(synthetic_images(d, b, seed=6), return_embeds=True)
    ids = torch.randint(0, d.vocab - 5, (b * G, T), generator=torch.Generator().manual_seed(7))
    mask = torch.ones(b * G, T, dtype=torch.long)
    mask[1, 9:] = 0                                 # a right-padded completion
    lp = m.score(emb, ids, num_generations=G, attention_mask=mask).cpu()
    logits = m.forward(emb, ids, num_generations=G, attention_mask=mask).logits.cpu()
    eng = m.model.engine
    prefix = eng.prefill_embeds(emb, return_logits=True).cpu().repeat(G, 1)     # t = 0 from the prefix logits
    ref = _gather_lp(torch.cat([prefix[:, None], logits[:, :-1]], dim=1), ids) * mask
    assert (lp[mask == 0] == 0).all()
    assert (lp - ref).abs().max().item() < 5e-2, (lp - ref).abs().max().item()
    assert (lp - ref).abs().mean().item() < 5e-3
    m.model.engine.close()


SVGS = ["<t11><t12><t13><t14><t15><t16><t17>", "<t21><t22>", "<t31><t32><t33><t34><t35>", "<t41>",
        "<t51><t52><t53><t54>"]


@pytest.mark.parametrize("variant", ["v1", "v2"])
def test_im2svg_loss_matches_oracle(variant):
    v2 = variant == "v2"
    d = dims_tiny_v2() if v2 else dims_tiny(max_batch=4)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    m = StarVectorForCausalLM.from_config(dims=d, state_dict=sd)
    svgs = ["<t11><t12><t13><t14>", "<t21><t22><t23><t24>"] if v2 else SVGS     # v2: equal lengths (left padding)
    img = synthetic_images(d, len(svgs), seed=8)
    loss = float(m.model({"image": img, "svg": svgs}))
    tok = m.model.svg_transformer.tokenizer
    if v2:
        o16, o32 = OracleStarVectorV2(d, sd, dtype=torch.bfloat16), OracleStarVectorV2(d, sd, dtype=torch.float32)
    else:
        o16 = OracleStarVector(d, sd, dtype=torch.bfloat16, pad_token_id=d.vocab - 4)
        o32 = OracleStarVector(d, sd, dtype=torch.float32, pad_token_id=d.vocab - 4)
    ml = m.model.max_length
    r16 = float(oracle_im2svg_loss(o16, img, svgs, tok, ml, v2=v2))
    r32 = float(oracle_im2svg_loss(o32, img.float(), svgs, tok, ml, v2=v2))
    assert abs(loss - r32) <= 2 * abs(r16 - r32) + 1e-3, (loss, r16, r32)
    m.model.engine.close()


# ---- full widths: several chunks per call, against the engine's own decode steps ----------------
def _score_vs_decode(d, B, T, seed):
    sd = synthetic_state_dict(d, seed=seed, device="cuda")
    eng = Engine(d, 0)
    eng.load_state_dict(sd)
    del sd
    g = torch.Generator().manual_seed(seed)
    emb = (torch.randn(B, 40, d.hidden, generator=g) * 0.5).to(torch.bfloat16).cuda()
    ids = torch.randint(0, d.vocab, (B, T), generator=g).cuda()
    first = eng.prefill_embeds(emb, return_logits=True)
    got = eng.score(ids)
    eng.prefill_embeds(emb)
    ref = torch.empty(B, T, device="cuda")
    prev = first
    for t in range(T):
        ref[:, t] = _gather_lp(prev, ids[:, t])
        prev = eng.decode_step(ids[:, t])
    e_max, e_mean = _err(got, ref)
    eng.close()
    return e_max, e_mean


# bf16 tolerance at full widths: the bound tests/test_full_1b_gpu.py holds the decode path's logits to against the oracle
FULL_MAX, FULL_MEAN = 0.25, 0.03


def test_full_1b_dims_several_chunks():
    e_max, e_mean = _score_vs_decode(dims_1b(max_batch=8, max_len=1200), B=8, T=1024, seed=11)
    assert e_max < FULL_MAX and e_mean < FULL_MEAN, (e_max, e_mean)


def test_8b_widths_sliding_window():
    d = dims_8b(max_batch=2, max_len=700)
    d.n_layer, d.sliding_window = 2, 512
    e_max, e_mean = _score_vs_decode(d, B=2, T=600, seed=12)
    assert e_max < FULL_MAX and e_mean < FULL_MEAN, (e_max, e_mean)

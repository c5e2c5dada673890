"""16 cache rows per GPU on the ring-GEMV graph decode path (two row groups of 8 sharing one weight stream).

Column n of an MMA does not depend on the other columns and every per-row reduction keeps its order, so a row decoded in a
16-row batch must carry exactly the bits it carries in an 8-row batch: the 16-row results are compared bit for bit with the
same images run as two 8-row calls on a max_batch=8 engine.  Beyond that: the oracle contract (tests/parity.py), the
per-op kernels, sampling streams, the device beam search against the host-stepped loop, and the Python surface."""
import dataclasses
import os

import pytest
import torch

from oracle.pipeline import OracleStarVector, OracleStarVectorV2
from parity import check_greedy_ids, oracle_greedy
from starvector_b200.beam_search import beam_search
from starvector_b200.config import ModelDims, dims_1b, dims_tiny
from starvector_b200.engine import Engine, GenerationParams
from starvector_b200.weights import synthetic_images, synthetic_state_dict

pytestmark = pytest.mark.gpu
PROMPT = [44, 78]


def _engine(d, sd, max_batch, env=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        eng = Engine(dataclasses.replace(d, max_batch=max_batch), 0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    eng.load_state_dict(sd)
    return eng


def _forced_id(step, row):
    return (7 * step + 3 * row) % 97 + 1


def _teacher_forced(eng, img, steps, row0=0, period=16):
    """Prefill logits, then the logits of `steps` teacher-forced decode steps: [1 + steps, B, V] bf16 values as fp32.
    Row b of this call is fed the ids of global row (row0 + b) % period, so split calls see the same histories."""
    eng.encode_images(img)
    out = [eng.prefill(torch.tensor([PROMPT] * img.shape[0]), return_logits=True).cpu()]
    for s in range(steps):
        ids = torch.tensor([_forced_id(s, (row0 + b) % period) for b in range(img.shape[0])], dtype=torch.int32)
        out.append(eng.decode_step(ids).cpu())
    return torch.stack(out)


def _greedy(eng, img, n_new, **kw):
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT] * img.shape[0]))
    return eng.generate(GenerationParams(max_new_tokens=n_new, pad_token_id=eng.dims.vocab - 4, **kw)).cpu()


@pytest.fixture(scope="module", params=[0, 1], ids=["layer_norm", "batch_norm"])
def tiny(request):
    d = dims_tiny(max_batch=16, adapter_norm=request.param)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    e16, e8 = _engine(d, sd, 16), _engine(d, sd, 8)
    yield d, sd, e16, e8, synthetic_images(d, 16, seed=1)
    e16.close()
    e8.close()


def test_describe_names_the_graph_path(tiny):
    d, sd, e16, e8, img = tiny
    assert "decode=ring-gemv-graph" in e16.describe() and "max_batch=16" in e16.describe()


def test_sixteen_rows_bitwise_equal_two_groups_of_eight(tiny):
    d, sd, e16, e8, img = tiny
    wide = _teacher_forced(e16, img, 6)
    two = torch.cat([_teacher_forced(e8, img[:8], 6), _teacher_forced(e8, img[8:], 6, row0=8)], dim=1)
    assert torch.equal(wide[0], two[0]), "prefill logits differ"
    for s in range(1, wide.shape[0]):
        assert torch.equal(wide[s], two[s]), f"decode step {s}: max diff {(wide[s] - two[s]).abs().max().item()}"
    g16 = _greedy(e16, img, 40, eos_token_id=None)
    g8 = torch.cat([_greedy(e8, img[:8], 40, eos_token_id=None), _greedy(e8, img[8:], 40, eos_token_id=None)])
    assert torch.equal(g16, g8)


def test_sixteen_rows_against_the_oracle_and_the_per_op_kernels(tiny):
    d, sd, e16, e8, img = tiny
    n_new = 24
    kw = dict(eos_token_id=0, stop_row0_only=False)
    got = _greedy(e16, img, n_new, **kw)
    o16 = OracleStarVector(d, sd, dtype=torch.bfloat16, pad_token_id=d.vocab - 4)
    ref_new, ref_logits = oracle_greedy(o16, img, PROMPT, (), n_new)
    tf = lambda ids: o16.teacher_forced_logits(img, PROMPT, ids)
    check_greedy_ids(got, ref_new, ref_logits, 0.05, tf, eos_token_id=o16.eos_token_id)
    legacy = _engine(d, sd, 16, {"SV_DECODE": "legacy"})
    try:
        assert "decode=legacy-kernels" in legacy.describe()
        lg = _greedy(legacy, img, n_new, **kw)
    finally:
        legacy.close()
    check_greedy_ids(lg, ref_new, ref_logits, 0.05, tf, eos_token_id=o16.eos_token_id)
    # token for token: the per-op kernels sum each dot product in another order, so the two bf16 logits of a near-tie may
    # swap; a row may only part where the oracle, over the shared history, puts the two tokens within 0.05 of each other
    assert lg.shape == got.shape
    for b in range(16):
        diff = (lg[b] != got[b]).nonzero()
        if len(diff):
            s = int(diff[0])
            row = o16.teacher_forced_logits(img[b: b + 1], PROMPT, got[b: b + 1, :s].long())[0, s]
            gap = abs(row[int(got[b, s])] - row[int(lg[b, s])]).item()
            assert gap < 0.05, f"row {b} step {s}: per-op {int(lg[b, s])} vs ring {int(got[b, s])}, oracle gap {gap:.4f}"


def test_sampling_rows_0_to_7_keep_their_stream(tiny):
    d, sd, e16, e8, img = tiny
    kw = dict(do_sample=True, temperature=0.9, top_p=0.8, seed=1234, eos_token_id=None)
    a = _greedy(e16, img, 32, **kw)
    b = _greedy(e16, img, 32, **kw)
    assert torch.equal(a, b), "a seeded 16-row run is not reproducible"
    c = _greedy(e8, img[:8], 32, **kw)
    assert torch.equal(a[:8], c)
    assert not torch.equal(a[8:], a[:8])
    # every token lies in the top-p nucleus of its step (HF TopPLogitsWarper after temperature): the mass of the strictly
    # more probable tokens is below top_p.  The logits are the engine's own, teacher-forced over the sampled sequence.
    e16.encode_images(img)
    logits = e16.prefill(torch.tensor([PROMPT] * 16), return_logits=True)
    for s in range(a.shape[1]):
        p = torch.softmax(logits.float().cpu() / 0.9, dim=-1)
        tok = a[:, s].long()
        above = torch.where(p > p.gather(1, tok[:, None]), p, torch.zeros(())).sum(1)
        assert (above < 0.8 + 1e-4).all(), (s, above.tolist())
        if s + 1 < a.shape[1]:
            logits = e16.decode_step(a[:, s].to(torch.int32))


@pytest.mark.parametrize("n_img,nb", [(8, 2), (4, 3), (2, 8)])
def test_device_beam_search_matches_the_host_loop(tiny, n_img, nb):
    d, sd, e16, e8, img = tiny
    kw = dict(num_beams=nb, max_new_tokens=14, eos_token_id=0, pad_token_id=d.vocab - 4, early_stopping=True)
    ids = torch.tensor([PROMPT] * n_img)
    dev = beam_search(e16, img[:n_img], ids, impl="device", **kw)
    host = beam_search(e16, img[:n_img], ids, impl="host", **kw)
    assert torch.equal(dev.cpu(), host.cpu()), (dev.tolist(), host.tolist())
    if nb == 2:      # the first 4 images through an 8-row engine: the same hypotheses
        four = beam_search(e8, img[:4], ids[:4], impl="device", **kw)
        assert torch.equal(four.cpu(), dev[:4].cpu()[:, : four.shape[1]])


def test_beam_sample_is_reproducible_and_keeps_the_8_row_stream(tiny):
    d, sd, e16, e8, img = tiny
    kw = dict(num_beams=2, max_new_tokens=14, do_sample=True, temperature=1.3, top_p=0.9, eos_token_id=0,
              pad_token_id=d.vocab - 4, seed=77, impl="device")
    ids = torch.tensor([PROMPT] * 8)
    a = beam_search(e16, img[:8], ids, **kw)
    b = beam_search(e16, img[:8], ids, **kw)
    assert torch.equal(a.cpu(), b.cpu())
    # images 0-3 are rows 0-7: the same Gumbel draws as on an 8-row engine, hence the same hypotheses
    four = beam_search(e8, img[:4], ids[:4], **kw)
    assert torch.equal(four.cpu(), a[:4].cpu()[:, : four.shape[1]])


def test_score_sixteen_rows_vs_two_calls(tiny):
    d, sd, e16, e8, img = tiny
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(1, d.vocab - 8, (16, 40), generator=g, dtype=torch.int32)
    e16.encode_images(img)
    e16.prefill(torch.tensor([PROMPT] * 16))
    wide = e16.score(ids).cpu()
    parts = []
    for h in (slice(0, 8), slice(8, 16)):
        e8.encode_images(img[h])
        e8.prefill(torch.tensor([PROMPT] * 8))
        parts.append(e8.score(ids[h]).cpu())
    assert (wide - torch.cat(parts)).abs().max().item() <= 1e-5


def test_limits(tiny):
    d, sd, e16, e8, img = tiny
    with pytest.raises(ValueError):
        Engine(dataclasses.replace(d, max_batch=17), 0)
    with pytest.raises(ValueError):
        beam_search(e16, img[:9], torch.tensor([PROMPT] * 9), num_beams=2, max_new_tokens=4, impl="device")
    with pytest.raises(ValueError):
        beam_search(e8, img[:5], torch.tensor([PROMPT] * 5), num_beams=2, max_new_tokens=4, impl="device")


def test_facade_reference_defaults_and_grpo():
    from starvector_b200.modeling import StarVectorForCausalLM

    d = dims_tiny(max_batch=16)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    m = StarVectorForCausalLM.from_config(dims=d, state_dict=sd)
    try:
        assert m.model.engine.dims.max_batch == 16
        img = synthetic_images(d, 8, seed=1)
        out = m.generate_im2svg({"image": img.to(torch.float16).cuda()}, max_length=d.query_length + 2 + 12)   # num_beams=2
        assert isinstance(out, list) and len(out) == 8 and all(isinstance(s, str) for s in out)
        r = m.model.generate_im2svg_grpo({"image": img[:2].cuda()}, num_return_sequences=8, max_length=d.query_length + 2 + 12,
                                         do_sample=True)
        assert len(r["raw_svg"]) == 16
    finally:
        m.model.engine.close()


def test_v2_sixteen_rows_on_the_per_op_kernels(golden_dir):
    g = torch.load(os.path.join(golden_dir, "tiny_v2_layer_norm.pt"), weights_only=False)
    d = ModelDims(**g["dims"])
    sd = synthetic_state_dict(d, seed=g["seed"], init=g["init"])
    img = synthetic_images(d, 16, seed=3)
    e16, e8 = _engine(d, sd, 16), _engine(d, sd, 8)
    try:
        assert "decode=legacy-kernels" in e16.describe()
        wide = _teacher_forced(e16, img, 4)
        two = torch.cat([_teacher_forced(e8, img[:8], 4), _teacher_forced(e8, img[8:], 4, row0=8)], dim=1)
        assert (wide - two).abs().max().item() <= 2e-2
        # the oracle's teacher-forced logits over the same history (prefill + the decode steps above)
        hist = torch.tensor([[_forced_id(s, b) for s in range(4)] for b in range(16)])
        o32 = OracleStarVectorV2(d, sd, dtype=torch.float32)
        emb, _, _ = o32.prepare_generation_inputs(img, PROMPT)
        x = torch.cat([emb, o32.llm.get_input_embeddings()(hist)], dim=1)
        with torch.no_grad():                                              # [16, 5, V]: after the prefix and each id
            ref = o32.llm(inputs_embeds=x, use_cache=False).logits[:, emb.shape[1] - 1:, :].float()
        got = wide.permute(1, 0, 2)
        ref = ref[:, : got.shape[1]]
        assert (got - ref).abs().max().item() <= 0.05 * ref.abs().max().item() + 0.05
    finally:
        e16.close()
        e8.close()


def test_full_1b_widths_two_layers_bitwise():
    d = dataclasses.replace(dims_1b(max_batch=16, max_len=512), n_layer=2)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    e16, e8 = _engine(d, sd, 16), _engine(d, sd, 8)
    try:
        four = synthetic_images(d, 8, seed=2)
        img = torch.cat([four, four])                     # 4 + 4 images, repeated to 16 rows
        wide = _teacher_forced(e16, img, 3, period=8)
        half = _teacher_forced(e8, img[:8], 3, period=8)
        assert torch.equal(wide[:, :8], half) and torch.equal(wide[:, 8:], half)
        g16 = _greedy(e16, img, 24, eos_token_id=None)
        g8 = _greedy(e8, img[:8], 24, eos_token_id=None)
        assert torch.equal(g16[:8], g8) and torch.equal(g16[8:], g8)
    finally:
        e16.close()
        e8.close()

"""Beam sessions (`sv_beam_session_*`, `Engine.beam_requests`, `generate_im2svg_continuous_beams`) on the GPU.

The contract: every request returns exactly the token ids and length of its one-image device beam search
(`beam_search(..., impl="device")`) with its own cap and seed, bit for bit, however the other groups are placed.  The
decode attention's partition comes from prefix + the session cap; every cap below gives the same partition as the session
cap (tiny v1: one 256-key cluster CTA; 1B: 4 CTAs; tiny v2 per-op path: one 32-key split bucket)."""
import pytest
import torch

from starvector_b200 import _lib
from starvector_b200.beam_search import beam_search
from starvector_b200.config import dims_1b, dims_tiny, dims_tiny_v2
from starvector_b200.continuous import ContinuousScheduler
from starvector_b200.engine import BeamSearchParams, Engine, GenerationParams
from starvector_b200.modeling import StarVectorForCausalLM
from starvector_b200.weights import synthetic_images, synthetic_state_dict

pytestmark = pytest.mark.gpu
PROMPT = [44, 78]


def _engine(d, sd):
    eng = Engine(d, 0)
    eng.load_state_dict(sd)
    return eng


def _random_head(d, sd, seed=3):
    """A randomised lm_head (as test_beam_gpu.py's fixture): beams reorder almost every step."""
    sd = dict(sd)
    g = torch.Generator().manual_seed(seed)
    sd["model.svg_transformer.transformer.lm_head.weight"] = (torch.randn(d.vocab, d.hidden, generator=g) * 0.2).to(torch.bfloat16)
    return sd


def _solo(eng, img, i, cap, seed, **kw):
    return beam_search(eng, img[i:i + 1], torch.tensor([PROMPT]), max_new_tokens=cap, seed=seed, impl="device", **kw).cpu()[0]


def _check(eng, img, caps, seeds, got, kw, which=None):
    for k in (range(len(got)) if which is None else which):
        ref = _solo(eng, img, k, caps[k], seeds[k], **kw)
        assert torch.equal(got[k].long(), ref), f"request {k}: session {got[k].tolist()[:10]}.. ({len(got[k])}) vs solo {ref.tolist()[:10]}.. ({len(ref)})"


@pytest.fixture(scope="module")
def tiny8():
    d = dims_tiny(max_batch=8)
    eng = _engine(d, _random_head(d, synthetic_state_dict(d, seed=0, init="randomized")))
    yield d, eng, synthetic_images(d, 11, seed=3)
    eng.close()


CASES = {
    "plain": dict(num_beams=2, eos_token_id=None),
    "quickstart": dict(num_beams=2, eos_token_id=None, length_penalty=-1.0, repetition_penalty=3.1),
    "early_false": dict(num_beams=2, eos_token_id=None, early_stopping=False, length_penalty=0.7),
    "never": dict(num_beams=2, eos_token_id=None, early_stopping="never", length_penalty=2.0),
    "beam_sample": dict(num_beams=2, eos_token_id=None, do_sample=True, temperature=0.9, top_p=0.9),
}


@pytest.mark.parametrize("case", list(CASES))
def test_requests_equal_one_image_searches(tiny8, case):
    d, eng, img = tiny8
    kw = dict(CASES[case], pad_token_id=d.vocab - 4)
    caps = [60, 17, 33, 60, 9, 41, 25, 60, 12, 50, 30]
    seeds = [700 + 13 * k for k in range(11)]
    order = []
    sch = ContinuousScheduler(eng, 8, num_beams=2)
    fill = kw["pad_token_id"] if kw.get("eos_token_id") is not None else -1
    params = BeamSearchParams(max_new_tokens=60, pad_token_id=fill, **{k: v for k, v in kw.items() if k != "pad_token_id"})
    got = sch.run(img, torch.tensor(PROMPT), params, max_new_tokens=caps, seeds=seeds, on_finish=lambda k, ids: order.append(k))
    assert sorted(order) == list(range(11)) and order != list(range(11))
    at = sch.stats["admit_step"]
    assert sch.stats["admissions"] > 2 and len(set(at)) > 2 and max(at) > 0     # groups joined mid-search of others
    _check(eng, img, caps, seeds, got, kw)


@pytest.mark.parametrize("nb,slots", [(3, 6), (4, 8)])
def test_wider_groups_with_eos_and_stop(tiny8, nb, slots):
    d, eng, img = tiny8
    free = _solo(eng, img, 0, 40, 0, num_beams=nb, eos_token_id=None, pad_token_id=d.vocab - 4).tolist()
    stop, eos = free[5:7], free[11]                 # a stop pair and an EOS id the model produces
    kw = dict(num_beams=nb, eos_token_id=eos, pad_token_id=d.vocab - 4, stop_ids=stop, length_penalty=1.3)
    caps = [40, 23, 31, 40, 15, 36, 28]
    got = eng.beam_requests(img[:7], torch.tensor(PROMPT), max_new_tokens=40, caps=caps, seed=5, slots=slots, **kw)
    assert any(len(g) < c for g, c in zip(got, caps)), "EOS / the stop pair should end some searches early"
    _check(eng, img, caps, [5 + k for k in range(7)], got, kw)


def test_full_1b_eight_groups():
    d = dims_1b(max_batch=16, max_len=1024)
    eng = _engine(d, synthetic_state_dict(d, seed=0))
    try:
        cap = 765                                       # prefix 259 + 510..765 keys: 4 CTAs per decode-attention cluster
        g = torch.Generator().manual_seed(1)
        caps = [int(c) for c in torch.randint(510, 600, (40,), generator=g)]
        caps[0], caps[1] = 765, 720
        img = synthetic_images(d, len(caps), seed=4)
        kw = dict(num_beams=2, eos_token_id=None, pad_token_id=d.vocab - 4, repetition_penalty=1.3)
        sch = ContinuousScheduler(eng, 16, num_beams=2)
        params = BeamSearchParams(max_new_tokens=cap, **dict(kw, pad_token_id=-1))
        got = sch.run(img, torch.tensor(PROMPT), params, max_new_tokens=caps, seeds=list(range(40)))
        assert [len(x) for x in got] == caps            # no EOS: every search runs to its cap
        at = sch.stats["admit_step"]
        for late in (8, 9):
            for early in (0, 1):
                assert at[late] - at[early] > 256, (late, early, at[late], at[early])
                assert at[early] + caps[early] - 1 > at[late], "the early request must still be decoding"
        _check(eng, img, caps, list(range(40)), got, kw, which=(0, 1, 8, 9))
    finally:
        eng.close()


def test_v2_sliding_window_per_op_path():
    d = dims_tiny_v2(max_batch=4)
    eng = _engine(d, _random_head(d, synthetic_state_dict(d, seed=0, init="randomized")))
    try:
        assert "legacy-kernels" in eng.describe()
        img = synthetic_images(d, 7, seed=2)
        caps = [60, 47, 55, 60, 49, 52, 58]             # prefix 18 + cap in (64, 96]: 3 key splits; the window is 24 keys
        kw = dict(num_beams=2, eos_token_id=None, pad_token_id=d.vocab - 4, repetition_penalty=1.2)
        got = eng.beam_requests(img, torch.tensor(PROMPT), max_new_tokens=60, caps=caps, seed=21, **kw)
        _check(eng, img, caps, [21 + k for k in range(7)], got, kw)
    finally:
        eng.close()


def test_facade_matches_one_image_calls():
    d = dims_tiny(max_batch=4)
    sd = _random_head(d, synthetic_state_dict(d, seed=0, init="randomized"))
    m = StarVectorForCausalLM.from_config(dims=d, state_dict=sd, max_batch=4)
    img = synthetic_images(d, 10, seed=6)
    kw = dict(max_length=d.query_length + 2 + 30, length_penalty=-1, repetition_penalty=3.1, seed=17)   # beam-sample
    got = m.generate_im2svg_continuous_beams({"image": img}, **kw)
    ref = [m.generate_im2svg({"image": img[i:i + 1]}, **dict(kw, seed=17 + i))[0] for i in range(10)]
    assert got == ref
    with pytest.raises(ValueError, match="generate_im2svg_continuous"):
        m.generate_im2svg_continuous_beams({"image": img}, num_beams=1, **kw)
    with pytest.raises(ValueError, match="num_return_sequences"):
        m.generate_im2svg_continuous_beams({"image": img}, num_return_sequences=2, **kw)


def test_refusals_and_state(tiny8):
    d, eng, img = tiny8
    kw = dict(num_beams=2, eos_token_id=None, pad_token_id=d.vocab - 4)
    before = _solo(eng, img, 1, 20, 3, **kw)
    with pytest.raises(ValueError, match="multiple"):
        eng.beam_session_begin(BeamSearchParams(2, 20), 5)
    with pytest.raises(ValueError, match="multiple"):
        eng.beam_session_begin(BeamSearchParams(1, 20), 4)
    eng.beam_session_begin(BeamSearchParams(2, 250), 4)        # prefix 19 + 250 > max_len 256: refused at admission
    try:
        with pytest.raises(ValueError, match="exceeds max_len"):
            eng.beam_session_admit(img[:1], torch.tensor([PROMPT]), [0])
    finally:
        eng.session_end()
    eng.beam_session_begin(BeamSearchParams(2, 20, eos_token_id=None, pad_token_id=-1), 4)
    try:
        with pytest.raises(_lib.EngineError, match="beam session"):
            eng.session_admit(img[:1], torch.tensor([PROMPT]), [0])
        with pytest.raises(_lib.EngineError):
            eng.encode_images(img[:2])
        with pytest.raises(_lib.EngineError):
            beam_search(eng, img[:1], torch.tensor([PROMPT]), max_new_tokens=20, impl="device", **kw)
        with pytest.raises(_lib.EngineError):
            eng.session_begin(GenerationParams(max_new_tokens=8), 4)
        eng.beam_session_admit(img[:1], torch.tensor([PROMPT]), [1])
        with pytest.raises(ValueError, match="busy"):
            eng.beam_session_admit(img[:1], torch.tensor([PROMPT]), [1])
    finally:
        eng.session_end()
    eng.session_begin(GenerationParams(max_new_tokens=8), 4)
    try:
        with pytest.raises(_lib.EngineError, match="sv_beam_session_begin"):
            eng.beam_session_admit(img[:1], torch.tensor([PROMPT]), [0])
    finally:
        eng.session_end()
    assert torch.equal(_solo(eng, img, 1, 20, 3, **kw), before)    # the rectangle search after the sessions
    caps = [20, 11, 17, 20, 8]
    runs = [eng.beam_requests(img[:5], torch.tensor(PROMPT), max_new_tokens=20, caps=caps, seed=3, slots=4, **kw)
            for _ in range(2)]                                       # the second replays the cached step graph
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    assert torch.equal(runs[0][1].long(), _solo(eng, img, 1, 11, 4, **kw))

"""Continuous batching (`sv_session_*`, `Engine.generate_requests`, `generate_im2svg_continuous`) on the GPU.

The contract: every request returns exactly the tokens a one-image `generate` of its image gives with the same parameters,
its own seed and the session cap (truncated to its own cap), bit for bit, however its neighbours in the session are
placed.  Each test runs more requests than there are slots, with caps that differ, so slots are refilled while other rows
are at other positions."""
import dataclasses
import os

import pytest
import torch

from oracle.pipeline import OracleStarVector
from parity import check_greedy_ids, oracle_greedy
from starvector_b200.config import dims_1b, dims_tiny, dims_tiny_v2
from starvector_b200.continuous import ContinuousScheduler
from starvector_b200.engine import Engine, GenerationParams
from starvector_b200.modeling import StarVectorForCausalLM
from starvector_b200.weights import synthetic_images, synthetic_state_dict

pytestmark = pytest.mark.gpu
PROMPT = [44, 78]


def _engine(d, sd):
    eng = Engine(d, 0)
    eng.load_state_dict(sd)
    return eng


def _params(d, cap, **kw):
    kw.setdefault("eos_token_id", None)
    return GenerationParams(max_new_tokens=cap, pad_token_id=d.vocab - 4, **kw)


def _solo(eng, img, i, params, seed=None):
    """Image i alone (a batch of one) through the rectangle path: its new tokens, [n]."""
    eng.encode_images(img[i:i + 1])
    eng.prefill(torch.tensor([PROMPT]))
    p = params if seed is None else dataclasses.replace(params, seed=seed)
    return eng.generate(p).cpu()[0]


def _check_all(eng, img, params, caps, got, seeds=None, n=1):
    for k, ids in enumerate(got):
        i = k // n
        ref = _solo(eng, img, i, params, None if seeds is None else seeds[k])
        ref = ref[: caps[i]]
        assert torch.equal(ids, ref), f"request {k}: session {ids.tolist()[:12]}... ({len(ids)}) vs solo {ref.tolist()[:12]}... ({len(ref)})"


@pytest.fixture(scope="module", params=[0, 1], ids=["layer_norm", "batch_norm"])
def tiny(request):
    d = dims_tiny(max_batch=4, adapter_norm=request.param)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    eng = _engine(d, sd)
    yield d, sd, eng, synthetic_images(d, 11, seed=3)
    eng.close()


def test_greedy_requests_equal_solo_runs(tiny):
    d, sd, eng, img = tiny
    cap = 48
    caps = [48, 5, 30, 12, 48, 1, 20, 33, 7, 48, 16]
    params = _params(d, cap)
    order = []
    got = eng.generate_requests(img, torch.tensor(PROMPT), params, max_new_tokens=caps, on_finish=lambda k, ids: order.append(k))
    assert sorted(order) == list(range(11)) and order != list(range(11)), "completion order should differ from request order"
    assert [len(g) for g in got] == caps
    _check_all(eng, img, params, caps, got)
    # one request against the CPU oracle (the reference path)
    o = OracleStarVector(d, sd, dtype=torch.bfloat16, pad_token_id=d.vocab - 4)
    ref_new, ref_logits = oracle_greedy(o, img[2:3], PROMPT, (), caps[2])
    check_greedy_ids(got[2][None], ref_new, ref_logits, 0.05, lambda ids: o.teacher_forced_logits(img[2:3], PROMPT, ids))


def test_eos_and_stop_sequence_finish_rows(tiny):
    d, sd, eng, img = tiny
    cap = 40
    # sampled rows (greedy rows of the synthetic tiny model repeat one token): request k draws with seed 900 + k
    base = _params(d, cap, do_sample=True, temperature=1.0, top_p=0.95, seed=900)
    free = [_solo(eng, img, i, base, seed=900 + i) for i in range(2)]
    eos = int(free[0][9])                              # request 0 stops at EOS by step 9 or earlier
    stop = (int(free[1][14]), int(free[1][15]))        # request 1 matches the stop pair by step 15 or earlier
    params = dataclasses.replace(base, eos_token_id=eos, stop_ids=stop, stop_row0_only=False)
    caps = [cap] * 11
    got = eng.generate_requests(img, torch.tensor(PROMPT), params)
    assert len(got[0]) <= 10 and len(got[1]) <= 16
    short = [g for g in got if len(g) < cap]
    assert len(short) >= 2 and len({len(g) for g in got}) >= 2, "rows should finish through the rule at different steps"
    for g in short:                                    # a row that ends before the cap ends with the rule's tokens
        assert int(g[-1]) == eos or tuple(int(t) for t in g[-2:]) == stop
    _check_all(eng, img, params, caps, got, seeds=[900 + k for k in range(11)])


def test_repetition_penalty_clears_seen_on_admission(tiny):
    d, sd, eng, img = tiny
    caps = [9, 4, 6, 3, 10, 5, 8, 2, 7, 6, 4]           # 11 requests on 4 slots: every slot is reused at least twice
    params = _params(d, 10, repetition_penalty=1.3)
    got = eng.generate_requests(img, torch.tensor(PROMPT), params, max_new_tokens=caps)
    _check_all(eng, img, params, caps, got)


def test_sampling_requests_use_their_own_seed(tiny):
    d, sd, eng, img = tiny
    caps = [24, 10, 18, 6, 24, 12, 3, 20, 9, 15, 24]
    params = _params(d, 24, do_sample=True, temperature=0.8, top_p=0.9, seed=777)
    got = eng.generate_requests(img, torch.tensor(PROMPT), params, max_new_tokens=caps)
    _check_all(eng, img, params, caps, got, seeds=[777 + k for k in range(11)])
    other = eng.generate_requests(img[:1], torch.tensor(PROMPT), params, seeds=[778])[0]
    assert not torch.equal(other, _solo(eng, img, 0, params, seed=777)), "two seeds gave the same tokens"


def test_n_completions_per_image(tiny):
    d, sd, eng, img = tiny
    params = _params(d, 20, do_sample=True, temperature=0.8, top_p=0.9, seed=5)
    got = eng.generate_requests(img[:3], torch.tensor(PROMPT), params, n=3, max_new_tokens=[20, 11, 16])
    assert len(got) == 9
    _check_all(eng, img, params, [20, 11, 16], got, seeds=[5 + k for k in range(9)], n=3)


def test_other_calls_refused_while_a_session_is_open(tiny):
    d, sd, eng, img = tiny
    eng.session_begin(_params(d, 8), 2)
    try:
        with pytest.raises(Exception, match="session"):
            eng.encode_images(img[:1])
        with pytest.raises(Exception, match="session"):
            eng.prefill(torch.tensor([PROMPT]))
        with pytest.raises(Exception, match="session"):
            eng.generate(_params(d, 8))
    finally:
        eng.session_end()
    eng.encode_images(img[:1])          # usable again
    eng.prefill(torch.tensor([PROMPT]))
    assert eng.generate(_params(d, 4)).shape == (1, 4)


def test_v2_sliding_window_per_op_path():
    d = dims_tiny_v2(max_batch=4)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    eng = _engine(d, sd)
    try:
        assert "legacy-kernels" in eng.describe()
        img = synthetic_images(d, 7, seed=2)
        caps = [60, 9, 41, 60, 17, 30, 60]               # the window is 24 keys: most rows run past it
        params = _params(d, 60, repetition_penalty=1.3)
        got = eng.generate_requests(img, torch.tensor(PROMPT), params, max_new_tokens=caps)
        _check_all(eng, img, params, caps, got)
    finally:
        eng.close()


def test_full_1b_sixteen_slots():
    d = dims_1b(max_batch=16, max_len=1024)
    sd = synthetic_state_dict(d, seed=0)
    eng = _engine(d, sd)
    try:
        cap = 560                                       # prefix 259 + 560 keys: 4 CTAs per decode-attention cluster
        g = torch.Generator().manual_seed(0)
        caps = [int(c) for c in torch.randint(16, 65, (112,), generator=g)]
        caps[0], caps[3], caps[110], caps[111] = 560, 500, 120, 200
        img = synthetic_images(d, len(caps), seed=4)
        params = _params(d, cap, repetition_penalty=1.3)
        sch = ContinuousScheduler(eng, 16)
        got = sch.run(img, torch.tensor(PROMPT), params, max_new_tokens=caps)
        assert [len(g) for g in got] == caps
        assert len(set(got[0].tolist())) > 20
        # 14 slots cycle short requests, so requests 110 and 111 join late: in the steps where they decode next to
        # requests 0 and 3, those rows are more than 256 keys further on
        at = sch.stats["admit_step"]
        for late in (110, 111):
            for early in (0, 3):
                assert at[late] - at[early] > 256, (late, early, at[late], at[early])
                assert at[early] + caps[early] - 1 > at[late], "the early request must still be decoding"
        for k in (0, 3, 110, 111):
            ref = _solo(eng, img, k, params)[: caps[k]]
            assert torch.equal(got[k], ref), f"request {k}"
    finally:
        eng.close()


def test_session_refreshes_slab_tiled_weights():
    """SV_TILED=1 streams slab-tiled copies of the decoder weights that are rebuilt after a weight load: a session on a
    freshly loaded engine, and again after new weights are loaded, must decode with the current weights."""
    d = dims_tiny(max_batch=4)
    old = os.environ.get("SV_TILED")
    os.environ["SV_TILED"] = "1"
    try:
        eng = _engine(d, synthetic_state_dict(d, seed=0, init="randomized"))
    finally:
        if old is None:
            os.environ.pop("SV_TILED")
        else:
            os.environ["SV_TILED"] = old
    try:
        if "weights=slab-tiled" not in eng.describe():
            pytest.skip(f"no slab-tiled ring weights on this engine: {eng.describe()}")
        img = synthetic_images(d, 6, seed=8)
        caps = [30, 7, 19, 30, 11, 24]
        params = _params(d, 30, do_sample=True, temperature=0.8, top_p=0.9, seed=31)
        seeds = [31 + k for k in range(6)]
        for sd_seed in (0, 1):
            if sd_seed:
                eng.load_state_dict(synthetic_state_dict(d, seed=sd_seed, init="randomized"))
            got = eng.generate_requests(img, torch.tensor(PROMPT), params, max_new_tokens=caps)   # before any solo run
            _check_all(eng, img, params, caps, got, seeds=seeds)
    finally:
        eng.close()


def test_facade_matches_one_image_calls():
    d = dims_tiny(max_batch=4)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    m = StarVectorForCausalLM.from_config(dims=d, state_dict=sd, max_batch=4)
    img = synthetic_images(d, 10, seed=6)
    kw = dict(use_nucleus_sampling=False, max_length=d.query_length + 2 + 30)
    got = m.generate_im2svg_continuous({"image": img}, **kw)
    ref = [m.generate_im2svg({"image": img[i:i + 1]}, num_beams=1, **kw)[0] for i in range(10)]
    assert got == ref
    kws = dict(use_nucleus_sampling=True, temperature=0.8, seed=11, max_length=d.query_length + 2 + 20)
    got = m.generate_im2svg_continuous({"image": img[:5]}, **kws)
    ref = [m.generate_im2svg({"image": img[i:i + 1]}, num_beams=1, **dict(kws, seed=11 + i))[0] for i in range(5)]
    assert got == ref
    with pytest.raises(NotImplementedError, match="beam"):
        m.generate_im2svg_continuous({"image": img}, num_beams=2, **kw)

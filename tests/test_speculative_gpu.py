"""Prompt-lookup speculative decoding on the GPU (`sv_generate_speculative`, DESIGN.md §7g): for every input a one-image
`generate` accepts, the speculative call returns the same tokens and length bit for bit; the drafts change the speed only."""
import os

import pytest
import torch

from starvector_b200.config import dims_1b, dims_tiny, dims_tiny_v2
from starvector_b200.engine import Engine, GenerationParams
from starvector_b200.modeling import StarVectorForCausalLM
from starvector_b200.weights import synthetic_images, synthetic_state_dict

from test_speculative_logic import draft

pytestmark = pytest.mark.gpu
PROMPT = [44, 78]


def _engine(d, sd, env=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        eng = Engine(d, 0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    eng.load_state_dict(sd)
    return eng


def _run(eng, img, n_new, on_tokens=None, **kw):
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT] * img.shape[0]))
    kw.setdefault("pad_token_id", eng.dims.vocab - 4)
    kw.setdefault("eos_token_id", None)
    out = eng.generate(GenerationParams(max_new_tokens=n_new, **kw), on_tokens=on_tokens).cpu()
    return out


def simulate_schedule(toks, k, g, eos, max_new):
    """The verify steps a speculative run of these (plain) tokens takes: each step drafts from the history with the host
    rule (sv_spec_draft_host), then emits one token plus the drafts that match the tokens, cut at the finish (the end of
    `toks`).  -> the counters sv_last_spec_stats reports."""
    n, m = len(toks), 1
    steps = drafted = accepted = 0
    while m < n:
        d = draft(toks[:m], k, g, -1 if eos is None else eos, max_new - m - 1)
        a = 0
        while a < len(d) and m + a + 1 < n and toks[m + a] == d[a]:
            a += 1
        steps, drafted, accepted, m = steps + 1, drafted + len(d), accepted + a, m + 1 + a
    return dict(steps=steps, drafted=drafted, accepted=accepted)


def _pair(eng, img, n_new, k, **kw):
    plain = _run(eng, img, n_new, **kw)
    spec = _run(eng, img, n_new, prompt_lookup_num_tokens=k, **kw)
    st = eng.last_spec_stats()
    if plain.shape[0] == 1:     # the device drafts are the host rule's: the schedule of the plain tokens
        want = simulate_schedule(plain[0].tolist(), k, kw.get("max_matching_ngram_size", 2), kw.get("eos_token_id"), n_new)
        assert {key: st[key] for key in want} == want, (st, want)
    return plain, spec, st


def _late_first(seq, width):
    """The width-gram of seq whose first occurrence starts latest (so that a stop on it falls deep inside the run)."""
    first = {}
    for j in range(len(seq) - width + 1):
        first.setdefault(tuple(seq[j:j + width]), j)
    return list(max(first, key=first.get))


@pytest.fixture(scope="module", params=[0, 1], ids=["layer_norm", "batch_norm"])
def tiny(request):
    d = dims_tiny(max_batch=8, adapter_norm=request.param)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    eng = _engine(d, sd)
    yield d, sd, eng, synthetic_images(d, 1, seed=1)
    eng.close()


CASES = {
    "greedy": dict(),
    "penalty1.3": dict(repetition_penalty=1.3),
    "penalty3.1": dict(repetition_penalty=3.1),
    "sample_seed7": dict(do_sample=True, temperature=0.9, top_p=0.9, seed=7),
    "sample_seed1234": dict(do_sample=True, temperature=0.7, top_p=1.0, seed=1234, repetition_penalty=1.3),
}


@pytest.mark.parametrize("k", [1, 3, 7])
@pytest.mark.parametrize("case", list(CASES))
def test_speculative_equals_plain(tiny, k, case):
    d, sd, eng, img = tiny
    n_new = d.max_len - d.query_length - len(PROMPT)
    plain, spec, st = _pair(eng, img, n_new, k, **CASES[case])
    assert torch.equal(plain, spec), (plain.tolist(), spec.tolist())
    assert st["steps"] >= 1 and st["accepted"] <= st["drafted"]
    assert st["steps"] + st["accepted"] == plain.shape[1] - 1          # every token after token 0 is a column's


@pytest.mark.parametrize("k", [1, 3, 7])
def test_eos_and_stop_inside_accepted_runs(tiny, k):
    d, sd, eng, img = tiny
    n_new = d.max_len - d.query_length - len(PROMPT)
    for kw in (dict(), dict(do_sample=True, temperature=0.8, top_p=0.9, seed=3)):
        ref = _run(eng, img, n_new, **kw)[0].tolist()
        eos = _late_first(ref, 1)[0]
        stop = _late_first(ref, 2)
        for extra in (dict(eos_token_id=eos), dict(stop_ids=stop), dict(eos_token_id=eos, stop_ids=stop)):
            plain, spec, st = _pair(eng, img, n_new, k, **kw, **extra)
            assert plain.shape[1] <= n_new and torch.equal(plain, spec), extra
        # a cap in the middle of a run
        for n in (1, 2, 17, 61):
            plain, spec, _ = _pair(eng, img, n, k, **kw)
            assert plain.shape[1] == n and torch.equal(plain, spec)


def test_drafts_are_accepted_and_rejected(tiny):
    d, sd, eng, img = tiny
    n_new = d.max_len - d.query_length - len(PROMPT)
    plain, spec, st = _pair(eng, img, n_new, 7)
    assert torch.equal(plain, spec)
    assert st["accepted"] > 0 and st["steps"] < n_new // 2, st        # the tiny model's greedy text repeats
    plain, spec, st = _pair(eng, img, n_new, 7, do_sample=True, temperature=1.5, top_p=1.0, seed=5)
    assert torch.equal(plain, spec)
    assert st["drafted"] > st["accepted"], st                          # a hot sampler rejects drafts


@pytest.mark.parametrize("k", [1, 3, 7])
def test_verify_columns_equal_successive_decode_steps(tiny, k):
    d, sd, eng, img = tiny
    ids = [(37 * c + 11) % d.vocab for c in range(k + 1)]
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT]))
    cols = eng.spec_verify_step(ids).cpu()
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT]))
    for c, t in enumerate(ids):
        step = eng.decode_step(torch.tensor([t]))[0].cpu()
        assert torch.equal(cols[c], step), f"column {c}: max diff {(cols[c] - step).abs().max().item()}"


def test_streaming_delivers_the_plain_tokens(tiny):
    d, sd, eng, img = tiny
    n_new = d.max_len - d.query_length - len(PROMPT)
    for kw in (dict(poll_interval=4), dict(poll_interval=16, do_sample=True, temperature=0.9, top_p=0.9, seed=11)):
        plain = _run(eng, img, n_new, **kw)
        chunks = []
        spec = _run(eng, img, n_new, on_tokens=lambda ids, first: chunks.append((first, ids.clone())) and False,
                    prompt_lookup_num_tokens=5, **kw)
        assert torch.equal(plain, spec)
        assert [f for f, _ in chunks] == [sum(c.shape[1] for _, c in chunks[:i]) for i in range(len(chunks))]
        assert torch.equal(torch.cat([c for _, c in chunks], dim=1), plain)


def test_refusals(tiny):
    d, sd, eng, img = tiny
    img2 = synthetic_images(d, 2, seed=1)
    with pytest.raises(NotImplementedError, match="one image"):
        _run(eng, img2, 8, prompt_lookup_num_tokens=3)
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens"):
        _run(eng, img, 8, prompt_lookup_num_tokens=d.max_batch)
    with pytest.raises(ValueError, match="max_matching_ngram_size"):
        _run(eng, img, 8, prompt_lookup_num_tokens=3, max_matching_ngram_size=0)
    eng.session_begin(GenerationParams(max_new_tokens=8), 2)
    try:
        with pytest.raises(NotImplementedError, match="session"):
            eng.generate(GenerationParams(max_new_tokens=8, prompt_lookup_num_tokens=3))
    finally:
        eng.session_end()
    legacy = _engine(d, sd, {"SV_DECODE": "legacy"})
    try:
        with pytest.raises(NotImplementedError, match="legacy"):
            _run(legacy, img, 8, prompt_lookup_num_tokens=3)
    finally:
        legacy.close()
    dv2 = dims_tiny_v2()
    v2 = _engine(dv2, synthetic_state_dict(dv2, seed=0, init="randomized"))
    try:
        with pytest.raises(NotImplementedError, match="v2"):
            _run(v2, synthetic_images(dv2, 1, seed=1), 8, prompt_lookup_num_tokens=3)
    finally:
        v2.close()
    flow = _engine(d, sd, {"SV_FLOW": "1"})
    try:
        assert "speculative decoding: graph path" in flow.describe()
        plain, spec, _ = _pair(flow, img, 64, 3)
        assert torch.equal(plain, spec)
    finally:
        flow.close()


def test_speculative_ngram_sizes(tiny):
    d, sd, eng, img = tiny
    n_new = d.max_len - d.query_length - len(PROMPT)
    for g in (1, 3, 8):
        plain, spec, st = _pair(eng, img, n_new, 4, max_matching_ngram_size=g)
        assert torch.equal(plain, spec)


# ---- facades -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    d = dims_tiny()
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    m = StarVectorForCausalLM.from_config(dims=d, state_dict=sd)
    yield d, m
    m.model.engine.close()


def test_facades(model):
    d, m = model
    img = synthetic_images(d, 2, seed=1)
    emb, _ = m.model.engine.encode_images(img, return_embeds=True)
    prompt = torch.tensor([m.model.svg_transformer.tokenizer("<svg")["input_ids"]] * 2)
    embeds = torch.cat([emb, m.model._get_embeddings(prompt)], dim=1)
    gen = m.model.svg_transformer.transformer.generate
    for kw in (dict(do_sample=False), dict(do_sample=True, top_p=0.9, temperature=0.8, seed=4)):
        kw.update(num_beams=1, max_length=embeds.shape[1] + 120)
        a = gen(inputs_embeds=embeds[:1], **kw)
        b = gen(inputs_embeds=embeds[:1], prompt_lookup_num_tokens=3, **kw)
        st = m.model.engine.last_spec_stats()
        assert st["steps"] + st["accepted"] == a.shape[1] - 1            # the speculative path ran
        c = gen(inputs_embeds=embeds[:1], prompt_lookup_num_tokens=2, max_matching_ngram_size=1, **kw)
        assert torch.equal(a.cpu(), b.cpu()) and torch.equal(a.cpu(), c.cpu())
    with pytest.raises(ValueError, match="assisted generate is only supported for batch_size = 1"):
        gen(inputs_embeds=embeds, prompt_lookup_num_tokens=3, max_length=embeds.shape[1] + 8)
    with pytest.warns(UserWarning, match="prompt_lookup_num_tokens"):
        a = gen(inputs_embeds=embeds[:1], num_beams=2, max_length=embeds.shape[1] + 8)
        b = gen(inputs_embeds=embeds[:1], num_beams=2, prompt_lookup_num_tokens=3, max_length=embeds.shape[1] + 8)
    assert torch.equal(a.cpu(), b.cpu())
    for kw in (dict(use_nucleus_sampling=False, num_beams=1), dict(use_nucleus_sampling=True, num_beams=1, seed=9),
               dict(num_beams=2)):
        kw.update(max_length=d.query_length + 2 + 100)
        for n in (1, 2):
            batch = {"image": img[:n].cuda()}
            a = m.generate_im2svg(batch, **kw)
            b = m.generate_im2svg(batch, prompt_lookup_num_tokens=10, **kw)     # a hint: clamped to max_batch - 1
            assert a == b, kw


# ---- StarVector-1B dimensions, synthetic weights -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sd_1b():
    return synthetic_state_dict(dims_1b(max_batch=8, max_len=1024), seed=0, init="randomized")


@pytest.mark.parametrize("max_batch,k", [(8, 7), (16, 15)])
def test_1b_speculative_equals_plain(sd_1b, max_batch, k):
    d = dims_1b(max_batch=max_batch, max_len=1024)
    eng = _engine(d, sd_1b)
    try:
        img = synthetic_images(d, 1, seed=2)
        n_new = 600
        assert d.query_length + len(PROMPT) + n_new <= d.max_len
        plain, spec, st = _pair(eng, img, n_new, k)
        assert plain.shape[1] == n_new and torch.equal(plain, spec)
        assert st["steps"] + st["accepted"] == n_new - 1
        ids = plain[0, :k + 1].tolist()                                 # the logits of every column, bit for bit
        eng.encode_images(img)
        eng.prefill(torch.tensor([PROMPT]))
        cols = eng.spec_verify_step(ids).cpu()
        eng.encode_images(img)
        eng.prefill(torch.tensor([PROMPT]))
        for c, t in enumerate(ids):
            assert torch.equal(cols[c], eng.decode_step(torch.tensor([t]))[0].cpu()), c
    finally:
        eng.close()


def test_1b_long_history_eight_cta_clusters():
    """1B widths with 2 layers, 4096 cache slots and a prefix + max_new > 2048: 8-CTA cluster attention, drafts searched
    over histories past both 1024-token strides, k = 15 on a 16-row engine; greedy with a repetition penalty and nucleus
    sampling.  Speculative = plain, and the counters = the host schedule of the plain tokens."""
    d = dims_1b(max_batch=16, max_len=4096)
    d.n_layer = 2
    eng = _engine(d, synthetic_state_dict(d, seed=0, init="randomized"))
    try:
        img = synthetic_images(d, 1, seed=2)
        n_new = 2300
        assert 2048 < d.query_length + len(PROMPT) + n_new <= d.max_len
        for kw in (dict(repetition_penalty=1.3), dict(do_sample=True, temperature=0.9, top_p=0.9, seed=7)):
            plain, spec, st = _pair(eng, img, n_new, 15, **kw)
            assert torch.equal(plain, spec), kw
            print(f"1b long history {kw}: {plain.shape[1]} tokens, stats {st}")
    finally:
        eng.close()

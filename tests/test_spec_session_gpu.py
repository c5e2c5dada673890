"""Prompt-lookup speculation inside continuous-batching sessions on the GPU (`sv_session_begin_speculative`, DESIGN.md
§7i): every request of a speculative session returns the tokens a plain session gives it, and so the tokens a one-image
`generate` gives, bit for bit; the drafts change the speed only."""
import ctypes as C
import dataclasses
import os

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200.config import dims_1b, dims_tiny, dims_tiny_v2
from starvector_b200.engine import Engine, GenerationParams, op_spec_session_select
from starvector_b200.modeling import StarVectorForCausalLM
from starvector_b200.weights import synthetic_images, synthetic_state_dict

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


def _params(d, cap, **kw):
    kw.setdefault("eos_token_id", None)
    return GenerationParams(max_new_tokens=cap, pad_token_id=d.vocab - 4, **kw)


def _solo(eng, img, i, params, seed):
    eng.encode_images(img[i:i + 1])
    eng.prefill(torch.tensor([PROMPT]))
    return eng.generate(dataclasses.replace(params, seed=seed, prompt_lookup_num_tokens=0)).cpu()[0]


def _both(eng, img, params, k, slots=None, **kw):
    """The same requests through a plain and a speculative session: (plain, spec, spec stats)."""
    from starvector_b200.continuous import ContinuousScheduler

    plain = eng.generate_requests(img, torch.tensor(PROMPT), dataclasses.replace(params, prompt_lookup_num_tokens=0),
                                  slots=slots, **kw)
    sched = ContinuousScheduler(eng, slots)
    spec = sched.run(img, torch.tensor(PROMPT), dataclasses.replace(params, prompt_lookup_num_tokens=k), **kw)
    return plain, spec, sched.stats.get("spec")


def _equal(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"request {i}: {x.tolist()[:12]} ({len(x)}) vs {y.tolist()[:12]} ({len(y)})"


@pytest.fixture(scope="module", params=[0, 1], ids=["layer_norm", "batch_norm"])
def tiny(request):
    d = dims_tiny(max_batch=8, adapter_norm=request.param)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    eng = _engine(d, sd)
    yield d, sd, eng, synthetic_images(d, 13, seed=3)
    eng.close()


CAPS = [48, 5, 30, 12, 48, 1, 20, 33, 7, 48, 16, 40, 9]


@pytest.mark.parametrize("k", [1, 3, 7])
def test_greedy_equals_plain_and_solo(tiny, k):
    """13 requests on 8 slots with ragged caps: rows are admitted while other rows have drafts in flight."""
    d, sd, eng, img = tiny
    for rp in (1.0, 1.3):
        params = _params(d, 48, repetition_penalty=rp)
        plain, spec, st = _both(eng, img, params, k, max_new_tokens=CAPS)
        _equal(plain, spec)
        assert [len(g) for g in spec] == CAPS
        assert st["accepted"] > 0 and st["steps"] < sum(CAPS) - len(CAPS)
        for i in (0, 2, 5, 12):
            assert torch.equal(spec[i], _solo(eng, img, i, params, params.seed + i)[:CAPS[i]])


@pytest.mark.parametrize("k", [1, 3, 7])
def test_sampling_with_own_seeds(tiny, k):
    d, sd, eng, img = tiny
    params = _params(d, 40, do_sample=True, temperature=0.8, top_p=0.9, seed=777, repetition_penalty=1.2)
    caps = [40, 10, 18, 6, 40, 12, 3, 20, 9, 15, 40, 25, 31]
    plain, spec, st = _both(eng, img, params, k, max_new_tokens=caps)
    _equal(plain, spec)
    for i in (0, 3, 11):
        assert torch.equal(spec[i], _solo(eng, img, i, params, 777 + i)[:caps[i]])


def test_eos_and_stop_inside_accepted_runs(tiny):
    """Greedy rows of the synthetic model repeat, so drafts are accepted in runs; an EOS and a stop pair picked from those
    runs end rows inside them (and a stop pair may straddle two verify steps)."""
    d, sd, eng, img = tiny
    base = _params(d, 40)
    free = [_solo(eng, img, i, base, base.seed + i) for i in range(3)]
    eos = int(free[0][12])
    stop = (int(free[1][20]), int(free[1][21]))
    params = dataclasses.replace(base, eos_token_id=eos, stop_ids=stop, stop_row0_only=False)
    for k in (3, 7):
        plain, spec, st = _both(eng, img, params, k)
        _equal(plain, spec)
        assert len(spec[0]) <= 13 and len(spec[1]) <= 22
    for i in range(3):
        assert torch.equal(spec[i], _solo(eng, img, i, params, params.seed + i))


def test_n_completions(tiny):
    d, sd, eng, img = tiny
    params = _params(d, 30, do_sample=True, temperature=0.8, top_p=0.9, seed=5)
    plain, spec, st = _both(eng, img[:5], params, 3, n=2, max_new_tokens=[30, 11, 16, 25, 4])
    _equal(plain, spec)


def test_drafting_is_real(tiny):
    d, sd, eng, img = tiny
    params = _params(d, 64)
    plain, spec, st = _both(eng, img[:2], params, 7)           # 2 rows, 8 slots: 6 spare columns
    _equal(plain, spec)
    tokens = sum(len(s) for s in spec)
    assert st["accepted"] > 0 and st["steps"] < tokens / 2
    # every slot busy and no row finishing before the others: no spare column, no draft
    plain, spec, st = _both(eng, img[:8], params, 3)
    _equal(plain, spec)
    assert st["drafted"] == 0 and st["accepted"] == 0


def test_engine_settings(tiny):
    d, sd, eng, img = tiny
    params = _params(d, 48, repetition_penalty=1.2)
    ref = eng.generate_requests(img, torch.tensor(PROMPT), params, max_new_tokens=CAPS)
    for env in ({"SV_TILED": "1"}, {"SV_FLOW": "1"}):
        other = _engine(d, sd, env)
        try:
            if "SV_FLOW" in env:
                assert "sessions, beam sessions and speculative decoding: graph path" in other.describe()
            _, spec, st = _both(other, img, params, 3, max_new_tokens=CAPS)
            _equal(ref, spec)
            assert st["accepted"] > 0
        finally:
            other.close()


def test_abi_refusals(tiny):
    d, sd, eng, img = tiny
    lib = _lib.load()
    cp = _params(d, 8).to_c()
    for k, g, code in ((0, 2, _lib.SV_ERR_INVALID), (8, 2, _lib.SV_ERR_INVALID), (3, 0, _lib.SV_ERR_INVALID)):
        sp = _lib.SpecParams(k, g)
        assert lib.sv_session_begin_speculative(eng._h, C.byref(cp), C.byref(sp), 8) == code
    sp = _lib.SpecParams(3, 2)
    assert lib.sv_session_begin_speculative(eng._h, C.byref(cp), C.byref(sp), 8) == 0
    try:
        assert lib.sv_session_begin_speculative(eng._h, C.byref(cp), C.byref(sp), 8) == _lib.SV_ERR_STATE
        out = torch.empty(1, 8, dtype=torch.int32, device="cuda")
        assert lib.sv_generate(eng._h, C.byref(cp), C.c_void_p(out.data_ptr()), None, None) == _lib.SV_ERR_STATE
    finally:
        assert lib.sv_session_end(eng._h) == 0
    assert lib.sv_session_spec_stats(eng._h, None, None, None) == _lib.SV_ERR_STATE
    for env, dd in (({"SV_DECODE": "legacy"}, d), ({}, dims_tiny_v2())):
        other = _engine(dd, sd if dd is d else synthetic_state_dict(dd, seed=0, init="randomized"), env)
        try:
            assert lib.sv_session_begin_speculative(other._h, C.byref(cp), C.byref(sp), 8) == _lib.SV_ERR_UNSUPPORTED
            # through the Python layer the hint is ignored there: a plain session, the same tokens
            params = _params(dd, 12)
            spec = other.generate_requests(synthetic_images(dd, 3, seed=1), torch.tensor(PROMPT),
                                           dataclasses.replace(params, prompt_lookup_num_tokens=3))
            plain = other.generate_requests(synthetic_images(dd, 3, seed=1), torch.tensor(PROMPT), params)
            _equal(plain, spec)
        finally:
            other.close()


def test_1b_widths_sixteen_slots_long_history():
    """StarVector-1B widths (2 layers), 16 slots, histories past 2048 keys: the 8-CTA cluster partition; greedy with a
    repetition penalty and nucleus sampling, speculative session = plain session."""
    d = dims_1b(max_batch=16, max_len=4096)
    d.n_layer = 2
    eng = _engine(d, synthetic_state_dict(d, seed=0, init="randomized"))
    try:
        img = synthetic_images(d, 5, seed=2)
        cap = 2300
        assert 2048 < d.query_length + len(PROMPT) + cap <= d.max_len
        caps = [2300, 700, 2300, 90, 1500]
        for kw in (dict(repetition_penalty=1.3), dict(do_sample=True, temperature=0.9, top_p=0.9, seed=7)):
            params = _params(d, cap, **kw)
            plain, spec, st = _both(eng, img, params, 15, slots=16, max_new_tokens=caps)
            _equal(plain, spec)
            print(f"1b 16 slots {kw}: stats {st}")
    finally:
        eng.close()


def test_one_launch_against_host_replay():
    """The three kernels one launch at a time at the real 1B vocabulary against sv_spec_session_tail_host."""
    d = dims_1b(max_batch=16)
    V, H, S, stride, tcap = d.vocab, 64, 6, 256, 2080
    g = torch.Generator().manual_seed(3)
    wte = (torch.randn(V, H, generator=g) * 0.1).to(torch.bfloat16).cuda()
    wpe = (torch.randn(1024, H, generator=g) * 0.1).to(torch.bfloat16).cuda()
    lib = _lib.load()
    for impl in (_lib.SV_SPEC_SESSION_GREEDY, _lib.SV_SPEC_SESSION_SAMPLE, _lib.SV_SPEC_SESSION_TAIL):
        params = _params(d, 200, eos_token_id=5, stop_ids=(11, 12), repetition_penalty=1.2, do_sample=True, temperature=0.9,
                         top_p=0.9)
        rows = _lib.SessionRows()
        hist = torch.randint(20, 30, (S, stride), generator=g, dtype=torch.int32)
        for r in range(S):
            rows.row_active[r] = int(r != 2)
            rows.row_step[r], rows.row_len[r], rows.row_max_new[r] = 30 + 7 * r, 300 + 7 * r, 200
            rows.row_seed[r] = 100 + r
        ss = _lib.SpecSessionState(ncols=S, k=3, max_ngram=2)
        cp = params.to_c()
        out_h = (C.c_int32 * (S * stride))(*hist.flatten().tolist())
        assert lib.sv_spec_session_tail_host(C.byref(cp), C.byref(rows), out_h, stride, C.byref(ss), 0, tcap) >= 1
        logits = (torch.randn(S, V, generator=g) * 3).to(torch.bfloat16).cuda()
        seen = torch.zeros(S, V, dtype=torch.uint8)
        for r in range(S):
            seen[r, hist[r, :rows.row_step[r]].long()] = 1
        # device: from the same state
        rows_d, ss_d = _lib.SessionRows.from_buffer_copy(rows), _lib.SpecSessionState.from_buffer_copy(ss)
        out_d, seen_d = torch.tensor(list(out_h), dtype=torch.int32).view(S, stride).cuda(), seen.cuda()
        x = torch.empty(S, H, dtype=torch.bfloat16, device="cuda")
        op_spec_session_select(impl, params, seen_d, out_d, torch.zeros(S, dtype=torch.int32, device="cuda"), rows_d, ss_d,
                               wte, wpe, x, 1024, tcap, logits=logits if impl != _lib.SV_SPEC_SESSION_TAIL else None)
        # host: the selected tokens the device wrote, then the same tail
        if impl == _lib.SV_SPEC_SESSION_TAIL:
            sel = list(ss.sel)
        else:
            sel = []
            lf = logits.float().cpu()
            for c in range(ss.n_live):
                r = ss.row[c]
                assert 0 <= ss_d.sel[c] < V if impl == _lib.SV_SPEC_SESSION_SAMPLE else True
                if impl == _lib.SV_SPEC_SESSION_GREEDY:
                    v = lf[c].clone()
                    pen = seen[r].bool().clone()
                    for j in range(1, ss.off[c] + 1):
                        pen[ss.tok[c - ss.off[c] + j]] = True
                    v[pen] = torch.where(v[pen] < 0, v[pen] * 1.2, v[pen] / 1.2)
                    sel.append(int(torch.argmax(v)))
                else:
                    sel.append(None)
        if impl == _lib.SV_SPEC_SESSION_SAMPLE:
            # the device's samples are checked against their own replay in the session tests; here the tail takes them
            sel = [ss_d.sel[c] for c in range(ss.n_live)]
        for c in range(len(sel)):
            ss.sel[c] = sel[c]
        assert lib.sv_spec_session_tail_host(C.byref(cp), C.byref(rows), out_h, stride, C.byref(ss), 1, tcap) >= 0
        if impl == _lib.SV_SPEC_SESSION_GREEDY:       # the greedy kernel keeps its selections in shared memory
            ss.sel = ss_d.sel
        assert bytes(rows) == bytes(rows_d), impl
        for f, _ in _lib.SpecSessionState._fields_:
            assert bytes(getattr(ss, f)) == bytes(getattr(ss_d, f)) if hasattr(getattr(ss, f), "_length_") else \
                getattr(ss, f) == getattr(ss_d, f), (impl, f)
        assert out_d.cpu().flatten().tolist() == list(out_h)
        # the next step's column inputs: wte[tok] + wpe[pos]
        ref = (wte[torch.tensor(list(ss.tok)[:S]).long().cuda()].float() + wpe[torch.tensor(list(ss.pos)[:S]).long().cuda()].float())
        assert torch.equal(x, ref.to(torch.bfloat16))


# ---- facade -----------------------------------------------------------------------------------------------------------
def test_facade_strings_do_not_change():
    """`generate_im2svg_continuous` gives the same strings with and without the hint; a v2 model given it runs plain."""
    for dims in (dims_tiny(max_batch=8), dims_tiny_v2()):
        m = StarVectorForCausalLM.from_config(dims=dims, state_dict=synthetic_state_dict(dims, seed=0, init="randomized"))
        try:
            img = synthetic_images(dims, 5, seed=4).cuda()
            for kw in (dict(use_nucleus_sampling=False), dict(use_nucleus_sampling=True, seed=3)):
                kw.update(max_length=dims.query_length + 2 + 60)
                plain = m.generate_im2svg_continuous({"image": img}, **kw)
                spec = m.generate_im2svg_continuous({"image": img}, prompt_lookup_num_tokens=3, max_matching_ngram_size=2, **kw)
                assert plain == spec, kw
        finally:
            m.model.engine.close()

"""CPU check of the device beam-search bookkeeping (csrc/sv_beam_core.h) at 16 cache rows: whole searches through the
library's host replays of the device stages over 8 images x 2 beams, 4 x 4 and 2 x 8, against HF generate(num_beams > 1)
and the torch loop (starvector_b200/beam_search.py); the beam-sample Gumbel stream of rows 0-7 is the 8-row engine's, and
no two (step, row, token) draws share a Philox counter.  No GPU: the library only has to load."""
import ctypes as C
import struct

import pytest
import torch

from oracle.pipeline import OracleStarVector
from starvector_b200 import _lib
from starvector_b200.beam_search import beam_search
from starvector_b200.config import dims_tiny
from starvector_b200.weights import synthetic_images, synthetic_state_dict
from test_beam_core import PROMPT, _fp, _ip, _SeededLogitsEngine
from test_beam_logic import OracleBackedEngine


def wide_core_beam_search(eng, image, prompt_ids, *, num_beams, max_new_tokens, length_penalty=1.0, repetition_penalty=1.0,
                          early_stopping=True, eos_token_id=0, pad_token_id=0, do_sample=False, temperature=1.0, top_p=1.0,
                          seed=0):
    """tests/test_beam_core.py's host loop for up to 16 rows: the same stages and state blob, read out with the 16-row entry
    point (the 8-row one keeps its contract)."""
    lib = _lib.load()
    B, nb = image.shape[0], num_beams
    R, K, V = B * nb, 2 * nb, eng.dims.vocab
    bp = _lib.BeamParams()
    bp.num_beams, bp.max_new_tokens, bp.do_sample = nb, max_new_tokens, int(do_sample)
    bp.early_stopping = 2 if early_stopping == "never" else int(bool(early_stopping))
    bp.temperature, bp.top_p, bp.repetition_penalty, bp.length_penalty = temperature, top_p, repetition_penalty, length_penalty
    bp.eos_token_id = -1 if eos_token_id is None else eos_token_id
    bp.pad_token_id = pad_token_id
    bp.seed = seed
    assert lib.sv_beam_params_check_rows(C.byref(bp), B, 16) == 0
    state = C.create_string_buffer(lib.sv_beam_state_bytes())
    prefix_len = eng.dims.query_length + prompt_ids.shape[1]
    assert lib.sv_beam_state_init_host(C.byref(bp), B, prefix_len, state) == 0
    stride = max_new_tokens
    run_seq = torch.full((2, R, stride), pad_token_id, dtype=torch.int32)
    fin_seq = torch.full((2, R, stride), pad_token_id, dtype=torch.int32)
    eng.encode_images(image.repeat_interleave(nb, dim=0))
    logits = eng.prefill(prompt_ids.repeat_interleave(nb, dim=0), return_logits=True)
    key, val = torch.empty(R, K, dtype=torch.float32), torch.empty(R, K, dtype=torch.float32)
    tok = torch.empty(R, K, dtype=torch.int32)
    nxt, src = torch.empty(R, dtype=torch.int32), torch.empty(R, dtype=torch.int32)
    parity, cur = C.c_int32(), C.c_int32()
    fin_len, scores = (C.c_int32 * 16)(), (C.c_float * 16)()
    cache_hi, step = prefix_len - 1, 0
    while True:
        lg = logits.float().contiguous()
        assert lib.sv_beam_state_read16_host(state, C.byref(parity), C.byref(cur), fin_len, None, scores) == 0
        for r in range(R):
            seq = run_seq[parity.value, r, : cur.value].contiguous()
            assert lib.sv_beam_row_candidates_host(C.byref(bp), _fp(lg[r]), V, _ip(seq), cur.value, float(scores[r]), step, r,
                                                   _fp(key[r]), _fp(val[r]), _ip(tok[r])) == 0
        cont = lib.sv_beam_step_host(C.byref(bp), B, V, stride, state, _fp(key), _fp(val), _ip(tok), _ip(run_seq), _ip(fin_seq),
                                     cache_hi, _ip(nxt), _ip(src), None)
        assert cont in (0, 1)
        step += 1
        cache_hi += 1
        if not cont:
            break
        eng.reorder_cache(src)
        logits = eng.decode_step(nxt)
    lib.sv_beam_state_read16_host(state, C.byref(parity), C.byref(cur), fin_len, None, None)
    n_gen = max(fin_len[b * nb] for b in range(B))
    return fin_seq[parity.value, 0::nb, :n_gen].long()


@pytest.fixture(scope="module")
def setup():
    torch.set_num_threads(1)
    d = dims_tiny(max_batch=16)
    sd = dict(synthetic_state_dict(d, seed=0, init="randomized"))
    g = torch.Generator().manual_seed(3)
    sd["model.svg_transformer.transformer.lm_head.weight"] = (torch.randn(d.vocab, d.hidden, generator=g) * 0.2).to(torch.bfloat16)
    o = OracleStarVector(d, sd, dtype=torch.float32, pad_token_id=d.vocab - 4)
    o.llm.lm_head.weight = torch.nn.Parameter(sd["model.svg_transformer.transformer.lm_head.weight"].float())
    return d, o, synthetic_images(d, 8, seed=1).float()


SHAPES = [(8, 2), (4, 4), (2, 8)]


@pytest.mark.parametrize("n_img,nb", SHAPES)
def test_sixteen_rows_match_hf(setup, n_img, nb):
    d, o, imgs = setup
    img, n_new = imgs[:n_img], 12
    kw = dict(use_nucleus_sampling=False, num_beams=nb, length_penalty=1.0, repetition_penalty=1.0,
              max_length=d.query_length + len(PROMPT) + n_new)
    ref = o.generate_im2svg_ids(img, PROMPT, (), **kw)[:, len(PROMPT):]
    got = wide_core_beam_search(OracleBackedEngine(o), img, torch.tensor([PROMPT] * n_img), num_beams=nb, max_new_tokens=n_new,
                                early_stopping=True, eos_token_id=0, pad_token_id=d.vocab - 4)
    assert got.shape == ref.shape and torch.equal(got, ref), (got.tolist(), ref.tolist())


@pytest.mark.parametrize("es", [True, False, "never"])
@pytest.mark.parametrize("n_img,nb", SHAPES)
def test_sixteen_rows_match_the_torch_loop(setup, n_img, nb, es):
    d, o, imgs = setup
    img = imgs[:n_img]
    kw = dict(num_beams=nb, max_new_tokens=10, length_penalty=-1.0 if es == "never" else 1.0, early_stopping=es, eos_token_id=0,
              pad_token_id=d.vocab - 4)
    ids = torch.tensor([PROMPT] * n_img)
    ref = beam_search(OracleBackedEngine(o), img, ids, **kw)
    got = wide_core_beam_search(OracleBackedEngine(o), img, ids, **kw)
    assert got.shape == ref.shape and torch.equal(got, ref), (got.tolist(), ref.tolist())


def test_sixteen_rows_at_the_1b_vocabulary():
    """Seeded bf16 logits over the real 49,156-entry vocabulary, 8 images x 2 beams, repetition penalty and "never"."""
    V, n_new, n_img = 49156, 24, 8
    kw = dict(num_beams=2, max_new_tokens=n_new, repetition_penalty=3.1, length_penalty=-1.0, early_stopping="never",
              eos_token_id=None, pad_token_id=49152)
    img, ids = torch.zeros(n_img, 3, 4, 4), torch.tensor([[1, 2]] * n_img)
    eng = _SeededLogitsEngine(V, 2)
    eng.dims.max_batch = 16
    ref = beam_search(eng, img, ids, **kw)
    eng = _SeededLogitsEngine(V, 2)
    got = wide_core_beam_search(eng, img, ids, **kw)
    assert ref.shape == (n_img, n_new) and torch.equal(got, ref)


def test_row_limits_and_the_8_row_readout():
    lib = _lib.load()
    bp = _lib.BeamParams()
    bp.num_beams, bp.max_new_tokens, bp.repetition_penalty, bp.temperature = 2, 4, 1.0, 1.0
    assert lib.sv_beam_params_check_rows(C.byref(bp), 8, 16) == 0
    assert lib.sv_beam_params_check_rows(C.byref(bp), 9, 16) != 0          # 18 rows
    assert lib.sv_beam_params_check_rows(C.byref(bp), 5, 8) != 0           # more rows than the engine holds
    assert lib.sv_beam_params_check_rows(C.byref(bp), 1, 17) != 0
    bp.num_beams = 9                                                      # 2 * num_beams candidates > 16
    assert lib.sv_beam_params_check_rows(C.byref(bp), 1, 16) != 0
    bp.num_beams = 2
    state = C.create_string_buffer(lib.sv_beam_state_bytes())
    assert lib.sv_beam_state_init_host(C.byref(bp), 8, 7, state) == 0
    fin8, sc8 = (C.c_int32 * 9)(*([-5] * 9)), (C.c_float * 9)(*([7.0] * 9))
    assert lib.sv_beam_state_read_host(state, None, None, fin8, sc8) == 0
    assert fin8[8] == -5 and sc8[8] == 7.0                                 # the 8-entry read-out writes 8 entries
    run = (C.c_float * 16)()
    assert lib.sv_beam_state_read16_host(state, None, None, None, None, run) == 0
    assert list(run) == [0.0, -1e9] * 8
    # the plan read-out holds rows 0-7: refused above 8 rows
    z = torch.zeros(64, dtype=torch.int32)
    kf = torch.zeros(16, 4)
    kt = torch.zeros(16, 4, dtype=torch.int32)
    seq = torch.zeros(2, 16, 4, dtype=torch.int32)
    assert lib.sv_beam_step_host(C.byref(bp), 8, 8, 4, state, _fp(kf), _fp(kf), _ip(kt), _ip(seq), _ip(seq.clone()), 6, None,
                                 None, _ip(z)) < 0


# ---- the beam-sample noise stream -----------------------------------------------------------------------------------------
M32 = 0xFFFFFFFF


def philox_u01(seed, c0, c1):
    """Python restatement of svbeam::philox_u01 (Philox4x32-10 -> (x0 >> 8 + 0.5) / 2^24, in fp32)."""
    k0, k1 = seed & M32, (seed >> 32) & M32
    x0, x1, x2, x3 = c0 & M32, c1 & M32, 0x4245414D, 0x53563032
    for _ in range(10):
        w0, w1 = 0xD2511F53 * x0, 0xCD9E8D57 * x2
        hi0, lo0, hi1, lo1 = w0 >> 32, w0 & M32, w1 >> 32, w1 & M32
        x0, x1, x2, x3 = hi1 ^ x1 ^ k0, lo1, hi0 ^ x3 ^ k1, lo0
        k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
    f32 = lambda v: struct.unpack("f", struct.pack("f", v))[0]
    return f32(f32(float(x0 >> 8) + 0.5) * f32(1.0 / 16777216.0))


def old_counter(step, row, token):
    """The 8-row engine's counter: (token, step * 8 + row)."""
    return token, step * 8 + row


def new_counter(step, row, token):
    return token + ((row >> 3) << 24), step * 8 + (row & 7)


_LIBM = C.CDLL("libm.so.6")
_LIBM.logf.restype, _LIBM.logf.argtypes = C.c_float, [C.c_float]


def gumbel(seed, c0, c1):
    """-logf(-logf(u)) in fp32 with the C library's logf, as the host replay computes it."""
    u = philox_u01(seed, c0, c1)
    return _LIBM.logf(-_LIBM.logf(u)) * -1.0


def _key_noise(seed, step, row, token, V=8):
    """The Gumbel noise the library adds to `token`: the ordering key of a row whose only finite score is that token
    (its log-prob is exactly 0 and the running score 0, so the key is the noise itself)."""
    lib = _lib.load()
    bp = _lib.BeamParams()
    bp.num_beams, bp.max_new_tokens, bp.do_sample = 2, 8, 1
    bp.temperature, bp.top_p, bp.repetition_penalty, bp.length_penalty = 1.0, 1.0, 1.0, 1.0
    bp.eos_token_id, bp.pad_token_id, bp.seed = -1, 0, seed
    logits = torch.full((V,), -1e30)
    logits[token] = 0.0
    key, val, tok = torch.empty(4), torch.empty(4), torch.empty(4, dtype=torch.int32)
    empty = torch.zeros(1, dtype=torch.int32)
    assert lib.sv_beam_row_candidates_host(C.byref(bp), _fp(logits), V, _ip(empty), 0, 0.0, step, row, _fp(key), _fp(val), _ip(tok)) == 0
    assert int(tok[0]) == token and float(val[0]) == 0.0
    return float(key[0])


@pytest.mark.parametrize("seed", [0, 12345, 2**40 + 7])
def test_gumbel_draws_follow_the_counter_bit_for_bit(seed):
    """Rows 0-7: the 8-row engine's counter (token, step * 8 + row); rows 8-15: (token + 2^24, step * 8 + row - 8).  The
    library's noise equals the restatement exactly, for several steps and tokens."""
    for step in (0, 1, 37):
        for row in range(16):
            for token in (0, 3, 7):
                c0, c1 = (old_counter if row < 8 else new_counter)(step, row, token)
                assert _key_noise(seed, step, row, token) == gumbel(seed, c0, c1), (step, row, token)
                if row < 8:
                    assert new_counter(step, row, token) == old_counter(step, row, token)


def test_no_two_draws_share_a_counter():
    """The library draws with new_counter (previous test); no two (step, row, token) with row < 16 share its value."""
    V = 49156
    seen = set()
    for step in range(64):
        for row in range(16):
            for token in (0, 1, V // 2, V - 1):
                c = new_counter(step, row, token)
                assert c not in seen, (step, row, token)
                seen.add(c)
    # the full argument: c1 fixes (step, row % 8), c0 fixes (row // 8, token) because token < 2^24
    assert V < 1 << 24
    for row in range(16):
        c0, c1 = new_counter(5, row, V - 1)
        assert (c1 // 8, c1 % 8, c0 >> 24, c0 & ((1 << 24) - 1)) == (5, row & 7, row >> 3, V - 1)

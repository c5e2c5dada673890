"""CPU tests of the host side: ABI surface, config/tokenizer/params plumbing, loud failure without a GPU."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200.config import StarVectorConfig, dims_1b, dims_tiny
from starvector_b200.engine import GenerationParams
from starvector_b200.tokenizer import SyntheticTokenizer
from starvector_b200.weights import synthetic_state_dict, weight_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "starvector_b200.h")).read()
    return set(re.findall(r"SV_API\s+[\w\s\*]+?\b(sv_\w+)\s*\(", text))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    declared = _header_symbols()
    assert declared, "no SV_API declarations parsed"
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (sv_\w+)", out))
    assert declared == exported, (declared ^ exported)
    assert declared == set(_lib.SIGNATURES), (declared ^ set(_lib.SIGNATURES))
    assert lib.sv_abi_version() == _lib.ABI_VERSION


def test_struct_layout_matches_header():
    assert C.sizeof(_lib.ModelDesc) == 22 * 4
    assert C.sizeof(_lib.GenParams) == 88 and _lib.GenParams.seed.offset == 72


def test_create_rejects_bad_descriptors_without_touching_cuda():
    lib = _lib.load()
    h = C.c_void_p()
    d = _lib.ModelDesc(variant=7)
    assert lib.sv_engine_create(C.byref(d), 0, C.byref(h)) == _lib.SV_ERR_UNSUPPORTED
    d = _lib.ModelDesc(variant=1, rope_theta=0.0)
    assert lib.sv_engine_create(C.byref(d), 0, C.byref(h)) == _lib.SV_ERR_INVALID
    assert b"rope_theta" in lib.sv_last_error(None)
    d = _lib.ModelDesc(vit_width=100, vit_heads=2)
    assert lib.sv_engine_create(C.byref(d), 0, C.byref(h)) == _lib.SV_ERR_INVALID


DECODE_OPS = ("sv_op_attention_decode", "sv_op_gemv_ring", "sv_op_ring_ntiles", "sv_op_ring_row_stride",
              "sv_op_rope_table", "sv_op_rope")


def test_decode_op_symbols_and_descriptor_layout():
    assert _lib.ABI_VERSION == 7                       # test hooks only: no existing entry point changed
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    for name in DECODE_OPS:
        assert name in _header_symbols() and name in _lib.SIGNATURES and name in exported, name
    # sv_op_ring: 7 pointers, 6 int32, float (+4 padding), 2 pointers, 4 int32, 3 pointers
    assert C.sizeof(_lib.OpRing) == 144
    assert (_lib.OpRing.ln_eps.offset, _lib.OpRing.kcache.offset, _lib.OpRing.n_head.offset,
            _lib.OpRing.pos_host.offset, _lib.OpRing.amax_idx.offset) == (80, 88, 104, 120, 136)


def _bad_decode_attention(**kw):
    a = dict(impl=0, per_row=0, lens=[5], n_head=16, n_kv=1, tcap=64, nsplit=2, window=0, ptr=0x10000)
    a.update(kw)
    lens = a["lens"]
    arr = (C.c_int32 * len(lens))(*lens)
    p = C.c_void_p(a["ptr"])
    lib = _lib.load()
    return lib.sv_op_attention_decode(a["impl"], a["per_row"], p, p, p, p, arr, len(lens), a["n_head"], a["n_kv"], a["tcap"],
                                      a["nsplit"], a["window"], None)


@pytest.mark.parametrize("kw", [dict(n_head=6, n_kv=4), dict(n_head=17, n_kv=1), dict(tcap=48), dict(lens=[0]),
                                dict(lens=[65]), dict(lens=[5, 6]), dict(lens=[1] * 17, per_row=1), dict(nsplit=0),
                                dict(nsplit=129), dict(impl=1, nsplit=9), dict(impl=2), dict(window=-1), dict(ptr=0x10008),
                                dict(ptr=0), dict(per_row=3), dict(per_row=2), dict(per_row=2, impl=1, window=4),
                                dict(per_row=2, impl=1, lens=[64]), dict(per_row=2, impl=1, lens=[3, -1]),
                                dict(per_row=2, impl=1, lens=[0] * 17)], ids=str)
def test_decode_attention_op_rejects_on_the_host(kw):
    """Checked before any CUDA call: these return SV_ERR_INVALID on a machine without a GPU too."""
    assert _bad_decode_attention(**kw) == _lib.SV_ERR_INVALID
    assert b"attention_decode" in _lib.load().sv_last_error(None)


@pytest.mark.parametrize("kw", [dict(K=48), dict(K=0), dict(B=0), dict(B=17), dict(N=0), dict(x=0x10008),
                                dict(w=0x10004), dict(ln=True, ln_b=0x10008), dict(ln=False, epi=1), dict(ln=False, epi=2),
                                dict(ln=True, K=4608, B=9), dict(ln=True, K=640, B=9), dict(ln=True, K=4608, epi=1),
                                dict(ln=True, epi=2, amax=False), dict(ln=True, epi=1, N=2304, tcap=40),
                                dict(ln=True, epi=1, N=2300), dict(ln=True, epi=1, N=2304, pos=[65]),
                                dict(ln=True, epi=1, N=2304, pos=[3, -1], per_row=1, B=2), dict(act=4), dict(epi=3),
                                dict(ln=True, epi=1, N=2304, per_row=3), dict(ln=True, epi=1, N=2304, per_row=2, n_live=-1),
                                dict(ln=True, epi=1, N=2304, pos=[3, 4], per_row=2, B=2, n_live=3),
                                dict(ln=True, epi=1, N=2304, pos=[3, 65], per_row=2, B=2, n_live=1),
                                dict(ln=True, epi=1, N=2304, pos=[64], per_row=2, n_live=0),
                                dict(ln=True, epi=1, N=2304, pos=[63, 63], per_row=2, B=2, n_live=2)], ids=str)
def test_gemv_ring_op_rejects_on_the_host(kw):
    """Among them the LayerNorm GEMV over K > 2048 with more than 8 rows, which has no ring kernel (the launcher would abort)."""
    a = dict(B=1, N=2304, K=2048, ln=False, epi=0, act=0, tcap=64, pos=[3], per_row=0, amax=True, n_live=1)
    a.update(kw)
    posl = a["pos"] + ([a["n_live"]] if a["per_row"] == 2 else [])      # the column map's n_live follows the positions
    pos = (C.c_int32 * len(posl))(*posl)
    o = _lib.OpRing(x=a.get("x", 0x10000), w=a.get("w", 0x20000), y=0x30000, B=a["B"], N=a["N"], K=a["K"], act=a["act"],
                    epi=a["epi"], n_head=16, n_kv=1, tcap=a["tcap"], per_row=a["per_row"], kcache=0x40000, vtcache=0x50000,
                    pos_host=C.cast(pos, C.POINTER(C.c_int32)))
    if a["ln"]:
        o.ln_w, o.ln_b = 0x60000, a.get("ln_b", 0x70000)
    if a["amax"]:
        o.amax_val, o.amax_idx = 0x80000, 0x90000
    lib = _lib.load()
    assert lib.sv_op_gemv_ring(C.byref(o), None) == _lib.SV_ERR_INVALID
    assert b"gemv_ring" in lib.sv_last_error(None)


def test_rope_ops_reject_on_the_host():
    lib = _lib.load()
    p = C.c_void_p(0x10000)
    assert lib.sv_op_rope_table(p, p, 16, 127, 1e4, None) == _lib.SV_ERR_INVALID
    assert lib.sv_op_rope_table(p, p, 0, 128, 1e4, None) == _lib.SV_ERR_INVALID
    assert lib.sv_op_rope_table(p, p, 16, 128, 0.0, None) == _lib.SV_ERR_INVALID
    two = (C.c_int32 * 2)(3, 4)
    assert lib.sv_op_rope(p, p, p, 2, 1, 4, 2, 16, 0, two, 0, None, None, 0, None) == _lib.SV_ERR_INVALID   # unequal, per_row 0
    assert lib.sv_op_rope(p, p, p, 2, 1, 4, 2, 16, 0, two, 1, p, p, 40, None) == _lib.SV_ERR_INVALID        # tcap % 32
    assert lib.sv_op_rope(p, p, p, 2, 1, 4, 2, 16, 0, None, 0, p, p, 64, None) == _lib.SV_ERR_INVALID      # append without pos
    assert lib.sv_op_rope(p, p, p, 2, 1, 4, 2, 16, -1, None, 0, None, None, 0, None) == _lib.SV_ERR_INVALID


PREFILL_OPS = ("sv_op_im2col", "sv_op_vit_assemble", "sv_op_adapter_norm", "sv_op_embed_prefix", "sv_op_attention_prefill",
               "sv_op_lm_logits")


def test_prefill_op_symbols():
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    for name in PREFILL_OPS:
        assert name in _header_symbols() and name in _lib.SIGNATURES and name in exported, name


_A, _U = 0x10000, 0x10008      # a 16-byte aligned and a misaligned device address (never dereferenced: rejected first)


def _prefill_op_calls():
    p, u, n = C.c_void_p(_A), C.c_void_p(_U), None
    RG, WG, AUTO = _lib.SV_LINEAR_ROWGROUP, _lib.SV_LINEAR_TCGEN05, _lib.SV_LINEAR_AUTO
    return {
        "layernorm null": ("sv_op_layernorm", (n, p, p, p, 4, 64, 1e-5, n)),
        "layernorm rows 0": ("sv_op_layernorm", (p, p, p, p, 0, 64, 1e-5, n)),
        "layernorm cols % 8": ("sv_op_layernorm", (p, p, p, p, 4, 60, 1e-5, n)),
        "layernorm misaligned": ("sv_op_layernorm", (u, p, p, p, 4, 64, 1e-5, n)),
        "linear null": ("sv_op_linear", (WG, p, n, n, n, p, 4, 64, 64, 0, n)),
        "linear M 0": ("sv_op_linear", (WG, p, p, n, n, p, 0, 64, 64, 0, n)),
        "linear N 0": ("sv_op_linear", (RG, p, p, n, n, p, 4, 0, 64, 0, n)),
        "linear rowgroup K % 32": ("sv_op_linear", (RG, p, p, n, n, p, 4, 64, 48, 0, n)),
        "linear wgmma N % 8": ("sv_op_linear", (WG, p, p, n, n, p, 64, 60, 64, 0, n)),
        "linear wgmma K % 64": ("sv_op_linear", (WG, p, p, n, n, p, 64, 64, 96, 0, n)),
        "linear auto no kernel": ("sv_op_linear", (AUTO, p, p, n, n, p, 64, 64, 48, 0, n)),
        "linear impl": ("sv_op_linear", (3, p, p, n, n, p, 4, 64, 64, 0, n)),
        "linear act": ("sv_op_linear", (RG, p, p, n, n, p, 4, 64, 64, 4, n)),
        "linear misaligned bias": ("sv_op_linear", (RG, p, p, u, n, p, 4, 64, 64, 0, n)),
        "attention_vit null": ("sv_op_attention_vit", (n, p, 1, 17, 2, n)),
        "attention_vit heads 0": ("sv_op_attention_vit", (p, p, 1, 17, 0, n)),
        "attention_vit seq 0": ("sv_op_attention_vit", (p, p, 1, 0, 2, n)),
        "im2col null": ("sv_op_im2col", (n, p, 1, 224, 14, 640, n)),
        "im2col image % patch": ("sv_op_im2col", (p, p, 1, 225, 14, 640, n)),
        "im2col kpad": ("sv_op_im2col", (p, p, 1, 224, 14, 587, n)),
        "im2col batch 0": ("sv_op_im2col", (p, p, 0, 224, 14, 640, n)),
        "vit_assemble null pos": ("sv_op_vit_assemble", (p, p, n, p, 1, 256, 1024, n)),
        "vit_assemble np 0": ("sv_op_vit_assemble", (p, p, p, p, 1, 0, 1024, n)),
        "adapter_norm kind": ("sv_op_adapter_norm", (2, p, p, p, p, p, p, 1, 257, 2048, 1e-5, n)),
        "adapter_norm tokens without stats": ("sv_op_adapter_norm", (1, p, p, p, n, p, p, 1, 257, 2048, 1e-5, n)),
        "adapter_norm slab % 8": ("sv_op_adapter_norm", (0, p, p, p, n, n, p, 1, 3, 3, 1e-5, n)),
        "adapter_norm misaligned": ("sv_op_adapter_norm", (0, u, p, p, n, n, p, 1, 257, 2048, 1e-5, n)),
        "adapter_norm q 0": ("sv_op_adapter_norm", (1, p, p, p, p, p, p, 1, 0, 2048, 1e-5, n)),
        "adapter_norm eps < 0": ("sv_op_adapter_norm", (0, p, p, p, n, n, p, 1, 257, 2048, -1.0, n)),
        "embed_prefix no visual": ("sv_op_embed_prefix", (n, p, p, p, p, 1, 257, 2, 2048, 49156, 0, 2, n)),
        "embed_prefix no ids": ("sv_op_embed_prefix", (p, n, p, p, p, 1, 257, 2, 2048, 49156, 0, 2, n)),
        "embed_prefix h % 8": ("sv_op_embed_prefix", (p, p, p, p, p, 1, 257, 2, 2044, 49156, 0, 2, n)),
        "embed_prefix empty": ("sv_op_embed_prefix", (p, p, p, p, p, 1, 0, 0, 2048, 49156, 0, 0, n)),
        "embed_prefix id_stride < p": ("sv_op_embed_prefix", (n, p, p, p, p, 1, 0, 16, 2048, 49156, 300, 8, n)),
        "embed_prefix pos0 < 0": ("sv_op_embed_prefix", (n, p, p, p, p, 1, 0, 16, 2048, 49156, -1, 16, n)),
        "embed_prefix misaligned wpe": ("sv_op_embed_prefix", (p, p, p, u, p, 1, 257, 2, 2048, 49156, 0, 2, n)),
        "attention_prefill null": ("sv_op_attention_prefill", (p, n, p, p, 1, 40, 16, 1, 64, 0, n)),
        "attention_prefill group": ("sv_op_attention_prefill", (p, p, p, p, 1, 40, 6, 4, 64, 0, n)),
        "attention_prefill group > 16": ("sv_op_attention_prefill", (p, p, p, p, 1, 40, 17, 1, 64, 0, n)),
        "attention_prefill tcap % 32": ("sv_op_attention_prefill", (p, p, p, p, 1, 40, 16, 1, 48, 0, n)),
        "attention_prefill seq > tcap": ("sv_op_attention_prefill", (p, p, p, p, 1, 65, 16, 1, 64, 0, n)),
        "attention_prefill window < 0": ("sv_op_attention_prefill", (p, p, p, p, 1, 40, 16, 1, 64, -1, n)),
        "attention_prefill misaligned": ("sv_op_attention_prefill", (p, u, p, p, 1, 40, 16, 1, 64, 0, n)),
        "attention_prefill batch 0": ("sv_op_attention_prefill", (p, p, p, p, 0, 40, 16, 1, 64, 0, n)),
        "attention_mqa heads > 16": ("sv_op_attention_mqa", (p, p, 1, 40, 17, n)),
        "lm_logits K % 64": ("sv_op_lm_logits", (p, p, p, 1, 49156, 2000, n)),
        "lm_logits M 0": ("sv_op_lm_logits", (p, p, p, 0, 49156, 2048, n)),
        "lm_logits null": ("sv_op_lm_logits", (p, p, n, 1, 49156, 2048, n)),
        "lm_logits misaligned": ("sv_op_lm_logits", (u, p, p, 1, 49156, 2048, n)),
    }


@pytest.mark.parametrize("case", sorted(_prefill_op_calls()))
def test_prefill_ops_reject_on_the_host(case):
    """The encoder / adapter / prefill entry points check every argument before any CUDA call: SV_ERR_INVALID here, on a
    machine without a GPU too."""
    name, args = _prefill_op_calls()[case]
    lib = _lib.load()
    assert getattr(lib, name)(*args) == _lib.SV_ERR_INVALID
    assert b"bad" in lib.sv_last_error(None)


SCORE_OPS = ("sv_op_attention_score", "sv_op_logits_logprob", "sv_op_lm_logprob", "sv_op_attention_chunk")


def test_score_op_symbols():
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    for name in SCORE_OPS:
        assert name in _header_symbols() and name in _lib.SIGNATURES and name in exported, name


def _score_op_calls():
    p, u, n = C.c_void_p(_A), C.c_void_p(_U), None
    u2 = C.c_void_p(_A + 2)                   # not even 4-byte aligned
    #              qkv kc vc out  B  C    pos0 nh nkv tcap  window
    ok = (p, p, p, p, 1, 256, 259, 16, 1, 544, 0, n)

    def score(i, v):
        a = list(ok)
        a[i] = v
        return ("sv_op_attention_score", tuple(a))
    return {
        "attention_score null qkv": score(0, n),
        "attention_score null vtcache": score(2, n),
        "attention_score null out": score(3, n),
        "attention_score batch 0": score(4, 0),
        "attention_score C 0": score(5, 0),
        "attention_score pos0 < 0": score(6, -1),
        "attention_score pos0 + C > tcap": score(6, 289),
        "attention_score group": ("sv_op_attention_score", (p, p, p, p, 1, 256, 259, 6, 4, 544, 0, n)),
        "attention_score group > 16": score(7, 17),
        "attention_score n_kv 0": score(8, 0),
        "attention_score tcap % 32": score(9, 528),
        "attention_score window < 0": score(10, -1),
        "attention_score misaligned qkv": score(0, u),
        "attention_score misaligned kcache": score(1, u),
        "attention_chunk q0 >= seq": ("sv_op_attention_chunk", (p, p, 1, 40, 40, 16, 1, 0, n)),
        "attention_chunk group": ("sv_op_attention_chunk", (p, p, 1, 40, 8, 6, 4, 0, n)),
        "lm_logprob null targets": ("sv_op_lm_logprob", (p, p, n, p, 4, 49156, 2048, n)),
        "lm_logprob null out": ("sv_op_lm_logprob", (p, p, p, n, 4, 49156, 2048, n)),
        "lm_logprob M 0": ("sv_op_lm_logprob", (p, p, p, p, 0, 49156, 2048, n)),
        "lm_logprob N 0": ("sv_op_lm_logprob", (p, p, p, p, 4, 0, 2048, n)),
        "lm_logprob K % 64": ("sv_op_lm_logprob", (p, p, p, p, 4, 49156, 2000, n)),
        "lm_logprob misaligned x": ("sv_op_lm_logprob", (u, p, p, p, 4, 49156, 2048, n)),
        "lm_logprob misaligned w": ("sv_op_lm_logprob", (p, u, p, p, 4, 49156, 2048, n)),
        "lm_logprob misaligned targets": ("sv_op_lm_logprob", (p, p, u2, p, 4, 49156, 2048, n)),
        "logits_logprob null logits": ("sv_op_logits_logprob", (n, p, p, 4, 49156, n)),
        "logits_logprob null targets": ("sv_op_logits_logprob", (p, n, p, 4, 49156, n)),
        "logits_logprob null out": ("sv_op_logits_logprob", (p, p, n, 4, 49156, n)),
        "logits_logprob M 0": ("sv_op_logits_logprob", (p, p, p, 0, 49156, n)),
        "logits_logprob vocab 0": ("sv_op_logits_logprob", (p, p, p, 4, 0, n)),
        "logits_logprob misaligned logits": ("sv_op_logits_logprob", (u, p, p, 4, 49156, n)),
        "logits_logprob misaligned out": ("sv_op_logits_logprob", (p, p, u2, 4, 49156, n)),
    }


@pytest.mark.parametrize("case", sorted(_score_op_calls()))
def test_score_ops_reject_on_the_host(case):
    """The scoring entry points check every argument before any CUDA call: SV_ERR_INVALID here, on a machine without a
    GPU too."""
    name, args = _score_op_calls()[case]
    lib = _lib.load()
    assert getattr(lib, name)(*args) == _lib.SV_ERR_INVALID
    assert b"bad" in lib.sv_last_error(None)


def test_select_op_symbols_and_descriptor_layout():
    assert _lib.ABI_VERSION == 7
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    for name in ("sv_op_select", "sv_op_beam_candidates"):
        assert name in _header_symbols() and name in _lib.SIGNATURES and name in exported, name
    # sv_op_select_args: 2 int32, pointer, 2 int32, sv_gen_params (88), 3 pointers, 3 int32 (+4), 7 pointers, uint32 (+4),
    # 6 pointers, 2 int32
    o = _lib.OpSelect
    assert C.sizeof(o) == 272
    assert (o.params.offset, o.seen.offset, o.out_stride.offset, o.counters_host.offset, o.row_seed_host.offset,
            o.row_mask.offset, o.event_host.offset, o.amax_val.offset, o.x.offset, o.h.offset) == (
        24, 112, 136, 152, 200, 208, 216, 224, 256, 264)


def _bad_select(**kw):
    a = dict(impl=0, per_row=0, B=2, vocab=500, nsteps=1, out_stride=8, advance_len=1, step=0, cur_len=5, logits=0x10000,
             seen=0x20000, out_ids=0x30000, next_ids=0x40000, do_sample=False, temperature=1.0, top_p=1.0, rp=1.0, stop=(),
             row_step=None, row_len=None, h=64, n_positions=16, wte=0x50000, wpe=0x60000, x=0x70000, amax=False,
             counters=True, event=True)
    a.update(kw)
    B = max(1, min(a["B"], 32))
    o = _lib.OpSelect(impl=a["impl"], per_row=a["per_row"], logits=a["logits"], vocab=a["vocab"], B=a["B"], seen=a["seen"],
                      out_ids=a["out_ids"], next_ids=a["next_ids"], out_stride=a["out_stride"], advance_len=a["advance_len"],
                      nsteps=a["nsteps"], row_mask=0xffff, h=a["h"], n_positions=a["n_positions"], wte=a["wte"],
                      wpe=a["wpe"], x=a["x"])
    p = o.params
    p.max_new_tokens, p.do_sample, p.temperature, p.top_p = 8, int(a["do_sample"]), a["temperature"], a["top_p"]
    p.repetition_penalty, p.eos_token_id, p.n_stop_ids = a["rp"], 0, a["stop"] if isinstance(a["stop"], int) else len(a["stop"])
    i32 = lambda v: C.cast((C.c_int32 * len(v))(*v), C.POINTER(C.c_int32))
    keep = [i32([a["step"], a["cur_len"], 0]), i32([1] * B), i32(a["row_len"] or [5] * B), i32(a["row_step"] or [0] * B),
            i32([1] * B), i32([8] * B), C.cast((C.c_uint64 * B)(), C.POINTER(C.c_uint64)), i32([0])]
    if a["counters"]:
        o.counters_host, o.unfinished_host = keep[0], keep[1]
    o.row_len_host, o.row_step_host, o.row_active_host, o.row_max_new_host, o.row_seed_host = keep[2:7]
    if a["event"]:
        o.event_host = keep[7]
    if a["amax"]:
        o.amax_val, o.amax_idx = 0x80000, 0x90000
    return _lib.load().sv_op_select(C.byref(o), None)


@pytest.mark.parametrize("kw", [dict(impl=3), dict(per_row=2), dict(logits=0), dict(seen=0), dict(out_ids=0), dict(next_ids=0),
                                dict(B=0), dict(B=17), dict(vocab=0), dict(nsteps=0), dict(advance_len=2),
                                dict(impl=1, temperature=0.0), dict(do_sample=True, temperature=-1.0), dict(impl=1, top_p=0.0),
                                dict(impl=1, top_p=1.5), dict(impl=1, top_p=float("nan")), dict(rp=0.0), dict(stop=9),
                                dict(stop=-1), dict(step=7, nsteps=2), dict(step=-1), dict(counters=False),
                                dict(per_row=1, row_step=[0, 8]), dict(per_row=1, row_len=[-1, 0]),
                                dict(per_row=1, event=False), dict(impl=2, h=60), dict(impl=2, h=0), dict(impl=2, wte=0),
                                dict(impl=2, x=0), dict(impl=2, n_positions=0), dict(impl=2, wpe=0x60008),
                                dict(impl=2, amax=True, nsteps=2)], ids=str)
def test_select_op_rejects_on_the_host(kw):
    assert _bad_select(**kw) == _lib.SV_ERR_INVALID
    assert b"bad select arguments" in _lib.load().sv_last_error(None)


def test_spec_select_op_symbol_and_descriptor_layout():
    assert _lib.ABI_VERSION == 7
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    assert "sv_op_spec_select" in _header_symbols() and "sv_op_spec_select" in _lib.SIGNATURES and "sv_op_spec_select" in exported
    # sv_spec_state = svspec::State: n_live, row[16], pos[16], tok[16], sel[16], ncols, k, max_ngram, steps, drafted, accepted
    s = _lib.SpecState
    assert C.sizeof(s) == 71 * 4
    assert (s.row.offset, s.pos.offset, s.tok.offset, s.sel.offset, s.ncols.offset, s.max_ngram.offset, s.accepted.offset) == (
        4, 68, 132, 196, 260, 268, 280)
    # sv_op_spec_args: int32 (+4), pointer, int32 (+4), sv_gen_params (88), 3 pointers, int32 (+4), 8 pointers, 2 int32
    o = _lib.OpSpec
    assert C.sizeof(o) == 208
    assert (o.logits.offset, o.vocab.offset, o.params.offset, o.seen.offset, o.out_stride.offset, o.gen_host.offset,
            o.spec_host.offset, o.amax_val.offset, o.wte.offset, o.x.offset, o.h.offset, o.n_positions.offset) == (
        8, 16, 24, 112, 136, 144, 152, 160, 176, 192, 200, 204)


def _bad_spec(**kw):
    a = dict(impl=0, vocab=500, out_stride=64, max_new=32, step=5, cur_len=40, done=0, logits=0x10000, seen=0x20000,
             out_ids=0x30000, next_ids=0x40000, temperature=1.0, top_p=1.0, rp=1.0, stop=0, h=64, n_positions=128,
             wte=0x50000, wpe=0x60000, x=0x70000, amax=None, gen=True, spec=True, ncols=4, n_live=2, k=None, max_ngram=2,
             pos=None, row=None)
    a.update(kw)
    st = _lib.SpecState(n_live=a["n_live"], ncols=a["ncols"], k=a["ncols"] - 1 if a["k"] is None else a["k"],
                        max_ngram=a["max_ngram"])
    for c in range(16):
        st.pos[c] = a["cur_len"] + min(c, 1) if a["pos"] is None else a["pos"]
        st.row[c] = 0 if a["row"] is None else a["row"]
    gen = (C.c_int32 * 4)(a["step"], a["cur_len"], a["done"], 1)
    o = _lib.OpSpec(impl=a["impl"], logits=a["logits"], vocab=a["vocab"], seen=a["seen"], out_ids=a["out_ids"],
                    next_ids=a["next_ids"], out_stride=a["out_stride"], wte=a["wte"], wpe=a["wpe"], x=a["x"], h=a["h"],
                    n_positions=a["n_positions"])
    if a["gen"]:
        o.gen_host = C.cast(gen, C.POINTER(C.c_int32))
    if a["spec"]:
        o.spec_host = C.pointer(st)
    p = o.params
    p.max_new_tokens, p.temperature, p.top_p, p.repetition_penalty = a["max_new"], a["temperature"], a["top_p"], a["rp"]
    p.eos_token_id, p.n_stop_ids = 0, a["stop"]
    if a["amax"] is not None:
        o.amax_val, o.amax_idx = a["amax"]
    return _lib.load().sv_op_spec_select(C.byref(o), None)


@pytest.mark.parametrize("kw", [dict(impl=3), dict(impl=-1), dict(seen=0), dict(out_ids=0), dict(next_ids=0), dict(gen=False),
                                dict(spec=False), dict(logits=0), dict(impl=1, logits=0), dict(vocab=0),
                                dict(impl=1, temperature=0.0), dict(impl=1, temperature=float("nan")), dict(impl=1, top_p=0.0),
                                dict(impl=1, top_p=1.5), dict(rp=0.0), dict(stop=9), dict(stop=-1), dict(max_new=0),
                                dict(max_new=65), dict(step=0), dict(step=64), dict(cur_len=-1), dict(cur_len=128, pos=3),
                                dict(wte=0), dict(x=0), dict(h=60), dict(h=0), dict(n_positions=0), dict(wpe=0x60008),
                                dict(x=0x70004), dict(amax=(0x80000, 0)), dict(amax=(0, 0x90000)),
                                dict(impl=1, amax=(0x80000, 0x90000)), dict(impl=2, amax=(0x80000, 0x90000)), dict(ncols=0),
                                dict(ncols=17, k=16), dict(n_live=-1), dict(n_live=5), dict(k=2), dict(ncols=1, k=1),
                                dict(max_ngram=0), dict(pos=-1), dict(pos=128), dict(row=1)], ids=str)
def test_spec_select_op_rejects_on_the_host(kw):
    """Checked before any CUDA call: these return SV_ERR_INVALID on a machine without a GPU too."""
    assert _bad_spec(**kw) == _lib.SV_ERR_INVALID
    assert b"bad spec_select arguments" in _lib.load().sv_last_error(None)


@pytest.mark.parametrize("kw", [dict(num_beams=1), dict(num_beams=9), dict(batch=9), dict(max_new_tokens=0), dict(n_stop_ids=9),
                                dict(early_stopping=3), dict(do_sample=1, temperature=0.0), dict(do_sample=1, top_p=0.0),
                                dict(do_sample=1, top_p=1.01), dict(repetition_penalty=0.0), dict(vocab=0), dict(vocab=60000),
                                dict(cur_len=-1), dict(cur_len=9), dict(logits=0), dict(run_seq=0), dict(cand=0),
                                dict(scores=False)], ids=str)
def test_beam_candidates_op_rejects_on_the_host(kw):
    """Among them a vocabulary whose fp32 row plus seen-bits exceed the shared memory the kernel may ask for."""
    a = dict(num_beams=2, batch=2, max_new_tokens=8, n_stop_ids=0, early_stopping=1, do_sample=0, temperature=1.0, top_p=1.0,
             repetition_penalty=1.0, vocab=500, cur_len=3, logits=0x10000, run_seq=0x20000, cand=0x30000, scores=True)
    a.update(kw)
    bp = _lib.BeamParams(**{k: a[k] for k in ("num_beams", "max_new_tokens", "n_stop_ids", "early_stopping", "do_sample",
                                              "temperature", "top_p", "repetition_penalty")}, length_penalty=1.0)
    scores = (C.c_float * 16)() if a["scores"] else None
    lib = _lib.load()
    c = C.c_void_p(a["cand"])
    assert lib.sv_op_beam_candidates(C.c_void_p(a["logits"]), a["vocab"], C.byref(bp), a["batch"], a["cur_len"], scores,
                                     C.c_void_p(a["run_seq"]), 8, c, c, c, None) == _lib.SV_ERR_INVALID
    assert b"bad beam_candidates arguments" in lib.sv_last_error(None)


BEAM_OPS = ("sv_op_beam_step", "sv_op_beam_kv_copy", "sv_op_kv_gather", "sv_op_session_admit")


def test_beam_op_symbols_and_struct_layouts():
    assert _lib.ABI_VERSION == 7
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    for name in BEAM_OPS:
        assert name in _header_symbols() and name in _lib.SIGNATURES and name in exported, name
    # sv_beam_state = svbeam::State: 4 int32, running_scores[16], beam_scores[16], is_finished[16], fin_len[16],
    # unsatisfied[16], div[16][16]
    s = _lib.BeamState
    assert C.sizeof(s) == 340 * 4 == _lib.load().sv_beam_state_bytes()
    assert (s.running_scores.offset, s.beam_scores.offset, s.is_finished.offset, s.fin_len.offset, s.unsatisfied.offset,
            s.div.offset) == (16, 80, 144, 208, 272, 336)
    # sv_beam_plan = svbeam::Plan: 7 x int32[16], copy_hi, cont, old_len
    p = _lib.BeamPlan
    assert C.sizeof(p) == 115 * 4
    assert (p.run_tok.offset, p.fin_old.offset, p.fin_parent.offset, p.fin_tok.offset, p.copy_src.offset, p.copy_lo.offset,
            p.copy_hi.offset, p.cont.offset, p.old_len.offset) == (64, 128, 192, 256, 320, 384, 448, 452, 456)
    # sv_op_beam_step_args: pointer, 4 int32, 10 pointers, 2 int32, 2 pointers
    o = _lib.OpBeamStep
    assert C.sizeof(o) == 128
    assert (o.batch.offset, o.advance.offset, o.state_host.offset, o.cand_tok.offset, o.fin_seq.offset, o.gen_host.offset,
            o.wpe.offset, o.x.offset, o.h.offset, o.n_positions.offset, o.next_ids.offset, o.plan_host.offset) == (
        8, 20, 24, 48, 64, 72, 88, 96, 104, 108, 112, 120)
    # sv_op_admit_args: 2 int32, 5 pointers, int32 (+4), pointer, 2 int32, 6 pointers
    a = _lib.OpAdmit
    assert C.sizeof(a) == 120
    assert (a.slot_host.offset, a.seed_host.offset, a.seen.offset, a.vocab.offset, a.out_ids.offset, a.out_stride.offset,
            a.pad_id.offset, a.row_len_host.offset, a.row_seed_host.offset, a.event_host.offset) == (
        8, 32, 40, 48, 56, 64, 68, 72, 104, 112)


def test_beam_state_struct_is_the_host_replay_blob():
    """sv_beam_state_init_host writes svbeam::State: read through the ctypes mirror, every field sits where it should."""
    lib = _lib.load()
    bp = _lib.BeamParams(num_beams=4, max_new_tokens=8, temperature=1.0, repetition_penalty=1.0, length_penalty=1.0)
    s = _lib.BeamState()
    C.memset(C.byref(s), 0x55, C.sizeof(s))
    assert lib.sv_beam_state_init_host(C.byref(bp), 4, 261, C.byref(s)) == 0
    assert (s.cur_len, s.done, s.parity, s.pad_) == (0, 0, 0, 0)
    assert list(s.running_scores) == [0.0 if r % 4 == 0 else -1e9 for r in range(16)]
    assert list(s.beam_scores) == [-1e9] * 16
    assert list(s.is_finished) == [0] * 16 and list(s.fin_len) == [0] * 16 and list(s.unsatisfied) == [1] * 16
    assert all(list(row) == [261] * 16 for row in s.div)


def _bad_beam_step(**kw):
    a = dict(num_beams=2, batch=2, vocab=500, seq_stride=64, advance=1, cur_len=5, parity=0, fin_len=0, gen_cur=300, h=64,
             n_positions=512, wpe=0x60000, x=0x70000, null=None, descriptor=True)
    a.update(kw)
    bp = _lib.BeamParams(num_beams=a["num_beams"], max_new_tokens=64, early_stopping=1, temperature=1.0, repetition_penalty=1.0,
                         length_penalty=1.0)
    st = _lib.BeamState(cur_len=a["cur_len"], parity=a["parity"])
    st.fin_len[1] = a["fin_len"]
    plan = _lib.BeamPlan()
    gen = (C.c_int32 * 2)(a["gen_cur"], 0)
    o = _lib.OpBeamStep(params=C.pointer(bp), batch=a["batch"], vocab=a["vocab"], seq_stride=a["seq_stride"],
                        advance=a["advance"], state_host=C.pointer(st), cand_key=0x10000, cand_val=0x11000, cand_tok=0x12000,
                        run_seq=0x20000, fin_seq=0x30000, gen_host=C.cast(gen, C.POINTER(C.c_int32)), wte=0x50000,
                        wpe=a["wpe"], x=a["x"], h=a["h"], n_positions=a["n_positions"], next_ids=0x40000,
                        plan_host=C.pointer(plan))
    if a["null"]:
        setattr(o, a["null"], None)
    return _lib.load().sv_op_beam_step(C.byref(o) if a["descriptor"] else None, None)


@pytest.mark.parametrize("kw", [dict(descriptor=False), dict(null="params"), dict(null="state_host"), dict(null="cand_key"),
                                dict(null="cand_val"), dict(null="cand_tok"), dict(null="run_seq"), dict(null="fin_seq"),
                                dict(null="gen_host"), dict(null="wte"), dict(null="x"), dict(null="next_ids"),
                                dict(null="plan_host"), dict(num_beams=1), dict(num_beams=9), dict(batch=9), dict(batch=0),
                                dict(vocab=0), dict(seq_stride=0), dict(advance=2), dict(advance=-1), dict(h=60), dict(h=0),
                                dict(n_positions=0), dict(wpe=0x60008), dict(x=0x70004), dict(gen_cur=-1),
                                dict(cur_len=64), dict(cur_len=-1), dict(parity=2), dict(fin_len=65), dict(fin_len=-1)],
                         ids=str)
def test_beam_step_op_rejects_on_the_host(kw):
    """Checked before any CUDA call: these return SV_ERR_INVALID on a machine without a GPU too."""
    assert _bad_beam_step(**kw) == _lib.SV_ERR_INVALID
    assert b"bad beam_step arguments" in _lib.load().sv_last_error(None)


def _bad_kv_copy(**kw):
    a = dict(k=0x10000, v=0x20000, n_layer=2, rows=4, n_kv=2, tcap=64, stride=None, plan=True, copy_hi=40, src=1, lo=30)
    a.update(kw)
    stride = a["rows"] * a["n_kv"] * a["tcap"] * 128 if a["stride"] is None else a["stride"]
    plan = _lib.BeamPlan(copy_hi=a["copy_hi"], cont=1)
    for r in range(16):
        plan.copy_src[r], plan.copy_lo[r] = -1, 0
    plan.copy_src[0], plan.copy_lo[0] = a["src"], a["lo"]
    return _lib.load().sv_op_beam_kv_copy(C.c_void_p(a["k"]), C.c_void_p(a["v"]), stride, a["n_layer"], a["rows"], a["n_kv"],
                                          a["tcap"], C.byref(plan) if a["plan"] else None, None)


@pytest.mark.parametrize("kw", [dict(k=0), dict(v=0), dict(plan=False), dict(n_layer=0), dict(rows=0), dict(rows=17),
                                dict(n_kv=0), dict(tcap=48), dict(tcap=0), dict(stride=4 * 2 * 64 * 128 - 8), dict(stride=65540),
                                dict(k=0x10008), dict(v=0x20002), dict(copy_hi=64), dict(src=4), dict(src=-2),
                                dict(lo=-1)], ids=str)
def test_beam_kv_copy_op_rejects_on_the_host(kw):
    assert _bad_kv_copy(**kw) == _lib.SV_ERR_INVALID
    assert b"bad beam_kv_copy arguments" in _lib.load().sv_last_error(None)


@pytest.mark.parametrize("kw", [dict(ks=0), dict(vs=0), dict(kd=0), dict(vd=0), dict(rows=0), dict(rows=17), dict(n_kv=0),
                                dict(tcap=48), dict(len=0), dict(len=65), dict(ks=0x10008), dict(vd=0x40004)], ids=str)
def test_kv_gather_op_rejects_on_the_host(kw):
    a = dict(ks=0x10000, vs=0x20000, kd=0x30000, vd=0x40000, rows=4, n_kv=2, tcap=64, len=64)
    a.update(kw)
    lib = _lib.load()
    assert lib.sv_op_kv_gather(*(C.c_void_p(a[n]) for n in ("ks", "vs", "kd", "vd")), None, a["rows"], a["n_kv"], a["tcap"],
                               a["len"], None) == _lib.SV_ERR_INVALID
    assert b"bad kv_gather arguments" in lib.sv_last_error(None)


@pytest.mark.parametrize("kw", [dict(descriptor=False), dict(null="slot_host"), dict(null="len_host"), dict(null="max_new_host"),
                                dict(null="seed_host"), dict(null="seen"), dict(null="out_ids"), dict(null="row_len_host"),
                                dict(null="row_seed_host"), dict(null="event_host"), dict(S=0), dict(S=17), dict(k=0),
                                dict(k=5), dict(vocab=0), dict(out_stride=0), dict(slots=[1, 1]), dict(slots=[0, 4]),
                                dict(slots=[-1, 0]), dict(lens=[3, -1])], ids=str)
def test_session_admit_op_rejects_on_the_host(kw):
    a = dict(k=2, S=4, slots=[2, 0], lens=[7, 7], vocab=500, out_stride=64, null=None, descriptor=True)
    a.update(kw)
    i32p = C.POINTER(C.c_int32)
    arr = lambda v, t=C.c_int32: (t * max(16, len(v)))(*v)
    keep = [arr(a["slots"]), arr(a["lens"]), arr([8] * 16), arr([1] * 16, C.c_uint64), arr([0] * 16), arr([0] * 16, C.c_uint64)]
    o = _lib.OpAdmit(k=a["k"], S=a["S"], slot_host=C.cast(keep[0], i32p), len_host=C.cast(keep[1], i32p),
                     max_new_host=C.cast(keep[2], i32p), seed_host=C.cast(keep[3], C.POINTER(C.c_uint64)), seen=0x10000,
                     vocab=a["vocab"], out_ids=0x20000, out_stride=a["out_stride"], pad_id=0,
                     row_seed_host=C.cast(keep[5], C.POINTER(C.c_uint64)), event_host=C.cast(keep[4], i32p))
    for n in ("row_len_host", "row_step_host", "row_active_host", "row_max_new_host"):
        setattr(o, n, C.cast(keep[4], i32p))
    if a["null"]:
        setattr(o, a["null"], None)
    lib = _lib.load()
    assert lib.sv_op_session_admit(C.byref(o) if a["descriptor"] else None, None) == _lib.SV_ERR_INVALID
    assert b"bad session_admit arguments" in lib.sv_last_error(None)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_engine_fails_loudly_without_gpu():
    from starvector_b200.engine import Engine

    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        Engine(dims_tiny())
    lib = _lib.load()
    h = C.c_void_p()
    t = dims_tiny()
    d = _lib.ModelDesc(image_size=t.image_size, patch_size=t.patch_size, vit_width=t.vit_width, vit_layers=1,
                       vit_heads=t.vit_heads, vit_mlp=t.vit_mlp, hidden=t.hidden, n_layer=1, n_head=t.n_head,
                       n_kv_head=1, head_dim=128, n_inner=t.n_inner, n_positions=64, vocab=500, ln_eps=1e-5,
                       max_batch=1, max_len=64)
    assert lib.sv_engine_create(C.byref(d), 0, C.byref(h)) == _lib.SV_ERR_CUDA
    assert b"no CPU fallback" in lib.sv_last_error(None)


def test_1b_dimensions_match_survey():
    d = dims_1b()
    assert d.query_length == 257 and d.patch_k == 588 and d.patch_k_padded == 640
    assert d.decoder_weight_bytes() == 2_240_876_544          # SURVEY.md §8d `W`
    assert d.kv_bytes_per_token() == 12_288
    n = sum(int(torch.tensor(s).prod()) for _, s, _ in weight_shapes(d))
    assert 1.42e9 < n < 1.45e9                                  # ViT 290.6M + adapter ~7.3M(+norm) + decoder 1137M


def test_config_roundtrip_and_dims():
    c = StarVectorConfig()
    d = c.to_dims(max_batch=2, max_len=4096)
    assert (d.hidden, d.n_layer, d.vocab, d.max_len) == (2048, 24, 49156, 4096)
    d8 = StarVectorConfig(starcoder_model_name="bigcode/starcoder2-7b", image_encoder_type="siglip_384", image_size=384,
                          hidden_size=4608, num_attention_heads=36, max_length=16384).to_dims(max_batch=2)
    assert (d8.variant, d8.query_length, d8.hidden, d8.n_kv_head, d8.sliding_window) == (1, 576, 4608, 4, 4096)
    assert d8.decoder_weight_bytes() == 14_347_893_760 and d8.kv_bytes_per_token() == 65_536   # SURVEY.md §8d (8B)
    c2 = StarVectorConfig(**{k: v for k, v in c.to_dict().items() if k not in ("model_type", "_name_or_path")})
    assert c2.hidden_size == c.hidden_size


def test_synthetic_tokenizer_roundtrip():
    t = SyntheticTokenizer(49156)
    assert t("<svg", add_special_tokens=False)["input_ids"] == [44, 5678]
    assert t.pad_token_id == 49152 and t.eos_token_id == 0
    ids = t(["<svg"] * 3, return_tensors="pt")["input_ids"]
    assert ids.shape == (3, 2)
    s = t.batch_decode([[44, 5678, 9, 10, 1245, 7, 29, 0, 49152]])[0]
    assert s == "<svg<t9><t10></svg>" and t.encode(s) == [44, 5678, 9, 10, 1245, 7, 29]


def test_generation_params_to_c():
    p = GenerationParams(max_new_tokens=7, do_sample=True, temperature=0.8, top_p=0.9, repetition_penalty=3.1,
                         eos_token_id=None, pad_token_id=49152, stop_ids=[1, 2, 3], seed=5).to_c()
    assert (p.max_new_tokens, p.do_sample, p.eos_token_id, p.n_stop_ids, list(p.stop_ids)[:3]) == (7, 1, -1, 3, [1, 2, 3])
    with pytest.raises(ValueError):
        GenerationParams(max_new_tokens=1, stop_ids=list(range(9))).to_c()


def test_state_dict_names_follow_reference_tree():
    sd = synthetic_state_dict(dims_tiny(), seed=0)
    assert "model.image_encoder.visual_encoder.transformer.resblocks.0.attn.in_proj_weight" in sd
    assert "model.image_projection.norm.weight" in sd
    assert sd["model.svg_transformer.transformer.lm_head.weight"] is sd["model.svg_transformer.transformer.transformer.wte.weight"]


def test_real_tokenizer_directory_is_prepared_like_the_reference(tmp_path):
    """llm/starcoder.py:40-53: eos/pad added when missing, the three start tokens appended; the facade's calls on it."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, trainers
    from transformers import PreTrainedTokenizerFast

    from starvector_b200.tokenizer import load_tokenizer

    tk = Tokenizer(models.BPE(unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tk.decoder = decoders.ByteLevel()
    corpus = ['<svg xmlns="http://www.w3.org/2000/svg" viewBox="0 0 24 24"><path d="M12 2L2 7l10 5 10-5z"/></svg>'] * 4
    tk.train_from_iterator(corpus, trainers.BpeTrainer(vocab_size=120, special_tokens=["<unk>"]))
    PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>").save_pretrained(str(tmp_path))
    tok = load_tokenizer(str(tmp_path), vocab_size=500)
    assert not isinstance(tok, SyntheticTokenizer)
    assert tok.eos_token == "[EOS]" and tok.pad_token == "[PAD]" and tok.eos_token_id != tok.pad_token_id
    for t in ("<svg-start>", "<image-start>", "<caption-start>"):
        assert len(tok.encode(t)) == 1
    stop = tok("</svg>", add_special_tokens=False)["input_ids"]                 # starvector_base.py:226
    prompt = tok(["<svg"] * 2, add_special_tokens=False, return_tensors="pt", padding="longest", truncation=True)["input_ids"]
    assert prompt.shape[0] == 2 and 1 <= len(stop) <= 8
    ids = prompt[0].tolist() + tok(' viewBox="0 0 24 24">')["input_ids"] + stop + [tok.eos_token_id, tok.pad_token_id]
    assert tok.batch_decode([ids], skip_special_tokens=True)[0] == '<svg viewBox="0 0 24 24"></svg>'
    assert isinstance(load_tokenizer(None, 500), SyntheticTokenizer)
    assert isinstance(load_tokenizer(str(tmp_path / "missing"), 500), SyntheticTokenizer)


def test_checkpoint_directory_round_trip(tmp_path):
    """write_checkpoint -> read_checkpoint: config fields, every tensor bit for bit, tied lm_head stored once, shards merged."""
    from safetensors.torch import save_file

    from starvector_b200.config import StarVectorConfig, dims_tiny
    from starvector_b200.modeling import read_checkpoint, write_checkpoint
    from starvector_b200.weights import synthetic_state_dict

    d = dims_tiny()
    sd = dict(synthetic_state_dict(d, seed=0, init="randomized"))
    cfg = StarVectorConfig(max_length_train=100, image_size=d.image_size)
    write_checkpoint(str(tmp_path), cfg, sd)
    cfg2, sd2 = read_checkpoint(str(tmp_path))
    assert cfg2.to_dict() == {**cfg.to_dict(), "_name_or_path": str(tmp_path)} or cfg2.max_length_train == 100
    stored = {k for k in sd if not k.endswith("lm_head.weight")}
    assert set(sd2) == stored and all(torch.equal(sd2[k], sd[k]) for k in stored)
    # a second shard is merged in
    save_file({"extra.tensor": torch.arange(4, dtype=torch.float32)}, str(tmp_path / "model-00002.safetensors"))
    assert "extra.tensor" in read_checkpoint(str(tmp_path))[1]
    with pytest.raises(FileNotFoundError):
        read_checkpoint(str(tmp_path / "nowhere"))
    (tmp_path / "empty").mkdir()
    (tmp_path / "empty" / "config.json").write_text((tmp_path / "config.json").read_text())
    with pytest.raises(FileNotFoundError):
        read_checkpoint(str(tmp_path / "empty"))


def test_untied_lm_head_survives_a_checkpoint_round_trip(tmp_path):
    """The reference always re-ties (train/util.py:68-77); the engine also takes an un-tied head, so saving must keep it."""
    from starvector_b200.config import StarVectorConfig
    from starvector_b200.modeling import read_checkpoint, write_checkpoint

    d = dims_tiny()
    sd = dict(synthetic_state_dict(d, seed=0))
    head = "model.svg_transformer.transformer.lm_head.weight"
    write_checkpoint(str(tmp_path / "tied"), StarVectorConfig(), sd)
    assert head not in read_checkpoint(str(tmp_path / "tied"))[1]                 # equal to wte: stored once
    sd[head] = sd[head].clone() + 1.0
    write_checkpoint(str(tmp_path / "untied"), StarVectorConfig(), sd)
    back = read_checkpoint(str(tmp_path / "untied"))[1]
    assert head in back and torch.equal(back[head], sd[head])


def test_decoder_dims_follow_the_checkpoint_tensors():
    """config.json fields that disagree with the tensors (max_length vs wpe rows, another model size) must not break loading."""
    import dataclasses

    from starvector_b200.config import dims_tiny_v2, refine_dims_from_state_dict

    for d in (dims_tiny(), dims_tiny_v2()):
        sd = synthetic_state_dict(d, seed=0)
        wrong = dataclasses.replace(d, n_layer=7, n_inner=64, vocab=123, hidden=128 * 5, n_head=5,
                                    n_positions=999 if d.variant == 0 else d.n_positions)
        assert refine_dims_from_state_dict(wrong, sd) == d


def test_v2_tokenizer_preparation(tmp_path):
    """llm/starcoder2.py:36-53: four added tokens (incl. <svg-end>) and left padding; the synthetic stand-in mirrors both."""
    from tokenizers import Tokenizer, models, pre_tokenizers, trainers
    from transformers import PreTrainedTokenizerFast

    from starvector_b200.tokenizer import load_tokenizer

    tk = Tokenizer(models.BPE(unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tk.train_from_iterator(["<svg></svg>"] * 4, trainers.BpeTrainer(vocab_size=60, special_tokens=["<unk>"]))
    PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>").save_pretrained(str(tmp_path))
    tok = load_tokenizer(str(tmp_path), vocab_size=500, v2=True)
    assert tok.padding_side == "left"
    for t in ("<svg-start>", "<image-start>", "<caption-start>", "<svg-end>"):
        assert len(tok.encode(t)) == 1
    syn = load_tokenizer(None, 500, v2=True)
    assert isinstance(syn, SyntheticTokenizer) and syn.padding_side == "left" and syn.pad_token_id == 495


def test_decode_chain_op_symbol_and_descriptor_layout():
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    assert "sv_op_decode_chain" in _header_symbols() and "sv_op_decode_chain" in _lib.SIGNATURES and "sv_op_decode_chain" in exported
    assert _lib.ABI_VERSION == 7
    assert C.sizeof(_lib.OpChainLayer) == 12 * 8
    # 12 int32, float, int32, 10 pointers, int64, 2 pointers, 5 pointers, 5 int64, int32 (+4), 3 pointers, 6 int32
    o = _lib.OpChain
    assert C.sizeof(o) == 296
    assert (o.ln_eps.offset, o.layers.offset, o.layer_stride.offset, o.pos_host.offset, o.x.offset, o.x_stride.offset,
            o.lm_head_tail.offset, o.logits.offset, o.pdl.offset, o.parts_used.offset, o.pdl_used.offset) == \
        (48, 56, 136, 152, 160, 200, 240, 248, 272, 288, 292)


def _bad_chain(**kw):
    """A v1 1B-shaped descriptor (2 layers, 2 rows) with fake aligned pointers, changed by kw; returns the call's code."""
    a = dict(mode=0, n_layer=2, B=2, per_row=0, hidden=2048, n_inner=8192, n_head=16, n_kv=1, vocab=49156, n_positions=8192,
             tcap=8224, window=0, ln_eps=1e-5, rope=0, pos=[100, 100], graph=0, pdl=1, tiled=0, parts=0, lm_head_tail=1,
             layer_stride=2 * 8224 * 128, x_stride=0, h_stride=0, null_layer_field=None, ptr=0x10000, ids=0x20000, amax=True,
             ln=0x30000, rope_tables=False)
    a.update(kw)
    layers = (_lib.OpChainLayer * 2)()
    for L in layers:
        for f in _lib.CHAIN_LAYER_FIELDS:
            setattr(L, f, a["ptr"])
    if a["null_layer_field"]:
        setattr(layers[1], a["null_layer_field"], 0)
    pos = (C.c_int32 * len(a["pos"]))(*a["pos"])
    o = _lib.OpChain(mode=a["mode"], n_layer=a["n_layer"], B=a["B"], per_row=a["per_row"], hidden=a["hidden"],
                     n_inner=a["n_inner"], n_head=a["n_head"], n_kv=a["n_kv"], vocab=a["vocab"], n_positions=a["n_positions"],
                     tcap=a["tcap"], window=a["window"], ln_eps=a["ln_eps"], rope=a["rope"], layers=layers,
                     layer_stride=a["layer_stride"], pos_host=C.cast(pos, C.POINTER(C.c_int32)), graph=a["graph"],
                     pdl=a["pdl"], tiled=a["tiled"], parts=a["parts"], lm_head_tail=a["lm_head_tail"],
                     x_stride=a["x_stride"], h_stride=a["h_stride"])
    for f in ("wte", "wpe", "lnf_w", "lnf_b", "lm_head", "kcache", "vtcache", "x", "qkv", "attn", "h", "logits"):
        setattr(o, f, 0x40000)
    o.ln, o.ids = a["ln"], a["ids"]
    if a["amax"]:
        o.amax_val, o.amax_idx = 0x50000, 0x60000
    if a["rope_tables"]:
        o.rope_cos, o.rope_sin = 0x70000, 0x80000
    lib = _lib.load()
    return lib.sv_op_decode_chain(C.byref(o), None), lib.sv_last_error(None)


@pytest.mark.parametrize("kw", [
    dict(mode=2), dict(n_layer=0), dict(B=0), dict(B=17), dict(per_row=2), dict(n_head=16, n_kv=3), dict(n_head=17),
    dict(hidden=2050), dict(n_inner=100), dict(vocab=0), dict(tcap=8200), dict(window=-1), dict(ln_eps=-1.0), dict(pdl=2),
    dict(graph=-1), dict(rope=1), dict(mode=1, tiled=1), dict(parts=9), dict(mode=1, parts=129), dict(parts=-1),
    dict(pos=[100, 101]), dict(pos=[8224, 8224]), dict(pos=[-1, -1]), dict(per_row=1, pos=[5, 8224]),
    dict(layer_stride=8224 * 128), dict(x_stride=2048), dict(x_stride=2 * 2048 + 4), dict(h_stride=-8),
    dict(null_layer_field="fc2_b"), dict(ptr=0x10008), dict(mode=1, ln=0), dict(ln=0x30008), dict(amax=False),
    # 8B widths on the FUSED chain: v1 (no RoPE) has no QKV epilogue behind a streamed LayerNorm; v2 holds 8 rows
    dict(hidden=4608, n_inner=18432, n_head=36, n_kv=4, layer_stride=2 * 4 * 8224 * 128),
    dict(hidden=4608, n_inner=18432, n_head=36, n_kv=4, layer_stride=9 * 4 * 8224 * 128, rope=1, rope_tables=True, B=9,
         pos=[7] * 9),
], ids=str)
def test_decode_chain_op_rejects_on_the_host(kw):
    """Checked before any CUDA call: SV_ERR_INVALID on a machine without a GPU too."""
    code, msg = _bad_chain(**kw)
    assert code == _lib.SV_ERR_INVALID and b"decode_chain" in msg, (code, msg)


def test_decode_chain_op_null_descriptor():
    lib = _lib.load()
    assert lib.sv_op_decode_chain(None, None) == _lib.SV_ERR_INVALID


def test_decode_flow_op_symbols_and_descriptor_layout():
    exported = set(re.findall(r" T (sv_\w+)", subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                                                             capture_output=True, text=True, check=True).stdout))
    for name in ("sv_op_decode_flow", "sv_op_flow_buffer_bytes"):
        assert name in _header_symbols() and name in _lib.SIGNATURES and name in exported, name
    # 9 int32, float, pointer, 7 pointers, int64, 8 int32, sv_gen_params (88), int32 (+4), 14 pointers, 2 int32
    o = _lib.OpFlow
    assert C.sizeof(o) == 360
    assert (o.ln_eps.offset, o.layers.offset, o.wte.offset, o.layer_stride.offset, o.nsteps.offset, o.clear.offset,
            o.params.offset, o.out_stride.offset, o.counters_host.offset, o.x_plain.offset, o.xa.offset, o.amax.offset,
            o.ncta_used.offset, o.realloc_used.offset) == \
        (36, 40, 48, 104, 112, 140, 144, 232, 240, 280, 296, 344, 352, 356)
    text = open(os.path.join(ROOT, "include", "starvector_b200.h")).read()
    order = re.search(r"enum \{ SV_FLOW_XA = 0, SV_FLOW_XB = 1, SV_FLOW_QKV = 2, SV_FLOW_ATT = 3, SV_FLOW_HB = 4, "
                      r"SV_FLOW_PART = 5, SV_FLOW_AMAX = 6 \};", text)
    assert order and _lib.FLOW_BUFFERS == ("xa", "xb", "qkv", "att", "hb", "part", "amax")


def test_decode_flow_buffer_bytes():
    """One flagged 32-bit word per value, each 8-value fragment in its own 256-byte chunk; attention partials: 64 splits of
    (m[16], l[16], acc[16][128]) 64-bit words per (row, kv head); argmax partials: 8 rows of 64-bit words per lm_head tile,
    room for one tile per vocabulary row."""
    lib = _lib.load()
    size = lambda w, B=8, H=2048, I=8192, kv=1, V=49157: lib.sv_op_flow_buffer_bytes(w, B, H, I, kv, V)
    assert size(_lib.SV_FLOW_XA) == size(_lib.SV_FLOW_XB) == size(_lib.SV_FLOW_ATT) == 8 * 256 * 256
    assert size(_lib.SV_FLOW_QKV) == 8 * (2304 // 8) * 256 and size(_lib.SV_FLOW_QKV, kv=2, H=512) == 8 * (1024 // 8) * 256
    assert size(_lib.SV_FLOW_HB) == 8 * 1024 * 256
    assert size(_lib.SV_FLOW_PART, B=3, kv=2) == 3 * 2 * 64 * (32 + 16 * 128) * 8
    assert size(_lib.SV_FLOW_AMAX) == 49157 * 64
    for bad in (dict(B=0), dict(H=2044), dict(I=0), dict(kv=0), dict(V=0)):
        assert size(_lib.SV_FLOW_XA, **bad) == -1, bad
    assert size(7) == -1 and size(-1) == -1


def _bad_flow(**kw):
    """A 1B-shaped descriptor (2 layers, 8 rows, greedy selection) with fake aligned pointers, changed by kw."""
    a = dict(n_layer=2, B=8, hidden=2048, n_inner=8192, n_head=16, n_kv=1, vocab=49156, n_positions=8192, tcap=8224,
             ln_eps=1e-5, layer_stride=8 * 8224 * 128, nsteps=16, step0=0, cur_len0=100, first_plain=1, do_select=1,
             l2_ahead=0, realloc=1, clear=1, rp=1.0, do_sample=0, n_stop=0, out_stride=64, counters=[0, 100, 0],
             unfinished=True, null_layer_field=None, ptr=0x10000, wte=0x40000, xa=0x50000, amax=0x60000, x_plain=0x70000,
             seen=0x80000)
    a.update(kw)
    layers = (_lib.OpChainLayer * max(1, a["n_layer"]))()
    for L in layers:
        for f in _lib.CHAIN_LAYER_FIELDS:
            setattr(L, f, a["ptr"])
    if a["null_layer_field"]:
        setattr(layers[-1], a["null_layer_field"], 0)
    p = GenerationParams(max_new_tokens=64, repetition_penalty=a["rp"], do_sample=bool(a["do_sample"]),
                         stop_ids=[7] * a["n_stop"] if a["n_stop"] <= 8 else []).to_c()
    if a["n_stop"] > 8 or a["n_stop"] < 0:
        p.n_stop_ids = a["n_stop"]
    o = _lib.OpFlow(n_layer=a["n_layer"], B=a["B"], hidden=a["hidden"], n_inner=a["n_inner"], n_head=a["n_head"],
                    n_kv=a["n_kv"], vocab=a["vocab"], n_positions=a["n_positions"], tcap=a["tcap"], ln_eps=a["ln_eps"],
                    layers=layers, layer_stride=a["layer_stride"], nsteps=a["nsteps"], step0=a["step0"],
                    cur_len0=a["cur_len0"], first_plain=a["first_plain"], do_select=a["do_select"], l2_ahead=a["l2_ahead"],
                    realloc=a["realloc"], clear=a["clear"], params=p, out_stride=a["out_stride"])
    for f in ("wpe", "lnf_w", "lnf_b", "lm_head", "kcache", "vtcache", "logits", "xb", "qkv", "att", "hb", "part", "out_ids",
              "next_ids"):
        setattr(o, f, 0x40000)
    o.wte, o.xa, o.amax, o.x_plain, o.seen = a["wte"], a["xa"], a["amax"], a["x_plain"], a["seen"]
    counters = (C.c_int32 * 3)(*a["counters"]) if a["counters"] else None
    unfinished = (C.c_int32 * 8)(*([1] * 8)) if a["unfinished"] else None
    if counters:
        o.counters_host = C.cast(counters, C.POINTER(C.c_int32))
    if unfinished:
        o.unfinished_host = C.cast(unfinished, C.POINTER(C.c_int32))
    lib = _lib.load()
    return lib.sv_op_decode_flow(C.byref(o), None), lib.sv_last_error(None)


@pytest.mark.parametrize("kw", [
    dict(B=0), dict(B=9), dict(n_layer=0), dict(n_layer=25), dict(n_head=16, n_kv=3), dict(n_head=17),
    # widths the kernel does not take: the 8B decoder, a hidden vector that is not 2^k fragments, a staged c_fc output
    # that is not either, a wide one that is not whole slabs, RoPE-free GQA beyond 16 heads per group
    dict(hidden=4608, n_inner=18432, n_head=36, n_kv=4, layer_stride=8 * 4 * 8224 * 128), dict(hidden=768, n_head=6),
    dict(n_inner=1536), dict(n_inner=2560), dict(hidden=2048, n_head=16, n_kv=1, n_inner=96),
    dict(vocab=0), dict(n_positions=0), dict(tcap=8200), dict(tcap=0), dict(ln_eps=-1.0),
    dict(first_plain=2), dict(do_select=-1), dict(realloc=2), dict(clear=3),
    dict(nsteps=0), dict(step0=-1), dict(cur_len0=-1), dict(cur_len0=8208), dict(cur_len0=8208, nsteps=16),
    dict(tcap=16416, layer_stride=8 * 16416 * 128, cur_len0=16380, nsteps=5), dict(l2_ahead=-1), dict(l2_ahead=65),
    dict(clear=1, first_plain=0), dict(wte=0), dict(x_plain=0), dict(xa=0), dict(amax=0), dict(wte=0x40004),
    dict(xa=0x50008), dict(amax=0x60008), dict(x_plain=0x70002), dict(layer_stride=8 * 8224 * 128 - 8),
    dict(layer_stride=8 * 8224 * 128 + 4), dict(null_layer_field="ln2_b"), dict(ptr=0x10008), dict(rp=0.0), dict(rp=-1.0),
    dict(do_sample=1), dict(n_stop=9), dict(n_stop=-1), dict(seen=0), dict(counters=None), dict(unfinished=False),
    dict(out_stride=0), dict(counters=[-1, 100, 0]), dict(counters=[60, 100, 0]), dict(counters=[0, -1, 0]),
], ids=str)
def test_decode_flow_op_rejects_on_the_host(kw):
    """Every combination the kernel could not complete (its polls would spin until the watchdog traps) or would compute
    wrong is refused before any CUDA call: SV_ERR_INVALID on a machine without a GPU too."""
    code, msg = _bad_flow(**kw)
    assert code == _lib.SV_ERR_INVALID and b"decode_flow" in msg, (code, msg)


def test_decode_flow_op_accepts_what_it_should_on_the_host():
    """The base descriptor and its edge cases pass every host check: on a machine without a GPU the call then fails in the
    first CUDA call, not as SV_ERR_INVALID.  (A finished generation may run past out_stride: nothing is written then.)"""
    if torch.cuda.is_available():
        pytest.skip("a GPU would run these launches over fake pointers")
    for kw in (dict(), dict(cur_len0=8207, nsteps=16), dict(do_select=0, seen=0,
               counters=None, unfinished=False), dict(counters=[60, 100, 1]), dict(hidden=512, n_head=4, n_kv=2, n_inner=1024,
               layer_stride=8 * 2 * 8224 * 128), dict(n_layer=24), dict(B=1, layer_stride=8224 * 128), dict(l2_ahead=64)):
        code, msg = _bad_flow(**kw)
        assert code != _lib.SV_ERR_INVALID, (kw, msg)


def test_decode_flow_op_null_descriptor():
    lib = _lib.load()
    assert lib.sv_op_decode_flow(None, None) == _lib.SV_ERR_INVALID

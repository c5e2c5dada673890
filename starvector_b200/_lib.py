"""ctypes binding of the C-ABI in include/starvector_b200.h (the whole product boundary).

No torch types cross this boundary: tensors are passed as raw device pointers plus sizes and
the current CUDA stream handle.  Loading fails loudly when the library has not been built —
there is no Python/CPU fallback for any entry point.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SV_LIB_PATH") or os.path.join(_HERE, "libstarvector_b200.so")   # SV_LIB_PATH: A/B builds

SV_OK, SV_ERR_INVALID, SV_ERR_CUDA, SV_ERR_UNSUPPORTED, SV_ERR_STATE = 0, -1, -2, -3, -4
SV_DTYPE_BF16, SV_DTYPE_F32, SV_DTYPE_F16 = 0, 1, 2
SV_ACT_NONE, SV_ACT_QUICKGELU, SV_ACT_GELU_TANH, SV_ACT_SILU = 0, 1, 2, 3
SV_LINEAR_AUTO, SV_LINEAR_ROWGROUP, SV_LINEAR_TCGEN05 = 0, 1, 2
ABI_VERSION = 7
SV_ALPHA_WHITE, SV_ALPHA_DROP = 0, 1


class ModelDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "variant", "image_size", "patch_size", "vit_width", "vit_layers", "vit_heads", "vit_mlp", "adapter_norm",
        "hidden", "n_layer", "n_head", "n_kv_head", "head_dim", "n_inner", "n_positions", "vocab")] + [
        ("ln_eps", C.c_float), ("max_batch", C.c_int32), ("max_len", C.c_int32),
        ("rope_theta", C.c_float), ("sliding_window", C.c_int32), ("vit_ln_eps", C.c_float)]


class GenParams(C.Structure):
    _fields_ = [
        ("max_new_tokens", C.c_int32), ("do_sample", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float),
        ("repetition_penalty", C.c_float), ("eos_token_id", C.c_int32), ("pad_token_id", C.c_int32),
        ("n_stop_ids", C.c_int32), ("stop_ids", C.c_int32 * 8), ("stop_row0_only", C.c_int32),
        ("seed", C.c_uint64), ("poll_interval", C.c_int32),
    ]


class BeamParams(C.Structure):
    _fields_ = [
        ("num_beams", C.c_int32), ("max_new_tokens", C.c_int32), ("do_sample", C.c_int32), ("early_stopping", C.c_int32),
        ("temperature", C.c_float), ("top_p", C.c_float), ("repetition_penalty", C.c_float), ("length_penalty", C.c_float),
        ("eos_token_id", C.c_int32), ("pad_token_id", C.c_int32), ("n_stop_ids", C.c_int32), ("stop_ids", C.c_int32 * 8),
        ("poll_interval", C.c_int32), ("seed", C.c_uint64),
    ]


class PreprocDesc(C.Structure):
    _fields_ = [("out_size", C.c_int32), ("alpha_mode", C.c_int32), ("pad_square", C.c_int32), ("out_dtype", C.c_int32),
                ("mean", C.c_float * 3), ("std", C.c_float * 3)]


class ImageU8(C.Structure):
    _fields_ = [("data", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32),
                ("row_stride", C.c_int32)]


SV_ATTN_DECODE_SPLIT, SV_ATTN_DECODE_CLUSTER = 0, 1


class OpRing(C.Structure):   # sv_op_ring
    _fields_ = [(n, C.c_void_p) for n in ("x", "w", "bias", "residual", "ln_w", "ln_b", "y")] + [
        (n, C.c_int32) for n in ("B", "N", "K", "act", "epi", "tiled")] + [
        ("ln_eps", C.c_float), ("kcache", C.c_void_p), ("vtcache", C.c_void_p)] + [
        (n, C.c_int32) for n in ("n_head", "n_kv", "tcap", "per_row")] + [
        ("pos_host", C.POINTER(C.c_int32)), ("amax_val", C.c_void_p), ("amax_idx", C.c_void_p)]


SV_CHAIN_FUSED, SV_CHAIN_PER_OP = 0, 1
CHAIN_LAYER_FIELDS = ("ln1_w", "ln1_b", "attn_w", "attn_b", "proj_w", "proj_b", "ln2_w", "ln2_b", "fc_w", "fc_b", "fc2_w", "fc2_b")


class OpChainLayer(C.Structure):   # sv_op_chain_layer
    _fields_ = [(n, C.c_void_p) for n in CHAIN_LAYER_FIELDS]


class OpChain(C.Structure):   # sv_op_chain
    _fields_ = [(n, C.c_int32) for n in ("mode", "n_layer", "B", "per_row", "hidden", "n_inner", "n_head", "n_kv", "vocab",
                                         "n_positions", "tcap", "window")] + [
        ("ln_eps", C.c_float), ("rope", C.c_int32), ("layers", C.POINTER(OpChainLayer))] + [
        (n, C.c_void_p) for n in ("wte", "wpe", "lnf_w", "lnf_b", "lm_head", "rope_cos", "rope_sin", "kcache", "vtcache")] + [
        ("layer_stride", C.c_int64), ("ids", C.c_void_p), ("pos_host", C.POINTER(C.c_int32))] + [
        (n, C.c_void_p) for n in ("x", "ln", "qkv", "attn", "h")] + [
        (n, C.c_int64) for n in ("x_stride", "ln_stride", "qkv_stride", "attn_stride", "h_stride")] + [
        ("lm_head_tail", C.c_int32), ("logits", C.c_void_p), ("amax_val", C.c_void_p), ("amax_idx", C.c_void_p)] + [
        (n, C.c_int32) for n in ("pdl", "graph", "tiled", "parts", "parts_used", "pdl_used")]


SV_FLOW_XA, SV_FLOW_XB, SV_FLOW_QKV, SV_FLOW_ATT, SV_FLOW_HB, SV_FLOW_PART, SV_FLOW_AMAX = range(7)
FLOW_BUFFERS = ("xa", "xb", "qkv", "att", "hb", "part", "amax")    # in SV_FLOW_* order


class OpFlow(C.Structure):   # sv_op_flow
    _fields_ = [(n, C.c_int32) for n in ("n_layer", "B", "hidden", "n_inner", "n_head", "n_kv", "vocab", "n_positions",
                                         "tcap")] + [
        ("ln_eps", C.c_float), ("layers", C.POINTER(OpChainLayer))] + [
        (n, C.c_void_p) for n in ("wte", "wpe", "lnf_w", "lnf_b", "lm_head", "kcache", "vtcache")] + [
        ("layer_stride", C.c_int64)] + [
        (n, C.c_int32) for n in ("nsteps", "step0", "cur_len0", "first_plain", "do_select", "l2_ahead", "realloc", "clear")] + [
        ("params", GenParams), ("out_stride", C.c_int32), ("counters_host", C.POINTER(C.c_int32)),
        ("unfinished_host", C.POINTER(C.c_int32)), ("seen", C.c_void_p), ("out_ids", C.c_void_p), ("next_ids", C.c_void_p),
        ("x_plain", C.c_void_p), ("logits", C.c_void_p)] + [(n, C.c_void_p) for n in FLOW_BUFFERS] + [
        ("ncta_used", C.c_int32), ("realloc_used", C.c_int32)]


SV_SELECT_GREEDY, SV_SELECT_SAMPLE, SV_SELECT_FUSED = 0, 1, 2
SV_ADAPTER_NORM_SLAB, SV_ADAPTER_NORM_TOKENS = 0, 1


class OpSelect(C.Structure):   # sv_op_select_args
    _fields_ = [("impl", C.c_int32), ("per_row", C.c_int32), ("logits", C.c_void_p), ("vocab", C.c_int32), ("B", C.c_int32),
                ("params", GenParams), ("seen", C.c_void_p), ("out_ids", C.c_void_p), ("next_ids", C.c_void_p),
                ("out_stride", C.c_int32), ("advance_len", C.c_int32), ("nsteps", C.c_int32),
                ("counters_host", C.POINTER(C.c_int32)), ("unfinished_host", C.POINTER(C.c_int32)),
                ("row_len_host", C.POINTER(C.c_int32)), ("row_step_host", C.POINTER(C.c_int32)),
                ("row_active_host", C.POINTER(C.c_int32)), ("row_max_new_host", C.POINTER(C.c_int32)),
                ("row_seed_host", C.POINTER(C.c_uint64)), ("row_mask", C.c_uint32), ("event_host", C.POINTER(C.c_int32)),
                ("amax_val", C.c_void_p), ("amax_idx", C.c_void_p), ("wte", C.c_void_p), ("wpe", C.c_void_p),
                ("x", C.c_void_p), ("h", C.c_int32), ("n_positions", C.c_int32)]


SV_SPEC_GREEDY, SV_SPEC_SAMPLE, SV_SPEC_ACCEPT = 0, 1, 2


class SpecState(C.Structure):   # sv_spec_state (svspec::State)
    _fields_ = [("n_live", C.c_int32), ("row", C.c_int32 * 16), ("pos", C.c_int32 * 16), ("tok", C.c_int32 * 16),
                ("sel", C.c_int32 * 16)] + [(n, C.c_int32) for n in ("ncols", "k", "max_ngram", "steps", "drafted", "accepted")]


class OpSpec(C.Structure):   # sv_op_spec_args
    _fields_ = [("impl", C.c_int32), ("logits", C.c_void_p), ("vocab", C.c_int32), ("params", GenParams),
                ("seen", C.c_void_p), ("out_ids", C.c_void_p), ("next_ids", C.c_void_p), ("out_stride", C.c_int32),
                ("gen_host", C.POINTER(C.c_int32)), ("spec_host", C.POINTER(SpecState)),
                ("amax_val", C.c_void_p), ("amax_idx", C.c_void_p), ("wte", C.c_void_p), ("wpe", C.c_void_p),
                ("x", C.c_void_p), ("h", C.c_int32), ("n_positions", C.c_int32)]


class BeamState(C.Structure):   # sv_beam_state (svbeam::State): also the state blob of sv_beam_state_init_host / _step_host
    _fields_ = [(n, C.c_int32) for n in ("cur_len", "done", "parity", "pad_")] + [
        ("running_scores", C.c_float * 16), ("beam_scores", C.c_float * 16), ("is_finished", C.c_int32 * 16),
        ("fin_len", C.c_int32 * 16), ("unsatisfied", C.c_int32 * 16), ("div", (C.c_int32 * 16) * 16)]


class BeamPlan(C.Structure):   # sv_beam_plan (svbeam::Plan)
    _fields_ = [(n, C.c_int32 * 16) for n in ("run_parent", "run_tok", "fin_old", "fin_parent", "fin_tok", "copy_src",
                                              "copy_lo")] + [(n, C.c_int32) for n in ("copy_hi", "cont", "old_len")]


class OpBeamStep(C.Structure):   # sv_op_beam_step_args
    _fields_ = [("params", C.POINTER(BeamParams))] + [(n, C.c_int32) for n in ("batch", "vocab", "seq_stride", "advance")] + [
        ("state_host", C.POINTER(BeamState)), ("cand_key", C.c_void_p), ("cand_val", C.c_void_p), ("cand_tok", C.c_void_p),
        ("run_seq", C.c_void_p), ("fin_seq", C.c_void_p), ("gen_host", C.POINTER(C.c_int32)), ("wte", C.c_void_p),
        ("wpe", C.c_void_p), ("x", C.c_void_p), ("h", C.c_int32), ("n_positions", C.c_int32), ("next_ids", C.c_void_p),
        ("plan_host", C.POINTER(BeamPlan))]


class OpAdmit(C.Structure):   # sv_op_admit_args
    _fields_ = [("k", C.c_int32), ("S", C.c_int32), ("slot_host", C.POINTER(C.c_int32)), ("len_host", C.POINTER(C.c_int32)),
                ("max_new_host", C.POINTER(C.c_int32)), ("seed_host", C.POINTER(C.c_uint64)), ("seen", C.c_void_p),
                ("vocab", C.c_int32), ("out_ids", C.c_void_p), ("out_stride", C.c_int32), ("pad_id", C.c_int32),
                ("row_len_host", C.POINTER(C.c_int32)), ("row_step_host", C.POINTER(C.c_int32)),
                ("row_active_host", C.POINTER(C.c_int32)), ("row_max_new_host", C.POINTER(C.c_int32)),
                ("row_seed_host", C.POINTER(C.c_uint64)), ("event_host", C.POINTER(C.c_int32))]


class SpecParams(C.Structure):   # sv_spec_params
    _fields_ = [("num_tokens", C.c_int32), ("max_matching_ngram_size", C.c_int32)]


class SessionRows(C.Structure):   # sv_session_rows (RowState)
    _fields_ = [("row_len", C.c_int32 * 16), ("row_step", C.c_int32 * 16), ("row_active", C.c_int32 * 16),
                ("event", C.c_int32), ("pad_", C.c_int32), ("row_max_new", C.c_int32 * 16), ("row_seed", C.c_uint64 * 16)]


class SpecSessionState(C.Structure):   # sv_spec_session_state (svspec::SessionState)
    _fields_ = [("n_live", C.c_int32)] + [(n, C.c_int32 * 16) for n in ("row", "pos", "tok", "sel", "off")] + [
        (n, C.c_int32) for n in ("ncols", "k", "max_ngram", "steps", "drafted", "accepted")]


SV_SPEC_SESSION_GREEDY, SV_SPEC_SESSION_SAMPLE, SV_SPEC_SESSION_TAIL = 0, 1, 2


class OpSpecSession(C.Structure):   # sv_op_spec_session_args
    _fields_ = [("impl", C.c_int32), ("accept", C.c_int32), ("logits", C.c_void_p), ("vocab", C.c_int32),
                ("params", GenParams), ("seen", C.c_void_p), ("out_ids", C.c_void_p), ("next_ids", C.c_void_p),
                ("out_stride", C.c_int32), ("tcap", C.c_int32), ("rows_host", C.POINTER(SessionRows)),
                ("ss_host", C.POINTER(SpecSessionState)), ("amax_val", C.c_void_p), ("amax_idx", C.c_void_p),
                ("wte", C.c_void_p), ("wpe", C.c_void_p), ("x", C.c_void_p), ("h", C.c_int32), ("n_positions", C.c_int32)]


TOKEN_CALLBACK =C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32)   # sv_token_callback

# name -> (restype, argtypes); must list every SV_API symbol of the header (tests check this)
_P, _I, _F = C.c_void_p, C.c_int32, C.c_float
SIGNATURES = {
    "sv_abi_version": (C.c_int, []),
    "sv_engine_create": (C.c_int, [C.POINTER(ModelDesc), C.c_int, C.POINTER(_P)]),
    "sv_engine_destroy": (None, [_P]),
    "sv_last_error": (C.c_char_p, [_P]),
    "sv_engine_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), _I, _I]),
    "sv_engine_missing_weights": (C.c_int, [_P]),
    "sv_encode_images": (C.c_int, [_P, _P, _I, _P, _P, _P]),
    "sv_prefill": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "sv_prefill_embeds": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "sv_decode_step": (C.c_int, [_P, _P, _P, _P]),
    "sv_score_tokens": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "sv_reorder_cache": (C.c_int, [_P, _P, _P]),
    "sv_expand_batch": (C.c_int, [_P, _P, C.c_int32, _P]),
    "sv_beam_search": (C.c_int, [_P, C.POINTER(BeamParams), _I, _P, _P, _P]),
    "sv_beam_params_check": (C.c_int, [C.POINTER(BeamParams), _I]),
    "sv_beam_params_check_rows": (C.c_int, [C.POINTER(BeamParams), _I, _I]),
    "sv_beam_state_bytes": (C.c_int, []),
    "sv_beam_state_init_host": (C.c_int, [C.POINTER(BeamParams), _I, _I, _P]),
    "sv_beam_state_read_host": (C.c_int, [_P, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I), C.POINTER(C.c_float)]),
    "sv_beam_state_read16_host": (C.c_int, [_P, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I), C.POINTER(C.c_float),
                                            C.POINTER(C.c_float)]),
    "sv_beam_row_candidates_host": (C.c_int, [C.POINTER(BeamParams), C.POINTER(C.c_float), _I, C.POINTER(_I), _I, _F, _I, _I,
                                              C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(_I)]),
    "sv_beam_step_host": (C.c_int, [C.POINTER(BeamParams), _I, _I, _I, _P, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                    C.POINTER(_I), C.POINTER(_I), C.POINTER(_I), _I, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)]),
    "sv_generate": (C.c_int, [_P, C.POINTER(GenParams), _P, _P, _P]),
    "sv_generate_stream": (C.c_int, [_P, C.POINTER(GenParams), _P, _P, TOKEN_CALLBACK, _P, _P]),
    "sv_generate_im2svg_host": (C.c_int, [_P, _P, _I, _P, _I, C.POINTER(GenParams), _P, _P, _P]),
    "sv_generate_speculative": (C.c_int, [_P, C.POINTER(GenParams), C.POINTER(SpecParams), _P, _P, TOKEN_CALLBACK, _P, _P]),
    "sv_last_spec_stats": (C.c_int, [_P, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)]),
    "sv_spec_verify_step": (C.c_int, [_P, C.POINTER(_I), _I, _P, _P]),
    "sv_spec_draft_host": (C.c_int, [C.POINTER(_I), _I, _I, _I, _I, _I, C.POINTER(_I)]),
    "sv_spec_accept_host": (C.c_int, [C.POINTER(GenParams), C.POINTER(_I), C.POINTER(_I), _I, C.POINTER(_I), C.POINTER(_I), _I]),
    "sv_session_begin": (C.c_int, [_P, C.POINTER(GenParams), _I]),
    "sv_session_admit": (C.c_int, [_P, _P, _I, _P, _I, _P, _P, _P, _P, _P]),
    "sv_session_run": (C.c_int, [_P, _I, _P, _P, _P]),
    "sv_session_read": (C.c_int, [_P, _I, _P, _P]),
    "sv_session_end": (C.c_int, [_P]),
    "sv_session_begin_speculative": (C.c_int, [_P, C.POINTER(GenParams), C.POINTER(SpecParams), _I]),
    "sv_session_spec_stats": (C.c_int, [_P, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)]),
    "sv_spec_session_plan_host": (C.c_int, [_I, C.POINTER(_I), C.POINTER(_I), _I, C.POINTER(_I), C.POINTER(_I)]),
    "sv_spec_session_tail_host": (C.c_int, [C.POINTER(GenParams), C.POINTER(SessionRows), C.POINTER(_I), _I,
                                            C.POINTER(SpecSessionState), _I, _I]),
    "sv_beam_session_begin": (C.c_int, [_P, C.POINTER(BeamParams), _I]),
    "sv_beam_session_admit": (C.c_int, [_P, _P, _I, _P, _I, _P, _P, _P, _P]),
    "sv_launch_count": (C.c_int64, [_P]),
    "sv_engine_describe": (C.c_char_p, [_P]),
    "sv_debug_read_timeline": (C.c_int, [_P, C.POINTER(C.c_longlong), _I]),
    "sv_last_decode_timing": (C.c_int, [_P, C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
    "sv_op_layernorm": (C.c_int, [_P, _P, _P, _P, _I, _I, _F, _P]),
    "sv_op_linear": (C.c_int, [_I, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "sv_op_attention_vit": (C.c_int, [_P, _P, _I, _I, _I, _P]),
    "sv_op_attention_mqa": (C.c_int, [_P, _P, _I, _I, _I, _P]),
    "sv_op_attention_chunk": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "sv_op_lm_logprob": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "sv_op_attention_decode": (C.c_int, [_I, _I, _P, _P, _P, _P, C.POINTER(_I), _I, _I, _I, _I, _I, _I, _P]),
    "sv_op_gemv_ring": (C.c_int, [C.POINTER(OpRing), _P]),
    "sv_op_ring_ntiles": (C.c_int32, [_I]),
    "sv_op_ring_row_stride": (C.c_int32, [_I]),
    "sv_op_rope_table": (C.c_int, [_P, _P, _I, _I, _F, _P]),
    "sv_op_rope": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, C.POINTER(_I), _I, _P, _P, _I, _P]),
    "sv_op_decode_chain": (C.c_int, [C.POINTER(OpChain), _P]),
    "sv_op_flow_buffer_bytes": (C.c_int64, [_I, _I, _I, _I, _I, _I]),
    "sv_op_decode_flow": (C.c_int, [C.POINTER(OpFlow), _P]),
    "sv_op_select": (C.c_int, [C.POINTER(OpSelect), _P]),
    "sv_op_spec_select": (C.c_int, [C.POINTER(OpSpec), _P]),
    "sv_op_spec_session_select": (C.c_int, [C.POINTER(OpSpecSession), _P]),
    "sv_op_beam_candidates": (C.c_int, [_P, _I, C.POINTER(BeamParams), _I, _I, C.POINTER(C.c_float), _P, _I, _P, _P, _P, _P]),
    "sv_op_beam_step": (C.c_int, [C.POINTER(OpBeamStep), _P]),
    "sv_op_beam_kv_copy": (C.c_int, [_P, _P, C.c_int64, _I, _I, _I, _I, C.POINTER(BeamPlan), _P]),
    "sv_op_kv_gather": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "sv_op_session_admit": (C.c_int, [C.POINTER(OpAdmit), _P]),
    "sv_op_im2col": (C.c_int, [_P, _P, _I, _I, _I, _I, _P]),
    "sv_op_vit_assemble": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "sv_op_adapter_norm": (C.c_int, [_I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _P]),
    "sv_op_embed_prefix": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "sv_op_attention_prefill": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "sv_op_lm_logits": (C.c_int, [_P, _P, _P, _I, _I, _I, _P]),
    "sv_op_attention_score": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "sv_op_logits_logprob": (C.c_int, [_P, _P, _P, _I, _I, _P]),
    "sv_preproc_create": (C.c_int, [C.POINTER(PreprocDesc), C.c_int, C.POINTER(_P)]),
    "sv_preproc_destroy": (None, [_P]),
    "sv_preproc_last_error": (C.c_char_p, [_P]),
    "sv_preproc_run_host": (C.c_int, [_P, C.POINTER(ImageU8), _I, _P, _P]),
    "sv_preproc_launch_count": (C.c_longlong, [_P]),
    "sv_resample_coeffs_host": (C.c_int, [_I, _I, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I), _I]),
    "sv_preproc_lut_host": (C.c_int, [C.POINTER(PreprocDesc), C.POINTER(C.c_float)]),
    "sv_preproc_plan_host": (C.c_int, [C.POINTER(PreprocDesc), C.POINTER(ImageU8), _I, _P, C.c_int64, C.POINTER(C.c_int64)]),
}

_lib = None


def load() -> C.CDLL:
    """Load libstarvector_b200.so (built by `python -m starvector_b200.build` / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA library has not been built. Run `python -m starvector_b200.build` "
            "(needs nvcc). starvector_b200 has no CPU or PyTorch fallback path."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.sv_abi_version() != ABI_VERSION:
        raise RuntimeError(f"ABI mismatch: library {lib.sv_abi_version()} vs binding {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


class EngineError(RuntimeError):
    """Any non-zero return of the C-ABI (SV_ERR_INVALID is raised as ValueError instead)."""


def check(lib, code: int, handle=None) -> None:
    if code == SV_OK:
        return
    msg = lib.sv_last_error(handle)
    text = msg.decode("utf-8", "replace") if msg else ""
    if code == SV_ERR_INVALID:
        raise ValueError(f"starvector_b200: {text}")
    if code == SV_ERR_UNSUPPORTED:
        raise NotImplementedError(f"starvector_b200: {text}")
    raise EngineError(f"starvector_b200 (code {code}): {text}")

/*
 * starvector_b200 — C-ABI of the H100-native im2svg generation engine.
 *
 * The reference (joanrod/star-vector) has no FFI: its boundary for this path is the Python
 * method surface `StarVectorForCausalLM.generate_im2svg` / `.model.svg_transformer
 * .transformer.generate` (reference: starvector/model/starvector_arch.py:186-187,
 * starvector/model/models/starvector_base.py:203-259).  The Python facade in
 * `starvector_b200/modeling.py` keeps that surface and binds THESE entry points with ctypes
 * (see INTEGRATION.md).  Each entry point below names the reference code it replaces.
 *
 * Conventions: plain pointers and sizes only (no torch types); every pointer is a DEVICE
 * pointer unless the name ends in `_host` or the comment says "host or device"; `stream` is
 * a `cudaStream_t` passed as `void*` (NULL = legacy default stream); return 0 on success,
 * <0 on error with the message available from `sv_last_error`; no exceptions cross the
 * ABI; an engine is not re-entrant (the caller serialises; the Python shim holds a lock).
 * There is no CPU fallback: every call fails with SV_ERR_CUDA if no sm_90 (H100) device is usable.
 */
#ifndef STARVECTOR_B200_H
#define STARVECTOR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SV_ABI_VERSION 7
#if defined(__GNUC__)
#define SV_API __attribute__((visibility("default")))
#else
#define SV_API
#endif

enum {
  SV_OK = 0,
  SV_ERR_INVALID = -1,     /* bad argument / shape / name */
  SV_ERR_CUDA = -2,        /* CUDA runtime or driver error (message has the cudaError string) */
  SV_ERR_UNSUPPORTED = -3, /* valid request this build does not implement */
  SV_ERR_STATE = -4        /* call order violated (weights missing, no prefill before generate, ...) */
};

enum { SV_DTYPE_BF16 = 0, SV_DTYPE_F32 = 1, SV_DTYPE_F16 = 2 };

/* activation selectors of the fused linear epilogue */
enum {
  SV_ACT_NONE = 0,
  SV_ACT_QUICKGELU = 1, /* x*sigmoid(1.702x)  — clip_model.py:126-128 */
  SV_ACT_GELU_TANH = 2, /* gelu_pytorch_tanh  — GPTBigCodeMLP */
  SV_ACT_SILU = 3       /* x*sigmoid(x)       — adapters/adapter.py:5-10 */
};

/* implementation selector for sv_op_linear (tests cross-check the two kernels) */
enum { SV_LINEAR_AUTO = 0, SV_LINEAR_ROWGROUP = 1, SV_LINEAR_TCGEN05 = 2 };

typedef struct sv_engine sv_engine;

/* Dimensions of one StarVector model (SURVEY.md §8; reference: image_encoder.py:50-61,
 * starvector_base.py:87-104, adapters/adapter.py:13-31, bigcode/starcoderbase-1b config). */
typedef struct sv_model_desc {
  int32_t variant;      /* 0 = v1 (1B): CLIP ViT-L/14 + Adapter + GPTBigCode (MQA, learned positions).
                           1 = v2 (8B): SigLIP tower (no class token, LN eps 1e-6, gelu_tanh, patch bias, post_layernorm)
                               + StarCoder2 (GQA, RoPE, sliding-window attention, biased linears) — models/starvector_v2.py */
  int32_t image_size;   /* 224 */
  int32_t patch_size;   /* 14  */
  int32_t vit_width;    /* 1024 */
  int32_t vit_layers;   /* 23 (penultimate-layer CLIP ViT-L/14) */
  int32_t vit_heads;    /* 16 (head dim must be 64) */
  int32_t vit_mlp;      /* 4096 */
  int32_t adapter_norm; /* 0 = LayerNorm([Q,H]); 1 = BatchNorm1d(Q) in eval mode */
  int32_t hidden;       /* 2048 */
  int32_t n_layer;      /* 24 */
  int32_t n_head;       /* 16 */
  int32_t n_kv_head;    /* 1 (multi-query) */
  int32_t head_dim;     /* 128 */
  int32_t n_inner;      /* 8192 */
  int32_t n_positions;  /* 8192 learned absolute positions */
  int32_t vocab;        /* 49156 = 49152 + [PAD] + 3 added tokens (llm/starcoder.py:43-53) */
  float ln_eps;         /* 1e-5 */
  int32_t max_batch;    /* cache rows (images x beams / completions) per call on this GPU, [1,16] */
  int32_t max_len;      /* KV-cache capacity in tokens (prefix + generated) */
  /* v2 only (ignored for variant 0) */
  float rope_theta;       /* StarCoder2 rope_theta (hub config of bigcode/starcoder2-7b; default 10000 in transformers) */
  int32_t sliding_window; /* 4096 for starcoder2-7b; 0 = full causal attention */
  float vit_ln_eps;       /* 1e-6 for SigLIP (1e-5 is used for variant 0) */
} sv_model_desc;

/* Decoding parameters = the kwargs the reference forwards to HF generate()
 * (starvector_base.py:223-241, :289-295) after HF's own length fix-up (SURVEY.md App. B). */
typedef struct sv_gen_params {
  int32_t max_new_tokens;    /* = max_length - (Q + P)  (generation/utils.py:1629-1638) */
  int32_t do_sample;         /* use_nucleus_sampling; 0 = greedy argmax (lowest index wins ties) */
  float temperature;
  float top_p;
  float repetition_penalty;  /* applies to generated ids only (App. B.4) */
  int32_t eos_token_id;      /* -1 = none (throughput configs) */
  int32_t pad_token_id;
  int32_t n_stop_ids;        /* 0..8: ids of '</svg>' (StoppingCriteriaSub, starvector_base.py:9-20) */
  int32_t stop_ids[8];
  int32_t stop_row0_only;    /* 1 = reference behaviour D6 (row 0 matching ends the WHOLE batch);
                                0 = per-row: a matching row is finished/padded, batch ends when all rows are */
  uint64_t seed;             /* Philox seed for sampling */
  int32_t poll_interval;     /* host polls the device stop flag every this many steps (0 -> 16) */
} sv_gen_params;

/* Beam search / beam-sample parameters = what HF `generate(num_beams > 1)` receives from the reference
 * (starvector_base.py:231-241: num_beams=2, do_sample, top_p, temperature, repetition_penalty, length_penalty;
 * :289-295: early_stopping=True, pad_token_id; starvector_v2.py:53-57: nothing -> HF defaults). */
typedef struct sv_beam_params {
  int32_t num_beams;          /* >= 2 and <= 8; batch * num_beams <= 16 cache rows (and <= the engine's max_batch) */
  int32_t max_new_tokens;
  int32_t do_sample;          /* 1 = beam-sample (candidates drawn without replacement, device Philox stream) */
  int32_t early_stopping;     /* 0 = False (HF default), 1 = True (v1), 2 = "never" */
  float temperature;
  float top_p;
  float repetition_penalty;   /* on the log-probs, over each running beam's own generated ids */
  float length_penalty;
  int32_t eos_token_id;       /* -1 = none */
  int32_t pad_token_id;       /* fill of the returned rectangle (HF: pad if given, else eos) */
  int32_t n_stop_ids;         /* 0..8: StoppingCriteriaSub, candidate 0 of image 0 matching ends every beam */
  int32_t stop_ids[8];
  int32_t poll_interval;      /* host polls the device done flag every this many steps (0 -> 16) */
  uint64_t seed;
} sv_beam_params;

/* ---- lifecycle ------------------------------------------------------------------------ */
SV_API int sv_abi_version(void);
/* Replaces module construction (starvector_base.py:22-48): allocates packed weights, KV cache
 * and workspaces on `device`. */
SV_API int sv_engine_create(const sv_model_desc* desc, int device, sv_engine** out);
SV_API void sv_engine_destroy(sv_engine* e);
/* Message for the last failing call on `e` (or the last failing create when e == NULL). */
SV_API const char* sv_last_error(const sv_engine* e);
/* Replaces load_state_dict/from_pretrained: copy one tensor by its reference state-dict name
 * (SURVEY.md §8b "Ownership"), e.g. "model.image_encoder.visual_encoder.conv1.weight".
 * `data` may be a host or device pointer (UVA); borrowed only during the call. */
SV_API int sv_engine_load_weight(sv_engine* e, const char* hf_name, const void* data, const int64_t* shape,
                          int32_t ndim, int32_t dtype);
/* Number of tensors still missing (0 = ready); names (newline separated) via sv_last_error. */
SV_API int sv_engine_missing_weights(sv_engine* e);

/* ---- the hot path --------------------------------------------------------------------- */
/* ImageEncoder.forward + Adapter.forward (image_encoder.py:91-94, adapter.py:33-39,
 * starvector_base.py:206-209).  pixels: bf16 [B,3,S,S].  Result stays resident as the visual
 * prefix; if out_embeds != NULL it is also copied there (bf16 [B,Q,H]).  If vit_out != NULL the
 * pre-adapter `ln_vision` output (bf16 [B,Q,W]) is copied there (parity tests). */
SV_API int sv_encode_images(sv_engine* e, const void* pixels, int32_t batch, void* out_embeds, void* vit_out,
                     void* stream);
/* Prompt embedding + concat (starvector_base.py:213-219) and the decoder prefill over the
 * Q+P prefix (the first forward inside generate(), SURVEY.md §3.1).  prompt_ids int32 [B,P].
 * last_logits (optional) float [B,V]: logits of the last prefix position. */
SV_API int sv_prefill(sv_engine* e, const int32_t* prompt_ids, int32_t batch, int32_t prompt_len,
               float* last_logits, void* stream);
/* The same prefill from caller-provided inputs_embeds bf16 [B,T,H] (the `.generate(inputs_embeds=...)`
 * form of starvector_base.py:255; wpe is added inside, as GPTBigCodeModel.forward does). */
SV_API int sv_prefill_embeds(sv_engine* e, const void* inputs_embeds, int32_t batch, int32_t seq_len,
                             float* last_logits, void* stream);
/* One teacher-forced decode step: feed ids int32 [B], append to the KV cache, return fp32 logits
 * [B,V] (optional).  The parity-test hook; also the body the generate loop replays. */
SV_API int sv_decode_step(sv_engine* e, const int32_t* ids, float* logits, void* stream);
/* Teacher forcing at prefill speed: after sv_prefill / sv_prefill_embeds / sv_expand_batch / sv_decode_step /
 * sv_score_tokens, feed ids int32 [batch, n_tokens] (device; batch == the current batch) at cache positions
 * cur_len .. cur_len+n_tokens-1.  logprobs fp32 [batch, n_tokens] (device): logprobs[b][t] =
 * log softmax(logits before ids[b][t])[ids[b][t]], where t = 0 uses the logits left resident by the previous call.  The
 * logits are bf16 (as HF's lm_head output) and the log-softmax is fp32 over them; they are never written to memory.
 * Leaves the engine as n_tokens sv_decode_step calls would (KV rows appended, cur_len advanced, the last position's bf16
 * logits resident), and the scored tokens become part of the prefix, so sv_generate, a decode step or another
 * sv_score_tokens may follow.  Out-of-range ids are clamped to [0, vocab) for both the embedding and the target.
 * SV_ERR_STATE before a prefill; SV_ERR_INVALID when batch != the current batch, n_tokens < 1 or
 * cur_len + n_tokens > max_len. */
SV_API int sv_score_tokens(sv_engine* e, const int32_t* ids, int32_t batch, int32_t n_tokens, float* logprobs, void* stream);
/* Beam search support (SURVEY.md §8f-1): permute the image rows of the KV cache, row r <- row src_rows[r]
 * (int32 [B] on the device) for the tokens cached so far = HF `_reorder_cache` (vendored modeling_gpt_bigcode.py:1282-1291). */
SV_API int sv_reorder_cache(sv_engine* e, const int32_t* src_rows, void* stream);
/* Prefix-KV sharing (SURVEY.md §8f-4; reference starvector_base.py:261-286 `num_return_sequences`, starvector_arch.py:161-184
 * `vision_embeds.repeat(num_generations, 1, 1)`): directly after sv_prefill / sv_prefill_embeds of b rows, make the engine hold
 * new_batch rows where row r is a copy of prefilled row src_rows_host[r] (HOST int32 [new_batch]): KV cache, last-position
 * logits and generation state are replicated, so the visual prefix is encoded and prefilled once per image, not once per
 * completion.  new_batch <= max_batch. */
SV_API int sv_expand_batch(sv_engine* e, const int32_t* src_rows_host, int32_t new_batch, void* stream);
/* `GenerationMixin._beam_search` after a prefill of batch * num_beams rows (every image repeated num_beams times,
 * adjacent: HF `_expand_inputs_for_generation`): the whole search runs on the device -- per decode step the candidate
 * selection, the beam bookkeeping and the cache permutation (as suffix copies between rows that diverged) follow the
 * lm_head inside the replayed CUDA graph; the host only polls a done flag.  out_ids int32 [batch, max_new_tokens] = the best
 * hypothesis per image (new tokens only, padded with pad_token_id), out_len int32 [batch] = rectangular length (HF's
 * max_generated).  SV_ERR_UNSUPPORTED when a logits row does not fit the SM's shared memory (vocab > ~55k): use the
 * host-stepped loop (sv_decode_step + sv_reorder_cache, starvector_b200/beam_search.py).  Synchronises `stream`. */
SV_API int sv_beam_search(sv_engine* e, const sv_beam_params* p, int32_t batch, int32_t* out_ids, int32_t* out_len,
                          void* stream);
/* Host replays of the device stages of sv_beam_search (no GPU needed; the same bookkeeping code, sv_beam_core.h):
 * parameter validation; size / initialisation / read-out of the opaque state blob; one logits row (fp32 values of the bf16
 * logits) -> its 2 * num_beams best continuations {ordering key, log-prob + running score, token}; one bookkeeping step
 * over row candidates [batch * num_beams][2 * num_beams] with the double-buffered sequence arrays
 * [2][batch * num_beams][seq_stride] -> next tokens, parent rows (= HF beam_idx), returns 1 while the search continues.
 * tests/test_beam_core.py runs whole searches with them against HF generate(num_beams > 1). */
SV_API int sv_beam_params_check(const sv_beam_params* p, int32_t batch);   /* for an engine of 8 rows (the default) */
SV_API int sv_beam_params_check_rows(const sv_beam_params* p, int32_t batch, int32_t max_rows);   /* max_rows <= 16 */
SV_API int sv_beam_state_bytes(void);
SV_API int sv_beam_state_init_host(const sv_beam_params* p, int32_t batch, int32_t first_cache_pos, void* state);
SV_API int sv_beam_state_read_host(const void* state, int32_t* parity, int32_t* cur_len, int32_t* fin_len8,
                                   float* beam_scores8);           /* rows 0-7 */
SV_API int sv_beam_state_read16_host(const void* state, int32_t* parity, int32_t* cur_len, int32_t* fin_len16,
                                     float* beam_scores16, float* running_scores16);
SV_API int sv_beam_row_candidates_host(const sv_beam_params* p, const float* logits, int32_t vocab, const int32_t* seq,
                                       int32_t seq_len, float running_score, int32_t step, int32_t row, float* cand_key,
                                       float* cand_val, int32_t* cand_tok);
SV_API int sv_beam_step_host(const sv_beam_params* p, int32_t batch, int32_t vocab, int32_t seq_stride, void* state,
                             const float* cand_key, const float* cand_val, const int32_t* cand_tok, int32_t* run_seq,
                             int32_t* fin_seq, int32_t cache_hi, int32_t* next_tokens, int32_t* src_rows, int32_t* plan_out);
/* GenerationMixin.generate() after the prefill (greedy / sampling loop, App. B): runs up to
 * max_new_tokens steps as a replayed CUDA graph.  out_ids int32 [B,max_new_tokens] (new tokens
 * only, padded with pad_token_id), out_len int32 [B] = rectangular generated length.
 * Synchronises `stream` before returning. */
SV_API int sv_generate(sv_engine* e, const sv_gen_params* p, int32_t* out_ids, int32_t* out_len, void* stream);
/* sv_generate with token streaming (SURVEY.md §8f-4: serve/model_worker.py:161-181 hands a `streamer` to generate(),
 * which the reference's kwarg whitelist drops, starvector_base.py:223-241).  Every `poll_interval` steps, and once at the
 * end, `on_tokens(user, ids_host, batch, first_step, n_steps)` is called on the calling thread with the new tokens of
 * every row, ids_host int32 [batch][n_steps] (valid during the call); the concatenation over calls is exactly the
 * rectangle sv_generate returns.  A non-zero return cancels the generation after the current poll. */
typedef int (*sv_token_callback)(void* user, const int32_t* ids_host, int32_t batch, int32_t first_step, int32_t n_steps);
SV_API int sv_generate_stream(sv_engine* e, const sv_gen_params* p, int32_t* out_ids, int32_t* out_len,
                              sv_token_callback on_tokens, void* user, void* stream);
/* Whole path with HOST buffers (copies inside): pixels_host bf16 [B,3,S,S], prompt_ids_host
 * int32 [B,P] -> out_ids_host int32 [B,max_new_tokens], out_len_host int32 [B]. */
SV_API int sv_generate_im2svg_host(sv_engine* e, const void* pixels_host, int32_t batch,
                            const int32_t* prompt_ids_host, int32_t prompt_len, const sv_gen_params* p,
                            int32_t* out_ids_host, int32_t* out_len_host, void* stream);

/* ---- prompt-lookup speculative decoding (HF generate(prompt_lookup_num_tokens=k), DESIGN.md §7g) ------------------ */
typedef struct sv_spec_params {
  int32_t num_tokens;               /* k = prompt_lookup_num_tokens: drafts per verify step, 1 <= k <= max_batch - 1 (<= 15) */
  int32_t max_matching_ngram_size;  /* >= 1 (HF default 2) */
} sv_spec_params;
/* sv_generate (sv_generate_stream when on_tokens != NULL) with drafts from n-gram matches in the row's own generated
 * tokens, verified k + 1 columns of one cache row per weight stream.  Returns the same out_ids rectangle, out_len and
 * cache length as sv_generate with the same parameters, bit for bit (greedy and sampling, every stop rule): the drafts
 * change the speed only.  One image (batch 1), v1 engines on the fused graph decode path (SV_FLOW engines run it on the
 * graph path).  SV_ERR_UNSUPPORTED for v2, SV_DECODE=legacy, batch > 1 or an open session; SV_ERR_INVALID for k outside
 * [1, max_batch - 1] or an n-gram size < 1.  Synchronises `stream`. */
SV_API int sv_generate_speculative(sv_engine* e, const sv_gen_params* p, const sv_spec_params* sp, int32_t* out_ids,
                                   int32_t* out_len, sv_token_callback on_tokens, void* user, void* stream);
/* Counters of the last sv_generate_speculative: verify steps, drafts proposed, drafts accepted (any pointer may be NULL). */
SV_API int sv_last_spec_stats(const sv_engine* e, int32_t* steps, int32_t* drafted, int32_t* accepted);
/* Teacher-forced verify step (tests): after a one-image prefill (and any sv_decode_step calls), feeds ids_host[0, ncols) as
 * the columns of one verify forward at positions cur_len + c and writes their logits, fp32 [ncols][vocab].  Column c's
 * logits are those the (c + 1)-th of ncols successive sv_decode_step calls with these ids returns, bit for bit, when the
 * decode attention's cluster size (attention_decode_cluster_ncta of the length) is the same for all of them.  The K/V of
 * the columns are written, the cache length does not advance.  Synchronises `stream`. */
SV_API int sv_spec_verify_step(sv_engine* e, const int32_t* ids_host, int32_t ncols, float* logits, void* stream);
/* Host replays of the device rules (tests): the drafts proposed after the history hist[0, n) (returns their count, <= k,
 * written to out), and one accept walk: columns' selected tokens sel[0, n_live) against the column inputs cols (cols[c] =
 * draft c for c >= 1) with the plain path's per-token bookkeeping on state {cur_len, step, done} and out_ids (returns the
 * number of tokens emitted). */
SV_API int sv_spec_draft_host(const int32_t* hist, int32_t n, int32_t k, int32_t max_ngram, int32_t eos_id, int32_t budget,
                              int32_t* out);
SV_API int sv_spec_accept_host(const sv_gen_params* p, int32_t* state, int32_t* out_ids, int32_t out_stride,
                               const int32_t* sel, const int32_t* cols, int32_t n_live);

/* ---- continuous batching (vLLM-style serving; the reference's fast validator backend,
 * starvector/validation/starvector_vllm_svg_validator.py) -------------------------------------- */
/* A decode session keeps `slots` (<= max_batch) cache rows; every row decodes at its own position, has its own token cap
 * and Philox seed and finishes on its own (EOS, the '</svg>' stop sequence over its own tokens, or its cap).  A finished
 * row is refilled by sv_session_admit while the other rows keep their caches; the decode graph (captured once per session
 * shape) then continues.  Every request gets the tokens a one-image sv_generate with the same parameters gives
 * (greedy and sampling, bit for bit), up to and including its stop.  While a session is open, sv_encode_images,
 * sv_prefill*, sv_decode_step, sv_score_tokens, sv_generate*, sv_beam_search, sv_reorder_cache, sv_expand_batch and
 * sv_engine_load_weight return SV_ERR_STATE.  The session runs the CUDA-graph decode path (never the SV_FLOW dataflow kernel).
 * Beam search has its own session form (sv_beam_session_begin / sv_beam_session_admit below).
 *
 * sv_session_begin: p = the session's generation parameters: max_new_tokens is the session cap (it fixes the decode
 * attention's split count together with the prompt length, as prefix + max_new_tokens does in sv_generate), eos, stop ids
 * (always per row; stop_row0_only is ignored), sampling parameters, seed (the default of admitted rows), poll_interval. */
SV_API int sv_session_begin(sv_engine* e, const sv_gen_params* p, int32_t slots);
/* Encode and prefill images into free slots.  pixels bf16 [n_img,3,S,S] and prompt_ids int32 [n_img,prompt_len] (device);
 * slots_host int32 [k]: the slots to fill; src_host int32 [k] (NULL = identity): the image index of each slot, so an
 * image listed for n slots is prefilled once and its cache rows copied (n completions); max_new_host int32 [k] (NULL =
 * the session cap, else in [1, cap]); seeds_host uint64 [k] (NULL = the session seed).  Token 0 of every admitted slot is
 * selected here.  The prompt length is fixed by the first admission of the session; prefix + cap <= max_len.  Each image
 * is encoded and prefilled at batch 1, with the kernels a one-image generate uses.  Synchronises `stream`. */
SV_API int sv_session_admit(sv_engine* e, const void* pixels, int32_t k, const int32_t* prompt_ids, int32_t prompt_len,
                            const int32_t* slots_host, const int32_t* max_new_host, const uint64_t* seeds_host,
                            const int32_t* src_host, void* stream);
/* Replay the decode graph for up to max_steps steps, polling every poll_interval steps; returns (the number of steps run,
 * >= 0) as soon as a poll finds a finished slot or no slot decoding.  finished_host int32 [slots] (optional): 1 for the
 * slots whose finish this call reports (each finish is reported once; the slot is free again), len_host int32 [slots]
 * (optional): tokens each slot holds.  Synchronises `stream`. */
SV_API int sv_session_run(sv_engine* e, int32_t max_steps, int32_t* finished_host, int32_t* len_host, void* stream);
/* Speculative session (DESIGN.md §7i): sv_session_begin with prompt-lookup drafts in the columns the live rows leave
 * free.  Every verify step streams the weights once for `slots` columns: each live row gets one column for its last token,
 * and the spare columns carry drafts from n-gram matches in the rows' own tokens (up to sp->num_tokens per row, handed
 * out round-robin in slot order).  Every request gets the tokens it gets in a plain session, bit for bit; the drafts change
 * the speed only.  Admit, run (max_steps counts verify steps), read and end as for a plain session.  v1 engines on the fused
 * graph decode path (SV_FLOW engines run it on the graph path).  SV_ERR_UNSUPPORTED for v2 and SV_DECODE=legacy;
 * SV_ERR_INVALID for num_tokens outside [1, slots - 1] or an n-gram size < 1. */
SV_API int sv_session_begin_speculative(sv_engine* e, const sv_gen_params* p, const sv_spec_params* sp, int32_t slots);
/* Counters of the open speculative session: verify steps, drafts proposed, drafts accepted (any pointer may be NULL).
 * SV_ERR_STATE unless a speculative session is open.  Synchronises the engine's stream. */
SV_API int sv_session_spec_stats(sv_engine* e, int32_t* steps, int32_t* drafted, int32_t* accepted);
/* Copy the tokens of `slot` (as of the last sv_session_run) to ids (int32, host or device); returns their count. */
SV_API int sv_session_read(sv_engine* e, int32_t slot, int32_t* ids, void* stream);
/* Close the session: the rectangle-batch entry points work again (after a new prefill). */
SV_API int sv_session_end(sv_engine* e);
/* Beam sessions: continuous batching of sv_beam_search.  The `slots` cache rows form slots / num_beams groups; group g owns
 * rows [g * num_beams, (g + 1) * num_beams) and runs one image's beam search (beam-sample with do_sample) with its own
 * token cap and seed, while the other groups keep decoding.  A request whose cap equals the session cap gets the token ids
 * and length the one-image sv_beam_search (after a prefill of the image repeated num_beams times) returns with the same
 * parameters, bit for bit; a smaller cap gets the same as the one-image search at that cap when the decode attention's
 * partition of prefix + cap equals that of prefix + session cap.  sv_session_run, sv_session_read and sv_session_end serve
 * beam sessions: the run reports a finished group at its first slot, sv_session_read(first slot) returns its best
 * hypothesis.  sv_session_admit is refused in a beam session, sv_beam_session_admit in a plain one.
 *
 * sv_beam_session_begin: p->max_new_tokens is the session cap; num_beams >= 2, slots a multiple of num_beams, <= max_batch.
 * p->seed is the default seed of admitted groups.  SV_ERR_UNSUPPORTED when a logits row does not fit the candidate kernel. */
SV_API int sv_beam_session_begin(sv_engine* e, const sv_beam_params* p, int32_t slots);
/* Encode and prefill k images into free groups: pixels bf16 [k,3,S,S] and prompt_ids int32 [k,prompt_len] (device);
 * groups_host int32 [k] the groups to fill; max_new_host int32 [k] (NULL = the session cap, else in [1, cap]); seeds_host
 * uint64 [k] (NULL = the session seed).  Each image is encoded and prefilled repeated num_beams times, as a one-image
 * beam search does, and the search's first step runs here.  The prompt length is fixed by the first admission; prefix +
 * cap <= max_len.  Synchronises `stream`. */
SV_API int sv_beam_session_admit(sv_engine* e, const void* pixels, int32_t k, const int32_t* prompt_ids, int32_t prompt_len,
                                 const int32_t* groups_host, const int32_t* max_new_host, const uint64_t* seeds_host,
                                 void* stream);

/* ---- introspection for bench/profiles ------------------------------------------------- */
/* Kernel launches issued by this engine since creation (graph replays count their nodes). */
SV_API int64_t sv_launch_count(const sv_engine* e);
/* Human-readable configuration of the engine (decode mode, PDL, kernel selection) for logs/bench JSON. */
SV_API const char* sv_engine_describe(sv_engine* e);
/* Debug (SV_MEGA_DEBUG=1): timeline records of CTA 0 for the first token of the last persistent-decode launch,
 * `id << 48 | SM clock` (ids: sv_decode_flow.cu); entries [0,4096) consumer thread 0, [4096,8192) producer warp;
 * unused entries are 0; n <= 8192. */
SV_API int sv_debug_read_timeline(sv_engine* e, long long* out_host, int32_t n);
/* Device time (ms) of the last sv_generate decode loop and its step count, from CUDA events
 * recorded on the launching stream. */
SV_API int sv_last_decode_timing(const sv_engine* e, float* ms, int32_t* steps);

/* ---- single-kernel entry points (unit parity tests; all bf16 unless noted) -------------- */
SV_API int sv_op_layernorm(const void* x, const void* w, const void* b, void* y, int32_t rows, int32_t cols,
                    float eps, void* stream);
/* y[M,N] = act(x[M,K] . w[N,K]^T + bias[N]) (+ residual[M,N]); rounding points follow the
 * reference's bf16 module boundaries (DESIGN.md §numerics). */
SV_API int sv_op_linear(int32_t impl, const void* x, const void* w, const void* bias, const void* residual, void* y,
                 int32_t M, int32_t N, int32_t K, int32_t act, void* stream);
/* ViT self-attention over packed qkv [B*L, 3*heads*64] -> out [B*L, heads*64]. */
SV_API int sv_op_attention_vit(const void* qkv, void* out, int32_t batch, int32_t seq, int32_t heads, void* stream);
/* Causal multi-query attention over packed qkv [B*T, heads*D + 2*D] (D=128) -> out [B*T, heads*D]: sv_op_attention_prefill
 * over zeroed caches this call allocates. */
SV_API int sv_op_attention_mqa(const void* qkv, void* out, int32_t batch, int32_t seq, int32_t heads, void* stream);
/* The scoring chunk attention: packed qkv [B*seq, (n_head + 2*n_kv)*D] (D=128) fills a cache with all seq positions;
 * the queries of positions [q0, seq) attend causally (keys > pos - window when window > 0) -> out [B*(seq-q0), n_head*D].
 * sv_op_attention_score over zeroed caches this call allocates. */
SV_API int sv_op_attention_chunk(const void* qkv, void* out, int32_t batch, int32_t seq, int32_t q0, int32_t n_head,
                                 int32_t n_kv, int32_t window, void* stream);
/* The fused lm_head log-likelihood: logprob fp32 [M] = log_softmax(float(bf16(x[M,K] . w[N,K]^T)))[m, targets[m]],
 * targets int32 [M] (device); any N >= 1, K % 64 == 0, x and w 16-byte aligned.  A target outside [0, N) gives NaN.
 * Checked on the host (SV_ERR_INVALID before any launch); synchronous on `stream`. */
SV_API int sv_op_lm_logprob(const void* x, const void* w, const int32_t* targets, float* logprob, int32_t M, int32_t N,
                            int32_t K, void* stream);

/* The decode-step kernels one at a time, over caches the caller fills (D = 128; kcache [batch][n_kv][tcap][D], vtcache
 * [batch][n_kv][D][tcap], packed qkv rows [batch][(n_head + 2 n_kv) * D]).  Every argument is checked on the host:
 * SV_ERR_INVALID before any launch.  Synchronous on `stream`. */
enum { SV_ATTN_DECODE_SPLIT = 0 /* split + merge, nsplit in [1, 128] */, SV_ATTN_DECODE_CLUSTER = 1 /* nsplit = CTAs in [1, 8] */ };
/* Decode attention: row b's query (qkv row b) attends to keys [0, lens_host[b]) of its cache (the last, lens - 1, is the
 * new token; keys > lens - 1 - window when window > 0) -> out [batch][n_head * D].  per_row = 0: the plain kernels
 * (equal lengths); 1: the session kernels.  1 <= lens <= tcap, tcap % 32 == 0, batch <= 16, n_head / n_kv <= 16.
 * per_row = 2: the column map of a speculative verify step (SV_ATTN_DECODE_CLUSTER only, window 0): column c (qkv row c)
 * attends to keys [0, lens_host[c]] of cache row 0, i.e. lens_host[c] is the column's position, in [0, tcap - 1]. */
SV_API int sv_op_attention_decode(int32_t impl, int32_t per_row, const void* qkv, const void* kcache, const void* vtcache,
                                  void* out, const int32_t* lens_host, int32_t batch, int32_t n_head, int32_t n_kv,
                                  int32_t tcap, int32_t nsplit, int32_t window, void* stream);
/* One weight-ring GEMV launch: y[B,N] = epi(LN?(x)[B,K] . w[N,K]^T) with the decode step's rounding points. */
typedef struct sv_op_ring {
  const void *x, *w, *bias, *residual; /* residual may alias y (in place) */
  const void *ln_w, *ln_b;             /* both NULL: no LayerNorm */
  void* y;
  int32_t B, N, K, act;
  int32_t epi;                         /* 0 plain, 1 QKV + KV append (needs LN), 2 lm_head + argmax partials (needs LN) */
  int32_t tiled;                       /* 1: stream a slab-tiled copy of w (built by the call) instead of w's rows */
  float ln_eps;
  void *kcache, *vtcache;              /* epi 1 */
  int32_t n_head, n_kv, tcap, per_row;
  const int32_t* pos_host;             /* epi 1: the append position (per_row = 0: [0] for every row; 1: one per row;
                                          2: the column map of a speculative verify step, [B + 1]: pos_host[c] = column c's
                                          position in cache row 0, in [0, tcap - 1], then n_live = pos_host[B]: columns
                                          [0, n_live) append their K/V, the others write nothing; pos_host[0] + n_live <= tcap) */
  float* amax_val;                     /* epi 2: [sv_op_ring_ntiles(N)][sv_op_ring_row_stride(B)] */
  int32_t* amax_idx;
} sv_op_ring;
SV_API int sv_op_gemv_ring(const sv_op_ring* args, void* stream);
SV_API int32_t sv_op_ring_ntiles(int32_t N);
SV_API int32_t sv_op_ring_row_stride(int32_t B);
/* The bf16 RoPE tables cos/sin [max_pos][d / 2] the engine builds for theta. */
SV_API int sv_op_rope_table(void* cos_t, void* sin_t, int32_t max_pos, int32_t d, float theta, void* stream);
/* RoPE in place on the q and k heads of packed qkv [rows][(n_head + 2 n_kv) * D] (positions >= max_pos use max_pos - 1).
 * pos_host == NULL: the prefill kernel, row r at pos0 + r % seq.  Otherwise one token per row at pos_host[0] (per_row = 0,
 * equal positions) or pos_host[r] (per_row = 1); with kcache != NULL the append kernel: q rotated in place, rotated k
 * and v written to the caches at the row's position when it is < tcap. */
SV_API int sv_op_rope(void* qkv, const void* cos_t, const void* sin_t, int32_t rows, int32_t seq, int32_t n_head,
                      int32_t n_kv, int32_t max_pos, int32_t pos0, const int32_t* pos_host, int32_t per_row, void* kcache,
                      void* vtcache, int32_t tcap, void* stream);
/* The decode step as the engine chains it (the same host code as sv_decode_step), over weights, caches and activation
 * buffers the caller owns: layers [0, n_layer) then, optionally, the lm_head.  Same conventions as the ops above (every
 * argument checked on the host, SV_ERR_INVALID before any launch; synchronous on `stream`).
 * SV_CHAIN_FUSED: per layer the c_attn ring GEMV (LayerNorm fused; v1 appends K/V in its epilogue, RoPE models run the
 * RoPE + append kernel after it), the cluster attention, and the c_proj / c_fc / c_fc2 ring GEMVs; the tail is the lm_head
 * ring with its argmax partials.  SV_CHAIN_PER_OP: LayerNorm, rowgroup GEMVs, RoPE, KV append and split attention; the
 * tail is ln_f + the rowgroup lm_head.
 * Activation slots: x[2l] is layer l's input (the embedding of ids, or the caller's when ids is NULL), x[2l + 1] the
 * residual stream after its attention, x[2l + 2] its output; ln[2l], ln[2l + 1] its two LayerNorm outputs and ln[2 n_layer]
 * ln_f's (PER_OP only); qkv[l], attn[l], h[l].  Slot k of buffer p is p + k * p_stride elements: stride 0 reuses one
 * buffer for every layer (the engine's aliasing, the residual stream updated in place); a nonzero stride is at least one
 * slot ([B][width]) and keeps every layer's intermediates. */
enum { SV_CHAIN_FUSED = 0, SV_CHAIN_PER_OP = 1 };
typedef struct sv_op_chain_layer {
  const void *ln1_w, *ln1_b, *attn_w, *attn_b, *proj_w, *proj_b, *ln2_w, *ln2_b, *fc_w, *fc_b, *fc2_w, *fc2_b;
} sv_op_chain_layer;
typedef struct sv_op_chain {
  int32_t mode;                        /* SV_CHAIN_* */
  int32_t n_layer, B;                  /* layers run (from layer 0) >= 1; rows in [1, 16] */
  int32_t per_row;                     /* 0: every row at pos_host[0] (GenState); 1: row b at pos_host[b] (RowState, sessions) */
  int32_t hidden, n_inner, n_head, n_kv, vocab, n_positions, tcap, window;   /* hidden = n_head * 128 */
  float ln_eps;
  int32_t rope;                        /* 1: StarCoder2 (RoPE on q and k; rope_cos / rope_sin [n_positions][64]) */
  const sv_op_chain_layer* layers;     /* host array [n_layer] */
  const void *wte, *wpe;               /* wpe may be NULL (no learned positions) */
  const void *lnf_w, *lnf_b, *lm_head, *rope_cos, *rope_sin;
  void *kcache, *vtcache;              /* [layer][B][n_kv][tcap][128] / [layer][B][n_kv][128][tcap], layer_stride apart */
  int64_t layer_stride;
  const int32_t* ids;                  /* device int32 [B] or NULL */
  const int32_t* pos_host;             /* [B]: the position each row's token takes, in [0, tcap - 1] (the appended slot) */
  void *x, *ln, *qkv, *attn, *h;
  int64_t x_stride, ln_stride, qkv_stride, attn_stride, h_stride;
  int32_t lm_head_tail;                /* 1: the tail; logits [B][vocab], FUSED also amax_val / amax_idx */
  void* logits;                        /*   [sv_op_ring_ntiles(vocab)][sv_op_ring_row_stride(B)] */
  float* amax_val;
  int32_t* amax_idx;
  int32_t pdl;                         /* FUSED: programmatic dependent launch between the chain's kernels */
  int32_t graph;                       /* 1: capture the chain in a CUDA graph once and launch the graph */
  int32_t tiled;                       /* FUSED: stream slab-tiled copies of the weights (built by the call) */
  int32_t parts;                       /* CTAs per cluster (FUSED, <= 8) / splits (PER_OP, <= 128); 0: the engine's rule */
  int32_t parts_used;                  /* out: the cluster size / split count the attention ran with */
  int32_t pdl_used;                    /* out: 1 if the chain ran with PDL edges (graph: the PDL capture was accepted) */
} sv_op_chain;
SV_API int sv_op_decode_chain(sv_op_chain* args, void* stream);

/* The dataflow decode kernel (SV_FLOW=1 engines: decode_flow_kernel, `nsteps` whole tokens per cooperative launch) over
 * weights, caches and exchange buffers the caller owns.  The call builds the slab-tiled weight copies the kernel streams,
 * runs ONE launch and waits for it.  Activations travel between CTAs as flagged words: a 32-bit word holds a bf16 value
 * (low half) and a phase tag (high half), word i of a row sits at (i >> 3) * 64 + (i & 7), rows are (n >> 3) * 64 words
 * apart; attention partials are 64-bit words (fp32 value, 32-bit tag), each lm_head argmax partial a 64-bit word
 * [tag16 | bf16 | index] at tile * 8 + row.  The tag of phase gp = step * (n_layer + 1) + layer is
 * ((gp & 0x7fff) + 1) << 16 (the lm_head is "layer n_layer"; tag32: (gp + 1) << 32).  After a launch the buffers hold the
 * last step's words: qkv, att, xb, hb of the last layer, xa its output (tag of the lm_head phase), or with do_select the
 * next step's input (tag of (step + 1) * (n_layer + 1)).
 * Every argument is checked on the host and refused with SV_ERR_INVALID before any launch, including every combination
 * the kernel could not complete: first_plain = 0 needs xa words carrying the first step's tag (the call reads them back).
 * Synchronous on `stream`. */
enum { SV_FLOW_XA = 0, SV_FLOW_XB = 1, SV_FLOW_QKV = 2, SV_FLOW_ATT = 3, SV_FLOW_HB = 4, SV_FLOW_PART = 5, SV_FLOW_AMAX = 6 };
/* bytes of exchange buffer `which` (SV_FLOW_*) for these dims (amax: room for any number of SMs); -1 if out of range */
SV_API int64_t sv_op_flow_buffer_bytes(int32_t which, int32_t B, int32_t hidden, int32_t n_inner, int32_t n_kv, int32_t vocab);
typedef struct sv_op_flow {
  int32_t n_layer, B;                  /* [1, 24] layers from layer 0; rows in [1, 8] */
  int32_t hidden, n_inner, n_head, n_kv, vocab, n_positions, tcap;   /* hidden = n_head * 128 */
  float ln_eps;
  const sv_op_chain_layer* layers;     /* host array [n_layer] */
  const void *wte, *wpe;               /* wpe may be NULL */
  const void *lnf_w, *lnf_b, *lm_head;
  void *kcache, *vtcache;              /* [layer][B][n_kv][tcap][128] / [layer][B][n_kv][128][tcap], layer_stride apart */
  int64_t layer_stride;
  int32_t nsteps;                      /* tokens in the launch */
  int32_t step0;                       /* phase-tag epoch of its first step (steps since the buffers were cleared) */
  int32_t cur_len0;                    /* tokens in the cache at the start; cur_len0 + nsteps <= tcap - 1 */
  int32_t first_plain;                 /* 1: the first step's input is x_plain (bf16 [B][hidden]) */
  int32_t do_select;                   /* 1: greedy selection + HF bookkeeping + the next token's embedding after every step */
  int32_t l2_ahead;                    /* weight slabs the L2 prefetch warp runs ahead of the ring, [0, 64] */
  int32_t realloc;                     /* 1: the register-reallocating variant (SV_FLOW=1), 0: the plain one (SV_FLOW=3) */
  int32_t clear;                       /* 1: zero the seven exchange buffers first (a new sequence; needs first_plain) */
  sv_gen_params params;                /* do_select: greedy (do_sample = 0); repetition_penalty is read in any case */
  int32_t out_stride;                  /* do_select: columns of out_ids */
  int32_t* counters_host;              /* do_select: [3] step, cur_len, done; read on entry, written back */
  int32_t* unfinished_host;            /* do_select: [B], read on entry, written back */
  void* seen;                          /* do_select: uint8 [B][vocab] */
  int32_t *out_ids, *next_ids;         /* do_select: [B][out_stride], [B] */
  void *x_plain, *logits;              /* bf16 [B][hidden] (refreshed by every select), bf16 [B][vocab] (the last step's) */
  void *xa, *xb, *qkv, *att, *hb, *part, *amax;   /* exchange buffers, sv_op_flow_buffer_bytes each */
  int32_t ncta_used;                   /* out: CTAs of the launch (one per SM) */
  int32_t realloc_used;                /* out: 1 if the register-reallocating variant ran */
} sv_op_flow;
SV_API int sv_op_decode_flow(sv_op_flow* args, void* stream);

/* The token-selection kernels one launch at a time: what follows the logits of a decode step.  The caller owns the device
 * tensors; the generation state travels as HOST arrays that are read on entry and written back on return.  The same
 * logits are selected from `nsteps` times in one call, the bookkeeping advancing between the launches (B x nsteps draws
 * of the sampler).  Every argument is checked on the host: SV_ERR_INVALID before any launch.  Synchronous on `stream`. */
enum {
  SV_SELECT_GREEDY = 0, /* select_greedy(_rows)_kernel; per_row = 0: followed by gen_finalize_kernel */
  SV_SELECT_SAMPLE = 1, /* select_sample(_rows)_kernel; per_row = 0: followed by gen_finalize_kernel (fp32 scratch allocated here) */
  SV_SELECT_FUSED = 2   /* select_fused(_rows)_kernel: greedy + bookkeeping + the next token's embedding in one launch */
};
typedef struct sv_op_select_args {
  int32_t impl;                 /* SV_SELECT_* */
  int32_t per_row;              /* 0: the rectangle-batch kernels; 1: the session kernels (every row has its own state) */
  const void* logits;           /* bf16 [B][vocab] */
  int32_t vocab, B;             /* vocab >= 1, B in [1, 16] */
  sv_gen_params params;         /* max_new_tokens is the plain kernels' cap; poll_interval is ignored */
  void* seen;                   /* uint8 [B][vocab]: ids generated so far (repetition penalty), updated */
  int32_t* out_ids;             /* [B][out_stride] */
  int32_t* next_ids;            /* [B] */
  int32_t out_stride, advance_len, nsteps;
  /* per_row = 0 (GenState) */
  int32_t* counters_host;       /* [3]: step, cur_len, done */
  int32_t* unfinished_host;     /* [B] */
  /* per_row = 1 (RowState): rows b with bit b of row_mask set and row_active[b] != 0 select */
  int32_t *row_len_host, *row_step_host, *row_active_host, *row_max_new_host;   /* [B] each */
  uint64_t* row_seed_host;      /* [B] */
  uint32_t row_mask;
  int32_t* event_host;          /* [1] */
  /* SV_SELECT_FUSED only */
  const float* amax_val;        /* lm_head argmax partials [sv_op_ring_ntiles(vocab)][sv_op_ring_row_stride(B)], or NULL: */
  const int32_t* amax_idx;      /*   the logits rows are scanned (always so when repetition_penalty != 1) */
  const void *wte, *wpe;        /* bf16 [vocab][h], [n_positions][h]; wpe may be NULL (RoPE models) */
  void* x;                      /* bf16 [B][h]: the selected tokens' embeddings at their post-advance positions */
  int32_t h, n_positions;       /* h % 8 == 0 */
} sv_op_select_args;
SV_API int sv_op_select(const sv_op_select_args* args, void* stream);
/* The selection kernels of a speculative verify step (sv_generate_speculative, one image row) one launch at a time, same
 * conventions as sv_op_select: the state travels as host structs read on entry and written back. */
enum {
  SV_SPEC_GREEDY = 0,  /* select_fused_spec_kernel: per-column greedy selection, the accept walk, next drafts and embeddings */
  SV_SPEC_SAMPLE = 1,  /* select_sample_spec_kernel (writes sel), then spec_accept_kernel, as the sampled verify graph runs them */
  SV_SPEC_ACCEPT = 2   /* spec_accept_kernel alone on the given sel (n_live = 0: the first drafts of a generation) */
};
/* The device state of one speculative generation (svspec::State, sv_spec_core.h), field for field. */
typedef struct sv_spec_state {
  int32_t n_live, row[16], pos[16];  /* the column map: column c < n_live decodes (row[c], pos[c]); the others are inert */
  int32_t tok[16], sel[16];          /* column inputs (tok[0] the last token, tok[c] draft c) and selected tokens */
  int32_t ncols, k, max_ngram;       /* columns (k + 1), drafts per step, the largest n-gram matched */
  int32_t steps, drafted, accepted;  /* counters */
} sv_spec_state;
typedef struct sv_op_spec_args {
  int32_t impl;                 /* SV_SPEC_* */
  const void* logits;           /* bf16 [ncols][vocab] (GREEDY, SAMPLE) */
  int32_t vocab;                /* >= 1 */
  sv_gen_params params;         /* max_new_tokens <= out_stride is the cap; do_sample and poll_interval are ignored */
  void* seen;                   /* uint8 [vocab]: ids generated so far (repetition penalty), updated */
  int32_t* out_ids;             /* [out_stride]: the generated ids (the draft history), updated */
  int32_t* next_ids;            /* [1] */
  int32_t out_stride;
  int32_t* gen_host;            /* [4]: step, cur_len, done, unfinished[0] */
  sv_spec_state* spec_host;
  const float* amax_val;        /* GREEDY only: lm_head argmax partials [sv_op_ring_ntiles(vocab)][sv_op_ring_row_stride(ncols)], */
  const int32_t* amax_idx;      /*   or NULL: the logits rows are scanned (always so when repetition_penalty != 1) */
  const void *wte, *wpe;        /* bf16 [vocab][h], [n_positions][h]; wpe may be NULL */
  void* x;                      /* bf16 [ncols][h]: the next step's column inputs */
  int32_t h, n_positions;       /* h % 8 == 0 */
} sv_op_spec_args;
SV_API int sv_op_spec_select(const sv_op_spec_args* args, void* stream);

/* ---- speculative sessions: host replays and one-launch hooks (tests) ---- */
/* The per-row state of a session (RowState), field for field. */
typedef struct sv_session_rows {
  int32_t row_len[16], row_step[16], row_active[16], event, pad_, row_max_new[16];
  uint64_t row_seed[16];
} sv_session_rows;
/* The device state of a speculative session (svspec::SessionState), field for field. */
typedef struct sv_spec_session_state {
  int32_t n_live, row[16], pos[16];  /* the column map: column c < n_live decodes (row[c], pos[c]); the others are inert */
  int32_t tok[16], sel[16], off[16]; /* column inputs, selected tokens, each column's offset within its row */
  int32_t ncols, k, max_ngram;       /* columns (the session's slots), drafts per row at most, the largest n-gram matched */
  int32_t steps, drafted, accepted;  /* counters */
} sv_spec_session_state;
/* The column allocation of a verify step: S slots, active[r] != 0 for the live rows, want[r] the drafts row r asks for,
 * at most `budget` (and S) columns in all.  Every live row gets one column; the spare columns go round-robin in slot order,
 * one draft per pass to each row below its want.  Writes g[r] (drafts granted) and first[r] (the row's first column, -1
 * for idle rows); returns n_live (the columns used), or SV_ERR_INVALID. */
SV_API int sv_spec_session_plan_host(int32_t S, const int32_t* active, const int32_t* want, int32_t budget, int32_t* g,
                                     int32_t* first);
/* What the session's tail kernel does, on the host: with `accept`, every live row's accept walk on ss->sel with the plain
 * session's per-token bookkeeping (rows, out_ids [S][out_stride]); then the next drafts, the allocation (column budget:
 * tcap, the KV cache's row capacity, see DESIGN.md §7i) and the column map into ss.  Returns the next n_live, or
 * SV_ERR_INVALID. */
SV_API int sv_spec_session_tail_host(const sv_gen_params* p, sv_session_rows* rows, int32_t* out_ids, int32_t out_stride,
                                     sv_spec_session_state* ss, int32_t accept, int32_t tcap);
enum {
  SV_SPEC_SESSION_GREEDY = 0,  /* spec_session_select_fused_kernel: per-column greedy selection, then the tail */
  SV_SPEC_SESSION_SAMPLE = 1,  /* spec_session_select_sample_kernel (writes sel), then spec_session_tail_kernel with accept */
  SV_SPEC_SESSION_TAIL = 2     /* spec_session_tail_kernel alone on the given sel, accept as given */
};
typedef struct sv_op_spec_session_args {
  int32_t impl;                 /* SV_SPEC_SESSION_* */
  int32_t accept;               /* TAIL: 1 accepts ss->sel first, 0 only re-plans (as after an admission) */
  const void* logits;           /* bf16 [ncols][vocab] (GREEDY, SAMPLE) */
  int32_t vocab;                /* >= 1 */
  sv_gen_params params;         /* eos, stop ids, penalty, sampling; do_sample, seed and poll_interval are ignored */
  void* seen;                   /* uint8 [ncols][vocab]: each slot's generated ids (repetition penalty), updated */
  int32_t* out_ids;             /* [ncols][out_stride]: each slot's generated ids (the draft history), updated */
  int32_t* next_ids;            /* [ncols] */
  int32_t out_stride;
  int32_t tcap;                 /* >= every live row's row_max_new + its prefix: the KV row capacity the budget uses */
  sv_session_rows* rows_host;
  sv_spec_session_state* ss_host;
  const float* amax_val;        /* GREEDY only: lm_head argmax partials [sv_op_ring_ntiles(vocab)][sv_op_ring_row_stride(ncols)], */
  const int32_t* amax_idx;      /*   or NULL: the logits rows are scanned (always so when repetition_penalty != 1) */
  const void *wte, *wpe;        /* bf16 [vocab][h], [n_positions][h]; wpe may be NULL */
  void* x;                      /* bf16 [ncols][h]: the next step's column inputs */
  int32_t h, n_positions;       /* h % 8 == 0 */
} sv_op_spec_session_args;
SV_API int sv_op_spec_session_select(const sv_op_spec_session_args* args, void* stream);
/* One beam_candidates_kernel launch over R = batch * num_beams rows: logits bf16 [R][vocab]; cur_len = tokens every
 * running beam holds (0: no repetition penalty yet), running_scores_host float [R], run_seq int32 [R][seq_stride] (device,
 * the beams' generated ids) -> cand_key / cand_val float and cand_tok int32 [R][2 * num_beams] (device).  p is checked as
 * sv_beam_params_check_rows(p, batch, 16) does; a vocab whose row does not fit the SM's shared memory is SV_ERR_INVALID. */
SV_API int sv_op_beam_candidates(const void* logits, int32_t vocab, const sv_beam_params* p, int32_t batch, int32_t cur_len,
                                 const float* running_scores_host, const int32_t* run_seq, int32_t seq_stride,
                                 float* cand_key, float* cand_val, int32_t* cand_tok, void* stream);

/* The beam-search bookkeeping and KV-cache movement kernels one launch at a time (what follows beam_candidates_kernel in
 * sv_beam_search, and the cache copies of sv_reorder_cache, sv_expand_batch and sv_session_admit).  Same conventions as
 * sv_op_select: the caller owns the device tensors, host-side state travels as host structs read on entry and written
 * back, every argument is checked on the host (SV_ERR_INVALID before any launch), synchronous on `stream`. */
/* The device state of one beam search (svbeam::State, sv_beam_core.h), field for field; the same bytes as the state blob
 * of sv_beam_state_init_host / sv_beam_step_host.  Rows r = b * num_beams + j. */
typedef struct sv_beam_state {
  int32_t cur_len, done, parity, pad_;   /* generated tokens per running beam, search over, live half of the sequence arrays */
  float running_scores[16], beam_scores[16];
  int32_t is_finished[16], fin_len[16];
  int32_t unsatisfied[16];               /* per image */
  int32_t div[16][16];                   /* first cache position at which rows r and q (same image) differ */
} sv_beam_state;
/* What one step decided (svbeam::Plan): new running row r = old row run_parent[r] + run_tok[r]; finished slot r = old
 * finished row fin_old[r] (>= 0) or old running row fin_parent[r] + fin_tok[r]; KV row r <- row copy_src[r] (-1: none)
 * over cache positions [copy_lo[r], copy_hi]; cont: the search goes on; old_len: cur_len before the step. */
typedef struct sv_beam_plan {
  int32_t run_parent[16], run_tok[16], fin_old[16], fin_parent[16], fin_tok[16], copy_src[16], copy_lo[16];
  int32_t copy_hi, cont, old_len;
} sv_beam_plan;
typedef struct sv_op_beam_step_args {
  const sv_beam_params* params;  /* checked as sv_beam_params_check_rows(params, batch, 16) */
  int32_t batch, vocab, seq_stride;
  int32_t advance;               /* 0: the first step (candidates of the prefill logits), 1: a decode step; cache_hi =
                                    cur_len - 1 + advance, and cur_len += advance when the search goes on */
  sv_beam_state* state_host;     /* in/out; 0 <= cur_len < seq_stride, parity 0 or 1, fin_len in [0, seq_stride] */
  const float *cand_key, *cand_val;   /* device [R][2 * num_beams], R = batch * num_beams: each row's candidates best-first, */
  const int32_t* cand_tok;            /*   as beam_candidates_kernel writes them */
  int32_t *run_seq, *fin_seq;    /* device [2][R][seq_stride]: the double-buffered sequences, updated */
  int32_t* gen_host;             /* [2]: cur_len (the position of the token fed next, >= 0), done; in/out */
  const void *wte, *wpe;         /* bf16 [vocab][h], [n_positions][h]; wpe may be NULL (RoPE models) */
  void* x;                       /* bf16 [R][h]: the next tokens' embeddings at position min(cur_len, n_positions - 1) */
  int32_t h, n_positions;        /* h % 8 == 0 */
  int32_t* next_ids;             /* device [R] */
  sv_beam_plan* plan_host;       /* in/out: the device plan starts as this and is read back (rows >= R are not defined
                                    after a step that ran) */
} sv_op_beam_step_args;
SV_API int sv_op_beam_step(const sv_op_beam_step_args* args, void* stream);
/* Both phases of the KV suffix copies (parent rows -> a staging cache this call allocates -> child rows) over caches
 * kcache [n_layer][>= rows][n_kv][tcap][D] and vtcache [n_layer][>= rows][n_kv][D][tcap] (D = 128), layer_stride elements
 * apart, following *plan_host for rows [0, rows).  copy_src in [-1, rows), copy_hi < tcap, copy_lo >= 0, tcap % 32 == 0,
 * caches 16-byte aligned. */
SV_API int sv_op_beam_kv_copy(void* kcache, void* vtcache, int64_t layer_stride, int32_t n_layer, int32_t rows,
                              int32_t n_kv, int32_t tcap, const sv_beam_plan* plan_host, void* stream);
/* One layer's cache-row gather (sv_reorder_cache, sv_expand_batch, the n-completions copy of sv_session_admit): row r of
 * kdst / vdst takes K positions [0, len) and V^T positions [0, round_up(len, 8)) of source row idx[r] (idx: device int32
 * [rows] with entries in the source's rows, or NULL: r).  Layouts as sv_op_attention_decode; 1 <= len <= tcap,
 * tcap % 32 == 0, rows <= 16. */
SV_API int sv_op_kv_gather(const void* ksrc, const void* vsrc, void* kdst, void* vdst, const int32_t* idx, int32_t rows,
                           int32_t n_kv, int32_t tcap, int32_t len, void* stream);
/* Admission of k session slots in one launch: slot slot_host[j] gets seen[slot] cleared, out_ids[slot] filled with pad_id
 * and its RowState fields row_len = len_host[j], row_step = 0, row_active = 1, row_max_new = max_new_host[j], row_seed =
 * seed_host[j].  The RowState travels as the host arrays [S] (and event [1]), read on entry and written back. */
typedef struct sv_op_admit_args {
  int32_t k, S;                  /* 1 <= k <= S <= 16 */
  const int32_t *slot_host, *len_host, *max_new_host;   /* [k]: distinct slots in [0, S), len >= 0 */
  const uint64_t* seed_host;     /* [k] */
  void* seen;                    /* uint8 [S][vocab] (device) */
  int32_t vocab;
  int32_t* out_ids;              /* [S][out_stride] (device) */
  int32_t out_stride, pad_id;
  int32_t *row_len_host, *row_step_host, *row_active_host, *row_max_new_host;   /* [S] each */
  uint64_t* row_seed_host;       /* [S] */
  int32_t* event_host;           /* [1] */
} sv_op_admit_args;
SV_API int sv_op_session_admit(const sv_op_admit_args* args, void* stream);

/* The image-encoder, adapter and prefill kernels one launch at a time (the half of a request before the first decode
 * step).  The caller owns the device tensors; every argument is checked on the host: SV_ERR_INVALID before any launch.
 * Synchronous on `stream`.  sv_op_layernorm, sv_op_linear and sv_op_attention_vit above are the rest of that half. */
/* pixels [batch][3][image][image] -> patches [batch * (image / patch)^2][kpad]: row = one patch, columns (c, iy, ix)
 * row-major, zero from 3 * patch^2 to kpad (the conv as a GEMM). */
SV_API int sv_op_im2col(const void* pixels, void* patches, int32_t batch, int32_t image, int32_t patch, int32_t kpad,
                        void* stream);
/* x [batch][np (+1)][width] = bf16(cat(cls, pe[b]) + pos), or bf16(pe[b] + pos) when cls == NULL (SigLIP);
 * pe [batch][np][width], cls [width], pos [np (+1)][width]. */
SV_API int sv_op_vit_assemble(const void* pe, const void* cls, const void* pos, void* x, int32_t batch, int32_t np,
                              int32_t width, void* stream);
/* The adapter norm over z [batch][q][h] -> y.  SV_ADAPTER_NORM_SLAB: LayerNorm([q, h]) per image, w and b [q][h]
 * (rmean, rvar unused; q * h % 8 == 0).  SV_ADAPTER_NORM_TOKENS: eval BatchNorm1d(q), channel = token, w, b, rmean,
 * rvar [q]. */
enum { SV_ADAPTER_NORM_SLAB = 0, SV_ADAPTER_NORM_TOKENS = 1 };
SV_API int sv_op_adapter_norm(int32_t kind, const void* z, const void* w, const void* b, const void* rmean, const void* rvar,
                              void* y, int32_t batch, int32_t q, int32_t h, float eps, void* stream);
/* x [batch][q + p][h]: row t = visual[b][t] for t < q, else wte[clamp(ids[b * id_stride + t - q], 0, vocab - 1)]; plus
 * wpe[pos0 + t] unless wpe == NULL (RoPE models).  ids int32 (device); q = 0, pos0 > 0 is the scoring chunk's form. */
SV_API int sv_op_embed_prefix(const void* visual, const int32_t* ids, const void* wte, const void* wpe, void* x,
                              int32_t batch, int32_t q, int32_t p, int32_t h, int32_t vocab, int32_t pos0, int32_t id_stride,
                              void* stream);
/* The prefill attention over caches the caller owns (D = 128; kcache [batch][n_kv][tcap][D], vtcache
 * [batch][n_kv][D][tcap]): the K/V columns of packed qkv [batch * seq][(n_head + 2 n_kv) * D] are written to slots
 * [0, seq), then token t of each image attends to keys [0, t] (keys > t - window when window > 0) -> out
 * [batch * seq][n_head * D].  Slots >= seq are not written.  seq <= tcap, tcap % 32 == 0, n_head / n_kv <= 16. */
SV_API int sv_op_attention_prefill(const void* qkv, void* kcache, void* vtcache, void* out, int32_t batch, int32_t seq,
                                   int32_t n_head, int32_t n_kv, int32_t tcap, int32_t window, void* stream);
/* y [M][N] = bf16(x[M,K] . w[N,K]^T) for any N: the resident last-position logits of a scoring call, with the tiling and
 * rounding of sv_op_lm_logprob.  Only the M * N outputs are written; K % 64 == 0. */
SV_API int sv_op_lm_logits(const void* x, const void* w, void* y, int32_t M, int32_t N, int32_t K, void* stream);

/* The teacher-forced scoring kernels one launch at a time (sv_score_tokens), same conventions as above.
 * The chunk attention over caches the caller owns (D = 128; kcache [batch][n_kv][tcap][D], vtcache [batch][n_kv][D][tcap]):
 * row [b][t] of packed qkv [batch * C][(n_head + 2 n_kv) * D] is position pos0 + t.  Its K/V columns are written to slots
 * [pos0, pos0 + C) of image b, then query t attends to keys [0, pos0 + t] (keys > pos0 + t - window when window > 0) ->
 * out [batch * C][n_head * D].  Slots < pos0 are the prefix an earlier call wrote; slots >= pos0 + C are neither written
 * nor read into the result.  pos0 + C <= tcap, tcap % 32 == 0, n_head / n_kv <= 16. */
SV_API int sv_op_attention_score(const void* qkv, void* kcache, void* vtcache, void* out, int32_t batch, int32_t C,
                                 int32_t pos0, int32_t n_head, int32_t n_kv, int32_t tcap, int32_t window, void* stream);
/* Position 0 of a scoring call: logprob fp32 [M] = log_softmax(float(logits[m]))[targets[m]] over resident bf16 logits
 * [M][vocab] (16-byte aligned), with the tiles and merge of sv_op_lm_logprob.  A target outside [0, vocab) gives NaN. */
SV_API int sv_op_logits_logprob(const void* logits, const int32_t* targets, float* logprob, int32_t M, int32_t vocab,
                                void* stream);

/* ---- image preprocessing (SURVEY.md §8f-2) ------------------------------------------------ */
/* Replaces `ImageTrainProcessor.__call__` (reference starvector/data/util.py:40-66: RGBA pasted on white, pad to
 * square with 255, `transforms.Resize(size, BICUBIC)` on the PIL image, ToTensor, Normalize) and
 * `SimpleStarVectorProcessor.transform` (starvector_arch.py:39-45: the same with `convert("RGB")` for RGBA),
 * bit for bit with Pillow's 8-bit resample.  On-wire input = what PIL holds: uint8 HWC host buffers. */
enum { SV_ALPHA_WHITE = 0 /* data/util.py:63-66 */, SV_ALPHA_DROP = 1 /* starvector_arch.py:40 */ };

typedef struct sv_preproc sv_preproc;

typedef struct sv_preproc_desc {
  int32_t out_size;    /* S: output is [n,3,S,S] (224 for CLIP ViT-L/14, data/util.py:41) */
  int32_t alpha_mode;  /* SV_ALPHA_WHITE | SV_ALPHA_DROP: what happens to a 4th channel */
  int32_t pad_square;  /* 1: pad the shorter side with 255 to a centred square first (data/util.py:55-61); 0: resize (w,h)->(S,S) */
  int32_t out_dtype;   /* SV_DTYPE_BF16 (what sv_encode_images takes) | SV_DTYPE_F32 (the reference's tensor, for parity) */
  float mean[3];       /* Normalize(mean, std), data/util.py:33-38 */
  float std[3];
} sv_preproc_desc;

typedef struct sv_image_u8 {
  const uint8_t* data; /* HOST pointer, uint8 [height][width][channels]; pinned memory makes the upload asynchronous */
  int32_t width, height;
  int32_t channels;    /* 3 (RGB) or 4 (RGBA) */
  int32_t row_stride;  /* bytes between rows; 0 = width*channels */
} sv_image_u8;

SV_API int sv_preproc_create(const sv_preproc_desc* desc, int device, sv_preproc** out);
SV_API void sv_preproc_destroy(sv_preproc* p);
/* Message for the last failing call on `p` (or the last failing create when p == NULL). */
SV_API const char* sv_preproc_last_error(const sv_preproc* p);
/* `[processor(img) for img in images]` + stack: uploads the n images (ragged sizes), runs the horizontal and the
 * vertical resample pass, writes DEVICE out_pixels [n,3,S,S] (out_dtype).  Asynchronous on `stream`. */
SV_API int sv_preproc_run_host(sv_preproc* p, const sv_image_u8* images_host, int32_t n, void* out_pixels, void* stream);
/* Kernels launched by `p` so far. */
SV_API long long sv_preproc_launch_count(const sv_preproc* p);
/* Host-only pieces of the above, exported so that they can be checked against Pillow / torch without a GPU:
 * the fixed-point resample taps of one axis (Pillow Resample.c precompute_coeffs + normalize_coeffs_8bpc; call with
 * bounds == taps == NULL to query ksize; bounds int32 [out_size][2] = first tap, tap count; taps int32
 * [out_size][ksize]) and the 3x256 ToTensor+Normalize table (float [3][256]). */
SV_API int sv_resample_coeffs_host(int32_t in_size, int32_t out_size, int32_t* ksize, int32_t* bounds, int32_t* taps,
                                   int32_t taps_capacity);
SV_API int sv_preproc_lut_host(const sv_preproc_desc* desc, float* lut768);
/* The batch plan sv_preproc_run_host uploads: per-image metadata (padding, arena offsets) followed by the coefficient
 * arena.  sizes[5] = {blob bytes, metadata bytes, input-arena bytes, intermediate pixels, max input rows}; blob may be
 * NULL to query sizes.  Test hook: tests/test_preprocess_emul.py replays the kernels' index arithmetic from it. */
SV_API int sv_preproc_plan_host(const sv_preproc_desc* desc, const sv_image_u8* images_host, int32_t n, void* blob,
                                int64_t blob_capacity, int64_t sizes[5]);

#ifdef __cplusplus
}
#endif
#endif /* STARVECTOR_B200_H */

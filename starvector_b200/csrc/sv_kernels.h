// Launcher declarations shared by the kernel translation units and sv_engine.cu.
// All tensors are bf16 unless noted; `st` is the stream every launch goes to.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sv_beam_core.h"
#include "sv_common.cuh"
#include "sv_spec_core.h"

namespace sv {

// Counts kernel launches issued through the launchers (sv_launch_count()).
extern thread_local int64_t* g_launch_counter;
inline void count_launch(int n = 1) { if (g_launch_counter) *g_launch_counter += n; }

// Device-resident generation state, read/written by kernels so a captured graph can be replayed.
struct GenState {
  int32_t cur_len;      // tokens in the KV cache == position of the token fed next
  int32_t step;         // generated tokens so far == next free column of out_ids
  int32_t done;         // all rows finished (or row-0 stop fired)
  int32_t row0_stop;    // scratch: row 0 matched the stop sequence this step
  int32_t unfinished[64];
};

struct GenParamsDev {
  int32_t max_new, do_sample, eos_id, pad_id, n_stop, stop_ids[8], stop_row0_only, out_stride;
  float temperature, top_p, rep_penalty;
  unsigned long long seed;
};

// Per-row state of a continuous-batching session (sv_session_*): every cache row ("slot") has its own position, step,
// token cap and Philox seed, and finishes on its own.  The kernels' session variants (the `rows` argument of the
// launchers below) read positions from here instead of GenState::cur_len; GenState itself is left as it is (the
// dataflow kernel copies it into shared memory).
constexpr int kSessionRows = 16;
struct RowState {
  int32_t row_len[kSessionRows];      // tokens in the row's KV cache == position of the token fed next
  int32_t row_step[kSessionRows];     // tokens generated == next free column of the row's out_ids
  int32_t row_active[kSessionRows];   // 1 while the row decodes; the select kernels skip rows with 0
  int32_t event;                      // set to 1 by the select kernels when a row finishes; the host polls and clears it
  int32_t pad_;
  int32_t row_max_new[kSessionRows];
  unsigned long long row_seed[kSessionRows];
};
// The per-row fields of the slots one admission fills, passed by value to launch_session_admit.
struct SessionAdmit {
  int32_t n, slot[kSessionRows], len[kSessionRows], max_new[kSessionRows];
  unsigned long long seed[kSessionRows];
};

// ---- sv_kernels_basic.cu
void launch_layernorm(const bf16* x, const bf16* w, const bf16* b, bf16* y, int rows, int cols, float eps,
                      int64_t x_row_stride, cudaStream_t st);
void launch_convert_to_bf16(const void* src, int dtype, bf16* dst, int64_t n, cudaStream_t st);
void launch_pad_rows(const bf16* src, bf16* dst, int rows, int src_cols, int dst_cols, cudaStream_t st);
void launch_im2col(const bf16* pixels, bf16* patches, int batch, int image, int patch, int kpad, cudaStream_t st);
void launch_vit_assemble(const bf16* pe, const bf16* cls, const bf16* pos, bf16* x, int batch, int np, int width,
                         cudaStream_t st);   // cls == nullptr: no class token (SigLIP): x = pe + pos
void launch_vit_transpose_v(const bf16* qkv, bf16* vt, int batch, int seq, int heads, int seq_pad, cudaStream_t st);
void launch_slab_layernorm(const bf16* z, const bf16* w, const bf16* b, bf16* y, float* partial, int batch,
                           int64_t slab, float eps, cudaStream_t st);
void launch_batchnorm_tokens(const bf16* z, const bf16* w, const bf16* b, const bf16* rmean, const bf16* rvar, bf16* y,
                             int batch, int q, int h, float eps, cudaStream_t st);
// rows [b][t] of x: visual[b][t] for t < q, else wte[prompt_ids[b * id_stride + t - q]]; + wpe[pos0 + t] when wpe != nullptr
void launch_embed_prefix(const bf16* visual, const int32_t* prompt_ids, const bf16* wte, const bf16* wpe, bf16* x,
                         int batch, int q, int p, int h, int vocab, int pos0, int id_stride, cudaStream_t st);
// rows != nullptr (here and below): the session variant, row b at position rows->row_len[b]
void launch_embed_tokens(const int32_t* ids, const bf16* wte, const bf16* wpe, const GenState* state, bf16* x,
                         int batch, int h, int vocab, int n_positions, cudaStream_t st, const RowState* rows = nullptr);
// K/V of qkv rows [b][0, seq) -> cache positions t0 .. t0+seq-1
void launch_kv_scatter(const bf16* qkv, bf16* kcache, bf16* vtcache, int batch, int seq, int q_cols, int n_kv, int d,
                       int tcap, int t0, cudaStream_t st);
void launch_kv_append(const bf16* qkv, bf16* kcache, bf16* vtcache, const GenState* state, int batch, int q_cols,
                      int n_kv, int d, int tcap, cudaStream_t st, const RowState* rows = nullptr);
void launch_kv_gather(const bf16* ksrc, const bf16* vsrc, bf16* kdst, bf16* vdst, const int32_t* idx, int rows, int n_kv,
                      int tcap, int d, int len, cudaStream_t st);
void launch_gather_rows(const bf16* x, bf16* y, int batch, int seq, int row, int h, cudaStream_t st);
void launch_logits_to_float(const bf16* logits, float* out, int64_t n, cudaStream_t st);
// Session variants (rows != nullptr): only rows b with bit b of row_mask set and rows->row_active[b] select a token; each
// keeps its own bookkeeping (out_ids[b][row_step[b]], stop sequence over its own history, EOS / stop / row_max_new finish
// the row and set rows->event, row_step += 1, row_len += advance_len); sampling draws from Philox(row_seed[b], 0,
// row_step[b]), the stream a one-row generate with that seed uses.  GenState is not touched.
void launch_select_greedy(const bf16* logits, int vocab, int batch, GenState* state, const GenParamsDev* params,
                          uint8_t* seen, int32_t* next_ids, int32_t* out_ids, cudaStream_t st, RowState* rows = nullptr,
                          uint32_t row_mask = 0, int advance_len = 0);
void launch_select_sample(const bf16* logits, int vocab, int batch, GenState* state, const GenParamsDev* params,
                          uint8_t* seen, int32_t* next_ids, int32_t* out_ids, float* probs, cudaStream_t st,
                          RowState* rows = nullptr, uint32_t row_mask = 0, int advance_len = 0);
void launch_gen_finalize(GenState* state, const GenParamsDev* params, int batch, int advance_len, cudaStream_t st);
// Admission of a.n session slots in one launch: for each slot a.slot[j], its repetition-penalty row seen[slot] is cleared,
// its output row out_ids[slot][0, out_stride) filled with pad_id, and its RowState fields set (row_len = a.len[j],
// row_step = 0, row_active = 1, row_max_new, row_seed).  Every other slot's rows are left as they are.
void launch_session_admit(RowState* rows, const SessionAdmit& a, uint8_t* seen, int vocab, int32_t* out_ids, int out_stride,
                          int pad_id, cudaStream_t st);
void launch_advance_len(GenState* state, cudaStream_t st);
void launch_fill_i32(int32_t* p, int32_t v, int n, cudaStream_t st);

// ---- sv_gemm_rowgroup.cu : y[M,N] = epi(x[M,K] . w[N,K]^T) with mma.sync, weight streaming
void launch_linear_rowgroup(const bf16* x, const bf16* w, const bf16* bias, const bf16* res, bf16* y, int M, int N,
                            int K, int act, cudaStream_t st);

// ---- sv_gemm_wgmma.cu : same contract on wgmma + TMA (M >= 1, N % 8 == 0, K % 64 == 0)
bool wgmma_supported(int M, int N, int K);
// returns cudaSuccess or the error of tensor-map creation / launch
cudaError_t launch_linear_wgmma(const bf16* x, const bf16* w, const bf16* bias, const bf16* res, bf16* y, int M, int N,
                                int K, int act, cudaStream_t st);
// fused lm_head log-likelihood, first half: logits = bf16(x[M,K] . w[N,K]^T) stay on chip; per (row, 128-column tile)
// part[row * lm_logprob_ntiles(N) + tile] = (max, sum exp(logit - max)) and tgt_logit[row] = logit[targets[row]]
// (any N; K % 64 == 0; targets must lie in [0, N))
int lm_logprob_ntiles(int N);
// y[M,N] = bf16(x . w^T) for any N, with the same tiling and rounding as launch_lm_logprob_partials
cudaError_t launch_lm_logits(const bf16* x, const bf16* w, bf16* y, int M, int N, int K, cudaStream_t st);
cudaError_t launch_lm_logprob_partials(const bf16* x, const bf16* w, const int32_t* targets, float2* part, float* tgt_logit,
                                       int M, int N, int K, cudaStream_t st);

// ---- sv_score.cu : the rest of teacher-forced scoring
// tgt[b * C + t] = clamp(ids[b * n + c0 + t + 1], 0, vocab) (0 past the end of the row)
void launch_score_targets(const int32_t* ids, int n, int c0, int batch, int C, int vocab, int32_t* tgt, cudaStream_t st);
// the partials of launch_lm_logprob_partials for resident bf16 logits rows [batch][vocab]
void launch_logits_logprob_partials(const bf16* logits, int vocab, int batch, const int32_t* targets, float2* part,
                                    float* tgt_logit, cudaStream_t st);
// logprob of row r = tgt_logit[r] - (m + log s) over its tiles' partials, written to out[(r / C) * n + off + r % C]
// when off + r % C < n
void launch_logprob_merge(const float2* part, int ntiles, const float* tgt_logit, int rows, int C, int off, int n,
                          float* out, cudaStream_t st);

// ---- sv_attention.cu
void launch_attention_vit(const bf16* qkv, const bf16* vt, bf16* out, int batch, int seq, int heads, int seq_pad,
                          cudaStream_t st);
// causal attention of `seq` new tokens per row against the cache (prefill: cache already holds them)
void launch_attention_heads(const bf16* qkv, int q_cols_total, const bf16* kcache, const bf16* vtcache, bf16* out,
                            int batch, int seq, int n_head, int n_kv, int d, int tcap, int window, cudaStream_t st);
// scoring chunk: queries of qkv rows [b * q_rows_per_b + t], t < C, at cache positions q0 + t (the cache already holds
// positions <= q0 + C - 1); out rows [b * C + t]
cudaError_t launch_attention_chunk(const bf16* qkv, int q_cols_total, int q_rows_per_b, const bf16* kcache,
                                   const bf16* vtcache, bf16* out, int batch, int C, int q0, int n_head, int n_kv, int d,
                                   int tcap, int window, cudaStream_t st);
void launch_attention_decode(const bf16* qkv, int q_cols_total, const bf16* kcache, const bf16* vtcache, bf16* out,
                             float* partial, const GenState* state, int batch, int n_head, int n_kv, int d, int tcap,
                             int nsplit, int window, cudaStream_t st, const RowState* rows = nullptr);
// RoPE in place on the q and k parts of packed qkv rows [rows][qkv_cols] (StarCoder2, rotate_half convention);
// cos/sin tables are bf16 [max_pos][D/2]; position of row r = pos0 + (r % seq) or state->cur_len when state != nullptr
// (or row_pos->row_len[r] when row_pos != nullptr: the session variant, one token per row).
void launch_rope(bf16* qkv, int rows, int seq, int qkv_cols, int n_rot_heads, int d, const bf16* cos_t, const bf16* sin_t,
                 const GenState* state, int max_pos, int pos0, cudaStream_t st, const RowState* row_pos = nullptr);
void launch_rope_append(bf16* qkv, int batch, int qkv_cols, int n_head, int n_kv, int d, const bf16* cos_t,
                        const bf16* sin_t, bf16* kcache, bf16* vtcache, const GenState* state, int tcap, int max_pos,
                        bool pdl, cudaStream_t st, const RowState* rows = nullptr);
constexpr int kRopeMaxHalf = 256;     // d / 2 of a RoPE table
void launch_rope_table(bf16* cos_t, bf16* sin_t, int max_pos, int d, float theta, cudaStream_t st);

// decode attention (PDL-ready): the ncta <= 8 CTAs of one image form a thread-block cluster
int attention_decode_cluster_ncta(int total_len);
cudaError_t attention_decode_cluster_init();
cudaError_t launch_attention_decode_cluster(const bf16* qkv, int q_cols_total, const bf16* kcache, const bf16* vtcache,
                                            bf16* out, const GenState* state, int batch, int n_head, int n_kv, int d,
                                            int tcap, int ncta, int window, bool pdl, cudaStream_t st,
                                            const RowState* rows = nullptr, const svspec::ColMap* cmap = nullptr);

// ---- sv_decode_fused.cu : token selection fused with the next step's embedding, PDL-ready
// rows != nullptr: the session variant (see launch_select_greedy); only the selecting rows' embeddings are written.
void launch_select_fused(const bf16* logits, int vocab, int batch, const float* amax_val, const int* amax_idx,
                         int ntiles, int amax_stride, GenState* state, const GenParamsDev* params, uint8_t* seen, int32_t* next_ids,
                         int32_t* out_ids, int advance_len, const bf16* wte, const bf16* wpe, bf16* x, int h,
                         int n_positions, bool pdl, cudaStream_t st, RowState* rows = nullptr, uint32_t row_mask = 0);

// ---- sv_decode_fused.cu : the verify step of sv_generate_speculative (one cache row, sp->ncols columns; sv_spec_core.h).
// Greedy: per-column selection as launch_select_fused, then accept, next drafts, column map and the columns' embeddings.
void launch_select_fused_spec(const bf16* logits, int vocab, const float* amax_val, const int* amax_idx, int ntiles,
                              int amax_stride, GenState* state, const GenParamsDev* params, uint8_t* seen,
                              int32_t* next_ids, int32_t* out_ids, const bf16* wte, const bf16* wpe, bf16* x, int h,
                              int n_positions, svspec::State* sp, bool pdl, cudaStream_t st);
// The same after launch_select_sample_spec (tokens in sp->sel); with sp->map.n_live = 0 it only drafts and embeds.
void launch_spec_accept(GenState* state, const GenParamsDev* params, uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                        int vocab, const bf16* wte, const bf16* wpe, bf16* x, int h, int n_positions, svspec::State* sp,
                        bool pdl, cudaStream_t st);
// ---- sv_kernels_basic.cu : sampling of the live columns of a verify step (select_sample_kernel per column, Philox counter
// (0, step + c), repetition-penalty set = row 0's seen plus drafts 1..c), tokens to sp->sel
void launch_select_sample_spec(const bf16* logits, int vocab, int ncols, GenState* state, const GenParamsDev* params,
                               uint8_t* seen, float* probs, svspec::State* sp, cudaStream_t st);

// ---- sv_spec_session.cu : the verify step of a speculative session (S = ss->ncols columns; sv_spec_core.h, sv_select.cuh).
// Greedy: per-column selection as launch_select_fused_spec, then every live row's accept walk, the next drafts, the column
// allocation and map, and the columns' embeddings.  Sampled: launch_spec_session_select_sample (tokens to ss->sel), then
// launch_spec_session_tail with accept; the tail without accept re-plans after an admission.
void launch_spec_session_select_fused(const bf16* logits, int vocab, const float* amax_val, const int* amax_idx, int ntiles,
                                      int amax_stride, RowState* rows, const GenParamsDev* params, uint8_t* seen,
                                      int32_t* next_ids, int32_t* out_ids, const bf16* wte, const bf16* wpe, bf16* x, int h,
                                      int n_positions, int tcap, svspec::SessionState* ss, bool pdl, cudaStream_t st);
void launch_spec_session_select_sample(const bf16* logits, int vocab, int ncols, RowState* rows, const GenParamsDev* params,
                                       uint8_t* seen, float* probs, svspec::SessionState* ss, cudaStream_t st);
void launch_spec_session_tail(bool accept, RowState* rows, const GenParamsDev* params, uint8_t* seen, int32_t* next_ids,
                              int32_t* out_ids, int vocab, const bf16* wte, const bf16* wpe, bf16* x, int h, int n_positions,
                              int tcap, svspec::SessionState* ss, bool pdl, cudaStream_t st);

// ---- sv_decode_mega.cu : per-phase weight-ring decode GEMV; layer descriptor shared with sv_decode_flow.cu
struct MegaLayer {
  const bf16 *ln1_w, *ln1_b, *attn_w, *attn_b, *proj_w, *proj_b, *ln2_w, *ln2_b, *fc_w, *fc_b, *fc2_w, *fc2_b;
  bf16 *kc, *vc;
  const bf16 *attn_t, *proj_t, *fc_t, *fc2_t;   // slab-tiled copies for the dataflow decode kernel (sv_decode_flow.cu flow_repack_kernel)
};
// one-phase weight-ring GEMV (same device code as the persistent kernel's GEMV phases)
struct RingGemvLaunch {
  const bf16 *X, *W, *bias, *res, *ln_w, *ln_b;
  const uint8_t* Wt;              // slab-tiled copy of W (flow_repack_kernel) or nullptr: then W's rows are copied one by one
  bf16* Y;
  int B, N, K, act, epi;          // epi: 0 plain, 1 QKV (+KV append), 2 lm_head (+argmax partials)
  float ln_eps;
  int n_head, n_kv, tcap;
  const GenState* state;
  bf16 *kcache, *vtcache;
  float* amax_val;
  int* amax_idx;
  bool pdl;
  const RowState* rows;           // != nullptr with epi 1: the session variant, KV appended at rows->row_len[row]
  const svspec::ColMap* cmap;     // != nullptr with epi 1: a verify step, column c's KV appended at (row[c], pos[c]) if live
};
cudaError_t gemv_ring_init();
bool gemv_ring_supported(int K, bool has_ln);
// LayerNorm GEMVs over such K stream their statistics: kernels for <= 8 rows and the plain / lm_head epilogues only
bool gemv_ring_ln_streamed(int K);
int gemv_ring_ntiles(int N);
int gemv_ring_ncta();
int gemv_ring_max_rows();
// Row groups of 8 a decode launch over B image rows uses (1 up to 8 rows, 2 for 9-16); the lm_head's argmax partials have
// a row stride of 8 * groups.
inline int ring_row_groups(int B) { return B > 8 ? 2 : 1; }
void launch_gemv_ring(const RingGemvLaunch& g, cudaStream_t st);
// ---- sv_decode_flow.cu : dataflow persistent decode kernel (flagged activation words through L2, no grid barriers)
struct FlowLaunch {
  const MegaLayer* layers_dev;
  int n_layer, B, H, I, n_head, n_kv, qkv_cols, vocab, tcap, n_positions;
  float ln_eps;
  const bf16 *wte, *wpe, *lnf_w, *lnf_b, *lm_head, *lm_head_t;
  bf16 *x_plain, *logits;
  uint32_t *xa, *xb, *qkv, *att, *hb;          // flagged bf16 words
  unsigned long long *part, *amax;             // flagged fp32 words / argmax partials
  GenState* state;
  const GenParamsDev* params;
  uint8_t* seen;
  int32_t *next_ids, *out_ids;
  int nsteps;          // tokens in this launch
  int step0;           // phase-tag epoch of the first step (monotonic since the exchange buffers were cleared)
  int cur_len0;        // tokens in the KV cache when the launch starts
  int first_plain;     // 1: the first step's input is x_plain (plain bf16) and gets converted to flagged words
  int do_select;       // 1: greedy select + embed after every step; 0: stop after the logits (teacher forcing)
  int l2_ahead;        // weight slabs per CTA prefetched into L2 ahead of the shared-memory ring (0 = off)
  long long* dbg;
  bool realloc;
};
cudaError_t decode_flow_init();
int decode_flow_ncta();
int decode_flow_max_splits();
int decode_flow_partial_floats();
const char* decode_flow_status();
bool decode_flow_supported(int H, int I, int head_dim, int max_batch, int window, bool rope);
bool decode_flow_shape_ok(int H, int I, int head_dim, int max_batch, int window, bool rope);   // host only: no device query
int decode_flow_max_keys();         // longest row (keys, the new token included) the attention's item split covers
int decode_flow_max_layers();
bool decode_flow_realloc_supported();
cudaError_t launch_decode_flow(const FlowLaunch& m, cudaStream_t st);
size_t flow_tiled_bytes(int N, int K, int ncta);      // bytes of the slab-tiled copy of a [N][K] decode weight matrix
void launch_flow_repack(const bf16* W, const bf16* bias, void* T, int N, int K, int ncta, cudaStream_t st);

// ---- sv_beam.cu : beam search / beam-sample bookkeeping inside the decode graph (state structs: sv_beam_core.h)
size_t beam_candidates_smem(int vocab);
cudaError_t beam_init(int vocab);          // cudaErrorInvalidValue: a logits row does not fit the SM's shared memory
void launch_beam_candidates(const bf16* logits, int vocab, int rows, const svbeam::Params* p, const svbeam::State* st,
                            const int32_t* run_seq, float* cand_key, float* cand_val, int32_t* cand_tok, cudaStream_t st_);
void launch_beam_step(const svbeam::Params* p, svbeam::State* st, svbeam::Plan* plan, const float* cand_key,
                      const float* cand_val, const int32_t* cand_tok, int32_t* run_seq, int32_t* fin_seq, GenState* gs,
                      int advance, const bf16* wte, const bf16* wpe, bf16* x, int h, int n_positions,
                      int32_t* next_ids, cudaStream_t st_);
void launch_beam_kv_copy(bf16* kc, bf16* vc, bf16* kc2, bf16* vc2, int64_t layer_stride, int n_layer, int rows, int n_kv,
                         int tcap, int D, const svbeam::Plan* plan, cudaStream_t st_);
// Beam-session variants (sv_beam_session_*): group g of num_beams = p[0].nb slots owns rows [g * nb, (g + 1) * nb) and its
// own p[g] (B = 1), st[g], plan[g] in group-local rows; run_seq / fin_seq are [2][kMaxRows][seq_stride] by global row, each
// group flipping its own parity half.  Groups outside group_mask, not live (rows->row_active of their first slot) or done
// are left as they are.  Positions come from rows->row_len; the step kernel advances row_len / row_step of a continuing
// group's slots and, at its finish, clears their row_active, writes the best hypothesis' length to row_step of its first
// slot and raises rows->event.  (sv_beam_session.cu)
cudaError_t beam_session_init(int vocab);  // cudaErrorInvalidValue: as beam_init
void launch_beam_session_candidates(const bf16* logits, int vocab, int slots, const svbeam::Params* p,
                                    const svbeam::State* st, const int32_t* run_seq, float* cand_key, float* cand_val,
                                    int32_t* cand_tok, const RowState* rows, uint32_t group_mask, cudaStream_t st_);
void launch_beam_session_step(const svbeam::Params* p, svbeam::State* st, svbeam::Plan* plan, const float* cand_key,
                              const float* cand_val, const int32_t* cand_tok, int32_t* run_seq, int32_t* fin_seq,
                              RowState* rows, uint32_t group_mask, int slots, int advance, const bf16* wte, const bf16* wpe,
                              bf16* x, int h, int n_positions, int32_t* next_ids, cudaStream_t st_);
void launch_beam_session_kv_copy(bf16* kc, bf16* vc, bf16* kc2, bf16* vc2, int64_t layer_stride, int n_layer, int slots,
                                 int n_kv, int tcap, int D, const svbeam::Params* p, const svbeam::Plan* plan,
                                 const RowState* rows, uint32_t group_mask, cudaStream_t st_);

}  // namespace sv

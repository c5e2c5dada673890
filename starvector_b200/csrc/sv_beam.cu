// Beam search / beam-sample inside the replayed decode graph (SURVEY.md §8f-1: the reference's default generate() mode is
// num_beams=2, starvector_base.py:231-241,289-295).  Three small kernels follow the lm_head of every decode step, so the
// host never sees a logit, a score or a cache permutation:
//   beam_candidates_kernel  one CTA per cache row (= running beam): log-softmax of the bf16 logits row in shared memory,
//                           HF's logits processors on the log-probs (repetition penalty over the beam's own tokens,
//                           temperature, top-p), + the beam's running score, then the row's K best continuations
//                           (beam-sample: the K first draws without replacement, by Gumbel-perturbed top-K);
//   beam_step_kernel        one CTA: merges the rows of each image, runs the bookkeeping of
//                           `GenerationMixin._beam_search` (sv_beam_core.h, shared with the host replay), moves the
//                           token sequences, and writes the next tokens' embeddings for the following decode step;
//   beam_kv_copy_kernel     `_reorder_cache` without moving the cache: a child row only receives the suffix of its
//                           parent's K / V^T rows from the position where the two rows diverged (a per-image divergence
//                           matrix is part of the state) -- typically a handful of tokens, not 2 x the live cache.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/starvector_b200.h"
#include "sv_beam_body.cuh"

namespace sv {

// ---- K1: per-row candidates (body: sv_beam_body.cuh) ----------------------------------------------------------------
__global__ void __launch_bounds__(kBeamThreads) beam_candidates_kernel(const bf16* __restrict__ logits,
                                                                       const Params* __restrict__ pp, const State* st,
                                                                       const int32_t* __restrict__ run_seq,
                                                                       float* __restrict__ cand_key,
                                                                       float* __restrict__ cand_val,
                                                                       int32_t* __restrict__ cand_tok) {
  beam_candidates_body<false>(logits, pp, st, run_seq, cand_key, cand_val, cand_tok, nullptr, 0u);
}

// ---- K2: bookkeeping, sequence moves, next-token embedding -----------------------------------------------------------
__global__ void __launch_bounds__(kBeamThreads) beam_step_kernel(const Params* __restrict__ pp, State* st, Plan* plan_out,
                                                                 const float* __restrict__ cand_key,
                                                                 const float* __restrict__ cand_val,
                                                                 const int32_t* __restrict__ cand_tok, int32_t* run_seq,
                                                                 int32_t* fin_seq, GenState* gs, int advance,
                                                                 const bf16* __restrict__ wte,
                                                                 const bf16* __restrict__ wpe, bf16* __restrict__ x, int h,
                                                                 int n_positions, int32_t* next_ids) {
  // every thread reads the flag BEFORE thread 0 can rewrite the state below (it may set done in this very step)
  const int was_done = st->done;
  __syncthreads();
  if (was_done) return;
  __shared__ Plan plan;
  __shared__ int s_oldp, s_pos;
  __shared__ int s_finlen[svbeam::kMaxRows];
  const int tid = threadIdx.x;
  const int nb = pp->nb, K = pp->K, R = pp->B * nb, stride = pp->seq_stride;
  const int pad_fill = pp->pad_id;          // (from the device-resident parameters: the captured graph serves every call)
  if (tid == 0) {
    const Params p = *pp;
    float mval[svbeam::kMaxRows * 2];
    int32_t mbeam[svbeam::kMaxRows * 2], mtok[svbeam::kMaxRows * 2];    // B * K = 2 * B * nb <= 16
    for (int b = 0; b < p.B; ++b)
      svbeam::merge_candidates(p, cand_key + b * nb * K, cand_val + b * nb * K, cand_tok + b * nb * K, mval + b * K,
                               mbeam + b * K, mtok + b * K);
    State s = *st;
    s_oldp = s.parity;
    const int cache_hi = advance ? gs->cur_len : gs->cur_len - 1;
    svbeam::beam_step(p, s, mval, mbeam, mtok, run_seq + (int64_t)s.parity * R * stride, cache_hi, plan);
    *st = s;
    *plan_out = plan;
    if (plan.cont && advance) gs->cur_len += 1;
    gs->done = plan.cont ? 0 : 1;
    s_pos = gs->cur_len;
    for (int r = 0; r < R; ++r) s_finlen[r] = s.fin_len[r];
  }
  __syncthreads();
  const int oldp = s_oldp, newp = oldp ^ 1, L = plan.old_len;
  for (int r = 0; r < R; ++r) {
    const int32_t* src = run_seq + ((int64_t)oldp * R + plan.run_parent[r]) * stride;
    int32_t* dst = run_seq + ((int64_t)newp * R + r) * stride;
    for (int i = tid; i <= L; i += kBeamThreads) dst[i] = i < L ? src[i] : plan.run_tok[r];
    int32_t* dstf = fin_seq + ((int64_t)newp * R + r) * stride;
    if (plan.fin_old[r] >= 0) {
      const int32_t* srcf = fin_seq + ((int64_t)oldp * R + plan.fin_old[r]) * stride;
      const int n = s_finlen[r];
      for (int i = tid; i <= L; i += kBeamThreads) dstf[i] = i < n ? srcf[i] : pad_fill;
    } else {
      const int32_t* srcp = run_seq + ((int64_t)oldp * R + plan.fin_parent[r]) * stride;
      for (int i = tid; i <= L; i += kBeamThreads) dstf[i] = i < L ? srcp[i] : plan.fin_tok[r];
    }
  }
  if (!plan.cont) return;
  // next step's input rows: wte[token] + wpe[position] (bf16 add), as select_fused_kernel does for one beam
  int pos = s_pos;
  pos = pos >= n_positions ? n_positions - 1 : pos;
  const int hv = h >> 3, V = pp->vocab;
  for (int i = tid; i < R * hv; i += kBeamThreads) {
    const int b = i / hv, c = (i % hv) * 8;
    int id = plan.run_tok[b];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);
    float e[8], q[8];
    unpack8(ldg_cached(wte + (int64_t)id * h + c), e);
    if (wpe) {
      unpack8(ldg_cached(wpe + (int64_t)pos * h + c), q);
#pragma unroll
      for (int j = 0; j < 8; ++j) e[j] += q[j];
    }
    *reinterpret_cast<uint4*>(x + (int64_t)b * h + c) = pack8(e);
  }
  if (tid < R) next_ids[tid] = plan.run_tok[tid];
}

// ---- K3: KV suffix copies (body: sv_beam_body.cuh) ----------------------------------------------------------------
__global__ void __launch_bounds__(256) beam_kv_copy_kernel(bf16* kc, bf16* vc, bf16* kc2, bf16* vc2, int64_t layer_stride,
                                                           int n_kv, int tcap, int D, const Plan* __restrict__ plan,
                                                           int phase) {
  beam_kv_copy_body<false>(kc, vc, kc2, vc2, layer_stride, n_kv, tcap, D, plan, phase, nullptr, nullptr, 0u);
}
// ---- launchers ----------------------------------------------------------------------------------------------------
size_t beam_candidates_smem(int vocab) { return (size_t)vocab * 4 + (size_t)((vocab + 31) / 32) * 4; }

cudaError_t beam_init(int vocab) {
  const size_t need = beam_candidates_smem(vocab);
  if (need > 220 * 1024) return cudaErrorInvalidValue;          // a logits row must fit the SM's shared memory
  return cudaFuncSetAttribute(beam_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need);
}

void launch_beam_candidates(const bf16* logits, int vocab, int rows, const Params* p, const State* st, const int32_t* run_seq,
                            float* cand_key, float* cand_val, int32_t* cand_tok, cudaStream_t st_) {
  beam_candidates_kernel<<<rows, kBeamThreads, beam_candidates_smem(vocab), st_>>>(logits, p, st, run_seq, cand_key, cand_val,
                                                                                   cand_tok);
  count_launch();
}

void launch_beam_step(const Params* p, State* st, Plan* plan, const float* cand_key, const float* cand_val,
                      const int32_t* cand_tok, int32_t* run_seq, int32_t* fin_seq, GenState* gs, int advance,
                      const bf16* wte, const bf16* wpe, bf16* x, int h, int n_positions, int32_t* next_ids,
                      cudaStream_t st_) {
  beam_step_kernel<<<1, kBeamThreads, 0, st_>>>(p, st, plan, cand_key, cand_val, cand_tok, run_seq, fin_seq, gs, advance,
                                                wte, wpe, x, h, n_positions, next_ids);
  count_launch();
}

void launch_beam_kv_copy(bf16* kc, bf16* vc, bf16* kc2, bf16* vc2, int64_t layer_stride, int n_layer, int rows, int n_kv,
                         int tcap, int D, const Plan* plan, cudaStream_t st_) {
  for (int phase = 0; phase < 2; ++phase)
    beam_kv_copy_kernel<<<dim3(4, rows, n_layer), 256, 0, st_>>>(kc, vc, kc2, vc2, layer_stride, n_kv, tcap, D, plan, phase);
  count_launch(2);
}

}  // namespace sv

// =====================================================================================================================
// Host replays of the two device stages (no GPU needed): the test hooks behind tests/test_beam_core.py, which runs a whole
// beam search with them on the CPU oracle's logits and compares with HF generate(num_beams > 1).
extern "C" {

static svbeam::Params params_from_abi(const sv_beam_params* bp, int32_t batch, int32_t vocab, int32_t seq_stride) {
  svbeam::Params p;
  memset(&p, 0, sizeof(p));
  p.B = batch; p.nb = bp->num_beams; p.K = 2 * bp->num_beams; p.vocab = vocab; p.max_length = bp->max_new_tokens;
  p.eos_id = bp->eos_token_id;
  p.pad_id = bp->pad_token_id;
  p.n_stop = bp->n_stop_ids;
  for (int i = 0; i < bp->n_stop_ids && i < svbeam::kMaxStop; ++i) p.stop_ids[i] = bp->stop_ids[i];
  p.do_sample = bp->do_sample; p.early_stopping = bp->early_stopping;
  p.min_keep = std::max(2, 1 + (bp->eos_token_id >= 0 ? 1 : 0));
  p.seq_stride = seq_stride;
  p.temperature = bp->temperature; p.top_p = bp->top_p; p.rep_penalty = bp->repetition_penalty;
  p.length_penalty = bp->length_penalty; p.seed = bp->seed;
  return p;
}

int sv_beam_params_check_rows(const sv_beam_params* bp, int32_t batch, int32_t max_rows) {
  if (!bp || batch < 1 || max_rows < 1 || max_rows > svbeam::kMaxRows) return SV_ERR_INVALID;
  if (bp->num_beams < 2 || batch * bp->num_beams > max_rows || 2 * bp->num_beams > svbeam::kMaxK) return SV_ERR_INVALID;
  if (bp->max_new_tokens < 1 || bp->n_stop_ids < 0 || bp->n_stop_ids > svbeam::kMaxStop) return SV_ERR_INVALID;
  if (bp->early_stopping < 0 || bp->early_stopping > 2) return SV_ERR_INVALID;
  if (bp->do_sample && !(bp->temperature > 0.f)) return SV_ERR_INVALID;
  if (!(bp->repetition_penalty > 0.f)) return SV_ERR_INVALID;
  return SV_OK;
}

int sv_beam_params_check(const sv_beam_params* bp, int32_t batch) { return sv_beam_params_check_rows(bp, batch, 8); }

int sv_beam_state_bytes(void) { return (int)sizeof(svbeam::State); }

int sv_beam_state_init_host(const sv_beam_params* bp, int32_t batch, int32_t first_cache_pos, void* state) {
  if (sv_beam_params_check_rows(bp, batch, svbeam::kMaxRows) != SV_OK || !state) return SV_ERR_INVALID;
  svbeam::Params p = params_from_abi(bp, batch, 8, bp->max_new_tokens);
  svbeam::init_state(p, *reinterpret_cast<svbeam::State*>(state), first_cache_pos);
  return SV_OK;
}

// One logits row (fp32 values of the bf16 logits) -> its K = 2 * num_beams best continuations, serially and with HF's
// exact top-p (sort + cumulative sum).  seq: the row's generated tokens so far.
int sv_beam_row_candidates_host(const sv_beam_params* bp, const float* logits, int32_t vocab, const int32_t* seq,
                                int32_t seq_len, float running_score, int32_t step, int32_t row, float* cand_key,
                                float* cand_val, int32_t* cand_tok) {
  if (!bp || !logits || vocab < 1 || !cand_key || !cand_val || !cand_tok) return SV_ERR_INVALID;
  const int K = 2 * bp->num_beams;
  const bool sample = bp->do_sample != 0;
  const int min_keep = std::max(2, 1 + (bp->eos_token_id >= 0 ? 1 : 0));
  std::vector<char> seen(vocab, 0);
  for (int i = 0; i < seq_len; ++i) if (seq[i] >= 0 && seq[i] < vocab) seen[seq[i]] = 1;
  float mx = -INFINITY;
  for (int i = 0; i < vocab; ++i) mx = std::max(mx, logits[i]);
  double z = 0.0;                       // the device sums in a tree: a serial fp32 sum of 49k terms is off by ~1e-4
  for (int i = 0; i < vocab; ++i) z += expf(logits[i] - mx);
  const float logz = logf((float)z);
  std::vector<float> s(vocab);
  for (int i = 0; i < vocab; ++i)
    s[i] = svbeam::process_logprob((logits[i] - mx) - logz, seq_len > 0 && seen[i], bp->repetition_penalty, sample, bp->temperature);
  std::vector<float> val = s;
  if (sample && bp->top_p < 1.0f) {
    std::vector<int> order(vocab);
    for (int i = 0; i < vocab; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return s[a] < s[b]; });    // ascending, as torch.sort
    const float m2 = s[order[vocab - 1]];
    double zd = 0.0;
    for (int i = 0; i < vocab; ++i) zd += expf(s[i] - m2);
    const float z2 = (float)zd;
    float cum = 0.f;
    for (int j = 0; j < vocab; ++j) {
      cum += expf(s[order[j]] - m2) / z2;
      if (cum <= 1.0f - bp->top_p && j < vocab - min_keep) val[order[j]] = -INFINITY;
    }
  }
  std::vector<float> key(vocab);
  for (int i = 0; i < vocab; ++i) {
    key[i] = val[i] + running_score;
    if (sample && key[i] > -INFINITY) key[i] += svbeam::gumbel_noise(bp->seed, step, row, i);
  }
  for (int k = 0; k < K; ++k) {
    int best = -1;
    for (int i = 0; i < vocab; ++i)
      if (best < 0 || key[i] > key[best]) best = i;            // ties: the lower index
    cand_key[k] = key[best];
    cand_val[k] = key[best] == -INFINITY ? -INFINITY : val[best] + running_score;
    cand_tok[k] = best;
    key[best] = -INFINITY;
  }
  return SV_OK;
}

// One bookkeeping step on the host: row candidates [batch * num_beams][K] -> merged -> beam_step.  `state` is the opaque
// State blob; run_seq / fin_seq are the double-buffered sequence arrays [2][batch * num_beams][seq_stride].  plan_out (optional)
// receives the plan of rows 0-7 as int32 [7 * 8 + 3]: run_parent, run_tok, fin_old, fin_parent, fin_tok, copy_src, copy_lo
// (8 entries each), copy_hi, cont, old_len; it must be NULL above 8 rows.  Returns 1 while the search continues, 0 when it
// is over, < 0 on error.
int sv_beam_step_host(const sv_beam_params* bp, int32_t batch, int32_t vocab, int32_t seq_stride, void* state,
                      const float* cand_key, const float* cand_val, const int32_t* cand_tok, int32_t* run_seq,
                      int32_t* fin_seq, int32_t cache_hi, int32_t* next_tokens, int32_t* src_rows, int32_t* plan_out) {
  if (sv_beam_params_check_rows(bp, batch, svbeam::kMaxRows) != SV_OK || !state || !cand_key || !cand_val || !cand_tok ||
      !run_seq || !fin_seq || (plan_out && batch * bp->num_beams > 8))
    return SV_ERR_INVALID;
  svbeam::Params p = params_from_abi(bp, batch, vocab, seq_stride);
  svbeam::State& s = *reinterpret_cast<svbeam::State*>(state);
  const int nb = p.nb, K = p.K, R = batch * nb;
  float mval[svbeam::kMaxRows * 2];
  int32_t mbeam[svbeam::kMaxRows * 2], mtok[svbeam::kMaxRows * 2];
  for (int b = 0; b < batch; ++b)
    svbeam::merge_candidates(p, cand_key + b * nb * K, cand_val + b * nb * K, cand_tok + b * nb * K, mval + b * K, mbeam + b * K,
                             mtok + b * K);
  const int oldp = s.parity;
  svbeam::Plan plan;
  memset(&plan, 0, sizeof(plan));
  svbeam::beam_step(p, s, mval, mbeam, mtok, run_seq + (int64_t)oldp * R * seq_stride, cache_hi, plan);
  const int newp = oldp ^ 1, L = plan.old_len;
  const int fill = bp->pad_token_id;
  for (int r = 0; r < R; ++r) {                                // the same moves beam_step_kernel makes
    const int32_t* src = run_seq + ((int64_t)oldp * R + plan.run_parent[r]) * seq_stride;
    int32_t* dst = run_seq + ((int64_t)newp * R + r) * seq_stride;
    for (int i = 0; i <= L; ++i) dst[i] = i < L ? src[i] : plan.run_tok[r];
    int32_t* dstf = fin_seq + ((int64_t)newp * R + r) * seq_stride;
    if (plan.fin_old[r] >= 0) {
      const int32_t* srcf = fin_seq + ((int64_t)oldp * R + plan.fin_old[r]) * seq_stride;
      for (int i = 0; i <= L; ++i) dstf[i] = i < s.fin_len[r] ? srcf[i] : fill;
    } else {
      const int32_t* srcp = run_seq + ((int64_t)oldp * R + plan.fin_parent[r]) * seq_stride;
      for (int i = 0; i <= L; ++i) dstf[i] = i < L ? srcp[i] : plan.fin_tok[r];
    }
    if (next_tokens) next_tokens[r] = plan.run_tok[r];
    if (src_rows) src_rows[r] = plan.run_parent[r];
  }
  if (plan_out) {
    const int32_t* rows[7] = {plan.run_parent, plan.run_tok, plan.fin_old, plan.fin_parent, plan.fin_tok, plan.copy_src, plan.copy_lo};
    for (int a = 0; a < 7; ++a) memcpy(plan_out + 8 * a, rows[a], 8 * sizeof(int32_t));
    plan_out[56] = plan.copy_hi; plan_out[57] = plan.cont; plan_out[58] = plan.old_len;
  }
  return plan.cont;
}

// Final read-out of a State blob: parity of the live sequence buffers and the lengths of the finished hypotheses.
int sv_beam_state_read_host(const void* state, int32_t* parity, int32_t* cur_len, int32_t* fin_len8, float* beam_scores8) {
  if (!state) return SV_ERR_INVALID;
  const svbeam::State& s = *reinterpret_cast<const svbeam::State*>(state);
  if (parity) *parity = s.parity;
  if (cur_len) *cur_len = s.cur_len;
  for (int r = 0; r < 8; ++r) {
    if (fin_len8) fin_len8[r] = s.fin_len[r];
    if (beam_scores8) beam_scores8[r] = s.beam_scores[r];
  }
  return SV_OK;
}

// The same for all 16 rows, with the running scores.
int sv_beam_state_read16_host(const void* state, int32_t* parity, int32_t* cur_len, int32_t* fin_len16, float* beam_scores16,
                              float* running_scores16) {
  if (!state) return SV_ERR_INVALID;
  const svbeam::State& s = *reinterpret_cast<const svbeam::State*>(state);
  if (parity) *parity = s.parity;
  if (cur_len) *cur_len = s.cur_len;
  for (int r = 0; r < svbeam::kMaxRows; ++r) {
    if (fin_len16) fin_len16[r] = s.fin_len[r];
    if (beam_scores16) beam_scores16[r] = s.beam_scores[r];
    if (running_scores16) running_scores16[r] = s.running_scores[r];
  }
  return SV_OK;
}

}  // extern "C"

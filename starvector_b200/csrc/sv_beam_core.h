// Beam-search bookkeeping shared by the device kernels (sv_beam.cu) and their host replay (sv_beam_step_host,
// tests/test_beam_core.py): one step of transformers' `GenerationMixin._beam_search` for the decoder-only /
// `inputs_embeds` case the reference uses (starvector_base.py:231-241,289-295 -> num_beams=2, early_stopping=True;
// starvector_v2.py:53-57 -> HF defaults), restated from the installed transformers 5.5 (generation/utils.py
// `_get_top_k_continuations`, `_get_running_beams_for_next_iteration`, `_update_finished_beams`,
// `_check_early_stop_heuristic`, `_beam_search_has_unfinished_sequences`) exactly as starvector_b200/beam_search.py
// does with torch ops -- that file is this one's oracle.  Plain scalar code over <= 16 cache rows and <= 16 candidates.
//
// Everything is in GENERATED-token coordinates (prompt_len = 0: the reference calls generate(inputs_embeds=...)).
// fp32 arithmetic and its order follow the torch expressions (a python scalar operand is an fp32 scalar there).
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define SVB_HD __host__ __device__ __forceinline__
#else
#define SVB_HD inline
#endif

namespace svbeam {

constexpr int kMaxRows = 16;     // image rows of the engine = batch * num_beams
constexpr int kMaxK = 16;        // beams_to_keep = max(2, 1 + n_eos) * num_beams = 2 * num_beams
constexpr int kMaxStop = 8;
constexpr float kNegBig = -1.0e9f;

struct Params {
  int32_t B, nb, K, vocab, max_length;      // max_length = max_new_tokens (generated coordinates)
  int32_t eos_id;                           // -1: none
  int32_t pad_id;                           // fill of the sequence rectangles (HF: pad if given, else eos)
  int32_t n_stop, stop_ids[kMaxStop];       // StoppingCriteriaSub (row 0 of the flattened candidates ends everything)
  int32_t do_sample;
  int32_t early_stopping;                   // 0 False, 1 True, 2 "never"
  int32_t min_keep;                         // TopPLogitsWarper min_tokens_to_keep = max(2, 1 + n_eos)
  int32_t seq_stride;                       // ints per sequence row (>= max_length)
  float temperature, top_p, rep_penalty, length_penalty;
  unsigned long long seed;
};

struct State {
  int32_t cur_len;                          // generated tokens held by every running beam
  int32_t done;
  int32_t parity;                           // which half of the double-buffered sequence arrays is current
  int32_t pad_;
  float running_scores[kMaxRows];           // [B][nb]
  float beam_scores[kMaxRows];              // finished beams
  int32_t is_finished[kMaxRows];
  int32_t fin_len[kMaxRows];                // tokens of the finished hypothesis (= count of beam_indices != -1 in HF)
  int32_t unsatisfied[kMaxRows];            // per image: is_early_stop_heuristic_unsatisfied
  int32_t div[kMaxRows][kMaxRows];          // first CACHE position at which the KV rows r and s differ (same image)
};

// What one step decided; the data movers (sequence copies, token embedding, KV suffix copies) act on it.
struct Plan {
  int32_t run_parent[kMaxRows], run_tok[kMaxRows];   // new running row r = old running row run_parent[r] + run_tok[r]
  int32_t fin_old[kMaxRows];                         // new finished slot: >= 0 -> old finished row; -1 -> a candidate:
  int32_t fin_parent[kMaxRows], fin_tok[kMaxRows];   //   old running row fin_parent + fin_tok
  int32_t copy_src[kMaxRows], copy_lo[kMaxRows];     // KV: row r <- row copy_src[r] over cache positions [copy_lo, copy_hi]; -1: none
  int32_t copy_hi;
  int32_t cont;                                      // the search goes on (a forward pass for run_tok follows)
  int32_t old_len;                                   // State.cur_len before this step (sequence copy length)
};

// ---- per-row score processing (beam_search.py `_process_log_probs` on the log-softmax of one logits row)
// Philox4x32-10 -> uniform in (0,1); the beam-sample path perturbs scores with Gumbel noise drawn from it.
SVB_HD uint32_t mulhilo32(uint32_t a, uint32_t b, uint32_t* hi) {
  const unsigned long long w = (unsigned long long)a * b;
  *hi = (uint32_t)(w >> 32);
  return (uint32_t)w;
}
SVB_HD float philox_u01(unsigned long long seed, uint32_t c0, uint32_t c1) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t x0 = c0, x1 = c1, x2 = 0x4245414Du, x3 = 0x53563032u;
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, hi1;
    const uint32_t lo0 = mulhilo32(0xD2511F53u, x0, &hi0);
    const uint32_t lo1 = mulhilo32(0xCD9E8D57u, x2, &hi1);
    const uint32_t y0 = hi1 ^ x1 ^ k0, y1 = lo1, y2 = hi0 ^ x3 ^ k1, y3 = lo0;
    x0 = y0; x1 = y1; x2 = y2; x3 = y3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return ((float)(x0 >> 8) + 0.5f) * (1.0f / 16777216.0f);
}
// Gumbel(0,1) for (step, row, token): sorting `score + gumbel` in descending order draws WITHOUT replacement from
// softmax(score) in exactly the order sequential sampling would (Plackett-Luce) = torch.multinomial(softmax, K).
// Counter: (token + (row / 8) * 2^24, step * 8 + row % 8).  Rows 0-7 draw what they drew when the engine held 8 rows, rows
// 8-15 are told apart through the first word (vocabularies are < 2^24, the engine takes <= 2^20).
SVB_HD float gumbel_noise(unsigned long long seed, int step, int row, int token) {
  const float u = philox_u01(seed, (uint32_t)token + ((uint32_t)(row >> 3) << 24), (uint32_t)(step * 8 + (row & 7)));
  return -logf(-logf(u));
}
// log-softmax value -> RepetitionPenaltyLogitsProcessor (on log-probs, generated ids only) -> TemperatureLogitsWarper
SVB_HD float process_logprob(float lp, bool seen, float rep_penalty, bool do_sample, float temperature) {
  if (seen && rep_penalty != 1.0f) lp = lp < 0.0f ? lp * rep_penalty : lp / rep_penalty;
  if (do_sample && temperature != 1.0f) lp = lp / temperature;
  return lp;
}

SVB_HD void init_state(const Params& p, State& s, int first_cache_pos) {
  s.cur_len = 0; s.done = 0; s.parity = 0; s.pad_ = 0;
  for (int r = 0; r < kMaxRows; ++r) {
    s.running_scores[r] = (r % p.nb) == 0 ? 0.0f : kNegBig;       // running_beam_scores[:, 1:] = -1e9
    s.beam_scores[r] = kNegBig;
    s.is_finished[r] = 0; s.fin_len[r] = 0; s.unsatisfied[r] = 1;
    for (int q = 0; q < kMaxRows; ++q) s.div[r][q] = first_cache_pos;   // beams of one image share the whole prefill
  }
}

// fp32 `x / (n ** length_penalty)` as torch evaluates `tensor / python_float`
SVB_HD float len_norm(float x, int n, float length_penalty) {
  return x / (float)pow((double)n, (double)length_penalty);
}

// Merge the per-row candidate lists (each sorted best-first) of one image into its K best: `key` orders (the log-prob for
// beam search, the Gumbel-perturbed log-prob for beam-sample = the order torch.multinomial would have drawn them in),
// ties go to the lower flat index beam * vocab + token.
SVB_HD void merge_candidates(const Params& p, const float* row_key, const float* row_val, const int32_t* row_tok,   // [nb][K]
                             float* out_val, int32_t* out_beam, int32_t* out_tok) {
  int head[kMaxRows];
  for (int j = 0; j < p.nb; ++j) head[j] = 0;
  for (int k = 0; k < p.K; ++k) {
    int best = -1;
    for (int j = 0; j < p.nb; ++j) {
      if (head[j] >= p.K) continue;
      if (best < 0) { best = j; continue; }
      const float a = row_key[j * p.K + head[j]], b = row_key[best * p.K + head[best]];
      if (a > b) best = j;                       // equal keys: the lower beam index (already `best`) wins
    }
    out_val[k] = row_val[best * p.K + head[best]];
    out_tok[k] = row_tok[best * p.K + head[best]];
    out_beam[k] = best;
    head[best]++;
  }
}

// One bookkeeping step over all images.  cand_*: [B][K] from merge_candidates.  run_seq: the CURRENT running sequences
// [B*nb][seq_stride] (read only: the row-0 stop check).  cache_hi: last cache position the forward pass that produced these
// candidates wrote (prefix_len - 1 on the first step: nothing to copy yet).
SVB_HD void beam_step(const Params& p, State& s, const float* cand_val, const int32_t* cand_beam, const int32_t* cand_tok,
                      const int32_t* run_seq, int cache_hi, Plan& plan) {
  const int nb = p.nb, K = p.K, cur = s.cur_len;
  // ---- stopping criteria on the flattened candidates: MaxLength | EOS | StoppingCriteriaSub(row 0 -> everyone)
  bool stop_all = false;
  if (p.n_stop > 0 && cur + 1 >= p.n_stop) {
    const int32_t* parent = run_seq + (int64_t)(0 * nb + cand_beam[0]) * p.seq_stride;
    stop_all = true;
    for (int j = 0; j < p.n_stop; ++j) {
      const int pos = cur + 1 - p.n_stop + j;
      const int32_t t = pos == cur ? cand_tok[0] : parent[pos];
      stop_all = stop_all && (t == p.stop_ids[j]);
    }
  }
  const bool at_max = cur + 1 >= p.max_length;
  bool all_hits = true;
  State n = s;
  for (int b = 0; b < p.B; ++b) {
    const float* val = cand_val + b * K;
    const int32_t* cb = cand_beam + b * K;
    const int32_t* ct = cand_tok + b * K;
    bool hit[kMaxK];
    float run_lp[kMaxK];
    for (int k = 0; k < K; ++k) {
      hit[k] = at_max || stop_all || (p.eos_id >= 0 && ct[k] == p.eos_id);
      all_hits = all_hits && hit[k];
      run_lp[k] = val[k] + (hit[k] ? 1.0f : 0.0f) * kNegBig;          // topk_log_probs + hits * -1e9
    }
    // ---- _get_running_beams_for_next_iteration: top nb of run_lp (stable: lower k first)
    bool used[kMaxK];
    for (int k = 0; k < K; ++k) used[k] = false;
    for (int j = 0; j < nb; ++j) {
      int best = -1;
      for (int k = 0; k < K; ++k)
        if (!used[k] && (best < 0 || run_lp[k] > run_lp[best])) best = k;
      used[best] = true;
      const int r = b * nb + j;
      plan.run_parent[r] = b * nb + cb[best];
      plan.run_tok[r] = ct[best];
      n.running_scores[r] = run_lp[best];
    }
    // ---- _update_finished_beams
    bool all_fin = true;
    for (int j = 0; j < nb; ++j) all_fin = all_fin && s.is_finished[b * nb + j] != 0;
    const float full = (all_fin && p.early_stopping == 1) ? 1.0f : 0.0f;
    const float unsat_not = s.unsatisfied[b] ? 0.0f : 1.0f;
    float merged[kMaxRows + kMaxK];
    bool jf[kMaxK];
    for (int j = 0; j < nb; ++j) merged[j] = s.beam_scores[b * nb + j];
    for (int k = 0; k < K; ++k) {
      jf[k] = hit[k] && k < nb;                                       // hits & top_num_beam_mask
      float f = len_norm(val[k], cur + 1, p.length_penalty);
      f = f + full * kNegBig;
      f = f + unsat_not * kNegBig;
      f = f + (jf[k] ? 0.0f : 1.0f) * kNegBig;
      merged[nb + k] = f;
    }
    bool mused[kMaxRows + kMaxK];
    for (int i = 0; i < nb + K; ++i) mused[i] = false;
    for (int j = 0; j < nb; ++j) {
      int best = -1;
      for (int i = 0; i < nb + K; ++i)
        if (!mused[i] && (best < 0 || merged[i] > merged[best])) best = i;
      mused[best] = true;
      const int r = b * nb + j;
      n.beam_scores[r] = merged[best];
      if (best < nb) {
        plan.fin_old[r] = b * nb + best; plan.fin_parent[r] = -1; plan.fin_tok[r] = -1;
        n.is_finished[r] = s.is_finished[b * nb + best];
        n.fin_len[r] = s.fin_len[b * nb + best];
      } else {
        const int k = best - nb;
        plan.fin_old[r] = -1; plan.fin_parent[r] = b * nb + cb[k]; plan.fin_tok[r] = ct[k];
        n.is_finished[r] = jf[k] ? 1 : 0;
        n.fin_len[r] = cur + 1;
      }
    }
  }
  // ---- KV plan: row r becomes a copy of its parent's row; rows of one image agree below div[r][parent]
  plan.copy_hi = cache_hi;
  for (int r = 0; r < p.B * nb; ++r) {
    const int par = plan.run_parent[r];
    plan.copy_src[r] = par == r ? -1 : par;
    plan.copy_lo[r] = par == r ? 0 : s.div[r][par];
    for (int q = 0; q < p.B * nb; ++q) {
      if (q / nb != r / nb) continue;
      const int pq = plan.run_parent[q];
      n.div[r][q] = pq == par ? cache_hi + 1 : s.div[par][pq];
    }
  }
  // ---- loop bookkeeping
  plan.old_len = cur;
  n.cur_len = cur + 1;
  bool any_unsat = false, all_finished = true;
  for (int b = 0; b < p.B; ++b) {
    // _check_early_stop_heuristic
    const int best_len = (p.early_stopping == 2 && p.length_penalty > 0.0f) ? p.max_length : n.cur_len;
    const float best_running = len_norm(n.running_scores[b * nb], best_len, p.length_penalty);
    float worst = n.beam_scores[b * nb];
    for (int j = 1; j < nb; ++j) worst = fminf(worst, n.beam_scores[b * nb + j]);
    bool any = false;
    for (int j = 0; j < nb; ++j) {
      const float w = n.is_finished[b * nb + j] ? worst : kNegBig;
      any = any || best_running > w;
      all_finished = all_finished && n.is_finished[b * nb + j] != 0;
    }
    n.unsatisfied[b] = (s.unsatisfied[b] && any) ? 1 : 0;
    any_unsat = any_unsat || n.unsatisfied[b];
  }
  // _beam_search_has_unfinished_sequences
  const bool open = !(all_finished && p.early_stopping == 1);
  plan.cont = (any_unsat && open && !all_hits) ? 1 : 0;
  n.done = plan.cont ? 0 : 1;
  n.parity = s.parity ^ 1;
  s = n;
}

}  // namespace svbeam

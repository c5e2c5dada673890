// Token append + HF stop bookkeeping shared by the select kernels (executed by ONE thread).
// Semantics: transformers GenerationMixin._sample loop body (SURVEY.md App. B.3-6) and the reference's
// StoppingCriteriaSub (starvector/model/models/starvector_base.py:9-20, row 0 stops the batch).
#pragma once
#include "sv_kernels.h"

namespace sv {

struct AmaxPair { float v; int i; };
SV_DEVINL AmaxPair amax_better(AmaxPair a, AmaxPair b) { return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a; }

// toks[b] in: selected ids; out: ids after the EOS->pad rule (what gets fed to the next step).  Also compiled for the host:
// sv_spec_accept_host replays the speculative accept walk with it.
__host__ __device__ __forceinline__ void select_apply_tokens(int* toks, int batch, int vocab, GenState* state, const GenParamsDev* p,
                                   uint8_t* seen, int32_t* next_ids, int32_t* out_ids, int advance_len) {
  const int step = state->step;
  for (int b = 0; b < batch; ++b) {
    int tok = toks[b];
    const bool unfinished = state->unfinished[b] != 0;
    if (p->eos_id >= 0 && !unfinished) tok = p->pad_id;                 // next*unfinished + pad*(1-unfinished)
    int32_t* row = out_ids + (int64_t)b * p->out_stride;
    row[step] = tok;
    next_ids[b] = tok;
    toks[b] = tok;
    if (tok >= 0 && tok < vocab) seen[(int64_t)b * vocab + tok] = 1;
    if (p->eos_id >= 0 && tok == p->eos_id) state->unfinished[b] = 0;   // EosTokenCriteria
    const int n = p->n_stop;
    if (n > 0 && step + 1 >= n && (b == 0 || !p->stop_row0_only)) {     // StoppingCriteriaSub
      bool match = true;
      for (int j = 0; j < n; ++j) match = match && (row[step + 1 - n + j] == p->stop_ids[j]);
      if (match) { if (p->stop_row0_only) state->row0_stop = 1; else state->unfinished[b] = 0; }
    }
  }
  // unfinished &= ~stop ; this_peer_finished = unfinished.max()==0 ; advance the counters
  if (state->row0_stop) { for (int b = 0; b < batch; ++b) state->unfinished[b] = 0; state->row0_stop = 0; }
  state->step = step + 1;
  if (advance_len) state->cur_len += 1;
  int any = 0;
  for (int b = 0; b < batch; ++b) any |= state->unfinished[b];
  if (!any || state->step >= p->max_new) state->done = 1;
}

// Session bookkeeping of one row (one thread; sv_session_*): the token goes to out_ids[b][row_step[b]]; EOS, the stop
// sequence matched against the row's own history, or the row's own cap finish the row.  For a batch of one row this is
// exactly select_apply_tokens / append_token + gen_finalize (the row-0 and the per-row stop rule agree there).
SV_DEVINL void session_append_token(int b, int tok, RowState* rows, const GenParamsDev* p, uint8_t* seen, int vocab,
                                    int32_t* next_ids, int32_t* out_ids, int advance_len) {
  const int step = rows->row_step[b];
  int32_t* row = out_ids + (int64_t)b * p->out_stride;
  row[step] = tok;
  next_ids[b] = tok;
  if (tok >= 0 && tok < vocab) seen[(int64_t)b * vocab + tok] = 1;
  bool fin = p->eos_id >= 0 && tok == p->eos_id;                      // EosTokenCriteria
  const int n = p->n_stop;
  if (n > 0 && step + 1 >= n) {                                       // StoppingCriteriaSub on this row
    bool match = true;
    for (int j = 0; j < n; ++j) match = match && (row[step + 1 - n + j] == p->stop_ids[j]);
    fin = fin || match;
  }
  rows->row_step[b] = step + 1;
  if (advance_len) rows->row_len[b] += 1;
  if (fin || step + 1 >= rows->row_max_new[b]) { rows->row_active[b] = 0; rows->event = 1; }
}

// a session row selects this step
SV_DEVINL bool session_row_selects(const RowState* rows, uint32_t row_mask, int b) {
  return ((row_mask >> b) & 1u) && rows->row_active[b] != 0;
}

}  // namespace sv

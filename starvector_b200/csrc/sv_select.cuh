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
__host__ __device__ __forceinline__ void session_append_token(int b, int tok, RowState* rows, const GenParamsDev* p, uint8_t* seen, int vocab,
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

// ---- speculative sessions (sv_spec_session.cu; host replay sv_spec_session_tail_host) --------------------------------
// The accept walk of every live row of ss's map (one thread): row r's columns emit their selected tokens `sel` with the
// plain session's bookkeeping (session_append_token, row_len advanced per token) while each equals the row's next draft.
__host__ __device__ __forceinline__ void spec_session_accept(svspec::SessionState* ss, const int32_t* sel, RowState* rows,
                                                            const GenParamsDev* p, uint8_t* seen, int vocab,
                                                            int32_t* next_ids, int32_t* out_ids) {
  const int n_live = ss->map.n_live;
  if (n_live <= 0) return;
  int nrows = 0, acc = 0;
  for (int c0 = 0; c0 < n_live;) {
    const int r = ss->map.row[c0];
    int m = 1;
    while (c0 + m < n_live && ss->off[c0 + m] != 0) ++m;          // row r's columns [c0, c0 + m)
    acc += svspec::accept(sel + c0, ss->tok + c0, m, [&](int t) {
      session_append_token(r, t, rows, p, seen, vocab, next_ids, out_ids, /*advance_len=*/1);
      return rows->row_active[r] == 0;
    }) - 1;
    ++nrows;
    c0 += m;
  }
  ss->steps += 1; ss->drafted += n_live - nrows; ss->accepted += acc;
}

// Columns of the next verify step at most: the session's slots, and at most tcap - row_len of the first live row beyond
// the live rows' own columns (the QKV epilogue's L2 prefetch reads that row's keys up to pos[0] + n_live).
__host__ __device__ __forceinline__ int spec_session_budget(const RowState* rows, int S, int tcap) {
  int live = 0, room = S;
  for (int r = S - 1; r >= 0; --r)
    if (rows->row_active[r]) { ++live; room = tcap - rows->row_len[r]; }
  room = room > live ? room : live;
  return room < S ? room : S;
}

// The next column map from each live row's want w[r] and drafts d[r][0, w[r]) (svspec::plan_session): row r's first
// column feeds its last emitted token at row_len[r], its column j draft j at row_len[r] + j.  Inert columns repeat the last
// live column's row, position and token (row 0, position 0, token 0 when no row is live).  Returns n_live.
__host__ __device__ __forceinline__ int spec_session_plan(svspec::SessionState* ss, const RowState* rows, const int32_t* out_ids,
                                                          int out_stride, const int32_t* w, const int32_t (*d)[svspec::kMaxCols],
                                                          int tcap) {
  const int S = ss->ncols;
  int32_t g[svspec::kMaxCols], first[svspec::kMaxCols];
  const int n_live = svspec::plan_session(S, rows->row_active, w, spec_session_budget(rows, S, tcap), g, first);
  for (int r = 0; r < S; ++r) {
    const int c = first[r];
    if (c < 0) continue;
    for (int j = 0; j <= g[r]; ++j) {
      ss->map.row[c + j] = r;
      ss->map.pos[c + j] = rows->row_len[r] + j;
      ss->off[c + j] = j;
      ss->tok[c + j] = j == 0 ? out_ids[(int64_t)r * out_stride + rows->row_step[r] - 1] : d[r][j - 1];
    }
  }
  for (int c = n_live; c < S; ++c) {
    const int l = n_live - 1;
    ss->map.row[c] = l >= 0 ? ss->map.row[l] : 0;
    ss->map.pos[c] = l >= 0 ? ss->map.pos[l] : 0;
    ss->tok[c] = l >= 0 ? ss->tok[l] : 0;
    ss->off[c] = 0;
  }
  ss->map.n_live = n_live;
  return n_live;
}

}  // namespace sv

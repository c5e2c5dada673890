// Prompt-lookup speculative decoding (sv_generate_speculative, and inside sessions sv_session_begin_speculative): the column
// map of a verify step, the draft rule, the accept walk and the session's column allocation, shared by the device kernels
// (spec_tail in sv_decode_fused.cu, sv_spec_session.cu) and their host replays (sv_spec_draft_host, sv_spec_accept_host,
// sv_spec_session_plan_host, tests/test_speculative_logic.py, tests/test_spec_session_logic.py).
//
// A verify step feeds the last emitted token and up to k drafted tokens as k + 1 columns of ONE cache row, column c at
// position cur_len + c.  Every column of the weight-ring GEMVs is an independent dot product and every per-row reduction
// keeps its order (DESIGN.md §7e, §7f), so column c's logits are bit-identical to what plain decoding computes at that
// position with that history.  Selection per column is the plain path's (Philox counter step + c), so accepting a draft
// only while the token selected before it equals it reproduces sv_generate's token sequence exactly (DESIGN.md §7g).
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define SVS_HD __host__ __device__ __forceinline__
#else
#define SVS_HD inline
#endif

namespace svspec {

constexpr int kMaxCols = 16;     // columns of a verify step: the rows of one ring GEMV launch

// Per-column map of a verify step.  Column c < n_live decodes cache row row[c] at position pos[c] and appends its K/V
// there; a column c >= n_live is inert: it appends nothing, attends over at most the live keys, and its output is
// discarded.  After the generation finished n_live = 0, so a replay of the step graph writes nothing.
struct ColMap {
  int32_t n_live;
  int32_t row[kMaxCols];
  int32_t pos[kMaxCols];
};

// Device-resident state of one speculative generation.
struct State {
  ColMap map;
  int32_t tok[kMaxCols];           // column inputs: tok[0] = the last emitted token, tok[c] = draft c
  int32_t sel[kMaxCols];           // token selected at each live column (sampled path: written by the select kernel)
  int32_t ncols;                   // columns of the captured step (k + 1)
  int32_t k, max_ngram;            // prompt_lookup_num_tokens, max_matching_ngram_size
  int32_t steps, drafted, accepted;   // verify steps run, drafts proposed, drafts accepted
};

// Length of the longest common suffix of h[0, e) and h[0, n), capped at g (e < n).  The window h[e - l, e) equals the last
// l tokens exactly for l <= this length, so e is where the continuation of an l-gram match starts.
SVS_HD int suffix_match(const int32_t* h, int n, int e, int g) {
  int l = 0;
  while (l < g && l < e && h[e - 1 - l] == h[n - 1 - l]) ++l;
  return l;
}

// The draft taken at continuation start e: h[e, min(e + k, n)), cropped before the first EOS and to `budget` tokens.
SVS_HD int draft_at(const int32_t* h, int n, int e, int k, int eos_id, int budget, int32_t* out) {
  int m = 0;
  for (int i = e; i < n && m < k && m < budget; ++i) {
    if (eos_id >= 0 && h[i] == eos_id) break;
    out[m++] = h[i];
  }
  return m;
}

// transformers' PromptLookupCandidateGenerator.get_candidates over the history h[0, n) (without its forbidden-token crop,
// which only matters for logits processors that output -inf): n-gram sizes from min(max_ngram, n - 1) down to 1, the
// earliest match whose continuation is non-empty, up to k tokens of it, cropped at the first EOS; then clamped to the
// remaining budget.  The largest size with a usable match is max_e suffix_match(e) over continuation starts e < n, and
// its earliest match is the smallest such e: the device computes both with one CTA-wide reduction each.
SVS_HD int draft_host(const int32_t* h, int n, int k, int max_ngram, int eos_id, int budget, int32_t* out) {
  if (n < 2 || k < 1 || budget < 1) return 0;
  int best = 0, at = -1;
  for (int e = 1; e < n; ++e) {
    const int l = suffix_match(h, n, e, max_ngram);
    if (l > best) { best = l; at = e; }
  }
  return best > 0 ? draft_at(h, n, at, k, eos_id, budget, out) : 0;
}

// Column b's repetition-penalty set is the row's seen set plus drafts 1..b: whether id i is one of those drafts
// (cols[c] = input token of column c).
SVS_HD bool drafted(const int* cols, int b, int i) {
  bool hit = false;
  for (int j = 1; j <= b; ++j) hit = hit || cols[j] == i;
  return hit;
}

// The accept walk of one verify step: column c's selected token is emitted (with the plain path's per-token bookkeeping,
// `emit`, which returns true once the generation is done), and the walk continues while it equals draft c + 1.
// Returns the number of tokens emitted.
template <class Emit>
SVS_HD int accept(const int32_t* sel, const int32_t* tok, int n_live, Emit&& emit) {
  int m = 0;
  for (int c = 0; c < n_live; ++c) {
    ++m;
    if (emit(sel[c]) || c + 1 >= n_live || sel[c] != tok[c + 1]) break;
  }
  return m;
}

// ---- speculation inside a continuous-batching session (sv_session_begin_speculative, DESIGN.md §7i) ----------------
// A verify step of a session of S slots has S columns.  Live row r gets 1 + g_r contiguous columns, the rows in slot order:
// its first column feeds its last emitted token at row_len[r], column j of the row its draft j at row_len[r] + j.  Each
// column selects with the plain session's rule for that token (sv_spec_session.cu), so the drafts change the speed only.
struct SessionState {
  ColMap map;                      // first, so that &ss->map is the step's column map
  int32_t tok[kMaxCols];           // column inputs
  int32_t sel[kMaxCols];           // token selected at each live column (sampled path: written by the select kernel)
  int32_t off[kMaxCols];           // column's offset within its row: 0 at the row's first column, j at its draft j
  int32_t ncols;                   // columns of the captured step (the session's slots)
  int32_t k, max_ngram;            // prompt_lookup_num_tokens, max_matching_ngram_size
  int32_t steps, drafted, accepted;   // verify steps run, drafts proposed, drafts accepted
};

// The column allocation: every live row (active[r] != 0) gets its own first column; the spare columns (at most `budget`
// columns in all, and at most S) are handed out round-robin in slot order, one draft per pass to each live row still below
// its want w[r], until none are left or no row wants more.  Writes g[r] (drafts granted, 0 for idle rows) and first[r] (the
// row's first column, -1 for idle rows); returns n_live, the sum of 1 + g[r] over the live rows.
SVS_HD int plan_session(int S, const int32_t* active, const int32_t* w, int budget, int32_t* g, int32_t* first) {
  int live = 0;
  for (int r = 0; r < S; ++r) { g[r] = 0; live += active[r] != 0; }
  int spare = (budget < S ? budget : S) - live;
  for (bool more = true; spare > 0 && more;) {
    more = false;
    for (int r = 0; r < S && spare > 0; ++r)
      if (active[r] && g[r] < w[r]) { ++g[r]; --spare; more = true; }
  }
  int c = 0;
  for (int r = 0; r < S; ++r) {
    first[r] = active[r] ? c : -1;
    if (active[r]) c += 1 + g[r];
  }
  return c;
}

// The column map after an accept: live columns at cur_len + c; inert ones at the last live position (after the finish,
// n_live = 0: the last position already in the cache), so they never read a key this step did not write.
SVS_HD void set_map(ColMap& m, int ncols, int n_live, int cur_len) {
  m.n_live = n_live;
  int last = cur_len + n_live - 1;
  if (last < 0) last = 0;
  for (int c = 0; c < ncols; ++c) {
    m.row[c] = 0;
    m.pos[c] = c < n_live ? cur_len + c : last;
  }
}

}  // namespace svspec

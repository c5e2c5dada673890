// Sampled token selection (select_sample_body) and the helpers it shares with the other kernels of sv_kernels_basic.cu.
// A header so that the speculative-session select kernel (sv_spec_session.cu) instantiates the same body, and so the same
// bits, as the plain session's sampler.
#pragma once
#include "sv_select.cuh"

namespace sv {

// ------------------------------------------------------------------------------------------
// block reductions
template <int NT>
SV_DEVINL float block_sum(float v, float* sm) {
  v = warp_sum(v);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sm[w] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int i = 0; i < NT / 32; ++i) r += sm[i];
  return r;
}

SV_DEVINL void append_token(int b, int tok, GenState* state, const GenParamsDev* p, uint8_t* seen, int vocab,
                            int32_t* next_ids, int32_t* out_ids) {
  const int step = state->step;
  const bool unfinished = state->unfinished[b] != 0;
  if (p->eos_id >= 0 && !unfinished) tok = p->pad_id;                 // next*unfinished + pad*(1-unfinished)
  int32_t* row = out_ids + (int64_t)b * p->out_stride;
  row[step] = tok;
  next_ids[b] = tok;
  if (tok >= 0 && tok < vocab) seen[(int64_t)b * vocab + tok] = 1;
  if (p->eos_id >= 0 && tok == p->eos_id) state->unfinished[b] = 0;   // EosTokenCriteria
  const int n = p->n_stop;
  if (n > 0 && step + 1 >= n && (b == 0 || !p->stop_row0_only)) {     // StoppingCriteriaSub (row 0 only)
    bool match = true;
    for (int j = 0; j < n; ++j) match = match && (row[step + 1 - n + j] == p->stop_ids[j]);
    if (match) {
      if (p->stop_row0_only) state->row0_stop = 1;
      else state->unfinished[b] = 0;
    }
  }
}

// ---- sampling: repetition penalty -> temperature -> top-p -> multinomial (App. B.3), Philox stream.
SV_DEVINL uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
  unsigned long long p = (unsigned long long)a * b;
  *hi = (uint32_t)(p >> 32);
  return (uint32_t)p;
}
SV_DEVINL float philox_uniform(unsigned long long seed, uint32_t c0, uint32_t c1) {   // Philox4x32-10
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t x0 = c0, x1 = c1, x2 = 0x5356u, x3 = 0x42323030u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, hi1;
    uint32_t lo0 = mulhilo(0xD2511F53u, x0, &hi0);
    uint32_t lo1 = mulhilo(0xCD9E8D57u, x2, &hi1);
    uint32_t y0 = hi1 ^ x1 ^ k0, y1 = lo1, y2 = hi0 ^ x3 ^ k1, y3 = lo0;
    x0 = y0; x1 = y1; x2 = y2; x3 = y3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return ((float)(x0 >> 8) + 0.5f) * (1.0f / 16777216.0f);
}

constexpr int kSampleThreads = 1024;

// `probs` is an fp32 scratch row [B][vocab] (L2 resident): the kernel makes ~34 passes over it.
// SPEC (the verify step of sv_generate_speculative): block b is column b of cache row 0; only live columns select, with
// row 0's seen set plus drafts 1..b and the counter of the token the column would be in a plain run (0, step + b); the
// token goes to sp->sel[b] and the bookkeeping is left to spec_accept_kernel.
// SESS (the verify step of a speculative session): block b is column b of ss's map, at offset j = ss->off[b] in cache row
// r = ss->map.row[b]; only live columns select, with row r's seen set plus the row's drafts 1..j and the counter a plain
// session gives that token (row_seed[r], 0, row_step[r] + j); the token goes to ss->sel[b].
template <bool ROWS, bool SPEC = false, bool SESS = false>
SV_DEVINL void select_sample_body(const bf16* __restrict__ logits, int vocab, GenState* state,
                                  const GenParamsDev* __restrict__ p, uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                                  float* __restrict__ probs, RowState* rows, uint32_t row_mask, int advance_len,
                                  svspec::State* sp = nullptr, svspec::SessionState* ss = nullptr) {
  const int b = blockIdx.x, tid = threadIdx.x;
  if constexpr (SESS) {
    if (b >= ss->map.n_live) return;
  } else if constexpr (ROWS) {
    if (!session_row_selects(rows, row_mask, b)) return;
  } else {
    if (state->done) return;
  }
  if constexpr (SPEC) {
    if (b >= sp->map.n_live) return;
  }
  __shared__ float smf[32];
  __shared__ float s_bcast;
  __shared__ int s_tok;
  __shared__ int s_cols[(SPEC || SESS) ? svspec::kMaxCols : 1];
  if constexpr (SPEC) {
    if (tid < svspec::kMaxCols) s_cols[tid] = sp->tok[tid];
    __syncthreads();
  }
  int srow = SPEC ? 0 : b, dbase = 0, nd = b;      // seen row; the drafts that join it: cols[dbase + 1 .. dbase + nd]
  if constexpr (SESS) {
    if (tid < svspec::kMaxCols) s_cols[tid] = ss->tok[tid];
    __syncthreads();
    srow = ss->map.row[b];
    nd = ss->off[b];
    dbase = b - nd;
  }
  const bf16* lr = logits + (int64_t)b * vocab;
  const uint8_t* sr = seen + (int64_t)srow * vocab;
  float* pr = probs + (int64_t)b * vocab;
  const float rp = p->rep_penalty, invT = 1.0f / p->temperature;
  float mx = -INFINITY;
  for (int i = tid; i < vocab; i += kSampleThreads) {
    float v = __bfloat162float(lr[i]);
    if (rp != 1.0f && (sr[i] || ((SPEC || SESS) && svspec::drafted(s_cols + dbase, nd, i)))) v = v < 0.f ? v * rp : v / rp;   // RepetitionPenaltyLogitsProcessor
    v *= invT;                                                         // TemperatureLogitsWarper
    pr[i] = v;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  if ((tid & 31) == 0) smf[tid >> 5] = mx;
  __syncthreads();
  mx = smf[0];
  for (int w = 1; w < 32; ++w) mx = fmaxf(mx, smf[w]);
  float z = 0.f;
  for (int i = tid; i < vocab; i += kSampleThreads) { float e = __expf(pr[i] - mx); pr[i] = e; z += e; }
  z = block_sum<kSampleThreads>(z, smf);
  const float invz = 1.0f / z;
  // TopPLogitsWarper: keep a token iff the mass of strictly more probable tokens is < top_p.
  // Bisection on the probability threshold: find (the infimum of) q with mass(p > q) < top_p.
  float lo = 0.f, hi = 1.f;
  const float top_p = p->top_p;
  if (top_p < 1.0f) {
    for (int it = 0; it < 30; ++it) {
      const float mid = 0.5f * (lo + hi);
      float m = 0.f;
      for (int i = tid; i < vocab; i += kSampleThreads) { float q = pr[i] * invz; m += q > mid ? q : 0.f; }
      m = block_sum<kSampleThreads>(m, smf);
      if (m < top_p) hi = mid; else lo = mid;
    }
  }                                                                   // top_p == 1: lo stays 0, every id with p > 0 is kept
  // kept set = { p > lo }.  Thread `tid` owns ids [tid*per, tid*per+per) so the scan runs in id order.
  const int per = (vocab + kSampleThreads - 1) / kSampleThreads;
  const int i0 = tid * per, i1 = min(i0 + per, vocab);
  float own = 0.f;
  for (int i = i0; i < i1; ++i) { float q = pr[i] * invz; own += q > lo ? q : 0.f; }
  float incl = own;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { float n = __shfl_up_sync(0xffffffffu, incl, o); if ((tid & 31) >= o) incl += n; }
  __syncthreads();
  if ((tid & 31) == 31) smf[tid >> 5] = incl;
  __syncthreads();
  float base = 0.f, total = 0.f;
  for (int w = 0; w < 32; ++w) { if (w < (tid >> 5)) base += smf[w]; total += smf[w]; }
  if (tid == 0) {
    // session rows: the counter of a one-row generate with the row's own seed (the slot index does not enter it)
    if constexpr (SESS) {   // row and offset read again: keeping them live through the body costs a spill
      const int r = ss->map.row[b];
      s_bcast = philox_uniform(rows->row_seed[r], 0u, (uint32_t)(rows->row_step[r] + ss->off[b])) * total;
    } else if constexpr (ROWS) s_bcast = philox_uniform(rows->row_seed[b], 0u, (uint32_t)rows->row_step[b]) * total;
    else if constexpr (SPEC) s_bcast = philox_uniform(p->seed, 0u, (uint32_t)(state->step + b)) * total;
    else s_bcast = philox_uniform(p->seed, (uint32_t)b, (uint32_t)state->step) * total;
    s_tok = -1;
  }
  __syncthreads();
  const float target = s_bcast;
  // torch.multinomial(probs, 1): every thread whose interval starts at or below the target proposes the id its scan stops
  // at, or its last kept id when the scan runs off its end; ids rise with the thread index, so the maximum is the proposal
  // of the last such thread.  (Also requiring `target < excl + own` leaves gaps: a thread's upper end and its neighbour's
  // lower end are different fp32 expressions, and a target between them was claimed by nobody.)
  const float excl = base + incl - own;
  if (own > 0.f && target >= excl) {
    float acc = excl; int tok = -1;
    for (int i = i0; i < i1; ++i) {
      float q = pr[i] * invz;
      if (q > lo) { tok = i; acc += q; if (target < acc) break; }
    }
    atomicMax(&s_tok, tok);
  }
  __syncthreads();
  if (tid == 0) {
    int tok = s_tok;
    if (tok < 0) {                                                     // no id has any mass (a row of -inf): last kept id
      for (int i = vocab - 1; i >= 0; --i) if (pr[i] * invz > lo) { tok = i; break; }
      if (tok < 0) tok = 0;
    }
    if constexpr (SESS) ss->sel[b] = tok;
    else if constexpr (ROWS) session_append_token(b, tok, rows, p, seen, vocab, next_ids, out_ids, advance_len);
    else if constexpr (SPEC) sp->sel[b] = tok;
    else append_token(b, tok, state, p, seen, vocab, next_ids, out_ids);
  }
}

}  // namespace sv

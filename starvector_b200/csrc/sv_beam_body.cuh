// Device bodies of the beam-search kernels, shared by sv_beam.cu (one search over the rectangle of rows) and
// sv_beam_session.cu (beam sessions: groups of rows with their own state).  The two forms are instantiated in separate
// translation units, so each one's code generation (inlining included) does not depend on the other.
#pragma once
#include <cmath>

#include "sv_beam_core.h"
#include "sv_kernels.h"

namespace sv {

using svbeam::Params;
using svbeam::Plan;
using svbeam::State;

constexpr int kBeamThreads = 1024;

namespace {

SV_DEVINL float block_max_f(float v, float* sm) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sm[0];
#pragma unroll
  for (int w = 1; w < kBeamThreads / 32; ++w) r = fmaxf(r, sm[w]);
  return r;
}
SV_DEVINL float block_sum_f(float v, float* sm) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int w = 0; w < kBeamThreads / 32; ++w) r += sm[w];     // fixed order: deterministic
  return r;
}
// (value desc, index asc) order: is (bv, bi) ahead of (av, ai)?
SV_DEVINL bool ahead(float bv, int bi, float av, int ai) { return bv > av || (bv == av && bi < ai); }

// block-wide first element in (value desc, index asc) order among those strictly BEHIND (lim_v, lim_i)
SV_DEVINL void block_argmax_behind(const float* __restrict__ s, int V, float lim_v, int lim_i, float* smf, int* smi,
                                   float& out_v, int& out_i) {
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += kBeamThreads) {
    const float v = s[i];
    if (ahead(lim_v, lim_i, v, i) && ahead(v, i, bv, bi)) { bv = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ahead(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { smf[threadIdx.x >> 5] = bv; smi[threadIdx.x >> 5] = bi; }
  __syncthreads();
  bv = smf[0]; bi = smi[0];
#pragma unroll
  for (int w = 1; w < kBeamThreads / 32; ++w)
    if (ahead(smf[w], smi[w], bv, bi)) { bv = smf[w]; bi = smi[w]; }
  out_v = bv; out_i = bi;
}

}  // namespace

// ---- K1: per-row candidates -------------------------------------------------------------------------------------
// dynamic shared memory: float score[V] | uint32 seen[(V + 31) / 32]
// SESSION: the beam-session variant.  CTA r serves group g = r / nb at local row j = r % nb: the group's own Params /
// State (pp[g], st[g], group-local rows, B = 1), the sequence buffers [2][kMaxRows][stride] by global row.  Groups outside
// group_mask or not live (rows->row_active of their first row) return, as do finished ones.
template <bool SESSION>
SV_DEVINL void beam_candidates_body(const bf16* __restrict__ logits, const Params* __restrict__ pp, const State* st,
                                    const int32_t* __restrict__ run_seq, float* __restrict__ cand_key,
                                    float* __restrict__ cand_val, int32_t* __restrict__ cand_tok, const RowState* rows,
                                    uint32_t group_mask) {
  const int r = blockIdx.x, tid = threadIdx.x;
  int j = r, half;
  if constexpr (SESSION) {
    const int nb = pp->nb, g = r / nb;
    if (!((group_mask >> g) & 1u) || !rows->row_active[g * nb]) return;
    pp += g; st += g; j = r % nb; half = svbeam::kMaxRows;
  }
  if (st->done) return;
  extern __shared__ float sc[];
  __shared__ float smf[kBeamThreads / 32];
  __shared__ int smi[kBeamThreads / 32];
  const int V = pp->vocab, K = pp->K, R = pp->B * pp->nb, cur = st->cur_len;
  if constexpr (!SESSION) half = R;
  const float rp = pp->rep_penalty, T = pp->temperature, top_p = pp->top_p;
  const bool sample = pp->do_sample != 0;
  uint32_t* seen = reinterpret_cast<uint32_t*>(sc + V);
  const bool use_rp = rp != 1.0f && cur > 0;
  if (use_rp) {                       // tokens this running beam has generated (RepetitionPenaltyLogitsProcessor input)
    for (int i = tid; i < (V + 31) / 32; i += kBeamThreads) seen[i] = 0u;
    __syncthreads();
    const int32_t* seq = run_seq + ((int64_t)st->parity * half + r) * pp->seq_stride;
    for (int i = tid; i < cur; i += kBeamThreads) {
      const int t = seq[i];
      if (t >= 0 && t < V) atomicOr(&seen[t >> 5], 1u << (t & 31));
    }
    __syncthreads();
  }
  const bf16* lr = logits + (int64_t)r * V;
  // log_softmax(logits.float()): x - max - log(sum(exp(x - max)))
  float mx = -INFINITY;
  for (int i = tid; i < V; i += kBeamThreads) { const float x = __bfloat162float(lr[i]); sc[i] = x; mx = fmaxf(mx, x); }
  mx = block_max_f(mx, smf);
  float z = 0.f;
  for (int i = tid; i < V; i += kBeamThreads) z += expf(sc[i] - mx);
  z = block_sum_f(z, smf);
  const float logz = logf(z);
  for (int i = tid; i < V; i += kBeamThreads) {
    const bool sn = use_rp && ((seen[i >> 5] >> (i & 31)) & 1u);
    sc[i] = svbeam::process_logprob((sc[i] - mx) - logz, sn, rp, sample, T);
  }
  __syncthreads();
  if (sample && top_p < 1.0f) {
    // TopPLogitsWarper(min_tokens_to_keep): a token stays iff the mass of strictly more probable tokens is < top_p, or it is
    // one of the min_keep most probable.  Bisection on the probability threshold (as the one-beam sampler does).
    float m2 = -INFINITY;
    for (int i = tid; i < V; i += kBeamThreads) m2 = fmaxf(m2, sc[i]);
    m2 = block_max_f(m2, smf);
    float z2 = 0.f;
    for (int i = tid; i < V; i += kBeamThreads) z2 += expf(sc[i] - m2);
    z2 = block_sum_f(z2, smf);
    const float inv = 1.0f / z2;
    float lo = 0.f, hi = 1.f;
    for (int it = 0; it < 30; ++it) {
      const float mid = 0.5f * (lo + hi);
      float m = 0.f;
      for (int i = tid; i < V; i += kBeamThreads) { const float q = expf(sc[i] - m2) * inv; m += q > mid ? q : 0.f; }
      m = block_sum_f(m, smf);
      if (m < top_p) hi = mid; else lo = mid;
    }
    float kv = INFINITY;                 // the min_keep-th best (value, index): everything not behind it is kept
    int ki = -1;
    for (int j = 0; j < pp->min_keep; ++j) block_argmax_behind(sc, V, kv, ki, smf, smi, kv, ki);
    __syncthreads();
    for (int i = tid; i < V; i += kBeamThreads) {
      const float v = sc[i];
      const bool keep = (expf(v - m2) * inv > lo) || !ahead(kv, ki, v, i);
      if (!keep) sc[i] = -INFINITY;
    }
    __syncthreads();
  }
  // ordering keys: score + running beam score (+ Gumbel noise for beam-sample); K rounds of block argmax with removal
  const float rs = st->running_scores[j];
  for (int i = tid; i < V; i += kBeamThreads) {
    float key = sc[i] + rs;
    if (sample && key > -INFINITY) key += svbeam::gumbel_noise(pp->seed, cur, j, i);    // a one-image search's counter
    sc[i] = key;
  }
  __syncthreads();
  for (int k = 0; k < K; ++k) {
    float bv; int bi;
    block_argmax_behind(sc, V, INFINITY, -1, smf, smi, bv, bi);
    if (tid == 0) {
      const int tok = bi == 0x7fffffff ? 0 : bi;
      // the candidate's log-prob, recomputed from the logit (the key may carry noise)
      const bool sn = use_rp && ((seen[tok >> 5] >> (tok & 31)) & 1u);
      const float s = svbeam::process_logprob((__bfloat162float(lr[tok]) - mx) - logz, sn, rp, sample, T);
      cand_key[r * K + k] = bv;
      cand_val[r * K + k] = bv == -INFINITY ? -INFINITY : s + rs;
      cand_tok[r * K + k] = tok;
      sc[tok] = -INFINITY;
    }
    __syncthreads();
  }
}

// ---- K3: KV suffix copies (phase 0: parent rows -> staging, phase 1: staging -> child rows) -------------------------------
// grid (chunks, rows, layers).  K [row][kvh][tcap][D]: one contiguous run per kv head; V^T [row][kvh][D][tcap]: one short
// run per (kv head, dim).  SESSION: row r follows its group's plan (plan[r / nb], group-local rows); groups outside
// group_mask or not live copy nothing.
template <bool SESSION>
SV_DEVINL void beam_kv_copy_body(bf16* kc, bf16* vc, bf16* kc2, bf16* vc2, int64_t layer_stride, int n_kv, int tcap, int D,
                                 const Plan* __restrict__ plan, int phase, const Params* __restrict__ pp,
                                 const RowState* rows, uint32_t group_mask) {
  const int r = blockIdx.y, layer = blockIdx.z;
  int j = r, row0 = 0;
  if constexpr (SESSION) {
    const int nb = pp->nb, g = r / nb;
    if (!((group_mask >> g) & 1u) || !rows->row_active[g * nb]) return;
    plan += g; j = r % nb; row0 = g * nb;
  }
  if (!plan->cont) return;
  const int src_row = plan->copy_src[j];
  if (src_row < 0) return;
  const int lo = plan->copy_lo[j], hi = plan->copy_hi;
  if (lo > hi) return;
  const int n = hi - lo + 1;
  const int64_t row_elems = (int64_t)n_kv * tcap * D;
  const bf16* ks = (phase == 0 ? kc : kc2) + layer * layer_stride + (phase == 0 ? row0 + src_row : r) * row_elems;
  const bf16* vs = (phase == 0 ? vc : vc2) + layer * layer_stride + (phase == 0 ? row0 + src_row : r) * row_elems;
  bf16* kd = (phase == 0 ? kc2 : kc) + layer * layer_stride + r * row_elems;
  bf16* vd = (phase == 0 ? vc2 : vc) + layer * layer_stride + r * row_elems;
  const int vec_per_key = D / 8;
  const int nk = n_kv * n * vec_per_key;                       // 16-byte vectors of K
  const int t0 = blockIdx.x * blockDim.x + threadIdx.x, ts = gridDim.x * blockDim.x;
  for (int i = t0; i < nk; i += ts) {
    const int kvh = i / (n * vec_per_key), rem = i % (n * vec_per_key);
    const int64_t off = ((int64_t)kvh * tcap + lo) * D + (int64_t)rem * 8;
    *reinterpret_cast<uint4*>(kd + off) = *reinterpret_cast<const uint4*>(ks + off);
  }
  const int nv = n_kv * D * n;                                 // 2-byte elements of V^T
  for (int i = t0; i < nv; i += ts) {
    const int line = i / n, t = i % n;                         // line = kvh * D + dim
    const int64_t off = (int64_t)line * tcap + lo + t;
    vd[off] = vs[off];
  }
}

}  // namespace sv

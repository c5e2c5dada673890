// Beam sessions (sv_beam_session_*, DESIGN.md §7h): the beam kernels of sv_beam.cu for groups of cache rows, each group
// one image's search with its own Params / State / Plan.  The candidate and KV-copy kernels are the session instantiations
// of the bodies in sv_beam_body.cuh; they live in a translation unit of their own so that the rectangle kernels of
// sv_beam.cu compile to the code they had before these existed (nvcc's inlining of shared callees such as pow depends on
// how many kernels of a unit call them).
#include "sv_beam_body.cuh"

namespace sv {

__global__ void __launch_bounds__(kBeamThreads) beam_session_candidates_kernel(
    const bf16* __restrict__ logits, const Params* __restrict__ pp, const State* st, const int32_t* __restrict__ run_seq,
    float* __restrict__ cand_key, float* __restrict__ cand_val, int32_t* __restrict__ cand_tok, const RowState* rows,
    uint32_t group_mask) {
  beam_candidates_body<true>(logits, pp, st, run_seq, cand_key, cand_val, cand_tok, rows, group_mask);
}

// ---- K2 of a beam session: one CTA per group g = blockIdx.x (CTAs past the session's slots return).  The bookkeeping,
// sequence moves and next-token embedding of beam_step_kernel (sv_beam.cu) on the group's own Params / State / Plan
// (B = 1, group-local rows), its candidates and its slots' rows, with positions from rows->row_len instead of GenState.
// While the search goes on, its slots advance together; at the finish they leave row_active, row_step of its first slot
// receives the length of the best hypothesis (sv_beam_search's n_gen) and rows->event is raised.  (beam_step_kernel
// itself is left as it is: routing it through a shared template body changes the code nvcc makes for it.)
__global__ void __launch_bounds__(kBeamThreads) beam_session_step_kernel(
    const Params* __restrict__ pp, State* st, Plan* plan_out, const float* __restrict__ cand_key,
    const float* __restrict__ cand_val, const int32_t* __restrict__ cand_tok, int32_t* run_seq, int32_t* fin_seq,
    RowState* rows, uint32_t group_mask, int slots, int advance, const bf16* __restrict__ wte, const bf16* __restrict__ wpe,
    bf16* __restrict__ x, int h, int n_positions, int32_t* next_ids) {
  const int g = blockIdx.x, row0 = g * pp->nb;
  // every thread reads the flags BEFORE thread 0 can rewrite them below (the group may finish in this very step)
  if (row0 >= slots || !((group_mask >> g) & 1u) || !rows->row_active[row0]) return;
  pp += g; st += g; plan_out += g;
  const int was_done = st->done;
  __syncthreads();
  if (was_done) return;
  __shared__ Plan plan;
  __shared__ int s_oldp, s_pos;
  __shared__ int s_finlen[svbeam::kMaxRows];
  const int tid = threadIdx.x;
  const int nb = pp->nb, K = pp->K, stride = pp->seq_stride;
  constexpr int HR = svbeam::kMaxRows;                      // rows per parity half of the sequence buffers
  cand_key += row0 * K; cand_val += row0 * K; cand_tok += row0 * K;
  run_seq += (int64_t)row0 * stride; fin_seq += (int64_t)row0 * stride;
  const int pad_fill = pp->pad_id;
  if (tid == 0) {
    const Params p = *pp;                    // B = 1
    float mval[svbeam::kMaxK];
    int32_t mbeam[svbeam::kMaxK], mtok[svbeam::kMaxK];
    svbeam::merge_candidates(p, cand_key, cand_val, cand_tok, mval, mbeam, mtok);
    State s = *st;
    s_oldp = s.parity;
    const int len = rows->row_len[row0];
    svbeam::beam_step(p, s, mval, mbeam, mtok, run_seq + (int64_t)s.parity * HR * stride, advance ? len : len - 1, plan);
    *st = s;
    *plan_out = plan;
    const int nlen = plan.cont && advance ? len + 1 : len;
    for (int r = 0; r < nb; ++r) {
      rows->row_len[row0 + r] = nlen;
      rows->row_step[row0 + r] = s.cur_len;
      if (!plan.cont) rows->row_active[row0 + r] = 0;
    }
    if (!plan.cont) {
      rows->row_step[row0] = s.fin_len[0] < p.max_length ? s.fin_len[0] : p.max_length;
      rows->event = 1;
    }
    s_pos = nlen;
    for (int r = 0; r < nb; ++r) s_finlen[r] = s.fin_len[r];
  }
  __syncthreads();
  const int oldp = s_oldp, newp = oldp ^ 1, L = plan.old_len;
  for (int r = 0; r < nb; ++r) {
    const int32_t* src = run_seq + ((int64_t)oldp * HR + plan.run_parent[r]) * stride;
    int32_t* dst = run_seq + ((int64_t)newp * HR + r) * stride;
    for (int i = tid; i <= L; i += kBeamThreads) dst[i] = i < L ? src[i] : plan.run_tok[r];
    int32_t* dstf = fin_seq + ((int64_t)newp * HR + r) * stride;
    if (plan.fin_old[r] >= 0) {
      const int32_t* srcf = fin_seq + ((int64_t)oldp * HR + plan.fin_old[r]) * stride;
      const int n = s_finlen[r];
      for (int i = tid; i <= L; i += kBeamThreads) dstf[i] = i < n ? srcf[i] : pad_fill;
    } else {
      const int32_t* srcp = run_seq + ((int64_t)oldp * HR + plan.fin_parent[r]) * stride;
      for (int i = tid; i <= L; i += kBeamThreads) dstf[i] = i < L ? srcp[i] : plan.fin_tok[r];
    }
  }
  if (!plan.cont) return;
  // the group's next input rows: wte[token] + wpe[its position] (bf16 add), as beam_step_kernel writes them
  int pos = s_pos;
  pos = pos >= n_positions ? n_positions - 1 : pos;
  const int hv = h >> 3, V = pp->vocab;
  for (int i = tid; i < nb * hv; i += kBeamThreads) {
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
    *reinterpret_cast<uint4*>(x + (int64_t)(row0 + b) * h + c) = pack8(e);
  }
  if (tid < nb) next_ids[row0 + tid] = plan.run_tok[tid];
}

__global__ void __launch_bounds__(256) beam_session_kv_copy_kernel(bf16* kc, bf16* vc, bf16* kc2, bf16* vc2,
                                                                   int64_t layer_stride, int n_kv, int tcap, int D,
                                                                   const Plan* __restrict__ plan, int phase,
                                                                   const Params* __restrict__ pp, const RowState* rows,
                                                                   uint32_t group_mask) {
  beam_kv_copy_body<true>(kc, vc, kc2, vc2, layer_stride, n_kv, tcap, D, plan, phase, pp, rows, group_mask);
}

cudaError_t beam_session_init(int vocab) {
  const size_t need = beam_candidates_smem(vocab);
  if (need > 220 * 1024) return cudaErrorInvalidValue;
  return cudaFuncSetAttribute(beam_session_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need);
}

void launch_beam_session_candidates(const bf16* logits, int vocab, int slots, const Params* p, const State* st,
                                    const int32_t* run_seq, float* cand_key, float* cand_val, int32_t* cand_tok,
                                    const RowState* rows, uint32_t group_mask, cudaStream_t st_) {
  beam_session_candidates_kernel<<<slots, kBeamThreads, beam_candidates_smem(vocab), st_>>>(
      logits, p, st, run_seq, cand_key, cand_val, cand_tok, rows, group_mask);
  count_launch();
}

void launch_beam_session_step(const Params* p, State* st, Plan* plan, const float* cand_key, const float* cand_val,
                              const int32_t* cand_tok, int32_t* run_seq, int32_t* fin_seq, RowState* rows,
                              uint32_t group_mask, int slots, int advance, const bf16* wte, const bf16* wpe, bf16* x, int h,
                              int n_positions, int32_t* next_ids, cudaStream_t st_) {
  // one CTA per group of the smallest beam width (2); the CTAs past the session's groups return
  beam_session_step_kernel<<<(slots + 1) / 2, kBeamThreads, 0, st_>>>(p, st, plan, cand_key, cand_val, cand_tok, run_seq,
                                                                       fin_seq, rows, group_mask, slots, advance, wte, wpe,
                                                                       x, h, n_positions, next_ids);
  count_launch();
}

void launch_beam_session_kv_copy(bf16* kc, bf16* vc, bf16* kc2, bf16* vc2, int64_t layer_stride, int n_layer, int slots,
                                 int n_kv, int tcap, int D, const Params* p, const Plan* plan, const RowState* rows,
                                 uint32_t group_mask, cudaStream_t st_) {
  for (int phase = 0; phase < 2; ++phase)
    beam_session_kv_copy_kernel<<<dim3(4, slots, n_layer), 256, 0, st_>>>(kc, vc, kc2, vc2, layer_stride, n_kv, tcap, D,
                                                                          plan, phase, p, rows, group_mask);
  count_launch(2);
}

}  // namespace sv

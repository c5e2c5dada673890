// Prompt-lookup speculation inside a continuous-batching session (sv_session_begin_speculative, DESIGN.md §7i): the
// selection and bookkeeping kernels of a session verify step.  The decode step itself is the engine's, run over the S
// columns of svspec::SessionState::map (the EPI_QKV_MAP ring GEMV and the cluster attention's map variant).
//
// Column c of live row r at offset j selects the token a plain session selects at row_step[r] + j with the same history:
// its repetition-penalty set is seen[r] plus the row's drafts 1..j, its Philox counter (row_seed[r], 0, row_step[r] + j).
// Accepting a draft only while the token selected before it equals it therefore reproduces the plain session's tokens.
#include "sv_kernels.h"
#include "sv_sample.cuh"

namespace sv {
namespace {

SV_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
SV_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
void launch_ex(void (*kern)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, args...);
  count_launch();
}

// What follows the selection of a session verify step, in one 1024-thread CTA: with `accept`, every live row's accept
// walk (spec_session_accept); then, when the live rows leave spare columns, each live row's prompt-lookup draft over its
// own tokens out_ids[r, 0, row_step[r]) (svspec::draft_host's rule, its two searches spread over the CTA, cropped to the
// row's remaining cap), the column allocation and map (spec_session_plan), and the embeddings wte[tok] + wpe[pos] of every
// column of the next step.
SV_DEVINL void spec_session_tail(const int32_t* sel, bool accept, svspec::SessionState* ss, RowState* rows,
                                 const GenParamsDev* __restrict__ p, uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                                 int vocab, const bf16* __restrict__ wte, const bf16* __restrict__ wpe, bf16* __restrict__ x,
                                 int h, int n_positions, int tcap) {
  __shared__ int s_best, s_at, s_spare;
  __shared__ int32_t s_w[svspec::kMaxCols], s_d[svspec::kMaxCols][svspec::kMaxCols];
  __shared__ int s_n[svspec::kMaxCols], s_room[svspec::kMaxCols];
  __shared__ int s_col_tok[svspec::kMaxCols], s_col_pos[svspec::kMaxCols];
  const int tid = threadIdx.x, S = ss->ncols;
  if (tid == 0) {
    if (accept) spec_session_accept(ss, sel, rows, p, seen, vocab, next_ids, out_ids);
    int live = 0;
    for (int r = 0; r < S; ++r) {
      s_w[r] = 0;
      const bool on = rows->row_active[r] != 0;
      live += on;
      s_n[r] = rows->row_step[r];
      s_room[r] = on ? rows->row_max_new[r] - rows->row_step[r] - 1 : 0;
    }
    s_spare = spec_session_budget(rows, S, tcap) - live;
  }
  __syncthreads();
  const int k = ss->k, g = ss->max_ngram;
  if (s_spare > 0) {             // a fully loaded session skips the search
    for (int r = 0; r < S; ++r) {
      const int n = s_n[r];
      if (s_room[r] < 1 || n < 2) continue;
      const int32_t* hist = out_ids + (int64_t)r * p->out_stride;
      if (tid == 0) { s_best = 0; s_at = 0x7fffffff; }
      __syncthreads();
      for (int e = 1 + tid; e < n; e += 1024) {
        const int l = svspec::suffix_match(hist, n, e, g);
        if (l > 0) atomicMax(&s_best, l);
      }
      __syncthreads();
      const int best = s_best;
      if (best > 0) {
        for (int e = best + tid; e < n; e += 1024)
          if (svspec::suffix_match(hist, n, e, g) >= best) atomicMin(&s_at, e);
      }
      __syncthreads();
      if (tid == 0 && best > 0) s_w[r] = svspec::draft_at(hist, n, s_at, k, p->eos_id, s_room[r], s_d[r]);
      __syncthreads();
    }
  }
  if (tid == 0) {
    spec_session_plan(ss, rows, out_ids, p->out_stride, s_w, s_d, tcap);
    for (int c = 0; c < S; ++c) { s_col_tok[c] = ss->tok[c]; s_col_pos[c] = ss->map.pos[c]; }
  }
  __syncthreads();
  // every column's input: wte[token] + wpe[position] (bf16 add), as select_fused_body embeds the plain step's token
  const int hv = h >> 3;
  for (int i = tid; i < S * hv; i += 1024) {
    const int b = i / hv, c = (i % hv) * 8;
    const int pos = min(s_col_pos[b], n_positions - 1);
    int id = s_col_tok[b];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    float e[8], q[8];
    unpack8(ldg_cached(wte + (int64_t)id * h + c), e);
    if (wpe) {
      unpack8(ldg_cached(wpe + (int64_t)pos * h + c), q);
#pragma unroll
      for (int j = 0; j < 8; ++j) e[j] += q[j];
    }
    *reinterpret_cast<uint4*>(x + (int64_t)b * h + c) = pack8(e);
  }
}

}  // namespace

// Greedy session verify step: select_fused_body's selection per live column (the lm_head's argmax partials at column c
// without a repetition penalty; otherwise the logits row scanned with the column's row's seen set plus its drafts), then
// spec_session_tail.  Argmax with the lowest-index tie-break is exact, so the reduction order does not enter the result.
__global__ void __launch_bounds__(1024) spec_session_select_fused_kernel(
    const bf16* __restrict__ logits, int vocab, const float* __restrict__ amax_val, const int* __restrict__ amax_idx,
    int ntiles, int amax_stride, RowState* rows, const GenParamsDev* __restrict__ p, uint8_t* seen, int32_t* next_ids,
    int32_t* out_ids, const bf16* __restrict__ wte, const bf16* __restrict__ wpe, bf16* __restrict__ x, int h,
    int n_positions, int tcap, svspec::SessionState* ss) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ AmaxPair sm[32];
  __shared__ int s_cols[svspec::kMaxCols], s_sel[svspec::kMaxCols];
  const int tid = threadIdx.x;
  const float rp = p->rep_penalty;
  const bool use_partials = (rp == 1.0f) && amax_val != nullptr;
  if (tid < svspec::kMaxCols) s_cols[tid] = ss->tok[tid];
  __syncthreads();
  const int n_live = ss->map.n_live;
  for (int b = 0; b < n_live; ++b) {
    AmaxPair best{-INFINITY, 0x7fffffff};
    if (use_partials) {
      for (int i = tid; i < ntiles; i += 1024) {
        const float v = __ldcg(amax_val + (int64_t)i * amax_stride + b);
        const int id = __ldcg(amax_idx + (int64_t)i * amax_stride + b);
        best = amax_better(best, AmaxPair{v, id});
      }
    } else {
      const int nd = ss->off[b];
      const bf16* lr = logits + (int64_t)b * vocab;
      const uint8_t* sr = seen + (int64_t)ss->map.row[b] * vocab;
      for (int i = tid; i < vocab; i += 1024) {
        float v = __bfloat162float(__ldcg(lr + i));
        if (sr[i] || svspec::drafted(s_cols + b - nd, nd, i)) v = v < 0.f ? v * rp : v / rp;
        best = amax_better(best, AmaxPair{v, i});
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      AmaxPair other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
      best = amax_better(best, other);
    }
    __syncthreads();
    if ((tid & 31) == 0) sm[tid >> 5] = best;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 32; ++w) best = amax_better(best, sm[w]);
      s_sel[b] = best.i == 0x7fffffff ? 0 : best.i;
    }
  }
  __syncthreads();
  spec_session_tail(s_sel, true, ss, rows, p, seen, next_ids, out_ids, vocab, wte, wpe, x, h, n_positions, tcap);
}

// Sampled session verify step: select_sample_body per live column (block c = column c), tokens to ss->sel.
__global__ void __launch_bounds__(kSampleThreads) spec_session_select_sample_kernel(
    const bf16* __restrict__ logits, int vocab, RowState* rows, const GenParamsDev* __restrict__ p, uint8_t* seen,
    float* __restrict__ probs, svspec::SessionState* ss) {
  select_sample_body<false, false, true>(logits, vocab, nullptr, p, seen, nullptr, nullptr, probs, rows, 0u, 0, nullptr, ss);
}

// The tail after spec_session_select_sample_kernel (accept = 1, tokens in ss->sel), and the re-plan after an admission
// (accept = 0: the admitted rows' first tokens were selected by the plain session kernels).
__global__ void __launch_bounds__(1024) spec_session_tail_kernel(int accept, RowState* rows, const GenParamsDev* __restrict__ p,
                                                                 uint8_t* seen, int32_t* next_ids, int32_t* out_ids, int vocab,
                                                                 const bf16* __restrict__ wte, const bf16* __restrict__ wpe,
                                                                 bf16* __restrict__ x, int h, int n_positions, int tcap,
                                                                 svspec::SessionState* ss) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ int32_t s_sel[svspec::kMaxCols];
  if (threadIdx.x < svspec::kMaxCols) s_sel[threadIdx.x] = ss->sel[threadIdx.x];
  __syncthreads();
  spec_session_tail(s_sel, accept != 0, ss, rows, p, seen, next_ids, out_ids, vocab, wte, wpe, x, h, n_positions, tcap);
}

void launch_spec_session_select_fused(const bf16* logits, int vocab, const float* amax_val, const int* amax_idx, int ntiles,
                                      int amax_stride, RowState* rows, const GenParamsDev* params, uint8_t* seen,
                                      int32_t* next_ids, int32_t* out_ids, const bf16* wte, const bf16* wpe, bf16* x, int h,
                                      int n_positions, int tcap, svspec::SessionState* ss, bool pdl, cudaStream_t st) {
  launch_ex(spec_session_select_fused_kernel, dim3(1), dim3(1024), st, pdl, logits, vocab, amax_val, amax_idx, ntiles,
            amax_stride, rows, params, seen, next_ids, out_ids, wte, wpe, x, h, n_positions, tcap, ss);
}
void launch_spec_session_select_sample(const bf16* logits, int vocab, int ncols, RowState* rows, const GenParamsDev* params,
                                       uint8_t* seen, float* probs, svspec::SessionState* ss, cudaStream_t st) {
  spec_session_select_sample_kernel<<<ncols, kSampleThreads, 0, st>>>(logits, vocab, rows, params, seen, probs, ss);
  count_launch();
}
void launch_spec_session_tail(bool accept, RowState* rows, const GenParamsDev* params, uint8_t* seen, int32_t* next_ids,
                              int32_t* out_ids, int vocab, const bf16* wte, const bf16* wpe, bf16* x, int h, int n_positions,
                              int tcap, svspec::SessionState* ss, bool pdl, cudaStream_t st) {
  launch_ex(spec_session_tail_kernel, dim3(1), dim3(1024), st, pdl, accept ? 1 : 0, rows, params, seen, next_ids, out_ids,
            vocab, wte, wpe, x, h, n_positions, tcap, ss);
}

}  // namespace sv

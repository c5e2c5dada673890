// Token selection fused with the next decode step's input (used by the CUDA-graph decode path): one single-CTA kernel finishes
// the greedy argmax from the lm_head kernel's per-tile partials (or scans the penalised logits), applies the HF stop / EOS
// bookkeeping (sv_select.cuh) and writes the next token's embedding.  Programmatic-dependent-launch ready: everything the
// previous kernel produced is read after `griddepcontrol.wait` with L2-only loads.
#include "sv_kernels.h"
#include "sv_select.cuh"

namespace sv {

SV_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
SV_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
SV_DEVINL uint4 ldcg16(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }

template <typename... KArgs, typename... Args>
static void launch_ex(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                      Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, args...);
  count_launch();
}

// ------------------------------------------------------------------------------------------
// What follows the selection of a verify step, in one 1024-thread CTA: the accept walk over the live columns' tokens `sel`
// (the plain path's bookkeeping per emitted token), the next drafts (svspec::draft_host's rule, its two searches spread
// over the CTA), the next column map, and the embeddings wte[tok] + wpe[pos] of every column of the next step.
SV_DEVINL void spec_tail(const int* sel, svspec::State* sp, GenState* state, const GenParamsDev* __restrict__ p,
                         uint8_t* seen, int32_t* next_ids, int32_t* out_ids, int vocab, const bf16* __restrict__ wte,
                         const bf16* __restrict__ wpe, bf16* __restrict__ x, int h, int n_positions) {
  __shared__ int s_best, s_at;
  __shared__ int s_col_tok[svspec::kMaxCols], s_col_pos[svspec::kMaxCols];
  const int tid = threadIdx.x;
  if (tid == 0) {
    const int n_live = sp->map.n_live;
    if (n_live > 0) {
      const int m = svspec::accept(sel, sp->tok, n_live, [&](int t) {
        int tk[1] = {t};
        select_apply_tokens(tk, 1, vocab, state, p, seen, next_ids, out_ids, /*advance_len=*/1);
        return state->done != 0;
      });
      sp->steps += 1; sp->drafted += n_live - 1; sp->accepted += m - 1;
    }
    s_best = 0; s_at = 0x7fffffff;
  }
  __syncthreads();
  const int n = state->step, g = sp->max_ngram;
  const bool done = state->done != 0;
  if (!done) {
    for (int e = 1 + tid; e < n; e += 1024) {
      const int l = svspec::suffix_match(out_ids, n, e, g);
      if (l > 0) atomicMax(&s_best, l);
    }
  }
  __syncthreads();
  const int best = s_best;
  if (!done && best > 0) {
    for (int e = best + tid; e < n; e += 1024)
      if (svspec::suffix_match(out_ids, n, e, g) >= best) atomicMin(&s_at, e);
  }
  __syncthreads();
  const int ncols = sp->ncols;
  if (tid == 0) {
    int nd = 0;
    if (!done && best > 0) nd = svspec::draft_at(out_ids, n, s_at, sp->k, p->eos_id, p->max_new - n - 1, sp->tok + 1);
    sp->tok[0] = out_ids[n - 1];
    for (int c = 1 + nd; c < ncols; ++c) sp->tok[c] = sp->tok[0];    // inert columns: any valid id
    svspec::set_map(sp->map, ncols, done ? 0 : 1 + nd, state->cur_len);
    for (int c = 0; c < ncols; ++c) { s_col_tok[c] = sp->tok[c]; s_col_pos[c] = sp->map.pos[c]; }
  }
  __syncthreads();
  // every column's input: wte[token] + wpe[position] (bf16 add), as select_fused_body embeds the plain step's token
  const int hv = h >> 3;
  for (int i = tid; i < ncols * hv; i += 1024) {
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

// ------------------------------------------------------------------------------------------
// Token selection + HF stop bookkeeping + next-token embedding in ONE single-CTA kernel.
// Greedy without a repetition penalty reduces the lm_head's per-tile argmax partials; otherwise the
// full bf16 logits row is scanned (penalty changes the order).  Semantics: SURVEY.md App. B.3-6.
// ROWS (the session variant): rows that do not select this step (session_row_selects) are skipped, each selecting row
// keeps its own bookkeeping (session_append_token) and is embedded at its own position.
// SPEC (the verify step of sv_generate_speculative): image row b is column b of one cache row; only the live columns
// select, column b's repetition-penalty set is the row's plus drafts 1..b, and spec_tail accepts, drafts and embeds.
template <bool ROWS, bool SPEC = false>
SV_DEVINL void select_fused_body(const bf16* __restrict__ logits, int vocab, int batch, const float* __restrict__ amax_val,
                                 const int* __restrict__ amax_idx, int ntiles, int amax_stride, GenState* state,
                                 const GenParamsDev* __restrict__ p, uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                                 int advance_len, const bf16* __restrict__ wte, const bf16* __restrict__ wpe,
                                 bf16* __restrict__ x, int h, int n_positions, RowState* rows, uint32_t row_mask,
                                 svspec::State* sp = nullptr) {
  pdl_launch_dependents();
  pdl_wait();
  if constexpr (!ROWS) {
    if (state->done) return;
  }
  __shared__ AmaxPair sm[32];
  __shared__ int s_tok[16];
  __shared__ int s_sel[16];
  const int tid = threadIdx.x;
  const float rp = p->rep_penalty;
  const bool use_partials = (rp == 1.0f) && amax_val != nullptr;
  if constexpr (ROWS) {
    if (tid < batch) s_sel[tid] = session_row_selects(rows, row_mask, tid) ? 1 : 0;
    __syncthreads();
  }
  if constexpr (SPEC) {
    batch = sp->map.n_live;
    if (tid < svspec::kMaxCols) s_sel[tid] = sp->tok[tid];        // the column inputs: drafts are s_sel[1..]
    __syncthreads();
  }
  for (int b = 0; b < batch; ++b) {
    if constexpr (ROWS) {
      if (!s_sel[b]) continue;
    }
    AmaxPair best{-INFINITY, 0x7fffffff};
    if (use_partials) {
      for (int i = tid; i < ntiles; i += 1024) {
        const float v = __ldcg(amax_val + (int64_t)i * amax_stride + b);
        const int id = __ldcg(amax_idx + (int64_t)i * amax_stride + b);
        best = amax_better(best, AmaxPair{v, id});
      }
    } else {
      const bf16* lr = logits + (int64_t)b * vocab;
      const uint8_t* sr = seen + (int64_t)(SPEC ? 0 : b) * vocab;
      for (int i = tid; i < vocab; i += 1024) {
        float v = __bfloat162float(__ldcg(lr + i));
        if (sr[i] || (SPEC && svspec::drafted(s_sel, b, i))) v = v < 0.f ? v * rp : v / rp;
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
      s_tok[b] = best.i == 0x7fffffff ? 0 : best.i;
    }
  }
  __syncthreads();
  if constexpr (SPEC) {
    spec_tail(s_tok, sp, state, p, seen, next_ids, out_ids, vocab, wte, wpe, x, h, n_positions);
    return;
  }
  if constexpr (ROWS) {
    if (tid < batch && s_sel[tid])
      session_append_token(tid, s_tok[tid], rows, p, seen, vocab, next_ids, out_ids, advance_len);
  } else {
    if (tid == 0) select_apply_tokens(s_tok, batch, vocab, state, p, seen, next_ids, out_ids, advance_len);
  }
  __syncthreads();
  // --- next step's input: wte[token] + wpe[position] (bf16 add), GPTBigCodeModel.forward
  int pos = ROWS ? 0 : state->cur_len;
  pos = pos >= n_positions ? n_positions - 1 : pos;
  const int hv = h >> 3;
  for (int i = tid; i < batch * hv; i += 1024) {
    const int b = i / hv, c = (i % hv) * 8;
    if constexpr (ROWS) {
      if (!s_sel[b]) continue;
      pos = min(rows->row_len[b], n_positions - 1);
    }
    int id = s_tok[b];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    float e[8], q[8];
    unpack8(ldg_cached(wte + (int64_t)id * h + c), e);
    if (wpe) {                                                  // RoPE models have no learned position table
      unpack8(ldg_cached(wpe + (int64_t)pos * h + c), q);
#pragma unroll
      for (int j = 0; j < 8; ++j) e[j] += q[j];
    }
    *reinterpret_cast<uint4*>(x + (int64_t)b * h + c) = pack8(e);
  }
}
__global__ void __launch_bounds__(1024) select_fused_kernel(const bf16* __restrict__ logits, int vocab, int batch,
                                                            const float* __restrict__ amax_val,
                                                            const int* __restrict__ amax_idx, int ntiles, int amax_stride,
                                                            GenState* state, const GenParamsDev* __restrict__ p,
                                                            uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                                                            int advance_len, const bf16* __restrict__ wte,
                                                            const bf16* __restrict__ wpe, bf16* __restrict__ x, int h,
                                                            int n_positions) {
  select_fused_body<false>(logits, vocab, batch, amax_val, amax_idx, ntiles, amax_stride, state, p, seen, next_ids, out_ids,
                           advance_len, wte, wpe, x, h, n_positions, nullptr, 0u);
}
__global__ void __launch_bounds__(1024) select_fused_rows_kernel(const bf16* __restrict__ logits, int vocab, int batch,
                                                                 const float* __restrict__ amax_val,
                                                                 const int* __restrict__ amax_idx, int ntiles,
                                                                 int amax_stride, RowState* rows, uint32_t row_mask,
                                                                 const GenParamsDev* __restrict__ p, uint8_t* seen,
                                                                 int32_t* next_ids, int32_t* out_ids, int advance_len,
                                                                 const bf16* __restrict__ wte,
                                                                 const bf16* __restrict__ wpe, bf16* __restrict__ x,
                                                                 int h, int n_positions) {
  select_fused_body<true>(logits, vocab, batch, amax_val, amax_idx, ntiles, amax_stride, nullptr, p, seen, next_ids, out_ids,
                          advance_len, wte, wpe, x, h, n_positions, rows, row_mask);
}

// Greedy verify step: per-column selection exactly as select_fused_kernel, then spec_tail.
__global__ void __launch_bounds__(1024) select_fused_spec_kernel(const bf16* __restrict__ logits, int vocab,
                                                                 const float* __restrict__ amax_val,
                                                                 const int* __restrict__ amax_idx, int ntiles,
                                                                 int amax_stride, GenState* state,
                                                                 const GenParamsDev* __restrict__ p, uint8_t* seen,
                                                                 int32_t* next_ids, int32_t* out_ids,
                                                                 const bf16* __restrict__ wte,
                                                                 const bf16* __restrict__ wpe, bf16* __restrict__ x,
                                                                 int h, int n_positions, svspec::State* sp) {
  select_fused_body<false, true>(logits, vocab, 0, amax_val, amax_idx, ntiles, amax_stride, state, p, seen, next_ids,
                                 out_ids, 1, wte, wpe, x, h, n_positions, nullptr, 0u, sp);
}
// Sampled verify step (after select_sample_kernel's SPEC variant wrote sp->sel) and the first drafts of a generation
// (n_live = 0: nothing to accept).
__global__ void __launch_bounds__(1024) spec_accept_kernel(GenState* state, const GenParamsDev* __restrict__ p,
                                                           uint8_t* seen, int32_t* next_ids, int32_t* out_ids, int vocab,
                                                           const bf16* __restrict__ wte, const bf16* __restrict__ wpe,
                                                           bf16* __restrict__ x, int h, int n_positions,
                                                           svspec::State* sp) {
  pdl_launch_dependents();
  pdl_wait();
  if (state->done) return;
  __shared__ int s_sel[svspec::kMaxCols];
  if (threadIdx.x < svspec::kMaxCols) s_sel[threadIdx.x] = sp->sel[threadIdx.x];
  __syncthreads();
  spec_tail(s_sel, sp, state, p, seen, next_ids, out_ids, vocab, wte, wpe, x, h, n_positions);
}

void launch_select_fused_spec(const bf16* logits, int vocab, const float* amax_val, const int* amax_idx, int ntiles,
                              int amax_stride, GenState* state, const GenParamsDev* params, uint8_t* seen,
                              int32_t* next_ids, int32_t* out_ids, const bf16* wte, const bf16* wpe, bf16* x, int h,
                              int n_positions, svspec::State* sp, bool pdl, cudaStream_t st) {
  launch_ex(select_fused_spec_kernel, dim3(1), dim3(1024), 0, st, pdl, logits, vocab, amax_val, amax_idx, ntiles,
            amax_stride, state, params, seen, next_ids, out_ids, wte, wpe, x, h, n_positions, sp);
}
void launch_spec_accept(GenState* state, const GenParamsDev* params, uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                        int vocab, const bf16* wte, const bf16* wpe, bf16* x, int h, int n_positions, svspec::State* sp,
                        bool pdl, cudaStream_t st) {
  launch_ex(spec_accept_kernel, dim3(1), dim3(1024), 0, st, pdl, state, params, seen, next_ids, out_ids, vocab, wte, wpe,
            x, h, n_positions, sp);
}

void launch_select_fused(const bf16* logits, int vocab, int batch, const float* amax_val, const int* amax_idx,
                         int ntiles, int amax_stride, GenState* state, const GenParamsDev* params, uint8_t* seen, int32_t* next_ids,
                         int32_t* out_ids, int advance_len, const bf16* wte, const bf16* wpe, bf16* x, int h,
                         int n_positions, bool pdl, cudaStream_t st, RowState* rows, uint32_t row_mask) {
  if (rows)
    launch_ex(select_fused_rows_kernel, dim3(1), dim3(1024), 0, st, pdl, logits, vocab, batch, amax_val, amax_idx, ntiles,
              amax_stride, rows, row_mask, params, seen, next_ids, out_ids, advance_len, wte, wpe, x, h, n_positions);
  else
    launch_ex(select_fused_kernel, dim3(1), dim3(1024), 0, st, pdl, logits, vocab, batch, amax_val, amax_idx, ntiles,
              amax_stride, state, params, seen, next_ids, out_ids, advance_len, wte, wpe, x, h, n_positions);
}

}  // namespace sv

// Teacher-forced scoring (sv_score_tokens): the small kernels around the fused lm_head log-likelihood of
// sv_gemm_wgmma.cu.  Numerics (DESIGN.md §3): the logits are bf16 (HF's lm_head output); the log-softmax runs in fp32
// over those bf16 values, as CrossEntropyLoss(logits.float()) does.  A row's softmax is split into 128-column tiles,
// each tile contributes (max, sum of exp(logit - max)) and the merge combines them:
//   logprob = logit[target] - (M + log sum_tiles s_tile * exp(m_tile - M)),  M = max over tiles of m_tile.
#include "sv_kernels.h"

namespace sv {

__global__ void score_targets_kernel(const int32_t* __restrict__ ids, int n, int c0, int C, int vocab,
                                     int32_t* __restrict__ tgt) {
  const int b = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= C) return;
  const int j = c0 + t + 1;
  int id = j < n ? ids[(int64_t)b * n + j] : 0;
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);              // the clamp the embedding kernels apply
  tgt[(int64_t)b * C + t] = id;
}
void launch_score_targets(const int32_t* ids, int n, int c0, int batch, int C, int vocab, int32_t* tgt, cudaStream_t st) {
  score_targets_kernel<<<dim3((C + 127) / 128, batch), 128, 0, st>>>(ids, n, c0, C, vocab, tgt);
  count_launch();
}

// one CTA per (128-column tile, row) of resident bf16 logits: the same partials as the wgmma epilogue
__global__ void __launch_bounds__(128) logits_logprob_partials_kernel(const bf16* __restrict__ logits, int vocab,
                                                                      const int32_t* __restrict__ targets,
                                                                      float2* __restrict__ part,
                                                                      float* __restrict__ tgt_logit) {
  __shared__ float red[4];
  const int tile = blockIdx.x, row = blockIdx.y, col = tile * 128 + threadIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float v = col < vocab ? __bfloat162float(logits[(int64_t)row * vocab + col]) : -INFINITY;
  if (col < vocab && col == targets[row]) tgt_logit[row] = v;      // the padded tail of the last tile is no target
  float m = warp_max(v);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float s = warp_sum(expf(v - m));
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) part[(int64_t)row * gridDim.x + tile] = make_float2(m, (red[0] + red[1]) + (red[2] + red[3]));
}
void launch_logits_logprob_partials(const bf16* logits, int vocab, int batch, const int32_t* targets, float2* part,
                                    float* tgt_logit, cudaStream_t st) {
  logits_logprob_partials_kernel<<<dim3(lm_logprob_ntiles(vocab), batch), 128, 0, st>>>(logits, vocab, targets, part, tgt_logit);
  count_launch();
}

// one warp per row; tiles merged in a fixed order per lane, then a fixed shuffle tree (deterministic)
__global__ void __launch_bounds__(256) logprob_merge_kernel(const float2* __restrict__ part, int ntiles,
                                                            const float* __restrict__ tgt_logit, int rows, int C, int off,
                                                            int n, float* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int b = row / C, t = row % C;
  if (off + t >= n) return;
  const float2* p = part + (int64_t)row * ntiles;
  float m = -INFINITY;
  for (int i = lane; i < ntiles; i += 32) m = fmaxf(m, p[i].x);
  m = warp_max(m);
  float s = 0.f;
  for (int i = lane; i < ntiles; i += 32) s += p[i].y * expf(p[i].x - m);
  s = warp_sum(s);
  if (lane == 0) out[(int64_t)b * n + off + t] = tgt_logit[row] - (m + logf(s));
}
void launch_logprob_merge(const float2* part, int ntiles, const float* tgt_logit, int rows, int C, int off, int n,
                          float* out, cudaStream_t st) {
  logprob_merge_kernel<<<(rows + 7) / 8, 256, 0, st>>>(part, ntiles, tgt_logit, rows, C, off, n, out);
  count_launch();
}

}  // namespace sv

// Small-M linear layer: y[M,N] = epilogue(x[M,K] . w[N,K]^T + bias).  This is the decode-time
// "GEMV" (M = images on this GPU <= 8): purely weight-streaming, so it is built for HBM, not FLOPs:
//   * one CTA owns 16 output features (16 weight rows) and all of K; its 8 warps take interleaved
//     32-element K chunks, so the CTA's loads sweep 16 contiguous row segments;
//   * every lane issues 128-bit loads straight from the row-major [N,K] weight (no repacking): the
//     dot product is invariant under a permutation of k applied to both operands, so lane (g,t)
//     feeds the 8 contiguous elements k0+8t..k0+8t+7 of rows g / g+8 to TWO m16n8k16 MMAs as their
//     (k=2t,2t+1 | 2t+8,2t+9) slots, and loads the same 8 elements of activation row g as B;
//   * weights are the MMA "A" operand (M=16 features), the <=8 activation rows are "B" (N=8), so
//     one legacy-path tensor-core instruction covers 16x8x16 MACs and the SM stays load-bound;
//   * split-K partials are reduced across the 8 warps in shared memory in a fixed order
//     (deterministic), then the reference's bf16 rounding points are applied (sv_common.cuh).
// For M > 8 the CTA loops over 8-row groups (weights then come from L2): a correctness fallback
// for shapes the wgmma GEMM does not take, never the fast path for large M.
#include "sv_kernels.h"

namespace sv {

constexpr int kRgWarps = 8;
constexpr int kRgGroupsPerCta = 4;

__global__ void __launch_bounds__(kRgWarps * 32) linear_rowgroup_kernel(
    const bf16* __restrict__ X, const bf16* __restrict__ W, const bf16* __restrict__ bias,
    const bf16* __restrict__ res, bf16* __restrict__ Y, int M, int N, int K, int act) {
  __shared__ float red[kRgWarps][16][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.x * 16;
  const int r0 = min(n0 + g, N - 1), r1 = min(n0 + g + 8, N - 1);
  const bf16* w0 = W + (int64_t)r0 * K + 8 * t;
  const bf16* w1 = W + (int64_t)r1 * K + 8 * t;
  const int nchunks = K >> 5;
  const bool stream_w = (M <= 8);

  for (int grp = 0; grp < kRgGroupsPerCta; ++grp) {
    const int m0 = (blockIdx.y * kRgGroupsPerCta + grp) * 8;
    if (m0 >= M) break;
    const int m = m0 + g;
    const bool mvalid = m < M;
    const bf16* xp = X + (int64_t)(mvalid ? m : M - 1) * K + 8 * t;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
    for (int ch = warp; ch < nchunks; ch += kRgWarps) {
      uint4 a, b;
      if (stream_w) { a = ldg_stream(w0 + ch * 32); b = ldg_stream(w1 + ch * 32); }
      else          { a = ldg_cached(w0 + ch * 32); b = ldg_cached(w1 + ch * 32); }
      uint4 xv = make_uint4(0u, 0u, 0u, 0u);
      if (mvalid) xv = ldg_cached(xp + ch * 32);
      mma_bf16_16816(c, a.x, b.x, a.y, b.y, xv.x, xv.y);
      mma_bf16_16816(c, a.z, b.z, a.w, b.w, xv.z, xv.w);
    }
    // c0,c1: (feature g, rows 2t,2t+1)   c2,c3: (feature g+8, rows 2t,2t+1)
    red[warp][g][2 * t] = c[0];
    red[warp][g][2 * t + 1] = c[1];
    red[warp][g + 8][2 * t] = c[2];
    red[warp][g + 8][2 * t + 1] = c[3];
    __syncthreads();
    if (threadIdx.x < 128) {
      const int n = threadIdx.x & 15, mm = threadIdx.x >> 4;
      float acc = 0.f;
#pragma unroll
      for (int w = 0; w < kRgWarps; ++w) acc += red[w][n][mm];
      const int row = m0 + mm, col = n0 + n;
      if (row < M && col < N) {
        const float bv = bias ? __bfloat162float(bias[col]) : 0.f;
        const float rv = res ? __bfloat162float(res[(int64_t)row * N + col]) : 0.f;
        Y[(int64_t)row * N + col] = __float2bfloat16_rn(epilogue_elem(acc, bv, act, res != nullptr, rv));
      }
    }
    __syncthreads();
  }
}

void launch_linear_rowgroup(const bf16* x, const bf16* w, const bf16* bias, const bf16* res, bf16* y, int M, int N,
                            int K, int act, cudaStream_t st) {
  if (M <= 0 || N <= 0) return;
  dim3 grid((N + 15) / 16, (M + 8 * kRgGroupsPerCta - 1) / (8 * kRgGroupsPerCta));
  linear_rowgroup_kernel<<<grid, kRgWarps * 32, 0, st>>>(x, w, bias, res, y, M, N, K, act);
  count_launch();
}

}  // namespace sv

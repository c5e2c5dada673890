// Shared device helpers for the starvector_b200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "starvector_b200 kernels are written for sm_90a (H100) only"
#endif

typedef __nv_bfloat16 bf16;

#define SV_DEVINL __device__ __forceinline__

// ---- bf16 <-> fp32 (round-to-nearest-even, the rounding every reference module boundary applies)
SV_DEVINL float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
SV_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
SV_DEVINL float2 unpack_bf16x2(uint32_t w) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&w);
  return __bfloat1622float2(v);
}
SV_DEVINL void unpack8(const uint4& v, float (&f)[8]) {
  float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
SV_DEVINL uint4 pack8(const float (&f)[8]) {
  uint4 v;
  v.x = pack_bf16x2(f[0], f[1]); v.y = pack_bf16x2(f[2], f[3]);
  v.z = pack_bf16x2(f[4], f[5]); v.w = pack_bf16x2(f[6], f[7]);
  return v;
}

// ---- 128-bit global loads
// Streaming (read-once weights): bypass L1 allocation.
SV_DEVINL uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// Re-used data (activations, K/V re-read by neighbouring warps): default caching, read-only path.
SV_DEVINL uint4 ldg_cached(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// ---- warp reductions
SV_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SV_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
SV_DEVINL float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}
SV_DEVINL float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  return v;
}

// ---- legacy-path tensor core MMA (bandwidth-bound small-M work only; big GEMMs use wgmma)
// D[16x8] += A[16x16] * B[16x8], bf16 in, fp32 accumulate.  Fragment layout (PTX ISA, g = lane>>2,
// t = lane&3):  a0:(g, 2t..) a1:(g+8, 2t..) a2:(g, 2t+8..) a3:(g+8, 2t+8..);  b0:(k=2t.., n=g)
// b1:(k=2t+8.., n=g);  c0,c1:(g, 2t..2t+1)  c2,c3:(g+8, 2t..2t+1).
SV_DEVINL void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                              uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// ---- activations with the reference's bf16 rounding points (DESIGN.md "numerics")
// Input v is the already bf16-rounded Linear output; the result is NOT yet rounded.
SV_DEVINL float act_quickgelu(float v) {          // x * sigmoid(1.702 * x): three bf16 tensor ops
  float t = bf16_round(1.702f * v);               // 1.702 * x            -> bf16
  float s = bf16_round(1.0f / (1.0f + __expf(-t)));  // torch.sigmoid(...) -> bf16
  return v * s;                                   // x * (...)            -> rounded by caller
}
SV_DEVINL float act_silu(float v) {               // x * sigmoid(x)
  float s = bf16_round(1.0f / (1.0f + __expf(-v)));
  return v * s;
}
SV_DEVINL float act_gelu_tanh(float v) {          // nn.GELU(approximate="tanh"): one fused op in fp32
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (v + k1 * v * v * v);
  return 0.5f * v * (1.0f + tanhf(u));
}
SV_DEVINL float apply_act(int act, float v) {
  switch (act) {
    case 1: return act_quickgelu(v);
    case 2: return act_gelu_tanh(v);
    case 3: return act_silu(v);
    default: return v;
  }
}
// Full epilogue for one element: acc(fp32) + bias -> bf16 -> act -> bf16 -> (+ residual -> bf16).
SV_DEVINL float epilogue_elem(float acc, float bias, int act, bool has_res, float res) {
  float v = bf16_round(acc + bias);
  if (act != 0) v = bf16_round(apply_act(act, v));
  if (has_res) v = bf16_round(v + res);
  return v;
}

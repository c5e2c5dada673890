// Shared device pieces of the weight-ring decode kernels (sv_decode_mega.cu: per-phase ring GEMV + barrier-synchronised
// persistent kernel; sv_decode_flow.cu: dataflow persistent kernel): CTA shape constants, mbarrier / bulk-copy helpers,
// the static tile plan, the producer warp's weight streaming loop and the split-KV attention core.
#pragma once
#include "sv_kernels.h"

namespace sv {
namespace mega {

// Build-time shape of a GEMV CTA.  The shipped library uses the defaults (8 consumer warps, 5 ring slots, one CTA per
// SM).  `python -m starvector_b200.build --variant nwc4` builds a second library (selected at run time with SV_LIB_PATH)
// with 4 consumer warps, 3 slots and TWO CTAs per SM, so that under PDL the next kernel's CTAs are already resident —
// and their producer warps already streaming — while the previous kernel drains (DESIGN.md §7c experiment (c)).
#ifndef SV_NWC
#define SV_NWC 8
#endif
#ifndef SV_STAGES
#define SV_STAGES 5
#endif
#ifndef SV_MINBLOCKS
#define SV_MINBLOCKS 1
#endif
constexpr int NWC = SV_NWC;                          // consumer warps
static_assert(NWC == 8 || NWC == 4, "the 128-thread tile epilogue needs >= 4 consumer warps; chunking assumes 32 % NWC == 0");
constexpr int NCT = NWC * 32;                        // consumer threads
constexpr int NTHREADS = NCT + 32;                   // + producer warp
constexpr int KS_MAX = 1024;                         // k elements per ring slot row
constexpr int CPW = KS_MAX / 32 / NWC;               // 32-wide k chunks per consumer warp and slot (4 with 8 warps)
constexpr int SLOT_BYTES = 16 * (KS_MAX * 2 + 64);   // 16 rows x (2 KB + 64 B pad)
constexpr int STAGES = SV_STAGES;
constexpr int RING_MINBLOCKS = SV_MINBLOCKS;         // gemv_ring_kernel CTAs per SM
constexpr int D = 128;
constexpr int PSZ = 32 + 16 * D;                     // floats per attention partial: m[16] l[16] acc[16][D]
constexpr int ATT_BYTES = 4 * PSZ * 4;               // tree-merge buffer: 4 warp partials
constexpr int RED_BYTES = 2 * NWC * 16 * 8 * 4;
constexpr int OFF_ATT = STAGES * SLOT_BYTES;
constexpr int OFF_RED = OFF_ATT + ATT_BYTES;
constexpr int OFF_STAT = OFF_RED + RED_BYTES;
constexpr int OFF_BAR = OFF_STAT + NWC * 8 * 4;
constexpr int OFF_TOK = OFF_BAR + 2 * STAGES * 8;
constexpr int SMEM_BYTES = OFF_TOK + 64 + 128;       // + alignment slack

SV_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
SV_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
SV_DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
SV_DEVINL void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
SV_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
  for (uint32_t it = 0;; ++it) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
    if (it > (1u << 22)) __trap();
  }
}
SV_DEVINL void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
SV_DEVINL uint4 lds16(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}
SV_DEVINL void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(NCT) : "memory"); }
SV_DEVINL uint4 ldcg16(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }

using Layer = MegaLayer;
struct Args {
  const Layer* layers;
  int n_layer, B, H, I, n_head, n_kv, qkv_cols, vocab, tcap, n_positions;
  float ln_eps;
  const bf16 *wte, *wpe, *lnf_w, *lnf_b, *lm_head;
  bf16 *x, *qkv, *attn, *h, *logits;
  float* attn_partial;
  float* amax_val;
  int* amax_idx;
  GenState* state;
  const GenParamsDev* params;
  uint8_t* seen;
  int32_t *next_ids, *out_ids;
  unsigned int* barrier_ctr;
  int nsteps, att_ncta;
  long long* dbg;      // optional: CTA 0 / thread 0 clock64() stamps around every grid barrier of the first token
};

// ---- static description of one GEMV phase (identical on producer and consumers)
struct Plan {
  int R, tpc, ntiles, tile0, ntile, KS, nstg, pitch;
};
SV_DEVINL Plan make_plan(int N, int K, int cta, int ncta) {
  Plan p;
  const int rows_per_cta = (N + ncta - 1) / ncta;
  p.tpc = (rows_per_cta + 15) / 16;
  p.R = (rows_per_cta + p.tpc - 1) / p.tpc;
  p.ntiles = (N + p.R - 1) / p.R;
  p.tile0 = cta * p.tpc;
  p.ntile = max(0, min(p.tpc, p.ntiles - p.tile0));
  // slab width: the largest of {1024, 768, 512, 256, 128, 64, 32} that divides K (4608 -> 768, 18432 -> 1024)
  p.KS = 32;
  for (int ks : {1024, 768, 512, 256, 128, 64}) if (ks <= K && K % ks == 0) { p.KS = ks; break; }
  p.nstg = K / p.KS;
  p.pitch = p.KS * 2 + 64;
  return p;
}

// make_plan's slab width on the host
inline int slab_width(int K) {
  for (int ks : {1024, 768, 512, 256, 128, 64}) if (ks <= K && K % ks == 0) return ks;
  return 32;
}

struct Ring {
  uint32_t base, full0, empty0;      // shared addresses
  uint32_t slot, phase, nslots;
  SV_DEVINL void advance() { if (++slot == nslots) { slot = 0; phase ^= 1u; } }
};

// ---- producer warp: stream one phase's weight slabs for this CTA.  Lane 0 arms the slot's "full"
// barrier, then lane i issues the bulk copy of row i (16 copies in flight per slot, issued in parallel).
SV_DEVINL void produce_phase(Ring& r, const bf16* W, int N, int K, int cta, int ncta, int lane) {
  const Plan p = make_plan(N, K, cta, ncta);
  for (int tl = 0; tl < p.ntile; ++tl) {
    const int row0 = (p.tile0 + tl) * p.R;
    const int rows = min(p.R, N - row0);
    for (int ks = 0; ks < p.nstg; ++ks) {
      const uint32_t fb = r.full0 + 8u * r.slot;
      if (lane == 0) {
        mbar_wait(r.empty0 + 8u * r.slot, r.phase ^ 1u);
        mbar_expect_tx(fb, (uint32_t)(rows * p.KS * 2));
      }
      __syncwarp();
      if (lane < rows)
        bulk_g2s(r.base + r.slot * SLOT_BYTES + lane * p.pitch, W + (int64_t)(row0 + lane) * K + (int64_t)ks * p.KS,
                 (uint32_t)(p.KS * 2), fb);
      r.advance();
    }
  }
}

// ---- the same on the slab-tiled copy of W (flow_repack_kernel in sv_decode_flow.cu): a slab is SLOT_BYTES-aligned and already
// has the shared-memory row pitch, so ONE bulk copy fills a slot instead of one 2 KB copy per row.  Rows past N are zero in the copy.
SV_DEVINL void produce_phase_tiled(Ring& r, const uint8_t* T, int N, int K, int cta, int ncta, int lane) {
  if (lane != 0) return;
  const Plan p = make_plan(N, K, cta, ncta);
  const uint8_t* src = T + (int64_t)cta * p.tpc * p.nstg * SLOT_BYTES;
  const uint32_t bytes = (uint32_t)(p.R * p.pitch);
  const int nslab = p.ntile * p.nstg;
  for (int i = 0; i < nslab; ++i) {
    const uint32_t fb = r.full0 + 8u * r.slot;
    mbar_wait(r.empty0 + 8u * r.slot, r.phase ^ 1u);
    mbar_expect_tx(fb, bytes);
    bulk_g2s(r.base + r.slot * SLOT_BYTES, src + (int64_t)i * SLOT_BYTES, bytes, fb);
    r.advance();
  }
}

// ---- attention core on L2-only loads (same fragment walk as sv_attention.cu, see the comments there)
SV_DEVINL void attn_block(const uint32_t (&qa)[D / 16][4], const bf16* __restrict__ kbase,
                          const bf16* __restrict__ vtbase, int tcap, int kb, int key_end, float scale_log2,
                          float (&acc)[D / 8][4], float (&mrow)[2], float (&lrow)[2], int g, int t) {
  float s[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
    int key = kb + 8 * (g >> 1) + 2 * j + (g & 1);
    key = key < key_end ? key : key_end - 1;
    const bf16* kp = kbase + (int64_t)key * D + 8 * t;
#pragma unroll
    for (int jj = 0; jj < D / 32; ++jj) {
      const uint4 w = ldcg16(kp + 32 * jj);
      mma_bf16_16816(s[j], qa[2 * jj][0], qa[2 * jj][1], qa[2 * jj][2], qa[2 * jj][3], w.x, w.y);
      mma_bf16_16816(s[j], qa[2 * jj + 1][0], qa[2 * jj + 1][1], qa[2 * jj + 1][2], qa[2 * jj + 1][3], w.z, w.w);
    }
  }
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool valid = (kb + 8 * t + 2 * j + e) < key_end;
      s[j][e] = valid ? s[j][e] * scale_log2 : -INFINITY;
      s[j][2 + e] = valid ? s[j][2 + e] * scale_log2 : -INFINITY;
      mx0 = fmaxf(mx0, s[j][e]);
      mx1 = fmaxf(mx1, s[j][2 + e]);
    }
  }
  mx0 = quad_max(mx0); mx1 = quad_max(mx1);
  const float mn0 = fmaxf(mrow[0], mx0), mn1 = fmaxf(mrow[1], mx1);
  const float corr0 = exp2f(mrow[0] - mn0), corr1 = exp2f(mrow[1] - mn1);
  mrow[0] = mn0; mrow[1] = mn1;
  float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s[j][0] = exp2f(s[j][0] - mn0); s[j][1] = exp2f(s[j][1] - mn0);
    s[j][2] = exp2f(s[j][2] - mn1); s[j][3] = exp2f(s[j][3] - mn1);
    rs0 += s[j][0] + s[j][1]; rs1 += s[j][2] + s[j][3];
  }
  lrow[0] = lrow[0] * corr0 + rs0;
  lrow[1] = lrow[1] * corr1 + rs1;
  uint32_t pa[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    pa[h][0] = pack_bf16x2(s[2 * h][0], s[2 * h][1]);
    pa[h][1] = pack_bf16x2(s[2 * h][2], s[2 * h][3]);
    pa[h][2] = pack_bf16x2(s[2 * h + 1][0], s[2 * h + 1][1]);
    pa[h][3] = pack_bf16x2(s[2 * h + 1][2], s[2 * h + 1][3]);
  }
#pragma unroll
  for (int nd = 0; nd < D / 8; ++nd) {
    acc[nd][0] *= corr0; acc[nd][1] *= corr0; acc[nd][2] *= corr1; acc[nd][3] *= corr1;
    const uint4 w = ldcg16(vtbase + (int64_t)(8 * nd + g) * tcap + kb + 8 * t);
    mma_bf16_16816(acc[nd], pa[0][0], pa[0][1], pa[0][2], pa[0][3], w.x, w.y);
    mma_bf16_16816(acc[nd], pa[1][0], pa[1][1], pa[1][2], pa[1][3], w.z, w.w);
  }
}

// merge another warp's partial (in shared memory, fragment layout) into this warp's registers
SV_DEVINL void attn_merge_from(const float* ws, float (&acc)[D / 8][4], float (&mrow)[2], float (&lq)[2], int g, int t) {
  const float m0 = ws[g], m1 = ws[g + 8];
  const float n0 = fmaxf(mrow[0], m0), n1 = fmaxf(mrow[1], m1);
  const float a0 = (mrow[0] == -INFINITY) ? 0.f : exp2f(mrow[0] - n0), b0 = (m0 == -INFINITY) ? 0.f : exp2f(m0 - n0);
  const float a1 = (mrow[1] == -INFINITY) ? 0.f : exp2f(mrow[1] - n1), b1 = (m1 == -INFINITY) ? 0.f : exp2f(m1 - n1);
  lq[0] = lq[0] * a0 + ws[16 + g] * b0;
  lq[1] = lq[1] * a1 + ws[16 + g + 8] * b1;
  mrow[0] = n0; mrow[1] = n1;
#pragma unroll
  for (int nd = 0; nd < D / 8; ++nd) {
    const float2 lo = *reinterpret_cast<const float2*>(ws + 32 + g * D + 8 * nd + 2 * t);
    const float2 hi = *reinterpret_cast<const float2*>(ws + 32 + (g + 8) * D + 8 * nd + 2 * t);
    acc[nd][0] = acc[nd][0] * a0 + lo.x * b0; acc[nd][1] = acc[nd][1] * a0 + lo.y * b0;
    acc[nd][2] = acc[nd][2] * a1 + hi.x * b1; acc[nd][3] = acc[nd][3] * a1 + hi.y * b1;
  }
}
SV_DEVINL void attn_store_to(float* ws, const float (&acc)[D / 8][4], const float (&mrow)[2], const float (&lq)[2],
                             int g, int t) {
  if (t == 0) { ws[g] = mrow[0]; ws[g + 8] = mrow[1]; ws[16 + g] = lq[0]; ws[16 + g + 8] = lq[1]; }
#pragma unroll
  for (int nd = 0; nd < D / 8; ++nd) {
    *reinterpret_cast<float2*>(ws + 32 + g * D + 8 * nd + 2 * t) = make_float2(acc[nd][0], acc[nd][1]);
    *reinterpret_cast<float2*>(ws + 32 + (g + 8) * D + 8 * nd + 2 * t) = make_float2(acc[nd][2], acc[nd][3]);
  }
}

}  // namespace mega
}  // namespace sv

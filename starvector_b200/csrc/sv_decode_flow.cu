// Dataflow decode kernel: `nsteps` whole tokens (all layers, lm_head, greedy token selection) in ONE cooperative launch,
// one CTA per SM, and NO grid barriers and NO fences on the token's critical path.
//
// The decode step of the reference (GPTBigCodeBlock, starvector/model/gpt_bigcode/modeling_gpt_bigcode.py:670-755; loop:
// HF GenerationMixin._sample, SURVEY.md App. B) is a chain of ~146 small all-to-all dependent phases that streams 2.24 GB
// of weights.  As separate kernels every phase pays a launch boundary (round 1: 122 launches, 1.0 ms/token = 0.34 of the HBM
// roofline); behind grid barriers it pays red.release + polling + membar + re-load (1.4 ms/token).  Here:
//
//   * weights: a producer warp per CTA walks the STATIC weight schedule of the whole launch and keeps a 5-slot shared
//     memory ring full with cp.async.bulk (sv_ring.cuh), never waiting for activations: HBM streams straight through
//     phase boundaries;
//   * activations travel between CTAs as FLAGGED WORDS through L2 (the point of coherence): a 32-bit word holds one bf16
//     value + a 16-bit phase tag (fp32 payloads: 64-bit word, 32-bit tag).  A single aligned 4/8-byte store is
//     single-copy atomic, so the consumer polls the data itself with ld.relaxed.gpu and needs neither a flag, a fence nor a
//     barrier: one phase hop costs one L2 store + one L2 load (~0.3 us) instead of ~2 us.  Tags come from a monotonic
//     phase counter, buffers are cleared when a new sequence starts, so a stale word can never carry the expected tag;
//   * a buffer is only rewritten one full all-to-all phase after its last read (DESIGN.md "flow hazards"), so no
//     double buffering and no back-pressure signalling is needed;
//   * attention: split-KV items of 8 warps x 32 keys spread over CTAs, CTA-local tree merge, partials (m,l,acc) as flagged
//     fp32 words, then a distributed merge (one warp per (image, head, 32 dims)) -- two short hops instead of a
//     cluster barrier; the current token's k/v never round-trip through the cache before they are used: the CTA that owns
//     the last key block takes them from the flagged QKV vector and appends them to the cache itself;
//   * the KV cache of older tokens is read with ld.global.cg one full token after it was written with st.global.cg.
//
// Every wait is bounded and traps instead of hanging the GPU.
#include <cstdio>
#include <cstdlib>

#include "sv_kernels.h"
#include "sv_ring.cuh"
#include "sv_select.cuh"

namespace sv {
namespace flow {

using namespace mega;

constexpr int MAXS = 64;                      // attention key splits per (image, kv head)
constexpr int FLOW_OFF_STAT = OFF_STAT;       // [2][NWC][8] floats: needs 2x the mega layout's room
constexpr int FLOW_OFF_BAR = FLOW_OFF_STAT + 2 * NWC * 8 * 4;
constexpr int FLOW_OFF_TOK = FLOW_OFF_BAR + 2 * STAGES * 8 + 4 * 8;      // + 2 full / 2 empty barriers of the LayerNorm ring
constexpr int LN_MAX_H = 2 * KS_MAX;          // LayerNorm width the parameter ring holds (the flow kernel needs H <= 2048)
constexpr int LN_SLOT_BYTES = 2 * LN_MAX_H * 2;                          // weight row + bias row, bf16
constexpr int FLOW_OFF_PROG = FLOW_OFF_TOK + 48;                         // producer progress counter + "ring full" flag (read by the L2 prefetch warp)
constexpr int FLOW_OFF_STATE = FLOW_OFF_TOK + 64;                        // CTA 0: GenState + GenParamsDev working copies
constexpr int FLOW_OFF_LN = (FLOW_OFF_STATE + (int)sizeof(GenState) + (int)sizeof(GenParamsDev) + 127) & ~127;   // [2][LN_SLOT_BYTES]
// per-layer pointer table and the five tile plans: read on every phase change, so they live in shared memory (as device-memory
// pointer chasing / integer divisions they cost ~1-2K cycles of the token's critical path per phase)
constexpr int FLOW_MAX_LAYERS = 24;
constexpr int FLOW_OFF_LAYERS = FLOW_OFF_LN + 2 * LN_SLOT_BYTES;
constexpr int FLOW_OFF_PLANS = FLOW_OFF_LAYERS + FLOW_MAX_LAYERS * (int)sizeof(Layer);
constexpr int FLOW_SMEM_BYTES = FLOW_OFF_PLANS + 5 * (int)sizeof(Plan) + 128;
static_assert(FLOW_SMEM_BYTES <= 232448, "dataflow decode kernel: shared memory over the 227 KB per-CTA limit");

struct FlowArgs {
  const Layer* layers;
  int n_layer, B, H, I, n_head, n_kv, qkv_cols, vocab, tcap, n_positions;
  float ln_eps;
  const bf16 *wte, *wpe, *lnf_w, *lnf_b, *lm_head;
  const bf16* lm_head_t;         // lm_head in the slab-tiled layout (see flow_repack_kernel)
  bf16* x_plain;                 // [B][H] bf16: input of the first step when first_plain; refreshed by every select
  bf16* logits;                  // [B][vocab] bf16 (plain stores; read by the host path / the penalised scan)
  uint32_t *xa, *xb, *qkv, *att, *hb;          // flagged bf16 words: [B][H], [B][H], [B][qkv_cols], [B][H], [B][I]
  unsigned long long *part, *amax;             // flagged fp32 words [B*n_kv][MAXS][PSZ]; argmax partials [ntiles][8]
  GenState* state;
  const GenParamsDev* params;
  uint8_t* seen;
  int32_t *next_ids, *out_ids;
  int nsteps, step0, cur_len0, first_plain, do_select;
  int l2_ahead;                  // weight slabs the producer asks L2 to fetch ahead of the shared-memory ring (0 = off)
  long long* dbg;                // optional: CTA 0 / thread 0 clock64() stamps of the first step
};

// ---- relaxed gpu-scope accesses (always served by L2)
SV_DEVINL uint4 ld_rlx16(const void* p) {
  uint4 r;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
SV_DEVINL uint32_t ld_rlx32(const void* p) {
  uint32_t r;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
  return r;
}
SV_DEVINL unsigned long long ld_rlx64(const void* p) {
  unsigned long long r;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
  return r;
}
SV_DEVINL void st_rlx32(void* p, uint32_t v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
SV_DEVINL void st_rlx64(void* p, unsigned long long v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
SV_DEVINL void st_rlx16B(void* p, uint4 v) {
  asm volatile("st.relaxed.gpu.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
SV_DEVINL void spin_guard(uint32_t& it) { if (++it > (1u << 26)) __trap(); }

SV_DEVINL Plan plan_of(const uint8_t* smem, int kind) { return reinterpret_cast<const Plan*>(smem + FLOW_OFF_PLANS)[kind]; }

// phase tags
SV_DEVINL uint32_t tag16(uint32_t gp) { return ((gp & 0x7fffu) + 1u) << 16; }   // in the upper half of a bf16 word (a stale word is <= 2 phases old)
SV_DEVINL unsigned long long tag32(uint32_t gp) { return (unsigned long long)(gp + 1u) << 32; }
SV_DEVINL unsigned long long fword(float v, unsigned long long T) { return T | (unsigned long long)__float_as_uint(v); }

// Layout of a flagged bf16 vector [B][n]: the 8 words of one MMA fragment (32 bytes = one L2 sector) are contiguous,
// consecutive fragments are FRAG_STRIDE words (256 bytes) apart.  All CTAs (one per SM) poll the same vector at the same moment:
// packed densely (8 KB for n = 2048) those reads hit a few L2 slices; one fragment per 256-byte chunk (the L2 slice hash works
// on address bits >= 8) spreads them over the whole L2.
constexpr int FRAG_STRIDE = 64;
SV_DEVINL int64_t ll_words(int n) { return (int64_t)(n >> 3) * FRAG_STRIDE; }                       // words per image row
SV_DEVINL int64_t ll_off(int i) { return (int64_t)(i >> 3) * FRAG_STRIDE + (i & 7); }              // word i of a row

// A poll = ISSUE every load first, CHECK afterwards.  (Checking each fragment right behind its own loads made the `asm
// volatile` loads issue one L2 round trip after the other: 8 serialised round trips per poll of a GEMV prologue.)
struct LLRaw { uint4 a, b; };
SV_DEVINL void ll_issue(const uint32_t* p, LLRaw& r) { r.a = ld_rlx16(p); r.b = ld_rlx16(p + 4); }
// 8 consecutive bf16 values out of flagged words; nonzero result = at least one word does not carry tag E yet
SV_DEVINL uint32_t ll_finish(const LLRaw& r, uint32_t E, uint4& out) {
  out.x = __byte_perm(r.a.x, r.a.y, 0x5410); out.y = __byte_perm(r.a.z, r.a.w, 0x5410);
  out.z = __byte_perm(r.b.x, r.b.y, 0x5410); out.w = __byte_perm(r.b.z, r.b.w, 0x5410);
  return ((r.a.x ^ E) | (r.a.y ^ E) | (r.a.z ^ E) | (r.a.w ^ E) | (r.b.x ^ E) | (r.b.y ^ E) | (r.b.z ^ E) | (r.b.w ^ E)) >> 16;
}
SV_DEVINL void ll_put8(uint32_t* p, uint32_t E, const uint4& v) {
  st_rlx16B(p, make_uint4(E | (v.x & 0xffffu), E | (v.x >> 16), E | (v.y & 0xffffu), E | (v.y >> 16)));
  st_rlx16B(p + 4, make_uint4(E | (v.z & 0xffffu), E | (v.z >> 16), E | (v.w & 0xffffu), E | (v.w >> 16)));
}

struct FCtx {
  const FlowArgs* a;
  uint8_t* smem;
  int cta, ncta, warp, lane, g, t;
  float* red;     // [2][NWC][16][8]
  float* stat;    // [2][NWC][8]
  long long* dbg; // nullptr unless this thread records the timeline
  int dbg_i;
  bool slow_select;   // repetition penalty armed: the select phase scans the full logits row
};
// timeline records (SV_MEGA_DEBUG): [id << 48 | clock64], CTA 0 only; consumer thread 0 fills dbg[0..4096), the producer
// warp's lane 0 dbg[4096..8192).  ids: 8 * kind + {1 enter, 2 x ready, 3 LayerNorm done, 4 first weight slab landed, 5 last
// slab consumed, 6 outputs stored} with kind 0 qkv, 1 c_proj, 2 fc, 3 mlp.c_proj, 4 lm_head; 40.. attention; 64 + 2 * kind
// (+1) = producer starts (has issued) the kind's slabs.
enum { ST_ENTER = 1, ST_XREADY = 2, ST_LN = 3, ST_W0 = 4, ST_WLAST = 5, ST_DONE = 6, ST_ATT_ENTER = 40, ST_ATT_Q = 41, ST_ATT_BLK = 42,
       ST_ATT_TREE = 43, ST_ATT_DONE = 44, ST_MERGE_DONE = 46, ST_SELECT_DONE = 47, ST_PROD = 64 };
constexpr int DBG_HALF = 4096;
SV_DEVINL void stamp_raw(long long* dbg, int& i, int id) {
  if (dbg && i < DBG_HALF) dbg[i++] = (long long)(((unsigned long long)id << 48) | ((unsigned long long)clock64() & 0xffffffffffffull));
}
#ifndef SV_FLOW_TIMELINE
#define SV_FLOW_TIMELINE 0        // 1: compile the timeline records in (scripts/flow_timeline.py builds that variant library)
#endif
SV_DEVINL void stamp(FCtx& cx, int id) {
#if SV_FLOW_TIMELINE
  stamp_raw(cx.dbg, cx.dbg_i, id);
#endif
}

enum { EPI_LL = 0, EPI_LMHEAD = 2 };

// LayerNorm parameters ride the producer's schedule too: (weight, bias) rows land in a 2-slot shared-memory mini-ring one or
// two phases before the consumers need them, instead of 16 dependent trips to HBM in the LayerNorm prologue.
struct LnRing {
  uint32_t base, full0, empty0, slot, phase;
  SV_DEVINL void advance() { if (++slot == 2u) { slot = 0; phase ^= 1u; } }
};
SV_DEVINL void produce_ln(LnRing& lr, const bf16* ln_w, const bf16* ln_b, int N, int K, int cta, int ncta, int lane) {
  if (lane == 0) {
    const uint32_t fb = lr.full0 + 8u * lr.slot, dst = lr.base + lr.slot * LN_SLOT_BYTES;
    mbar_wait(lr.empty0 + 8u * lr.slot, lr.phase ^ 1u);
    mbar_expect_tx(fb, (uint32_t)(4 * K));
    bulk_g2s(dst, ln_w, (uint32_t)(2 * K), fb);
    bulk_g2s(dst + LN_MAX_H * 2, ln_b, (uint32_t)(2 * K), fb);
  }
  lr.advance();
}

// ---- consumer: one GEMV phase  Y[B,N] = epi( LN?(X)[B,K] . W[N,K]^T ) on flagged activations.
// X: flagged [B][K] carrying tag EX.  res (optional): flagged [B][N], tag ER.  EPI_LL: Y flagged [B][N], tag EY.
// EPI_LMHEAD: plain bf16 logits + one flagged argmax partial per (tile, image).
// ---- waiting for a flagged vector without flooding L2.  While a CTA waits for a phase's input, 256 threads re-issuing their
// polls back to back put ~1 sector request per clock and CTA on L2 -- with most of the CTAs waiting (e.g. for the one or
// two CTAs that run the attention) that alone saturates L2 and slows exactly the CTAs everybody is waiting for.  So one warp
// watches 32 fragments spread over the vector, sleeping between looks; only when those carry the tag does every thread poll
// its own share (which then mostly succeeds at once).
SV_DEVINL void wait_vector(const FCtx& cx, const uint32_t* __restrict__ V, uint32_t E, int nfrag) {
  if (cx.warp == 0) {
    const uint32_t* p = V + (int64_t)((int)(((long long)cx.lane * nfrag) >> 5)) * FRAG_STRIDE;
    uint32_t it = 0;
    for (;;) {
      LLRaw raw;
      uint4 v;
      ll_issue(p, raw);
      const uint32_t bad = ll_finish(raw, E, v);
      if (!__any_sync(0xffffffffu, bad != 0)) break;
      __nanosleep(100);
      spin_guard(it);
    }
  }
  consumer_sync();
}

// ---- cooperative poll (+ LayerNorm): the consumer threads fetch a flagged [B][n] vector ONCE per CTA into shared memory,
// one fragment (8 values, two 16-byte loads) per thread and pass, all loads in flight together, then spin on the tags.
// With LayerNorm (GPTBigCodeBlock ln_1 / ln_2 / ln_f, vendored modeling_gpt_bigcode.py:700,733; fp32 statistics, bf16 output)
// every thread also normalises the fragments it fetched, so the work is spread over all 256 threads instead of the few
// lanes that feed the MMA B operand at small batch, and nothing but the staged bf16 vector has to stay in registers.
// Statistics are reduced per 32-fragment chunk (one warp, one pass) and summed in chunk order: deterministic.
// Staged rows are xs_pitch(n) bytes apart (+64: the MMA fragment reads of the 8 image rows then hit different banks).
// Ends with the consumer threads synchronised: the staged vector may be read.
SV_DEVINL int xs_pitch(int n) { return n * 2 + 64; }
SV_DEVINL void stage_vector(FCtx& cx, LnRing* lr, const uint32_t* __restrict__ V, uint32_t E, int n, uint8_t* xs, int kind) {
  const FlowArgs& a = *cx.a;
  const int fpr = n >> 3, total = a.B * fpr;           // fragments per row / in all (fpr is a multiple of 32)
  const int tid = threadIdx.x;
  const int fs = 31 - __clz(fpr);                     // fpr is a power of two (n = 256 .. 2048)
  auto slot = [&](int f) { return reinterpret_cast<uint4*>(xs + (f >> fs) * xs_pitch(n) + (f & (fpr - 1)) * 16); };
  wait_vector(cx, V, E, total);
  // (the fragments live in shared memory between the steps below, each thread re-reads only what it wrote itself)
#pragma unroll 1
  for (int f0 = tid; f0 < total; f0 += 4 * NCT) {      // 4 fragments = 8 loads in flight per thread
    // (indices past the end are clamped: their loads are real, only their stores are dropped -- no partially defined arrays,
    // which ptxas would put into local memory, and local memory is an L2 round trip here: 227 KB of the SM are shared memory)
    const int f1 = min(f0 + NCT, total - 1), f2 = min(f0 + 2 * NCT, total - 1), f3 = min(f0 + 3 * NCT, total - 1);
    LLRaw r0, r1, r2, r3;
    uint4 v0, v1, v2, v3;
    uint32_t bad, it = 0;
    do {
      ll_issue(V + (int64_t)f0 * FRAG_STRIDE, r0);       // row b's fragments follow row b - 1's
      ll_issue(V + (int64_t)f1 * FRAG_STRIDE, r1);
      ll_issue(V + (int64_t)f2 * FRAG_STRIDE, r2);
      ll_issue(V + (int64_t)f3 * FRAG_STRIDE, r3);
      bad = ll_finish(r0, E, v0) | ll_finish(r1, E, v1) | ll_finish(r2, E, v2) | ll_finish(r3, E, v3);
      if (bad) { __nanosleep(40); spin_guard(it); }
    } while (bad);
    *slot(f0) = v0;
    if (f0 + NCT < total) *slot(f1) = v1;
    if (f0 + 2 * NCT < total) *slot(f2) = v2;
    if (f0 + 3 * NCT < total) *slot(f3) = v3;
  }
  stamp(cx, 8 * kind + ST_XREADY);
  if (lr != nullptr) {
    float* stat = cx.stat;                              // [2][64]: per-chunk sums, then per-chunk centred squares
    const int cpr = fpr >> 5;                           // 32-fragment chunks per row
#pragma unroll 1
    for (int f = tid; f < total; f += NCT) {            // warp-uniform trip count: total is a multiple of 32
      float fv[8];
      unpack8(*slot(f), fv);
      float sum = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) sum += fv[e];
      sum = warp_sum(sum);
      if (cx.lane == 0) stat[f >> 5] = sum;
    }
    consumer_sync();
#pragma unroll 1
    for (int f = tid; f < total; f += NCT) {
      const int c0 = (f >> fs) * cpr;
      float m = 0.f;
      for (int c = 0; c < cpr; ++c) m += stat[c0 + c];
      const float mean = m / (float)n;
      float fv[8];
      unpack8(*slot(f), fv);
      float q = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float dlt = fv[e] - mean; q += dlt * dlt; }
      q = warp_sum(q);
      if (cx.lane == 0) stat[64 + (f >> 5)] = q;
    }
    consumer_sync();
    mbar_wait(lr->full0 + 8u * lr->slot, lr->phase);    // (weight, bias) rows staged by the producer warp, normally long ago
    const uint32_t lnw = lr->base + lr->slot * LN_SLOT_BYTES, lnb = lnw + LN_MAX_H * 2;
#pragma unroll 1
    for (int f = tid; f < total; f += NCT) {
      const int c0 = (f >> fs) * cpr, fr = f & (fpr - 1);
      float m = 0.f, var = 0.f;
      for (int c = 0; c < cpr; ++c) { m += stat[c0 + c]; var += stat[64 + c0 + c]; }
      const float mean = m / (float)n, rstd = 1.0f / sqrtf(var / (float)n + a.ln_eps);
      float fv[8], wf[8], bfv[8];
      unpack8(*slot(f), fv);
      unpack8(lds16(lnw + fr * 16), wf);
      unpack8(lds16(lnb + fr * 16), bfv);
#pragma unroll
      for (int e = 0; e < 8; ++e) fv[e] = (fv[e] - mean) * rstd * wf[e] + bfv[e];
      *slot(f) = pack8(fv);                              // the LayerNorm output is a bf16 tensor in the reference
    }
    __syncwarp();
    if (cx.lane == 0) mbar_arrive(lr->empty0 + 8u * lr->slot);
    lr->advance();
  }
  consumer_sync();
  if (lr != nullptr) stamp(cx, 8 * kind + ST_LN);
}

// has_ln / epi are run-time (warp-uniform) switches on purpose: the kernel holds ONE copy of this code for its five call
// patterns (a 256 KB kernel thrashed the instruction cache at every phase change).
SV_DEVINL void gemv_flow(FCtx& cx, Ring& r, LnRing& lr, const bool has_ln, const int epi, const uint32_t* __restrict__ X, uint32_t EX,
                         const bf16* __restrict__ bias, const uint32_t* res, uint32_t ER, uint32_t* Y, uint32_t EY, int N, int K, int act,
                         uint32_t gp, int kind) {
  const FlowArgs& a = *cx.a;
  const Plan p = plan_of(cx.smem, kind);
  if (p.ntile <= 0) return;
  stamp(cx, 8 * kind + ST_ENTER);                          // nothing to do here: go and wait where this CTA has work
  const int warp = cx.warp, g = cx.g, t = cx.t;
  const int cps = p.KS >> 5;                         // 32-wide chunks per slot row
  const int cpws = (cps + NWC - 1) / NWC;            // chunks per warp per slot (<= CPW)
  const bool row_ok = g < a.B;
  const uint32_t* xp = X + (int64_t)(row_ok ? g : 0) * ll_words(K) + (int64_t)t * FRAG_STRIDE;   // fragment t of chunk 0
  constexpr int CHUNK = 4 * FRAG_STRIDE;             // words between the fragments of consecutive 32-wide k chunks
  const bool big_k = p.nstg > 2;

  // activations of the whole phase live in registers when K <= 2048 (8 fragments per lane)
  uint4 xr[2 * CPW];
#pragma unroll
  for (int i = 0; i < 2 * CPW; ++i) xr[i] = make_uint4(0u, 0u, 0u, 0u);
  if (!big_k) {
    uint8_t* xs = cx.smem + OFF_ATT;                   // the attention scratch is free during a GEMV phase
    stage_vector(cx, has_ln ? &lr : nullptr, X, EX, K, xs, kind);
    if (row_ok) {
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int j = 0; j < CPW; ++j)
          if (ks < p.nstg && j < cpws && (warp + NWC * j) < cps)
            xr[ks * CPW + j] = *reinterpret_cast<const uint4*>(xs + g * xs_pitch(K) + ((ks * cps + warp + NWC * j) * 4 + t) * 16);
    }
  }

  float c[4] = {0.f, 0.f, 0.f, 0.f};
  for (int tl = 0; tl < p.ntile; ++tl) {
    const int tile = p.tile0 + tl;
    // the epilogue thread's residual word: requested now, checked after the MMAs (it was written a phase ago)
    const int en = threadIdx.x & 15, emm = threadIdx.x >> 4;
    const int ecol = tile * p.R + en;
    const bool eok = threadIdx.x < 128 && en < p.R && ecol < N && emm < a.B;
    uint32_t rword = 0;
    if (res != nullptr && eok) rword = ld_rlx32(res + emm * ll_words(N) + ll_off(ecol));
    float bias_v = 0.f;                                  // read from the padding of the tile's last slab (flow_repack_kernel)
    if (!big_k) {
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        if (ks < p.nstg) {
          mbar_wait(r.full0 + 8u * r.slot, r.phase);
          if (tl == 0 && ks == 0) stamp(cx, 8 * kind + ST_W0);
          const uint32_t sb = r.base + r.slot * SLOT_BYTES + g * p.pitch + t * 16;
#pragma unroll
          for (int j = 0; j < CPW; ++j) {
            const int cl = warp + NWC * j;
            if (j < cpws && cl < cps) {
              const uint4 lo = lds16(sb + cl * 64), hi = lds16(sb + 8 * p.pitch + cl * 64);
              const uint4 xv = xr[ks * CPW + j];
              mma_bf16_16816(c, lo.x, hi.x, lo.y, hi.y, xv.x, xv.y);
              mma_bf16_16816(c, lo.z, hi.z, lo.w, hi.w, xv.z, xv.w);
            }
          }
          if (bias != nullptr && ks == p.nstg - 1 && threadIdx.x < 128)
            bias_v = __uint_as_float(*reinterpret_cast<const uint32_t*>(cx.smem + r.slot * SLOT_BYTES + en * p.pitch + p.KS * 2) << 16);
          __syncwarp();
          if (cx.lane == 0) mbar_arrive(r.empty0 + 8u * r.slot);
          r.advance();
        }
      }
    } else {
      // K > 2048: activation fragments are fetched per slab from L2, one slab ahead of their use.  The loads of slab
      // ks + 1 are ISSUED before the MMAs of slab ks and only CHECKED after them, so the L2 round trip hides behind the
      // weight wait + MMAs (checking at once cost one exposed round trip per slab: 8 per mlp.c_proj tile).
      uint4 xc[CPW], xn[CPW], ra[CPW], rb[CPW];
      auto issue = [&](int ks) {
#pragma unroll
        for (int j = 0; j < CPW; ++j) {
          const int cl = warp + NWC * j;
          if (row_ok && ks < p.nstg && j < cpws && cl < cps) {
            const uint32_t* q = xp + (int64_t)(ks * cps + cl) * CHUNK;
            ra[j] = ld_rlx16(q); rb[j] = ld_rlx16(q + 4);
          }
        }
      };
      auto finish = [&](int ks) {                          // raw words -> fragments; spins (re-loading) until every tag matches
#pragma unroll
        for (int j = 0; j < CPW; ++j) xn[j] = make_uint4(0u, 0u, 0u, 0u);
        if (row_ok && ks < p.nstg) {
          uint32_t it = 0;
          for (;;) {
            uint32_t bad = 0;
#pragma unroll
            for (int j = 0; j < CPW; ++j) {
              const int cl = warp + NWC * j;
              if (j < cpws && cl < cps) {
                bad |= ((ra[j].x ^ EX) | (ra[j].y ^ EX) | (ra[j].z ^ EX) | (ra[j].w ^ EX) | (rb[j].x ^ EX) | (rb[j].y ^ EX) | (rb[j].z ^ EX) |
                        (rb[j].w ^ EX)) >> 16;
                xn[j].x = __byte_perm(ra[j].x, ra[j].y, 0x5410); xn[j].y = __byte_perm(ra[j].z, ra[j].w, 0x5410);
                xn[j].z = __byte_perm(rb[j].x, rb[j].y, 0x5410); xn[j].w = __byte_perm(rb[j].z, rb[j].w, 0x5410);
              }
            }
            if (!bad) break;
            __nanosleep(40);
            spin_guard(it);
            issue(ks);
          }
        }
      };
      issue(0);
      finish(0);
      if (tl == 0) stamp(cx, 8 * kind + ST_XREADY);
      for (int ks = 0; ks < p.nstg; ++ks) {
#pragma unroll
        for (int j = 0; j < CPW; ++j) xc[j] = xn[j];
        issue(ks + 1);
        mbar_wait(r.full0 + 8u * r.slot, r.phase);
        if (tl == 0 && ks == 0) stamp(cx, 8 * kind + ST_W0);
        const uint32_t sb = r.base + r.slot * SLOT_BYTES + g * p.pitch + t * 16;
#pragma unroll
        for (int j = 0; j < CPW; ++j) {
          const int cl = warp + NWC * j;
          if (j < cpws && cl < cps) {
            const uint4 lo = lds16(sb + cl * 64), hi = lds16(sb + 8 * p.pitch + cl * 64);
            mma_bf16_16816(c, lo.x, hi.x, lo.y, hi.y, xc[j].x, xc[j].y);
            mma_bf16_16816(c, lo.z, hi.z, lo.w, hi.w, xc[j].z, xc[j].w);
          }
        }
        if (bias != nullptr && ks == p.nstg - 1 && threadIdx.x < 128)
          bias_v = __uint_as_float(*reinterpret_cast<const uint32_t*>(cx.smem + r.slot * SLOT_BYTES + en * p.pitch + p.KS * 2) << 16);
        __syncwarp();
        if (cx.lane == 0) mbar_arrive(r.empty0 + 8u * r.slot);
        r.advance();
        finish(ks + 1);
      }
    }
    // ---- tile finished: deterministic cross-warp split-K reduction + epilogue
    if (tl == p.ntile - 1) stamp(cx, 8 * kind + ST_WLAST);
    float* rd = cx.red + (tl & 1) * (NWC * 16 * 8);
    rd[(warp * 16 + g) * 8 + 2 * t] = c[0]; rd[(warp * 16 + g) * 8 + 2 * t + 1] = c[1];
    rd[(warp * 16 + g + 8) * 8 + 2 * t] = c[2]; rd[(warp * 16 + g + 8) * 8 + 2 * t + 1] = c[3];
    c[0] = c[1] = c[2] = c[3] = 0.f;
    consumer_sync();
    if (threadIdx.x < 128) {
      float acc = 0.f;
#pragma unroll
      for (int w = 0; w < NWC; ++w) acc += rd[(w * 16 + en) * 8 + emm];
      float v = 0.f, v_bf = 0.f;          // v_bf: the value as the bf16 logits tensor holds it
      if (eok) {
        const float bv = bias_v;
        float rv = 0.f;
        if (res != nullptr) {
          uint32_t it = 0;
          while ((rword ^ ER) >> 16) { spin_guard(it); rword = ld_rlx32(res + emm * ll_words(N) + ll_off(ecol)); }
          rv = __uint_as_float(rword << 16);
        }
        v = epilogue_elem(acc, bv, act, res != nullptr, rv);
        const bf16 vb = __float2bfloat16_rn(v);
        v_bf = __bfloat162float(vb);
        if (epi == EPI_LL) {
          st_rlx32(Y + emm * ll_words(N) + ll_off(ecol), EY | (uint32_t)__bfloat16_as_ushort(vb));
        } else {
          a.logits[(int64_t)emm * N + ecol] = vb;
        }
      }
      if (epi == EPI_LMHEAD) {
        // penalised selection reads the logits themselves: order them before the partial word that announces the tile
        // (all 16 stores a partial covers come from this half-warp)
        if (cx.slow_select) { __threadfence(); __syncwarp(); }
        // greedy = argmax over the bf16 logits cast to float, lowest index wins ties (HF _sample; SURVEY.md App. B.3)
        float bv = eok ? v_bf : -INFINITY;
        int bi = eok ? ecol : 0x7fffffff;
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (en == 0 && emm < a.B) {
          // [tag16 | bf16 bits of the value | index]: one atomic 8-byte word
          const unsigned long long w = ((unsigned long long)(tag16(gp) | (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(bv))) << 32) |
                                       (unsigned long long)(uint32_t)bi;
          st_rlx64(a.amax + (int64_t)tile * 8 + emm, w);
        }
      }
    }
    // red[] is double-buffered by tile parity: one barrier per tile
  }
  stamp(cx, 8 * kind + ST_DONE);
}

// ---- attention, hop 1.  item = (image, kv head, key range c) = one CTA.
// Two sub-phases with different work splits, so that no (m, l, acc) partial ever has to be merged across warps:
//   1. keys split over warps: warp w computes S = q.K^T for key blocks w (and w + 8) of the item on the tensor cores
//      (the <= 16 query heads of the kv head are the MMA M dimension), the row maxima go through shared memory, and with the
//      item-wide maximum every warp turns its scores into P = exp2(S - M) once; P is parked in shared memory in exactly the
//      register layout the P.V MMA wants as its A operand (so there is no transpose);
//   2. output dims split over warps: warp w computes out[:, 16w .. 16w+15] = P . V over ALL keys of the item: it owns a
//      disjoint slice of the output, its V^T rows are 16-byte coalesced loads that are issued before the softmax finishes.
// One item covers <= ATT_BLKS = 8 key blocks (256 keys).  Up to 256 keys of context (the new token included) a single
// item holds the whole row: it normalises and writes the attention output directly (no merge hop).  Longer rows are cut
// into MAXS items or fewer of <= 8 blocks each, whose (m, l, acc) partials go to merge_flow as flagged fp32 words: at most
// MAXS * 256 = 16384 keys (decode_flow_max_keys).
constexpr int ATT_R = 1;                                  // key blocks per warp and item (2: a warp's blocks run one after the other)
constexpr int ATT_BLKS = NWC * ATT_R;                     // key blocks per item
constexpr int ATT_P_BYTES = ATT_BLKS * 2 * 32 * 16;       // P fragments: [block][h][lane] x 16 bytes
constexpr int OFF_ATT_M = OFF_ATT + ATT_P_BYTES;          // float [ATT_BLKS][16] block row maxima, then [ATT_BLKS][16] block row sums
constexpr int OFF_ATT_Q = OFF_ATT_M + 2 * ATT_BLKS * 16 * 4;   // the item's query heads, bf16 [16][D]
static_assert(ATT_P_BYTES + 2 * ATT_BLKS * 16 * 4 + 16 * D * 2 + 2 * D * 2 <= ATT_BYTES, "attention scratch must fit the mega layout's tree-merge buffer");
static_assert(8 * (2 * KS_MAX * 2 + 64) <= ATT_BYTES, "the staged activation vector (8 rows x 2048 values) shares that buffer");

SV_DEVINL void attn_split(int nkeys, int& nact, int& per) {
  const int nblk = (nkeys + 31) / 32;
  if (nblk <= ATT_BLKS) { nact = 1; per = nblk; return; }
  nact = min(MAXS, (nblk + NWC - 1) / NWC);
  per = (nblk + nact - 1) / nact;
  nact = (nblk + per - 1) / per;
}

// S (log2 domain, scaled, masked) of one 32-key block: thread (g, t) gets keys kb + 8t + 2j + e for head rows g (s[j][e])
// and g + 8 (s[j][2 + e]) -- the layout the P.V A operand needs (sv_attention.cu, fragment trick).  The row of key `cur_key`
// (the token being decoded: not in the cache yet) is read from shared memory at `ks` instead.
SV_DEVINL void qk_block(const uint32_t (&qa)[D / 16][4], const bf16* __restrict__ kbase, int kb, int key_end, int cur_key, uint32_t ks,
                        float scale_log2, float (&s)[4][4], int g, int t) {
  // all 16 K fragments of the lane are requested before the first MMA (one L2 round trip for the block, not sixteen);
  // the current token's row is fetched from global like any other (valid memory, stale content) and replaced by a select
  uint4 w[4][D / 32];
  bool cur[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int key = kb + 8 * (g >> 1) + 2 * j + (g & 1);
    key = key < key_end ? key : key_end - 1;
    cur[j] = key == cur_key;
    const bf16* kp = kbase + (int64_t)key * D + 8 * t;
#pragma unroll
    for (int jj = 0; jj < D / 32; ++jj) w[j][jj] = ldcg16(kp + 32 * jj);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int jj = 0; jj < D / 32; ++jj) {
      const uint4 c = lds16(ks + (32 * jj + 8 * t) * 2);
      uint4 v = w[j][jj];
      v.x = cur[j] ? c.x : v.x; v.y = cur[j] ? c.y : v.y; v.z = cur[j] ? c.z : v.z; v.w = cur[j] ? c.w : v.w;
      mma_bf16_16816(s[j], qa[2 * jj][0], qa[2 * jj][1], qa[2 * jj][2], qa[2 * jj][3], v.x, v.y);
      mma_bf16_16816(s[j], qa[2 * jj + 1][0], qa[2 * jj + 1][1], qa[2 * jj + 1][2], qa[2 * jj + 1][3], v.z, v.w);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool valid = (kb + 8 * t + 2 * j + e) < key_end;
      s[j][e] = valid ? s[j][e] * scale_log2 : -INFINITY;
      s[j][2 + e] = valid ? s[j][2 + e] * scale_log2 : -INFINITY;
    }
  }
}

// 8 keys of one V^T row (what the P.V B operand of a lane holds for a block): the element of key index `e` (0..7) is replaced
// by `val` -- the current token's v, which is not in the cache yet.  Written with selects only (no register indexing).
SV_DEVINL void patch_v(uint4& w, int e, uint32_t val) {
  const uint32_t lo = (e & 1) ? 0x0000ffffu : 0xffff0000u, ins = (e & 1) ? (val << 16) : val;
  w.x = (e >> 1) == 0 ? ((w.x & lo) | ins) : w.x;
  w.y = (e >> 1) == 1 ? ((w.y & lo) | ins) : w.y;
  w.z = (e >> 1) == 2 ? ((w.z & lo) | ins) : w.z;
  w.w = (e >> 1) == 3 ? ((w.w & lo) | ins) : w.w;
}

SV_DEVINL void attention_flow(FCtx& cx, const Layer* L, int cur_len, uint32_t E, uint32_t gp) {
  const FlowArgs& a = *cx.a;
  const int warp = cx.warp, lane = cx.lane, g = cx.g, t = cx.t;
  const int group = a.n_head / a.n_kv;
  const int nkeys = cur_len + 1;
  const int nblk = (nkeys + 31) / 32;
  int nact, per;
  attn_split(nkeys, nact, per);
  const float scale_log2 = 1.4426950408889634f / sqrtf((float)D);
  const uint32_t pbuf = smem_u32(cx.smem + OFF_ATT);
  float* mbuf = reinterpret_cast<float*>(cx.smem + OFF_ATT_M);
  float* lbuf = mbuf + ATT_BLKS * 16;
  uint8_t* qs = cx.smem + OFF_ATT_Q;                       // staged: the group's query heads [16][D], then k_cur [D], v_cur [D]
  const uint32_t ks = smem_u32(qs + 16 * D * 2);
  const unsigned short* vs = reinterpret_cast<const unsigned short*>(qs + 16 * D * 2 + D * 2);
  const unsigned long long T = tag32(gp);
  const int nitems = a.B * a.n_kv * nact;
  stamp(cx, ST_ATT_ENTER);
  for (int item = cx.cta; item < nitems; item += cx.ncta) {
    const int c = item % nact, bk = item / nact, kvh = bk % a.n_kv, b = bk / a.n_kv;
    const int blk0 = c * per, blk1 = min(nblk, blk0 + per), nb = blk1 - blk0;
    const bool has_cur = blk1 == nblk;                     // this item's last block holds the token being decoded
    const int cur_key = has_cur ? cur_len : -1;
    bf16* kb_ = L->kc + (int64_t)bk * a.tcap * D;
    bf16* vb_ = L->vc + (int64_t)bk * D * a.tcap;
    const uint32_t* qkv_row = a.qkv + b * ll_words(a.qkv_cols);
    // ---- one cooperative poll: the group's query heads and (last item only) the current token's k, v -> shared memory.
    // The cache append itself happens after the math: the current key / value are used from shared memory
    // (GPTBigCodeAttention.forward: key_value = cat(layer_past, key_value), vendored modeling_gpt_bigcode.py:265-267).
    {
      const int nq = group * (D / 8), nfr = nq + (has_cur ? 2 * (D / 8) : 0);
      wait_vector(cx, qkv_row + (int64_t)(kvh * nq) * FRAG_STRIDE, E, nq);
      for (int f0 = threadIdx.x; f0 < nfr; f0 += NCT) {
        const int frag = f0 < nq ? kvh * nq + f0
                                 : (f0 < nq + D / 8 ? (a.n_head + kvh) * (D / 8) + (f0 - nq) : (a.n_head + a.n_kv + kvh) * (D / 8) + (f0 - nq - D / 8));
        LLRaw raw;
        uint4 v;
        uint32_t it = 0;
        for (;;) {
          ll_issue(qkv_row + (int64_t)frag * FRAG_STRIDE, raw);
          if (!ll_finish(raw, E, v)) break;
          __nanosleep(40);
          spin_guard(it);
        }
        *reinterpret_cast<uint4*>(qs + (f0 < nq ? f0 : 16 * (D / 8) + (f0 - nq)) * 16) = v;
      }
      consumer_sync();
    }
    stamp(cx, ST_ATT_Q);
    // ---- V^T loads of every key block of the item: issued now, used after the scores (they only depend on addresses)
    const bf16* v0 = vb_ + (int64_t)(16 * warp + g) * a.tcap + blk0 * 32 + 8 * t;       // V^T row of n-tile 0; n-tile 1: + 8 rows
    uint4 vv[ATT_BLKS][2];
#pragma unroll
    for (int i = 0; i < ATT_BLKS / 2; ++i) {               // first half now, second half once the K fragments are consumed
      const int bi = min(i, nb - 1);
      vv[i][0] = ldcg16(v0 + bi * 32);
      vv[i][1] = ldcg16(v0 + 8 * (int64_t)a.tcap + bi * 32);
    }
    // ---- sub-phase 1: scores of this warp's key blocks.  Every block is finished on the spot with ITS OWN row maxima
    // (P = exp2(S - m_block), bf16, parked as MMA A fragments; m_block and the row sums go to shared memory): no score outlives
    // its block, the item-wide maximum enters later as one scale factor per (block, head) on the block's P.V product.
    if (warp < nb) {
      uint32_t qa[D / 16][4];
#pragma unroll
      for (int jj = 0; jj < D / 32; ++jj) {
        uint4 lo = make_uint4(0u, 0u, 0u, 0u), hi = make_uint4(0u, 0u, 0u, 0u);
        if (g < group) lo = *reinterpret_cast<const uint4*>(qs + (g * (D / 8) + 4 * jj + t) * 16);
        if (g + 8 < group) hi = *reinterpret_cast<const uint4*>(qs + ((g + 8) * (D / 8) + 4 * jj + t) * 16);
        qa[2 * jj][0] = lo.x; qa[2 * jj][1] = hi.x; qa[2 * jj][2] = lo.y; qa[2 * jj][3] = hi.y;
        qa[2 * jj + 1][0] = lo.z; qa[2 * jj + 1][1] = hi.z; qa[2 * jj + 1][2] = lo.w; qa[2 * jj + 1][3] = hi.w;
      }
#pragma unroll 1
      for (int r = 0; r < ATT_R; ++r) {
        const int bi = warp + r * NWC;
        if (bi < nb) {
          const int kb = (blk0 + bi) * 32;
          float s[4][4];
          qk_block(qa, kb_, kb, min(nkeys, kb + 32), cur_key, ks, scale_log2, s, g, t);
          float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
            mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
          }
          mx0 = quad_max(mx0); mx1 = quad_max(mx1);           // finite: a block always holds at least one real key
          float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            s[j][0] = exp2f(s[j][0] - mx0); s[j][1] = exp2f(s[j][1] - mx0);
            s[j][2] = exp2f(s[j][2] - mx1); s[j][3] = exp2f(s[j][3] - mx1);
            rs0 += s[j][0] + s[j][1]; rs1 += s[j][2] + s[j][3];
          }
          rs0 = quad_sum(rs0); rs1 = quad_sum(rs1);
          if (t == 0) { mbuf[bi * 16 + g] = mx0; mbuf[bi * 16 + g + 8] = mx1; lbuf[bi * 16 + g] = rs0; lbuf[bi * 16 + g + 8] = rs1; }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint4 pa;
            pa.x = pack_bf16x2(s[2 * h][0], s[2 * h][1]);
            pa.y = pack_bf16x2(s[2 * h][2], s[2 * h][3]);
            pa.z = pack_bf16x2(s[2 * h + 1][0], s[2 * h + 1][1]);
            pa.w = pack_bf16x2(s[2 * h + 1][2], s[2 * h + 1][3]);
            asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(pbuf + ((bi * 2 + h) * 32 + lane) * 16), "r"(pa.x), "r"(pa.y),
                         "r"(pa.z), "r"(pa.w) : "memory");
          }
        }
      }
    }
#pragma unroll
    for (int i = ATT_BLKS / 2; i < ATT_BLKS; ++i) {
      const int bi = min(i, nb - 1);
      vv[i][0] = ldcg16(v0 + bi * 32);
      vv[i][1] = ldcg16(v0 + 8 * (int64_t)a.tcap + bi * 32);
    }
    consumer_sync();
    stamp(cx, ST_ATT_BLK);
    // ---- sub-phase 2: out[:, 16 * warp + {0..15}] = sum over the item's key blocks of 2^(m_block - M) * P_block . V_block
    float M0 = -INFINITY, M1 = -INFINITY;
    for (int bi = 0; bi < nb; ++bi) { M0 = fmaxf(M0, mbuf[bi * 16 + g]); M1 = fmaxf(M1, mbuf[bi * 16 + g + 8]); }
    float acc[2][4], L0 = 0.f, L1 = 0.f;
#pragma unroll
    for (int n = 0; n < 2; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
    // the lane whose 8 keys of the last block contain the current token takes its v from shared memory
    const int cur_e = cur_len - (nblk - 1) * 32 - 8 * t;       // element index inside that lane's 8 keys, if in [0, 8)
    const bool patch = has_cur && cur_e >= 0 && cur_e < 8;
#pragma unroll
    for (int bi = 0; bi < ATT_BLKS; ++bi) {
      if (bi < nb) {
        if (patch && bi == nb - 1) {
          patch_v(vv[bi][0], cur_e, (uint32_t)vs[16 * warp + g]);
          patch_v(vv[bi][1], cur_e, (uint32_t)vs[16 * warp + 8 + g]);
        }
        const uint4 p0 = lds16(pbuf + ((bi * 2 + 0) * 32 + lane) * 16), p1 = lds16(pbuf + ((bi * 2 + 1) * 32 + lane) * 16);
        const float sc0 = exp2f(mbuf[bi * 16 + g] - M0), sc1 = exp2f(mbuf[bi * 16 + g + 8] - M1);
        L0 += lbuf[bi * 16 + g] * sc0; L1 += lbuf[bi * 16 + g + 8] * sc1;
#pragma unroll
        for (int n = 0; n < 2; ++n) {
          float pv[4] = {0.f, 0.f, 0.f, 0.f};
          mma_bf16_16816(pv, p0.x, p0.y, p0.z, p0.w, vv[bi][n].x, vv[bi][n].y);
          mma_bf16_16816(pv, p1.x, p1.y, p1.z, p1.w, vv[bi][n].z, vv[bi][n].w);
          acc[n][0] += pv[0] * sc0; acc[n][1] += pv[1] * sc0; acc[n][2] += pv[2] * sc1; acc[n][3] += pv[3] * sc1;
        }
      }
    }
    stamp(cx, ST_ATT_TREE);
    if (nact == 1) {
      // the whole row was in this item: normalise and publish the attention output (bf16, like the reference's attn_output)
      uint32_t* orow = a.att + b * ll_words(a.n_head * D);
      const float i0 = 1.0f / L0, i1 = 1.0f / L1;
#pragma unroll
      for (int n = 0; n < 2; ++n) {
        const int d = 16 * warp + 8 * n + 2 * t;           // d, d + 1 share a fragment
        if (g < group) {
          uint32_t* o = orow + ll_off((kvh * group + g) * D + d);
          st_rlx32(o, E | (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(acc[n][0] * i0)));
          st_rlx32(o + 1, E | (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(acc[n][1] * i0)));
        }
        if (g + 8 < group) {
          uint32_t* o = orow + ll_off((kvh * group + g + 8) * D + d);
          st_rlx32(o, E | (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(acc[n][2] * i1)));
          st_rlx32(o + 1, E | (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(acc[n][3] * i1)));
        }
      }
    } else {
      unsigned long long* ws = a.part + ((int64_t)bk * MAXS + c) * PSZ;
      if (warp == 0 && t == 0) {
        st_rlx64(ws + g, fword(M0, T)); st_rlx64(ws + g + 8, fword(M1, T));
        st_rlx64(ws + 16 + g, fword(L0, T)); st_rlx64(ws + 16 + g + 8, fword(L1, T));
      }
#pragma unroll
      for (int n = 0; n < 2; ++n) {
        const int d = 16 * warp + 8 * n + 2 * t;
        st_rlx64(ws + 32 + g * D + d, fword(acc[n][0], T)); st_rlx64(ws + 32 + g * D + d + 1, fword(acc[n][1], T));
        st_rlx64(ws + 32 + (g + 8) * D + d, fword(acc[n][2], T)); st_rlx64(ws + 32 + (g + 8) * D + d + 1, fword(acc[n][3], T));
      }
    }
    stamp(cx, ST_ATT_DONE);
    // ---- the cache append, off the critical path: K row (16 x 16 bytes) and V^T column (D x 2 bytes) from the staged copies
    if (has_cur && cur_len < a.tcap) {
      const int tid = threadIdx.x;
      if (tid < D / 8) __stcg(reinterpret_cast<uint4*>(kb_ + (int64_t)cur_len * D) + tid, *reinterpret_cast<const uint4*>(qs + 16 * D * 2 + tid * 16));
      if (tid >= 32 && tid < 32 + D)
        __stcg(reinterpret_cast<unsigned short*>(vb_) + (int64_t)(tid - 32) * a.tcap + cur_len, vs[tid - 32]);
    }
    consumer_sync();                                      // the scratch is reused by the CTA's next item
  }
}

// ---- attention, hop 2: distributed merge of the item partials; task = (image, head, 32 output dims) = one warp
SV_DEVINL void merge_flow(FCtx& cx, int cur_len, uint32_t E, uint32_t gp) {
  const FlowArgs& a = *cx.a;
  const int group = a.n_head / a.n_kv;
  int nact, per;
  attn_split(cur_len + 1, nact, per);
  if (nact == 1) return;                               // the single item published the output itself
  const unsigned long long T = tag32(gp);
  const int ntasks = a.B * a.n_head * (D / 32);
  for (int task = cx.cta + cx.ncta * cx.warp; task < ntasks; task += cx.ncta * NWC) {
    const int q4 = task % (D / 32), head = (task / (D / 32)) % a.n_head, b = task / ((D / 32) * a.n_head);
    const int kvh = head / group, rr = head % group, dim = q4 * 32 + cx.lane;
    const unsigned long long* p0 = a.part + ((int64_t)(b * a.n_kv + kvh) * MAXS) * PSZ;
    float M = -INFINITY, Lsum = 0.f, A = 0.f;
    for (int c0 = 0; c0 < nact; c0 += 8) {
      unsigned long long wm[8], wl[8], wa[8];
      uint32_t it = 0;
      bool bad;
      do {
#pragma unroll
        for (int j = 0; j < 8; ++j) {                    // every load of the poll first ...
          if (c0 + j < nact) {
            const unsigned long long* pc = p0 + (int64_t)(c0 + j) * PSZ;
            wm[j] = ld_rlx64(pc + rr); wl[j] = ld_rlx64(pc + 16 + rr); wa[j] = ld_rlx64(pc + 32 + rr * D + dim);
          }
        }
        unsigned long long x = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j)                      // ... then the tags
          if (c0 + j < nact) x |= (wm[j] ^ T) | (wl[j] ^ T) | (wa[j] ^ T);
        bad = (x >> 32) != 0;
        if (bad) { __nanosleep(100); spin_guard(it); }
      } while (bad);
      float Mn = M;
#pragma unroll
      for (int j = 0; j < 8; ++j) if (c0 + j < nact) Mn = fmaxf(Mn, __uint_as_float((uint32_t)wm[j]));
      const float sc0 = (M == -INFINITY) ? 0.f : exp2f(M - Mn);
      Lsum *= sc0; A *= sc0; M = Mn;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (c0 + j < nact) {
          const float m = __uint_as_float((uint32_t)wm[j]);
          const float sc = (m == -INFINITY) ? 0.f : exp2f(m - M);
          Lsum += __uint_as_float((uint32_t)wl[j]) * sc;
          A += __uint_as_float((uint32_t)wa[j]) * sc;
        }
      }
    }
    const bf16 o = __float2bfloat16_rn(A / Lsum);
    st_rlx32(a.att + b * ll_words(a.n_head * D) + ll_off(head * D + dim), E | (uint32_t)__bfloat16_as_ushort(o));
  }
}

// ---- next step's input: x = wte[token] + wpe[position] (GPTBigCodeModel.forward), as flagged words (+ a plain copy)
SV_DEVINL void embed_flow(const FCtx& cx, const int* toks, int pos, uint32_t E) {
  const FlowArgs& a = *cx.a;
  pos = pos >= a.n_positions ? a.n_positions - 1 : pos;
  const int hv = a.H >> 3;
  for (int i = threadIdx.x; i < a.B * hv; i += NCT) {
    const int b = i / hv, col = (i % hv) * 8;
    int id = toks[b];
    id = id < 0 ? 0 : (id >= a.vocab ? a.vocab - 1 : id);
    float e[8], q[8];
    unpack8(ldg_cached(a.wte + (int64_t)id * a.H + col), e);
    if (a.wpe) {
      unpack8(ldg_cached(a.wpe + (int64_t)pos * a.H + col), q);
#pragma unroll
      for (int j = 0; j < 8; ++j) e[j] += q[j];
    }
    const uint4 v = pack8(e);
    ll_put8(a.xa + b * ll_words(a.H) + ll_off(col), E, v);
    *reinterpret_cast<uint4*>(a.x_plain + (int64_t)b * a.H + col) = v;
  }
}

// ---- token selection (CTA 0): argmax partials (or penalised scan of the logits) -> HF bookkeeping -> embedding
SV_DEVINL void select_flow(FCtx& cx, int ntiles, uint32_t gp, int next_pos, uint32_t Enext) {
  const FlowArgs& a = *cx.a;
  AmaxPair* sm = reinterpret_cast<AmaxPair*>(cx.red);
  int* s_tok = reinterpret_cast<int*>(cx.smem + FLOW_OFF_TOK);
  GenState* st = reinterpret_cast<GenState*>(cx.smem + FLOW_OFF_STATE);          // working copies (decode_flow_kernel prologue):
  const GenParamsDev* prm = reinterpret_cast<const GenParamsDev*>(st + 1);         // no global round trips in the bookkeeping
  const int tid = threadIdx.x;
  const float rp = prm->rep_penalty;
  const uint32_t T16 = tag16(gp) >> 16;
  const bool done = st->done != 0;                 // only this CTA ever writes the state during the launch
  for (int b = 0; b < a.B; ++b) {
    AmaxPair best{-INFINITY, 0x7fffffff};
    // the partial words double as "this tile's logits are complete" (the penalised path fenced before writing them)
    for (int i0 = tid; i0 < ntiles; i0 += 4 * NCT) {
      unsigned long long w[4];
      uint32_t it = 0;
      bool bad;
      do {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (i0 + j * NCT < ntiles) w[j] = ld_rlx64(a.amax + (int64_t)(i0 + j * NCT) * 8 + b);
        bad = false;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (i0 + j * NCT < ntiles) bad |= (uint32_t)(w[j] >> 48) != T16;
        if (bad) { __nanosleep(100); spin_guard(it); }
      } while (bad);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (i0 + j * NCT < ntiles) {
          const float v = __uint_as_float(((uint32_t)(w[j] >> 32) & 0xffffu) << 16);
          best = amax_better(best, AmaxPair{v, (int)(uint32_t)w[j]});
        }
      }
    }
    if (rp != 1.0f) {
      best = AmaxPair{-INFINITY, 0x7fffffff};
      consumer_sync();                                // every partial seen by some thread -> all logits are in L2
      const bf16* lr = a.logits + (int64_t)b * a.vocab;
      const uint8_t* sr = a.seen + (int64_t)b * a.vocab;
      for (int i = tid; i < a.vocab; i += NCT) {
        float v = __bfloat162float(__ldcg(lr + i));
        if (__ldcg(sr + i)) v = v < 0.f ? v * rp : v / rp;
        best = amax_better(best, AmaxPair{v, i});
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      AmaxPair other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
      best = amax_better(best, other);
    }
    consumer_sync();
    if (cx.lane == 0) sm[cx.warp] = best;
    consumer_sync();
    if (tid == 0) {
      for (int w = 1; w < NWC; ++w) best = amax_better(best, sm[w]);
      s_tok[b] = best.i == 0x7fffffff ? 0 : best.i;
    }
  }
  consumer_sync();
  if (tid == 0 && !done) {
    select_apply_tokens(s_tok, a.B, a.vocab, st, prm, a.seen, a.next_ids, a.out_ids, 1);
    a.state->cur_len = st->cur_len; a.state->step = st->step; a.state->done = st->done;      // for the host / the next launch
    for (int b = 0; b < a.B; ++b) a.state->unfinished[b] = st->unfinished[b];
  }
  consumer_sync();
  embed_flow(cx, s_tok, next_pos, Enext);           // after `done` the other CTAs keep stepping until the launch ends
}

// ---- the static schedule: phase q of a token = layer q / 4, kind q % 4 (0 c_attn, 1 attn.c_proj, 2 mlp.c_fc, 3 mlp.c_proj);
// q == 4 * n_layer is the lm_head
struct PhaseW { const bf16 *W, *ln_w, *ln_b; int N, K, kind; };     // W: the slab-tiled copy of the phase's weight matrix
SV_DEVINL PhaseW phase_weights(const FlowArgs& a, const Layer* layers, int q) {
  PhaseW w;
  w.ln_w = nullptr; w.ln_b = nullptr;
  if (q == 4 * a.n_layer) { w.W = a.lm_head_t; w.N = a.vocab; w.K = a.H; w.kind = 4; w.ln_w = a.lnf_w; w.ln_b = a.lnf_b; return w; }
  const Layer* L = layers + (q >> 2);
  w.kind = q & 3;
  switch (w.kind) {
    case 0: w.W = L->attn_t; w.N = a.qkv_cols; w.K = a.H; w.ln_w = L->ln1_w; w.ln_b = L->ln1_b; break;
    case 1: w.W = L->proj_t; w.N = a.H; w.K = a.H; break;
    case 2: w.W = L->fc_t; w.N = a.I; w.K = a.H; w.ln_w = L->ln2_w; w.ln_b = L->ln2_b; break;
    default: w.W = L->fc2_t; w.N = a.H; w.K = a.I; break;
  }
  return w;
}

// L2 prefetch that leaves the region L2-resident: one 4-byte ld.global.cg with the L2::128B prefetch size per 128-byte
// line.  `rows` pieces of `row_bytes` (a multiple of 128), `row_stride` bytes apart; one warp, 8 independent loads per lane in
// flight.  The loaded words are folded into `t.acc` only at the NEXT call (by then they have long arrived): that keeps the
// eight destination registers distinct and alive -- dead outputs would share one register and serialise on its scoreboard --
// without ever waiting for a load that was just issued.
struct L2Touch { uint32_t v[8], acc; };
SV_DEVINL void l2_touch(L2Touch& t, const char* base, int rows, int64_t row_stride, int row_bytes, int lane) {
  const int lpr = row_bytes >> 7, nlines = rows * lpr;
  for (int i0 = lane; i0 < nlines; i0 += 8 * 32) {
    t.acc ^= t.v[0] ^ t.v[1] ^ t.v[2] ^ t.v[3] ^ t.v[4] ^ t.v[5] ^ t.v[6] ^ t.v[7];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int i = min(i0 + k * 32, nlines - 1);
      asm volatile("ld.global.cg.L2::128B.u32 %0, [%1];" : "=r"(t.v[k]) : "l"(base + (int64_t)(i / lpr) * row_stride + (i % lpr) * 128) : "memory");
    }
  }
}

// The prefetch warp also pulls the K / V^T blocks this CTA's attention items of a layer will read (everything but the current
// token, which arrives as flagged words) into L2 a few microseconds before the attention phase.
SV_DEVINL void prefetch_kv_l2(L2Touch& tch, const FlowArgs& a, const Layer* L, int cur_len, int cta, int ncta, int lane) {
  if (cur_len <= 0) return;
  const int nkeys = cur_len + 1, nblk = (nkeys + 31) / 32;
  int nact, per;
  attn_split(nkeys, nact, per);
  const int nitems = a.B * a.n_kv * nact;
  for (int item = cta; item < nitems; item += ncta) {
    const int c = item % nact, bk = item / nact;
    const int key0 = c * per * 32, key1 = min(cur_len, min(nblk, c * per + per) * 32);       // cached keys of the item
    if (key1 <= key0) continue;
    const int kbytes = ((key1 - key0) * D * 2 + 127) & ~127;                                 // K rows are contiguous
    l2_touch(tch, reinterpret_cast<const char*>(L->kc + ((int64_t)bk * a.tcap + key0) * D), 1, 0, kbytes, lane);
    const int vbytes = ((key1 - key0) * 2 + 127) & ~127;                                     // V^T: D rows, tcap * 2 bytes apart
    l2_touch(tch, reinterpret_cast<const char*>(L->vc + (int64_t)bk * D * a.tcap + key0), D, (int64_t)a.tcap * 2, vbytes, lane);
  }
}

constexpr int FLOW_THREADS = NCT + 64;        // 8 consumer warps + producer warp + L2 prefetch warp
constexpr int FLOW_THREADS_REALLOC = NCT + 128;

template <bool REALLOC>
__global__ void __launch_bounds__(REALLOC ? FLOW_THREADS_REALLOC : FLOW_THREADS, 1) decode_flow_kernel(const FlowArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cta = blockIdx.x, ncta = gridDim.x;
  Ring ring;
  ring.base = smem_u32(smem);
  ring.full0 = smem_u32(smem + FLOW_OFF_BAR);
  ring.empty0 = ring.full0 + 8u * STAGES;
  ring.slot = 0; ring.phase = 0; ring.nslots = STAGES;
  LnRing lnr;
  lnr.base = smem_u32(smem + FLOW_OFF_LN);
  lnr.full0 = ring.empty0 + 8u * STAGES;
  lnr.empty0 = lnr.full0 + 16u;
  lnr.slot = 0; lnr.phase = 0;
  if (threadIdx.x == 0) {
    *reinterpret_cast<uint32_t*>(smem + FLOW_OFF_PROG) = 0u;
    *reinterpret_cast<uint32_t*>(smem + FLOW_OFF_PROG + 4) = 0u;
    for (int s = 0; s < STAGES; ++s) { mbar_init(ring.full0 + 8u * s, 1); mbar_init(ring.empty0 + 8u * s, NWC); }
    for (int s = 0; s < 2; ++s) { mbar_init(lnr.full0 + 8u * s, 1); mbar_init(lnr.empty0 + 8u * s, NWC); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const Layer* layers_s = reinterpret_cast<const Layer*>(smem + FLOW_OFF_LAYERS);
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(a.layers);
    uint32_t* dst = reinterpret_cast<uint32_t*>(smem + FLOW_OFF_LAYERS);
    for (int i = threadIdx.x; i < a.n_layer * (int)(sizeof(Layer) / 4); i += blockDim.x) dst[i] = src[i];
    if (threadIdx.x < 5) {
      const int k = threadIdx.x;
      const int N = k == 0 ? a.qkv_cols : (k == 2 ? a.I : (k == 4 ? a.vocab : a.H)), K = k == 3 ? a.I : a.H;
      reinterpret_cast<Plan*>(smem + FLOW_OFF_PLANS)[k] = make_plan(N, K, cta, ncta);
    }
  }
  __syncthreads();

  if (warp >= NWC) {
    if constexpr (REALLOC) {
      // the pool is what the launch allocated (384 x 168): the 4 x 32 x (168 - 56) registers given back here are exactly the
      // 8 x 32 x (224 - 168) the consumers ask for below -- any other split never gets its setmaxnreg.inc satisfied
      asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(56));
      if (warp > NWC + 1) return;
    }
    const uint32_t progress = smem_u32(smem + FLOW_OFF_PROG);                                   // slabs the producer has issued
    if (warp == NWC) {
      // =========================== producer: the static weight schedule of the whole launch ===========================
      // Plain nested loops (token, phase, tile, k slab): per slab only the wait for a free slot and <= 16 bulk copies,
      // one per lane -- this loop must stay far ahead of the consumers (an earlier version that re-derived its position
      // from a generic iterator for every slab fell behind them and halved the throughput).
      long long* pdbg = (a.dbg != nullptr && cta == 0 && lane == 0) ? a.dbg + DBG_HALF : nullptr;
      int pi = 0;
      uint32_t issued = 0;
      for (int s = 0; s < a.nsteps; ++s) {
        if (s == 1) pdbg = nullptr;
        for (int q = 0; q <= 4 * a.n_layer; ++q) {
          const PhaseW w = phase_weights(a, layers_s, q);
          const Plan p = plan_of(smem, w.kind);
          if (p.ntile <= 0) continue;                                    // the consumers skip the phase as well
          stamp_raw(pdbg, pi, ST_PROD + 2 * w.kind);
          if (w.ln_w != nullptr) produce_ln(lnr, w.ln_w, w.ln_b, w.N, w.K, cta, ncta, lane);
          // the CTA's slabs of this matrix are one contiguous run of SLOT_BYTES blocks in the tiled copy (flow_repack_kernel):
          // ONE bulk copy per slab (one large copy streams faster than one 2 KB copy per weight row)
          const char* src = reinterpret_cast<const char*>(w.W) + (int64_t)cta * p.tpc * p.nstg * SLOT_BYTES;
          const uint32_t bytes = (uint32_t)(p.R * p.pitch);
          const int nslab = p.ntile * p.nstg;
          for (int i = 0; i < nslab; ++i) {
            if (lane == 0) {
              const uint32_t fb = ring.full0 + 8u * ring.slot;
              // "blocked" = the ring is full and the consumers are not draining it (a latency-bound stretch): only then does
              // the prefetch warp run ahead -- its requests would otherwise queue in front of the slabs the ring is waiting for
              asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(progress + 4u), "r"(1u) : "memory");
              mbar_wait(ring.empty0 + 8u * ring.slot, ring.phase ^ 1u);
              asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(progress + 4u), "r"(0u) : "memory");
              mbar_expect_tx(fb, bytes);
              bulk_g2s(ring.base + ring.slot * SLOT_BYTES, src + (int64_t)i * SLOT_BYTES, bytes, fb);
              asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(progress), "r"(++issued) : "memory");
            }
            ring.advance();
          }
        }
      }
    } else {
      // =========================== L2 prefetcher: the same schedule, `l2_ahead` slabs in front of the producer ==========
      // cp.async.bulk.prefetch.L2 only: HBM keeps streaming into L2 while the ring is full and the consumers sit in a
      // latency-bound stretch (attention, hops); the ring then refills from L2.
      uint32_t j = 0;
      L2Touch tch;
#pragma unroll
      for (int k = 0; k < 8; ++k) tch.v[k] = 0u;
      tch.acc = 0u;
      for (int s = 0; s < a.nsteps; ++s) {
        for (int q = 0; q <= 4 * a.n_layer; ++q) {
          const PhaseW w = phase_weights(a, layers_s, q);
          const Plan p = plan_of(smem, w.kind);
          const char* src = reinterpret_cast<const char*>(w.W) + (int64_t)cta * p.tpc * p.nstg * SLOT_BYTES;
          const int nslab = p.ntile * p.nstg, bytes = (p.R * p.pitch + 127) & ~127;
          for (int i = 0; i < nslab; ++i, ++j) {
            uint32_t it = 0, prog, blocked;
            for (;;) {
              asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(prog) : "r"(progress) : "memory");
              asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(blocked) : "r"(progress + 4u) : "memory");
              if ((int32_t)(j - prog) < STAGES) break;                        // fell behind the ring: skip ahead
              if ((int32_t)(j - prog) <= a.l2_ahead && blocked) break;
              __nanosleep(100);
              spin_guard(it);
            }
            if (a.l2_ahead > 0 && (int32_t)(j - prog) >= STAGES)              // slabs the ring is about to copy need no hint
              l2_touch(tch, src + (int64_t)i * SLOT_BYTES, 1, 0, bytes, lane);
          }
          // K / V of the NEXT attention phase: while the schedule is in mlp.c_proj of the layer before (or the lm_head of the
          // previous token), i.e. roughly one phase ahead of the c_attn GEMV whose output the attention waits for
          if (w.kind == 3 && (q >> 2) + 1 < a.n_layer) prefetch_kv_l2(tch, a, layers_s + (q >> 2) + 1, a.cur_len0 + s, cta, ncta, lane);
          if (w.kind == 4 && s + 1 < a.nsteps) prefetch_kv_l2(tch, a, layers_s, a.cur_len0 + s + 1, cta, ncta, lane);
        }
      }
      // (never true: the fold only exists to keep the prefetch loads' registers alive)
      if ((tch.acc ^ tch.v[0] ^ tch.v[1] ^ tch.v[2] ^ tch.v[3] ^ tch.v[4] ^ tch.v[5] ^ tch.v[6] ^ tch.v[7]) == 0x9e3779b9u && a.nsteps < 0)
        asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(progress), "r"(tch.acc) : "memory");
    }
    return;   // in-flight bulk copies are all consumed (and thus complete) before the consumers exit
  }
  // =========================== consumers ===========================
  if constexpr (REALLOC) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(224));
  FCtx cx;
  cx.a = &a; cx.smem = smem; cx.cta = cta; cx.ncta = ncta; cx.warp = warp; cx.lane = lane; cx.g = lane >> 2; cx.t = lane & 3;
  cx.red = reinterpret_cast<float*>(smem + OFF_RED);
  cx.stat = reinterpret_cast<float*>(smem + FLOW_OFF_STAT);
  cx.dbg = (a.dbg != nullptr && cta == 0 && threadIdx.x == 0) ? a.dbg : nullptr;
  cx.dbg_i = 0;
  cx.slow_select = a.params->rep_penalty != 1.0f;
  if (cta == 0 && a.do_select) {
    uint32_t* dst = reinterpret_cast<uint32_t*>(smem + FLOW_OFF_STATE);
    const uint32_t* s0 = reinterpret_cast<const uint32_t*>(a.state);
    const uint32_t* s1 = reinterpret_cast<const uint32_t*>(a.params);
    constexpr int n0 = (int)sizeof(GenState) / 4, n1 = (int)sizeof(GenParamsDev) / 4;
    for (int i = threadIdx.x; i < n0 + n1; i += NCT) dst[i] = i < n0 ? s0[i] : s1[i - n0];
    consumer_sync();
  }
  const int ntiles_lm = plan_of(smem, 4).ntiles;
  const uint32_t nl1 = (uint32_t)a.n_layer + 1u;
  if (a.first_plain && cta == 0) {
    // the step-0 input was written as plain bf16 by the kernel that selected / embedded the previous token
    const uint32_t E0 = tag16((uint32_t)a.step0 * nl1);
    const int hv = a.H >> 3;
    for (int i = threadIdx.x; i < a.B * hv; i += NCT) {
      const int b = i / hv, col = (i % hv) * 8;
      ll_put8(a.xa + b * ll_words(a.H) + ll_off(col), E0, __ldcg(reinterpret_cast<const uint4*>(a.x_plain + (int64_t)b * a.H + col)));
    }
  }
  for (int s = 0; s < a.nsteps; ++s) {
    const uint32_t gs = (uint32_t)(a.step0 + s);
    const int cur_len = a.cur_len0 + s;
    if (s == 1) cx.dbg = nullptr;
    for (int q = 0; q <= 4 * a.n_layer; ++q) {
      const int l = q >> 2;
      const uint32_t gp = gs * nl1 + (uint32_t)l;          // the lm_head (q = 4 * n_layer) is "layer n_layer"
      const uint32_t E = tag16(gp), En = tag16(gp + 1u);
      const PhaseW w = phase_weights(a, layers_s, q);
      const Layer* L = layers_s + (l < a.n_layer ? l : 0);
      const uint32_t *X, *res = nullptr;
      uint32_t *Y = nullptr, EY = E;
      const bf16* bias = nullptr;
      int act = 0, epi = EPI_LL;
      switch (w.kind) {
        case 0: X = a.xa; bias = L->attn_b; Y = a.qkv; break;
        case 1: X = a.att; bias = L->proj_b; res = a.xa; Y = a.xb; break;
        case 2: X = a.xb; bias = L->fc_b; Y = a.hb; act = 2 /*gelu_tanh*/; break;
        case 3: X = a.hb; bias = L->fc2_b; res = a.xb; Y = a.xa; EY = En; break;
        default: X = a.xa; epi = EPI_LMHEAD; break;
      }
      gemv_flow(cx, ring, lnr, w.ln_w != nullptr, epi, X, E, bias, res, E, Y, EY, w.N, w.K, act, gp, w.kind);
      if (w.kind == 0) {
        attention_flow(cx, L, cur_len, E, gp);
        merge_flow(cx, cur_len, E, gp);
        stamp(cx, ST_MERGE_DONE);
      }
    }
    const uint32_t gp = gs * nl1 + (uint32_t)a.n_layer;
    if (a.do_select && cta == 0) {
      select_flow(cx, ntiles_lm, gp, cur_len + 1, tag16((gs + 1u) * nl1));
      stamp(cx, ST_SELECT_DONE);
    }
  }
}

// ---- slab-tiled copy of a decode weight matrix W [N][K] and its bias (made once, when the weights are loaded): for CTA c, tile t, k slab s
// the block ((c * tpc + t) * nstg + s) * SLOT_BYTES holds the R rows x KS columns of that slab with the shared-memory row pitch
// (KS * 2 + 64 bytes) already applied, rows beyond N and the padding zeroed -- exactly the bytes of one ring slot, so the
// producer moves a slab with a single bulk copy and a CTA's whole share of the matrix is one linear range.
__global__ void __launch_bounds__(256) flow_repack_kernel(const bf16* __restrict__ W, const bf16* __restrict__ bias, uint8_t* __restrict__ T, int N,
                                                          int K, int ncta) {
  const Plan p = make_plan(N, K, blockIdx.x, ncta);
  const int tl = blockIdx.y / p.nstg, ks = blockIdx.y % p.nstg;
  if (blockIdx.y >= p.tpc * p.nstg) return;
  uint8_t* dst = T + ((int64_t)(blockIdx.x * p.tpc + tl) * p.nstg + ks) * SLOT_BYTES;
  const int row0 = (p.tile0 + tl) * p.R;
  const int vec_per_row = p.pitch / 16;                                   // 16-byte vectors per padded row
  for (int i = threadIdx.x; i < 16 * vec_per_row; i += 256) {
    const int r = i / vec_per_row, v = i % vec_per_row;
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (tl < p.ntile && r < p.R && row0 + r < N && v * 8 < p.KS)
      val = *reinterpret_cast<const uint4*>(W + (int64_t)(row0 + r) * K + (int64_t)ks * p.KS + v * 8);
    // the first two bytes of a row's 64-byte padding carry that output row's bias: the epilogue thread takes it from the slab
    // it has just multiplied (a separate global load sat behind ~20 MB of queued weight traffic and stalled the ring)
    if (bias != nullptr && tl < p.ntile && r < p.R && row0 + r < N && v * 8 == p.KS)
      val.x = (uint32_t)__bfloat16_as_ushort(bias[row0 + r]);
    if (i * 16 < SLOT_BYTES) *reinterpret_cast<uint4*>(dst + (int64_t)i * 16) = val;
  }
}

}  // namespace flow

size_t flow_tiled_bytes(int N, int K, int ncta) {
  const int rows_per_cta = (N + ncta - 1) / ncta, tpc = (rows_per_cta + 15) / 16;
  int ks = 32;
  for (int c : {1024, 768, 512, 256, 128, 64}) if (c <= K && K % c == 0) { ks = c; break; }
  return (size_t)ncta * tpc * (K / ks) * mega::SLOT_BYTES;
}

void launch_flow_repack(const bf16* W, const bf16* bias, void* T, int N, int K, int ncta, cudaStream_t st) {
  const int rows_per_cta = (N + ncta - 1) / ncta, tpc = (rows_per_cta + 15) / 16;
  int ks = 32;
  for (int c : {1024, 768, 512, 256, 128, 64}) if (c <= K && K % c == 0) { ks = c; break; }
  flow::flow_repack_kernel<<<dim3(ncta, tpc * (K / ks)), 256, 0, st>>>(W, bias, reinterpret_cast<uint8_t*>(T), N, K, ncta);
  count_launch();
}

// ---- host side
static int g_flow_ncta = 0;
static bool g_flow_realloc_ok = false;
static char g_flow_why[256] = "decode_flow_init not called";
const char* decode_flow_status() { return g_flow_why; }

cudaError_t decode_flow_init() {
  cudaError_t e = cudaFuncSetAttribute(flow::decode_flow_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, flow::FLOW_SMEM_BYTES);
  if (e != cudaSuccess) return e;
  bool realloc_attr_ok = cudaFuncSetAttribute(flow::decode_flow_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              flow::FLOW_SMEM_BYTES) == cudaSuccess;
  if (!realloc_attr_ok) cudaGetLastError();
  int dev = 0, nsm = 0, per_sm = 0, per_sm_realloc = 0, coop = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, flow::decode_flow_kernel<false>, flow::FLOW_THREADS, flow::FLOW_SMEM_BYTES);
  if (e != cudaSuccess) return e;
  if (!realloc_attr_ok || cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_realloc, flow::decode_flow_kernel<true>, flow::FLOW_THREADS_REALLOC,
                                                                         flow::FLOW_SMEM_BYTES) != cudaSuccess) {
    per_sm_realloc = 0;
    cudaGetLastError();
  }
  g_flow_ncta = (coop && per_sm >= 1) ? nsm : 0;
  g_flow_realloc_ok = coop && per_sm_realloc >= 1;
  snprintf(g_flow_why, sizeof(g_flow_why), "sms=%d coop=%d blocks_per_sm=%d (setmaxnreg variant: %d) smem=%d threads=%d -> ncta=%d", nsm,
           coop, per_sm, per_sm_realloc, flow::FLOW_SMEM_BYTES, flow::FLOW_THREADS, g_flow_ncta);
  return cudaSuccess;
}
bool decode_flow_realloc_supported() { return g_flow_realloc_ok; }
int decode_flow_ncta() { return g_flow_ncta; }
int decode_flow_max_splits() { return flow::MAXS; }
int decode_flow_partial_floats() { return mega::PSZ; }
// The widths the kernel takes, without asking the device.  A vector the consumers stage in shared memory (the hidden
// vector, and the c_fc output when I <= 2048) must be a power-of-two number of 8-value fragments, a multiple of 32 of them
// (stage_vector): 256, 512, 1024 or 2048 values.  A wider c_fc output is streamed per slab: I % KS_MAX == 0.
bool decode_flow_shape_ok(int H, int I, int head_dim, int max_batch, int window, bool rope) {
  auto staged = [](int n) { return n == 256 || n == 512 || n == 1024 || n == 2048; };
  return mega::NWC == 8 && head_dim == mega::D && staged(H) && (staged(I) || (I > 2 * mega::KS_MAX && I % mega::KS_MAX == 0)) &&
         max_batch >= 1 && max_batch <= 8 && window == 0 && !rope;      // (+ n_layer <= FLOW_MAX_LAYERS, checked at launch)
}
bool decode_flow_supported(int H, int I, int head_dim, int max_batch, int window, bool rope) {
  return g_flow_ncta > 0 && decode_flow_shape_ok(H, I, head_dim, max_batch, window, rope);
}
int decode_flow_max_keys() { return flow::MAXS * flow::ATT_BLKS * 32; }
int decode_flow_max_layers() { return flow::FLOW_MAX_LAYERS; }

cudaError_t launch_decode_flow(const FlowLaunch& m, cudaStream_t st) {
  flow::FlowArgs a{};
  a.layers = reinterpret_cast<const mega::Layer*>(m.layers_dev);
  a.n_layer = m.n_layer; a.B = m.B; a.H = m.H; a.I = m.I; a.n_head = m.n_head; a.n_kv = m.n_kv; a.qkv_cols = m.qkv_cols;
  a.vocab = m.vocab; a.tcap = m.tcap; a.n_positions = m.n_positions; a.ln_eps = m.ln_eps;
  a.wte = m.wte; a.wpe = m.wpe; a.lnf_w = m.lnf_w; a.lnf_b = m.lnf_b; a.lm_head = m.lm_head; a.lm_head_t = m.lm_head_t;
  a.x_plain = m.x_plain; a.logits = m.logits;
  a.xa = m.xa; a.xb = m.xb; a.qkv = m.qkv; a.att = m.att; a.hb = m.hb; a.part = m.part; a.amax = m.amax;
  a.state = m.state; a.params = m.params; a.seen = m.seen; a.next_ids = m.next_ids; a.out_ids = m.out_ids;
  a.nsteps = m.nsteps; a.step0 = m.step0; a.cur_len0 = m.cur_len0; a.first_plain = m.first_plain; a.do_select = m.do_select;
  a.l2_ahead = m.l2_ahead;
  a.dbg = m.dbg;
  if (m.n_layer > flow::FLOW_MAX_LAYERS) return cudaErrorInvalidValue;
  void* args[] = {&a};
  cudaError_t e;
  if (m.realloc)
    e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(flow::decode_flow_kernel<true>), dim3(g_flow_ncta), dim3(flow::FLOW_THREADS_REALLOC), args,
                                    flow::FLOW_SMEM_BYTES, st);
  else
    e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(flow::decode_flow_kernel<false>), dim3(g_flow_ncta), dim3(flow::FLOW_THREADS), args,
                                    flow::FLOW_SMEM_BYTES, st);
  count_launch();
  return e;
}

}  // namespace sv

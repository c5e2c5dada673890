// Large-M linear layer on the Hopper tensor cores: y[M,N] = epilogue(x[M,K] . w[N,K]^T + bias).
// Used by the ViT blocks, the adapter and the decoder prefill (every GEMM with M >= ~64 rows).
//
// Structure (one 128 x BN output tile per CTA, warp-specialised, 288 threads):
//   warp 8    : TMA producer - cp.async.bulk.tensor.2d loads of the 128x64 activation tile and the
//               BNx64 weight tile (both K-major, 128-byte swizzle) into a STAGES-deep smem ring,
//               completion signalled on per-stage "full" mbarriers (expect_tx).
//   warps 0-7 : two consumer warpgroups, one per 64-row half of the tile.  Each issues 4 x wgmma.mma_async
//               (64 x BN x 16, bf16 in / fp32 accumulate in registers) per stage straight from the swizzled
//               tiles, keeps one stage of MMAs in flight and releases the stage before it on its "empty"
//               mbarrier.  Epilogue: the fp32 tile is staged in the (then idle) ring, and every thread applies
//               bias / activation / residual with the reference's bf16 rounding points to 8 consecutive
//               columns of a row, 16-byte global stores.
// Rows beyond M and weight rows beyond N are zero-filled by TMA (OOB fill) and masked at the store.
// EPI = kEpiLogprob (the fused lm_head log-likelihood of sv_score.cu) replaces the store: straight from the accumulator
// registers, every logit is rounded to bf16 and each (row, N-tile) writes its (max, sum of exp) pair and, in the tile that
// holds it, the target's logit; the [M, N] logits never reach global memory and N needs no alignment.
// Every mbarrier wait is bounded: a protocol bug traps (CUDA error) instead of hanging the GPU.
#include <cuda.h>

#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>

#include "sv_kernels.h"

namespace sv {

namespace wg {

constexpr int BM = 128;                // two warpgroups x 64 rows
constexpr int BK = 64;                 // 64 bf16 = 128 bytes = one swizzle row
constexpr int kConsumers = 256;        // warps 0-7
constexpr int kThreads = kConsumers + 32;

template <int BN> struct Cfg {
  static constexpr int kStageBytes = BM * BK * 2 + BN * BK * 2;
  static constexpr int kStages = (BN == 128) ? 3 : 4;                          // ~96 KB per CTA: two CTAs share an SM
  static constexpr int kOutStride = BN + 8;                                     // fp32 staging row; +8 spreads the banks
  static_assert(BM * kOutStride * 4 <= kStages * kStageBytes, "epilogue staging tile must fit in the ring");
  static constexpr int kBarBytes = 256;
  static constexpr int kSmemBytes = kStages * kStageBytes + kBarBytes + 1024;   // +1024: manual 1 KiB alignment
};

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
    if (it > (1u << 20)) __trap();   // ~seconds: pipeline protocol broken -> fail loudly, never hang
  }
}
SV_DEVINL void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y) : "memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (PTX "matrix descriptor", sm_90 wgmma format):
// start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major) | SBO>>4 [32,46) = 1024 B between
// 8-row groups | layout_type=1 (SWIZZLE_128B) [62,64).
SV_DEVINL uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

SV_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
SV_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> SV_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R> SV_DEVINL void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define SV_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])

// D[64 x BN] += A[64 x 16] * B[BN x 16]^T, bf16 -> fp32, both operands K-major in shared memory.
// Fragment of D: d[i] is row 16 * (warp % 4) + lane / 4 + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (lane % 4) + i % 2.
SV_DEVINL void wgmma_bf16(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"   // scale-d = true: accumulate into d
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : SV_ACC8(0), SV_ACC8(8), SV_ACC8(16), SV_ACC8(24)
      : "l"(a_desc), "l"(b_desc));
}
SV_DEVINL void wgmma_bf16(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"   // scale-d = true: accumulate into d
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : SV_ACC8(0), SV_ACC8(8), SV_ACC8(16), SV_ACC8(24), SV_ACC8(32), SV_ACC8(40), SV_ACC8(48), SV_ACC8(56)
      : "l"(a_desc), "l"(b_desc));
}
#undef SV_ACC8

// kEpiLogits: the plain epilogue for any N (columns masked one by one), so that resident logits carry exactly the bf16
// values the kEpiLogprob epilogue sees
constexpr int kEpiLinear = 0, kEpiLogprob = 1, kEpiLogits = 2;

template <int BN, int EPI = kEpiLinear>
__global__ void __launch_bounds__(kThreads, 2) linear_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x,
                                                                   const __grid_constant__ CUtensorMap tmap_w,
                                                                   const bf16* __restrict__ bias,
                                                                   const bf16* __restrict__ res, bf16* __restrict__ Y,
                                                                   int M, int N, int K, int act,
                                                                   const int32_t* __restrict__ targets,
                                                                   float2* __restrict__ part, float* __restrict__ tgt_logit) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bars = base + C::kStages * C::kStageBytes;
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (C::kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_blk = blockIdx.x, m_blk = blockIdx.y;
  const int nk = K / BK;

  if (threadIdx.x == kConsumers) {
    for (int s = 0; s < C::kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumers); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
  }
  __syncthreads();

  if (warp == kConsumers / 32) {   // producer; the consumers wait for every load it issues, so it may leave early
    if (lane == 0) {
      for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % C::kStages;
        const uint32_t ph = (uint32_t)(kb / C::kStages) & 1u;
        mbar_wait(empty_bar(s), ph ^ 1u);
        const uint32_t a_smem = base + s * C::kStageBytes;
        const uint32_t b_smem = a_smem + BM * BK * 2;
        mbar_expect_tx(full_bar(s), C::kStageBytes);
        tma_load_2d(a_smem, &tmap_x, full_bar(s), kb * BK, m_blk * BM);
        tma_load_2d(b_smem, &tmap_w, full_bar(s), kb * BK, n_blk * BN);
      }
    }
    return;
  }

  const int half = warp >> 2;            // warpgroup = 64-row half of the tile
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  fence_acc(acc);
  for (int kb = 0; kb < nk; ++kb) {
    const int s = kb % C::kStages;
    mbar_wait(full_bar(s), (uint32_t)(kb / C::kStages) & 1u);
    const uint32_t a_smem = base + s * C::kStageBytes + half * 64 * BK * 2;   // 8 KB: keeps the 1 KiB swizzle alignment
    const uint32_t b_smem = base + s * C::kStageBytes + BM * BK * 2;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)   // advance 16 elements (32 bytes) along K inside the 128-byte swizzle row
      wgmma_bf16(acc, make_sw128_desc(a_smem + k * 32), make_sw128_desc(b_smem + k * 32));
    wgmma_commit();
    wgmma_wait<1>();                     // the previous stage's MMAs are done: hand that stage back to the producer
    if (kb > 0) mbar_arrive(empty_bar((kb - 1) % C::kStages));
  }
  wgmma_wait<0>();
  fence_acc(acc);

  if constexpr (EPI == kEpiLogprob) {
    // d[i] is row r0 + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (lane % 4) + i % 2: the 4 lanes of a quad hold a row's BN columns
    const int r0 = m_blk * BM + half * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = n_blk * BN + 2 * (lane & 3);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      const int col = c0 + 8 * (i >> 2) + (i & 1);
      acc[i] = col < N ? bf16_round(acc[i]) : -INFINITY;          // HF: lm_head output is bf16
      mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], acc[i]);
    }
    mx[0] = quad_max(mx[0]);
    mx[1] = quad_max(mx[1]);
    float se[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) se[(i >> 1) & 1] += expf(acc[i] - mx[(i >> 1) & 1]);
    se[0] = quad_sum(se[0]);
    se[1] = quad_sum(se[1]);
    int tg0 = r0 < M ? targets[r0] : -1, tg1 = r0 + 8 < M ? targets[r0 + 8] : -1;
    tg0 = tg0 < N ? tg0 : -1;                                       // a column past N (-inf) is no target
    tg1 = tg1 < N ? tg1 : -1;
    float tv0 = 0.f, tv1 = 0.f;
    bool hit0 = false, hit1 = false;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      const int col = c0 + 8 * (i >> 2) + (i & 1);
      if ((i >> 1) & 1) { if (col == tg1) { tv1 = acc[i]; hit1 = true; } }
      else if (col == tg0) { tv0 = acc[i]; hit0 = true; }
    }
    if (hit0) tgt_logit[r0] = tv0;
    if (hit1) tgt_logit[r0 + 8] = tv1;
    if ((lane & 3) == 0) {
      if (r0 < M) part[(int64_t)r0 * gridDim.x + n_blk] = make_float2(mx[0], se[0]);
      if (r0 + 8 < M) part[(int64_t)(r0 + 8) * gridDim.x + n_blk] = make_float2(mx[1], se[1]);
    }
    return;
  }

  // both warpgroups are done reading the ring before either overwrites it with the fp32 tile
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
  float* tile = reinterpret_cast<float*>(smem_raw + (base - raw));
  {
    const int r0 = half * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int r = r0 + 8 * ((i >> 1) & 1), c = c0 + 8 * (i >> 2);
      *reinterpret_cast<float2*>(tile + r * C::kOutStride + c) = make_float2(acc[i], acc[i + 1]);
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
  const bool has_res = res != nullptr;
#pragma unroll 1
  for (int c = threadIdx.x; c < BM * BN / 8; c += kConsumers) {
    const int r = c / (BN / 8), c8 = (c % (BN / 8)) * 8;
    const int row = m_blk * BM + r, col = n_blk * BN + c8;
    if constexpr (EPI == kEpiLogits) {
      if (row >= M || col >= N) continue;
    } else {
      if (row >= M || col + 8 > N) continue;
    }
    const float4 lo = *reinterpret_cast<const float4*>(tile + r * C::kOutStride + c8);
    const float4 hi = *reinterpret_cast<const float4*>(tile + r * C::kOutStride + c8 + 4);
    const float a[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    float bv[8], rv[8], o[8];
    if (bias) unpack8(ldg_cached(bias + col), bv);
    else { for (int j = 0; j < 8; ++j) bv[j] = 0.f; }
    if (has_res) unpack8(ldg_cached(res + (int64_t)row * N + col), rv);
    else { for (int j = 0; j < 8; ++j) rv[j] = 0.f; }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = epilogue_elem(a[j], bv[j], act, has_res, rv[j]);
    if constexpr (EPI == kEpiLogits) {
      for (int j = 0; j < 8 && col + j < N; ++j) Y[(int64_t)row * N + col + j] = __float2bfloat16_rn(o[j]);
    } else {
      *reinterpret_cast<uint4*>(Y + (int64_t)row * N + col) = pack8(o);
    }
  }
}

// ---- host side: tensor maps through the driver entry point (no link-time libcuda dependency)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 2-D bf16 row-major [rows, cols] tensor, box = [box_rows, 64 cols], 128-byte swizzle, zero OOB fill.
static bool make_map(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

struct MapKey {
  const void* p; int64_t rows, cols; int box;
  bool operator<(const MapKey& o) const { return std::tie(p, rows, cols, box) < std::tie(o.p, o.rows, o.cols, o.box); }
};
static std::mutex g_map_mu;
static std::map<MapKey, CUtensorMap> g_maps;

static bool cached_map(CUtensorMap* out, const void* ptr, int64_t rows, int64_t cols, int box_rows) {
  std::lock_guard<std::mutex> lk(g_map_mu);
  MapKey k{ptr, rows, cols, box_rows};
  auto it = g_maps.find(k);
  if (it == g_maps.end()) {
    CUtensorMap m;
    if (!make_map(&m, ptr, rows, cols, box_rows)) return false;
    if (g_maps.size() > 4096) g_maps.clear();
    it = g_maps.emplace(k, m).first;
  }
  *out = it->second;
  return true;
}

template <int BN, int EPI = kEpiLinear>
static cudaError_t launch(const bf16* x, const bf16* w, const bf16* bias, const bf16* res, bf16* y, int M, int N,
                          int K, int act, cudaStream_t st, const int32_t* targets = nullptr, float2* part = nullptr,
                          float* tgt_logit = nullptr) {
  CUtensorMap mx, mw;
  if (!cached_map(&mx, x, M, K, BM) || !cached_map(&mw, w, N, K, BN)) return cudaErrorInvalidValue;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(linear_wgmma_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg<BN>::kSmemBytes);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  linear_wgmma_kernel<BN, EPI><<<grid, kThreads, Cfg<BN>::kSmemBytes, st>>>(mx, mw, bias, res, y, M, N, K, act, targets,
                                                                             part, tgt_logit);
  count_launch();
  return cudaGetLastError();
}

}  // namespace wg

bool wgmma_supported(int M, int N, int K) { return M >= 1 && N >= 8 && (N % 8) == 0 && K >= 64 && (K % 64) == 0; }

cudaError_t launch_linear_wgmma(const bf16* x, const bf16* w, const bf16* bias, const bf16* res, bf16* y, int M, int N,
                                int K, int act, cudaStream_t st) {
  if (!wgmma_supported(M, N, K)) return cudaErrorInvalidValue;
  // Tile-count heuristic for the small-M GEMMs of this path (M = 257..2072): every CTA pays a fixed cost (launch,
  // pipeline fill, epilogue), so never spill into a second wave if a wider tile avoids it: BN=64 while its tile count
  // fits one wave of SMs (two CTAs per SM with the 96 KB ring), else BN=128.
  const int mt = (M + wg::BM - 1) / wg::BM;
  static int nsm = 0;
  if (nsm == 0) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev); if (nsm <= 0) nsm = 132; }
  const bool wide = (N % 128 == 0) && ((int64_t)mt * ((N + 63) / 64) > (int64_t)nsm * 2);
  return wide ? wg::launch<128>(x, w, bias, res, y, M, N, K, act, st)
              : wg::launch<64>(x, w, bias, res, y, M, N, K, act, st);
}

int lm_logprob_ntiles(int N) { return (N + 127) / 128; }

cudaError_t launch_lm_logits(const bf16* x, const bf16* w, bf16* y, int M, int N, int K, cudaStream_t st) {
  if (M < 1 || N < 1 || K < 64 || K % 64) return cudaErrorInvalidValue;
  return wg::launch<128, wg::kEpiLogits>(x, w, nullptr, nullptr, y, M, N, K, /*act=*/0, st);
}

cudaError_t launch_lm_logprob_partials(const bf16* x, const bf16* w, const int32_t* targets, float2* part, float* tgt_logit,
                                       int M, int N, int K, cudaStream_t st) {
  if (M < 1 || N < 1 || K < 64 || K % 64) return cudaErrorInvalidValue;
  return wg::launch<128, wg::kEpiLogprob>(x, w, nullptr, nullptr, nullptr, M, N, K, /*act=*/0, st, targets, part, tgt_logit);
}

}  // namespace sv

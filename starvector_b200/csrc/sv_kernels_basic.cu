// Elementwise / normalisation / layout kernels of the im2svg path (all HBM-bound, bf16 storage,
// fp32 math).  Reference semantics are cited per kernel; rounding points follow DESIGN.md.
#include "sv_kernels.h"
#include "sv_sample.cuh"

namespace sv {

thread_local int64_t* g_launch_counter = nullptr;

// ------------------------------------------------------------------------------------------
// LayerNorm over the last dim (clip_model.py:117-124; nn.LayerNorm in GPTBigCode blocks):
// fp32 statistics (two-pass), y = bf16((x-mean)*rstd*w + b).
__global__ void __launch_bounds__(128) layernorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                        const bf16* __restrict__ b, bf16* __restrict__ y, int cols,
                                                        float eps, int64_t x_row_stride) {
  __shared__ float sm[4];
  const bf16* xr = x + (int64_t)blockIdx.x * x_row_stride;
  bf16* yr = y + (int64_t)blockIdx.x * cols;
  const int nvec = cols >> 3;
  float s = 0.f;
  for (int i = threadIdx.x; i < nvec; i += 128) {
    float f[8];
    unpack8(ldg_cached(xr + i * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += f[j];
  }
  const float mean = block_sum<128>(s, sm) / (float)cols;
  float q = 0.f;
  for (int i = threadIdx.x; i < nvec; i += 128) {
    float f[8];
    unpack8(ldg_cached(xr + i * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { float d = f[j] - mean; q += d * d; }
  }
  const float var = block_sum<128>(q, sm) / (float)cols;
  const float rstd = 1.0f / sqrtf(var + eps);
  for (int i = threadIdx.x; i < nvec; i += 128) {
    float f[8], wf[8], bf[8];
    unpack8(ldg_cached(xr + i * 8), f);
    unpack8(ldg_cached(w + i * 8), wf);
    unpack8(ldg_cached(b + i * 8), bf);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = (f[j] - mean) * rstd * wf[j] + bf[j];
    *reinterpret_cast<uint4*>(yr + i * 8) = pack8(f);
  }
}

void launch_layernorm(const bf16* x, const bf16* w, const bf16* b, bf16* y, int rows, int cols, float eps,
                      int64_t x_row_stride, cudaStream_t st) {
  if (rows <= 0) return;
  layernorm_kernel<<<rows, 128, 0, st>>>(x, w, b, y, cols, eps, x_row_stride);
  count_launch();
}

// ------------------------------------------------------------------------------------------
__global__ void convert_kernel(const void* __restrict__ src, int dtype, bf16* __restrict__ dst, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float v = dtype == 1 ? reinterpret_cast<const float*>(src)[i]
                         : __half2float(reinterpret_cast<const __half*>(src)[i]);
    dst[i] = __float2bfloat16_rn(v);
  }
}
void launch_convert_to_bf16(const void* src, int dtype, bf16* dst, int64_t n, cudaStream_t st) {
  if (n <= 0) return;
  int blocks = (int)((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256);
  convert_kernel<<<blocks, 256, 0, st>>>(src, dtype, dst, n);
  count_launch();
}

__global__ void pad_rows_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int src_cols, int dst_cols) {
  const int r = blockIdx.x;
  for (int c = threadIdx.x; c < dst_cols; c += blockDim.x)
    dst[(int64_t)r * dst_cols + c] = c < src_cols ? src[(int64_t)r * src_cols + c] : __float2bfloat16_rn(0.f);
}
void launch_pad_rows(const bf16* src, bf16* dst, int rows, int src_cols, int dst_cols, cudaStream_t st) {
  pad_rows_kernel<<<rows, 128, 0, st>>>(src, dst, src_cols, dst_cols);
  count_launch();
}

// ------------------------------------------------------------------------------------------
// Patch extraction for conv1 (clip_model.py:174,182): stride == kernel, so the conv is a GEMM over
// [B*G*G, 3*p*p] patches; K is zero-padded to a multiple of 64 for the TMA/UMMA tile.
__global__ void im2col_kernel(const bf16* __restrict__ px, bf16* __restrict__ out, int image, int patch, int kpad) {
  const int g = image / patch;
  const int np = g * g;
  const int b = blockIdx.x / np, pi = blockIdx.x % np;
  const int py = pi / g, pxi = pi % g;
  const int pp = patch * patch;
  for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
    bf16 v = __float2bfloat16_rn(0.f);
    if (k < 3 * pp) {
      int c = k / pp, r = k % pp, iy = r / patch, ix = r % patch;
      v = px[(((int64_t)b * 3 + c) * image + (py * patch + iy)) * image + (pxi * patch + ix)];
    }
    out[(int64_t)blockIdx.x * kpad + k] = v;
  }
}
void launch_im2col(const bf16* pixels, bf16* patches, int batch, int image, int patch, int kpad, cudaStream_t st) {
  int g = image / patch;
  im2col_kernel<<<batch * g * g, 128, 0, st>>>(pixels, patches, image, patch, kpad);
  count_launch();
}

// cat([class_embedding, patches]) + positional_embedding (clip_model.py:185-186); bf16 add.
__global__ void vit_assemble_kernel(const bf16* __restrict__ pe, const bf16* __restrict__ cls,
                                    const bf16* __restrict__ pos, bf16* __restrict__ x, int np, int width) {
  const int off = cls ? 1 : 0;                     // SigLIP has no class token (modeling_siglip.py:178-187)
  const int q = np + off;
  const int b = blockIdx.x / q, t = blockIdx.x % q;
  const bf16* src = (cls && t == 0) ? cls : pe + ((int64_t)b * np + (t - off)) * width;
  for (int c = threadIdx.x; c < width; c += blockDim.x)
    x[(int64_t)blockIdx.x * width + c] =
        __float2bfloat16_rn(__bfloat162float(src[c]) + __bfloat162float(pos[(int64_t)t * width + c]));
}
void launch_vit_assemble(const bf16* pe, const bf16* cls, const bf16* pos, bf16* x, int batch, int np, int width,
                         cudaStream_t st) {
  vit_assemble_kernel<<<batch * (np + (cls ? 1 : 0)), 128, 0, st>>>(pe, cls, pos, x, np, width);
  count_launch();
}

// V^T per (image, head): vt[b][h][d][l] = qkv[b*L+l][2W + h*64 + d], zero for l >= L (keeps P.V clean).
__global__ void vit_transpose_v_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ vt, int seq, int heads,
                                       int seq_pad) {
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int W = heads * 64;
  const int total = 64 * seq_pad;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    int d = i / seq_pad, l = i % seq_pad;
    bf16 v = __float2bfloat16_rn(0.f);
    if (l < seq) v = qkv[((int64_t)b * seq + l) * (3 * W) + 2 * W + h * 64 + d];
    vt[((int64_t)blockIdx.x * 64 + d) * seq_pad + l] = v;
  }
}
void launch_vit_transpose_v(const bf16* qkv, bf16* vt, int batch, int seq, int heads, int seq_pad, cudaStream_t st) {
  vit_transpose_v_kernel<<<batch * heads, 256, 0, st>>>(qkv, vt, seq, heads, seq_pad);
  count_launch();
}

// ------------------------------------------------------------------------------------------
// Adapter norm, LayerNorm([Q,H]) flavour (adapters/adapter.py:25-26,37): statistics over the whole
// [Q,H] slab of one image, elementwise affine of the same shape.  Two kernels: per-chunk partial
// (sum, sumsq) then normalise (each block recombines the 64 partials in double).
constexpr int kSlabChunks = 64;
__global__ void __launch_bounds__(256) slab_stats_kernel(const bf16* __restrict__ z, float* __restrict__ partial,
                                                         int64_t slab) {
  __shared__ float sm[8];
  const int b = blockIdx.y, c = blockIdx.x;
  const int64_t per = (slab + kSlabChunks - 1) / kSlabChunks;
  const int64_t lo = c * per, hi = (lo + per < slab) ? lo + per : slab;
  const bf16* zr = z + (int64_t)b * slab;
  float s = 0.f, q = 0.f;
  for (int64_t i = lo + threadIdx.x; i < hi; i += 256) {
    float v = __bfloat162float(zr[i]);
    s += v; q += v * v;
  }
  s = block_sum<256>(s, sm);
  q = block_sum<256>(q, sm);
  if (threadIdx.x == 0) {
    partial[((int64_t)b * kSlabChunks + c) * 2 + 0] = s;
    partial[((int64_t)b * kSlabChunks + c) * 2 + 1] = q;
  }
}
__global__ void __launch_bounds__(256) slab_norm_kernel(const bf16* __restrict__ z, const bf16* __restrict__ w,
                                                        const bf16* __restrict__ bb, bf16* __restrict__ y,
                                                        const float* __restrict__ partial, int64_t slab, float eps) {
  __shared__ float stat[2];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    double s = 0.0, q = 0.0;
    for (int c = 0; c < kSlabChunks; ++c) {
      s += (double)partial[((int64_t)b * kSlabChunks + c) * 2 + 0];
      q += (double)partial[((int64_t)b * kSlabChunks + c) * 2 + 1];
    }
    double mean = s / (double)slab;
    double var = q / (double)slab - mean * mean;
    if (var < 0.0) var = 0.0;
    stat[0] = (float)mean;
    stat[1] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  const float mean = stat[0], rstd = stat[1];
  const int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 8;
  if (i >= slab) return;
  float f[8], wf[8], bf[8];
  unpack8(ldg_cached(z + (int64_t)b * slab + i), f);
  unpack8(ldg_cached(w + i), wf);
  unpack8(ldg_cached(bb + i), bf);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = (f[j] - mean) * rstd * wf[j] + bf[j];
  *reinterpret_cast<uint4*>(y + (int64_t)b * slab + i) = pack8(f);
}
void launch_slab_layernorm(const bf16* z, const bf16* w, const bf16* b, bf16* y, float* partial, int batch,
                           int64_t slab, float eps, cudaStream_t st) {
  slab_stats_kernel<<<dim3(kSlabChunks, batch), 256, 0, st>>>(z, partial, slab);
  int64_t nvec = slab / 8;
  slab_norm_kernel<<<dim3((unsigned)((nvec + 255) / 256), batch), 256, 0, st>>>(z, w, b, y, partial, slab, eps);
  count_launch(2);
}

// Adapter norm, BatchNorm1d(Q) eval flavour (adapter.py:27-28): channel = token index q.
__global__ void batchnorm_tokens_kernel(const bf16* __restrict__ z, const bf16* __restrict__ w,
                                        const bf16* __restrict__ b, const bf16* __restrict__ rmean,
                                        const bf16* __restrict__ rvar, bf16* __restrict__ y, int q, int h, float eps) {
  const int t = blockIdx.x % q;
  const float mean = __bfloat162float(rmean[t]);
  const float invstd = 1.0f / sqrtf(__bfloat162float(rvar[t]) + eps);
  const float ww = __bfloat162float(w[t]), bb = __bfloat162float(b[t]);
  for (int c = threadIdx.x; c < h; c += blockDim.x) {
    float v = __bfloat162float(z[(int64_t)blockIdx.x * h + c]);
    y[(int64_t)blockIdx.x * h + c] = __float2bfloat16_rn((v - mean) * invstd * ww + bb);
  }
}
void launch_batchnorm_tokens(const bf16* z, const bf16* w, const bf16* b, const bf16* rmean, const bf16* rvar, bf16* y,
                             int batch, int q, int h, float eps, cudaStream_t st) {
  batchnorm_tokens_kernel<<<batch * q, 128, 0, st>>>(z, w, b, rmean, rvar, y, q, h, eps);
  count_launch();
}

// ------------------------------------------------------------------------------------------
// inputs_embeds = cat([visual, wte(prompt)]) (starvector_base.py:218-219) + wpe[position]
// (GPTBigCodeModel.forward: hidden = inputs_embeds + position_embeds), bf16 add.  Row t sits at position pos0 + t
// (pos0 > 0: a scoring chunk appended to a filled cache); prompt row b starts at prompt + b * id_stride.
__global__ void embed_prefix_kernel(const bf16* __restrict__ visual, const int32_t* __restrict__ prompt,
                                    const bf16* __restrict__ wte, const bf16* __restrict__ wpe, bf16* __restrict__ x,
                                    int q, int p, int h, int vocab, int pos0, int id_stride) {
  const int t0 = q + p;
  const int b = blockIdx.x / t0, t = blockIdx.x % t0;
  const bf16* src;
  if (t < q) {
    src = visual + ((int64_t)b * q + t) * h;
  } else {
    int id = prompt[(int64_t)b * id_stride + (t - q)];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    src = wte + (int64_t)id * h;
  }
  const bf16* pos = wpe ? wpe + (int64_t)(pos0 + t) * h : nullptr;   // RoPE models (StarCoder2) have no learned positions
  for (int c = threadIdx.x * 8; c < h; c += blockDim.x * 8) {
    float a[8], d[8];
    unpack8(ldg_cached(src + c), a);
    if (pos) {
      unpack8(ldg_cached(pos + c), d);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += d[j];
    }
    *reinterpret_cast<uint4*>(x + (int64_t)blockIdx.x * h + c) = pack8(a);
  }
}
void launch_embed_prefix(const bf16* visual, const int32_t* prompt_ids, const bf16* wte, const bf16* wpe, bf16* x,
                         int batch, int q, int p, int h, int vocab, int pos0, int id_stride, cudaStream_t st) {
  embed_prefix_kernel<<<batch * (q + p), 128, 0, st>>>(visual, prompt_ids, wte, wpe, x, q, p, h, vocab, pos0, id_stride);
  count_launch();
}

// ROWS: the session variant (position of row b = rows->row_len[b]); the plain kernels instantiate ROWS = false.
template <bool ROWS>
SV_DEVINL void embed_tokens_body(const int32_t* __restrict__ ids, const bf16* __restrict__ wte,
                                 const bf16* __restrict__ wpe, const GenState* __restrict__ state,
                                 const RowState* __restrict__ rows, bf16* __restrict__ x, int h, int vocab,
                                 int n_positions) {
  const int b = blockIdx.x;
  int id = ids[b];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  int pos = ROWS ? rows->row_len[b] : state->cur_len;
  pos = pos >= n_positions ? n_positions - 1 : pos;
  const bf16* src = wte + (int64_t)id * h;
  const bf16* pe = wpe ? wpe + (int64_t)pos * h : nullptr;
  for (int c = threadIdx.x * 8; c < h; c += blockDim.x * 8) {
    float a[8], d[8];
    unpack8(ldg_cached(src + c), a);
    if (pe) {
      unpack8(ldg_cached(pe + c), d);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += d[j];
    }
    *reinterpret_cast<uint4*>(x + (int64_t)b * h + c) = pack8(a);
  }
}
__global__ void embed_tokens_kernel(const int32_t* __restrict__ ids, const bf16* __restrict__ wte,
                                    const bf16* __restrict__ wpe, const GenState* __restrict__ state,
                                    bf16* __restrict__ x, int h, int vocab, int n_positions) {
  embed_tokens_body<false>(ids, wte, wpe, state, nullptr, x, h, vocab, n_positions);
}
__global__ void embed_tokens_rows_kernel(const int32_t* __restrict__ ids, const bf16* __restrict__ wte,
                                         const bf16* __restrict__ wpe, const RowState* __restrict__ rows,
                                         bf16* __restrict__ x, int h, int vocab, int n_positions) {
  embed_tokens_body<true>(ids, wte, wpe, nullptr, rows, x, h, vocab, n_positions);
}
void launch_embed_tokens(const int32_t* ids, const bf16* wte, const bf16* wpe, const GenState* state, bf16* x,
                         int batch, int h, int vocab, int n_positions, cudaStream_t st, const RowState* rows) {
  if (rows) embed_tokens_rows_kernel<<<batch, 128, 0, st>>>(ids, wte, wpe, rows, x, h, vocab, n_positions);
  else embed_tokens_kernel<<<batch, 128, 0, st>>>(ids, wte, wpe, state, x, h, vocab, n_positions);
  count_launch();
}

// ------------------------------------------------------------------------------------------
// KV cache write.  Layout per layer: K [max_batch][n_kv][tcap][d] (rows), V^T [max_batch][n_kv][d][tcap]
// (so the P.V tensor-core operand is a contiguous 16-byte load per lane; see sv_attention.cu).
// The reference re-allocates and copies the whole cache every step (torch.cat, SURVEY.md K15).
__global__ void kv_write_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ kcache, bf16* __restrict__ vtcache,
                                const GenState* __restrict__ state, int t0, int seq, int q_cols, int n_kv, int d, int tcap) {
  const int b = blockIdx.y, ts = blockIdx.x;
  const int t = (state ? state->cur_len : t0) + ts;
  if (t >= tcap) return;
  const int cols = q_cols + 2 * n_kv * d;
  const bf16* row = qkv + ((int64_t)b * seq + ts) * cols;
  for (int i = threadIdx.x; i < n_kv * d; i += blockDim.x) {
    int kvh = i / d, dim = i % d;
    kcache[(((int64_t)b * n_kv + kvh) * tcap + t) * d + dim] = row[q_cols + i];
    vtcache[(((int64_t)b * n_kv + kvh) * d + dim) * tcap + t] = row[q_cols + n_kv * d + i];
  }
}
void launch_kv_scatter(const bf16* qkv, bf16* kcache, bf16* vtcache, int batch, int seq, int q_cols, int n_kv, int d,
                       int tcap, int t0, cudaStream_t st) {
  kv_write_kernel<<<dim3(seq, batch), 128, 0, st>>>(qkv, kcache, vtcache, nullptr, t0, seq, q_cols, n_kv, d, tcap);
  count_launch();
}
// Session variant of the decode-step append: row b's K/V go to position rows->row_len[b].
__global__ void kv_append_rows_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ kcache, bf16* __restrict__ vtcache,
                                      const RowState* __restrict__ rows, int q_cols, int n_kv, int d, int tcap) {
  const int b = blockIdx.y;
  const int t = rows->row_len[b];
  if (t >= tcap) return;
  const int cols = q_cols + 2 * n_kv * d;
  const bf16* row = qkv + (int64_t)b * cols;
  for (int i = threadIdx.x; i < n_kv * d; i += blockDim.x) {
    int kvh = i / d, dim = i % d;
    kcache[(((int64_t)b * n_kv + kvh) * tcap + t) * d + dim] = row[q_cols + i];
    vtcache[(((int64_t)b * n_kv + kvh) * d + dim) * tcap + t] = row[q_cols + n_kv * d + i];
  }
}
void launch_kv_append(const bf16* qkv, bf16* kcache, bf16* vtcache, const GenState* state, int batch, int q_cols,
                      int n_kv, int d, int tcap, cudaStream_t st, const RowState* rows) {
  if (rows) kv_append_rows_kernel<<<dim3(1, batch), 128, 0, st>>>(qkv, kcache, vtcache, rows, q_cols, n_kv, d, tcap);
  else kv_write_kernel<<<dim3(1, batch), 128, 0, st>>>(qkv, kcache, vtcache, state, 0, 1, q_cols, n_kv, d, tcap);
  count_launch();
}

// Beam search cache reorder (HF `_reorder_cache` / `Cache.reorder_cache`, generation/utils.py beam loop): image row r of
// the destination takes the first `len` tokens of source row idx[r].  One layer at a time through a scratch layer
// (gather), then copied back with idx == nullptr (identity).  grid = (n_kv * 2, rows); 16-byte vectors.
__global__ void kv_gather_kernel(const bf16* __restrict__ ksrc, const bf16* __restrict__ vsrc, bf16* __restrict__ kdst,
                                 bf16* __restrict__ vdst, const int32_t* __restrict__ idx, int n_kv, int tcap, int d,
                                 int len) {
  const int r = blockIdx.y, kvh = blockIdx.x >> 1, which = blockIdx.x & 1;
  const int sr = idx ? idx[r] : r;
  if (which == 0) {            // K rows: contiguous [len][d]
    const uint4* s = reinterpret_cast<const uint4*>(ksrc + ((int64_t)sr * n_kv + kvh) * tcap * d);
    uint4* t = reinterpret_cast<uint4*>(kdst + ((int64_t)r * n_kv + kvh) * tcap * d);
    const int n = len * d / 8;
    for (int i = threadIdx.x; i < n; i += blockDim.x) t[i] = s[i];
  } else {                     // V^T: d rows of `len` (rounded up to 8) keys
    const int per = (len + 7) / 8;
    for (int i = threadIdx.x; i < d * per; i += blockDim.x) {
      const int dim = i / per, c = i % per;
      const int64_t off = (((int64_t)0 * n_kv + kvh) * d + dim) * tcap + c * 8;
      *reinterpret_cast<uint4*>(vdst + ((int64_t)r * n_kv * d) * tcap + off) =
          *reinterpret_cast<const uint4*>(vsrc + ((int64_t)sr * n_kv * d) * tcap + off);
    }
  }
}
void launch_kv_gather(const bf16* ksrc, const bf16* vsrc, bf16* kdst, bf16* vdst, const int32_t* idx, int rows, int n_kv,
                      int tcap, int d, int len, cudaStream_t st) {
  kv_gather_kernel<<<dim3(n_kv * 2, rows), 256, 0, st>>>(ksrc, vsrc, kdst, vdst, idx, n_kv, tcap, d, len);
  count_launch();
}

__global__ void gather_rows_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int seq, int row, int h) {
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < h; c += blockDim.x) y[(int64_t)b * h + c] = x[((int64_t)b * seq + row) * h + c];
}
void launch_gather_rows(const bf16* x, bf16* y, int batch, int seq, int row, int h, cudaStream_t st) {
  gather_rows_kernel<<<batch, 256, 0, st>>>(x, y, seq, row, h);
  count_launch();
}

__global__ void logits_to_float_kernel(const bf16* __restrict__ l, float* __restrict__ o, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = __bfloat162float(l[i]);
}
void launch_logits_to_float(const bf16* logits, float* out, int64_t n, cudaStream_t st) {
  logits_to_float_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(logits, out, n);
  count_launch();
}

// ------------------------------------------------------------------------------------------
// Token selection = the body of HF `_sample` (SURVEY.md App. B.3-6): fp32 cast of the bf16 logits,
// repetition penalty over generated ids, argmax with lowest-index tie-break, EOS->pad for finished
// rows, append, EOS / '</svg>' stop bookkeeping.  One block per batch row.
struct ArgMax { float v; int i; };
SV_DEVINL ArgMax better(ArgMax a, ArgMax b) { return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a; }

template <bool ROWS>
SV_DEVINL void select_greedy_body(const bf16* __restrict__ logits, int vocab, GenState* state,
                                  const GenParamsDev* __restrict__ p, uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                                  RowState* rows, uint32_t row_mask, int advance_len) {
  const int b = blockIdx.x;
  if constexpr (ROWS) {
    if (!session_row_selects(rows, row_mask, b)) return;
  } else {
    if (state->done) return;
  }
  __shared__ ArgMax sm[32];
  const bf16* lr = logits + (int64_t)b * vocab;
  const uint8_t* sr = seen + (int64_t)b * vocab;
  const float rp = p->rep_penalty;
  const bool use_rp = rp != 1.0f;
  ArgMax best{-INFINITY, 0x7fffffff};
  for (int i = threadIdx.x; i < vocab; i += 1024) {
    float v = __bfloat162float(lr[i]);
    if (use_rp && sr[i]) v = v < 0.f ? v * rp : v / rp;               // RepetitionPenaltyLogitsProcessor
    best = better(best, ArgMax{v, i});
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
    best = better(best, other);
  }
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 32; ++w) best = better(best, sm[w]);
    int tok = best.i == 0x7fffffff ? 0 : best.i;
    if constexpr (ROWS) session_append_token(b, tok, rows, p, seen, vocab, next_ids, out_ids, advance_len);
    else append_token(b, tok, state, p, seen, vocab, next_ids, out_ids);
  }
}
__global__ void __launch_bounds__(1024) select_greedy_kernel(const bf16* __restrict__ logits, int vocab,
                                                             GenState* state, const GenParamsDev* __restrict__ p,
                                                             uint8_t* seen, int32_t* next_ids, int32_t* out_ids) {
  select_greedy_body<false>(logits, vocab, state, p, seen, next_ids, out_ids, nullptr, 0u, 0);
}
__global__ void __launch_bounds__(1024) select_greedy_rows_kernel(const bf16* __restrict__ logits, int vocab,
                                                                  RowState* rows, const GenParamsDev* __restrict__ p,
                                                                  uint8_t* seen, int32_t* next_ids, int32_t* out_ids,
                                                                  uint32_t row_mask, int advance_len) {
  select_greedy_body<true>(logits, vocab, nullptr, p, seen, next_ids, out_ids, rows, row_mask, advance_len);
}
void launch_select_greedy(const bf16* logits, int vocab, int batch, GenState* state, const GenParamsDev* params,
                          uint8_t* seen, int32_t* next_ids, int32_t* out_ids, cudaStream_t st, RowState* rows,
                          uint32_t row_mask, int advance_len) {
  if (rows)
    select_greedy_rows_kernel<<<batch, 1024, 0, st>>>(logits, vocab, rows, params, seen, next_ids, out_ids, row_mask, advance_len);
  else
    select_greedy_kernel<<<batch, 1024, 0, st>>>(logits, vocab, state, params, seen, next_ids, out_ids);
  count_launch();
}

__global__ void __launch_bounds__(kSampleThreads) select_sample_spec_kernel(const bf16* __restrict__ logits, int vocab,
                                                                            GenState* state,
                                                                            const GenParamsDev* __restrict__ p,
                                                                            uint8_t* seen, float* __restrict__ probs,
                                                                            svspec::State* sp) {
  select_sample_body<false, true>(logits, vocab, state, p, seen, nullptr, nullptr, probs, nullptr, 0u, 0, sp);
}
void launch_select_sample_spec(const bf16* logits, int vocab, int ncols, GenState* state, const GenParamsDev* params,
                               uint8_t* seen, float* probs, svspec::State* sp, cudaStream_t st) {
  select_sample_spec_kernel<<<ncols, kSampleThreads, 0, st>>>(logits, vocab, state, params, seen, probs, sp);
  count_launch();
}
__global__ void __launch_bounds__(kSampleThreads) select_sample_kernel(const bf16* __restrict__ logits, int vocab,
                                                                       GenState* state,
                                                                       const GenParamsDev* __restrict__ p,
                                                                       uint8_t* seen, int32_t* next_ids,
                                                                       int32_t* out_ids, float* __restrict__ probs) {
  select_sample_body<false>(logits, vocab, state, p, seen, next_ids, out_ids, probs, nullptr, 0u, 0);
}
__global__ void __launch_bounds__(kSampleThreads) select_sample_rows_kernel(const bf16* __restrict__ logits, int vocab,
                                                                            RowState* rows,
                                                                            const GenParamsDev* __restrict__ p,
                                                                            uint8_t* seen, int32_t* next_ids,
                                                                            int32_t* out_ids, float* __restrict__ probs,
                                                                            uint32_t row_mask, int advance_len) {
  select_sample_body<true>(logits, vocab, nullptr, p, seen, next_ids, out_ids, probs, rows, row_mask, advance_len);
}
void launch_select_sample(const bf16* logits, int vocab, int batch, GenState* state, const GenParamsDev* params,
                          uint8_t* seen, int32_t* next_ids, int32_t* out_ids, float* probs, cudaStream_t st,
                          RowState* rows, uint32_t row_mask, int advance_len) {
  if (rows)
    select_sample_rows_kernel<<<batch, kSampleThreads, 0, st>>>(logits, vocab, rows, params, seen, next_ids, out_ids, probs,
                                                                row_mask, advance_len);
  else
    select_sample_kernel<<<batch, kSampleThreads, 0, st>>>(logits, vocab, state, params, seen, next_ids, out_ids, probs);
  count_launch();
}

// unfinished &= ~stop; this_peer_finished = unfinished.max()==0; then advance the step counter.
__global__ void gen_finalize_kernel(GenState* state, const GenParamsDev* __restrict__ p, int batch, int advance_len) {
  if (threadIdx.x != 0 || state->done) return;
  if (state->row0_stop) {
    for (int b = 0; b < batch; ++b) state->unfinished[b] = 0;
    state->row0_stop = 0;
  }
  state->step += 1;
  if (advance_len) state->cur_len += 1;
  int any = 0;
  for (int b = 0; b < batch; ++b) any |= state->unfinished[b];
  if (!any || state->step >= p->max_new) state->done = 1;
}
void launch_gen_finalize(GenState* state, const GenParamsDev* params, int batch, int advance_len, cudaStream_t st) {
  gen_finalize_kernel<<<1, 32, 0, st>>>(state, params, batch, advance_len);
  count_launch();
}
__global__ void session_admit_kernel(RowState* rows, const SessionAdmit a, uint8_t* seen, int vocab, int32_t* out_ids,
                                     int out_stride, int pad_id) {
  const int j = blockIdx.x, s = a.slot[j];
  for (int i = threadIdx.x; i < vocab; i += blockDim.x) seen[(int64_t)s * vocab + i] = 0;
  for (int i = threadIdx.x; i < out_stride; i += blockDim.x) out_ids[(int64_t)s * out_stride + i] = pad_id;
  if (threadIdx.x == 0) {
    rows->row_len[s] = a.len[j];
    rows->row_step[s] = 0;
    rows->row_active[s] = 1;
    rows->row_max_new[s] = a.max_new[j];
    rows->row_seed[s] = a.seed[j];
  }
}
void launch_session_admit(RowState* rows, const SessionAdmit& a, uint8_t* seen, int vocab, int32_t* out_ids, int out_stride,
                          int pad_id, cudaStream_t st) {
  if (a.n <= 0) return;
  session_admit_kernel<<<a.n, 256, 0, st>>>(rows, a, seen, vocab, out_ids, out_stride, pad_id);
  count_launch();
}
__global__ void advance_len_kernel(GenState* state) {
  if (threadIdx.x == 0) state->cur_len += 1;
}
void launch_advance_len(GenState* state, cudaStream_t st) {
  advance_len_kernel<<<1, 32, 0, st>>>(state);
  count_launch();
}

// ------------------------------------------------------------------------------------------
// Rotary position embedding of StarCoder2 (transformers modeling_starcoder2.py:72-107,265-329): cos/sin are computed
// in fp32, CAST TO bf16, and  q*cos + rotate_half(q)*sin  runs as three bf16 tensor ops (two products, one sum).
// inv_freq comes from the host, computed as transformers does in fp32 (1.0 / theta ** (arange(0, d, 2) / d): the exponent,
// the power and the reciprocal each rounded to fp32 once).  The device's powf may be an ulp or two off; at positions in the
// thousands that moves the angle enough to change bf16 entries by up to hundreds of ulps where cos / sin cross zero.
struct RopeInvFreq {
  float v[kRopeMaxHalf];
};
__global__ void rope_table_kernel(bf16* __restrict__ cos_t, bf16* __restrict__ sin_t, int max_pos, int half,
                                  const RopeInvFreq inv_freq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_pos * half) return;
  const int pos = i / half, j = i % half;
  const float ang = (float)pos * inv_freq.v[j];
  cos_t[i] = __float2bfloat16_rn(cosf(ang));
  sin_t[i] = __float2bfloat16_rn(sinf(ang));
}
void launch_rope_table(bf16* cos_t, bf16* sin_t, int max_pos, int d, float theta, cudaStream_t st) {
  RopeInvFreq f{};
  for (int j = 0; j < d / 2 && j < kRopeMaxHalf; ++j) {
    const float e = (float)(2 * j) / (float)d;
    f.v[j] = 1.0f / (float)std::pow((double)theta, (double)e);      // the fp32 power, correctly rounded
  }
  const int n = max_pos * (d / 2);
  rope_table_kernel<<<(n + 255) / 256, 256, 0, st>>>(cos_t, sin_t, max_pos, d / 2, f);
  count_launch();
}
template <bool ROWS>
SV_DEVINL void rope_body(bf16* __restrict__ qkv, int seq, int qkv_cols, int n_rot_heads, int d,
                         const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                         const GenState* __restrict__ state, const RowState* __restrict__ rows, int max_pos, int pos0) {
  const int row = blockIdx.x, half = d >> 1;
  int pos = ROWS ? rows->row_len[row] : (state ? state->cur_len : pos0 + (row % seq));
  pos = pos >= max_pos ? max_pos - 1 : pos;
  bf16* base = qkv + (int64_t)row * qkv_cols;
  for (int i = threadIdx.x; i < n_rot_heads * half; i += blockDim.x) {
    const int h = i / half, j = i % half;
    bf16* v = base + h * d;
    const float c = __bfloat162float(cos_t[(int64_t)pos * half + j]), s = __bfloat162float(sin_t[(int64_t)pos * half + j]);
    const float x1 = __bfloat162float(v[j]), x2 = __bfloat162float(v[j + half]);
    v[j] = __float2bfloat16_rn(bf16_round(x1 * c) + bf16_round(-x2 * s));
    v[j + half] = __float2bfloat16_rn(bf16_round(x2 * c) + bf16_round(x1 * s));
  }
}
__global__ void rope_kernel(bf16* __restrict__ qkv, int seq, int qkv_cols, int n_rot_heads, int d,
                            const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                            const GenState* __restrict__ state, int max_pos, int pos0) {
  rope_body<false>(qkv, seq, qkv_cols, n_rot_heads, d, cos_t, sin_t, state, nullptr, max_pos, pos0);
}
__global__ void rope_rows_kernel(bf16* __restrict__ qkv, int qkv_cols, int n_rot_heads, int d,
                                 const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                 const RowState* __restrict__ rows, int max_pos) {
  rope_body<true>(qkv, 1, qkv_cols, n_rot_heads, d, cos_t, sin_t, nullptr, rows, max_pos, 0);
}
// Decode-step companion of the fused QKV GEMV for RoPE models: rotate q in place, rotate k and append it (and v) to the
// KV cache at position cur_len (ROWS: rows->row_len[b]).  One block per image.
template <bool ROWS>
SV_DEVINL void rope_append_body(bf16* __restrict__ qkv, int qkv_cols, int n_head, int n_kv, int d,
                                const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                bf16* __restrict__ kcache, bf16* __restrict__ vtcache,
                                const GenState* __restrict__ state, const RowState* __restrict__ rows, int tcap,
                                int max_pos) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int b = blockIdx.x, half = d >> 1;
  const int pos = ROWS ? rows->row_len[b] : state->cur_len;
  const int tp = pos >= max_pos ? max_pos - 1 : pos;
  bf16* base = qkv + (int64_t)b * qkv_cols;
  for (int i = threadIdx.x; i < (n_head + n_kv) * half; i += blockDim.x) {
    const int h = i / half, j = i % half;
    bf16* v = base + h * d;
    const float c = __bfloat162float(cos_t[(int64_t)tp * half + j]), s = __bfloat162float(sin_t[(int64_t)tp * half + j]);
    const float x1 = __bfloat162float(__ldcg(v + j)), x2 = __bfloat162float(__ldcg(v + j + half));
    const bf16 o1 = __float2bfloat16_rn(bf16_round(x1 * c) + bf16_round(-x2 * s));
    const bf16 o2 = __float2bfloat16_rn(bf16_round(x2 * c) + bf16_round(x1 * s));
    if (h < n_head) {
      v[j] = o1; v[j + half] = o2;
    } else if (pos < tcap) {
      const int kvh = h - n_head;
      bf16* kr = kcache + (((int64_t)b * n_kv + kvh) * tcap + pos) * d;
      kr[j] = o1; kr[j + half] = o2;
    }
  }
  if (pos < tcap) {
    const bf16* vsrc = base + (n_head + n_kv) * d;
    for (int i = threadIdx.x; i < n_kv * d; i += blockDim.x) {
      const int kvh = i / d, dim = i % d;
      vtcache[(((int64_t)b * n_kv + kvh) * d + dim) * tcap + pos] = __ldcg(vsrc + i);
    }
  }
}
__global__ void rope_append_kernel(bf16* __restrict__ qkv, int qkv_cols, int n_head, int n_kv, int d,
                                   const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                   bf16* __restrict__ kcache, bf16* __restrict__ vtcache,
                                   const GenState* __restrict__ state, int tcap, int max_pos) {
  rope_append_body<false>(qkv, qkv_cols, n_head, n_kv, d, cos_t, sin_t, kcache, vtcache, state, nullptr, tcap, max_pos);
}
__global__ void rope_append_rows_kernel(bf16* __restrict__ qkv, int qkv_cols, int n_head, int n_kv, int d,
                                        const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                        bf16* __restrict__ kcache, bf16* __restrict__ vtcache,
                                        const RowState* __restrict__ rows, int tcap, int max_pos) {
  rope_append_body<true>(qkv, qkv_cols, n_head, n_kv, d, cos_t, sin_t, kcache, vtcache, nullptr, rows, tcap, max_pos);
}
void launch_rope_append(bf16* qkv, int batch, int qkv_cols, int n_head, int n_kv, int d, const bf16* cos_t,
                        const bf16* sin_t, bf16* kcache, bf16* vtcache, const GenState* state, int tcap, int max_pos,
                        bool pdl, cudaStream_t st, const RowState* rows) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(batch); cfg.blockDim = dim3(256); cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  if (rows)
    cudaLaunchKernelEx(&cfg, rope_append_rows_kernel, qkv, qkv_cols, n_head, n_kv, d, cos_t, sin_t, kcache, vtcache, rows,
                       tcap, max_pos);
  else
    cudaLaunchKernelEx(&cfg, rope_append_kernel, qkv, qkv_cols, n_head, n_kv, d, cos_t, sin_t, kcache, vtcache, state, tcap,
                       max_pos);
  count_launch();
}

void launch_rope(bf16* qkv, int rows, int seq, int qkv_cols, int n_rot_heads, int d, const bf16* cos_t, const bf16* sin_t,
                 const GenState* state, int max_pos, int pos0, cudaStream_t st, const RowState* row_pos) {
  if (row_pos) rope_rows_kernel<<<rows, 256, 0, st>>>(qkv, qkv_cols, n_rot_heads, d, cos_t, sin_t, row_pos, max_pos);
  else rope_kernel<<<rows, 256, 0, st>>>(qkv, seq, qkv_cols, n_rot_heads, d, cos_t, sin_t, state, max_pos, pos0);
  count_launch();
}

__global__ void fill_i32_kernel(int32_t* p, int32_t v, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
void launch_fill_i32(int32_t* p, int32_t v, int n, cudaStream_t st) {
  fill_i32_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, v, n);
  count_launch();
}

}  // namespace sv

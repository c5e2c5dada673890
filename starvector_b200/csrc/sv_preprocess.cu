// GPU image preprocessing (SURVEY.md §8f-2): uint8 HWC host images -> normalised [n,3,S,S] pixels in HBM, ready for
// sv_encode_images.  Replaces `ImageTrainProcessor.__call__` (reference starvector/data/util.py:40-66) and
// `SimpleStarVectorProcessor.transform` (starvector_arch.py:39-45), i.e. Pillow paste / pad / bicubic resize +
// torchvision ToTensor / Normalize, bit for bit (the integer arithmetic lives in sv_preprocess_core.h).
//
// HBM-bound byte work, two kernels per batch:
//   resize_h_kernel  one thread per (image, input row, output column): n_taps pixel fetches (paste/pad applied in the
//                    fetch), 3 int32 accumulators, one packed uint32 store into the 8-bit intermediate [in_h][S].
//   resize_v_kernel  one thread per (image, output pixel): n_taps coalesced uint32 loads down a column, clip, 256-entry
//                    per-channel table (ToTensor+Normalize evaluated on the host in fp32, exactly as torch does), three
//                    coalesced planar stores (bf16 or fp32).
// Algorithmic bytes per image = w*h*c in + 3*S*S*sizeof(out) out; the intermediate adds 2*in_h*S*4.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/starvector_b200.h"
#include "sv_preprocess_core.h"

namespace {

using svpre::ImageMeta;

std::string g_preproc_create_error;

// ---- host: Pillow's resample coefficients (Resample.c precompute_coeffs + normalize_coeffs_8bpc), box = whole axis ----
double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

struct Coeffs {
  int ksize = 0;
  std::vector<int32_t> data;   // bounds[out][2] (first tap, tap count) followed by taps[ksize][out] (tap-major)
};

Coeffs precompute_coeffs(int in_size, int out_size) {
  Coeffs c;
  double scale = (double)in_size / out_size, filterscale = scale;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  c.ksize = (int)std::ceil(support) * 2 + 1;
  c.data.assign((size_t)out_size * (2 + c.ksize), 0);
  int32_t* bounds = c.data.data();
  int32_t* taps = bounds + 2 * (size_t)out_size;
  std::vector<double> w(c.ksize);
  const double ss = 1.0 / filterscale;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = bicubic_filter((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    for (int x = 0; x < xmax; ++x) {
      const double v = ww != 0.0 ? w[x] / ww : w[x];
      taps[(size_t)x * out_size + xx] =
          v < 0 ? (int)(-0.5 + v * (1 << svpre::kPrecisionBits)) : (int)(0.5 + v * (1 << svpre::kPrecisionBits));
    }
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
  }
  return c;
}

// ToTensor (`byte.to(float32).div(255)`) + Normalize (`sub_(mean).div_(std)`): fp32 IEEE ops, one entry per byte value.
void build_lut(const float mean[3], const float stdv[3], float* lut /* [3][256] */) {
  for (int c = 0; c < 3; ++c)
    for (int i = 0; i < 256; ++i) {
      volatile float v = (float)i / 255.0f;
      volatile float d = v - mean[c];
      lut[c * 256 + i] = d / stdv[c];
    }
}

// ---- device -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) resize_h_kernel(const uint8_t* __restrict__ arena, const int32_t* __restrict__ coeffs,
                                                       const ImageMeta* __restrict__ metas, uint32_t* __restrict__ tmp,
                                                       int out_w) {
  const ImageMeta im = metas[blockIdx.y];
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= im.in_h * out_w) return;
  const int y = idx / out_w, xx = idx - y * out_w;
  tmp[im.tmp_off + idx] = svpre::horizontal_pixel(arena, coeffs, im, out_w, y, xx);
}

template <typename OutT>
__global__ void __launch_bounds__(256) resize_v_kernel(const uint32_t* __restrict__ tmp, const int32_t* __restrict__ coeffs,
                                                       const ImageMeta* __restrict__ metas, const float* __restrict__ lut,
                                                       OutT* __restrict__ out, int out_w, int out_h) {
  __shared__ float s_lut[768];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) s_lut[i] = lut[i];
  __syncthreads();
  const ImageMeta im = metas[blockIdx.y];
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= out_w * out_h) return;
  const int yy = idx / out_w, xx = idx - yy * out_w;
  int rgb[3];
  svpre::vertical_pixel(tmp, coeffs, im, out_w, out_h, yy, xx, rgb);
  const size_t plane = (size_t)out_w * out_h;
  OutT* o = out + (size_t)blockIdx.y * 3 * plane + idx;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = s_lut[c * 256 + rgb[c]];
    if constexpr (sizeof(OutT) == 2) o[c * plane] = __float2bfloat16_rn(v);
    else o[c * plane] = v;
  }
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

struct sv_preproc {
  int device = 0;
  sv_preproc_desc desc{};
  std::string err;
  float lut_host[768];
  float* lut_dev = nullptr;
  uint8_t* in_dev = nullptr;     size_t in_cap = 0;
  uint32_t* tmp_dev = nullptr;   size_t tmp_cap = 0;        // pixels
  uint8_t* meta_dev = nullptr;   size_t meta_cap = 0;       // ImageMeta[n] then the int32 coefficient arena
  uint8_t* meta_host = nullptr;  size_t meta_host_cap = 0;  // pinned mirror of meta_dev
  cudaEvent_t meta_copied = nullptr;
  bool meta_in_flight = false;
  std::map<std::pair<int, int>, Coeffs> coeff_cache;       // (in_size, out_size) -> taps; a serving process sees few sizes
  long long launches = 0;
};

namespace {

int fail(sv_preproc* p, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (p) p->err = buf; else g_preproc_create_error = buf;
  return code;
}

#define PRE_CK(p, call)                                                                                           \
  do {                                                                                                            \
    cudaError_t r_ = (call);                                                                                      \
    if (r_ != cudaSuccess) return fail(p, SV_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(r_));                  \
  } while (0)

template <typename T>
int grow(sv_preproc* p, T** ptr, size_t* cap, size_t need, bool pinned_host = false) {
  if (need <= *cap) return SV_OK;
  const size_t want = align_up(need + need / 4, 4096);
  if (*ptr) PRE_CK(p, pinned_host ? cudaFreeHost(*ptr) : cudaFree(*ptr));
  *ptr = nullptr;
  *cap = 0;
  void* q = nullptr;
  PRE_CK(p, pinned_host ? cudaMallocHost(&q, want * sizeof(T)) : cudaMalloc(&q, want * sizeof(T)));
  *ptr = (T*)q;
  *cap = want;
  return SV_OK;
}

// ---- host: the batch plan = ImageMeta[n] followed by the coefficient arena, plus arena sizes ----------------------------
struct Plan {
  std::vector<uint8_t> blob;
  size_t meta_bytes = 0, in_bytes = 0, tmp_px = 0;
  int max_rows = 0;
};

int plan_fail(std::string& err, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  err = buf;
  return SV_ERR_INVALID;
}

int make_plan(const sv_preproc_desc& desc, std::map<std::pair<int, int>, Coeffs>& cache, const sv_image_u8* images, int n,
              Plan& plan, std::string& err) {
  if (n < 1 || n > 4096) return plan_fail(err, "need 1..4096 images per call (got %d)", n);
  const int S = desc.out_size;
  std::vector<ImageMeta> metas(n);
  std::map<std::pair<int, int>, int32_t> placed;            // (in_size, S) -> int32 offset in this call's coefficient arena
  std::vector<const Coeffs*> order;
  size_t coeff_words = 0;
  for (int i = 0; i < n; ++i) {
    const sv_image_u8& im = images[i];
    if (!im.data || im.width < 1 || im.height < 1 || im.width > 16384 || im.height > 16384 || (im.channels != 3 && im.channels != 4))
      return plan_fail(err, "image %d: need uint8 HWC data, 1..16384 pixels per side, 3 or 4 channels (got %dx%dx%d)", i, im.width,
                       im.height, im.channels);
    const int tight = im.width * im.channels;
    if (im.row_stride != 0 && im.row_stride < tight) return plan_fail(err, "image %d: row_stride %d < width*channels", i, im.row_stride);
    ImageMeta& m = metas[i];
    std::memset(&m, 0, sizeof m);
    m.width = im.width; m.height = im.height; m.channels = im.channels; m.row_stride = tight;   // rows are tight in the arena
    m.alpha_white = desc.alpha_mode == SV_ALPHA_WHITE ? 1 : 0;
    if (desc.pad_square) {
      const int s = im.width > im.height ? im.width : im.height;
      m.in_w = m.in_h = s;
      m.pad_left = (s - im.width) / 2;
      m.pad_top = (s - im.height) / 2;
    } else {
      m.in_w = im.width; m.in_h = im.height;
    }
    m.src_off = (int64_t)plan.in_bytes;
    plan.in_bytes += align_up((size_t)tight * im.height, 16);
    m.tmp_off = (int64_t)plan.tmp_px;
    plan.tmp_px += (size_t)m.in_h * S;
    if (m.in_h > plan.max_rows) plan.max_rows = m.in_h;
    const int sizes[2] = {m.in_w, m.in_h};
    int32_t offs[2], ks[2];
    for (int a = 0; a < 2; ++a) {
      auto key = std::make_pair(sizes[a], S);
      auto c = cache.find(key);
      if (c == cache.end()) c = cache.emplace(key, precompute_coeffs(sizes[a], S)).first;   // std::map: references stay valid
      auto it = placed.find(key);
      if (it == placed.end()) {
        it = placed.emplace(key, (int32_t)coeff_words).first;
        coeff_words += c->second.data.size();
        order.push_back(&c->second);
      }
      offs[a] = it->second;
      ks[a] = c->second.ksize;
    }
    m.kx_off = offs[0]; m.ky_off = offs[1]; m.ksize_x = ks[0]; m.ksize_y = ks[1];
  }
  if (coeff_words > ((size_t)1 << 28)) return plan_fail(err, "coefficient arena too large");
  plan.meta_bytes = align_up(sizeof(ImageMeta) * (size_t)n, 16);
  plan.blob.assign(plan.meta_bytes + coeff_words * sizeof(int32_t), 0);
  std::memcpy(plan.blob.data(), metas.data(), sizeof(ImageMeta) * (size_t)n);
  uint8_t* w = plan.blob.data() + plan.meta_bytes;
  for (const Coeffs* c : order) {                           // same order as the offsets were handed out
    std::memcpy(w, c->data.data(), c->data.size() * sizeof(int32_t));
    w += c->data.size() * sizeof(int32_t);
  }
  return SV_OK;
}

}  // namespace

extern "C" {

int sv_resample_coeffs_host(int32_t in_size, int32_t out_size, int32_t* ksize, int32_t* bounds, int32_t* taps,
                            int32_t taps_capacity) {
  if (in_size < 1 || out_size < 1 || !ksize) return SV_ERR_INVALID;
  const Coeffs c = precompute_coeffs(in_size, out_size);
  *ksize = c.ksize;
  if (!bounds && !taps) return SV_OK;
  if (!bounds || !taps || (int64_t)taps_capacity < (int64_t)out_size * c.ksize) return SV_ERR_INVALID;
  std::memcpy(bounds, c.data.data(), sizeof(int32_t) * 2 * out_size);
  const int32_t* tm = c.data.data() + 2 * (size_t)out_size;          // stored tap-major; the export is [out][ksize]
  for (int xx = 0; xx < out_size; ++xx)
    for (int t = 0; t < c.ksize; ++t) taps[(size_t)xx * c.ksize + t] = tm[(size_t)t * out_size + xx];
  return SV_OK;
}

int sv_preproc_lut_host(const sv_preproc_desc* desc, float* lut768) {
  if (!desc || !lut768) return SV_ERR_INVALID;
  build_lut(desc->mean, desc->std, lut768);
  return SV_OK;
}

const char* sv_preproc_last_error(const sv_preproc* p) { return p ? p->err.c_str() : g_preproc_create_error.c_str(); }

int sv_preproc_create(const sv_preproc_desc* desc, int device, sv_preproc** out) {
  if (!desc || !out) return fail(nullptr, SV_ERR_INVALID, "sv_preproc_create: null argument");
  *out = nullptr;
  if (desc->out_size < 1 || desc->out_size > 4096) return fail(nullptr, SV_ERR_INVALID, "out_size %d not in 1..4096", desc->out_size);
  if (desc->out_dtype != SV_DTYPE_BF16 && desc->out_dtype != SV_DTYPE_F32)
    return fail(nullptr, SV_ERR_INVALID, "out_dtype must be SV_DTYPE_BF16 or SV_DTYPE_F32");
  for (int c = 0; c < 3; ++c)
    if (!(desc->std[c] > 0.0f)) return fail(nullptr, SV_ERR_INVALID, "std[%d] must be > 0", c);
  int count = 0;
  cudaError_t r = cudaGetDeviceCount(&count);
  if (r != cudaSuccess || device < 0 || device >= count)
    return fail(nullptr, SV_ERR_CUDA, "no usable CUDA device %d (%s): there is no CPU fallback", device,
                r == cudaSuccess ? "index out of range" : cudaGetErrorString(r));
  cudaDeviceProp prop;
  PRE_CK(nullptr, cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(nullptr, SV_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
  PRE_CK(nullptr, cudaSetDevice(device));
  sv_preproc* p = new sv_preproc();
  p->device = device;
  p->desc = *desc;
  build_lut(desc->mean, desc->std, p->lut_host);
  if (cudaMalloc((void**)&p->lut_dev, sizeof(p->lut_host)) != cudaSuccess ||
      cudaMemcpy(p->lut_dev, p->lut_host, sizeof(p->lut_host), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->meta_copied, cudaEventDisableTiming) != cudaSuccess) {
    const int code = fail(nullptr, SV_ERR_CUDA, "sv_preproc_create: %s", cudaGetErrorString(cudaGetLastError()));
    sv_preproc_destroy(p);
    return code;
  }
  *out = p;
  return SV_OK;
}

void sv_preproc_destroy(sv_preproc* p) {
  if (!p) return;
  cudaSetDevice(p->device);
  cudaDeviceSynchronize();
  if (p->lut_dev) cudaFree(p->lut_dev);
  if (p->in_dev) cudaFree(p->in_dev);
  if (p->tmp_dev) cudaFree(p->tmp_dev);
  if (p->meta_dev) cudaFree(p->meta_dev);
  if (p->meta_host) cudaFreeHost(p->meta_host);
  if (p->meta_copied) cudaEventDestroy(p->meta_copied);
  delete p;
}

long long sv_preproc_launch_count(const sv_preproc* p) { return p ? p->launches : 0; }

int sv_preproc_plan_host(const sv_preproc_desc* desc, const sv_image_u8* images_host, int32_t n, void* blob,
                         int64_t blob_capacity, int64_t sizes[5]) {
  if (!desc || !images_host || !sizes) return SV_ERR_INVALID;
  std::map<std::pair<int, int>, Coeffs> cache;
  Plan plan;
  std::string err;
  const int rc = make_plan(*desc, cache, images_host, n, plan, err);
  if (rc != SV_OK) {
    g_preproc_create_error = err;
    return rc;
  }
  sizes[0] = (int64_t)plan.blob.size(); sizes[1] = (int64_t)plan.meta_bytes; sizes[2] = (int64_t)plan.in_bytes;
  sizes[3] = (int64_t)plan.tmp_px; sizes[4] = plan.max_rows;
  if (blob) {
    if (blob_capacity < (int64_t)plan.blob.size()) return SV_ERR_INVALID;
    std::memcpy(blob, plan.blob.data(), plan.blob.size());
  }
  return SV_OK;
}

int sv_preproc_run_host(sv_preproc* p, const sv_image_u8* images_host, int32_t n, void* out_pixels, void* stream_) {
  if (!p) return SV_ERR_INVALID;
  if (!images_host || !out_pixels) return fail(p, SV_ERR_INVALID, "sv_preproc_run_host: null argument");
  cudaStream_t stream = (cudaStream_t)stream_;
  PRE_CK(p, cudaSetDevice(p->device));
  const int S = p->desc.out_size;
  if (p->coeff_cache.size() > 256) p->coeff_cache.clear();
  Plan plan;
  int rc = make_plan(p->desc, p->coeff_cache, images_host, n, plan, p->err);
  if (rc != SV_OK) return rc;
  const size_t blob_bytes = plan.blob.size();

  // ---- arenas (grown on demand, kept across calls)
  if (p->meta_in_flight) {                                  // the pinned mirror is reused: wait for the previous upload
    PRE_CK(p, cudaEventSynchronize(p->meta_copied));
    p->meta_in_flight = false;
  }
  if ((rc = grow(p, &p->in_dev, &p->in_cap, plan.in_bytes)) != SV_OK) return rc;
  if ((rc = grow(p, &p->tmp_dev, &p->tmp_cap, plan.tmp_px)) != SV_OK) return rc;
  if ((rc = grow(p, &p->meta_dev, &p->meta_cap, blob_bytes)) != SV_OK) return rc;
  if ((rc = grow(p, &p->meta_host, &p->meta_host_cap, blob_bytes, true)) != SV_OK) return rc;
  std::memcpy(p->meta_host, plan.blob.data(), blob_bytes);

  // ---- uploads: the blob (one copy) and every image (tight rows in the arena)
  PRE_CK(p, cudaMemcpyAsync(p->meta_dev, p->meta_host, blob_bytes, cudaMemcpyHostToDevice, stream));
  PRE_CK(p, cudaEventRecord(p->meta_copied, stream));
  p->meta_in_flight = true;
  const ImageMeta* metas = (const ImageMeta*)plan.blob.data();
  for (int i = 0; i < n; ++i) {
    const sv_image_u8& im = images_host[i];
    const size_t tight = (size_t)im.width * im.channels;
    const size_t pitch = im.row_stride ? (size_t)im.row_stride : tight;
    if (pitch == tight)
      PRE_CK(p, cudaMemcpyAsync(p->in_dev + metas[i].src_off, im.data, tight * im.height, cudaMemcpyHostToDevice, stream));
    else
      PRE_CK(p, cudaMemcpy2DAsync(p->in_dev + metas[i].src_off, tight, im.data, pitch, tight, im.height, cudaMemcpyHostToDevice, stream));
  }

  // ---- the two passes
  const ImageMeta* metas_dev = (const ImageMeta*)p->meta_dev;
  const int32_t* coeffs_dev = (const int32_t*)(p->meta_dev + plan.meta_bytes);
  {
    dim3 grid((unsigned)(((size_t)plan.max_rows * S + 255) / 256), (unsigned)n);
    resize_h_kernel<<<grid, 256, 0, stream>>>(p->in_dev, coeffs_dev, metas_dev, p->tmp_dev, S);
  }
  {
    dim3 grid((unsigned)(((size_t)S * S + 255) / 256), (unsigned)n);
    if (p->desc.out_dtype == SV_DTYPE_BF16)
      resize_v_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(p->tmp_dev, coeffs_dev, metas_dev, p->lut_dev, (__nv_bfloat16*)out_pixels, S, S);
    else
      resize_v_kernel<float><<<grid, 256, 0, stream>>>(p->tmp_dev, coeffs_dev, metas_dev, p->lut_dev, (float*)out_pixels, S, S);
  }
  PRE_CK(p, cudaGetLastError());
  p->launches += 2;
  return SV_OK;
}

}  // extern "C"

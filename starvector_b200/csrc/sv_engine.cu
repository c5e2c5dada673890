// C-ABI of the im2svg engine (include/starvector_b200.h): engine state, weight registry, the
// encode -> prefill -> decode orchestration and the CUDA-graph generation loop.
//
// Reference path being replaced: StarVectorBase.generate_im2svg
// (starvector/model/models/starvector_base.py:203-259) = ImageEncoder (image_encoder.py:91-94,
// clip_model.py:181-191) -> Adapter (adapters/adapter.py:33-39) -> prompt concat -> HF
// GenerationMixin.generate over GPTBigCodeForCausalLM (SURVEY.md §3.1, App. A/B).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/starvector_b200.h"
#include "sv_kernels.h"
#include "sv_select.cuh"

using namespace sv;

namespace {

constexpr int kMaxPrompt = 64;
constexpr int kStreamChunk = 1024;   // tokens per row handed to a streaming callback at once
constexpr int kMaxSplit = 128;
constexpr int kScoreRows = 4096;     // rows (batch x positions) of one sv_score_tokens chunk: keeps the layer GEMMs tensor-bound

std::string g_create_error;

struct Weight {
  bf16* p = nullptr;
  std::vector<int64_t> shape;      // shape expected from the caller (reference layout)
  int64_t numel = 0;
  bool loaded = false;
  bool optional = false;
};

struct VitLayer { bf16 *ln1_w, *ln1_b, *qkv_w, *qkv_b, *out_w, *out_b, *ln2_w, *ln2_b, *fc_w, *fc_b, *proj_w, *proj_b; };
struct DecLayer { bf16 *ln1_w, *ln1_b, *attn_w, *attn_b, *proj_w, *proj_b, *ln2_w, *ln2_b, *fc_w, *fc_b, *fc2_w, *fc2_b; };

// The decode-step graphs of generate, speculative generate, beam search and sessions share one cache.  Two captures that
// enqueue different kernels or arguments must never share a key: `rows` is the batch, the verify step's columns or the
// session's slots, `parts` the attention partition (decode_parts).
enum class StepKind { generate, speculative, beam, session, beam_session, spec_session };
struct StepKey {
  StepKind kind;
  int rows, parts;
  bool sample, fused, pdl;
  bool operator<(const StepKey& o) const {
    return std::tie(kind, rows, parts, sample, fused, pdl) < std::tie(o.kind, o.rows, o.parts, o.sample, o.fused, o.pdl);
  }
};
struct GraphEntry { cudaGraphExec_t exec = nullptr; int kernels = 0; bool pdl = false; };

}  // namespace

struct sv_engine {
  sv_model_desc d{};
  int device = 0;
  std::string err, describe;
  int64_t launches = 0;
  int linear_impl = SV_LINEAR_AUTO;

  int Q = 0, NP = 0, Kp = 0, Lpad = 0, qkv_cols = 0, tcap = 0;
  bool v2 = false;                 // SigLIP + StarCoder2 (StarVector-8B family)
  float vit_eps = 1e-5f;
  int vit_act = SV_ACT_QUICKGELU, window = 0;
  bf16 *conv_b = nullptr, *rope_cos = nullptr, *rope_sin = nullptr;
  std::map<std::string, Weight> w;
  std::vector<void*> allocs;

  // resolved weights
  bf16 *conv_w = nullptr, *conv_raw = nullptr, *cls = nullptr, *pos = nullptr, *lnpre_w = nullptr, *lnpre_b = nullptr;
  bf16 *lnv_w = nullptr, *lnv_b = nullptr;
  std::vector<VitLayer> vit;
  bf16 *afc_w = nullptr, *afc_b = nullptr, *aproj_w = nullptr, *aproj_b = nullptr, *anorm_w = nullptr, *anorm_b = nullptr,
       *anorm_rm = nullptr, *anorm_rv = nullptr;
  bf16 *wte = nullptr, *wpe = nullptr, *lnf_w = nullptr, *lnf_b = nullptr, *lm_head = nullptr;
  std::vector<DecLayer> dec;

  // activations / workspaces
  bf16 *v_patches, *v_pe, *v_x, *v_ln, *v_qkv, *v_vt, *v_attn, *v_h, *v_out, *a_h, *a_z, *visual;
  float* slab_partial;
  bf16 *p_x, *p_ln, *p_qkv, *p_attn, *p_h;
  bf16 *d_x, *d_ln, *d_qkv, *d_attn, *d_h, *d_last, *logits;
  float *logits_f32, *attn_partial, *amax_val;
  int* amax_idx;
  bool fused_decode = true, use_pdl = true;
  MegaLayer* mega_layers = nullptr;
  long long* mega_dbg = nullptr;
  bool mega_debug = false;
  // dataflow persistent decode kernel (sv_decode_flow.cu): flagged exchange buffers in one allocation
  bool use_flow = false, flow_realloc = false, flow_requested = false;
  bool use_tiles = false;           // slab-tiled weight copies exist (the dataflow kernel streams them)
  bool ring_tiles = false;          // SV_TILED=1: the ring GEMVs of the graph path stream them too
  uint8_t* flow_mem = nullptr;
  size_t flow_bytes = 0;
  uint32_t *f_xa = nullptr, *f_xb = nullptr, *f_qkv = nullptr, *f_att = nullptr, *f_hb = nullptr;
  unsigned long long *f_part = nullptr, *f_amax = nullptr;
  int flow_l2_ahead = 0;            // SV_FLOW_L2AHEAD: weight slabs per CTA prefetched into L2 ahead of the ring (measured: no gain, off)
  // slab-tiled copies of the decoder matrices for the dataflow kernel (made from the reference-layout weights when they change)
  std::vector<uint8_t*> t_attn, t_proj, t_fc, t_fc2;
  uint8_t* t_lm_head = nullptr;
  const bf16* t_lm_src = nullptr;   // which lm_head tensor t_lm_head was made from
  bool tiles_dirty = true;
  int flow_epoch = 0;               // phase-tag epoch: steps run through the flow kernel since the buffers were cleared
  bf16 *kscratch = nullptr, *vscratch = nullptr;   // one layer of cache, for beam-search reorders
  // device-resident beam search (sv_beam.cu), allocated by the first sv_beam_search or beam session (beam_alloc).  Params,
  // State and Plan hold one entry per group of a beam session (kMaxRows / 2); sv_beam_search uses the first
  svbeam::Params* beam_params = nullptr;
  svbeam::State* beam_state = nullptr;
  svbeam::Plan* beam_plan = nullptr;
  float *beam_key = nullptr, *beam_val = nullptr;
  int32_t *beam_tok = nullptr, *beam_run_seq = nullptr, *beam_fin_seq = nullptr;
  bf16 *kstage = nullptr, *vstage = nullptr;        // staging copy of the cache for the KV suffix moves (all layers)
  bf16 *kcache, *vtcache;           // [layer][max_batch][n_kv][tcap][D] / [layer][max_batch][n_kv][D][tcap]
  int64_t cache_layer_stride = 0;
  GenState* state = nullptr;
  GenParamsDev* params = nullptr;
  uint8_t* seen = nullptr;
  int32_t *next_ids = nullptr, *out_ids = nullptr, *ids_tmp = nullptr;
  bf16* im2svg_px = nullptr;        // staging of sv_generate_im2svg_host (pixels in, ids + lengths out): allocated by its first
  int32_t* im2svg_out = nullptr;    //   call, sized for max_batch rows, kept for the engine's lifetime
  int32_t* host_flag = nullptr;     // pinned
  int32_t* host_stream = nullptr;   // pinned staging of streamed tokens [max_batch][kStreamChunk], allocated on first use
  // sv_score_tokens chunk buffers (kScoreRows rows each), allocated by its first call: an engine that never scores keeps
  // the footprint it had without them
  bf16 *s_x = nullptr, *s_ln = nullptr, *s_qkv = nullptr, *s_attn = nullptr, *s_h = nullptr;
  int32_t* s_tgt = nullptr;
  float2* s_part = nullptr;
  float* s_tl = nullptr;

  // run state (host mirror)
  int cur_batch = 0, prefix_len = 0, host_cur_len = 0;
  bool encoded = false, prefilled = false;

  cudaStream_t gen_stream = nullptr;
  cudaEvent_t ev_in = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
  std::map<StepKey, GraphEntry> step_graphs;
  float last_decode_ms = 0.f;
  int last_decode_steps = 0;

  // continuous-batching session (sv_session_*): `sess_slots` cache rows decode with per-row positions (RowState); finished
  // rows are refilled by admission while the others keep their caches
  bool session = false;
  sv_gen_params sess_p{};
  int sess_slots = 0, sess_prompt_len = 0;   // the prompt length is fixed by the first admission
  RowState* rows = nullptr;                  // device, allocated by the first session
  RowState* rows_host = nullptr;             // pinned read-back of row_step / row_active
  bf16* sess_logits = nullptr;               // [max_batch][vocab]: the prefill logits of admitted slots (token 0 is read there)
  std::vector<int> sess_live;                // host: slot holds a request whose finish was not reported yet
  std::vector<int> sess_len;                 // host: tokens of each slot at the last poll
  // beam session (sv_beam_session_*): the slots form groups of num_beams, each one image's beam search with its own
  // beam_params / beam_state / beam_plan entry; sess_live / sess_len are kept at each group's first slot
  bool sess_beam = false;
  sv_beam_params sess_bp{};
  bf16* bsess_px = nullptr;                  // staging: one admitted image repeated num_beams times
  int32_t* bsess_ids = nullptr;              //   and its prompt
  // speculative session (sv_session_begin_speculative, DESIGN.md §7i): the verify step's columns belong to the live rows
  bool sess_spec = false;
  svspec::SessionState* spec_sess = nullptr; // device, allocated by the first speculative session

  // prompt-lookup speculative decoding (sv_generate_speculative): device state allocated by the first call
  svspec::State* spec = nullptr;
  RowState* spec_pos = nullptr;              // sv_spec_verify_step: the columns' embedding positions (row_len)
  int32_t spec_stats[3] = {0, 0, 0};         // steps, drafted, accepted of the last call
};

namespace {

int fail(sv_engine* e, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (e) e->err = buf; else g_create_error = buf;
  return code;
}

#define SV_CK(e, call)                                                                              \
  do {                                                                                              \
    cudaError_t _err = (call);                                                                      \
    if (_err != cudaSuccess)                                                                        \
      return fail((e), SV_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_err), __FILE__, __LINE__); \
  } while (0)

#define SV_TRY(call)              \
  do {                            \
    const int _r = (call);        \
    if (_r != SV_OK) return _r;   \
  } while (0)

struct LaunchScope {   // routes count_launch() of this thread to the engine's counter
  explicit LaunchScope(sv_engine* e) { g_launch_counter = &e->launches; }
  ~LaunchScope() { g_launch_counter = nullptr; }
};

template <typename T>
cudaError_t dev_alloc(sv_engine* e, T** p, int64_t n) {
  void* q = nullptr;
  cudaError_t r = cudaMalloc(&q, (size_t)std::max<int64_t>(n, 1) * sizeof(T));
  if (r == cudaSuccess) { e->allocs.push_back(q); *p = reinterpret_cast<T*>(q); }
  return r;
}

// `external` != nullptr registers the name as a view into storage that another entry owns (v2 packs the reference's
// separate q_proj / k_proj / v_proj tensors into one [q|k|v] matrix so both families share the same kernels).
bf16* add_weight(sv_engine* e, const std::string& name, std::vector<int64_t> shape, int64_t alloc_numel = -1,
                 bool optional = false, bf16* external = nullptr) {
  Weight wt;
  wt.shape = shape;
  wt.numel = 1;
  for (auto s : shape) wt.numel *= s;
  wt.optional = optional;
  if (external) {
    wt.p = external;
  } else {
    int64_t n = alloc_numel > 0 ? alloc_numel : wt.numel;
    if (dev_alloc(e, &wt.p, n) != cudaSuccess) return nullptr;
    cudaMemset(wt.p, 0, (size_t)n * sizeof(bf16));
  }
  bf16* p = wt.p;
  e->w[name] = std::move(wt);
  return p;
}

const char* VIS = "model.image_encoder.visual_encoder.";
const char* LNV = "model.image_encoder.ln_vision.";
const char* ADP = "model.image_projection.";
const char* DEC = "model.svg_transformer.transformer.transformer.";
const char* LMH = "model.svg_transformer.transformer.lm_head.weight";

bool build_weights_v2(sv_engine* e);

bool build_weights(sv_engine* e) {
  if (e->v2) return build_weights_v2(e);
  const sv_model_desc& d = e->d;
  const int64_t W = d.vit_width, Q = e->Q, H = d.hidden, kv = (int64_t)d.n_kv_head * d.head_dim, I = d.n_inner;
  bool ok = true;
  auto A = [&](const std::string& n, std::vector<int64_t> s, int64_t alloc = -1, bool opt = false) {
    bf16* p = add_weight(e, n, std::move(s), alloc, opt);
    ok = ok && p != nullptr;
    return p;
  };
  std::string v = VIS;
  e->conv_raw = A(v + "conv1.weight", {W, 3, d.patch_size, d.patch_size});
  ok = ok && dev_alloc(e, &e->conv_w, W * e->Kp) == cudaSuccess;
  e->cls = A(v + "class_embedding", {W});
  e->pos = A(v + "positional_embedding", {Q, W});
  e->lnpre_w = A(v + "ln_pre.weight", {W});
  e->lnpre_b = A(v + "ln_pre.bias", {W});
  e->vit.resize(d.vit_layers);
  for (int i = 0; i < d.vit_layers; ++i) {
    std::string p = v + "transformer.resblocks." + std::to_string(i) + ".";
    VitLayer& L = e->vit[i];
    L.ln1_w = A(p + "ln_1.weight", {W}); L.ln1_b = A(p + "ln_1.bias", {W});
    L.qkv_w = A(p + "attn.in_proj_weight", {3 * W, W}); L.qkv_b = A(p + "attn.in_proj_bias", {3 * W});
    L.out_w = A(p + "attn.out_proj.weight", {W, W}); L.out_b = A(p + "attn.out_proj.bias", {W});
    L.ln2_w = A(p + "ln_2.weight", {W}); L.ln2_b = A(p + "ln_2.bias", {W});
    L.fc_w = A(p + "mlp.c_fc.weight", {(int64_t)d.vit_mlp, W}); L.fc_b = A(p + "mlp.c_fc.bias", {(int64_t)d.vit_mlp});
    L.proj_w = A(p + "mlp.c_proj.weight", {W, (int64_t)d.vit_mlp}); L.proj_b = A(p + "mlp.c_proj.bias", {W});
  }
  e->lnv_w = A(std::string(LNV) + "weight", {W});
  e->lnv_b = A(std::string(LNV) + "bias", {W});
  std::string a = ADP;
  e->afc_w = A(a + "c_fc.weight", {2 * W, W}); e->afc_b = A(a + "c_fc.bias", {2 * W});
  e->aproj_w = A(a + "c_proj.weight", {H, 2 * W}); e->aproj_b = A(a + "c_proj.bias", {H});
  if (d.adapter_norm == 0) {
    e->anorm_w = A(a + "norm.weight", {Q, H}); e->anorm_b = A(a + "norm.bias", {Q, H});
  } else {
    e->anorm_w = A(a + "norm.weight", {Q}); e->anorm_b = A(a + "norm.bias", {Q});
    e->anorm_rm = A(a + "norm.running_mean", {Q}); e->anorm_rv = A(a + "norm.running_var", {Q});
  }
  std::string t = DEC;
  e->wte = A(t + "wte.weight", {(int64_t)d.vocab, H});
  e->wpe = A(t + "wpe.weight", {(int64_t)d.n_positions, H});
  e->dec.resize(d.n_layer);
  for (int i = 0; i < d.n_layer; ++i) {
    std::string p = t + "h." + std::to_string(i) + ".";
    DecLayer& L = e->dec[i];
    L.ln1_w = A(p + "ln_1.weight", {H}); L.ln1_b = A(p + "ln_1.bias", {H});
    L.attn_w = A(p + "attn.c_attn.weight", {H + 2 * kv, H}); L.attn_b = A(p + "attn.c_attn.bias", {H + 2 * kv});
    L.proj_w = A(p + "attn.c_proj.weight", {H, H}); L.proj_b = A(p + "attn.c_proj.bias", {H});
    L.ln2_w = A(p + "ln_2.weight", {H}); L.ln2_b = A(p + "ln_2.bias", {H});
    L.fc_w = A(p + "mlp.c_fc.weight", {I, H}); L.fc_b = A(p + "mlp.c_fc.bias", {I});
    L.fc2_w = A(p + "mlp.c_proj.weight", {H, I}); L.fc2_b = A(p + "mlp.c_proj.bias", {H});
  }
  e->lnf_w = A(t + "ln_f.weight", {H});
  e->lnf_b = A(t + "ln_f.bias", {H});
  e->lm_head = e->wte;   // tied (train/util.py:68-77); an explicit lm_head.weight un-ties it
  return ok;
}

// StarVector v2 (8B family) state dict: SiglipVisionTransformer keys under model.image_encoder.visual_encoder.
// (image_encoder.py:32-48,108-109), the same Adapter, Starcoder2ForCausalLM keys under
// model.svg_transformer.transformer. (llm/starcoder2.py:19-32).  q/k/v projections are packed [q|k|v] at load.
bool build_weights_v2(sv_engine* e) {
  const sv_model_desc& d = e->d;
  const int64_t W = d.vit_width, Q = e->Q, H = d.hidden, D = d.head_dim, kv = (int64_t)d.n_kv_head * D, I = d.n_inner;
  const int64_t HQ = (int64_t)d.n_head * D;
  bool ok = true;
  auto A = [&](const std::string& n, std::vector<int64_t> s, bf16* ext = nullptr, bool opt = false) {
    bf16* p = add_weight(e, n, std::move(s), -1, opt, ext);
    ok = ok && p != nullptr;
    return p;
  };
  auto raw = [&](int64_t n) { bf16* p = nullptr; ok = ok && dev_alloc(e, &p, n) == cudaSuccess; if (p) cudaMemset(p, 0, (size_t)n * 2); return p; };
  std::string v = VIS;
  e->conv_raw = A(v + "embeddings.patch_embedding.weight", {W, 3, d.patch_size, d.patch_size});
  ok = ok && dev_alloc(e, &e->conv_w, W * e->Kp) == cudaSuccess;
  e->conv_b = A(v + "embeddings.patch_embedding.bias", {W});
  e->pos = A(v + "embeddings.position_embedding.weight", {Q, W});
  e->vit.resize(d.vit_layers);
  for (int i = 0; i < d.vit_layers; ++i) {
    std::string p = v + "encoder.layers." + std::to_string(i) + ".";
    VitLayer& L = e->vit[i];
    L.ln1_w = A(p + "layer_norm1.weight", {W}); L.ln1_b = A(p + "layer_norm1.bias", {W});
    L.qkv_w = raw(3 * W * W); L.qkv_b = raw(3 * W);
    if (!ok) return false;
    const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      A(p + "self_attn." + nm[j] + ".weight", {W, W}, L.qkv_w + j * W * W);
      A(p + "self_attn." + nm[j] + ".bias", {W}, L.qkv_b + j * W);
    }
    L.out_w = A(p + "self_attn.out_proj.weight", {W, W}); L.out_b = A(p + "self_attn.out_proj.bias", {W});
    L.ln2_w = A(p + "layer_norm2.weight", {W}); L.ln2_b = A(p + "layer_norm2.bias", {W});
    L.fc_w = A(p + "mlp.fc1.weight", {(int64_t)d.vit_mlp, W}); L.fc_b = A(p + "mlp.fc1.bias", {(int64_t)d.vit_mlp});
    L.proj_w = A(p + "mlp.fc2.weight", {W, (int64_t)d.vit_mlp}); L.proj_b = A(p + "mlp.fc2.bias", {W});
  }
  e->lnv_w = A(v + "post_layernorm.weight", {W});
  e->lnv_b = A(v + "post_layernorm.bias", {W});
  std::string a = ADP;
  e->afc_w = A(a + "c_fc.weight", {2 * W, W}); e->afc_b = A(a + "c_fc.bias", {2 * W});
  e->aproj_w = A(a + "c_proj.weight", {H, 2 * W}); e->aproj_b = A(a + "c_proj.bias", {H});
  if (d.adapter_norm == 0) {
    e->anorm_w = A(a + "norm.weight", {Q, H}); e->anorm_b = A(a + "norm.bias", {Q, H});
  } else {
    e->anorm_w = A(a + "norm.weight", {Q}); e->anorm_b = A(a + "norm.bias", {Q});
    e->anorm_rm = A(a + "norm.running_mean", {Q}); e->anorm_rv = A(a + "norm.running_var", {Q});
  }
  std::string t = "model.svg_transformer.transformer.model.";
  e->wte = A(t + "embed_tokens.weight", {(int64_t)d.vocab, H});
  e->wpe = nullptr;
  e->dec.resize(d.n_layer);
  for (int i = 0; i < d.n_layer; ++i) {
    std::string p = t + "layers." + std::to_string(i) + ".";
    DecLayer& L = e->dec[i];
    L.ln1_w = A(p + "input_layernorm.weight", {H}); L.ln1_b = A(p + "input_layernorm.bias", {H});
    L.attn_w = raw((HQ + 2 * kv) * H); L.attn_b = raw(HQ + 2 * kv);
    if (!ok) return false;
    A(p + "self_attn.q_proj.weight", {HQ, H}, L.attn_w); A(p + "self_attn.q_proj.bias", {HQ}, L.attn_b);
    A(p + "self_attn.k_proj.weight", {kv, H}, L.attn_w + HQ * H); A(p + "self_attn.k_proj.bias", {kv}, L.attn_b + HQ);
    A(p + "self_attn.v_proj.weight", {kv, H}, L.attn_w + (HQ + kv) * H); A(p + "self_attn.v_proj.bias", {kv}, L.attn_b + HQ + kv);
    L.proj_w = A(p + "self_attn.o_proj.weight", {H, HQ}); L.proj_b = A(p + "self_attn.o_proj.bias", {H});
    L.ln2_w = A(p + "post_attention_layernorm.weight", {H}); L.ln2_b = A(p + "post_attention_layernorm.bias", {H});
    L.fc_w = A(p + "mlp.c_fc.weight", {I, H}); L.fc_b = A(p + "mlp.c_fc.bias", {I});
    L.fc2_w = A(p + "mlp.c_proj.weight", {H, I}); L.fc2_b = A(p + "mlp.c_proj.bias", {H});
  }
  e->lnf_w = A(t + "norm.weight", {H});
  e->lnf_b = A(t + "norm.bias", {H});
  e->lm_head = e->wte;
  // RoPE tables [n_positions][D/2]: computed on device at create; a host may overwrite them with its own values
  e->rope_cos = A("engine.rope_cos", {(int64_t)d.n_positions, D / 2}, nullptr, true);
  e->rope_sin = A("engine.rope_sin", {(int64_t)d.n_positions, D / 2}, nullptr, true);
  return ok;
}

bool build_buffers(sv_engine* e) {
  const sv_model_desc& d = e->d;
  const int64_t B = d.max_batch, W = d.vit_width, H = d.hidden, I = d.n_inner, D = d.head_dim;
  const int64_t Mv = B * e->Q, Mp = B * (e->Q + kMaxPrompt), heads = d.vit_heads;
  bool ok = true;
#define AL(ptr, n) ok = ok && (dev_alloc(e, &e->ptr, (n)) == cudaSuccess)
  AL(v_patches, B * e->NP * e->Kp); AL(v_pe, B * e->NP * W); AL(v_x, Mv * W); AL(v_ln, Mv * W);
  AL(v_qkv, Mv * 3 * W); AL(v_vt, B * heads * 64 * e->Lpad); AL(v_attn, Mv * W); AL(v_h, Mv * d.vit_mlp);
  AL(v_out, Mv * W); AL(a_h, Mv * 2 * W); AL(a_z, Mv * H); AL(visual, Mv * H);
  AL(slab_partial, B * 64 * 2);
  AL(p_x, Mp * H); AL(p_ln, Mp * H); AL(p_qkv, Mp * e->qkv_cols); AL(p_attn, Mp * H); AL(p_h, Mp * I);
  AL(d_x, B * H); AL(d_ln, B * H); AL(d_qkv, B * e->qkv_cols); AL(d_attn, B * H); AL(d_h, B * I); AL(d_last, B * H);
  AL(logits, B * d.vocab); AL(logits_f32, B * d.vocab);
  AL(attn_partial, B * d.n_kv_head * kMaxSplit * (32 + 16 * D));
  const int64_t amax_rows = gemv_ring_ntiles(d.vocab) * 8 * ring_row_groups((int)B);    // [tile][8 * row groups]
  AL(amax_val, amax_rows); AL(amax_idx, amax_rows);
  AL(mega_layers, d.n_layer); AL(mega_dbg, 8192);
  {
    // flagged exchange buffers of the dataflow decode kernel, cleared together when a sequence starts
    // a flagged word per value, one 8-value fragment per 256-byte chunk (sv_decode_flow.cu FRAG_STRIDE): 32 bytes per value
    const size_t n_x = (size_t)B * H * 32, n_qkv = (size_t)B * e->qkv_cols * 32, n_hb = (size_t)B * I * 32;
    const size_t n_part = (size_t)B * d.n_kv_head * decode_flow_max_splits() * decode_flow_partial_floats() * 8;
    const size_t n_amax = (size_t)gemv_ring_ntiles(d.vocab) * 8 * 8;
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    e->flow_bytes = 3 * up(n_x) + up(n_qkv) + up(n_hb) + up(n_part) + up(n_amax);
    AL(flow_mem, (int64_t)e->flow_bytes);
    if (ok) {
      uint8_t* q = e->flow_mem;
      e->f_xa = reinterpret_cast<uint32_t*>(q); q += up(n_x);
      e->f_xb = reinterpret_cast<uint32_t*>(q); q += up(n_x);
      e->f_att = reinterpret_cast<uint32_t*>(q); q += up(n_x);
      e->f_qkv = reinterpret_cast<uint32_t*>(q); q += up(n_qkv);
      e->f_hb = reinterpret_cast<uint32_t*>(q); q += up(n_hb);
      e->f_part = reinterpret_cast<unsigned long long*>(q); q += up(n_part);
      e->f_amax = reinterpret_cast<unsigned long long*>(q);
    }
  }
  e->cache_layer_stride = B * d.n_kv_head * (int64_t)e->tcap * D;
  AL(kcache, e->cache_layer_stride * d.n_layer); AL(vtcache, e->cache_layer_stride * d.n_layer);
  AL(kscratch, e->cache_layer_stride); AL(vscratch, e->cache_layer_stride);
  AL(state, 1); AL(params, 1); AL(seen, B * d.vocab); AL(next_ids, B); AL(out_ids, B * (int64_t)d.max_len);
  AL(ids_tmp, B * kMaxPrompt);
#undef AL
  if (!ok) return false;
  // zero the caches once: masked keys are never read as NaN (sv_attention.cu, P == 0 there)
  cudaMemset(e->kcache, 0, (size_t)e->cache_layer_stride * d.n_layer * sizeof(bf16));
  cudaMemset(e->vtcache, 0, (size_t)e->cache_layer_stride * d.n_layer * sizeof(bf16));
  cudaMemset(e->state, 0, sizeof(GenState));
  cudaMemset(e->flow_mem, 0, e->flow_bytes);
  return cudaMallocHost(reinterpret_cast<void**>(&e->host_flag), 64) == cudaSuccess;
}

int do_linear(sv_engine* e, int impl, const bf16* x, const bf16* w, const bf16* bias, const bf16* res, bf16* y, int M,
              int N, int K, int act, cudaStream_t st) {
  if (impl == SV_LINEAR_AUTO) impl = (M > 32 && wgmma_supported(M, N, K)) ? SV_LINEAR_TCGEN05 : SV_LINEAR_ROWGROUP;
  if (impl == SV_LINEAR_TCGEN05) {
    if (!wgmma_supported(M, N, K)) return fail(e, SV_ERR_INVALID, "wgmma linear needs N%%8==0, K%%64==0 (M=%d N=%d K=%d)", M, N, K);
    cudaError_t r = launch_linear_wgmma(x, w, bias, res, y, M, N, K, act, st);
    if (r != cudaSuccess) return fail(e, SV_ERR_CUDA, "wgmma linear launch failed: %s", cudaGetErrorString(r));
    return SV_OK;
  }
  if (K % 32 != 0) return fail(e, SV_ERR_INVALID, "rowgroup linear needs K%%32==0 (K=%d)", K);
  launch_linear_rowgroup(x, w, bias, res, y, M, N, K, act, st);
  return SV_OK;
}
#define LIN(...)                                   \
  do {                                             \
    int _r = do_linear(e, e->linear_impl, __VA_ARGS__); \
    if (_r != SV_OK) return _r;                    \
  } while (0)

// ---- stage: ViT + adapter -------------------------------------------------------------------
int run_encode(sv_engine* e, const bf16* pixels, int B, cudaStream_t st) {
  const sv_model_desc& d = e->d;
  const int W = d.vit_width, Q = e->Q, NP = e->NP, M = B * Q, H = d.hidden;
  const float veps = e->vit_eps;
  launch_im2col(pixels, e->v_patches, B, d.image_size, d.patch_size, e->Kp, st);
  LIN(e->v_patches, e->conv_w, e->conv_b, nullptr, e->v_pe, B * NP, W, e->Kp, SV_ACT_NONE, st);   // patch conv (bias: SigLIP only)
  if (e->v2) {
    launch_vit_assemble(e->v_pe, nullptr, e->pos, e->v_x, B, NP, W, st);                           // + position_embedding
  } else {
    launch_vit_assemble(e->v_pe, e->cls, e->pos, e->v_ln, B, NP, W, st);                           // cat cls + pos
    launch_layernorm(e->v_ln, e->lnpre_w, e->lnpre_b, e->v_x, M, W, veps, W, st);                  // ln_pre
  }
  for (int i = 0; i < d.vit_layers; ++i) {
    const VitLayer& L = e->vit[i];
    launch_layernorm(e->v_x, L.ln1_w, L.ln1_b, e->v_ln, M, W, veps, W, st);
    LIN(e->v_ln, L.qkv_w, L.qkv_b, nullptr, e->v_qkv, M, 3 * W, W, SV_ACT_NONE, st);
    launch_vit_transpose_v(e->v_qkv, e->v_vt, B, Q, d.vit_heads, e->Lpad, st);
    launch_attention_vit(e->v_qkv, e->v_vt, e->v_attn, B, Q, d.vit_heads, e->Lpad, st);
    LIN(e->v_attn, L.out_w, L.out_b, e->v_x, e->v_x, M, W, W, SV_ACT_NONE, st);                    // x += attn
    launch_layernorm(e->v_x, L.ln2_w, L.ln2_b, e->v_ln, M, W, veps, W, st);
    LIN(e->v_ln, L.fc_w, L.fc_b, nullptr, e->v_h, M, d.vit_mlp, W, e->vit_act, st);
    LIN(e->v_h, L.proj_w, L.proj_b, e->v_x, e->v_x, M, W, d.vit_mlp, SV_ACT_NONE, st);             // x += mlp
  }
  launch_layernorm(e->v_x, e->lnv_w, e->lnv_b, e->v_out, M, W, veps, W, st);                       // ln_vision | post_layernorm
  LIN(e->v_out, e->afc_w, e->afc_b, nullptr, e->a_h, M, 2 * W, W, SV_ACT_SILU, st);
  LIN(e->a_h, e->aproj_w, e->aproj_b, nullptr, e->a_z, M, H, 2 * W, SV_ACT_NONE, st);
  if (d.adapter_norm == 0)
    launch_slab_layernorm(e->a_z, e->anorm_w, e->anorm_b, e->visual, e->slab_partial, B, (int64_t)Q * H, 1e-5f, st);
  else
    launch_batchnorm_tokens(e->a_z, e->anorm_w, e->anorm_b, e->anorm_rm, e->anorm_rv, e->visual, B, Q, H, 1e-5f, st);
  return SV_OK;
}

// ---- stage: decoder prefill -----------------------------------------------------------------
// `prefix` is [B, q, H] embeddings (the resident visual prefix, or caller-provided inputs_embeds);
// `prompt_ids` [B, P] are embedded through wte and appended (P may be 0).
// `row0`: the prefilled images land in cache rows row0 .. row0+B-1 (a session admits into its free slots; every other row
// of the cache is left as it is), and the last-position logits go to `logits_out` (nullptr: e->logits).
int run_prefill(sv_engine* e, const bf16* prefix, int q, const int32_t* prompt_ids, int B, int P, cudaStream_t st,
                int row0 = 0, bf16* logits_out = nullptr) {
  const sv_model_desc& d = e->d;
  const int H = d.hidden, T0 = q + P, M = B * T0, D = d.head_dim;
  const int64_t row_off = (int64_t)row0 * d.n_kv_head * e->tcap * D;     // cache layout [layer][row][n_kv][tcap][D]
  launch_embed_prefix(prefix, prompt_ids, e->wte, e->wpe, e->p_x, B, q, P, H, d.vocab, 0, P, st);
  for (int i = 0; i < d.n_layer; ++i) {
    const DecLayer& L = e->dec[i];
    bf16* kc = e->kcache + e->cache_layer_stride * i + row_off;
    bf16* vc = e->vtcache + e->cache_layer_stride * i + row_off;
    launch_layernorm(e->p_x, L.ln1_w, L.ln1_b, e->p_ln, M, H, d.ln_eps, H, st);
    LIN(e->p_ln, L.attn_w, L.attn_b, nullptr, e->p_qkv, M, e->qkv_cols, H, SV_ACT_NONE, st);
    if (e->v2)   // RoPE on q and k (positions 0..T0-1), modeling_starcoder2.py:167-168
      launch_rope(e->p_qkv, M, T0, e->qkv_cols, d.n_head + d.n_kv_head, D, e->rope_cos, e->rope_sin, nullptr, d.n_positions, 0, st);
    launch_kv_scatter(e->p_qkv, kc, vc, B, T0, d.n_head * D, d.n_kv_head, D, e->tcap, 0, st);
    launch_attention_heads(e->p_qkv, e->qkv_cols, kc, vc, e->p_attn, B, T0, d.n_head, d.n_kv_head, D, e->tcap, e->window, st);
    LIN(e->p_attn, L.proj_w, L.proj_b, e->p_x, e->p_x, M, H, H, SV_ACT_NONE, st);
    launch_layernorm(e->p_x, L.ln2_w, L.ln2_b, e->p_ln, M, H, d.ln_eps, H, st);
    LIN(e->p_ln, L.fc_w, L.fc_b, nullptr, e->p_h, M, d.n_inner, H, SV_ACT_GELU_TANH, st);
    LIN(e->p_h, L.fc2_w, L.fc2_b, e->p_x, e->p_x, M, H, d.n_inner, SV_ACT_NONE, st);
  }
  // last-position logits only (HF computes all T0 positions; only [:, -1] is consumed)
  launch_gather_rows(e->p_x, e->d_last, B, T0, T0 - 1, H, st);
  launch_layernorm(e->d_last, e->lnf_w, e->lnf_b, e->d_ln, B, H, d.ln_eps, H, st);
  launch_linear_rowgroup(e->d_ln, e->lm_head, nullptr, nullptr, logits_out ? logits_out : e->logits, B, d.vocab, H, SV_ACT_NONE, st);
  return SV_OK;
}

// ---- stage: teacher-forced scoring chunk ------------------------------------------------------
// Rows [b][t] = ids[b][c0 + t] (row stride n) at cache positions pos0 + t, t < C, through the decoder at prefill shape:
// KV rows appended, the log-likelihood of ids[b][c0 + t + 1] written to logprobs[b][c0 + t + 1] without materialising
// the logits.  `last`: also leave the bf16 logits of the final position resident (as run_prefill does).
// Every GEMM runs on the wgmma kernel whatever M is, and the resident logits come from the same lm_head tiling as the
// fused log-likelihood, so the log-probs of a sequence do not depend on how it is split over calls or chunks.
int run_score_chunk(sv_engine* e, const int32_t* ids, int n, int c0, int C, int B, int pos0, float* logprobs, bool last,
                    cudaStream_t st) {
  const sv_model_desc& d = e->d;
  const int H = d.hidden, M = B * C, D = d.head_dim;
#define SLIN(...)                                           \
  do {                                                      \
    int _r = do_linear(e, SV_LINEAR_TCGEN05, __VA_ARGS__);  \
    if (_r != SV_OK) return _r;                             \
  } while (0)
  launch_embed_prefix(nullptr, ids + c0, e->wte, e->wpe, e->s_x, B, 0, C, H, d.vocab, pos0, n, st);
  for (int i = 0; i < d.n_layer; ++i) {
    const DecLayer& L = e->dec[i];
    bf16* kc = e->kcache + e->cache_layer_stride * i;
    bf16* vc = e->vtcache + e->cache_layer_stride * i;
    launch_layernorm(e->s_x, L.ln1_w, L.ln1_b, e->s_ln, M, H, d.ln_eps, H, st);
    SLIN(e->s_ln, L.attn_w, L.attn_b, nullptr, e->s_qkv, M, e->qkv_cols, H, SV_ACT_NONE, st);
    if (e->v2)
      launch_rope(e->s_qkv, M, C, e->qkv_cols, d.n_head + d.n_kv_head, D, e->rope_cos, e->rope_sin, nullptr, d.n_positions, pos0, st);
    launch_kv_scatter(e->s_qkv, kc, vc, B, C, d.n_head * D, d.n_kv_head, D, e->tcap, pos0, st);
    cudaError_t ce = launch_attention_chunk(e->s_qkv, e->qkv_cols, C, kc, vc, e->s_attn, B, C, pos0, d.n_head, d.n_kv_head, D,
                                            e->tcap, e->window, st);
    if (ce != cudaSuccess) return fail(e, SV_ERR_CUDA, "chunk attention launch failed: %s", cudaGetErrorString(ce));
    SLIN(e->s_attn, L.proj_w, L.proj_b, e->s_x, e->s_x, M, H, H, SV_ACT_NONE, st);
    launch_layernorm(e->s_x, L.ln2_w, L.ln2_b, e->s_ln, M, H, d.ln_eps, H, st);
    SLIN(e->s_ln, L.fc_w, L.fc_b, nullptr, e->s_h, M, d.n_inner, H, SV_ACT_GELU_TANH, st);
    SLIN(e->s_h, L.fc2_w, L.fc2_b, e->s_x, e->s_x, M, H, d.n_inner, SV_ACT_NONE, st);
  }
  launch_layernorm(e->s_x, e->lnf_w, e->lnf_b, e->s_ln, M, H, d.ln_eps, H, st);
  launch_score_targets(ids, n, c0, B, C, d.vocab, e->s_tgt, st);
  cudaError_t ce = launch_lm_logprob_partials(e->s_ln, e->lm_head, e->s_tgt, e->s_part, e->s_tl, M, d.vocab, H, st);
  if (ce != cudaSuccess) return fail(e, SV_ERR_CUDA, "lm_head log-likelihood launch failed: %s", cudaGetErrorString(ce));
  launch_logprob_merge(e->s_part, lm_logprob_ntiles(d.vocab), e->s_tl, M, C, c0 + 1, n, logprobs, st);
  if (last) {
    launch_gather_rows(e->s_x, e->d_last, B, C, C - 1, H, st);
    launch_layernorm(e->d_last, e->lnf_w, e->lnf_b, e->d_ln, B, H, d.ln_eps, H, st);
    ce = launch_lm_logits(e->d_ln, e->lm_head, e->logits, B, d.vocab, H, st);
    if (ce != cudaSuccess) return fail(e, SV_ERR_CUDA, "lm_head launch failed: %s", cudaGetErrorString(ce));
  }
#undef SLIN
  return SV_OK;
}

// ---- one decode step: token ids (device) at position state->cur_len -> logits ----------------
// The decode chain of one step as plain data.  The engine fills it from its own state with every activation stride 0
// (one buffer reused by every layer, the residual stream updated in place); sv_op_decode_chain fills it from the caller's
// tensors, where a nonzero stride (elements) keeps every layer's intermediates.  Slots: x[2l] is layer l's input,
// x[2l + 1] the residual stream after its attention, x[2l + 2] its output; ln[2l], ln[2l + 1] its LayerNorm outputs and
// ln[2 n_layer] ln_f's (per-op chain only); qkv[l], attn[l], h[l].
struct DecodeChain {
  int n_layer = 0;
  const DecLayer* layers = nullptr;
  uint8_t* const *t_attn = nullptr, *const *t_proj = nullptr, *const *t_fc = nullptr, *const *t_fc2 = nullptr;   // slab-tiled
  const uint8_t* t_lm_head = nullptr;                                                        //   copies, or nullptr
  bf16 *kcache = nullptr, *vtcache = nullptr;   // [layer][row][n_kv][tcap][D] / [layer][row][n_kv][D][tcap]
  int64_t layer_stride = 0;
  GenState* state = nullptr;
  const RowState* rows = nullptr;               // != nullptr: a session step, row b at rows->row_len[b]
  const svspec::ColMap* cmap = nullptr;         // != nullptr: a speculative verify step (fused chain, v1 only)
  int H = 0, I = 0, n_head = 0, n_kv = 0, D = 0, qkv_cols = 0, vocab = 0, n_positions = 0, tcap = 0, window = 0;
  float ln_eps = 0.f;
  bool rope = false;                            // StarCoder2: RoPE on q and k before the append
  const bf16 *rope_cos = nullptr, *rope_sin = nullptr, *wte = nullptr, *wpe = nullptr, *lnf_w = nullptr, *lnf_b = nullptr,
             *lm_head = nullptr;
  bf16 *x = nullptr, *ln = nullptr, *qkv = nullptr, *attn = nullptr, *h = nullptr;
  int64_t sx = 0, sln = 0, sqkv = 0, sattn = 0, sh = 0;
  float* attn_partial = nullptr;                // split partials of the per-op attention
  bool lm_tail = true;                          // ln_f + lm_head after the layers
  bf16* logits = nullptr;
  float* amax_val = nullptr;                    // fused chain: the lm_head's argmax partials
  int* amax_idx = nullptr;
};

DecodeChain engine_chain(sv_engine* e, const RowState* rows = nullptr, const svspec::ColMap* cmap = nullptr) {
  const sv_model_desc& d = e->d;
  DecodeChain c;
  c.n_layer = d.n_layer; c.layers = e->dec.data();
  if (e->ring_tiles) { c.t_attn = e->t_attn.data(); c.t_proj = e->t_proj.data(); c.t_fc = e->t_fc.data(); c.t_fc2 = e->t_fc2.data(); }
  c.t_lm_head = (e->ring_tiles && e->t_lm_src == e->lm_head) ? e->t_lm_head : nullptr;
  c.kcache = e->kcache; c.vtcache = e->vtcache; c.layer_stride = e->cache_layer_stride;
  c.state = e->state; c.rows = rows; c.cmap = cmap;
  c.H = d.hidden; c.I = d.n_inner; c.n_head = d.n_head; c.n_kv = d.n_kv_head; c.D = d.head_dim; c.qkv_cols = e->qkv_cols;
  c.vocab = d.vocab; c.n_positions = d.n_positions; c.tcap = e->tcap; c.window = e->window; c.ln_eps = d.ln_eps; c.rope = e->v2;
  c.rope_cos = e->rope_cos; c.rope_sin = e->rope_sin; c.wte = e->wte; c.wpe = e->wpe; c.lnf_w = e->lnf_w; c.lnf_b = e->lnf_b;
  c.lm_head = e->lm_head;
  c.x = e->d_x; c.ln = e->d_ln; c.qkv = e->d_qkv; c.attn = e->d_attn; c.h = e->d_h;
  c.attn_partial = e->attn_partial; c.logits = e->logits; c.amax_val = e->amax_val; c.amax_idx = e->amax_idx;
  return c;
}

inline bf16* slot(bf16* p, int64_t stride, int i) { return p + stride * i; }

// Per-op decode step: embedding, then per layer LayerNorm + rowgroup GEMVs, RoPE (v2), KV append and split attention.
void run_chain_per_op(const DecodeChain& c, const int32_t* ids, int B, int nsplit, cudaStream_t st) {
  const int H = c.H, D = c.D, n = c.n_layer;
  if (ids) launch_embed_tokens(ids, c.wte, c.wpe, c.state, c.x, B, H, c.vocab, c.n_positions, st, c.rows);
  for (int i = 0; i < n; ++i) {
    const DecLayer& L = c.layers[i];
    bf16* kc = c.kcache + c.layer_stride * i;
    bf16* vc = c.vtcache + c.layer_stride * i;
    bf16 *x0 = slot(c.x, c.sx, 2 * i), *x1 = slot(c.x, c.sx, 2 * i + 1), *x2 = slot(c.x, c.sx, 2 * i + 2);
    bf16 *ln1 = slot(c.ln, c.sln, 2 * i), *ln2 = slot(c.ln, c.sln, 2 * i + 1), *qkv = slot(c.qkv, c.sqkv, i);
    bf16 *attn = slot(c.attn, c.sattn, i), *h = slot(c.h, c.sh, i);
    launch_layernorm(x0, L.ln1_w, L.ln1_b, ln1, B, H, c.ln_eps, H, st);
    launch_linear_rowgroup(ln1, L.attn_w, L.attn_b, nullptr, qkv, B, c.qkv_cols, H, SV_ACT_NONE, st);
    if (c.rope)
      launch_rope(qkv, B, 1, c.qkv_cols, c.n_head + c.n_kv, D, c.rope_cos, c.rope_sin, c.state, c.n_positions, 0, st, c.rows);
    launch_kv_append(qkv, kc, vc, c.state, B, c.n_head * D, c.n_kv, D, c.tcap, st, c.rows);
    launch_attention_decode(qkv, c.qkv_cols, kc, vc, attn, c.attn_partial, c.state, B, c.n_head, c.n_kv, D, c.tcap, nsplit,
                            c.window, st, c.rows);
    launch_linear_rowgroup(attn, L.proj_w, L.proj_b, x0, x1, B, H, H, SV_ACT_NONE, st);
    launch_layernorm(x1, L.ln2_w, L.ln2_b, ln2, B, H, c.ln_eps, H, st);
    launch_linear_rowgroup(ln2, L.fc_w, L.fc_b, nullptr, h, B, c.I, H, SV_ACT_GELU_TANH, st);
    launch_linear_rowgroup(h, L.fc2_w, L.fc2_b, x1, x2, B, H, c.I, SV_ACT_NONE, st);
  }
  if (c.lm_tail) {
    bf16* lnf = slot(c.ln, c.sln, 2 * n);
    launch_layernorm(slot(c.x, c.sx, 2 * n), c.lnf_w, c.lnf_b, lnf, B, H, c.ln_eps, H, st);
    launch_linear_rowgroup(lnf, c.lm_head, nullptr, nullptr, c.logits, B, c.vocab, H, SV_ACT_NONE, st);
  }
}

// Fused decode step: 5 kernels per layer (4 weight-ring GEMVs with fused LayerNorm / bias / GELU / residual / KV append,
// 1 cluster attention) + lm_head, chained with programmatic dependent launch.  `ids` != nullptr embeds those tokens first
// (teacher forcing / sampling); with nullptr, x[0] was already written (by select_fused).
// Leaves bf16 logits and per-tile argmax partials in amax_*.
void run_chain_fused(const DecodeChain& c, const int32_t* ids, int B, int ncta, bool pdl, cudaStream_t st) {
  const int H = c.H, D = c.D, n = c.n_layer;
  if (ids) launch_embed_tokens(ids, c.wte, c.wpe, c.state, c.x, B, H, c.vocab, c.n_positions, st, c.rows);
  bool first = true;
  RingGemvLaunch g{};
  g.B = B; g.ln_eps = c.ln_eps; g.n_head = c.n_head; g.n_kv = c.n_kv; g.tcap = c.tcap; g.state = c.state; g.rows = c.rows;
  g.cmap = c.cmap;
  g.amax_val = c.amax_val; g.amax_idx = c.amax_idx;
  auto gemv = [&](const bf16* X, const bf16* W, const uint8_t* Wt, const bf16* bias, const bf16* res, bf16* Y, int N, int K, int act,
                  const bf16* lw, const bf16* lb, int epi, bf16* kc, bf16* vc, bool p) {
    g.X = X; g.W = W; g.Wt = Wt; g.bias = bias; g.res = res; g.Y = Y; g.N = N; g.K = K; g.act = act; g.ln_w = lw; g.ln_b = lb;
    g.epi = epi; g.kcache = kc; g.vtcache = vc; g.pdl = p;
    launch_gemv_ring(g, st);
  };
  for (int i = 0; i < n; ++i) {
    const DecLayer& L = c.layers[i];
    bf16* kc = c.kcache + c.layer_stride * i;
    bf16* vc = c.vtcache + c.layer_stride * i;
    bf16 *x0 = slot(c.x, c.sx, 2 * i), *x1 = slot(c.x, c.sx, 2 * i + 1), *x2 = slot(c.x, c.sx, 2 * i + 2);
    bf16 *qkv = slot(c.qkv, c.sqkv, i), *attn = slot(c.attn, c.sattn, i), *h = slot(c.h, c.sh, i);
    gemv(x0, L.attn_w, c.t_attn ? c.t_attn[i] : nullptr, L.attn_b, nullptr, qkv, c.qkv_cols, H, SV_ACT_NONE, L.ln1_w, L.ln1_b,
         c.rope ? 0 : 1, kc, vc, pdl && !first);
    first = false;
    if (c.rope)   // RoPE on q,k then append (the GEMV epilogue cannot rotate: the pair element lives in another tile)
      launch_rope_append(qkv, B, c.qkv_cols, c.n_head, c.n_kv, D, c.rope_cos, c.rope_sin, kc, vc, c.state, c.tcap,
                         c.n_positions, pdl, st, c.rows);
    launch_attention_decode_cluster(qkv, c.qkv_cols, kc, vc, attn, c.state, B, c.n_head, c.n_kv, D, c.tcap, std::min(ncta, 8),
                                    c.window, pdl, st, c.rows, c.cmap);
    gemv(attn, L.proj_w, c.t_proj ? c.t_proj[i] : nullptr, L.proj_b, x0, x1, H, H, SV_ACT_NONE, nullptr, nullptr, 0, nullptr,
         nullptr, pdl);
    gemv(x1, L.fc_w, c.t_fc ? c.t_fc[i] : nullptr, L.fc_b, nullptr, h, c.I, H, SV_ACT_GELU_TANH, L.ln2_w, L.ln2_b, 0, nullptr,
         nullptr, pdl);
    gemv(h, L.fc2_w, c.t_fc2 ? c.t_fc2[i] : nullptr, L.fc2_b, x1, x2, H, c.I, SV_ACT_NONE, nullptr, nullptr, 0, nullptr, nullptr,
         pdl);
  }
  if (c.lm_tail)
    gemv(slot(c.x, c.sx, 2 * n), c.lm_head, c.t_lm_head, nullptr, nullptr, c.logits, c.vocab, H, SV_ACT_NONE, c.lnf_w, c.lnf_b, 2,
         nullptr, nullptr, pdl);
}

// The attention partition of a decode step whose keys reach total_len: CTAs per image of the cluster kernel (fused chain)
// or key splits of the split / merge kernels (per-op chain).
int decode_parts(bool fused, int total_len) {
  if (fused) return attention_decode_cluster_ncta(total_len);
  return std::max(1, std::min(kMaxSplit, (total_len + 31) / 32));
}

void run_chain(const DecodeChain& c, bool fused, const int32_t* ids, int B, int parts, bool pdl, cudaStream_t st) {
  if (fused) run_chain_fused(c, ids, B, parts, pdl, st);
  else run_chain_per_op(c, ids, B, parts, st);
}

// The engine's step over its own buffers and caches.  rows != nullptr: a session step.  cmap != nullptr: a speculative
// verify step, B columns of one cache row placed by the column map (fused chain, v1 only).
void run_engine_step(sv_engine* e, const int32_t* ids, int B, int parts, bool pdl, cudaStream_t st,
                     const RowState* rows = nullptr, const svspec::ColMap* cmap = nullptr) {
  run_chain(engine_chain(e, rows, cmap), e->fused_decode, ids, B, parts, pdl, st);
}

// Captures `enqueue(pdl)` on `st` into g: the instantiated graph, its kernel count and whether the PDL capture was kept.
// A PDL capture the driver refuses is retried once in plain stream order.  The launch counter active before is restored.
template <typename Enqueue>
cudaError_t capture_step(cudaStream_t st, bool try_pdl, const Enqueue& enqueue, GraphEntry& g) {
  int64_t* const outer = g_launch_counter;
  cudaError_t ce = cudaSuccess;
  for (int attempt = try_pdl ? 0 : 1; attempt < 2; ++attempt) {
    int64_t counted = 0;
    g_launch_counter = &counted;
    cudaGraph_t graph = nullptr;
    ce = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
    if (ce != cudaSuccess) break;
    enqueue(attempt == 0);
    ce = cudaStreamEndCapture(st, &graph);
    if (ce == cudaSuccess) ce = cudaGraphInstantiate(&g.exec, graph, 0);
    if (graph) cudaGraphDestroy(graph);
    if (ce == cudaSuccess) {
      g.kernels = (int)counted;
      g.pdl = attempt == 0;
      break;
    }
    g.exec = nullptr;
    cudaGetLastError();
  }
  g_launch_counter = outer;
  return ce;
}

// Replays the step graph n times on the engine's stream.
int replay(sv_engine* e, const GraphEntry& g, int n) {
  for (int i = 0; i < n; ++i) {
    SV_CK(e, cudaGraphLaunch(g.exec, e->gen_stream));
    e->launches += g.kernels;
  }
  return SV_OK;
}

// Reads n device words into host_flag once the engine's stream has reached this point.
int read_flags(sv_engine* e, const int32_t* dev, int n) {
  SV_CK(e, cudaMemcpyAsync(e->host_flag, dev, n * sizeof(int32_t), cudaMemcpyDeviceToHost, e->gen_stream));
  SV_CK(e, cudaStreamSynchronize(e->gen_stream));
  return SV_OK;
}

// Orders the engine's stream after the work queued so far on the caller's.
int join_caller(sv_engine* e, void* stream) {
  SV_CK(e, cudaEventRecord(e->ev_in, (cudaStream_t)stream));
  SV_CK(e, cudaStreamWaitEvent(e->gen_stream, e->ev_in, 0));
  return SV_OK;
}

// (re)build the slab-tiled copies the dataflow kernel streams, after any weight changed
void ensure_flow_tiles(sv_engine* e, cudaStream_t st) {
  if (!e->use_tiles || (!e->tiles_dirty && e->t_lm_src == e->lm_head)) return;
  const sv_model_desc& d = e->d;
  const int nc = decode_flow_ncta();
  for (int i = 0; i < d.n_layer; ++i) {
    const DecLayer& L = e->dec[i];
    launch_flow_repack(L.attn_w, L.attn_b, e->t_attn[i], e->qkv_cols, d.hidden, nc, st);
    launch_flow_repack(L.proj_w, L.proj_b, e->t_proj[i], d.hidden, d.hidden, nc, st);
    launch_flow_repack(L.fc_w, L.fc_b, e->t_fc[i], d.n_inner, d.hidden, nc, st);
    launch_flow_repack(L.fc2_w, L.fc2_b, e->t_fc2[i], d.hidden, d.n_inner, nc, st);
  }
  launch_flow_repack(e->lm_head, nullptr, e->t_lm_head, d.vocab, d.hidden, nc, st);
  e->t_lm_src = e->lm_head;
  e->tiles_dirty = false;
}

// Both fillers of a FlowLaunch (this one and sv_op_decode_flow's) set every field: a field added to the descriptor changes
// its size, and this assert sends whoever adds it to both.
static_assert(sizeof(FlowLaunch) == 256, "FlowLaunch changed: fill the new field in flow_launch_desc AND sv_op_decode_flow");
FlowLaunch flow_launch_desc(sv_engine* e, int B) {
  FlowLaunch m{};
  m.layers_dev = e->mega_layers; m.n_layer = e->d.n_layer; m.B = B; m.H = e->d.hidden; m.I = e->d.n_inner;
  m.n_head = e->d.n_head; m.n_kv = e->d.n_kv_head; m.qkv_cols = e->qkv_cols; m.vocab = e->d.vocab; m.tcap = e->tcap;
  m.n_positions = e->d.n_positions; m.ln_eps = e->d.ln_eps; m.wte = e->wte; m.wpe = e->wpe; m.lnf_w = e->lnf_w;
  m.lnf_b = e->lnf_b; m.lm_head = e->lm_head; m.lm_head_t = reinterpret_cast<const bf16*>(e->t_lm_head); m.x_plain = e->d_x; m.logits = e->logits;
  m.xa = e->f_xa; m.xb = e->f_xb; m.qkv = e->f_qkv; m.att = e->f_att; m.hb = e->f_hb; m.part = e->f_part; m.amax = e->f_amax;
  m.state = e->state; m.params = e->params; m.seen = e->seen; m.next_ids = e->next_ids; m.out_ids = e->out_ids;
  m.dbg = e->mega_debug ? e->mega_dbg : nullptr;
  m.realloc = e->flow_realloc;
  m.l2_ahead = e->flow_l2_ahead;
  return m;
}

// Token selection from `logits` [B][vocab]: sampling, or greedy through the fused kernel (which also embeds the next step's
// input; `partials`: the lm_head left its argmax partials) on the fused decode path, or the plain greedy kernel.
// rows != nullptr: the session variants, rows in `mask` only, row_len advanced by advance_len.  Without rows, the
// sampling and plain greedy kernels leave the step bookkeeping to launch_gen_finalize.
void launch_token_select(sv_engine* e, const bf16* logits, int B, bool sample, bool partials, int advance_len, bool pdl,
                         cudaStream_t st, RowState* rows = nullptr, uint32_t mask = 0) {
  const sv_model_desc& d = e->d;
  if (sample)
    launch_select_sample(logits, d.vocab, B, e->state, e->params, e->seen, e->next_ids, e->out_ids, e->logits_f32, st, rows,
                         mask, advance_len);
  else if (e->fused_decode)
    launch_select_fused(logits, d.vocab, B, partials ? e->amax_val : nullptr, e->amax_idx, gemv_ring_ntiles(d.vocab),
                        8 * ring_row_groups(B), e->state, e->params, e->seen, e->next_ids, e->out_ids, advance_len, e->wte,
                        e->wpe, e->d_x, d.hidden, d.n_positions, pdl, st, rows, mask);
  else
    launch_select_greedy(logits, d.vocab, B, e->state, e->params, e->seen, e->next_ids, e->out_ids, st, rows, mask, advance_len);
}

// Entry points that use the cache as one rectangle of rows refuse to run while a session holds per-row state in it.
int session_guard(sv_engine* e, const char* what) {
  return e->session ? fail(e, SV_ERR_STATE, "%s: a decode session is open (call sv_session_end first)", what) : SV_OK;
}
#define SV_NO_SESSION(e, what)                 \
  do {                                        \
    int _g = session_guard((e), (what));      \
    if (_g != SV_OK) return _g;               \
  } while (0)

int check_ready(sv_engine* e) {
  for (auto& kv : e->w)
    if (!kv.second.loaded && !kv.second.optional) return fail(e, SV_ERR_STATE, "weight not loaded: %s", kv.first.c_str());
  return SV_OK;
}

}  // namespace

static int finish_prefill_impl(sv_engine* e, int batch, int prefix_len, float* last_logits, cudaStream_t st) {
  e->prefix_len = prefix_len;
  e->host_cur_len = e->prefix_len;
  GenState hs;
  memset(&hs, 0, sizeof(hs));
  hs.cur_len = e->prefix_len;
  for (int b = 0; b < batch; ++b) hs.unfinished[b] = 1;
  SV_CK(e, cudaMemcpyAsync(e->state, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));   // pageable: staged synchronously
  ensure_flow_tiles(e, st);          // (no-op unless a weight changed since the last sequence)
  if (e->use_flow) {                 // new sequence: no word of the exchange buffers may carry a tag of the coming epochs
    SV_CK(e, cudaMemsetAsync(e->flow_mem, 0, e->flow_bytes, st));
    e->flow_epoch = 0;
  }
  if (last_logits) launch_logits_to_float(e->logits, last_logits, (int64_t)batch * e->d.vocab, st);
  SV_CK(e, cudaGetLastError());
  e->prefilled = true;
  return SV_OK;
}

static int finish_prefill(sv_engine* e, int batch, int prefix_len, float* last_logits, cudaStream_t st) {
  LaunchScope scope(e);
  return finish_prefill_impl(e, batch, prefix_len, last_logits, st);
}

// =============================================================================================
extern "C" {

int sv_abi_version(void) { return SV_ABI_VERSION; }

const char* sv_last_error(const sv_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int sv_engine_create(const sv_model_desc* desc, int device, sv_engine** out) {
  if (!desc || !out) return fail(nullptr, SV_ERR_INVALID, "null argument");
  *out = nullptr;
  const sv_model_desc& d = *desc;
  if (d.variant != 0 && d.variant != 1) return fail(nullptr, SV_ERR_UNSUPPORTED, "unknown model variant %d", d.variant);
  if (d.variant == 1 && !(d.rope_theta > 1.0f)) return fail(nullptr, SV_ERR_INVALID, "variant 1 (StarCoder2) needs rope_theta > 1");
  if (d.variant == 1 && d.sliding_window < 0) return fail(nullptr, SV_ERR_INVALID, "sliding_window must be >= 0");
  if (d.vit_width != d.vit_heads * 64) return fail(nullptr, SV_ERR_INVALID, "ViT head dim must be 64");
  if (d.head_dim != 128 || d.hidden != d.n_head * d.head_dim) return fail(nullptr, SV_ERR_INVALID, "decoder head dim must be 128 and hidden == n_head*128");
  if (d.hidden % 64 || d.n_inner % 64) return fail(nullptr, SV_ERR_INVALID, "decoder widths must be multiples of 64");
  if (d.n_kv_head < 1 || d.n_head % d.n_kv_head || d.n_head / d.n_kv_head > 16) return fail(nullptr, SV_ERR_INVALID, "need 1 <= n_head/n_kv_head <= 16");
  if (d.image_size % d.patch_size) return fail(nullptr, SV_ERR_INVALID, "image_size %% patch_size != 0");
  if (d.vit_width % 64 || d.vit_mlp % 64 || d.hidden % 64 || d.n_inner % 64) return fail(nullptr, SV_ERR_INVALID, "widths must be multiples of 64");
  if (d.max_batch < 1 || d.max_batch > 16) return fail(nullptr, SV_ERR_INVALID, "max_batch must be in [1,16] (decode kernels hold two groups of 8 rows per MMA)");
  if (d.adapter_norm != 0 && d.adapter_norm != 1) return fail(nullptr, SV_ERR_INVALID, "adapter_norm must be 0 or 1");
  if (d.vocab < 8 || d.vocab > (1 << 20)) return fail(nullptr, SV_ERR_INVALID, "vocab out of range");

  int ndev = 0;
  cudaError_t r = cudaGetDeviceCount(&ndev);
  if (r != cudaSuccess || ndev <= device)
    return fail(nullptr, SV_ERR_CUDA, "no CUDA device %d (%s): this engine has no CPU fallback", device,
                r == cudaSuccess ? "device count too small" : cudaGetErrorString(r));
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0)
    return fail(nullptr, SV_ERR_CUDA, "device %d is sm_%d%d; kernels are built for sm_90a (H100) only", device, prop.major, prop.minor);
  if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, SV_ERR_CUDA, "cudaSetDevice(%d) failed", device);

  sv_engine* e = new sv_engine();
  e->d = d;
  e->device = device;
  const int g = d.image_size / d.patch_size;
  e->NP = g * g;
  e->v2 = d.variant == 1;
  e->Q = e->NP + (e->v2 ? 0 : 1);                       // SigLIP has no class token
  if (e->v2) {
    e->vit_eps = d.vit_ln_eps > 0.f ? d.vit_ln_eps : 1e-6f;
    e->vit_act = SV_ACT_GELU_TANH;
    e->window = d.sliding_window;
  }
  e->Kp = (3 * d.patch_size * d.patch_size + 63) / 64 * 64;
  e->Lpad = (e->Q + 31) / 32 * 32;
  e->qkv_cols = d.hidden + 2 * d.n_kv_head * d.head_dim;
  int max_len = std::min(d.max_len, d.n_positions);
  if (max_len < e->Q + 2) { delete e; return fail(nullptr, SV_ERR_INVALID, "max_len %d smaller than the visual prefix", d.max_len); }
  e->d.max_len = max_len;
  e->tcap = (max_len + 1 + 31) / 32 * 32;
  const char* impl = getenv("SV_LINEAR_IMPL");
  if (impl && !strcmp(impl, "rowgroup")) e->linear_impl = SV_LINEAR_ROWGROUP;
  if (impl && !strcmp(impl, "tcgen05")) e->linear_impl = SV_LINEAR_TCGEN05;
  const char* dec = getenv("SV_DECODE");          // "legacy" = the unfused per-op kernels (A/B checks)
  if (dec && !strcmp(dec, "legacy")) e->fused_decode = false;
  const char* pdl = getenv("SV_PDL");             // "0" = plain stream order between decode kernels
  if (pdl && !strcmp(pdl, "0")) e->use_pdl = false;
  e->mega_debug = getenv("SV_MEGA_DEBUG") != nullptr;
  { const char* fl = getenv("SV_FLOW");          // "1": dataflow persistent kernel for greedy decode / teacher forcing (opt-in: the
    // per-phase CUDA graph is still faster, DESIGN.md §4); "3": the same without setmaxnreg register reallocation
    e->use_flow = fl && (!strcmp(fl, "1") || !strcmp(fl, "2") || !strcmp(fl, "3"));
    e->flow_requested = e->use_flow;
    if (d.max_batch > 8) e->use_flow = false;     // the dataflow kernel holds 8 rows (decode_flow_supported); no tiled copies
    e->flow_realloc = !(fl && !strcmp(fl, "3"));
    const char* la = getenv("SV_FLOW_L2AHEAD");
    if (la) e->flow_l2_ahead = std::max(0, std::min(64, atoi(la))); }
  if (!gemv_ring_supported(d.hidden, true) || !gemv_ring_supported(d.n_inner, false)) e->fused_decode = false;
  // v1 appends K/V in the c_attn GEMV's epilogue, which the streamed-LayerNorm kernels do not have
  if (!e->v2 && gemv_ring_ln_streamed(d.hidden)) e->fused_decode = false;
  // v2 at full size: the per-op kernels measure faster (4.4 vs 5.8 ms/token at 8B; 768-wide slabs + per-slab LayerNorm
  // on the consumer path), so the fused ring step is opt-in for v2 (SV_DECODE=fused) until that is fixed.
  if (e->v2 && !(dec && !strcmp(dec, "fused"))) e->fused_decode = false;
  // above 8 rows the fused step needs the 16-row ring kernels: v1 without a streamed LayerNorm (they have none) and
  // 8 consumer warps
  if (d.max_batch > 8 && (e->v2 || gemv_ring_ln_streamed(d.hidden) || d.max_batch > gemv_ring_max_rows())) e->fused_decode = false;
  if (!build_weights(e) || !build_buffers(e)) {
    std::string msg = std::string("device allocation failed: ") + cudaGetErrorString(cudaGetLastError());
    sv_engine_destroy(e);
    return fail(nullptr, SV_ERR_CUDA, "%s", msg.c_str());
  }
  if (e->v2) {
    launch_rope_table(e->rope_cos, e->rope_sin, d.n_positions, d.head_dim, d.rope_theta, nullptr);
    if (cudaDeviceSynchronize() != cudaSuccess) {
      sv_engine_destroy(e);
      return fail(nullptr, SV_ERR_CUDA, "RoPE table setup failed");
    }
  }
  {
    std::vector<MegaLayer> ml(d.n_layer);
    for (int i = 0; i < d.n_layer; ++i) {
      const DecLayer& L = e->dec[i];
      ml[i] = MegaLayer{L.ln1_w, L.ln1_b, L.attn_w, L.attn_b, L.proj_w, L.proj_b, L.ln2_w, L.ln2_b, L.fc_w, L.fc_b,
                        L.fc2_w, L.fc2_b, e->kcache + e->cache_layer_stride * i, e->vtcache + e->cache_layer_stride * i,
                        nullptr, nullptr, nullptr, nullptr};
    }
    // slab-tiled copies of the decode weights (one bulk copy per ring slot instead of one per weight row): what the dataflow
    // kernel streams (SV_FLOW=1), and optionally the ring GEMVs of the graph path (SV_TILED=1).  The default keeps ONE copy
    // of the decoder in HBM (row-major) and leaves the tiled copy opt-in.
    const char* tl = getenv("SV_TILED");
    const bool want_tiles = e->use_flow || (tl && !strcmp(tl, "1"));
    if (want_tiles && decode_flow_init() == cudaSuccess && e->fused_decode && decode_flow_ncta() == gemv_ring_ncta()) {
      const int nc = decode_flow_ncta();
      e->use_tiles = true;
      e->ring_tiles = tl && !strcmp(tl, "1");
      bool ok = true;
      auto tiled = [&](int N, int K) -> uint8_t* {
        uint8_t* p = nullptr;
        ok = ok && dev_alloc(e, &p, (int64_t)flow_tiled_bytes(N, K, nc)) == cudaSuccess;
        return p;
      };
      e->t_attn.resize(d.n_layer); e->t_proj.resize(d.n_layer); e->t_fc.resize(d.n_layer); e->t_fc2.resize(d.n_layer);
      for (int i = 0; i < d.n_layer; ++i) {
        e->t_attn[i] = tiled(e->qkv_cols, d.hidden); e->t_proj[i] = tiled(d.hidden, d.hidden);
        e->t_fc[i] = tiled(d.n_inner, d.hidden); e->t_fc2[i] = tiled(d.hidden, d.n_inner);
        ml[i].attn_t = reinterpret_cast<const bf16*>(e->t_attn[i]); ml[i].proj_t = reinterpret_cast<const bf16*>(e->t_proj[i]);
        ml[i].fc_t = reinterpret_cast<const bf16*>(e->t_fc[i]); ml[i].fc2_t = reinterpret_cast<const bf16*>(e->t_fc2[i]);
      }
      e->t_lm_head = tiled(d.vocab, d.hidden);
      if (!ok) { sv_engine_destroy(e); return fail(nullptr, SV_ERR_CUDA, "allocation of the tiled decode weights failed"); }
    }
    if (cudaMemcpy(e->mega_layers, ml.data(), ml.size() * sizeof(MegaLayer), cudaMemcpyHostToDevice) != cudaSuccess ||
        decode_flow_init() != cudaSuccess || gemv_ring_init() != cudaSuccess) {
      sv_engine_destroy(e);
      return fail(nullptr, SV_ERR_CUDA, "persistent decode kernel setup failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    if (!decode_flow_supported(d.hidden, d.n_inner, d.head_dim, d.max_batch, e->window, e->v2) || !e->fused_decode || d.n_layer > decode_flow_max_layers() ||
        d.max_len > decode_flow_max_keys() || !e->use_tiles) e->use_flow = false;
    if (e->flow_realloc && !decode_flow_realloc_supported()) e->flow_realloc = false;
  }
  if (attention_decode_cluster_init() != cudaSuccess) {
    sv_engine_destroy(e);
    return fail(nullptr, SV_ERR_CUDA, "cannot raise the shared-memory limit of the decode attention kernel");
  }
  if (cudaStreamCreateWithFlags(&e->gen_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&e->ev_t0) != cudaSuccess || cudaEventCreate(&e->ev_t1) != cudaSuccess) {
    sv_engine_destroy(e);
    return fail(nullptr, SV_ERR_CUDA, "stream/event creation failed");
  }
  *out = e;
  return SV_OK;
}

void sv_engine_destroy(sv_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  for (auto& g : e->step_graphs) if (g.second.exec) cudaGraphExecDestroy(g.second.exec);
  for (void* p : e->allocs) cudaFree(p);
  if (e->host_flag) cudaFreeHost(e->host_flag);
  if (e->host_stream) cudaFreeHost(e->host_stream);
  if (e->rows_host) cudaFreeHost(e->rows_host);
  if (e->gen_stream) cudaStreamDestroy(e->gen_stream);
  if (e->ev_in) cudaEventDestroy(e->ev_in);
  if (e->ev_t0) cudaEventDestroy(e->ev_t0);
  if (e->ev_t1) cudaEventDestroy(e->ev_t1);
  delete e;
}

int sv_engine_load_weight(sv_engine* e, const char* hf_name, const void* data, const int64_t* shape, int32_t ndim,
                          int32_t dtype) {
  if (!e || !hf_name || !data || !shape) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_engine_load_weight");    // rows admitted earlier would continue on other weights
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  std::string name = hf_name;
  auto ends_with = [&](const char* s) { size_t n = strlen(s); return name.size() >= n && !name.compare(name.size() - n, n, s); };
  if (ends_with("num_batches_tracked") || ends_with(".attn.bias") || ends_with("transformer.bias") ||
      ends_with(".attn.masked_bias") || ends_with("rotary_emb.inv_freq") || ends_with("embeddings.position_ids"))
    return SV_OK;   // buffers that carry no parameters
  if (name.find("visual_encoder.head.") != std::string::npos)
    return SV_OK;   // SigLIP pooling head: computed and discarded by the reference (image_encoder.py:109)
  int64_t numel = 1;
  for (int i = 0; i < ndim; ++i) numel *= shape[i];
  if (name == LMH && e->w.find(name) == e->w.end()) {   // explicit (un-tied) lm_head
    const sv_model_desc& d = e->d;
    bf16* p = add_weight(e, name, {(int64_t)d.vocab, (int64_t)d.hidden}, -1, true);
    if (!p) return fail(e, SV_ERR_CUDA, "allocation failed for lm_head");
    e->lm_head = p;
  }
  auto it = e->w.find(name);
  if (it == e->w.end()) return fail(e, SV_ERR_INVALID, "unknown weight name: %s", hf_name);
  Weight& wt = it->second;
  if (numel != wt.numel || ndim != (int)wt.shape.size())
    return fail(e, SV_ERR_INVALID, "shape mismatch for %s: got %lld elements / %d dims, expected %lld / %zu", hf_name,
                (long long)numel, ndim, (long long)wt.numel, wt.shape.size());
  for (int i = 0; i < ndim; ++i)
    if (shape[i] != wt.shape[i]) return fail(e, SV_ERR_INVALID, "shape mismatch for %s at dim %d", hf_name, i);
  if (dtype == SV_DTYPE_BF16) {
    SV_CK(e, cudaMemcpy(wt.p, data, (size_t)numel * 2, cudaMemcpyDefault));
  } else if (dtype == SV_DTYPE_F32 || dtype == SV_DTYPE_F16) {
    const size_t es = dtype == SV_DTYPE_F32 ? 4 : 2;
    void* tmp = nullptr;
    SV_CK(e, cudaMalloc(&tmp, (size_t)numel * es));
    cudaError_t r = cudaMemcpy(tmp, data, (size_t)numel * es, cudaMemcpyDefault);
    if (r == cudaSuccess) {
      launch_convert_to_bf16(tmp, dtype, wt.p, numel, nullptr);
      r = cudaDeviceSynchronize();
    }
    cudaFree(tmp);
    SV_CK(e, r);
  } else {
    return fail(e, SV_ERR_INVALID, "unsupported dtype %d", dtype);
  }
  if (wt.p == e->conv_raw) {   // [W,3,p,p] -> [W, Kp] zero padded GEMM operand
    launch_pad_rows(e->conv_raw, e->conv_w, e->d.vit_width, 3 * e->d.patch_size * e->d.patch_size, e->Kp, nullptr);
    SV_CK(e, cudaDeviceSynchronize());
  }
  wt.loaded = true;
  e->tiles_dirty = true;
  return SV_OK;
}

int sv_engine_missing_weights(sv_engine* e) {
  if (!e) return SV_ERR_INVALID;
  int n = 0;
  std::string names;
  for (auto& kv : e->w)
    if (!kv.second.loaded && !kv.second.optional) { ++n; names += kv.first + "\n"; }
  e->err = names;
  return n;
}

int sv_encode_images(sv_engine* e, const void* pixels, int32_t batch, void* out_embeds, void* vit_out, void* stream) {
  if (!e || !pixels) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_encode_images");
  if (batch < 1 || batch > e->d.max_batch) return fail(e, SV_ERR_INVALID, "batch %d outside [1,%d]", batch, e->d.max_batch);
  int r = check_ready(e);
  if (r != SV_OK) return r;
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = (cudaStream_t)stream;
  r = run_encode(e, (const bf16*)pixels, batch, st);
  if (r != SV_OK) return r;
  const size_t M = (size_t)batch * e->Q;
  if (out_embeds) SV_CK(e, cudaMemcpyAsync(out_embeds, e->visual, M * e->d.hidden * 2, cudaMemcpyDeviceToDevice, st));
  if (vit_out) SV_CK(e, cudaMemcpyAsync(vit_out, e->v_out, M * e->d.vit_width * 2, cudaMemcpyDeviceToDevice, st));
  SV_CK(e, cudaGetLastError());
  e->cur_batch = batch;
  e->encoded = true;
  e->prefilled = false;
  return SV_OK;
}

int sv_prefill(sv_engine* e, const int32_t* prompt_ids, int32_t batch, int32_t prompt_len, float* last_logits,
               void* stream) {
  if (!e || !prompt_ids) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_prefill");
  if (!e->encoded || batch != e->cur_batch) return fail(e, SV_ERR_STATE, "sv_prefill needs sv_encode_images with the same batch first");
  if (prompt_len < 1 || prompt_len > kMaxPrompt) return fail(e, SV_ERR_INVALID, "prompt_len %d outside [1,%d]", prompt_len, kMaxPrompt);
  if (e->Q + prompt_len + 1 > e->d.max_len) return fail(e, SV_ERR_INVALID, "prefix longer than max_len");
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = (cudaStream_t)stream;
  int r = run_prefill(e, e->visual, e->Q, prompt_ids, batch, prompt_len, st);
  if (r != SV_OK) return r;
  return finish_prefill(e, batch, e->Q + prompt_len, last_logits, st);
}

int sv_prefill_embeds(sv_engine* e, const void* inputs_embeds, int32_t batch, int32_t seq_len, float* last_logits,
                      void* stream) {
  if (!e || !inputs_embeds) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_prefill_embeds");
  if (batch < 1 || batch > e->d.max_batch) return fail(e, SV_ERR_INVALID, "batch %d outside [1,%d]", batch, e->d.max_batch);
  if (seq_len < 1 || seq_len > e->Q + kMaxPrompt) return fail(e, SV_ERR_INVALID, "seq_len %d outside [1,%d]", seq_len, e->Q + kMaxPrompt);
  if (seq_len + 1 > e->d.max_len) return fail(e, SV_ERR_INVALID, "prefix longer than max_len");
  int r = check_ready(e);
  if (r != SV_OK) return r;
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = (cudaStream_t)stream;
  r = run_prefill(e, (const bf16*)inputs_embeds, seq_len, nullptr, batch, 0, st);
  if (r != SV_OK) return r;
  e->cur_batch = batch;
  return finish_prefill(e, batch, seq_len, last_logits, st);
}

int sv_decode_step(sv_engine* e, const int32_t* ids, float* logits, void* stream) {
  if (!e || !ids) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_decode_step");
  if (!e->prefilled) return fail(e, SV_ERR_STATE, "sv_decode_step needs sv_prefill first");
  if (e->host_cur_len + 1 > e->d.max_len) return fail(e, SV_ERR_INVALID, "KV cache full (max_len %d)", e->d.max_len);
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = (cudaStream_t)stream;
  if (e->use_flow) {
    // one token through the dataflow kernel: embed (plain) -> all layers -> logits, no selection
    const sv_model_desc& d = e->d;
    launch_embed_tokens(ids, e->wte, e->wpe, e->state, e->d_x, e->cur_batch, d.hidden, d.vocab, d.n_positions, st);
    ensure_flow_tiles(e, st);
    FlowLaunch m = flow_launch_desc(e, e->cur_batch);
    m.nsteps = 1; m.step0 = e->flow_epoch; m.cur_len0 = e->host_cur_len; m.first_plain = 1; m.do_select = 0;
    cudaError_t ce = launch_decode_flow(m, st);
    if (ce != cudaSuccess) return fail(e, SV_ERR_CUDA, "dataflow decode launch failed: %s", cudaGetErrorString(ce));
    e->flow_epoch += 1;
    launch_advance_len(e->state, st);
  } else {
    run_engine_step(e, ids, e->cur_batch, decode_parts(e->fused_decode, e->host_cur_len + 1), e->use_pdl, st);
    launch_advance_len(e->state, st);
  }
  if (logits) launch_logits_to_float(e->logits, logits, (int64_t)e->cur_batch * e->d.vocab, st);
  SV_CK(e, cudaGetLastError());
  e->host_cur_len += 1;
  return SV_OK;
}

int sv_score_tokens(sv_engine* e, const int32_t* ids, int32_t batch, int32_t n_tokens, float* logprobs, void* stream) {
  if (!e || !ids || !logprobs) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_score_tokens");
  if (!e->prefilled) return fail(e, SV_ERR_STATE, "sv_score_tokens needs sv_prefill first");
  if (batch != e->cur_batch) return fail(e, SV_ERR_INVALID, "batch %d != the current batch %d", batch, e->cur_batch);
  if (n_tokens < 1) return fail(e, SV_ERR_INVALID, "n_tokens must be >= 1");
  if ((int64_t)e->host_cur_len + n_tokens > e->d.max_len)
    return fail(e, SV_ERR_INVALID, "cache length %d + n_tokens %d exceeds max_len %d", e->host_cur_len, n_tokens, e->d.max_len);
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = (cudaStream_t)stream;
  const sv_model_desc& d = e->d;
  if (!e->s_x) {
    const int64_t R = kScoreRows;
    bool ok = true;
#define SAL(ptr, n) ok = ok && (dev_alloc(e, &e->ptr, (n)) == cudaSuccess)
    SAL(s_ln, R * d.hidden); SAL(s_qkv, R * e->qkv_cols); SAL(s_attn, R * d.hidden); SAL(s_h, R * d.n_inner);
    SAL(s_tgt, R); SAL(s_part, R * lm_logprob_ntiles(d.vocab)); SAL(s_tl, R); SAL(s_x, R * d.hidden);
#undef SAL
    if (!ok) { e->s_x = nullptr; return fail(e, SV_ERR_CUDA, "allocation of the scoring buffers failed: %s", cudaGetErrorString(cudaGetLastError())); }
  }
  const int B = batch, n = n_tokens, pos0 = e->host_cur_len, C = std::max(1, kScoreRows / B);
  // position 0: from the logits the previous call left resident, with the same partials + merge
  launch_score_targets(ids, n, -1, B, 1, d.vocab, e->s_tgt, st);
  launch_logits_logprob_partials(e->logits, d.vocab, B, e->s_tgt, e->s_part, e->s_tl, st);
  launch_logprob_merge(e->s_part, lm_logprob_ntiles(d.vocab), e->s_tl, B, 1, 0, n, logprobs, st);
  for (int c0 = 0; c0 < n; c0 += C) {
    const int Cc = std::min(C, n - c0);
    int r = run_score_chunk(e, ids, n, c0, Cc, B, pos0 + c0, logprobs, c0 + Cc == n, st);
    if (r != SV_OK) return r;
  }
  SV_CK(e, cudaGetLastError());
  // the scored tokens extend the prefix: a decode step, another scoring call or a generation continues from here
  return finish_prefill_impl(e, B, pos0 + n, nullptr, st);
}

// What every entry point checks in sv_gen_params: nullptr, or what is wrong.
static const char* gen_params_error(const sv_gen_params& p) {
  if (p.n_stop_ids < 0 || p.n_stop_ids > 8) return "n_stop_ids outside [0, 8]";
  if (p.do_sample && !(p.temperature > 0.f)) return "temperature must be > 0";
  if (!(p.repetition_penalty > 0.f)) return "repetition_penalty must be > 0";
  return nullptr;
}

// The device-side generation parameters (n_stop_ids already checked to lie in [0, 8]).
static GenParamsDev gen_params_dev(const sv_gen_params* p, int stop_row0_only, int out_stride) {
  GenParamsDev hp;
  memset(&hp, 0, sizeof(hp));
  hp.max_new = p->max_new_tokens; hp.do_sample = p->do_sample; hp.eos_id = p->eos_token_id; hp.pad_id = p->pad_token_id;
  hp.n_stop = p->n_stop_ids;
  for (int i = 0; i < p->n_stop_ids; ++i) hp.stop_ids[i] = p->stop_ids[i];
  hp.stop_row0_only = stop_row0_only; hp.out_stride = out_stride;
  hp.temperature = p->temperature; hp.top_p = p->top_p; hp.rep_penalty = p->repetition_penalty; hp.seed = p->seed;
  return hp;
}

// The generate loop.  `cb` (optional) receives the new tokens of every row each time the host polls the device
// (sv_generate_stream); with cb == NULL the code path is exactly sv_generate's.  `spec` != NULL: prompt-lookup
// speculative decoding (sv_generate_speculative): every replay of the step graph verifies k + 1 columns of the one cache
// row and emits 1 to k + 1 tokens.
static int generate_impl(sv_engine* e, const sv_gen_params* p, int32_t* out_ids, int32_t* out_len, void* stream,
                         sv_token_callback cb, void* cb_user, const sv_spec_params* spec = nullptr) {
  if (!e) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_generate");
  if (!p || !out_ids) return fail(e, SV_ERR_INVALID, "null argument");
  if (!e->prefilled) return fail(e, SV_ERR_STATE, "sv_generate needs sv_prefill first");
  if (e->host_cur_len != e->prefix_len) return fail(e, SV_ERR_STATE, "sv_generate must directly follow sv_prefill");
  const int B = e->cur_batch, max_new = p->max_new_tokens;
  if (max_new < 1) return fail(e, SV_ERR_INVALID, "max_new_tokens must be >= 1");
  if (e->prefix_len + max_new > e->d.max_len)
    return fail(e, SV_ERR_INVALID, "prefix %d + max_new_tokens %d exceeds max_len %d", e->prefix_len, max_new, e->d.max_len);
  if (const char* bad = gen_params_error(*p)) return fail(e, SV_ERR_INVALID, "%s", bad);
  const int ncols = spec ? spec->num_tokens + 1 : 0;
  if (spec) {
    if (e->v2) return fail(e, SV_ERR_UNSUPPORTED, "sv_generate_speculative: v2 engines decode through the per-op kernels; only v1 is built");
    if (!e->fused_decode) return fail(e, SV_ERR_UNSUPPORTED, "sv_generate_speculative needs the fused graph decode path (SV_DECODE=legacy is set)");
    if (B != 1) return fail(e, SV_ERR_UNSUPPORTED, "sv_generate_speculative decodes one image; batch is %d", B);
    if (spec->num_tokens < 1 || ncols > e->d.max_batch || ncols > svspec::kMaxCols)
      return fail(e, SV_ERR_INVALID, "prompt_lookup_num_tokens %d outside [1, %d] (max_batch - 1)", spec->num_tokens,
                  std::min(e->d.max_batch, svspec::kMaxCols) - 1);
    if (spec->max_matching_ngram_size < 1)
      return fail(e, SV_ERR_INVALID, "max_matching_ngram_size must be >= 1, got %d", spec->max_matching_ngram_size);
  }
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  if (spec && !e->spec && dev_alloc(e, &e->spec, 1) != cudaSuccess)
    return fail(e, SV_ERR_CUDA, "allocation of the speculative decoding state failed: %s", cudaGetErrorString(cudaGetLastError()));
  cudaStream_t st = e->gen_stream;
  SV_TRY(join_caller(e, stream));

  const GenParamsDev hp = gen_params_dev(p, p->stop_row0_only, e->d.max_len);
  SV_CK(e, cudaMemcpyAsync(e->params, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));
  SV_CK(e, cudaMemsetAsync(e->seen, 0, (size_t)B * e->d.vocab, st));
  launch_fill_i32(e->out_ids, p->pad_token_id, B * e->d.max_len, st);

  // token 0 comes from the prefill logits.  Greedy on the fused path: one kernel selects, applies the
  // HF stop rules and embeds the token for the first decode step.
  const bool fused = e->fused_decode;
  const bool fused_select = fused && !p->do_sample;
  auto select_step = [&](int advance_len, bool have_partials, bool pdl) {
    launch_token_select(e, e->logits, B, p->do_sample, have_partials, advance_len, pdl, st);
    if (!fused_select) launch_gen_finalize(e->state, e->params, B, advance_len, st);
  };
  select_step(/*advance_len=*/0, /*have_partials=*/false, /*pdl=*/false);
  if (spec) {   // nothing to accept yet (n_live = 0): the first drafts, the column map and the columns' embeddings
    svspec::State hs;
    memset(&hs, 0, sizeof(hs));
    hs.ncols = ncols; hs.k = spec->num_tokens; hs.max_ngram = spec->max_matching_ngram_size;
    SV_CK(e, cudaMemcpyAsync(e->spec, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));   // pageable: staged synchronously
    launch_spec_accept(e->state, e->params, e->seen, e->next_ids, e->out_ids, e->d.vocab, e->wte, e->wpe, e->d_x,
                       e->d.hidden, e->d.n_positions, e->spec, false, st);
  }

  const int parts = decode_parts(fused, e->prefix_len + max_new);
  GraphEntry& ge = e->step_graphs[{spec ? StepKind::speculative : StepKind::generate, spec ? ncols : B, parts, p->do_sample != 0,
                                   fused, e->use_pdl}];
  const bool flow = e->use_flow && fused_select && !spec;
  auto step = [&](bool pdl) {
    if (spec) {           // verify step: the columns' inputs were embedded by the previous accept
      run_engine_step(e, nullptr, ncols, parts, pdl, st, nullptr, &e->spec->map);
      if (fused_select) {
        launch_select_fused_spec(e->logits, e->d.vocab, e->amax_val, e->amax_idx, gemv_ring_ntiles(e->d.vocab),
                                 8 * ring_row_groups(ncols), e->state, e->params, e->seen, e->next_ids, e->out_ids, e->wte,
                                 e->wpe, e->d_x, e->d.hidden, e->d.n_positions, e->spec, pdl, st);
      } else {
        launch_select_sample_spec(e->logits, e->d.vocab, ncols, e->state, e->params, e->seen, e->logits_f32, e->spec, st);
        launch_spec_accept(e->state, e->params, e->seen, e->next_ids, e->out_ids, e->d.vocab, e->wte, e->wpe, e->d_x,
                           e->d.hidden, e->d.n_positions, e->spec, false, st);
      }
    } else {
      run_engine_step(e, fused_select ? nullptr : e->next_ids, B, parts, pdl, st);
      select_step(/*advance_len=*/1, /*have_partials=*/fused, pdl);
    }
  };
  if (!ge.exec && max_new > 1 && !flow) {
    SV_CK(e, capture_step(st, e->use_pdl && fused, step, ge));
    if (fused && !ge.pdl) e->use_pdl = false;     // programmatic edges refused by this driver: plain stream order
  }

  const int poll = p->poll_interval > 0 ? p->poll_interval : 16;
  const bool can_stop = p->eos_token_id >= 0 || p->n_stop_ids > 0;
  // streaming: at every poll, tokens [emitted, step) of every row go to the callback through a pinned staging buffer
  int emitted = 0;
  bool cancelled = false;
  auto emit_upto = [&](int upto) -> int {          // `st` must be idle (synchronised) when this is called
    while (cb && emitted < upto) {
      const int n = std::min(upto - emitted, kStreamChunk);
      if (!e->host_stream) SV_CK(e, cudaMallocHost(reinterpret_cast<void**>(&e->host_stream), (size_t)e->d.max_batch * kStreamChunk * 4));
      SV_CK(e, cudaMemcpy2DAsync(e->host_stream, (size_t)n * 4, e->out_ids + emitted, (size_t)e->d.max_len * 4, (size_t)n * 4, B,
                                 cudaMemcpyDeviceToHost, st));
      SV_CK(e, cudaStreamSynchronize(st));
      if (cb(cb_user, e->host_stream, B, emitted, n) != 0) cancelled = true;
      emitted += n;
    }
    return SV_OK;
  };
  auto poll_device = [&](bool& done_flag) -> int {  // {step, done} into host_flag, then the new tokens when streaming
    SV_TRY(read_flags(e, &e->state->step, 2));
    done_flag = e->host_flag[1] != 0;
    SV_TRY(emit_upto(std::min(e->host_flag[0], max_new)));
    if (cancelled) done_flag = true;
    return SV_OK;
  };
  SV_CK(e, cudaEventRecord(e->ev_t0, st));
  int steps = 0;
  bool done = false;
  if (flow) {
    // dataflow persistent kernel: up to `chunk` whole tokens per cooperative launch, no host work in between
    const int chunk = (can_stop || cb) ? poll : 512;
    ensure_flow_tiles(e, st);
    FlowLaunch m = flow_launch_desc(e, B);
    m.do_select = 1;
    if (e->mega_debug) cudaMemsetAsync(e->mega_dbg, 0, 8192 * sizeof(long long), st);
    int left = max_new - 1;
    bool first = true;
    while (left > 0 && !done) {
      m.nsteps = std::min(left, chunk);
      m.step0 = e->flow_epoch; m.cur_len0 = e->prefix_len + steps; m.first_plain = first ? 1 : 0;
      cudaError_t ce = launch_decode_flow(m, st);
      if (ce != cudaSuccess) return fail(e, SV_ERR_CUDA, "dataflow decode launch failed: %s", cudaGetErrorString(ce));
      first = false;
      m.dbg = nullptr;
      e->flow_epoch += m.nsteps;
      left -= m.nsteps;
      steps += m.nsteps;
      if ((cb || can_stop) && left > 0) SV_TRY(poll_device(done));
    }
  }
  if (spec) {
    // Each replay emits 1 to k + 1 tokens: replay as many times as the remaining budget needs at full acceptance (at most
    // `poll`), then read {step, done}.  So the device never runs past max_new_tokens, and past the finish only after an
    // EOS or a stop, as the plain loop does.
    int known = 1;
    while (!done && known < max_new) {
      const int n_rep = std::max(1, std::min(poll, (max_new - known + ncols - 1) / ncols));
      SV_TRY(replay(e, ge, n_rep));
      steps += n_rep;
      SV_TRY(poll_device(done));
      known = e->host_flag[0];
    }
  }
  // with neither a callback, an EOS nor a stop sequence armed, no host read and no sync until the end
  for (int s = 1; s < max_new && !done && !flow && !spec; ++s) {
    SV_TRY(replay(e, ge, 1));
    ++steps;
    if ((cb || can_stop) && s % poll == 0) SV_TRY(poll_device(done));
  }
  SV_CK(e, cudaEventRecord(e->ev_t1, st));
  // rectangular result: [B, n_generated] new tokens, padded (HF returns the same rectangle)
  SV_TRY(read_flags(e, &e->state->step, 1));
  const int n_gen = std::min(e->host_flag[0], max_new);
  SV_TRY(emit_upto(n_gen));
  SV_CK(e, cudaMemcpy2DAsync(out_ids, (size_t)max_new * 4, e->out_ids, (size_t)e->d.max_len * 4, (size_t)max_new * 4, B,
                             cudaMemcpyDeviceToDevice, st));
  if (out_len) launch_fill_i32(out_len, n_gen, B, st);
  SV_CK(e, cudaStreamSynchronize(st));
  SV_CK(e, cudaGetLastError());
  SV_CK(e, cudaEventElapsedTime(&e->last_decode_ms, e->ev_t0, e->ev_t1));
  e->last_decode_steps = steps;
  if (spec) SV_CK(e, cudaMemcpy(e->spec_stats, &e->spec->steps, sizeof(e->spec_stats), cudaMemcpyDeviceToHost));
  e->host_cur_len = e->prefix_len + std::max(0, n_gen - 1);
  e->prefilled = false;   // the cache now holds a finished generation; a new prefill is required
  return SV_OK;
}

int sv_generate(sv_engine* e, const sv_gen_params* p, int32_t* out_ids, int32_t* out_len, void* stream) {
  return generate_impl(e, p, out_ids, out_len, stream, nullptr, nullptr);
}

int sv_generate_stream(sv_engine* e, const sv_gen_params* p, int32_t* out_ids, int32_t* out_len, sv_token_callback on_tokens,
                       void* user, void* stream) {
  if (!on_tokens) return fail(e, SV_ERR_INVALID, "sv_generate_stream needs a callback (use sv_generate otherwise)");
  return generate_impl(e, p, out_ids, out_len, stream, on_tokens, user);
}

int sv_generate_speculative(sv_engine* e, const sv_gen_params* p, const sv_spec_params* sp, int32_t* out_ids,
                            int32_t* out_len, sv_token_callback on_tokens, void* user, void* stream) {
  if (!e || !sp) return fail(e, SV_ERR_INVALID, "null argument");
  if (e->session) return fail(e, SV_ERR_UNSUPPORTED, "sv_generate_speculative: a decode session is open (a session speculates when "
                                                     "opened with sv_session_begin_speculative)");
  return generate_impl(e, p, out_ids, out_len, stream, on_tokens, user, sp);
}

int sv_last_spec_stats(const sv_engine* e, int32_t* steps, int32_t* drafted, int32_t* accepted) {
  if (!e) return SV_ERR_INVALID;
  if (steps) *steps = e->spec_stats[0];
  if (drafted) *drafted = e->spec_stats[1];
  if (accepted) *accepted = e->spec_stats[2];
  return SV_OK;
}

int sv_spec_verify_step(sv_engine* e, const int32_t* ids_host, int32_t ncols, float* logits, void* stream) {
  if (!e || !ids_host || !logits) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_spec_verify_step");
  if (e->v2 || !e->fused_decode) return fail(e, SV_ERR_UNSUPPORTED, "sv_spec_verify_step: v1 engines on the fused decode path only");
  if (!e->prefilled || e->cur_batch != 1) return fail(e, SV_ERR_STATE, "sv_spec_verify_step needs a one-image prefill first");
  if (ncols < 1 || ncols > std::min(e->d.max_batch, svspec::kMaxCols))
    return fail(e, SV_ERR_INVALID, "ncols %d outside [1, %d]", ncols, std::min(e->d.max_batch, svspec::kMaxCols));
  if (e->host_cur_len + ncols > e->d.max_len) return fail(e, SV_ERR_INVALID, "KV cache full (max_len %d)", e->d.max_len);
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  if (!e->spec && dev_alloc(e, &e->spec, 1) != cudaSuccess)
    return fail(e, SV_ERR_CUDA, "allocation of the speculative decoding state failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (!e->spec_pos && dev_alloc(e, &e->spec_pos, 1) != cudaSuccess)
    return fail(e, SV_ERR_CUDA, "allocation of the column positions failed: %s", cudaGetErrorString(cudaGetLastError()));
  cudaStream_t st = (cudaStream_t)stream;
  const sv_model_desc& d = e->d;
  svspec::State hs;
  RowState rs;
  memset(&hs, 0, sizeof(hs));
  memset(&rs, 0, sizeof(rs));
  hs.ncols = ncols;
  svspec::set_map(hs.map, ncols, ncols, e->host_cur_len);
  for (int c = 0; c < ncols; ++c) rs.row_len[c] = e->host_cur_len + c;      // the columns' embedding positions
  SV_CK(e, cudaMemcpyAsync(e->spec, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));   // pageable: staged synchronously
  SV_CK(e, cudaMemcpyAsync(e->spec_pos, &rs, sizeof(rs), cudaMemcpyHostToDevice, st));
  SV_CK(e, cudaMemcpyAsync(e->ids_tmp, ids_host, (size_t)ncols * 4, cudaMemcpyHostToDevice, st));
  launch_embed_tokens(e->ids_tmp, e->wte, e->wpe, e->state, e->d_x, ncols, d.hidden, d.vocab, d.n_positions, st, e->spec_pos);
  run_engine_step(e, nullptr, ncols, decode_parts(true, e->host_cur_len + ncols), false, st, nullptr, &e->spec->map);
  launch_logits_to_float(e->logits, logits, (int64_t)ncols * d.vocab, st);
  SV_CK(e, cudaStreamSynchronize(st));
  SV_CK(e, cudaGetLastError());
  return SV_OK;
}

int sv_spec_draft_host(const int32_t* hist, int32_t n, int32_t k, int32_t max_ngram, int32_t eos_id, int32_t budget,
                       int32_t* out) {
  if ((!hist && n > 0) || !out || n < 0 || k < 0 || max_ngram < 1) return SV_ERR_INVALID;
  return svspec::draft_host(hist, n, k, max_ngram, eos_id, budget, out);
}

int sv_spec_accept_host(const sv_gen_params* p, int32_t* state, int32_t* out_ids, int32_t out_stride, const int32_t* sel,
                        const int32_t* cols, int32_t n_live) {
  if (!p || !state || !out_ids || !sel || !cols || n_live < 0 || n_live > svspec::kMaxCols) return SV_ERR_INVALID;
  if (p->n_stop_ids < 0 || p->n_stop_ids > 8 || out_stride < p->max_new_tokens) return SV_ERR_INVALID;
  GenState gs;
  memset(&gs, 0, sizeof(gs));
  gs.cur_len = state[0]; gs.step = state[1]; gs.done = state[2]; gs.unfinished[0] = state[2] ? 0 : 1;
  const GenParamsDev hp = gen_params_dev(p, p->stop_row0_only, out_stride);
  int m = 0;
  if (!gs.done) {
    m = svspec::accept(sel, cols, n_live, [&](int t) {
      int tk[1] = {t};
      select_apply_tokens(tk, 1, /*vocab=*/0, &gs, &hp, nullptr, tk, out_ids, /*advance_len=*/1);
      return gs.done != 0;
    });
  }
  state[0] = gs.cur_len; state[1] = gs.step; state[2] = gs.done;
  return m;
}

int sv_generate_im2svg_host(sv_engine* e, const void* pixels_host, int32_t batch, const int32_t* prompt_ids_host,
                            int32_t prompt_len, const sv_gen_params* p, int32_t* out_ids_host, int32_t* out_len_host,
                            void* stream) {
  if (!e || !pixels_host || !prompt_ids_host || !p || !out_ids_host) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_generate_im2svg_host");
  if (batch < 1 || batch > e->d.max_batch) return fail(e, SV_ERR_INVALID, "batch %d outside [1,%d]", batch, e->d.max_batch);
  if (prompt_len < 1 || prompt_len > kMaxPrompt) return fail(e, SV_ERR_INVALID, "prompt_len outside [1,%d]", kMaxPrompt);
  SV_CK(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  if (p->max_new_tokens < 1 || p->max_new_tokens > e->d.max_len)
    return fail(e, SV_ERR_INVALID, "max_new_tokens %d outside [1,%d]", p->max_new_tokens, e->d.max_len);
  const size_t px_bytes = (size_t)batch * 3 * e->d.image_size * e->d.image_size * 2;
  // device staging of the host entry point: one allocation for the engine's lifetime (no cudaMalloc / cudaFree per call)
  if (!e->im2svg_px && dev_alloc(e, &e->im2svg_px, (int64_t)e->d.max_batch * 3 * e->d.image_size * e->d.image_size) != cudaSuccess)
    return fail(e, SV_ERR_CUDA, "allocation of the pixel staging buffer failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (!e->im2svg_out && dev_alloc(e, &e->im2svg_out, (int64_t)e->d.max_batch * (e->d.max_len + 1)) != cudaSuccess)
    return fail(e, SV_ERR_CUDA, "allocation of the output staging buffer failed: %s", cudaGetErrorString(cudaGetLastError()));
  bf16* px = e->im2svg_px;
  int32_t* dout = e->im2svg_out;
  int32_t* dlen = dout + (size_t)batch * p->max_new_tokens;
  int r = SV_OK;
  cudaError_t ce = cudaMemcpyAsync(px, pixels_host, px_bytes, cudaMemcpyHostToDevice, st);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(e->ids_tmp, prompt_ids_host, (size_t)batch * prompt_len * 4, cudaMemcpyHostToDevice, st);
  if (ce != cudaSuccess) r = fail(e, SV_ERR_CUDA, "H2D copy failed: %s", cudaGetErrorString(ce));
  if (r == SV_OK) r = sv_encode_images(e, px, batch, nullptr, nullptr, stream);
  if (r == SV_OK) r = sv_prefill(e, e->ids_tmp, batch, prompt_len, nullptr, stream);
  if (r == SV_OK) r = sv_generate(e, p, dout, dlen, stream);
  if (r == SV_OK) {
    ce = cudaMemcpyAsync(out_ids_host, dout, (size_t)batch * p->max_new_tokens * 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess && out_len_host) ce = cudaMemcpyAsync(out_len_host, dlen, (size_t)batch * 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) r = fail(e, SV_ERR_CUDA, "D2H copy failed: %s", cudaGetErrorString(ce));
  }
  cudaStreamSynchronize(st);
  return r;
}

// The device-side beam parameters of a search over `batch` images (K = 2 * num_beams candidates per row).
static svbeam::Params beam_params_dev(const sv_beam_params* bp, int batch, int vocab, int seq_stride) {
  svbeam::Params hp;
  memset(&hp, 0, sizeof(hp));
  hp.B = batch; hp.nb = bp->num_beams; hp.K = 2 * bp->num_beams; hp.vocab = vocab; hp.max_length = bp->max_new_tokens;
  hp.eos_id = bp->eos_token_id;
  hp.pad_id = bp->pad_token_id;
  hp.n_stop = bp->n_stop_ids;
  for (int i = 0; i < bp->n_stop_ids; ++i) hp.stop_ids[i] = bp->stop_ids[i];
  hp.do_sample = bp->do_sample; hp.early_stopping = bp->early_stopping;
  hp.min_keep = std::max(2, 1 + (bp->eos_token_id >= 0 ? 1 : 0));
  hp.seq_stride = seq_stride;
  hp.temperature = bp->temperature; hp.top_p = bp->top_p; hp.rep_penalty = bp->repetition_penalty;
  hp.length_penalty = bp->length_penalty; hp.seed = bp->seed;
  return hp;
}

// The device state of sv_beam_search and beam sessions, allocated once per engine.
static int beam_alloc(sv_engine* e) {
  if (e->beam_state) return SV_OK;
  const sv_model_desc& d = e->d;
  const int stride = d.max_len;
  bool ok = true;
  const int MR = svbeam::kMaxRows, MK = svbeam::kMaxK, MG = svbeam::kMaxRows / 2;
#define BAL(ptr, n) ok = ok && (dev_alloc(e, &e->ptr, (n)) == cudaSuccess)
  BAL(beam_params, MG); BAL(beam_state, MG); BAL(beam_plan, MG);
  BAL(beam_key, MR * MK); BAL(beam_val, MR * MK); BAL(beam_tok, MR * MK);
  BAL(beam_run_seq, (int64_t)2 * MR * stride); BAL(beam_fin_seq, (int64_t)2 * MR * stride);
  BAL(kstage, e->cache_layer_stride * d.n_layer); BAL(vstage, e->cache_layer_stride * d.n_layer);
#undef BAL
  if (!ok) { e->beam_state = nullptr; return fail(e, SV_ERR_CUDA, "allocation of the beam-search state failed: %s", cudaGetErrorString(cudaGetLastError())); }
  return SV_OK;
}

// Beam search with the whole loop on the device.  Graph body = one decode step over the batch * num_beams cache rows, then
// candidates -> bookkeeping (+ next-token embeddings) -> KV suffix copies; the host replays it and polls `done`.
int sv_beam_search(sv_engine* e, const sv_beam_params* bp, int32_t batch, int32_t* out_ids, int32_t* out_len, void* stream) {
  if (!e || !bp || !out_ids) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_beam_search");
  if (sv_beam_params_check_rows(bp, batch, e->d.max_batch) != SV_OK)
    return fail(e, SV_ERR_INVALID, "bad beam parameters (need num_beams >= 2, batch * num_beams <= max_batch (%d), max_new_tokens >= 1, "
                                   "n_stop_ids in [0,8], early_stopping in {0,1,2}, temperature > 0, repetition_penalty > 0)", e->d.max_batch);
  if (!e->prefilled) return fail(e, SV_ERR_STATE, "sv_beam_search needs sv_prefill first");
  if (e->host_cur_len != e->prefix_len) return fail(e, SV_ERR_STATE, "sv_beam_search must directly follow sv_prefill");
  const sv_model_desc& d = e->d;
  const int nb = bp->num_beams, R = batch * nb, max_new = bp->max_new_tokens, K = 2 * nb;
  if (R != e->cur_batch) return fail(e, SV_ERR_STATE, "prefilled rows %d != batch %d x num_beams %d", e->cur_batch, batch, nb);
  if (e->prefix_len + max_new > d.max_len)
    return fail(e, SV_ERR_INVALID, "prefix %d + max_new_tokens %d exceeds max_len %d", e->prefix_len, max_new, d.max_len);
  SV_CK(e, cudaSetDevice(e->device));
  if (beam_init(d.vocab) != cudaSuccess) {
    cudaGetLastError();
    return fail(e, SV_ERR_UNSUPPORTED, "a logits row of %d entries does not fit the SM's shared memory: use the host-stepped beam loop", d.vocab);
  }
  LaunchScope scope(e);
  const int stride = d.max_len;
  SV_TRY(beam_alloc(e));
  cudaStream_t st = e->gen_stream;
  SV_TRY(join_caller(e, stream));

  const svbeam::Params hp = beam_params_dev(bp, batch, d.vocab, stride);
  svbeam::State hs;
  memset(&hs, 0, sizeof(hs));
  svbeam::init_state(hp, hs, e->prefix_len);
  SV_CK(e, cudaMemcpyAsync(e->beam_params, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));   // pageable: staged synchronously
  SV_CK(e, cudaMemcpyAsync(e->beam_state, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));
  SV_CK(e, cudaMemsetAsync(e->beam_plan, 0, sizeof(svbeam::Plan), st));
  launch_fill_i32(e->beam_run_seq, bp->pad_token_id, 2 * R * stride, st);
  launch_fill_i32(e->beam_fin_seq, bp->pad_token_id, 2 * R * stride, st);

  const bool fused = e->fused_decode;
  auto bookkeeping = [&](int advance) {
    launch_beam_candidates(e->logits, d.vocab, R, e->beam_params, e->beam_state, e->beam_run_seq, e->beam_key, e->beam_val,
                           e->beam_tok, st);
    launch_beam_step(e->beam_params, e->beam_state, e->beam_plan, e->beam_key, e->beam_val, e->beam_tok, e->beam_run_seq,
                     e->beam_fin_seq, e->state, advance, e->wte, e->wpe, e->d_x, d.hidden, d.n_positions, e->next_ids, st);
    launch_beam_kv_copy(e->kcache, e->vtcache, e->kstage, e->vstage, e->cache_layer_stride, d.n_layer, R, d.n_kv_head,
                        e->tcap, d.head_dim, e->beam_plan, st);
  };
  bookkeeping(/*advance=*/0);                       // step 0: candidates from the prefill logits

  const int parts = decode_parts(fused, e->prefix_len + max_new);
  // beam sampling is read from the device parameters: the same graph serves both
  GraphEntry& ge = e->step_graphs[{StepKind::beam, R, parts, false, fused, e->use_pdl}];
  auto step = [&](bool pdl) {
    run_engine_step(e, fused ? nullptr : e->next_ids, R, parts, pdl, st);
    bookkeeping(/*advance=*/1);
  };
  if (!ge.exec && max_new > 1) {
    SV_CK(e, capture_step(st, e->use_pdl && fused, step, ge));
    if (fused && !ge.pdl) e->use_pdl = false;
  }
  const int poll = bp->poll_interval > 0 ? bp->poll_interval : 16;
  SV_CK(e, cudaEventRecord(e->ev_t0, st));
  int steps = 0;
  bool done = false;
  for (int s = 1; s < max_new && !done; ++s) {
    SV_TRY(replay(e, ge, 1));
    ++steps;
    if (s % poll == 0) {
      SV_TRY(read_flags(e, &e->beam_state->done, 1));
      done = e->host_flag[0] != 0;
    }
  }
  SV_CK(e, cudaEventRecord(e->ev_t1, st));
  SV_CK(e, cudaMemcpyAsync(&hs, e->beam_state, sizeof(hs), cudaMemcpyDeviceToHost, st));
  SV_CK(e, cudaStreamSynchronize(st));
  SV_CK(e, cudaGetLastError());
  if (!hs.done) return fail(e, SV_ERR_STATE, "beam search did not terminate within max_new_tokens steps (internal error)");
  int n_gen = 0;
  for (int b = 0; b < batch; ++b) n_gen = std::max(n_gen, hs.fin_len[b * nb]);     // HF: max_generated over the best beams
  n_gen = std::min(n_gen, max_new);
  launch_fill_i32(out_ids, bp->pad_token_id, batch * max_new, st);
  // best hypothesis of image b = finished slot 0 = row b * nb of the live half of fin_seq
  SV_CK(e, cudaMemcpy2DAsync(out_ids, (size_t)max_new * 4, e->beam_fin_seq + ((int64_t)hs.parity * R) * stride, (size_t)nb * stride * 4,
                             (size_t)std::max(n_gen, 1) * 4, batch, cudaMemcpyDeviceToDevice, st));
  if (out_len) launch_fill_i32(out_len, n_gen, batch, st);
  SV_CK(e, cudaStreamSynchronize(st));
  SV_CK(e, cudaGetLastError());
  SV_CK(e, cudaEventElapsedTime(&e->last_decode_ms, e->ev_t0, e->ev_t1));
  e->last_decode_steps = steps;
  e->host_cur_len = e->prefix_len + hs.cur_len;
  e->prefilled = false;
  return SV_OK;
}

int sv_reorder_cache(sv_engine* e, const int32_t* src_rows, void* stream) {
  if (!e || !src_rows) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_reorder_cache");
  if (!e->prefilled) return fail(e, SV_ERR_STATE, "sv_reorder_cache needs a prefilled cache");
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = (cudaStream_t)stream;
  const sv_model_desc& d = e->d;
  const int B = e->cur_batch, len = e->host_cur_len;
  for (int i = 0; i < d.n_layer; ++i) {
    bf16* kc = e->kcache + e->cache_layer_stride * i;
    bf16* vc = e->vtcache + e->cache_layer_stride * i;
    launch_kv_gather(kc, vc, e->kscratch, e->vscratch, src_rows, B, d.n_kv_head, e->tcap, d.head_dim, len, st);
    launch_kv_gather(e->kscratch, e->vscratch, kc, vc, nullptr, B, d.n_kv_head, e->tcap, d.head_dim, len, st);
  }
  SV_CK(e, cudaGetLastError());
  return SV_OK;
}

int sv_expand_batch(sv_engine* e, const int32_t* src_rows_host, int32_t new_batch, void* stream) {
  if (!e || !src_rows_host) return fail(e, SV_ERR_INVALID, "null argument");
  SV_NO_SESSION(e, "sv_expand_batch");
  if (!e->prefilled || e->host_cur_len != e->prefix_len) return fail(e, SV_ERR_STATE, "sv_expand_batch must directly follow sv_prefill");
  if (new_batch < 1 || new_batch > e->d.max_batch) return fail(e, SV_ERR_INVALID, "new_batch %d outside [1,%d]", new_batch, e->d.max_batch);
  for (int r = 0; r < new_batch; ++r)
    if (src_rows_host[r] < 0 || src_rows_host[r] >= e->cur_batch) return fail(e, SV_ERR_INVALID, "src_rows[%d] = %d is not a prefilled row", r, src_rows_host[r]);
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = (cudaStream_t)stream;
  const sv_model_desc& d = e->d;
  const int len = e->host_cur_len;
  SV_CK(e, cudaMemcpyAsync(e->ids_tmp, src_rows_host, (size_t)new_batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  for (int i = 0; i < d.n_layer; ++i) {          // cache rows: gather through the one-layer scratch (as sv_reorder_cache)
    bf16* kc = e->kcache + e->cache_layer_stride * i;
    bf16* vc = e->vtcache + e->cache_layer_stride * i;
    launch_kv_gather(kc, vc, e->kscratch, e->vscratch, e->ids_tmp, new_batch, d.n_kv_head, e->tcap, d.head_dim, len, st);
    launch_kv_gather(e->kscratch, e->vscratch, kc, vc, nullptr, new_batch, d.n_kv_head, e->tcap, d.head_dim, len, st);
  }
  // the prefill's last-position logits (token 0 is selected from them) and the last hidden row, staged through logits_f32
  const size_t row = (size_t)d.vocab * sizeof(bf16);
  uint8_t* stage = reinterpret_cast<uint8_t*>(e->logits_f32);
  for (int r = 0; r < new_batch; ++r)
    SV_CK(e, cudaMemcpyAsync(stage + r * row, reinterpret_cast<uint8_t*>(e->logits) + src_rows_host[r] * row, row, cudaMemcpyDeviceToDevice, st));
  SV_CK(e, cudaMemcpyAsync(e->logits, stage, new_batch * row, cudaMemcpyDeviceToDevice, st));
  e->cur_batch = new_batch;
  return finish_prefill_impl(e, new_batch, e->prefix_len, nullptr, st);     // fresh GenState for the new rows, exchange buffers cleared
}

// ---- continuous batching --------------------------------------------------------------------------------------------
// The per-row state of a session, allocated by the first one.
static int session_alloc(sv_engine* e) {
  if (e->rows) return SV_OK;
  const sv_model_desc& d = e->d;
  bool ok = dev_alloc(e, &e->rows, 1) == cudaSuccess && dev_alloc(e, &e->sess_logits, (int64_t)d.max_batch * d.vocab) == cudaSuccess;
  if (ok && !e->rows_host) ok = cudaMallocHost(reinterpret_cast<void**>(&e->rows_host), sizeof(RowState)) == cudaSuccess;
  if (!ok) { e->rows = nullptr; return fail(e, SV_ERR_CUDA, "allocation of the session state failed: %s", cudaGetErrorString(cudaGetLastError())); }
  return SV_OK;
}

int sv_session_begin(sv_engine* e, const sv_gen_params* p, int32_t slots) {
  if (!e || !p) return fail(e, SV_ERR_INVALID, "null argument");
  if (e->session) return fail(e, SV_ERR_STATE, "a decode session is already open");
  if (slots < 1 || slots > e->d.max_batch) return fail(e, SV_ERR_INVALID, "slots %d outside [1,%d]", slots, e->d.max_batch);
  if (p->max_new_tokens < 1 || p->max_new_tokens > e->d.max_len)
    return fail(e, SV_ERR_INVALID, "max_new_tokens %d outside [1,%d]", p->max_new_tokens, e->d.max_len);
  if (const char* bad = gen_params_error(*p)) return fail(e, SV_ERR_INVALID, "%s", bad);
  int r = check_ready(e);
  if (r != SV_OK) return r;
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  const sv_model_desc& d = e->d;
  SV_TRY(session_alloc(e));
  cudaStream_t st = e->gen_stream;
  const GenParamsDev hp = gen_params_dev(p, /*stop_row0_only=*/0, d.max_len);
  SV_CK(e, cudaMemcpyAsync(e->params, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));   // pageable: staged synchronously
  SV_CK(e, cudaMemsetAsync(e->rows, 0, sizeof(RowState), st));
  ensure_flow_tiles(e, st);      // SV_TILED=1: the ring GEMVs stream the slab-tiled weights, rebuilt after a weight load
  SV_CK(e, cudaStreamSynchronize(st));
  e->sess_p = *p;
  e->sess_slots = slots;
  e->sess_prompt_len = 0;
  e->sess_live.assign(slots, 0);
  e->sess_len.assign(slots, 0);
  e->session = true;
  e->encoded = false;        // admission overwrites the resident visual prefix and the cache rows
  e->prefilled = false;
  return SV_OK;
}

int sv_session_admit(sv_engine* e, const void* pixels, int32_t k, const int32_t* prompt_ids, int32_t prompt_len,
                     const int32_t* slots_host, const int32_t* max_new_host, const uint64_t* seeds_host,
                     const int32_t* src_host, void* stream) {
  if (!e || !pixels || !prompt_ids || !slots_host) return fail(e, SV_ERR_INVALID, "null argument");
  if (!e->session) return fail(e, SV_ERR_STATE, "sv_session_admit needs sv_session_begin first");
  if (e->sess_beam) return fail(e, SV_ERR_STATE, "sv_session_admit: a beam session is open (admit with sv_beam_session_admit)");
  const sv_model_desc& d = e->d;
  const int S = e->sess_slots, cap = e->sess_p.max_new_tokens;
  if (k < 1 || k > S) return fail(e, SV_ERR_INVALID, "k %d outside [1,%d]", k, S);
  if (prompt_len < 1 || prompt_len > kMaxPrompt) return fail(e, SV_ERR_INVALID, "prompt_len %d outside [1,%d]", prompt_len, kMaxPrompt);
  if (e->sess_prompt_len != 0 && prompt_len != e->sess_prompt_len)
    return fail(e, SV_ERR_INVALID, "prompt_len %d differs from the session's %d (the split count of the decode graph is fixed by "
                                   "prefix + max_new_tokens)", prompt_len, e->sess_prompt_len);
  const int prefix = e->Q + prompt_len;
  if (prefix + cap > d.max_len)
    return fail(e, SV_ERR_INVALID, "prefix %d + max_new_tokens %d exceeds max_len %d", prefix, cap, d.max_len);
  std::vector<int> used(S, 0);
  int n_img = 0;
  for (int j = 0; j < k; ++j) {
    const int s = slots_host[j];
    if (s < 0 || s >= S) return fail(e, SV_ERR_INVALID, "slot %d outside [0,%d)", s, S);
    if (used[s] || e->sess_live[s]) return fail(e, SV_ERR_INVALID, "slot %d is busy or listed twice", s);
    used[s] = 1;
    if (max_new_host && (max_new_host[j] < 1 || max_new_host[j] > cap))
      return fail(e, SV_ERR_INVALID, "max_new[%d] = %d outside [1,%d] (the session cap)", j, max_new_host[j], cap);
    const int src = src_host ? src_host[j] : j;
    if (src < 0 || src >= k) return fail(e, SV_ERR_INVALID, "src[%d] = %d outside [0,%d)", j, src, k);
    n_img = std::max(n_img, src + 1);
  }
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = e->gen_stream;
  SV_TRY(join_caller(e, stream));
  const int64_t img = (int64_t)3 * d.image_size * d.image_size, row_stride = (int64_t)d.n_kv_head * e->tcap * d.head_dim;
  const size_t lrow = (size_t)d.vocab * sizeof(bf16);
  uint32_t mask = 0;
  // On an error below, the slots touched so far hold a partial admission; they are not marked live, so the caller may
  // admit into them again (or end the session).
  // Every image is encoded and prefilled on its own (B = 1): the same kernels, tilings and bits as a one-image generate.
  // Batching the admitted images would change M-dependent tile choices of the prefill GEMMs and of the last-logits GEMV.
  for (int i = 0; i < n_img; ++i) {
    int first = -1;
    for (int j = 0; j < k; ++j)
      if ((src_host ? src_host[j] : j) == i) { first = slots_host[j]; break; }
    if (first < 0) continue;
    int r = run_encode(e, (const bf16*)pixels + i * img, 1, st);
    if (r == SV_OK) r = run_prefill(e, e->visual, e->Q, prompt_ids + (int64_t)i * prompt_len, 1, prompt_len, st, first,
                                    e->sess_logits + (int64_t)first * d.vocab);
    if (r != SV_OK) return r;
    for (int j = 0; j < k; ++j) {      // n completions of one image: its prefilled rows copied into the other slots
      const int s = slots_host[j];
      if ((src_host ? src_host[j] : j) != i || s == first) continue;
      for (int l = 0; l < d.n_layer; ++l) {
        bf16* kc = e->kcache + e->cache_layer_stride * l;
        bf16* vc = e->vtcache + e->cache_layer_stride * l;
        launch_kv_gather(kc + first * row_stride, vc + first * row_stride, kc + s * row_stride, vc + s * row_stride, nullptr, 1,
                         d.n_kv_head, e->tcap, d.head_dim, prefix, st);
      }
      SV_CK(e, cudaMemcpyAsync(reinterpret_cast<uint8_t*>(e->sess_logits) + s * lrow,
                               reinterpret_cast<uint8_t*>(e->sess_logits) + first * lrow, lrow, cudaMemcpyDeviceToDevice, st));
    }
  }
  // the slots' own rows of the carried state (repetition-penalty set, output row, per-row fields), in one launch
  SessionAdmit adm;
  memset(&adm, 0, sizeof(adm));
  adm.n = k;
  for (int j = 0; j < k; ++j) {
    const int s = slots_host[j];
    adm.slot[j] = s;
    adm.len[j] = prefix;
    adm.max_new[j] = max_new_host ? max_new_host[j] : cap;
    adm.seed[j] = seeds_host ? seeds_host[j] : e->sess_p.seed;
    mask |= 1u << s;
  }
  launch_session_admit(e->rows, adm, e->seen, d.vocab, e->out_ids, d.max_len, e->sess_p.pad_token_id, st);
  // token 0 of the admitted slots from their prefill logits (generate_impl's first select, no position advance)
  launch_token_select(e, e->sess_logits, S, e->sess_p.do_sample, /*partials=*/false, /*advance_len=*/0, /*pdl=*/false, st,
                      e->rows, mask);
  // speculative session: nothing to accept; the next drafts, allocation and map over every live row, and every column's
  // embedding (the select above embedded the admitted rows at their slot index, which is not the column layout)
  if (e->sess_spec)
    launch_spec_session_tail(false, e->rows, e->params, e->seen, e->next_ids, e->out_ids, d.vocab, e->wte, e->wpe, e->d_x,
                             d.hidden, d.n_positions, e->tcap, e->spec_sess, false, st);
  SV_CK(e, cudaGetLastError());
  SV_CK(e, cudaStreamSynchronize(st));     // the caller may release pixels / prompt_ids on return
  for (int j = 0; j < k; ++j) e->sess_live[slots_host[j]] = 1;
  e->sess_prompt_len = prompt_len;
  return SV_OK;
}

int sv_session_run(sv_engine* e, int32_t max_steps, int32_t* finished_host, int32_t* len_host, void* stream) {
  if (!e) return fail(e, SV_ERR_INVALID, "null argument");
  if (!e->session) return fail(e, SV_ERR_STATE, "sv_session_run needs sv_session_begin first");
  if (max_steps < 0) return fail(e, SV_ERR_INVALID, "max_steps must be >= 0");
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  const int S = e->sess_slots;
  cudaStream_t st = e->gen_stream;
  SV_TRY(join_caller(e, stream));
  // the select kernels raise RowState::event when a row finishes (at admission too: a first token may end a row), so a
  // poll reads that one word; the per-row fields are read once, at the end, and the event is cleared with them
  bool any_live = false;
  for (int s = 0; s < S; ++s) any_live = any_live || e->sess_live[s];
  SV_TRY(read_flags(e, &e->rows->event, 1));
  bool any_fin = e->host_flag[0] != 0;
  int steps = 0;
  if (!any_fin && any_live && max_steps > 0) {
    ensure_flow_tiles(e, st);    // (no-op unless a weight was loaded since the tiles were built)
    const bool beam = e->sess_beam;
    const bool fused = e->fused_decode, sample = !beam && e->sess_p.do_sample != 0;
    const int cap = beam ? e->sess_bp.max_new_tokens : e->sess_p.max_new_tokens;
    const int total = e->Q + e->sess_prompt_len + cap;     // the session cap fixes the split count
    const int parts = decode_parts(fused, total);
    // (beam sessions: beam-sample and the beam width are read from the device parameters, as in sv_beam_search)
    const bool spec = e->sess_spec;
    const StepKind kind = beam ? StepKind::beam_session : spec ? StepKind::spec_session : StepKind::session;
    GraphEntry& ge = e->step_graphs[{kind, S, parts, sample, fused, e->use_pdl}];
    const sv_model_desc& d = e->d;
    auto step = [&](bool pdl) {
      if (spec) {              // verify step over the S columns of the map; the previous tail embedded their inputs
        run_engine_step(e, nullptr, S, parts, pdl, st, nullptr, &e->spec_sess->map);
        if (sample) {
          launch_spec_session_select_sample(e->logits, d.vocab, S, e->rows, e->params, e->seen, e->logits_f32, e->spec_sess, st);
          launch_spec_session_tail(true, e->rows, e->params, e->seen, e->next_ids, e->out_ids, d.vocab, e->wte, e->wpe, e->d_x,
                                   d.hidden, d.n_positions, e->tcap, e->spec_sess, false, st);
        } else {
          launch_spec_session_select_fused(e->logits, d.vocab, e->amax_val, e->amax_idx, gemv_ring_ntiles(d.vocab),
                                           8 * ring_row_groups(S), e->rows, e->params, e->seen, e->next_ids, e->out_ids,
                                           e->wte, e->wpe, e->d_x, d.hidden, d.n_positions, e->tcap, e->spec_sess, pdl, st);
        }
        return;
      }
      if (beam) {              // the decode step, then every live group's bookkeeping, as sv_beam_search runs it
        run_engine_step(e, fused ? nullptr : e->next_ids, S, parts, pdl, st, e->rows);
        launch_beam_session_candidates(e->logits, d.vocab, S, e->beam_params, e->beam_state, e->beam_run_seq, e->beam_key,
                                       e->beam_val, e->beam_tok, e->rows, ~0u, st);
        launch_beam_session_step(e->beam_params, e->beam_state, e->beam_plan, e->beam_key, e->beam_val, e->beam_tok,
                                 e->beam_run_seq, e->beam_fin_seq, e->rows, ~0u, S, /*advance=*/1, e->wte, e->wpe, e->d_x,
                                 d.hidden, d.n_positions, e->next_ids, st);
        launch_beam_session_kv_copy(e->kcache, e->vtcache, e->kstage, e->vstage, e->cache_layer_stride, d.n_layer, S,
                                    d.n_kv_head, e->tcap, d.head_dim, e->beam_params, e->beam_plan, e->rows, ~0u, st);
        return;
      }
      run_engine_step(e, fused && !sample ? nullptr : e->next_ids, S, parts, pdl, st, e->rows);
      launch_token_select(e, e->logits, S, sample, /*partials=*/true, /*advance_len=*/1, pdl, st, e->rows, (1u << S) - 1u);
    };
    if (!ge.exec) {
      SV_CK(e, capture_step(st, e->use_pdl && fused, step, ge));
      if (fused && !ge.pdl) e->use_pdl = false;
    }
    const int poll = beam ? e->sess_bp.poll_interval : e->sess_p.poll_interval;
    const int every = poll > 0 ? poll : 16;
    while (steps < max_steps && !any_fin && any_live) {
      const int n = std::min(every, max_steps - steps);
      SV_TRY(replay(e, ge, n));
      steps += n;
      SV_TRY(read_flags(e, &e->rows->event, 1));
      any_fin = e->host_flag[0] != 0;
    }
  }
  {
    const size_t off = offsetof(RowState, row_step), n = offsetof(RowState, event) - off;   // row_step, row_active
    SV_CK(e, cudaMemcpyAsync(reinterpret_cast<uint8_t*>(e->rows_host) + off, reinterpret_cast<uint8_t*>(e->rows) + off, n,
                             cudaMemcpyDeviceToHost, st));
    SV_CK(e, cudaMemsetAsync(&e->rows->event, 0, sizeof(int32_t), st));
    SV_CK(e, cudaStreamSynchronize(st));
  }
  SV_CK(e, cudaGetLastError());
  for (int s = 0; s < S; ++s) {
    const bool fin = e->sess_live[s] && !e->rows_host->row_active[s];
    e->sess_len[s] = e->rows_host->row_step[s];
    if (fin) e->sess_live[s] = 0;
    if (finished_host) finished_host[s] = fin ? 1 : 0;
    if (len_host) len_host[s] = e->sess_len[s];
  }
  return steps;
}

int sv_session_read(sv_engine* e, int32_t slot, int32_t* ids, void* stream) {
  if (!e || !ids) return fail(e, SV_ERR_INVALID, "null argument");
  if (!e->session) return fail(e, SV_ERR_STATE, "sv_session_read needs an open session");
  if (slot < 0 || slot >= e->sess_slots) return fail(e, SV_ERR_INVALID, "slot %d outside [0,%d)", slot, e->sess_slots);
  SV_CK(e, cudaSetDevice(e->device));
  cudaStream_t st = e->gen_stream;
  SV_TRY(join_caller(e, stream));
  const int n = e->sess_len[slot];
  const int32_t* src = e->out_ids + (int64_t)slot * e->d.max_len;
  if (e->sess_beam) {          // the best hypothesis = finished slot 0 of the group's live half of fin_seq
    const int nb = e->sess_bp.num_beams;
    if (slot % nb) return fail(e, SV_ERR_INVALID, "slot %d is not the first slot of a group of %d", slot, nb);
    SV_TRY(read_flags(e, &e->beam_state[slot / nb].parity, 1));
    src = e->beam_fin_seq + ((int64_t)e->host_flag[0] * svbeam::kMaxRows + slot) * e->d.max_len;
  }
  if (n > 0) SV_CK(e, cudaMemcpyAsync(ids, src, (size_t)n * 4, cudaMemcpyDefault, st));
  SV_CK(e, cudaStreamSynchronize(st));
  return n;
}

int sv_session_end(sv_engine* e) {
  if (!e) return SV_ERR_INVALID;
  if (!e->session) return fail(e, SV_ERR_STATE, "no decode session is open");
  SV_CK(e, cudaSetDevice(e->device));
  SV_CK(e, cudaStreamSynchronize(e->gen_stream));
  e->session = false;
  e->sess_beam = false;
  e->sess_spec = false;
  e->sess_slots = 0;
  e->sess_live.clear();
  e->sess_len.clear();
  return SV_OK;
}

// ---- speculative sessions (DESIGN.md §7i) ---------------------------------------------------------------------------
int sv_session_begin_speculative(sv_engine* e, const sv_gen_params* p, const sv_spec_params* sp, int32_t slots) {
  if (!e || !p || !sp) return fail(e, SV_ERR_INVALID, "null argument");
  if (e->session) return fail(e, SV_ERR_STATE, "a decode session is already open");
  if (e->v2) return fail(e, SV_ERR_UNSUPPORTED, "sv_session_begin_speculative: v2 engines decode through the per-op kernels; only v1 is built");
  if (!e->fused_decode) return fail(e, SV_ERR_UNSUPPORTED, "sv_session_begin_speculative needs the fused graph decode path (SV_DECODE=legacy is set)");
  if (slots < 2 || slots > std::min(e->d.max_batch, svspec::kMaxCols))
    return fail(e, SV_ERR_INVALID, "slots %d outside [2,%d] (a speculative session drafts into the columns of idle slots)", slots,
                std::min(e->d.max_batch, svspec::kMaxCols));
  if (sp->num_tokens < 1 || sp->num_tokens > slots - 1)
    return fail(e, SV_ERR_INVALID, "prompt_lookup_num_tokens %d outside [1, %d] (slots - 1)", sp->num_tokens, slots - 1);
  if (sp->max_matching_ngram_size < 1)
    return fail(e, SV_ERR_INVALID, "max_matching_ngram_size must be >= 1, got %d", sp->max_matching_ngram_size);
  SV_CK(e, cudaSetDevice(e->device));
  if (!e->spec_sess && dev_alloc(e, &e->spec_sess, 1) != cudaSuccess)
    return fail(e, SV_ERR_CUDA, "allocation of the speculative session state failed: %s", cudaGetErrorString(cudaGetLastError()));
  SV_TRY(sv_session_begin(e, p, slots));
  svspec::SessionState hs;
  memset(&hs, 0, sizeof(hs));          // n_live = 0: no column is live before the first admission
  hs.ncols = slots; hs.k = sp->num_tokens; hs.max_ngram = sp->max_matching_ngram_size;
  const cudaError_t r = cudaMemcpy(e->spec_sess, &hs, sizeof(hs), cudaMemcpyHostToDevice);
  if (r != cudaSuccess) {
    sv_session_end(e);
    return fail(e, SV_ERR_CUDA, "upload of the speculative session state failed: %s", cudaGetErrorString(r));
  }
  e->sess_spec = true;
  return SV_OK;
}

int sv_session_spec_stats(sv_engine* e, int32_t* steps, int32_t* drafted, int32_t* accepted) {
  if (!e) return SV_ERR_INVALID;
  if (!e->session || !e->sess_spec) return fail(e, SV_ERR_STATE, "sv_session_spec_stats needs an open speculative session");
  SV_CK(e, cudaSetDevice(e->device));
  SV_CK(e, cudaStreamSynchronize(e->gen_stream));
  int32_t v[3];
  SV_CK(e, cudaMemcpy(v, &e->spec_sess->steps, sizeof(v), cudaMemcpyDeviceToHost));
  if (steps) *steps = v[0];
  if (drafted) *drafted = v[1];
  if (accepted) *accepted = v[2];
  return SV_OK;
}

int sv_spec_session_plan_host(int32_t S, const int32_t* active, const int32_t* want, int32_t budget, int32_t* g,
                              int32_t* first) {
  if (S < 1 || S > svspec::kMaxCols || !active || !want || !g || !first) return SV_ERR_INVALID;
  return svspec::plan_session(S, active, want, budget, g, first);
}

// sv_spec_session_state mirrors svspec::SessionState and sv_session_rows RowState, field for field.
static_assert(sizeof(sv_spec_session_state) == sizeof(svspec::SessionState) &&
              offsetof(sv_spec_session_state, off) == offsetof(svspec::SessionState, off) &&
              offsetof(sv_spec_session_state, accepted) == offsetof(svspec::SessionState, accepted),
              "sv_spec_session_state mirrors svspec::SessionState");
static_assert(sizeof(sv_session_rows) == sizeof(RowState) && offsetof(sv_session_rows, event) == offsetof(RowState, event) &&
              offsetof(sv_session_rows, row_seed) == offsetof(RowState, row_seed), "sv_session_rows mirrors RowState");

int sv_spec_session_tail_host(const sv_gen_params* p, sv_session_rows* rows, int32_t* out_ids, int32_t out_stride,
                              sv_spec_session_state* ss, int32_t accept, int32_t tcap) {
  if (!p || !rows || !out_ids || !ss) return SV_ERR_INVALID;
  const int S = ss->ncols;
  if (S < 1 || S > svspec::kMaxCols || ss->n_live < 0 || ss->n_live > S || ss->k < 0 || ss->max_ngram < 1) return SV_ERR_INVALID;
  if (p->n_stop_ids < 0 || p->n_stop_ids > 8 || out_stride < 1) return SV_ERR_INVALID;
  for (int r = 0; r < S; ++r)
    if (rows->row_active[r] && (rows->row_step[r] < 1 || rows->row_step[r] >= rows->row_max_new[r] || rows->row_max_new[r] > out_stride))
      return SV_ERR_INVALID;
  svspec::SessionState* s = reinterpret_cast<svspec::SessionState*>(ss);
  RowState* rs = reinterpret_cast<RowState*>(rows);
  const GenParamsDev hp = gen_params_dev(p, 0, out_stride);
  int32_t next[svspec::kMaxCols];
  if (accept) spec_session_accept(s, s->sel, rs, &hp, nullptr, /*vocab=*/0, next, out_ids);
  int32_t w[svspec::kMaxCols] = {0}, dr[svspec::kMaxCols][svspec::kMaxCols];
  int live = 0;
  for (int r = 0; r < S; ++r) live += rs->row_active[r] != 0;
  if (spec_session_budget(rs, S, tcap) > live)
    for (int r = 0; r < S; ++r)
      if (rs->row_active[r])
        w[r] = svspec::draft_host(out_ids + (int64_t)r * out_stride, rs->row_step[r], s->k, s->max_ngram, hp.eos_id,
                                  rs->row_max_new[r] - rs->row_step[r] - 1, dr[r]);
  return spec_session_plan(s, rs, out_ids, out_stride, w, dr, tcap);
}

// ---- beam sessions (DESIGN.md §7h) ----------------------------------------------------------------------------------
int sv_beam_session_begin(sv_engine* e, const sv_beam_params* bp, int32_t slots) {
  if (!e || !bp) return fail(e, SV_ERR_INVALID, "null argument");
  if (e->session) return fail(e, SV_ERR_STATE, "a decode session is already open");
  const sv_model_desc& d = e->d;
  const int nb = bp->num_beams;
  if (nb < 2 || slots < nb || slots > d.max_batch || slots % nb)
    return fail(e, SV_ERR_INVALID, "slots %d must be a multiple of num_beams %d (>= 2) in [num_beams, %d]", slots, nb, d.max_batch);
  if (sv_beam_params_check_rows(bp, slots / nb, d.max_batch) != SV_OK)
    return fail(e, SV_ERR_INVALID, "bad beam parameters (need max_new_tokens >= 1, n_stop_ids in [0,8], early_stopping in {0,1,2}, "
                                   "temperature > 0, repetition_penalty > 0, 2 * num_beams <= 16)");
  if (bp->max_new_tokens > d.max_len) return fail(e, SV_ERR_INVALID, "max_new_tokens %d exceeds max_len %d", bp->max_new_tokens, d.max_len);
  int r = check_ready(e);
  if (r != SV_OK) return r;
  SV_CK(e, cudaSetDevice(e->device));
  if (beam_init(d.vocab) != cudaSuccess || beam_session_init(d.vocab) != cudaSuccess) {
    cudaGetLastError();
    return fail(e, SV_ERR_UNSUPPORTED, "a logits row of %d entries does not fit the SM's shared memory: beam sessions need the "
                                       "device candidate kernel", d.vocab);
  }
  LaunchScope scope(e);
  SV_TRY(session_alloc(e));
  SV_TRY(beam_alloc(e));
  if (!e->bsess_px) {
    const int64_t img = (int64_t)3 * d.image_size * d.image_size;
    if (dev_alloc(e, &e->bsess_px, d.max_batch * img) != cudaSuccess || dev_alloc(e, &e->bsess_ids, d.max_batch * kMaxPrompt) != cudaSuccess) {
      e->bsess_px = nullptr;
      return fail(e, SV_ERR_CUDA, "allocation of the beam-session staging failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
  }
  cudaStream_t st = e->gen_stream;
  SV_CK(e, cudaMemsetAsync(e->rows, 0, sizeof(RowState), st));          // no slot live
  const svbeam::Params hp = beam_params_dev(bp, 1, d.vocab, d.max_len);
  for (int g = 0; g < slots / nb; ++g)     // every group's entry holds the beam width the kernels read (admission fills the rest)
    SV_CK(e, cudaMemcpyAsync(e->beam_params + g, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));   // pageable: staged synchronously
  SV_CK(e, cudaMemsetAsync(e->beam_plan, 0, sizeof(svbeam::Plan) * (svbeam::kMaxRows / 2), st));
  ensure_flow_tiles(e, st);
  SV_CK(e, cudaStreamSynchronize(st));
  e->sess_bp = *bp;
  e->sess_beam = true;
  e->sess_slots = slots;
  e->sess_prompt_len = 0;
  e->sess_live.assign(slots, 0);
  e->sess_len.assign(slots, 0);
  e->session = true;
  e->encoded = false;
  e->prefilled = false;
  return SV_OK;
}

int sv_beam_session_admit(sv_engine* e, const void* pixels, int32_t k, const int32_t* prompt_ids, int32_t prompt_len,
                          const int32_t* groups_host, const int32_t* max_new_host, const uint64_t* seeds_host, void* stream) {
  if (!e || !pixels || !prompt_ids || !groups_host) return fail(e, SV_ERR_INVALID, "null argument");
  if (!e->session || !e->sess_beam) return fail(e, SV_ERR_STATE, "sv_beam_session_admit needs sv_beam_session_begin first");
  const sv_model_desc& d = e->d;
  const int nb = e->sess_bp.num_beams, S = e->sess_slots, G = S / nb, cap = e->sess_bp.max_new_tokens;
  if (k < 1 || k > G) return fail(e, SV_ERR_INVALID, "k %d outside [1,%d]", k, G);
  if (prompt_len < 1 || prompt_len > kMaxPrompt) return fail(e, SV_ERR_INVALID, "prompt_len %d outside [1,%d]", prompt_len, kMaxPrompt);
  if (e->sess_prompt_len != 0 && prompt_len != e->sess_prompt_len)
    return fail(e, SV_ERR_INVALID, "prompt_len %d differs from the session's %d (the split count of the decode graph is fixed by "
                                   "prefix + max_new_tokens)", prompt_len, e->sess_prompt_len);
  const int prefix = e->Q + prompt_len;
  if (prefix + cap > d.max_len)
    return fail(e, SV_ERR_INVALID, "prefix %d + max_new_tokens %d exceeds max_len %d", prefix, cap, d.max_len);
  std::vector<int> used(G, 0);
  for (int j = 0; j < k; ++j) {
    const int g = groups_host[j];
    if (g < 0 || g >= G) return fail(e, SV_ERR_INVALID, "group %d outside [0,%d)", g, G);
    if (used[g] || e->sess_live[g * nb]) return fail(e, SV_ERR_INVALID, "group %d is busy or listed twice", g);
    used[g] = 1;
    if (max_new_host && (max_new_host[j] < 1 || max_new_host[j] > cap))
      return fail(e, SV_ERR_INVALID, "max_new[%d] = %d outside [1,%d] (the session cap)", j, max_new_host[j], cap);
  }
  SV_CK(e, cudaSetDevice(e->device));
  LaunchScope scope(e);
  cudaStream_t st = e->gen_stream;
  SV_TRY(join_caller(e, stream));
  const int64_t img = (int64_t)3 * d.image_size * d.image_size;
  const int stride = d.max_len, fill = e->sess_bp.pad_token_id;
  SessionAdmit adm;
  memset(&adm, 0, sizeof(adm));
  uint32_t mask = 0;
  // Each image runs what a one-image beam search runs: the image and prompt repeated num_beams times are encoded and
  // prefilled at batch num_beams (GEMM tiles depend on M), into the group's rows.  On an error below, the groups touched so
  // far are not marked live, so the caller may admit into them again (or end the session).
  for (int j = 0; j < k; ++j) {
    const int g = groups_host[j], row0 = g * nb;
    for (int b = 0; b < nb; ++b) {
      SV_CK(e, cudaMemcpyAsync(e->bsess_px + b * img, (const bf16*)pixels + j * img, img * sizeof(bf16), cudaMemcpyDeviceToDevice, st));
      SV_CK(e, cudaMemcpyAsync(e->bsess_ids + b * prompt_len, prompt_ids + (int64_t)j * prompt_len, prompt_len * sizeof(int32_t),
                               cudaMemcpyDeviceToDevice, st));
    }
    int r = run_encode(e, e->bsess_px, nb, st);
    if (r == SV_OK) r = run_prefill(e, e->visual, e->Q, e->bsess_ids, nb, prompt_len, st, row0, e->sess_logits + (int64_t)row0 * d.vocab);
    if (r != SV_OK) return r;
    sv_beam_params bp = e->sess_bp;
    bp.max_new_tokens = max_new_host ? max_new_host[j] : cap;
    if (seeds_host) bp.seed = seeds_host[j];
    const svbeam::Params hp = beam_params_dev(&bp, 1, d.vocab, stride);
    svbeam::State hs;
    memset(&hs, 0, sizeof(hs));
    svbeam::init_state(hp, hs, prefix);
    SV_CK(e, cudaMemcpyAsync(e->beam_params + g, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));   // pageable: staged synchronously
    SV_CK(e, cudaMemcpyAsync(e->beam_state + g, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));
    SV_CK(e, cudaMemsetAsync(e->beam_plan + g, 0, sizeof(svbeam::Plan), st));
    for (int half = 0; half < 2; ++half) {
      const int64_t off = ((int64_t)half * svbeam::kMaxRows + row0) * stride;
      launch_fill_i32(e->beam_run_seq + off, fill, nb * stride, st);
      launch_fill_i32(e->beam_fin_seq + off, fill, nb * stride, st);
    }
    for (int b = 0; b < nb; ++b) {
      adm.slot[adm.n] = row0 + b; adm.len[adm.n] = prefix; adm.max_new[adm.n] = bp.max_new_tokens; adm.seed[adm.n] = bp.seed;
      ++adm.n;
    }
    mask |= 1u << g;
  }
  launch_session_admit(e->rows, adm, e->seen, d.vocab, e->out_ids, d.max_len, fill, st);     // row_len, row_active, ...
  // step 0 of the admitted groups from their prefill logits (sv_beam_search's first bookkeeping, no position advance)
  launch_beam_session_candidates(e->sess_logits, d.vocab, S, e->beam_params, e->beam_state, e->beam_run_seq, e->beam_key,
                                 e->beam_val, e->beam_tok, e->rows, mask, st);
  launch_beam_session_step(e->beam_params, e->beam_state, e->beam_plan, e->beam_key, e->beam_val, e->beam_tok, e->beam_run_seq,
                           e->beam_fin_seq, e->rows, mask, S, /*advance=*/0, e->wte, e->wpe, e->d_x, d.hidden, d.n_positions,
                           e->next_ids, st);
  launch_beam_session_kv_copy(e->kcache, e->vtcache, e->kstage, e->vstage, e->cache_layer_stride, d.n_layer, S, d.n_kv_head,
                              e->tcap, d.head_dim, e->beam_params, e->beam_plan, e->rows, mask, st);
  SV_CK(e, cudaGetLastError());
  SV_CK(e, cudaStreamSynchronize(st));     // the caller may release pixels / prompt_ids on return
  for (int j = 0; j < k; ++j) e->sess_live[groups_host[j] * nb] = 1;
  e->sess_prompt_len = prompt_len;
  return SV_OK;
}

int64_t sv_launch_count(const sv_engine* e) { return e ? e->launches : 0; }

int sv_debug_read_timeline(sv_engine* e, long long* out_host, int32_t n) {
  if (!e || !out_host || n < 1 || n > 8192) return SV_ERR_INVALID;
  cudaError_t r = cudaMemcpy(out_host, e->mega_dbg, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost);
  return r == cudaSuccess ? SV_OK : SV_ERR_CUDA;
}

const char* sv_engine_describe(sv_engine* e) {
  if (!e) return "";
  char buf[512];
  snprintf(buf, sizeof(buf), "decode=%s weights=%s attn=cluster-dsmem pdl=%d linear_impl=%d max_batch=%d flow[%s]%s%s",
           !e->fused_decode ? "legacy-kernels" : e->use_flow ? (e->flow_realloc ? "dataflow-kernel-setmaxnreg" : "dataflow-kernel") : "ring-gemv-graph",
           e->ring_tiles ? "slab-tiled" : "row-major", (int)e->use_pdl, e->linear_impl, e->d.max_batch, decode_flow_status(),
           e->flow_requested && !e->use_flow && e->d.max_batch > 8 ? " SV_FLOW ignored: the dataflow kernel holds 8 rows, max_batch > 8 runs the graph path" : "",
           e->use_flow ? " sessions, beam sessions and speculative decoding: graph path (the dataflow kernel has no per-row positions)" : "");
  e->describe = buf;
  return e->describe.c_str();
}

int sv_last_decode_timing(const sv_engine* e, float* ms, int32_t* steps) {
  if (!e) return SV_ERR_INVALID;
  if (ms) *ms = e->last_decode_ms;
  if (steps) *steps = e->last_decode_steps;
  return SV_OK;
}

// ---- single-kernel entry points ---------------------------------------------------------------
static std::string g_op_error;
static int op_fail(const char* what, cudaError_t r) {
  g_create_error = std::string(what) + ": " + cudaGetErrorString(r);
  return SV_ERR_CUDA;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

int sv_op_layernorm(const void* x, const void* w, const void* b, void* y, int32_t rows, int32_t cols, float eps,
                    void* stream) {
  const char* bad = nullptr;
  if (!x || !w || !b || !y) bad = "null pointer";
  else if (rows < 1 || cols < 8 || cols % 8) bad = "rows >= 1, cols >= 8 and cols % 8 == 0";
  else if (!(eps >= 0.f)) bad = "eps < 0";
  else if (!aligned16(x) || !aligned16(w) || !aligned16(b) || !aligned16(y)) bad = "x, w, b and y must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad layernorm arguments: %s", bad);
  launch_layernorm((const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)y, rows, cols, eps, cols, (cudaStream_t)stream);
  cudaError_t r = cudaGetLastError();
  return r == cudaSuccess ? SV_OK : op_fail("layernorm", r);
}

int sv_op_linear(int32_t impl, const void* x, const void* w, const void* bias, const void* residual, void* y, int32_t M,
                 int32_t N, int32_t K, int32_t act, void* stream) {
  const char* bad = nullptr;
  const bool wg_ok = wgmma_supported(M, N, K), rg_ok = K >= 32 && K % 32 == 0;
  if (!x || !w || !y) bad = "x, w and y are required";
  else if (impl != SV_LINEAR_AUTO && impl != SV_LINEAR_ROWGROUP && impl != SV_LINEAR_TCGEN05) bad = "unknown impl";
  else if (act < SV_ACT_NONE || act > SV_ACT_SILU) bad = "unknown act";
  else if (M < 1 || N < 1 || K < 1) bad = "M, N and K must be >= 1";
  else if (impl == SV_LINEAR_ROWGROUP && !rg_ok) bad = "rowgroup needs K % 32 == 0";
  else if (impl == SV_LINEAR_TCGEN05 && !wg_ok) bad = "wgmma needs N % 8 == 0 and K % 64 == 0";
  else if (impl == SV_LINEAR_AUTO && !rg_ok && !(M > 32 && wg_ok)) bad = "no kernel for this shape (AUTO)";
  else if (!aligned16(x) || !aligned16(w) || !aligned16(y) || !aligned16(bias) || !aligned16(residual))
    bad = "x, w, bias, residual and y must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad linear arguments: %s (M=%d N=%d K=%d)", bad, M, N, K);
  int r = do_linear(nullptr, impl, (const bf16*)x, (const bf16*)w, (const bf16*)bias, (const bf16*)residual, (bf16*)y, M,
                    N, K, act, (cudaStream_t)stream);
  if (r != SV_OK) return r;
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? SV_OK : op_fail("linear", ce);
}

int sv_op_attention_vit(const void* qkv, void* out, int32_t batch, int32_t seq, int32_t heads, void* stream) {
  const char* bad = nullptr;
  if (!qkv || !out) bad = "null pointer";
  else if (batch < 1 || seq < 1 || heads < 1) bad = "batch, seq and heads must be >= 1";
  else if (!aligned16(qkv) || !aligned16(out)) bad = "qkv and out must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad attention_vit arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int seq_pad = (seq + 31) / 32 * 32;
  bf16* vt = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&vt), (size_t)batch * heads * 64 * seq_pad * 2);
  if (r != cudaSuccess) return op_fail("attention_vit alloc", r);
  launch_vit_transpose_v((const bf16*)qkv, vt, batch, seq, heads, seq_pad, st);
  launch_attention_vit((const bf16*)qkv, vt, (bf16*)out, batch, seq, heads, seq_pad, st);
  r = cudaStreamSynchronize(st);
  cudaFree(vt);
  return r == cudaSuccess ? SV_OK : op_fail("attention_vit", r);
}

// The decoder prefill's attention as run_prefill issues it: the K/V columns of qkv rows [b][0, seq) go to cache slots
// [0, seq) of image b (kv_write_kernel), then every token attends causally to the cache (attention_heads_kernel).
int sv_op_attention_prefill(const void* qkv, void* kcache, void* vtcache, void* out, int32_t batch, int32_t seq,
                            int32_t n_head, int32_t n_kv, int32_t tcap, int32_t window, void* stream) {
  const char* bad = nullptr;
  if (!qkv || !kcache || !vtcache || !out) bad = "null pointer";
  else if (batch < 1 || seq < 1) bad = "batch and seq must be >= 1";
  else if (n_head < 1 || n_kv < 1 || n_head % n_kv || n_head / n_kv > 16) bad = "n_head % n_kv != 0 or group > 16";
  else if (tcap < 32 || tcap % 32) bad = "tcap % 32 != 0";
  else if (seq > tcap) bad = "seq > tcap";
  else if (window < 0) bad = "window < 0";
  else if (!aligned16(qkv) || !aligned16(kcache) || !aligned16(vtcache) || !aligned16(out))
    bad = "qkv, the caches and out must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad attention_prefill arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 128;
  launch_kv_scatter((const bf16*)qkv, (bf16*)kcache, (bf16*)vtcache, batch, seq, n_head * D, n_kv, D, tcap, 0, st);
  launch_attention_heads((const bf16*)qkv, (n_head + 2 * n_kv) * D, (const bf16*)kcache, (const bf16*)vtcache, (bf16*)out,
                         batch, seq, n_head, n_kv, D, tcap, window, st);
  cudaError_t r = cudaGetLastError();
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  return r == cudaSuccess ? SV_OK : op_fail("attention_prefill", r);
}

int sv_op_attention_mqa(const void* qkv, void* out, int32_t batch, int32_t seq, int32_t heads, void* stream) {
  if (!qkv || !out || batch < 1 || seq < 1 || heads < 1 || heads > 16) return fail(nullptr, SV_ERR_INVALID, "bad attention arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 128, tcap = (seq + 31) / 32 * 32;
  const size_t n = (size_t)batch * tcap * D;
  bf16* kc = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&kc), 2 * n * 2);
  if (r != cudaSuccess) return op_fail("attention_mqa alloc", r);
  r = cudaMemsetAsync(kc, 0, 2 * n * 2, st);
  const int rc = r == cudaSuccess ? sv_op_attention_prefill(qkv, kc, kc + n, out, batch, seq, heads, 1, tcap, 0, stream)
                                  : op_fail("attention_mqa", r);
  cudaFree(kc);
  return rc;
}

// The scoring chunk's attention as run_score_chunk issues it: the K/V columns of qkv rows [b][0, C) go to cache slots
// [pos0, pos0 + C) of image b (kv_write_kernel at pos0), then query t attends to keys [0, pos0 + t] of the cache
// (attention_chunk_kernel).  Slots < pos0 hold the prefix an earlier call wrote; slots >= pos0 + C are neither written
// nor used.
int sv_op_attention_score(const void* qkv, void* kcache, void* vtcache, void* out, int32_t batch, int32_t C, int32_t pos0,
                          int32_t n_head, int32_t n_kv, int32_t tcap, int32_t window, void* stream) {
  const char* bad = nullptr;
  if (!qkv || !kcache || !vtcache || !out) bad = "null pointer";
  else if (batch < 1 || C < 1 || pos0 < 0) bad = "batch, C >= 1 and pos0 >= 0";
  else if (n_head < 1 || n_kv < 1 || n_head % n_kv || n_head / n_kv > 16) bad = "n_head % n_kv != 0 or group > 16";
  else if (tcap < 32 || tcap % 32) bad = "tcap % 32 != 0";
  else if ((int64_t)pos0 + C > tcap) bad = "pos0 + C > tcap";
  else if (window < 0) bad = "window < 0";
  else if (!aligned16(qkv) || !aligned16(kcache) || !aligned16(vtcache) || !aligned16(out))
    bad = "qkv, the caches and out must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad attention_score arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 128, cols = (n_head + 2 * n_kv) * D;
  launch_kv_scatter((const bf16*)qkv, (bf16*)kcache, (bf16*)vtcache, batch, C, n_head * D, n_kv, D, tcap, pos0, st);
  cudaError_t r = launch_attention_chunk((const bf16*)qkv, cols, C, (const bf16*)kcache, (const bf16*)vtcache, (bf16*)out,
                                         batch, C, pos0, n_head, n_kv, D, tcap, window, st);
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  return r == cudaSuccess ? SV_OK : op_fail("attention_score", r);
}

// All `seq` positions of qkv go to zeroed caches this call allocates, then sv_op_attention_score runs the queries of
// [q0, seq) (copied to rows of their own) against them.
int sv_op_attention_chunk(const void* qkv, void* out, int32_t batch, int32_t seq, int32_t q0, int32_t n_head, int32_t n_kv,
                          int32_t window, void* stream) {
  if (!qkv || !out || batch < 1 || seq < 1 || q0 < 0 || q0 >= seq || n_kv < 1 || n_head % n_kv || n_head / n_kv > 16 ||
      window < 0)
    return fail(nullptr, SV_ERR_INVALID, "bad attention arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 128, tcap = (seq + 31) / 32 * 32, cols = (n_head + 2 * n_kv) * D, C = seq - q0;
  const size_t n = (size_t)batch * n_kv * tcap * D, row = (size_t)cols * 2;
  bf16* kc = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&kc), 2 * n * 2 + (size_t)batch * C * row);
  if (r != cudaSuccess) return op_fail("attention_chunk alloc", r);
  bf16* vc = kc + n;
  bf16* chunk = vc + n;
  r = cudaMemsetAsync(kc, 0, 2 * n * 2, st);
  if (r == cudaSuccess) r = cudaMemcpy2DAsync(chunk, C * row, (const bf16*)qkv + (size_t)q0 * cols, seq * row, C * row, batch,
                                              cudaMemcpyDeviceToDevice, st);
  int rc = SV_OK;
  if (r == cudaSuccess) {
    launch_kv_scatter((const bf16*)qkv, kc, vc, batch, seq, n_head * D, n_kv, D, tcap, 0, st);
    rc = sv_op_attention_score(chunk, kc, vc, out, batch, C, q0, n_head, n_kv, tcap, window, stream);
  } else {
    rc = op_fail("attention_chunk", r);
  }
  cudaFree(kc);
  return rc;
}

// Scratch for the (max, sum) partials of M rows and their target logits.  The target logits start as NaN, so a target
// that no column matches (outside [0, N)) gives NaN instead of whatever the memory held.
static cudaError_t logprob_scratch(int M, int N, cudaStream_t st, float2** part, float** tl) {
  const size_t np = (size_t)M * lm_logprob_ntiles(N);
  void* buf = nullptr;
  cudaError_t r = cudaMalloc(&buf, np * sizeof(float2) + (size_t)M * sizeof(float));
  if (r != cudaSuccess) return r;
  *part = reinterpret_cast<float2*>(buf);
  *tl = reinterpret_cast<float*>(*part + np);
  r = cudaMemsetAsync(*tl, 0xff, (size_t)M * sizeof(float), st);      // 0xffffffff: a quiet NaN
  if (r != cudaSuccess) cudaFree(buf);
  return r;
}

int sv_op_lm_logprob(const void* x, const void* w, const int32_t* targets, float* logprob, int32_t M, int32_t N, int32_t K,
                     void* stream) {
  const char* bad = nullptr;
  if (!x || !w || !targets || !logprob) bad = "null pointer";
  else if (M < 1 || N < 1 || K < 64 || K % 64) bad = "M, N >= 1 and K % 64 == 0";
  else if (!aligned16(x) || !aligned16(w) || !aligned4(targets) || !aligned4(logprob))
    bad = "x and w must be 16-byte aligned, targets and logprob 4-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad lm_logprob arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  float2* part = nullptr;
  float* tl = nullptr;
  cudaError_t r = logprob_scratch(M, N, st, &part, &tl);
  if (r != cudaSuccess) return op_fail("lm_logprob alloc", r);
  r = launch_lm_logprob_partials((const bf16*)x, (const bf16*)w, targets, part, tl, M, N, K, st);
  if (r == cudaSuccess) {
    launch_logprob_merge(part, lm_logprob_ntiles(N), tl, M, M, 0, M, logprob, st);
    r = cudaGetLastError();
    if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  }
  cudaFree(part);
  return r == cudaSuccess ? SV_OK : op_fail("lm_logprob", r);
}

// Position 0 of a scoring call: the log-likelihood of targets[m] under resident bf16 logits [M][vocab]
// (logits_logprob_partials_kernel, then the merge).
int sv_op_logits_logprob(const void* logits, const int32_t* targets, float* logprob, int32_t M, int32_t vocab, void* stream) {
  const char* bad = nullptr;
  if (!logits || !targets || !logprob) bad = "null pointer";
  else if (M < 1 || vocab < 1) bad = "M and vocab must be >= 1";
  else if (!aligned16(logits) || !aligned4(targets) || !aligned4(logprob))
    bad = "logits must be 16-byte aligned, targets and logprob 4-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad logits_logprob arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  float2* part = nullptr;
  float* tl = nullptr;
  cudaError_t r = logprob_scratch(M, vocab, st, &part, &tl);
  if (r != cudaSuccess) return op_fail("logits_logprob alloc", r);
  launch_logits_logprob_partials((const bf16*)logits, vocab, M, targets, part, tl, st);
  launch_logprob_merge(part, lm_logprob_ntiles(vocab), tl, M, M, 0, M, logprob, st);
  r = cudaGetLastError();
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(part);
  return r == cudaSuccess ? SV_OK : op_fail("logits_logprob", r);
}

// ---- the decode-step kernels one at a time, over caches the caller owns -------------------------------------------
// Every argument is checked on the host before anything is allocated or launched: a shape the kernels were not built
// for returns SV_ERR_INVALID instead of reaching a device trap (the ring's bounded waits) or an abort.
constexpr size_t kOpState = 512;     // scratch header holding the GenState / RowState the kernels read
static_assert(sizeof(GenState) <= kOpState && sizeof(RowState) <= kOpState, "the state structs fit the scratch header");

int sv_op_attention_decode(int32_t impl, int32_t per_row, const void* qkv, const void* kcache, const void* vtcache, void* out,
                           const int32_t* lens_host, int32_t batch, int32_t n_head, int32_t n_kv, int32_t tcap,
                           int32_t nsplit, int32_t window, void* stream) {
  const char* bad = nullptr;
  if (!qkv || !kcache || !vtcache || !out || !lens_host) bad = "null pointer";
  else if (impl != SV_ATTN_DECODE_SPLIT && impl != SV_ATTN_DECODE_CLUSTER) bad = "unknown impl";
  else if (per_row < 0 || per_row > 2) bad = "per_row is 0, 1 or 2";
  else if (per_row == 2 && (impl != SV_ATTN_DECODE_CLUSTER || window != 0)) bad = "the column map (per_row = 2) is cluster-only with window 0";
  else if (batch < 1 || batch > kSessionRows) bad = "batch not in [1, 16]";
  else if (n_head < 1 || n_kv < 1 || n_head % n_kv || n_head / n_kv > 16) bad = "n_head % n_kv != 0 or group > 16";
  else if (tcap < 32 || tcap % 32) bad = "tcap % 32 != 0";
  else if (nsplit < 1 || nsplit > (impl == SV_ATTN_DECODE_CLUSTER ? 8 : kMaxSplit)) bad = "nsplit not in [1, 128] (split) / [1, 8] (cluster)";
  else if (window < 0) bad = "window < 0";
  else if (!aligned16(qkv) || !aligned16(kcache) || !aligned16(vtcache)) bad = "qkv and the caches must be 16-byte aligned";
  for (int b = 0; !bad && b < batch; ++b) {
    if (per_row == 2) { if (lens_host[b] < 0 || lens_host[b] >= tcap) bad = "a column position is not in [0, tcap - 1]"; }
    else if (lens_host[b] < 1 || lens_host[b] > tcap) bad = "a length is not in [1, tcap]";
    else if (!per_row && lens_host[b] != lens_host[0]) bad = "per_row = 0 needs equal lengths";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad attention_decode arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 128, cols = (n_head + 2 * n_kv) * D;
  const size_t part_floats = impl == SV_ATTN_DECODE_SPLIT ? (size_t)batch * n_kv * nsplit * (32 + 16 * D) : 0;
  GenState gs{};
  RowState rs{};
  svspec::ColMap cm{};
  gs.cur_len = lens_host[0] - 1;
  for (int b = 0; b < batch; ++b) rs.row_len[b] = lens_host[b] - 1;    // the new token's key sits at lens - 1
  cm.n_live = batch;                                                   // every column reads cache row 0 (row[c] = 0)
  for (int b = 0; b < batch; ++b) cm.pos[b] = lens_host[b];
  static_assert(sizeof(svspec::ColMap) <= kOpState, "the column map fits the scratch header");
  void* buf = nullptr;
  cudaError_t r = cudaMalloc(&buf, kOpState + part_floats * sizeof(float));
  if (r != cudaSuccess) return op_fail("attention_decode alloc", r);
  GenState* d_gs = reinterpret_cast<GenState*>(buf);
  RowState* d_rs = reinterpret_cast<RowState*>(buf);
  svspec::ColMap* d_cm = reinterpret_cast<svspec::ColMap*>(buf);
  float* partial = reinterpret_cast<float*>(static_cast<char*>(buf) + kOpState);
  if (per_row == 2) r = cudaMemcpyAsync(d_cm, &cm, sizeof(cm), cudaMemcpyHostToDevice, st);
  else if (per_row) r = cudaMemcpyAsync(d_rs, &rs, sizeof(rs), cudaMemcpyHostToDevice, st);
  else r = cudaMemcpyAsync(d_gs, &gs, sizeof(gs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) {
    if (impl == SV_ATTN_DECODE_SPLIT) {
      launch_attention_decode((const bf16*)qkv, cols, (const bf16*)kcache, (const bf16*)vtcache, (bf16*)out, partial, d_gs,
                              batch, n_head, n_kv, D, tcap, nsplit, window, st, per_row == 1 ? d_rs : nullptr);
      r = cudaGetLastError();
    } else {
      r = attention_decode_cluster_init();
      if (r == cudaSuccess)
        r = launch_attention_decode_cluster((const bf16*)qkv, cols, (const bf16*)kcache, (const bf16*)vtcache, (bf16*)out, d_gs,
                                            batch, n_head, n_kv, D, tcap, nsplit, window, false, st, per_row == 1 ? d_rs : nullptr,
                                            per_row == 2 ? d_cm : nullptr);
    }
  }
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  return r == cudaSuccess ? SV_OK : op_fail("attention_decode", r);
}

int32_t sv_op_ring_ntiles(int32_t N) { return N < 1 ? 0 : gemv_ring_ntiles(N); }
int32_t sv_op_ring_row_stride(int32_t B) { return 8 * ring_row_groups(B); }

int sv_op_gemv_ring(const sv_op_ring* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad gemv_ring arguments: null descriptor");
  const sv_op_ring& o = *args;
  const bool ln = o.ln_w != nullptr;
  const char* bad = nullptr;
  if (!o.x || !o.w || !o.y) bad = "x, w and y are required";
  else if (o.B < 1 || o.B > gemv_ring_max_rows()) bad = "B not in [1, gemv_ring_max_rows()]";
  else if (o.N < 1 || !gemv_ring_supported(o.K, ln)) bad = "N < 1 or K % 32 != 0";
  else if (ln != (o.ln_b != nullptr)) bad = "ln_w and ln_b go together";
  else if (!aligned16(o.x) || !aligned16(o.w) || (ln && (!aligned16(o.ln_w) || !aligned16(o.ln_b))))
    bad = "x, w, ln_w and ln_b must be 16-byte aligned";
  else if (o.act < SV_ACT_NONE || o.act > SV_ACT_SILU) bad = "unknown act";
  else if (o.tiled != 0 && o.tiled != 1) bad = "tiled is 0 or 1";
  else if (o.epi < 0 || o.epi > 2 || (o.epi != 0 && !ln)) bad = "epi is 0 (plain), 1 (QKV) or 2 (lm_head); 1 and 2 need the LayerNorm";
  else if (ln && gemv_ring_ln_streamed(o.K) && (o.B > 8 || o.epi == 1))
    bad = "a LayerNorm over more than two slabs of K has ring kernels for <= 8 rows and no QKV epilogue";
  else if (o.epi == 2 && (!o.amax_val || !o.amax_idx)) bad = "lm_head needs amax_val and amax_idx";
  else if (o.epi == 1) {
    if (!o.kcache || !o.vtcache || !o.pos_host) bad = "QKV needs kcache, vtcache and pos_host";
    else if (o.n_head < 1 || o.n_kv < 1 || o.n_head % o.n_kv || o.N != (o.n_head + 2 * o.n_kv) * 128) bad = "N != (n_head + 2 n_kv) * 128";
    else if (o.tcap < 32 || o.tcap % 32) bad = "tcap % 32 != 0";
    else if (o.per_row < 0 || o.per_row > 2) bad = "per_row is 0, 1 or 2";
    else if (o.per_row == 2 && (o.B > svspec::kMaxCols || o.pos_host[o.B] < 0 || o.pos_host[o.B] > o.B))
      bad = "the column map needs 0 <= n_live = pos_host[B] <= B";
    for (int b = 0; !bad && b < (o.per_row ? o.B : 1); ++b)
      if (o.pos_host[b] < 0 || o.pos_host[b] > o.tcap) bad = "a position is not in [0, tcap]";
    // the map kernel prefetches row 0's keys [0, pos[0] + n_live): svspec::set_map's form keeps that inside the row
    for (int b = 0; !bad && o.per_row == 2 && b < o.B; ++b)
      if (o.pos_host[b] >= o.tcap || o.pos_host[0] + o.pos_host[o.B] > o.tcap) bad = "a column position is not in [0, tcap - 1] or pos[0] + n_live > tcap";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad gemv_ring arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int ncta = gemv_ring_ncta();
  const size_t tiled_bytes = o.tiled ? flow_tiled_bytes(o.N, o.K, ncta) : 0;
  void* buf = nullptr;
  cudaError_t r = cudaMalloc(&buf, kOpState + tiled_bytes);
  if (r != cudaSuccess) return op_fail("gemv_ring alloc", r);
  GenState gs{};
  RowState rs{};
  svspec::ColMap cm{};
  const bool map = o.epi == 1 && o.per_row == 2;
  if (o.epi == 1) {
    gs.cur_len = o.pos_host[0];
    for (int b = 0; o.per_row == 1 && b < o.B; ++b) rs.row_len[b] = o.pos_host[b];
    if (map) cm.n_live = o.pos_host[o.B];                              // svspec::set_map's form: every column in row 0
    for (int b = 0; map && b < o.B; ++b) cm.pos[b] = o.pos_host[b];
  }
  GenState* d_gs = reinterpret_cast<GenState*>(buf);
  RowState* d_rs = reinterpret_cast<RowState*>(buf);
  svspec::ColMap* d_cm = reinterpret_cast<svspec::ColMap*>(buf);
  uint8_t* wt = static_cast<uint8_t*>(buf) + kOpState;
  if (map) r = cudaMemcpyAsync(d_cm, &cm, sizeof(cm), cudaMemcpyHostToDevice, st);
  else if (o.per_row) r = cudaMemcpyAsync(d_rs, &rs, sizeof(rs), cudaMemcpyHostToDevice, st);
  else r = cudaMemcpyAsync(d_gs, &gs, sizeof(gs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = gemv_ring_init();
  if (r == cudaSuccess) {
    if (o.tiled) launch_flow_repack((const bf16*)o.w, (const bf16*)o.bias, wt, o.N, o.K, ncta, st);
    RingGemvLaunch g{};
    g.X = (const bf16*)o.x; g.W = (const bf16*)o.w; g.Wt = o.tiled ? wt : nullptr; g.bias = (const bf16*)o.bias;
    g.res = (const bf16*)o.residual; g.ln_w = (const bf16*)o.ln_w; g.ln_b = (const bf16*)o.ln_b; g.Y = (bf16*)o.y;
    g.B = o.B; g.N = o.N; g.K = o.K; g.act = o.act; g.epi = o.epi; g.ln_eps = o.ln_eps;
    g.n_head = o.n_head; g.n_kv = o.n_kv; g.tcap = o.tcap; g.state = d_gs;
    g.kcache = (bf16*)o.kcache; g.vtcache = (bf16*)o.vtcache; g.amax_val = o.amax_val; g.amax_idx = o.amax_idx;
    g.pdl = false; g.rows = (o.epi == 1 && o.per_row == 1) ? d_rs : nullptr; g.cmap = map ? d_cm : nullptr;
    launch_gemv_ring(g, st);
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  return r == cudaSuccess ? SV_OK : op_fail("gemv_ring", r);
}

int sv_op_rope_table(void* cos_t, void* sin_t, int32_t max_pos, int32_t d, float theta, void* stream) {
  if (!cos_t || !sin_t || max_pos < 1 || d < 2 || d % 2 || d / 2 > kRopeMaxHalf || !(theta > 0.f))
    return fail(nullptr, SV_ERR_INVALID, "bad rope_table arguments");
  cudaStream_t st = (cudaStream_t)stream;
  launch_rope_table((bf16*)cos_t, (bf16*)sin_t, max_pos, d, theta, st);
  cudaError_t r = cudaGetLastError();
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  return r == cudaSuccess ? SV_OK : op_fail("rope_table", r);
}

int sv_op_rope(void* qkv, const void* cos_t, const void* sin_t, int32_t rows, int32_t seq, int32_t n_head, int32_t n_kv,
               int32_t max_pos, int32_t pos0, const int32_t* pos_host, int32_t per_row, void* kcache, void* vtcache,
               int32_t tcap, void* stream) {
  const char* bad = nullptr;
  if (!qkv || !cos_t || !sin_t) bad = "null pointer";
  else if (rows < 1 || seq < 1 || n_head < 1 || n_kv < 1 || max_pos < 1 || pos0 < 0) bad = "rows, seq, n_head, n_kv, max_pos >= 1, pos0 >= 0";
  else if (kcache && (!vtcache || !pos_host || tcap < 32 || tcap % 32)) bad = "the KV append needs vtcache, pos_host and tcap % 32 == 0";
  else if (pos_host && (rows > kSessionRows || (per_row != 0 && per_row != 1))) bad = "one token per row: rows <= 16, per_row is 0 or 1";
  for (int b = 0; !bad && pos_host && b < rows; ++b) {
    if (pos_host[b] < 0) bad = "a position is < 0";
    else if (!per_row && pos_host[b] != pos_host[0]) bad = "per_row = 0 needs equal positions";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad rope arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 128, cols = (n_head + 2 * n_kv) * D;
  void* buf = nullptr;
  cudaError_t r = cudaSuccess;
  GenState* d_gs = nullptr;
  RowState* d_rs = nullptr;
  if (pos_host) {
    r = cudaMalloc(&buf, kOpState);
    if (r != cudaSuccess) return op_fail("rope alloc", r);
    GenState gs{};
    RowState rs{};
    gs.cur_len = pos_host[0];
    for (int b = 0; b < rows; ++b) rs.row_len[b] = pos_host[b];
    if (per_row) { d_rs = reinterpret_cast<RowState*>(buf); r = cudaMemcpyAsync(d_rs, &rs, sizeof(rs), cudaMemcpyHostToDevice, st); }
    else { d_gs = reinterpret_cast<GenState*>(buf); r = cudaMemcpyAsync(d_gs, &gs, sizeof(gs), cudaMemcpyHostToDevice, st); }
  }
  if (r == cudaSuccess) {
    if (kcache)
      launch_rope_append((bf16*)qkv, rows, cols, n_head, n_kv, D, (const bf16*)cos_t, (const bf16*)sin_t, (bf16*)kcache,
                         (bf16*)vtcache, d_gs, tcap, max_pos, false, st, d_rs);
    else
      launch_rope((bf16*)qkv, rows, pos_host ? 1 : seq, cols, n_head + n_kv, D, (const bf16*)cos_t, (const bf16*)sin_t, d_gs,
                  max_pos, pos0, st, d_rs);
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  if (buf) cudaFree(buf);
  return r == cudaSuccess ? SV_OK : op_fail("rope", r);
}

// ---- the decode step as the engine chains it, over weights, caches and buffers the caller owns ----------------------
static_assert(sizeof(sv_op_chain) == 296 && offsetof(sv_op_chain, layer_stride) == 136 && offsetof(sv_op_chain, pdl_used) == 292,
              "sv_op_chain layout (the ctypes binding mirrors it)");
int sv_op_decode_chain(sv_op_chain* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad decode_chain arguments: null descriptor");
  sv_op_chain& o = *args;
  const bool fused = o.mode == SV_CHAIN_FUSED;
  const int D = 128, B = o.B;
  const int64_t qkv_cols = (int64_t)o.hidden + 2 * (int64_t)o.n_kv * D;
  const char* bad = nullptr;
  auto al = [](const void* p) { return aligned16(p); };
  auto stride_ok = [&](int64_t s, int64_t width) { return s == 0 || (s >= (int64_t)B * width && s % 8 == 0); };
  if (o.mode != SV_CHAIN_FUSED && o.mode != SV_CHAIN_PER_OP) bad = "unknown mode";
  else if (o.n_layer < 1) bad = "n_layer < 1";
  else if (B < 1 || B > kSessionRows) bad = "B not in [1, 16]";
  else if (o.per_row != 0 && o.per_row != 1) bad = "per_row is 0 or 1";
  else if (o.n_head < 1 || o.n_kv < 1 || o.n_head % o.n_kv || o.n_head / o.n_kv > 16) bad = "n_head % n_kv != 0 or group > 16";
  else if (o.hidden != o.n_head * D) bad = "hidden != n_head * 128";
  else if (o.hidden % 64 || o.n_inner < 64 || o.n_inner % 64) bad = "hidden and n_inner must be multiples of 64";
  else if (o.vocab < 1 || o.n_positions < 1) bad = "vocab and n_positions must be >= 1";
  else if (o.tcap < 32 || o.tcap % 32) bad = "tcap % 32 != 0";
  else if (o.window < 0) bad = "window < 0";
  else if (!(o.ln_eps >= 0.f)) bad = "ln_eps < 0";
  else if ((o.rope | o.pdl | o.graph | o.tiled | o.lm_head_tail) & ~1) bad = "rope, pdl, graph, tiled and lm_head_tail are 0 or 1";
  else if (o.rope && (!o.rope_cos || !o.rope_sin || !al(o.rope_cos) || !al(o.rope_sin))) bad = "rope needs 16-byte aligned rope_cos and rope_sin";
  else if (o.tiled && !fused) bad = "tiled weights are streamed by the FUSED chain only";
  else if (fused && (!gemv_ring_supported(o.hidden, true) || !gemv_ring_supported(o.n_inner, false))) bad = "no ring GEMV for these widths";
  else if (fused && !o.rope && gemv_ring_ln_streamed(o.hidden))
    bad = "the FUSED v1 chain appends K/V in the c_attn epilogue, which a LayerNorm over more than two slabs does not have";
  else if (fused && B > 8 && (o.rope || gemv_ring_ln_streamed(o.hidden) || B > gemv_ring_max_rows()))
    bad = "the FUSED chain over more than 8 rows needs v1 with a register-resident LayerNorm";
  else if (o.parts < 0 || o.parts > (fused ? 8 : kMaxSplit)) bad = "parts not in [0, 8] (FUSED) / [0, 128] (PER_OP)";
  else if (!o.layers || !o.pos_host || !o.kcache || !o.vtcache || !o.x || !o.qkv || !o.attn || !o.h || (!fused && !o.ln))
    bad = "null pointer (layers, pos_host, caches, x, qkv, attn, h; PER_OP also ln)";
  else if (o.ids && (!o.wte || !al(o.wte) || (o.wpe && !al(o.wpe)))) bad = "ids need a 16-byte aligned wte (and wpe)";
  else if (o.lm_head_tail && (!o.lm_head || !o.lnf_w || !o.lnf_b || !o.logits || !al(o.lm_head) || !al(o.lnf_w) || !al(o.lnf_b) ||
                              !al(o.logits) || (fused && (!o.amax_val || !o.amax_idx))))
    bad = "the lm_head tail needs 16-byte aligned lm_head, lnf_w, lnf_b and logits (FUSED: amax_val and amax_idx)";
  else if (o.layer_stride < (int64_t)B * o.n_kv * o.tcap * D) bad = "layer_stride < B * n_kv * tcap * 128";
  else if (!stride_ok(o.x_stride, o.hidden) || !stride_ok(o.ln_stride, o.hidden) || !stride_ok(o.qkv_stride, qkv_cols) ||
           !stride_ok(o.attn_stride, o.hidden) || !stride_ok(o.h_stride, o.n_inner))
    bad = "an activation stride is neither 0 nor a multiple of 8 of at least one slot (B rows)";
  else if (!al(o.kcache) || !al(o.vtcache) || !al(o.x) || (o.ln && !al(o.ln)) || !al(o.qkv) || !al(o.attn) || !al(o.h))
    bad = "the caches and activation buffers must be 16-byte aligned";
  for (int b = 0; !bad && b < B; ++b) {
    if (o.pos_host[b] < 0 || o.pos_host[b] >= o.tcap) bad = "a position is not in [0, tcap - 1]";
    else if (!o.per_row && o.pos_host[b] != o.pos_host[0]) bad = "per_row = 0 needs equal positions";
  }
  for (int l = 0; !bad && l < o.n_layer; ++l) {
    const void* const* p = &o.layers[l].ln1_w;
    for (int k = 0; !bad && k < 12; ++k)
      if (!p[k] || !al(p[k])) bad = "every layer weight must be given and 16-byte aligned";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad decode_chain arguments: %s", bad);

  cudaStream_t st = (cudaStream_t)stream;
  int total = 0;
  for (int b = 0; b < B; ++b) total = std::max(total, o.pos_host[b] + 1);
  const int parts = o.parts ? o.parts : decode_parts(fused, total);
  std::vector<DecLayer> layers(o.n_layer);
  for (int l = 0; l < o.n_layer; ++l) {
    const sv_op_chain_layer& s = o.layers[l];
    auto w = [](const void* p) { return const_cast<bf16*>(static_cast<const bf16*>(p)); };
    layers[l] = DecLayer{w(s.ln1_w), w(s.ln1_b), w(s.attn_w), w(s.attn_b), w(s.proj_w), w(s.proj_b), w(s.ln2_w), w(s.ln2_b),
                         w(s.fc_w), w(s.fc_b), w(s.fc2_w), w(s.fc2_b)};
  }
  // scratch: the state header, the split partials (PER_OP), the slab-tiled copies (tiled)
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const int ncta = fused ? gemv_ring_ncta() : 0;
  const size_t part_bytes = fused ? 0 : up((size_t)B * o.n_kv * kMaxSplit * (32 + 16 * D) * sizeof(float));
  size_t tile_bytes = 0;
  if (o.tiled) {
    tile_bytes = (size_t)o.n_layer * (up(flow_tiled_bytes((int)qkv_cols, o.hidden, ncta)) + up(flow_tiled_bytes(o.hidden, o.hidden, ncta)) +
                                      up(flow_tiled_bytes(o.n_inner, o.hidden, ncta)) + up(flow_tiled_bytes(o.hidden, o.n_inner, ncta)));
    if (o.lm_head_tail) tile_bytes += up(flow_tiled_bytes(o.vocab, o.hidden, ncta));
  }
  void* buf = nullptr;
  cudaError_t r = cudaMalloc(&buf, kOpState + part_bytes + tile_bytes);
  if (r != cudaSuccess) return op_fail("decode_chain alloc", r);
  uint8_t* q = static_cast<uint8_t*>(buf) + kOpState;
  DecodeChain c;
  c.attn_partial = fused ? nullptr : reinterpret_cast<float*>(q);
  q += part_bytes;
  std::vector<uint8_t*> t_attn, t_proj, t_fc, t_fc2;
  if (o.tiled) {
    auto tile = [&](const bf16* W, const bf16* bias, int N, int K) {
      uint8_t* t = q;
      q += up(flow_tiled_bytes(N, K, ncta));
      launch_flow_repack(W, bias, t, N, K, ncta, st);
      return t;
    };
    for (const DecLayer& L : layers) {
      t_attn.push_back(tile(L.attn_w, L.attn_b, (int)qkv_cols, o.hidden));
      t_proj.push_back(tile(L.proj_w, L.proj_b, o.hidden, o.hidden));
      t_fc.push_back(tile(L.fc_w, L.fc_b, o.n_inner, o.hidden));
      t_fc2.push_back(tile(L.fc2_w, L.fc2_b, o.hidden, o.n_inner));
    }
    c.t_attn = t_attn.data(); c.t_proj = t_proj.data(); c.t_fc = t_fc.data(); c.t_fc2 = t_fc2.data();
    if (o.lm_head_tail) c.t_lm_head = tile((const bf16*)o.lm_head, nullptr, o.vocab, o.hidden);
  }
  GenState gs{};
  RowState rs{};
  gs.cur_len = o.pos_host[0];
  for (int b = 0; b < B; ++b) rs.row_len[b] = o.pos_host[b];
  c.n_layer = o.n_layer; c.layers = layers.data();
  c.kcache = (bf16*)o.kcache; c.vtcache = (bf16*)o.vtcache; c.layer_stride = o.layer_stride;
  c.state = reinterpret_cast<GenState*>(buf);
  c.rows = o.per_row ? reinterpret_cast<const RowState*>(buf) : nullptr;
  c.H = o.hidden; c.I = o.n_inner; c.n_head = o.n_head; c.n_kv = o.n_kv; c.D = D; c.qkv_cols = (int)qkv_cols; c.vocab = o.vocab;
  c.n_positions = o.n_positions; c.tcap = o.tcap; c.window = o.window; c.ln_eps = o.ln_eps; c.rope = o.rope != 0;
  c.rope_cos = (const bf16*)o.rope_cos; c.rope_sin = (const bf16*)o.rope_sin; c.wte = (const bf16*)o.wte; c.wpe = (const bf16*)o.wpe;
  c.lnf_w = (const bf16*)o.lnf_w; c.lnf_b = (const bf16*)o.lnf_b; c.lm_head = (const bf16*)o.lm_head;
  c.x = (bf16*)o.x; c.ln = (bf16*)o.ln; c.qkv = (bf16*)o.qkv; c.attn = (bf16*)o.attn; c.h = (bf16*)o.h;
  c.sx = o.x_stride; c.sln = o.ln_stride; c.sqkv = o.qkv_stride; c.sattn = o.attn_stride; c.sh = o.h_stride;
  c.lm_tail = o.lm_head_tail != 0; c.logits = (bf16*)o.logits; c.amax_val = o.amax_val; c.amax_idx = o.amax_idx;
  if (o.per_row) r = cudaMemcpyAsync(buf, &rs, sizeof(rs), cudaMemcpyHostToDevice, st);
  else r = cudaMemcpyAsync(buf, &gs, sizeof(gs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = gemv_ring_init();
  if (r == cudaSuccess) r = attention_decode_cluster_init();
  bool pdl_used = false;
  if (r == cudaSuccess && !o.graph) {
    run_chain(c, fused, o.ids, B, parts, fused && o.pdl, st);
    pdl_used = fused && o.pdl;
    r = cudaGetLastError();
  } else if (r == cudaSuccess) {
    // the capture goes to a stream of its own (the caller's may be the legacy stream, which cannot be captured)
    cudaStream_t cs = nullptr;
    GraphEntry g;
    r = cudaStreamSynchronize(st);
    if (r == cudaSuccess) r = cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
    if (r == cudaSuccess) r = capture_step(cs, fused && o.pdl, [&](bool pdl) { run_chain(c, fused, o.ids, B, parts, pdl, cs); }, g);
    if (r == cudaSuccess) r = cudaGraphLaunch(g.exec, cs);
    if (r == cudaSuccess) r = cudaStreamSynchronize(cs);
    pdl_used = g.pdl;
    if (g.exec) cudaGraphExecDestroy(g.exec);
    if (cs) cudaStreamDestroy(cs);
  }
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  if (r != cudaSuccess) return op_fail("decode_chain", r);
  o.parts_used = parts;
  o.pdl_used = pdl_used ? 1 : 0;
  return SV_OK;
}

// ---- the dataflow decode kernel over weights, caches and exchange buffers the caller owns ----------------------------
int64_t sv_op_flow_buffer_bytes(int32_t which, int32_t B, int32_t hidden, int32_t n_inner, int32_t n_kv, int32_t vocab) {
  if (B < 1 || hidden < 8 || hidden % 8 || n_inner < 8 || n_inner % 8 || n_kv < 1 || vocab < 1) return -1;
  const int64_t row = 64 * 4;          // bytes per 8 values: one flagged fragment per 256-byte chunk
  switch (which) {
    case SV_FLOW_XA: case SV_FLOW_XB: case SV_FLOW_ATT: return (int64_t)B * (hidden / 8) * row;
    case SV_FLOW_QKV: return (int64_t)B * ((hidden + 2 * (int64_t)n_kv * 128) / 8) * row;
    case SV_FLOW_HB: return (int64_t)B * (n_inner / 8) * row;
    case SV_FLOW_PART: return (int64_t)B * n_kv * decode_flow_max_splits() * decode_flow_partial_floats() * 8;
    case SV_FLOW_AMAX: return (int64_t)vocab * 8 * 8;        // a tile holds >= 1 row: at most `vocab` tiles on any device
    default: return -1;
  }
}

static_assert(sizeof(sv_op_flow) == 360 && offsetof(sv_op_flow, params) == 144 && offsetof(sv_op_flow, out_stride) == 232 &&
              offsetof(sv_op_flow, ncta_used) == 352, "sv_op_flow layout (the ctypes binding mirrors it)");
int sv_op_decode_flow(sv_op_flow* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad decode_flow arguments: null descriptor");
  sv_op_flow& o = *args;
  const int D = 128, B = o.B;
  const sv_gen_params& p = o.params;
  void* xbuf[7] = {o.xa, o.xb, o.qkv, o.att, o.hb, o.part, o.amax};
  const char* bad = nullptr;
  auto al = [](const void* q) { return aligned16(q); };
  if (o.n_layer < 1 || o.n_layer > decode_flow_max_layers()) bad = "n_layer not in [1, 24]";
  else if (B < 1 || B > 8) bad = "B not in [1, 8]";
  else if (o.n_head < 1 || o.n_kv < 1 || o.n_head % o.n_kv || o.n_head / o.n_kv > 16) bad = "n_head % n_kv != 0 or group > 16";
  else if (o.hidden != o.n_head * D) bad = "hidden != n_head * 128";
  else if (!decode_flow_shape_ok(o.hidden, o.n_inner, D, B, 0, false))
    bad = "the dataflow kernel takes hidden in {256, 512, 1024, 2048} and n_inner the same or a multiple of 1024 above 2048";
  else if (o.vocab < 1 || o.n_positions < 1) bad = "vocab and n_positions must be >= 1";
  else if (o.tcap < 32 || o.tcap % 32) bad = "tcap % 32 != 0";
  else if (!(o.ln_eps >= 0.f)) bad = "ln_eps < 0";
  else if ((o.first_plain | o.do_select | o.realloc | o.clear) & ~1) bad = "first_plain, do_select, realloc and clear are 0 or 1";
  else if (o.nsteps < 1 || o.step0 < 0 || o.cur_len0 < 0) bad = "nsteps must be >= 1, step0 and cur_len0 >= 0";
  else if ((int64_t)o.cur_len0 + o.nsteps > o.tcap - 1) bad = "cur_len0 + nsteps > tcap - 1";
  else if ((int64_t)o.cur_len0 + o.nsteps > decode_flow_max_keys()) bad = "cur_len0 + nsteps > 16384 (the attention's item split)";
  else if (o.l2_ahead < 0 || o.l2_ahead > 64) bad = "l2_ahead not in [0, 64]";
  else if (o.clear && !o.first_plain) bad = "clear zeroes the xa words: the first step's input must come from x_plain (first_plain = 1)";
  else if (!o.layers || !o.wte || !o.lnf_w || !o.lnf_b || !o.lm_head || !o.kcache || !o.vtcache || !o.x_plain || !o.logits)
    bad = "null pointer (layers, wte, lnf_w, lnf_b, lm_head, caches, x_plain, logits)";
  else if (!o.xa || !o.xb || !o.qkv || !o.att || !o.hb || !o.part || !o.amax) bad = "null exchange buffer (xa xb qkv att hb part amax)";
  else if (!al(o.wte) || !al(o.wpe) || !al(o.lnf_w) || !al(o.lnf_b) || !al(o.lm_head) || !al(o.kcache) || !al(o.vtcache) ||
           !al(o.x_plain) || !al(o.logits))
    bad = "wte, wpe, lnf_w, lnf_b, lm_head, the caches, x_plain and logits must be 16-byte aligned";
  else if (!al(o.xa) || !al(o.xb) || !al(o.qkv) || !al(o.att) || !al(o.hb) || !al(o.part) || !al(o.amax))
    bad = "the exchange buffers must be 16-byte aligned";
  else if (o.layer_stride < (int64_t)B * o.n_kv * o.tcap * D || o.layer_stride % 8) bad = "layer_stride < B * n_kv * tcap * 128 or not a multiple of 8";
  else if ((bad = gen_params_error(p))) {}
  else if (o.do_select) {
    if (p.do_sample) bad = "the dataflow kernel selects greedily: do_sample must be 0";
    else if (!o.seen || !o.out_ids || !o.next_ids || !o.counters_host || !o.unfinished_host)
      bad = "do_select needs seen, out_ids, next_ids, counters_host and unfinished_host";
    else if (o.out_stride < 1) bad = "out_stride < 1";
    else if (o.counters_host[0] < 0 || o.counters_host[1] < 0) bad = "step and cur_len must be >= 0";
    else if (!o.counters_host[2] && (int64_t)o.counters_host[0] + o.nsteps > o.out_stride) bad = "step + nsteps > out_stride";
  }
  for (int l = 0; !bad && l < o.n_layer; ++l) {
    const void* const* w = &o.layers[l].ln1_w;
    for (int k = 0; !bad && k < 12; ++k)
      if (!w[k] || !al(w[k])) bad = "every layer weight must be given and 16-byte aligned";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad decode_flow arguments: %s", bad);

  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t r = decode_flow_init();
  if (r != cudaSuccess) return op_fail("decode_flow init", r);
  if (!decode_flow_supported(o.hidden, o.n_inner, D, B, 0, false))
    return fail(nullptr, SV_ERR_UNSUPPORTED, "the dataflow kernel cannot run on this device: %s", decode_flow_status());
  if (o.realloc && !decode_flow_realloc_supported())
    return fail(nullptr, SV_ERR_UNSUPPORTED, "the register-reallocating variant cannot run on this device: %s", decode_flow_status());
  const int ncta = decode_flow_ncta();
  const int64_t qkv_cols = (int64_t)o.hidden + 2 * (int64_t)o.n_kv * D;
  if (o.clear) {
    for (int i = 0; r == cudaSuccess && i < 7; ++i)
      r = cudaMemsetAsync(xbuf[i], 0, (size_t)sv_op_flow_buffer_bytes(i, B, o.hidden, o.n_inner, o.n_kv, o.vocab), st);
    if (r != cudaSuccess) return op_fail("decode_flow clear", r);
  }
  if (!o.first_plain) {
    // the first step polls xa for the tag of phase step0 * (n_layer + 1): words without it would never be accepted
    std::vector<uint32_t> w((size_t)sv_op_flow_buffer_bytes(SV_FLOW_XA, B, o.hidden, o.n_inner, o.n_kv, o.vocab) / 4);
    r = cudaMemcpyAsync(w.data(), o.xa, w.size() * 4, cudaMemcpyDeviceToHost, st);
    if (r == cudaSuccess) r = cudaStreamSynchronize(st);
    if (r != cudaSuccess) return op_fail("decode_flow xa read-back", r);
    const uint32_t gp = (uint32_t)o.step0 * (uint32_t)(o.n_layer + 1), E0 = ((gp & 0x7fffu) + 1u) << 16;
    for (int b = 0; b < B; ++b)
      for (int i = 0; i < o.hidden; ++i)
        if ((w[(size_t)b * (o.hidden / 8) * 64 + (size_t)(i >> 3) * 64 + (i & 7)] & 0xffff0000u) != E0)
          return fail(nullptr, SV_ERR_INVALID,
                      "bad decode_flow arguments: first_plain = 0 but xa word %d of row %d does not carry the tag of step %d", i, b, o.step0);
  }
  // scratch: GenState, GenParamsDev, the layer table, the slab-tiled copies (built here, as the chain's tiled = 1 does)
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t t_attn = up(flow_tiled_bytes((int)qkv_cols, o.hidden, ncta)), t_proj = up(flow_tiled_bytes(o.hidden, o.hidden, ncta));
  const size_t t_fc = up(flow_tiled_bytes(o.n_inner, o.hidden, ncta)), t_fc2 = up(flow_tiled_bytes(o.hidden, o.n_inner, ncta));
  const size_t t_lm = up(flow_tiled_bytes(o.vocab, o.hidden, ncta));
  const size_t head = 2 * kOpState + up(sizeof(MegaLayer) * o.n_layer);
  static_assert(sizeof(GenState) <= kOpState && sizeof(GenParamsDev) <= kOpState, "the state fits a scratch slot");
  uint8_t* buf = nullptr;
  r = cudaMalloc(reinterpret_cast<void**>(&buf), head + o.n_layer * (t_attn + t_proj + t_fc + t_fc2) + t_lm);
  if (r != cudaSuccess) return op_fail("decode_flow alloc", r);
  GenState* d_gs = reinterpret_cast<GenState*>(buf);
  GenParamsDev* d_p = reinterpret_cast<GenParamsDev*>(buf + kOpState);
  MegaLayer* d_layers = reinterpret_cast<MegaLayer*>(buf + 2 * kOpState);
  uint8_t* q = buf + head;
  std::vector<MegaLayer> ml(o.n_layer);
  auto tile = [&](const void* W, const void* bias, int N, int K, size_t bytes) {
    uint8_t* t = q;
    q += bytes;
    launch_flow_repack((const bf16*)W, (const bf16*)bias, t, N, K, ncta, st);
    return reinterpret_cast<const bf16*>(t);
  };
  for (int l = 0; l < o.n_layer; ++l) {
    const sv_op_chain_layer& s = o.layers[l];
    auto w = [](const void* v) { return static_cast<const bf16*>(v); };
    ml[l] = MegaLayer{w(s.ln1_w), w(s.ln1_b), w(s.attn_w), w(s.attn_b), w(s.proj_w), w(s.proj_b), w(s.ln2_w), w(s.ln2_b),
                      w(s.fc_w), w(s.fc_b), w(s.fc2_w), w(s.fc2_b), (bf16*)o.kcache + o.layer_stride * l,
                      (bf16*)o.vtcache + o.layer_stride * l, nullptr, nullptr, nullptr, nullptr};
    ml[l].attn_t = tile(s.attn_w, s.attn_b, (int)qkv_cols, o.hidden, t_attn);
    ml[l].proj_t = tile(s.proj_w, s.proj_b, o.hidden, o.hidden, t_proj);
    ml[l].fc_t = tile(s.fc_w, s.fc_b, o.n_inner, o.hidden, t_fc);
    ml[l].fc2_t = tile(s.fc2_w, s.fc2_b, o.hidden, o.n_inner, t_fc2);
  }
  const bf16* lm_t = tile(o.lm_head, nullptr, o.vocab, o.hidden, t_lm);
  GenState gs{};
  if (o.do_select) {
    gs.step = o.counters_host[0]; gs.cur_len = o.counters_host[1]; gs.done = o.counters_host[2];
    for (int b = 0; b < B; ++b) gs.unfinished[b] = o.unfinished_host[b];
  }
  const GenParamsDev hp = gen_params_dev(&p, p.stop_row0_only, o.do_select ? o.out_stride : 1);
  r = cudaGetLastError();
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_gs, &gs, sizeof(gs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_p, &hp, sizeof(hp), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_layers, ml.data(), sizeof(MegaLayer) * o.n_layer, cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) {
    // every field flow_launch_desc sets for the engine, from the caller's tensors (the size assert above it keeps the two in
    // step), then the per-launch fields; the launch itself is the engine's launch_decode_flow
    FlowLaunch m{};
    m.layers_dev = d_layers; m.n_layer = o.n_layer; m.B = B; m.H = o.hidden; m.I = o.n_inner; m.n_head = o.n_head; m.n_kv = o.n_kv;
    m.qkv_cols = (int)qkv_cols; m.vocab = o.vocab; m.tcap = o.tcap; m.n_positions = o.n_positions; m.ln_eps = o.ln_eps;
    m.wte = (const bf16*)o.wte; m.wpe = (const bf16*)o.wpe; m.lnf_w = (const bf16*)o.lnf_w; m.lnf_b = (const bf16*)o.lnf_b;
    m.lm_head = (const bf16*)o.lm_head; m.lm_head_t = lm_t; m.x_plain = (bf16*)o.x_plain; m.logits = (bf16*)o.logits;
    m.xa = (uint32_t*)o.xa; m.xb = (uint32_t*)o.xb; m.qkv = (uint32_t*)o.qkv; m.att = (uint32_t*)o.att; m.hb = (uint32_t*)o.hb;
    m.part = (unsigned long long*)o.part; m.amax = (unsigned long long*)o.amax;
    m.state = d_gs; m.params = d_p; m.seen = (uint8_t*)o.seen; m.next_ids = o.next_ids; m.out_ids = o.out_ids;
    m.nsteps = o.nsteps; m.step0 = o.step0; m.cur_len0 = o.cur_len0; m.first_plain = o.first_plain; m.do_select = o.do_select;
    m.l2_ahead = o.l2_ahead; m.dbg = nullptr; m.realloc = o.realloc != 0;
    r = launch_decode_flow(m, st);
  }
  if (r == cudaSuccess) r = cudaMemcpyAsync(&gs, d_gs, sizeof(gs), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  if (r != cudaSuccess) return op_fail("decode_flow", r);
  if (o.do_select) {
    o.counters_host[0] = gs.step; o.counters_host[1] = gs.cur_len; o.counters_host[2] = gs.done;
    for (int b = 0; b < B; ++b) o.unfinished_host[b] = gs.unfinished[b];
  }
  o.ncta_used = ncta;
  o.realloc_used = o.realloc;
  return SV_OK;
}

// ---- the token-selection kernels one at a time ---------------------------------------------------------------------
int sv_op_select(const sv_op_select_args* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad select arguments: null descriptor");
  const sv_op_select_args& o = *args;
  const sv_gen_params& p = o.params;
  const bool sampling = o.impl == SV_SELECT_SAMPLE || p.do_sample != 0, fused = o.impl == SV_SELECT_FUSED;
  const char* bad = nullptr;
  if (o.impl != SV_SELECT_GREEDY && o.impl != SV_SELECT_SAMPLE && o.impl != SV_SELECT_FUSED) bad = "unknown impl";
  else if (o.per_row != 0 && o.per_row != 1) bad = "per_row is 0 or 1";
  else if (!o.logits || !o.seen || !o.out_ids || !o.next_ids) bad = "logits, seen, out_ids and next_ids are required";
  else if (o.B < 1 || o.B > kSessionRows) bad = "B not in [1, 16]";
  else if (o.vocab < 1) bad = "vocab < 1";
  else if (o.nsteps < 1 || o.out_stride < 1) bad = "nsteps and out_stride must be >= 1";
  else if (o.advance_len != 0 && o.advance_len != 1) bad = "advance_len is 0 or 1";
  else if (sampling && !(p.temperature > 0.f)) bad = "temperature must be > 0";
  else if (sampling && !(p.top_p > 0.f && p.top_p <= 1.f)) bad = "top_p not in (0, 1]";
  else if ((bad = gen_params_error(p))) {}
  else if (!o.per_row) {
    if (!o.counters_host || !o.unfinished_host) bad = "per_row = 0 needs counters_host and unfinished_host";
    else if (o.counters_host[0] < 0 || o.counters_host[1] < 0) bad = "step and cur_len must be >= 0";
    else if (o.counters_host[0] + o.nsteps > o.out_stride) bad = "step + nsteps > out_stride";
  } else {
    if (!o.row_len_host || !o.row_step_host || !o.row_active_host || !o.row_max_new_host || !o.row_seed_host || !o.event_host)
      bad = "per_row = 1 needs the row_*_host arrays and event_host";
    for (int b = 0; !bad && b < o.B; ++b) {
      if (o.row_len_host[b] < 0 || o.row_step_host[b] < 0) bad = "row_len and row_step must be >= 0";
      else if (o.row_step_host[b] + o.nsteps > o.out_stride) bad = "row_step + nsteps > out_stride";
    }
  }
  if (!bad && fused) {
    if (!o.wte || !o.x) bad = "fused needs wte and x";
    else if (o.h < 8 || o.h % 8) bad = "h % 8 != 0";
    else if (o.n_positions < 1) bad = "n_positions < 1";
    else if (!aligned16(o.wte) || !aligned16(o.wpe) || !aligned16(o.x)) bad = "wte, wpe and x must be 16-byte aligned";
    else if ((o.amax_val != nullptr) != (o.amax_idx != nullptr)) bad = "amax_val and amax_idx go together";
    else if (o.amax_val && o.nsteps > 1) bad = "the argmax partials describe one step: nsteps > 1 needs amax_val = NULL";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad select arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const GenParamsDev hp = gen_params_dev(&p, p.stop_row0_only, o.out_stride);
  GenState gs{};
  RowState rs{};
  if (o.per_row) {
    for (int b = 0; b < o.B; ++b) {
      rs.row_len[b] = o.row_len_host[b]; rs.row_step[b] = o.row_step_host[b]; rs.row_active[b] = o.row_active_host[b];
      rs.row_max_new[b] = o.row_max_new_host[b]; rs.row_seed[b] = o.row_seed_host[b];
    }
    rs.event = o.event_host[0];
  } else {
    gs.step = o.counters_host[0]; gs.cur_len = o.counters_host[1]; gs.done = o.counters_host[2];
    for (int b = 0; b < o.B; ++b) gs.unfinished[b] = o.unfinished_host[b];
  }
  const size_t probs_bytes = o.impl == SV_SELECT_SAMPLE ? (size_t)o.B * o.vocab * sizeof(float) : 0;
  char* buf = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&buf), 3 * kOpState + probs_bytes);
  if (r != cudaSuccess) return op_fail("select alloc", r);
  GenState* d_gs = reinterpret_cast<GenState*>(buf);
  RowState* d_rs = reinterpret_cast<RowState*>(buf + kOpState);
  GenParamsDev* d_p = reinterpret_cast<GenParamsDev*>(buf + 2 * kOpState);
  float* probs = reinterpret_cast<float*>(buf + 3 * kOpState);
  static_assert(sizeof(GenParamsDev) <= kOpState, "the parameters fit a scratch slot");
  r = cudaMemcpyAsync(d_gs, &gs, sizeof(gs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_rs, &rs, sizeof(rs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_p, &hp, sizeof(hp), cudaMemcpyHostToDevice, st);
  RowState* rows = o.per_row ? d_rs : nullptr;
  const bf16* lg = (const bf16*)o.logits;
  uint8_t* seen = (uint8_t*)o.seen;
  for (int s = 0; r == cudaSuccess && s < o.nsteps; ++s) {
    if (fused) {
      launch_select_fused(lg, o.vocab, o.B, o.amax_val, o.amax_idx, gemv_ring_ntiles(o.vocab), 8 * ring_row_groups(o.B), d_gs,
                          d_p, seen, o.next_ids, o.out_ids, o.advance_len, (const bf16*)o.wte, (const bf16*)o.wpe, (bf16*)o.x,
                          o.h, o.n_positions, false, st, rows, o.row_mask);
    } else {
      if (o.impl == SV_SELECT_SAMPLE)
        launch_select_sample(lg, o.vocab, o.B, d_gs, d_p, seen, o.next_ids, o.out_ids, probs, st, rows, o.row_mask, o.advance_len);
      else
        launch_select_greedy(lg, o.vocab, o.B, d_gs, d_p, seen, o.next_ids, o.out_ids, st, rows, o.row_mask, o.advance_len);
      if (!o.per_row) launch_gen_finalize(d_gs, d_p, o.B, o.advance_len, st);
    }
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaMemcpyAsync(&gs, d_gs, sizeof(gs), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(&rs, d_rs, sizeof(rs), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  if (r != cudaSuccess) return op_fail("select", r);
  if (o.per_row) {
    for (int b = 0; b < o.B; ++b) {
      o.row_len_host[b] = rs.row_len[b]; o.row_step_host[b] = rs.row_step[b]; o.row_active_host[b] = rs.row_active[b];
      o.row_max_new_host[b] = rs.row_max_new[b]; o.row_seed_host[b] = rs.row_seed[b];
    }
    o.event_host[0] = rs.event;
  } else {
    o.counters_host[0] = gs.step; o.counters_host[1] = gs.cur_len; o.counters_host[2] = gs.done;
    for (int b = 0; b < o.B; ++b) o.unfinished_host[b] = gs.unfinished[b];
  }
  return SV_OK;
}

// The selection kernels of a speculative verify step, launched as generate_impl launches them.
static_assert(sizeof(sv_spec_state) == sizeof(svspec::State) && offsetof(sv_spec_state, tok) == offsetof(svspec::State, tok) &&
              offsetof(sv_spec_state, ncols) == offsetof(svspec::State, ncols) &&
              offsetof(sv_spec_state, accepted) == offsetof(svspec::State, accepted),
              "sv_spec_state mirrors svspec::State");
int sv_op_spec_select(const sv_op_spec_args* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad spec_select arguments: null descriptor");
  const sv_op_spec_args& o = *args;
  const sv_gen_params& p = o.params;
  const char* bad = nullptr;
  if (o.impl != SV_SPEC_GREEDY && o.impl != SV_SPEC_SAMPLE && o.impl != SV_SPEC_ACCEPT) bad = "unknown impl";
  else if (!o.seen || !o.out_ids || !o.next_ids || !o.gen_host || !o.spec_host) bad = "seen, out_ids, next_ids, gen_host and spec_host are required";
  else if (o.impl != SV_SPEC_ACCEPT && !o.logits) bad = "GREEDY and SAMPLE need logits";
  else if (o.vocab < 1) bad = "vocab < 1";
  else if (o.impl == SV_SPEC_SAMPLE && !(p.temperature > 0.f)) bad = "temperature must be > 0";
  else if (o.impl == SV_SPEC_SAMPLE && !(p.top_p > 0.f && p.top_p <= 1.f)) bad = "top_p not in (0, 1]";
  else if ((bad = gen_params_error(p))) {}
  else if (p.max_new_tokens < 1 || p.max_new_tokens > o.out_stride) bad = "max_new_tokens not in [1, out_stride]";
  else if (o.gen_host[0] < 1 || o.gen_host[0] >= o.out_stride) bad = "step (the history's length) not in [1, out_stride)";
  else if (o.gen_host[1] < 0 || o.gen_host[1] >= o.n_positions) bad = "cur_len not in [0, n_positions - 1]";
  else if (!o.wte || !o.x) bad = "wte and x are required";
  else if (o.h < 8 || o.h % 8) bad = "h % 8 != 0";
  else if (o.n_positions < 1) bad = "n_positions < 1";
  else if (!aligned16(o.wte) || !aligned16(o.wpe) || !aligned16(o.x)) bad = "wte, wpe and x must be 16-byte aligned";
  else if ((o.amax_val != nullptr) != (o.amax_idx != nullptr)) bad = "amax_val and amax_idx go together";
  else if (o.amax_val && o.impl != SV_SPEC_GREEDY) bad = "the argmax partials are GREEDY's";
  if (!bad) {
    const sv_spec_state& q = *o.spec_host;
    if (q.ncols < 1 || q.ncols > svspec::kMaxCols) bad = "ncols not in [1, 16]";
    else if (q.n_live < 0 || q.n_live > q.ncols) bad = "n_live not in [0, ncols]";
    else if (q.k != q.ncols - 1) bad = "k != ncols - 1";
    else if (q.max_ngram < 1) bad = "max_ngram < 1";
    for (int c = 0; !bad && c < q.ncols; ++c)
      if (q.row[c] != 0 || q.pos[c] < 0 || q.pos[c] >= o.n_positions) bad = "a column is not in row 0 at a position in [0, n_positions - 1]";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad spec_select arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const GenParamsDev hp = gen_params_dev(&p, p.stop_row0_only, o.out_stride);
  GenState gs{};
  gs.step = o.gen_host[0]; gs.cur_len = o.gen_host[1]; gs.done = o.gen_host[2]; gs.unfinished[0] = o.gen_host[3];
  svspec::State sp;
  memcpy(&sp, o.spec_host, sizeof(sp));
  const int ncols = sp.ncols;
  const size_t probs_bytes = o.impl == SV_SPEC_SAMPLE ? (size_t)ncols * o.vocab * sizeof(float) : 0;
  char* buf = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&buf), 3 * kOpState + probs_bytes);
  if (r != cudaSuccess) return op_fail("spec_select alloc", r);
  GenState* d_gs = reinterpret_cast<GenState*>(buf);
  svspec::State* d_sp = reinterpret_cast<svspec::State*>(buf + kOpState);
  GenParamsDev* d_p = reinterpret_cast<GenParamsDev*>(buf + 2 * kOpState);
  float* probs = reinterpret_cast<float*>(buf + 3 * kOpState);
  static_assert(sizeof(svspec::State) <= kOpState, "the speculative state fits a scratch slot");
  r = cudaMemcpyAsync(d_gs, &gs, sizeof(gs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_sp, &sp, sizeof(sp), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_p, &hp, sizeof(hp), cudaMemcpyHostToDevice, st);
  const bf16* lg = (const bf16*)o.logits;
  uint8_t* seen = (uint8_t*)o.seen;
  if (r == cudaSuccess) {
    if (o.impl == SV_SPEC_GREEDY) {
      launch_select_fused_spec(lg, o.vocab, o.amax_val, o.amax_idx, gemv_ring_ntiles(o.vocab), 8 * ring_row_groups(ncols), d_gs,
                               d_p, seen, o.next_ids, o.out_ids, (const bf16*)o.wte, (const bf16*)o.wpe, (bf16*)o.x, o.h,
                               o.n_positions, d_sp, false, st);
    } else {
      if (o.impl == SV_SPEC_SAMPLE) launch_select_sample_spec(lg, o.vocab, ncols, d_gs, d_p, seen, probs, d_sp, st);
      launch_spec_accept(d_gs, d_p, seen, o.next_ids, o.out_ids, o.vocab, (const bf16*)o.wte, (const bf16*)o.wpe, (bf16*)o.x,
                         o.h, o.n_positions, d_sp, false, st);
    }
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaMemcpyAsync(&gs, d_gs, sizeof(gs), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(&sp, d_sp, sizeof(sp), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  if (r != cudaSuccess) return op_fail("spec_select", r);
  o.gen_host[0] = gs.step; o.gen_host[1] = gs.cur_len; o.gen_host[2] = gs.done; o.gen_host[3] = gs.unfinished[0];
  memcpy(o.spec_host, &sp, sizeof(sp));
  return SV_OK;
}

// The kernels of a speculative session's verify step, launched as sv_session_run / sv_session_admit launch them.
int sv_op_spec_session_select(const sv_op_spec_session_args* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad spec_session_select arguments: null descriptor");
  const sv_op_spec_session_args& o = *args;
  const sv_gen_params& p = o.params;
  const char* bad = nullptr;
  if (o.impl != SV_SPEC_SESSION_GREEDY && o.impl != SV_SPEC_SESSION_SAMPLE && o.impl != SV_SPEC_SESSION_TAIL) bad = "unknown impl";
  else if (!o.seen || !o.out_ids || !o.next_ids || !o.rows_host || !o.ss_host) bad = "seen, out_ids, next_ids, rows_host and ss_host are required";
  else if (o.impl != SV_SPEC_SESSION_TAIL && !o.logits) bad = "GREEDY and SAMPLE need logits";
  else if (o.vocab < 1) bad = "vocab < 1";
  else if (o.impl == SV_SPEC_SESSION_SAMPLE && !(p.temperature > 0.f)) bad = "temperature must be > 0";
  else if (o.impl == SV_SPEC_SESSION_SAMPLE && !(p.top_p > 0.f && p.top_p <= 1.f)) bad = "top_p not in (0, 1]";
  else if ((bad = gen_params_error(p))) {}
  else if (!o.wte || !o.x) bad = "wte and x are required";
  else if (o.h < 8 || o.h % 8) bad = "h % 8 != 0";
  else if (o.n_positions < 1) bad = "n_positions < 1";
  else if (!aligned16(o.wte) || !aligned16(o.wpe) || !aligned16(o.x)) bad = "wte, wpe and x must be 16-byte aligned";
  else if ((o.amax_val != nullptr) != (o.amax_idx != nullptr)) bad = "amax_val and amax_idx go together";
  else if (o.amax_val && o.impl != SV_SPEC_SESSION_GREEDY) bad = "the argmax partials are GREEDY's";
  if (!bad) {
    const sv_spec_session_state& q = *o.ss_host;
    const sv_session_rows& rw = *o.rows_host;
    const int S = q.ncols;
    if (S < 2 || S > svspec::kMaxCols) bad = "ncols not in [2, 16]";
    else if (q.n_live < 0 || q.n_live > S) bad = "n_live not in [0, ncols]";
    else if (q.k < 1 || q.k > S - 1 || q.max_ngram < 1) bad = "k not in [1, ncols - 1] or max_ngram < 1";
    for (int c = 0; !bad && c < S; ++c)
      if (q.row[c] < 0 || q.row[c] >= S || q.pos[c] < 0 || q.pos[c] >= std::min(o.n_positions, o.tcap) || q.off[c] < 0 || q.off[c] > c)
        bad = "a column's row, position or offset is out of range";
    for (int r = 0; !bad && r < S; ++r)
      if (rw.row_active[r] && (rw.row_step[r] < 1 || rw.row_step[r] >= rw.row_max_new[r] || rw.row_max_new[r] > o.out_stride ||
                               rw.row_len[r] < 0 || rw.row_len[r] + rw.row_max_new[r] > o.tcap || rw.row_len[r] + rw.row_max_new[r] > o.n_positions))
        bad = "a live row's step, cap or position is out of range (1 <= row_step < row_max_new <= out_stride, row_len + row_max_new <= min(tcap, n_positions))";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad spec_session_select arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const GenParamsDev hp = gen_params_dev(&p, 0, o.out_stride);
  const int S = o.ss_host->ncols;
  const size_t probs_bytes = o.impl == SV_SPEC_SESSION_SAMPLE ? (size_t)S * o.vocab * sizeof(float) : 0;
  char* buf = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&buf), 3 * kOpState + probs_bytes);
  if (r != cudaSuccess) return op_fail("spec_session_select alloc", r);
  static_assert(sizeof(svspec::SessionState) <= kOpState && sizeof(RowState) <= kOpState, "the session states fit scratch slots");
  RowState* d_rows = reinterpret_cast<RowState*>(buf);
  svspec::SessionState* d_ss = reinterpret_cast<svspec::SessionState*>(buf + kOpState);
  GenParamsDev* d_p = reinterpret_cast<GenParamsDev*>(buf + 2 * kOpState);
  float* probs = reinterpret_cast<float*>(buf + 3 * kOpState);
  r = cudaMemcpyAsync(d_rows, o.rows_host, sizeof(RowState), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_ss, o.ss_host, sizeof(svspec::SessionState), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_p, &hp, sizeof(hp), cudaMemcpyHostToDevice, st);
  const bf16* lg = (const bf16*)o.logits;
  uint8_t* seen = (uint8_t*)o.seen;
  if (r == cudaSuccess) {
    if (o.impl == SV_SPEC_SESSION_GREEDY) {
      launch_spec_session_select_fused(lg, o.vocab, o.amax_val, o.amax_idx, gemv_ring_ntiles(o.vocab), 8 * ring_row_groups(S), d_rows,
                                       d_p, seen, o.next_ids, o.out_ids, (const bf16*)o.wte, (const bf16*)o.wpe, (bf16*)o.x, o.h,
                                       o.n_positions, o.tcap, d_ss, false, st);
    } else {
      if (o.impl == SV_SPEC_SESSION_SAMPLE) launch_spec_session_select_sample(lg, o.vocab, S, d_rows, d_p, seen, probs, d_ss, st);
      launch_spec_session_tail(o.impl == SV_SPEC_SESSION_SAMPLE || o.accept != 0, d_rows, d_p, seen, o.next_ids, o.out_ids,
                               o.vocab, (const bf16*)o.wte, (const bf16*)o.wpe, (bf16*)o.x, o.h, o.n_positions, o.tcap, d_ss,
                               false, st);
    }
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaMemcpyAsync(o.rows_host, d_rows, sizeof(RowState), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(o.ss_host, d_ss, sizeof(svspec::SessionState), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  if (r != cudaSuccess) return op_fail("spec_session_select", r);
  return SV_OK;
}

int sv_op_beam_candidates(const void* logits, int32_t vocab, const sv_beam_params* p, int32_t batch, int32_t cur_len,
                          const float* running_scores_host, const int32_t* run_seq, int32_t seq_stride, float* cand_key,
                          float* cand_val, int32_t* cand_tok, void* stream) {
  const char* bad = nullptr;
  if (!logits || !p || !running_scores_host || !run_seq || !cand_key || !cand_val || !cand_tok) bad = "null pointer";
  else if (sv_beam_params_check_rows(p, batch, svbeam::kMaxRows) != SV_OK)
    bad = "beam parameters (num_beams in [2, 8], batch * num_beams <= 16, max_new_tokens >= 1, n_stop_ids in [0, 8], "
          "early_stopping in {0, 1, 2}, temperature > 0, repetition_penalty > 0)";
  else if (p->do_sample && !(p->top_p > 0.f && p->top_p <= 1.f)) bad = "top_p not in (0, 1]";
  else if (vocab < 1) bad = "vocab < 1";
  else if (seq_stride < 1 || cur_len < 0 || cur_len > seq_stride) bad = "cur_len not in [0, seq_stride]";
  cudaError_t r = bad ? cudaSuccess : beam_init(vocab);      // the last check: it sizes the kernel's shared memory
  if (r == cudaErrorInvalidValue) bad = "a logits row of this vocab does not fit the SM's shared memory";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad beam_candidates arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int R = batch * p->num_beams;
  const svbeam::Params hp = beam_params_dev(p, batch, vocab, seq_stride);
  svbeam::State hs;
  memset(&hs, 0, sizeof(hs));
  svbeam::init_state(hp, hs, 0);
  hs.cur_len = cur_len;
  for (int r = 0; r < R; ++r) hs.running_scores[r] = running_scores_host[r];
  if (r != cudaSuccess) { cudaGetLastError(); return op_fail("beam_candidates setup", r); }
  char* buf = nullptr;
  r = cudaMalloc(reinterpret_cast<void**>(&buf), sizeof(svbeam::Params) + sizeof(svbeam::State));
  if (r != cudaSuccess) return op_fail("beam_candidates alloc", r);
  svbeam::Params* d_p = reinterpret_cast<svbeam::Params*>(buf);
  svbeam::State* d_s = reinterpret_cast<svbeam::State*>(buf + sizeof(svbeam::Params));
  static_assert(sizeof(svbeam::Params) % 8 == 0, "State follows Params at its alignment");
  r = cudaMemcpyAsync(d_p, &hp, sizeof(hp), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_s, &hs, sizeof(hs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) {
    launch_beam_candidates((const bf16*)logits, vocab, R, d_p, d_s, run_seq, cand_key, cand_val, cand_tok, st);
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  return r == cudaSuccess ? SV_OK : op_fail("beam_candidates", r);
}

// The bookkeeping and KV-movement kernels of the beam loop, launched as sv_beam_search / sv_reorder_cache / sv_session_admit
// launch them.
static_assert(sizeof(sv_beam_state) == sizeof(svbeam::State) &&
              offsetof(sv_beam_state, running_scores) == offsetof(svbeam::State, running_scores) &&
              offsetof(sv_beam_state, beam_scores) == offsetof(svbeam::State, beam_scores) &&
              offsetof(sv_beam_state, is_finished) == offsetof(svbeam::State, is_finished) &&
              offsetof(sv_beam_state, fin_len) == offsetof(svbeam::State, fin_len) &&
              offsetof(sv_beam_state, unsatisfied) == offsetof(svbeam::State, unsatisfied) &&
              offsetof(sv_beam_state, div) == offsetof(svbeam::State, div),
              "sv_beam_state mirrors svbeam::State");
static_assert(sizeof(sv_beam_plan) == sizeof(svbeam::Plan) && offsetof(sv_beam_plan, run_tok) == offsetof(svbeam::Plan, run_tok) &&
              offsetof(sv_beam_plan, fin_old) == offsetof(svbeam::Plan, fin_old) &&
              offsetof(sv_beam_plan, fin_parent) == offsetof(svbeam::Plan, fin_parent) &&
              offsetof(sv_beam_plan, fin_tok) == offsetof(svbeam::Plan, fin_tok) &&
              offsetof(sv_beam_plan, copy_src) == offsetof(svbeam::Plan, copy_src) &&
              offsetof(sv_beam_plan, copy_lo) == offsetof(svbeam::Plan, copy_lo) &&
              offsetof(sv_beam_plan, copy_hi) == offsetof(svbeam::Plan, copy_hi) &&
              offsetof(sv_beam_plan, cont) == offsetof(svbeam::Plan, cont) &&
              offsetof(sv_beam_plan, old_len) == offsetof(svbeam::Plan, old_len),
              "sv_beam_plan mirrors svbeam::Plan");

int sv_op_beam_step(const sv_op_beam_step_args* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad beam_step arguments: null descriptor");
  const sv_op_beam_step_args& o = *args;
  const char* bad = nullptr;
  if (!o.params || !o.state_host || !o.cand_key || !o.cand_val || !o.cand_tok || !o.run_seq || !o.fin_seq || !o.gen_host ||
      !o.wte || !o.x || !o.next_ids || !o.plan_host)
    bad = "null pointer (only wpe may be NULL)";
  else if (sv_beam_params_check_rows(o.params, o.batch, svbeam::kMaxRows) != SV_OK)
    bad = "beam parameters (num_beams in [2, 8], batch * num_beams <= 16, max_new_tokens >= 1, n_stop_ids in [0, 8], "
          "early_stopping in {0, 1, 2}, temperature > 0, repetition_penalty > 0)";
  else if (o.vocab < 1 || o.seq_stride < 1) bad = "vocab and seq_stride must be >= 1";
  else if (o.advance != 0 && o.advance != 1) bad = "advance is 0 or 1";
  else if (o.h < 8 || o.h % 8) bad = "h % 8 != 0";
  else if (o.n_positions < 1) bad = "n_positions < 1";
  else if (!aligned16(o.wte) || !aligned16(o.wpe) || !aligned16(o.x)) bad = "wte, wpe and x must be 16-byte aligned";
  else if (o.gen_host[0] < 0) bad = "cur_len < 0";
  else {
    const sv_beam_state& s = *o.state_host;
    // the sequence moves write positions [0, cur_len] of every row; the row-0 stop check reads the n_stop - 1 before it
    if (s.cur_len < 0 || s.cur_len >= o.seq_stride) bad = "state cur_len not in [0, seq_stride)";
    else if (s.parity != 0 && s.parity != 1) bad = "state parity is 0 or 1";
    for (int r = 0; !bad && r < o.batch * o.params->num_beams; ++r)
      if (s.fin_len[r] < 0 || s.fin_len[r] > o.seq_stride) bad = "a state fin_len is not in [0, seq_stride]";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad beam_step arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const svbeam::Params hp = beam_params_dev(o.params, o.batch, o.vocab, o.seq_stride);
  GenState gs{};
  gs.cur_len = o.gen_host[0];
  gs.done = o.gen_host[1];
  char* buf = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&buf), 4 * kOpState + sizeof(svbeam::State));
  if (r != cudaSuccess) return op_fail("beam_step alloc", r);
  static_assert(sizeof(svbeam::Params) <= kOpState && sizeof(svbeam::Plan) <= kOpState, "params and plan fit a scratch slot");
  svbeam::Params* d_p = reinterpret_cast<svbeam::Params*>(buf);
  GenState* d_gs = reinterpret_cast<GenState*>(buf + kOpState);
  svbeam::Plan* d_plan = reinterpret_cast<svbeam::Plan*>(buf + 2 * kOpState);
  svbeam::State* d_s = reinterpret_cast<svbeam::State*>(buf + 4 * kOpState);
  r = cudaMemcpyAsync(d_p, &hp, sizeof(hp), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_gs, &gs, sizeof(gs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_plan, o.plan_host, sizeof(svbeam::Plan), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(d_s, o.state_host, sizeof(svbeam::State), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) {
    launch_beam_step(d_p, d_s, d_plan, o.cand_key, o.cand_val, o.cand_tok, o.run_seq, o.fin_seq, d_gs, o.advance,
                     (const bf16*)o.wte, (const bf16*)o.wpe, (bf16*)o.x, o.h, o.n_positions, o.next_ids, st);
    r = cudaGetLastError();
  }
  svbeam::State hs;
  svbeam::Plan hplan;
  if (r == cudaSuccess) r = cudaMemcpyAsync(&gs, d_gs, sizeof(gs), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(&hs, d_s, sizeof(hs), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaMemcpyAsync(&hplan, d_plan, sizeof(hplan), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  if (r != cudaSuccess) return op_fail("beam_step", r);
  memcpy(o.state_host, &hs, sizeof(hs));
  memcpy(o.plan_host, &hplan, sizeof(hplan));
  o.gen_host[0] = gs.cur_len;
  o.gen_host[1] = gs.done;
  return SV_OK;
}

int sv_op_beam_kv_copy(void* kcache, void* vtcache, int64_t layer_stride, int32_t n_layer, int32_t rows, int32_t n_kv,
                       int32_t tcap, const sv_beam_plan* plan_host, void* stream) {
  const int D = 128;
  const char* bad = nullptr;
  if (!kcache || !vtcache || !plan_host) bad = "null pointer";
  else if (n_layer < 1 || rows < 1 || rows > svbeam::kMaxRows || n_kv < 1) bad = "n_layer, n_kv >= 1 and rows in [1, 16]";
  else if (tcap < 32 || tcap % 32) bad = "tcap % 32 != 0";
  else if (layer_stride < (int64_t)rows * n_kv * tcap * D || layer_stride % 8) bad = "layer_stride < rows * n_kv * tcap * 128 or % 8 != 0";
  else if (!aligned16(kcache) || !aligned16(vtcache)) bad = "the caches must be 16-byte aligned";
  else if (plan_host->copy_hi >= tcap) bad = "copy_hi >= tcap";
  for (int r = 0; !bad && r < rows; ++r) {
    if (plan_host->copy_src[r] < -1 || plan_host->copy_src[r] >= rows) bad = "a copy_src is not in [-1, rows)";
    else if (plan_host->copy_src[r] >= 0 && plan_host->copy_lo[r] <= plan_host->copy_hi && plan_host->copy_lo[r] < 0)
      bad = "a copy_lo < 0";
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad beam_kv_copy arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t stage = layer_stride * n_layer;          // the staging cache has the caches' layout (as sv_beam_search's)
  char* buf = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&buf), kOpState + 2 * stage * sizeof(bf16));
  if (r != cudaSuccess) return op_fail("beam_kv_copy alloc", r);
  svbeam::Plan* d_plan = reinterpret_cast<svbeam::Plan*>(buf);
  bf16* kstage = reinterpret_cast<bf16*>(buf + kOpState);
  bf16* vstage = kstage + stage;
  r = cudaMemcpyAsync(d_plan, plan_host, sizeof(svbeam::Plan), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) {
    launch_beam_kv_copy((bf16*)kcache, (bf16*)vtcache, kstage, vstage, layer_stride, n_layer, rows, n_kv, tcap, D, d_plan, st);
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(buf);
  return r == cudaSuccess ? SV_OK : op_fail("beam_kv_copy", r);
}

int sv_op_kv_gather(const void* ksrc, const void* vsrc, void* kdst, void* vdst, const int32_t* idx, int32_t rows, int32_t n_kv,
                    int32_t tcap, int32_t len, void* stream) {
  const char* bad = nullptr;
  if (!ksrc || !vsrc || !kdst || !vdst) bad = "null pointer";
  else if (rows < 1 || rows > kSessionRows || n_kv < 1) bad = "rows in [1, 16] and n_kv >= 1";
  else if (tcap < 32 || tcap % 32) bad = "tcap % 32 != 0";
  else if (len < 1 || len > tcap) bad = "len not in [1, tcap]";
  else if (!aligned16(ksrc) || !aligned16(vsrc) || !aligned16(kdst) || !aligned16(vdst)) bad = "the caches must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad kv_gather arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  launch_kv_gather((const bf16*)ksrc, (const bf16*)vsrc, (bf16*)kdst, (bf16*)vdst, idx, rows, n_kv, tcap, 128, len, st);
  cudaError_t r = cudaGetLastError();
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  return r == cudaSuccess ? SV_OK : op_fail("kv_gather", r);
}

int sv_op_session_admit(const sv_op_admit_args* args, void* stream) {
  if (!args) return fail(nullptr, SV_ERR_INVALID, "bad session_admit arguments: null descriptor");
  const sv_op_admit_args& o = *args;
  const char* bad = nullptr;
  if (!o.slot_host || !o.len_host || !o.max_new_host || !o.seed_host || !o.seen || !o.out_ids || !o.row_len_host ||
      !o.row_step_host || !o.row_active_host || !o.row_max_new_host || !o.row_seed_host || !o.event_host)
    bad = "null pointer";
  else if (o.S < 1 || o.S > kSessionRows || o.k < 1 || o.k > o.S) bad = "1 <= k <= S <= 16";
  else if (o.vocab < 1 || o.out_stride < 1) bad = "vocab and out_stride must be >= 1";
  uint32_t used = 0;
  for (int j = 0; !bad && j < o.k; ++j) {
    const int s = o.slot_host[j];
    if (s < 0 || s >= o.S || (used >> s & 1u)) bad = "a slot is outside [0, S) or listed twice";
    else if (o.len_host[j] < 0) bad = "a len is < 0";
    else used |= 1u << s;
  }
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad session_admit arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  RowState rs{};
  for (int b = 0; b < o.S; ++b) {
    rs.row_len[b] = o.row_len_host[b]; rs.row_step[b] = o.row_step_host[b]; rs.row_active[b] = o.row_active_host[b];
    rs.row_max_new[b] = o.row_max_new_host[b]; rs.row_seed[b] = o.row_seed_host[b];
  }
  rs.event = o.event_host[0];
  SessionAdmit adm;
  memset(&adm, 0, sizeof(adm));
  adm.n = o.k;
  for (int j = 0; j < o.k; ++j) {
    adm.slot[j] = o.slot_host[j]; adm.len[j] = o.len_host[j]; adm.max_new[j] = o.max_new_host[j]; adm.seed[j] = o.seed_host[j];
  }
  RowState* d_rs = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&d_rs), kOpState);
  if (r != cudaSuccess) return op_fail("session_admit alloc", r);
  r = cudaMemcpyAsync(d_rs, &rs, sizeof(rs), cudaMemcpyHostToDevice, st);
  if (r == cudaSuccess) {
    launch_session_admit(d_rs, adm, (uint8_t*)o.seen, o.vocab, o.out_ids, o.out_stride, o.pad_id, st);
    r = cudaGetLastError();
  }
  if (r == cudaSuccess) r = cudaMemcpyAsync(&rs, d_rs, sizeof(rs), cudaMemcpyDeviceToHost, st);
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  cudaFree(d_rs);
  if (r != cudaSuccess) return op_fail("session_admit", r);
  for (int b = 0; b < o.S; ++b) {
    o.row_len_host[b] = rs.row_len[b]; o.row_step_host[b] = rs.row_step[b]; o.row_active_host[b] = rs.row_active[b];
    o.row_max_new_host[b] = rs.row_max_new[b]; o.row_seed_host[b] = rs.row_seed[b];
  }
  o.event_host[0] = rs.event;
  return SV_OK;
}

// ---- the image-encoder, adapter and prefill kernels one at a time --------------------------------------------------
static int op_sync(const char* what, cudaStream_t st) {
  cudaError_t r = cudaGetLastError();
  if (r == cudaSuccess) r = cudaStreamSynchronize(st);
  return r == cudaSuccess ? SV_OK : op_fail(what, r);
}

int sv_op_im2col(const void* pixels, void* patches, int32_t batch, int32_t image, int32_t patch, int32_t kpad, void* stream) {
  const char* bad = nullptr;
  if (!pixels || !patches) bad = "null pointer";
  else if (batch < 1 || patch < 1 || image < patch || image % patch) bad = "batch >= 1 and image a multiple of patch";
  else if (kpad < 3 * patch * patch) bad = "kpad < 3 * patch * patch";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad im2col arguments: %s", bad);
  launch_im2col((const bf16*)pixels, (bf16*)patches, batch, image, patch, kpad, (cudaStream_t)stream);
  return op_sync("im2col", (cudaStream_t)stream);
}

int sv_op_vit_assemble(const void* pe, const void* cls, const void* pos, void* x, int32_t batch, int32_t np, int32_t width,
                       void* stream) {
  const char* bad = nullptr;
  if (!pe || !pos || !x) bad = "pe, pos and x are required";
  else if (batch < 1 || np < 1 || width < 1) bad = "batch, np and width must be >= 1";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad vit_assemble arguments: %s", bad);
  launch_vit_assemble((const bf16*)pe, (const bf16*)cls, (const bf16*)pos, (bf16*)x, batch, np, width, (cudaStream_t)stream);
  return op_sync("vit_assemble", (cudaStream_t)stream);
}

int sv_op_adapter_norm(int32_t kind, const void* z, const void* w, const void* b, const void* rmean, const void* rvar,
                       void* y, int32_t batch, int32_t q, int32_t h, float eps, void* stream) {
  const char* bad = nullptr;
  if (kind != SV_ADAPTER_NORM_SLAB && kind != SV_ADAPTER_NORM_TOKENS) bad = "unknown kind";
  else if (!z || !w || !b || !y) bad = "z, w, b and y are required";
  else if (kind == SV_ADAPTER_NORM_TOKENS && (!rmean || !rvar)) bad = "the token BatchNorm needs rmean and rvar";
  else if (batch < 1 || q < 1 || h < 1) bad = "batch, q and h must be >= 1";
  else if (!(eps >= 0.f)) bad = "eps < 0";
  else if (kind == SV_ADAPTER_NORM_SLAB && ((int64_t)q * h) % 8) bad = "q * h % 8 != 0";
  else if (kind == SV_ADAPTER_NORM_SLAB && (!aligned16(z) || !aligned16(w) || !aligned16(b) || !aligned16(y)))
    bad = "z, w, b and y must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad adapter_norm arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  if (kind == SV_ADAPTER_NORM_TOKENS) {
    launch_batchnorm_tokens((const bf16*)z, (const bf16*)w, (const bf16*)b, (const bf16*)rmean, (const bf16*)rvar, (bf16*)y,
                            batch, q, h, eps, st);
    return op_sync("adapter_norm", st);
  }
  float* partial = nullptr;
  cudaError_t r = cudaMalloc(reinterpret_cast<void**>(&partial), (size_t)batch * 64 * 2 * sizeof(float));
  if (r != cudaSuccess) return op_fail("adapter_norm alloc", r);
  launch_slab_layernorm((const bf16*)z, (const bf16*)w, (const bf16*)b, (bf16*)y, partial, batch, (int64_t)q * h, eps, st);
  const int rc = op_sync("adapter_norm", st);
  cudaFree(partial);
  return rc;
}

int sv_op_embed_prefix(const void* visual, const int32_t* ids, const void* wte, const void* wpe, void* x, int32_t batch,
                       int32_t q, int32_t p, int32_t h, int32_t vocab, int32_t pos0, int32_t id_stride, void* stream) {
  const char* bad = nullptr;
  if (!wte || !x) bad = "wte and x are required";
  else if ((q > 0 && !visual) || (p > 0 && !ids)) bad = "q > 0 needs visual, p > 0 needs ids";
  else if (batch < 1 || q < 0 || p < 0 || q + p < 1) bad = "batch >= 1, q, p >= 0 and q + p >= 1";
  else if (h < 8 || h % 8) bad = "h % 8 != 0";
  else if (vocab < 1 || pos0 < 0 || id_stride < p) bad = "vocab >= 1, pos0 >= 0 and id_stride >= p";
  else if (!aligned16(visual) || !aligned16(wte) || !aligned16(wpe) || !aligned16(x))
    bad = "visual, wte, wpe and x must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad embed_prefix arguments: %s", bad);
  launch_embed_prefix((const bf16*)visual, ids, (const bf16*)wte, (const bf16*)wpe, (bf16*)x, batch, q, p, h, vocab, pos0,
                      id_stride, (cudaStream_t)stream);
  return op_sync("embed_prefix", (cudaStream_t)stream);
}

int sv_op_lm_logits(const void* x, const void* w, void* y, int32_t M, int32_t N, int32_t K, void* stream) {
  const char* bad = nullptr;
  if (!x || !w || !y) bad = "null pointer";
  else if (M < 1 || N < 1 || K < 64 || K % 64) bad = "M, N >= 1 and K % 64 == 0";
  else if (!aligned16(x) || !aligned16(w)) bad = "x and w must be 16-byte aligned";
  if (bad) return fail(nullptr, SV_ERR_INVALID, "bad lm_logits arguments: %s", bad);
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t r = launch_lm_logits((const bf16*)x, (const bf16*)w, (bf16*)y, M, N, K, st);
  if (r != cudaSuccess) return op_fail("lm_logits", r);
  return op_sync("lm_logits", st);
}

}  // extern "C"

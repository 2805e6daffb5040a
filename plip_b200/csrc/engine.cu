// plip_b200 — engine: packed weights, workspace, tower orchestration, C ABI (include/plip_b200.h).
//
// The forward pass of one micro-batch is a fixed sequence of stream-ordered kernel launches:
//   vision (TF:modeling_clip.py:667-691, 829-863)
//     im2col(+u8 normalise) -> patch GEMM (+pos emb, scatter past the class row) -> class rows -> pre-LN
//     -> bf16 copy + row statistics
//     12 x [ QKV GEMM (LN1 folded, +bias) -> fused attention -> out GEMM (+bias +residual, emits bf16 copy + stats)
//            fc1 GEMM (LN2 folded, +bias +QuickGELU) -> fc2 GEMM (+bias +residual, emits bf16 copy + stats) ]
//     CLS-row post-LN -> projection GEMM [-> L2 normalise]
//   text (TF:531-589, 793-825): token+pos gather & EOS search -> same 12 layers (causal/padding mask)
//     -> EOS-row final-LN -> projection GEMM [-> L2 normalise]
// Residual stream fp32 (X), GEMM operands bf16 (Xn = bf16(X), AO, QKV, H): cosine >= 1-1e-4 vs the fp32
// reference needs the fp32 residual / LN statistics / softmax (SURVEY.md §7).  No allocation and no host sync
// on this path.
#include "kernels.cuh"

#include <stdlib.h>
#include <string.h>

#include <array>
#include <map>
#include <string>
#include <tuple>
#include <vector>

namespace plip {
const char* get_last_error();

namespace {

struct Spec {
  std::string name;
  int dtype;  // 0 f32, 1 bf16
  int rows, cols, fused;
  uint64_t offset, numel;
};

void add(std::vector<Spec>& v, const std::string& name, int dtype, int rows, int cols, int fused = 0) {
  Spec s;
  s.name = name; s.dtype = dtype; s.rows = rows; s.cols = cols; s.fused = fused;
  s.numel = (uint64_t)rows * cols;
  s.offset = 0;
  v.push_back(s);
}

void add_tower(std::vector<Spec>& v, const std::string& pfx, int D, int FF) {
  for (int l = 0; l < kLayers; ++l) {
    const std::string p = pfx + ".encoder.layers." + std::to_string(l);
    // fused bit 0: q|k|v rows concatenated, q pre-scaled by 0.125; bit 1: LayerNorm folded in
    // (layer_norm1 for q_proj, layer_norm2 for fc1): W' = bf16(gamma o W), bias' = bias + W beta,
    // colsum[n] = sum_k W'[n,k].  layer_norm1/2 themselves never reach the device.
    add(v, p + ".self_attn.q_proj.weight", 1, 3 * D, D, 3);
    add(v, p + ".self_attn.q_proj.bias", 0, 3 * D, 1, 3);
    add(v, p + ".self_attn.q_proj.colsum", 0, 3 * D, 1, 3);
    add(v, p + ".self_attn.out_proj.weight", 1, D, D);
    add(v, p + ".self_attn.out_proj.bias", 0, D, 1);
    add(v, p + ".mlp.fc1.weight", 1, FF, D, 2);
    add(v, p + ".mlp.fc1.bias", 0, FF, 1, 2);
    add(v, p + ".mlp.fc1.colsum", 0, FF, 1, 2);
    add(v, p + ".mlp.fc2.weight", 1, D, FF);
    add(v, p + ".mlp.fc2.bias", 0, D, 1);
  }
}

std::vector<Spec> build_specs() {
  std::vector<Spec> v;
  add(v, "vision_model.embeddings.patch_embedding.weight", 1, kVisDim, kPatchK);
  add(v, "vision_model.embeddings.class_embedding", 0, kVisDim, 1);
  add(v, "vision_model.embeddings.position_embedding.weight", 0, kVisSeq, kVisDim);
  add(v, "vision_model.pre_layrnorm.weight", 0, kVisDim, 1);
  add(v, "vision_model.pre_layrnorm.bias", 0, kVisDim, 1);
  add_tower(v, "vision_model", kVisDim, kVisFF);
  add(v, "vision_model.post_layernorm.weight", 0, kVisDim, 1);
  add(v, "vision_model.post_layernorm.bias", 0, kVisDim, 1);
  add(v, "visual_projection.weight", 1, kProj, kVisDim);
  add(v, "text_model.embeddings.token_embedding.weight", 0, kVocab, kTxtDim);
  add(v, "text_model.embeddings.position_embedding.weight", 0, kTxtSeq, kTxtDim);
  add_tower(v, "text_model", kTxtDim, kTxtFF);
  add(v, "text_model.final_layer_norm.weight", 0, kTxtDim, 1);
  add(v, "text_model.final_layer_norm.bias", 0, kTxtDim, 1);
  add(v, "text_projection.weight", 1, kProj, kTxtDim);
  uint64_t off = 0;
  for (auto& s : v) {
    s.offset = off;
    off += s.numel * (s.dtype == 1 ? 2 : 4);
    off = (off + 255) & ~255ull;
  }
  return v;
}

const std::vector<Spec>& specs() {
  static const std::vector<Spec> v = build_specs();  // C++11: initialised once, thread-safe
  return v;
}

uint64_t blob_bytes() {
  const auto& v = specs();
  const Spec& s = v.back();
  return (s.offset + s.numel * (s.dtype == 1 ? 2 : 4) + 255) & ~255ull;
}

struct LayerW {
  const float *bqkv, *sqkv, *bo, *b1, *s1, *b2;
  const __nv_bfloat16 *wqkv, *wo, *w1, *w2;
};

constexpr int kEosId = 49407;  // TF:configuration_clip.py:63 (eos_token_id)

enum ProfKind { PK_QKV = 0, PK_ATTN, PK_OUT, PK_FC1, PK_FC2, PK_PATCH, PK_IM2COL, PK_LN, PK_ROWSTATS, PK_EMBED, PK_PROJ,
                PK_MISC, PK_ATTN_LONG, PK_ATTN_PROBS, PK_COUNT };
const char* const kProfNames[PK_COUNT] = {"gemm[ln1+qkv]", "attention", "gemm[out_proj+resid]", "gemm[ln2+fc1+gelu]",
                                          "gemm[fc2+resid]", "gemm[patch_embed]", "im2col", "layernorm",
                                          "rowstats_cast", "text_embed", "gemm[projection]", "misc", "attention[long]",
                                          "attention[probs]"};

size_t pixel_bytes(int fmt, int height = kImage, int width = kImage) {
  const size_t px = (size_t)3 * height * width;
  return fmt == PLIP_PIX_F32_NCHW ? px * 4 : (fmt == PLIP_PIX_BF16_NCHW ? px * 2 : px);
}

// Input geometry of the vision tower: H x W pixels -> gh x gw patches (the H % 32 / W % 32 remainder is ignored, as by
// the stride-32 conv), S = gh * gw + 1 tokens.  224 x 224 (7 x 7, S = 50) uses the stored position table; any other
// grid an interpolated one (TF:modeling_clip.py:161-218, interpolate_pos_encoding).
struct VisGeom {
  int H = kImage, W = kImage, gh = kGrid, gw = kGrid, S = kVisSeq;
};

VisGeom vis_geom(int height, int width) {
  VisGeom g;
  g.H = height; g.W = width; g.gh = height / kPatch; g.gw = width / kPatch; g.S = g.gh * g.gw + 1;
  return g;
}

// Pixels of a vision pass: mb tiles at `pixels` in `fmt`, or, when win.region is set, mb 224 x 224 windows of a uint8
// RGB region (plip_encode_windows; win.origins points at the pass's first origin).
struct VisInput {
  const void* pixels;
  int fmt;
  WindowSrc win;
};

VisInput tiles(const void* pixels, int fmt) { return VisInput{pixels, fmt, WindowSrc{nullptr, 0, nullptr}}; }

// The workspace holds kVisSeq * max_mb vision token rows (and max_mb pooled rows): images per pass at S tokens each.
int64_t images_per_pass(int max_mb, int S) {
  const int64_t n = (int64_t)kVisSeq * max_mb / S;
  return n < max_mb ? n : max_mb;
}

// Everything a captured launch sequence bakes in (the engine's buffers aside).  Unused fields are 0.
struct GraphKey {
  int tower;  // 0 vision, 1 text
  int n;
  int format;  // pixel format / ids dtype
  int normalize, seq_len, prefix_len, has_mask, pool_argmax, prune;
  auto fields() const {
    return std::tie(tower, n, format, normalize, seq_len, prefix_len, has_mask, pool_argmax, prune);
  }
  bool operator<(const GraphKey& o) const { return fields() < o.fields(); }
};

struct Graph {
  cudaGraphExec_t exec = nullptr;
  unsigned long long kernels = 0;  // kernel nodes: what one replay adds to g_launch_count
};

}  // namespace
}  // namespace plip

using namespace plip;

struct plip_engine {
  int device = 0;
  int max_mb = 0;
  int text_pool_argmax = 0;  // rows without an eos token: 0 = position 0 (HF, eos_token_id 49407), 1 = argmax of the ids (legacy / OpenAI)
  int prune_last = 0;  // plip_set_last_layer_pruning: embedding calls run the last layer's out_proj / MLP on the pooled rows only
  int f16 = 0;  // 16-bit operand format of the packed GEMM weights and of every activation operand: 0 bf16, 1 IEEE half
  float logit_scale_exp = 1.f;
  uint8_t* d_blob = nullptr;
  // vision
  const __nv_bfloat16 *v_patch_w = nullptr, *v_proj = nullptr;
  const float *v_cls = nullptr, *v_pos = nullptr, *v_pre_g = nullptr, *v_pre_b = nullptr, *v_post_g = nullptr,
              *v_post_b = nullptr;
  LayerW vis[kLayers], txt[kLayers];
  // text
  const float *t_tok = nullptr, *t_pos = nullptr, *t_fin_g = nullptr, *t_fin_b = nullptr;
  const __nv_bfloat16* t_proj = nullptr;
  // workspace (sized for max_mb)
  float* X = nullptr;            // residual stream fp32 [rows, D]
  __nv_bfloat16* Xn = nullptr;   // bf16 copy of the residual stream (A operand of the LN-folded GEMMs) [rows, D]
  __nv_bfloat16* AO = nullptr;   // attention output [rows, D]
  float2* stats = nullptr;       // per-row (sum, sumsq) partials of X [rows, kStatSlots]
  __nv_bfloat16* QKV = nullptr;  // [rows, 3D]
  __nv_bfloat16* H = nullptr;    // fc1 output [rows, FF]; aliases the im2col matrix [mb*49, 3072]
  __nv_bfloat16* pooled = nullptr;  // [mb, 768]
  int32_t* row_idx = nullptr;       // [mb] EOS rows
  int32_t* kmask = nullptr;         // [mb*77] key padding mask
  // last use of the shared workspace through the device-pointer API (any caller stream): the host-buffer
  // path, which runs on the engine's own streams, waits for it before touching the workspace
  cudaEvent_t ev_last = nullptr;
  // host-buffer path (lazy)
  cudaStream_t s_compute = nullptr, s_copy = nullptr;
  cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
  void* d_in[2] = {nullptr, nullptr};
  size_t d_in_bytes = 0;
  void* h_stage[2] = {nullptr, nullptr};
  size_t h_stage_bytes = 0;
  float* d_out = nullptr;
  size_t d_out_bytes = 0;
  void* d_aux = nullptr;  // ids + mask for the text host path
  size_t d_aux_bytes = 0;
  int32_t* d_win = nullptr;  // window origins of plip_encode_windows, int32 [n, 2] (lazy)
  size_t d_win_bytes = 0;
  // small-batch path: the ~67 launches of a tower are replayed as ONE CUDA graph per GraphKey on engine-owned
  // staging buffers (inputs are copied in, the [n,512] result copied out), which removes the host-side launch cost
  // that dominates when a forward is only a few hundred microseconds of GPU work (reference default:
  // batch_size = 8, plip.py:95-97).  PLIP_GRAPH_MAX (default 128, 0 = off) bounds n.
  int graph_max_n = 128;
  cudaStream_t s_cap = nullptr;
  void* g_in[2] = {nullptr, nullptr};  // staged pixels / ids, attention mask
  size_t g_in_bytes[2] = {0, 0};
  float* g_out = nullptr;      // [graph_max_n, 512]
  std::map<GraphKey, Graph> graphs;
  // in-step kernel timing (plip_profile_*): a CUDA event pair around every launch of a forward pass, recorded on
  // the launch stream, so bench.py can report each kernel's average duration INSIDE the step it belongs to
  bool prof_on = false;
  int prof_tower = 0;  // 0 vision, 1 text (set by the forward that is running)
  std::vector<cudaEvent_t> prof_ev;    // event pool, two per recorded launch
  struct ProfRec { int kind; int tower; double flops, bytes; };
  std::vector<ProfRec> prof_rec;
};

namespace {

// Records an event before / after one launch when profiling is on (no-op otherwise).
struct ProfScope {
  plip_engine* e;
  cudaStream_t st;
  bool on;
  ProfScope(plip_engine* e_, cudaStream_t st_, int kind, double flops, double bytes) : e(e_), st(st_), on(e_->prof_on) {
    if (!on) return;
    if (e->prof_rec.size() >= 8192) { on = false; return; }
    cudaEvent_t a = nullptr, b = nullptr;
    if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) { on = false; return; }
    e->prof_ev.push_back(a);
    e->prof_ev.push_back(b);
    e->prof_rec.push_back({kind, e->prof_tower, flops, bytes});
    cudaEventRecord(a, st);
  }
  ~ProfScope() {
    if (on) cudaEventRecord(e->prof_ev.back(), st);
  }
};

template <typename T>
const T* wptr(const plip_engine* e, const Spec& s) {
  return reinterpret_cast<const T*>(e->d_blob + s.offset);
}

int bind_weights(plip_engine* e) {
  const auto& v = specs();
  size_t i = 0;
  auto nextf = [&]() { return wptr<float>(e, v[i++]); };
  auto nextb = [&]() { return wptr<__nv_bfloat16>(e, v[i++]); };
  auto tower = [&](LayerW* L) {
    for (int l = 0; l < kLayers; ++l) {
      L[l].wqkv = nextb(); L[l].bqkv = nextf(); L[l].sqkv = nextf();
      L[l].wo = nextb(); L[l].bo = nextf();
      L[l].w1 = nextb(); L[l].b1 = nextf(); L[l].s1 = nextf();
      L[l].w2 = nextb(); L[l].b2 = nextf();
    }
  };
  e->v_patch_w = nextb();
  e->v_cls = nextf();
  e->v_pos = nextf();
  e->v_pre_g = nextf(); e->v_pre_b = nextf();
  tower(e->vis);
  e->v_post_g = nextf(); e->v_post_b = nextf();
  e->v_proj = nextb();
  e->t_tok = nextf();
  e->t_pos = nextf();
  tower(e->txt);
  e->t_fin_g = nextf(); e->t_fin_b = nextf();
  e->t_proj = nextb();
  PLIP_REQUIRE(i == v.size(), "internal: weight table mismatch (%zu vs %zu)", i, v.size());
  return 0;
}

struct WsLayout {
  size_t x, xn, ao, stats, qkv, h, pooled, rowidx, kmask, total;
};

WsLayout ws_layout(int mb) {
  const size_t rv = (size_t)mb * kVisSeq, rt = (size_t)mb * kTxtSeq;
  auto mx = [](size_t a, size_t b) { return a > b ? a : b; };
  auto al = [](size_t a) { return (a + 1023) & ~(size_t)1023; };
  WsLayout w;
  size_t off = 0;
  w.x = off; off += al(mx(rv * kVisDim, rt * kTxtDim) * 4);
  w.xn = off; off += al(mx(rv * kVisDim, rt * kTxtDim) * 2);
  w.ao = off; off += al(mx(rv * kVisDim, rt * kTxtDim) * 2);
  w.stats = off; off += al(mx(rv, rt) * kStatSlots * sizeof(float2));
  w.qkv = off; off += al(mx(rv * 3 * kVisDim, rt * 3 * kTxtDim) * 2);
  w.h = off; off += al(mx(mx(rv * kVisFF, rt * kTxtFF), (size_t)mb * kPatches * kPatchK) * 2);
  w.pooled = off; off += al((size_t)mb * kVisDim * 2);
  w.rowidx = off; off += al((size_t)mb * 4);
  w.kmask = off; off += al(rt * 4);
  w.total = off;
  return w;
}

// One GEMM of a forward pass in the engine's operand format, profiled as `kind` with its algorithmic work
// (DESIGN.md §4): 2·M·N·K FLOPs; A and W read once, the output written once (an fp32 residual read and written),
// plus the 16-bit copy of the updated rows when the residual epilogue emits one.
int gemm(plip_engine* e, int kind, GemmArgs g, cudaStream_t st) {
  g.f16 = e->f16;
  const double M = g.M, N = g.N, K = g.K;
  const double out_elem = g.epi == EPI_BIAS_RESID_F32 ? 8 : (g.epi == EPI_F32 || g.epi == EPI_PATCH_F32 ? 4 : 2);
  ProfScope ps(e, st, kind, 2 * M * N * K, M * K * 2 + N * K * 2 + M * N * out_elem + (g.xb_out ? M * N * 2 : 0));
  return launch_gemm(g, st);
}

// The rest of an encoder layer after attention, on `rows` rows of the attention output `ao` and the fp32 residual
// stream `x`:  x = x + out_proj(ao);  x = x + fc2(quick_gelu(fc1(LN2(x))))            TF:modeling_clip.py:370-382
// The residual GEMMs leave Xn / stats (the input of the next LayerNorm-folded GEMM) and the number of statistics
// partials in np; the last layer's fc2 does not, its output only feeds the pooled-row LayerNorm (fp32 x).
int layer_tail(plip_engine* e, const LayerW& w, int rows, int D, int FF, const __nv_bfloat16* ao, float* x, bool last,
               int& np, cudaStream_t st) {
  GemmArgs g;
  g.A = ao; g.lda = D; g.W = w.wo; g.ldw = D; g.M = rows; g.N = D; g.K = D;
  g.bias = w.bo; g.out = x; g.ldo = D; g.epi = EPI_BIAS_RESID_F32;
  g.xb_out = e->Xn; g.stats_out = e->stats; g.n_tiles_used = &np;
  if (int rc = gemm(e, PK_OUT, g, st)) return rc;
  g = GemmArgs();
  g.A = e->Xn; g.lda = D; g.W = w.w1; g.ldw = D; g.M = rows; g.N = FF; g.K = D;
  g.bias = w.b1; g.colsum = w.s1; g.stats_in = e->stats; g.n_partials = np;
  g.out = e->H; g.ldo = FF; g.epi = EPI_LN_BIAS_GELU_BF16;
  if (int rc = gemm(e, PK_FC1, g, st)) return rc;
  g = GemmArgs();
  g.A = e->H; g.lda = FF; g.W = w.w2; g.ldw = FF; g.M = rows; g.N = D; g.K = FF;
  g.bias = w.b2; g.out = x; g.ldo = D; g.epi = EPI_BIAS_RESID_F32;
  if (!last) { g.xb_out = e->Xn; g.stats_out = e->stats; g.n_tiles_used = &np; }
  return gemm(e, PK_FC2, g, st);
}

// What one pass writes (null: not requested): micro-batch [i0, i0 + mb) of an n-item call's plip_tower_outputs_t, i.e.
// the caller's buffers at the micro-batch's offsets.  The per-layer ones are written by run_layers:
//   hidden: X [n_seq * S, D] is copied to hidden on entry and to hidden + (l + 1) * hidden_stride after layer l
//   attn:   the attention probabilities of layer l go to attn + l * attn_stride ([n_seq, heads, S, S] fp32)
struct PassOut {
  float *embeds = nullptr, *pooled = nullptr, *last_hidden = nullptr;
  float* hidden = nullptr;
  int64_t hidden_stride = 0;  // floats between layers
  float* attn = nullptr;
  int64_t attn_stride = 0;
  int normalize = 0;
};

PassOut pass_out(const plip_tower_outputs_t& o, int64_t n, int64_t i0, int S, int D, int heads) {
  PassOut p;
  const int64_t tok = (int64_t)S * D, pp = (int64_t)heads * S * S;
  if (o.embeds) p.embeds = o.embeds + i0 * kProj;
  if (o.pooled) p.pooled = o.pooled + i0 * D;
  if (o.last_hidden) p.last_hidden = o.last_hidden + i0 * tok;
  if (o.hidden) { p.hidden = o.hidden + i0 * tok; p.hidden_stride = n * tok; }
  if (o.attn) { p.attn = o.attn + i0 * pp; p.attn_stride = n * pp; }
  p.normalize = o.normalize;
  return p;
}

// The embedding calls (plip_encode_*): [mb, 512] at out.
PassOut embeds_only(float* out, int normalize) {
  PassOut p;
  p.embeds = out;
  p.normalize = normalize;
  return p;
}

// Encoder layers with both LayerNorms folded into the consuming GEMMs.  On entry X holds the residual
// stream; Xn / stats are (re)derived from it here and afterwards maintained by the residual epilogues.
//
// prune (embedding calls with plip_set_last_layer_pruning on; never for hidden-state requests): only the pooled row of
// each sequence leaves the tower (CLS, TF:modeling_clip.py:685; first-EOS row, :571-584), and after the last layer's
// attention nothing mixes rows any more, so that layer's out_proj, LN2, fc1 and fc2 are run on the n_seq pooled rows
// alone (gathered into compact buffers) instead of all n_seq*S rows — same arithmetic per row, identical embeddings.
// pool_idx: device row indices of the pooled rows (null = row i*S).  A pruned pass sets *pooled_x to the compact fp32
// [n_seq, D] pooled rows and writes no per-layer outputs.
int run_layers(plip_engine* e, const LayerW* L, int64_t n_seq, int S, int D, int FF, int heads, bool causal,
               const int32_t* kmask, int num_layers, cudaStream_t st, bool prune = false,
               const int32_t* pool_idx = nullptr, const PassOut& out = PassOut(), const float** pooled_x = nullptr) {
  const int64_t M = n_seq * S;
  PLIP_REQUIRE(M <= 0x7fffffff / 4, "micro-batch too large");
  PLIP_REQUIRE(!prune || (pooled_x && !out.hidden && !out.attn), "internal: per-layer outputs of a pruned pass");
  const size_t x_bytes = (size_t)M * D * 4;
  if (out.hidden) PLIP_CUDA_CHECK(cudaMemcpyAsync(out.hidden, e->X, x_bytes, cudaMemcpyDeviceToDevice, st));
  if (num_layers <= 0) return 0;
  {
    ProfScope ps(e, st, PK_ROWSTATS, 0, (double)M * D * 6 + (double)M * 8);
    if (int rc = launch_rowstats_cast(e->X, M, D, e->Xn, e->stats, e->f16, st)) return rc;
  }
  const double b_att = (double)M * 3 * D * 2 + (double)M * D * 2;
  const double f_att = 4.0 * (double)n_seq * heads * S * S * kHeadDim;
  int np = 1;
  for (int l = 0; l < num_layers; ++l) {
    const LayerW& w = L[l];
    const bool last = l + 1 == num_layers;
    // LN1 + q/k/v projection, attention                                   TF:modeling_clip.py:370-376
    GemmArgs g;
    g.A = e->Xn; g.lda = D; g.W = w.wqkv; g.ldw = D; g.M = (int)M; g.N = 3 * D; g.K = D;
    g.bias = w.bqkv; g.colsum = w.sqkv; g.stats_in = e->stats; g.n_partials = np;
    g.out = e->QKV; g.ldo = 3 * D; g.epi = EPI_LN_BIAS_BF16;
    if (int rc = gemm(e, PK_QKV, g, st)) return rc;
    {
      ProfScope ps(e, st, S > 128 ? PK_ATTN_LONG : PK_ATTN, f_att, b_att);
      if (int rc = launch_attention(e->QKV, n_seq, S, heads, causal, kmask, e->AO, e->f16, st)) return rc;
    }
    if (out.attn) {
      // reads Q and K of QKV (intact until the next layer's QKV GEMM), writes heads * S^2 fp32 per sequence
      ProfScope ps(e, st, PK_ATTN_PROBS, 0.5 * f_att, (double)M * 2 * D * 2 + (double)n_seq * heads * S * S * 4);
      if (int rc = launch_attention_probs(e->QKV, n_seq, S, heads, causal, kmask, out.attn + l * out.attn_stride,
                                          e->f16, st)) return rc;
    }
    if (!(prune && last)) {
      if (int rc = layer_tail(e, w, (int)M, D, FF, e->AO, e->X, last, np, st)) return rc;
      if (out.hidden)
        PLIP_CUDA_CHECK(cudaMemcpyAsync(out.hidden + (l + 1) * out.hidden_stride, e->X, x_bytes,
                                        cudaMemcpyDeviceToDevice, st));
      continue;
    }
    // compact copies of the pooled rows: attention output -> head of the (now free) QKV buffer, residual rows behind it
    __nv_bfloat16* ao_p = e->QKV;
    float* x_p = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(e->QKV) + (((size_t)n_seq * D * 2 + 1023) & ~(size_t)1023));
    {
      ProfScope ps(e, st, PK_MISC, 0, (double)n_seq * D * 12);
      if (int rc = launch_gather_rows(e->AO, e->X, pool_idx, S, n_seq, D, ao_p, x_p, st)) return rc;
    }
    if (int rc = layer_tail(e, w, (int)n_seq, D, FF, ao_p, x_p, true, np, st)) return rc;
    *pooled_x = x_p;
  }
  return 0;
}

// Vision tower up to (and including) `num_layers` encoder layers; X holds the residual stream [mb * geo.S, 768].
int vision_trunk(plip_engine* e, const VisInput& in, int64_t mb, const VisGeom& geo, int num_layers,
                 cudaStream_t st, bool prune = false, const PassOut& out = PassOut(),
                 const float** pooled_x = nullptr) {
  e->prof_tower = 0;
  const double dmb = (double)mb;
  const int patches = geo.gh * geo.gw;
  // Position table of the grid.  An interpolated one goes to the QKV buffer, which nothing reads before the first
  // layer's QKV GEMM: [geo.S, 768] fp32 fits, since S <= kVisSeq * max_mb and QKV holds that many rows of 2 x 2304 B.
  const float* pos = e->v_pos;
  if (geo.gh != kGrid || geo.gw != kGrid) {
    float* table = reinterpret_cast<float*>(e->QKV);
    ProfScope ps(e, st, PK_MISC, 0, (double)kVisSeq * kVisDim * 4 + (double)geo.S * kVisDim * 4);
    if (int rc = launch_pos_interp(e->v_pos, geo.gh, geo.gw, table, st)) return rc;
    pos = table;
  }
  {
    // windows: fmt is PLIP_PIX_U8_NHWC and geo 224 x 224, so the bytes are those of the same windows as tiles
    ProfScope ps(e, st, PK_IM2COL, 0, dmb * (double)pixel_bytes(in.fmt, geo.H, geo.W) + dmb * patches * kPatchK * 2);
    const int rc = in.win.region ? launch_window_im2col(in.win, mb, e->H, e->f16, st)
                                 : launch_im2col(in.pixels, in.fmt, mb, geo.H, geo.W, e->H, e->f16, st);
    if (rc) return rc;
  }
  GemmArgs g;
  g.A = e->H; g.lda = kPatchK; g.W = e->v_patch_w; g.ldw = kPatchK;
  g.M = (int)(mb * patches); g.N = kVisDim; g.K = kPatchK;
  g.out = e->X; g.ldo = kVisDim; g.pos = pos; g.patches = patches; g.seq = geo.S; g.epi = EPI_PATCH_F32;
  if (int rc = gemm(e, PK_PATCH, g, st)) return rc;
  {
    ProfScope ps(e, st, PK_MISC, 0, dmb * kVisDim * 4);
    if (int rc = launch_cls_rows(e->v_cls, pos, mb, geo.S, e->X, st)) return rc;
  }
  const int64_t M = mb * geo.S;
  {
    ProfScope ps(e, st, PK_LN, 0, (double)M * kVisDim * 8);
    if (int rc = launch_layernorm(e->X, nullptr, kVisDim, M, kVisDim, e->v_pre_g, e->v_pre_b, e->X, nullptr, e->f16, st)) return rc;
  }
  return run_layers(e, e->vis, mb, geo.S, kVisDim, kVisFF, kVisHeads, false, nullptr, num_layers, st, prune, nullptr,
                    out, pooled_x);
}

// Tower head: LayerNorm of the pooled rows -> projection [-> L2 normalise].  The pooled rows are the compact
// pooled_x rows when the last layer was pruned, else rows pool_idx[i] of X (null: row i*S).
// pooled_f32 (optional): the LayerNorm-ed pooled rows in fp32 as well, [mb, D] (pooler_output); out null: no projection.
int pooled_head(plip_engine* e, const float* pooled_x, const int32_t* pool_idx, int64_t mb, int S, int D,
                const float* gamma, const float* beta, const __nv_bfloat16* proj, float* out, int normalize,
                cudaStream_t st, float* pooled_f32) {
  {
    ProfScope ps(e, st, PK_LN, 0, (double)mb * D * (pooled_f32 ? 10 : 6));
    const bool compact = pooled_x != nullptr;
    if (int rc = launch_layernorm(compact ? pooled_x : e->X, compact ? nullptr : pool_idx,
                                  compact || pool_idx ? (int64_t)D : (int64_t)S * D, mb, D, gamma, beta, pooled_f32,
                                  e->pooled, e->f16, st)) return rc;
  }
  if (!out) return 0;
  GemmArgs g;
  g.A = e->pooled; g.lda = D; g.W = proj; g.ldw = D;
  g.M = (int)mb; g.N = kProj; g.K = D; g.out = out; g.ldo = kProj; g.epi = EPI_F32;
  if (int rc = gemm(e, PK_PROJ, g, st)) return rc;
  if (normalize) {
    ProfScope ps(e, st, PK_MISC, 0, (double)mb * kProj * 8);
    return launch_l2_normalize(out, mb, kProj, st);
  }
  return 0;
}

// One vision pass over mb images: the whole tower, then what `out` asks for.  prune: see run_layers (the embedding
// calls only).  last_hidden_state is the residual stream after the last layer, before post_layernorm (TF:680-686).
int vision_pass(plip_engine* e, const VisInput& in, int64_t mb, const VisGeom& geo, const PassOut& out, bool prune,
                cudaStream_t st) {
  const float* pooled_x = nullptr;
  if (int rc = vision_trunk(e, in, mb, geo, kLayers, st, prune, out, &pooled_x)) return rc;
  if (out.last_hidden)
    PLIP_CUDA_CHECK(cudaMemcpyAsync(out.last_hidden, e->X, (size_t)mb * geo.S * kVisDim * 4, cudaMemcpyDeviceToDevice,
                                    st));
  if (!out.embeds && !out.pooled) return 0;
  // pooled = post_layernorm(last_hidden_state[:, 0, :])                  TF:modeling_clip.py:685-686
  return pooled_head(e, pooled_x, nullptr, mb, geo.S, kVisDim, e->v_post_g, e->v_post_b, e->v_proj, out.embeds,
                     out.normalize, st, out.pooled);
}

// S = number of leading token positions actually processed (<= stride, the row length of ids / mask).
// Causality makes rows after a caption's first EOS irrelevant to its pooled output (TF:571-584), so callers
// that know the longest caption of the batch may pass a shorter S: same result, proportionally less work.
int text_trunk(plip_engine* e, const void* ids, int ids_dtype, const void* mask, int64_t mb, int S, int stride,
               int num_layers, cudaStream_t st, bool prune = false, const PassOut& out = PassOut(),
               const float** pooled_x = nullptr) {
  e->prof_tower = 1;
  {
    ProfScope ps(e, st, PK_EMBED, 0, (double)mb * S * kTxtDim * 8);
    if (int rc = launch_text_embed(ids, ids_dtype, mb, S, stride, e->t_tok, e->t_pos, e->X, e->row_idx, kEosId, e->text_pool_argmax, st)) return rc;
  }
  const int32_t* km = nullptr;
  if (mask) {
    ProfScope ps(e, st, PK_MISC, 0, (double)mb * S * 12);
    if (int rc = launch_mask_to_i32(mask, ids_dtype, mb * S, S, stride, e->kmask, st)) return rc;
    km = e->kmask;
  }
  return run_layers(e, e->txt, mb, S, kTxtDim, kTxtFF, kTxtHeads, true, km, num_layers, st, prune, e->row_idx, out,
                    pooled_x);
}

// One text pass over mb captions (the first S of `stride` positions), then what `out` asks for.
// last_hidden_state = final_layer_norm of every row (TF:562).
int text_pass(plip_engine* e, const void* ids, int ids_dtype, const void* mask, int64_t mb, int S, int stride,
              const PassOut& out, bool prune, cudaStream_t st) {
  const float* pooled_x = nullptr;
  if (int rc = text_trunk(e, ids, ids_dtype, mask, mb, S, stride, kLayers, st, prune, out, &pooled_x)) return rc;
  if (out.last_hidden) {
    ProfScope ps(e, st, PK_LN, 0, (double)mb * S * kTxtDim * 8);
    if (int rc = launch_layernorm(e->X, nullptr, kTxtDim, mb * S, kTxtDim, e->t_fin_g, e->t_fin_b, out.last_hidden,
                                  nullptr, e->f16, st)) return rc;
  }
  if (!out.embeds && !out.pooled) return 0;
  // pooled = final_layer_norm(last_hidden_state)[b, first eos]            TF:modeling_clip.py:562-584
  return pooled_head(e, pooled_x, e->row_idx, mb, S, kTxtDim, e->t_fin_g, e->t_fin_b, e->t_proj, out.embeds,
                     out.normalize, st, out.pooled);
}

int ensure_host_path(plip_engine* e) {
  if (e->s_compute) return 0;
  PLIP_CUDA_CHECK(cudaStreamCreateWithFlags(&e->s_compute, cudaStreamNonBlocking));
  PLIP_CUDA_CHECK(cudaStreamCreateWithFlags(&e->s_copy, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    PLIP_CUDA_CHECK(cudaEventCreateWithFlags(&e->ev_copied[i], cudaEventDisableTiming));
    PLIP_CUDA_CHECK(cudaEventCreateWithFlags(&e->ev_done[i], cudaEventDisableTiming));
  }
  return 0;
}

int grow_dev(void** p, size_t* have, size_t want) {
  if (*have >= want) return 0;
  if (*p) PLIP_CUDA_CHECK(cudaFree(*p));
  *p = nullptr; *have = 0;
  PLIP_CUDA_CHECK(cudaMalloc(p, want));
  *have = want;
  return 0;
}

// Length-bucketed text batches (SURVEY §8 f3).  The pooled output of a caption depends only on its positions up to
// the first EOS, so captions sorted by that length can be processed bucket by bucket, each bucket only up to its own
// longest caption.  Buckets are chosen by dynamic programming over the (<= 77) distinct lengths: cost of a bucket
// = max(captions x prefix, kMinBucketRows) + kBucketOverheadRows token rows — a GEMM needs ~8k rows to fill the
// SMs once, and a 66-launch pass costs about as much as 2k token rows — so small or uniform batches stay in
// one bucket.  perm[i] = original index of the caption at sorted position i (stable); bucket k covers sorted
// positions [start[k], start[k+1]) and is processed with prefix[k].  Returns the number of buckets.
constexpr long long kMinBucketRows = 8192, kBucketOverheadRows = 2048;
constexpr int kMaxTextBuckets = 8;

int plan_text_buckets(const int32_t* lens, int64_t n, int seq_len, int32_t* perm, int32_t* start, int32_t* prefix,
                      int cap) {
  std::vector<int64_t> upto(seq_len + 1, 0);  // upto[L] = captions with length <= L
  for (int64_t i = 0; i < n; ++i) {
    const int L = lens[i] < 1 ? 1 : (lens[i] > seq_len ? seq_len : lens[i]);
    ++upto[L];
  }
  std::vector<int64_t> first(seq_len + 2, 0);  // counting sort offsets
  for (int L = 1; L <= seq_len; ++L) first[L + 1] = first[L] + upto[L];
  if (perm) {
    std::vector<int64_t> cur(first.begin(), first.end());
    for (int64_t i = 0; i < n; ++i) {
      const int L = lens[i] < 1 ? 1 : (lens[i] > seq_len ? seq_len : lens[i]);
      perm[cur[L]++] = (int32_t)i;
    }
  }
  std::vector<int> ends;  // lengths that occur: the only sensible bucket ends
  for (int L = 1; L <= seq_len; ++L)
    if (upto[L]) ends.push_back(L);
  for (int L = 1; L <= seq_len; ++L) upto[L] += upto[L - 1];
  const int m = (int)ends.size();
  const int kb = cap < kMaxTextBuckets ? cap : kMaxTextBuckets;
  // f[b][j]: cheapest cover of the captions up to length ends[j] with exactly b+1 buckets
  const long long INF = 1LL << 62;
  std::vector<std::vector<long long>> f(kb, std::vector<long long>(m, INF));
  std::vector<std::vector<int>> from(kb, std::vector<int>(m, -1));
  auto cost = [&](int jlo, int jhi) {  // bucket holding lengths ends[jlo..jhi]
    const long long cnt = upto[ends[jhi]] - (jlo ? upto[ends[jlo - 1]] : 0);
    const long long rows = cnt * ends[jhi];
    return (rows < kMinBucketRows ? kMinBucketRows : rows) + kBucketOverheadRows;
  };
  for (int j = 0; j < m; ++j) f[0][j] = cost(0, j);
  for (int b = 1; b < kb; ++b)
    for (int j = b; j < m; ++j)
      for (int i = b - 1; i < j; ++i)
        if (f[b - 1][i] < INF) {
          const long long c = f[b - 1][i] + cost(i + 1, j);
          if (c < f[b][j]) f[b][j] = c, from[b][j] = i;
        }
  int best_b = 0;
  for (int b = 1; b < kb; ++b)
    if (m > b && f[b][m - 1] < f[best_b][m - 1]) best_b = b;
  const int nb = best_b + 1;
  int j = m - 1;
  for (int b = best_b; b >= 0; --b) {
    prefix[b] = ends[j];
    const int i = b ? from[b][j] : -1;
    start[b] = (int32_t)(i >= 0 ? upto[ends[i]] : 0);
    j = i;
  }
  start[nb] = (int32_t)n;
  return nb;
}

bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

}  // namespace

namespace {

// Kernel nodes of a captured graph.
int count_kernel_nodes(cudaGraph_t g, unsigned long long* kernels) {
  size_t n = 0;
  PLIP_CUDA_CHECK(cudaGraphGetNodes(g, nullptr, &n));
  std::vector<cudaGraphNode_t> nodes(n);
  PLIP_CUDA_CHECK(cudaGraphGetNodes(g, nodes.data(), &n));
  *kernels = 0;
  for (cudaGraphNode_t node : nodes) {
    cudaGraphNodeType type;
    PLIP_CUDA_CHECK(cudaGraphNodeGetType(node, &type));
    *kernels += type == cudaGraphNodeTypeKernel;
  }
  return 0;
}

// Capture `body` (stream-ordered launches on e->s_cap, nothing executes) into an executable graph.  The captured
// launches were counted by launch_kernel but do not run: they come off g_launch_count and are added per replay.
template <typename F>
int capture_graph(plip_engine* e, F&& body, Graph* out) {
  if (!e->s_cap) PLIP_CUDA_CHECK(cudaStreamCreateWithFlags(&e->s_cap, cudaStreamNonBlocking));
  PLIP_CUDA_CHECK(cudaStreamBeginCapture(e->s_cap, cudaStreamCaptureModeThreadLocal));
  int rc = body(e->s_cap);
  cudaGraph_t g = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(e->s_cap, &g);
  if (g) {
    const int rc_count = count_kernel_nodes(g, &out->kernels);
    if (rc == 0) rc = rc_count;
    g_launch_count.fetch_sub(out->kernels, std::memory_order_relaxed);
  }
  if (rc != 0) {
    if (g) cudaGraphDestroy(g);
    return rc;
  }
  PLIP_CUDA_CHECK(ce);
  const cudaError_t ci = cudaGraphInstantiate(&out->exec, g, 0);
  cudaGraphDestroy(g);
  PLIP_CUDA_CHECK(ci);
  return 0;
}

// Arguments of a call on n images (interpolate_pos_encoding: any size): 32 <= H, W and a patch grid of at most
// kMaxGrid x kMaxGrid, and one image's tokens must fit the workspace's kVisSeq * max_micro_batch token rows.  Pointers
// and shapes are checked before the handle, so a bad argument is reported as such whatever else is wrong.
int check_pixels(const char* fn, const plip_engine* e, const void* in, const void* out, int fmt, int64_t n,
                 int height, int width) {
  PLIP_REQUIRE(in && out, "%s: null argument", fn);
  PLIP_REQUIRE(n > 0, "%s: n must be positive (got %lld)", fn, (long long)n);
  PLIP_REQUIRE(fmt >= 0 && fmt <= 2, "%s: unknown pixel format %d", fn, fmt);
  PLIP_REQUIRE(height >= kPatch && width >= kPatch && height / kPatch <= kMaxGrid && width / kPatch <= kMaxGrid,
               "%s: image size %dx%d out of range (32 <= height, width and at most %d patches of 32 per side)", fn,
               height, width, kMaxGrid);
  PLIP_REQUIRE(e != nullptr, "%s: null engine", fn);
  const int S = (height / kPatch) * (width / kPatch) + 1;
  PLIP_REQUIRE(S <= (int64_t)kVisSeq * e->max_mb,
               "%s: a %dx%d image has %d tokens, more than the %lld token rows of the workspace "
               "(%d x max_micro_batch %d); create the engine with max_micro_batch >= %d",
               fn, height, width, S, (long long)kVisSeq * e->max_mb, kVisSeq, e->max_mb, (S + kVisSeq - 1) / kVisSeq);
  return 0;
}

// Arguments of a call on n captions of seq_len ids (the TF message for a bad seq_len), of which the first prefix_len
// are processed; the same order as check_pixels.
int check_ids(const char* fn, const plip_engine* e, const void* ids, const void* out, int ids_dtype, int64_t n,
              int seq_len, int prefix_len) {
  PLIP_REQUIRE(ids && out, "%s: null argument", fn);
  PLIP_REQUIRE(n > 0, "%s: n must be positive (got %lld)", fn, (long long)n);
  PLIP_REQUIRE(seq_len >= 1 && seq_len <= kTxtSeq,
               "Sequence length must be less than max_position_embeddings (got `sequence length`: %d and "
               "max_position_embeddings: %d)", seq_len, kTxtSeq);  // message mirrors TF:243-247
  PLIP_REQUIRE(prefix_len >= 1 && prefix_len <= seq_len, "%s: prefix_len %d out of [1,%d]", fn, prefix_len, seq_len);
  PLIP_REQUIRE(ids_dtype == PLIP_IDS_I32 || ids_dtype == PLIP_IDS_I64, "%s: unknown ids dtype %d", fn, ids_dtype);
  PLIP_REQUIRE(e != nullptr, "%s: null engine", fn);
  return 0;
}

int check_outputs(const char* fn, const plip_tower_outputs_t* o) {
  PLIP_REQUIRE(o != nullptr, "%s: null outputs", fn);
  PLIP_REQUIRE(o->embeds || o->pooled || o->last_hidden || o->hidden || o->attn, "%s: no output requested", fn);
  return 0;
}

// Arguments of a call on n 224 x 224 windows of a height x width uint8 region of `channels` bytes per pixel (rows
// row_pitch bytes apart): every host origin (row, col) is checked against the region before anything is launched, and
// a bad one is named.
int check_windows(const char* fn, const void* region, int height, int width, int64_t row_pitch,
                  const int32_t* origins, int64_t n, const void* out, int channels = 3) {
  PLIP_REQUIRE(region && origins && out, "%s: null argument", fn);
  PLIP_REQUIRE(n > 0, "%s: n must be positive (got %lld)", fn, (long long)n);
  PLIP_REQUIRE(height >= kImage && width >= kImage, "%s: region %dx%d is smaller than one %dx%d window", fn, height,
               width, kImage, kImage);
  PLIP_REQUIRE(row_pitch >= (int64_t)channels * width, "%s: row pitch %lld bytes < %d * width = %lld", fn,
               (long long)row_pitch, channels, (long long)channels * width);
  for (int64_t i = 0; i < n; ++i) {
    const int r = origins[2 * i], c = origins[2 * i + 1];
    PLIP_REQUIRE(r >= 0 && c >= 0 && r <= height - kImage && c <= width - kImage,
                 "%s: window %lld at (%d, %d) is outside the %dx%d region (rows 0..%d, columns 0..%d)", fn,
                 (long long)i, r, c, height, width, height - kImage, width - kImage);
  }
  return 0;
}

// The protocol of an eager device-pointer call: calls on different streams share one workspace, so the call waits for
// its last use, runs pass(i, mb) over items [i, i + mb) in passes of at most per_pass, and marks its own last use.
template <typename F>
int micro_batches(plip_engine* e, int64_t n, int64_t per_pass, cudaStream_t st, F&& pass) {
  PLIP_CUDA_CHECK(cudaStreamWaitEvent(st, e->ev_last, 0));
  for (int64_t i = 0; i < n; i += per_pass)
    if (int rc = pass(i, n - i < per_pass ? n - i : per_pass)) return rc;
  PLIP_CUDA_CHECK(cudaEventRecord(e->ev_last, st));
  return 0;
}

bool graph_eligible(const plip_engine* e, int64_t n) {
  return e->graph_max_n > 0 && n <= e->graph_max_n && n <= e->max_mb && !e->prof_on;
}

// A caller that cycles through many batch sizes / formats must not accumulate executable graphs without bound.
constexpr size_t kMaxGraphs = 96;
void trim_graphs(plip_engine* e) {
  if (e->graphs.size() < kMaxGraphs) return;
  cudaDeviceSynchronize();  // none of them may still be running
  for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second.exec);
  e->graphs.clear();
}

// A caller's input buffer of a graph-replayed call (src null: absent); input i is staged in e->g_in[i].
struct Staged {
  const void* src;
  size_t bytes;
};

// Small-batch path (graph_eligible), waiting for and marking the workspace as micro_batches does: the first call of a
// key runs forward(stream, in0, in1, out) eagerly on the caller's buffers, which also configures every kernel, then
// records it as a graph on the staging buffers.  Later calls copy the inputs in, replay the graph and copy the [n, 512]
// result out.
template <typename F>
int graph_call(plip_engine* e, const GraphKey& key, std::array<Staged, 2> in, float* out, cudaStream_t st,
               F&& forward) {
  PLIP_CUDA_CHECK(cudaStreamWaitEvent(st, e->ev_last, 0));
  auto it = e->graphs.find(key);
  if (it == e->graphs.end()) {
    const size_t stage_bytes[2] = {(size_t)e->graph_max_n * pixel_bytes(PLIP_PIX_F32_NCHW),
                                   (size_t)e->graph_max_n * kTxtSeq * 8};
    for (int i = 0; i < 2; ++i)
      if (in[i].src)
        if (int rc = grow_dev(&e->g_in[i], &e->g_in_bytes[i], stage_bytes[i])) return rc;
    if (!e->g_out) PLIP_CUDA_CHECK(cudaMalloc(&e->g_out, (size_t)e->graph_max_n * kProj * 4));
    if (int rc = forward(st, in[0].src, in[1].src, out)) return rc;
    Graph graph;
    if (int rc = capture_graph(e, [&](cudaStream_t cs) {
          return forward(cs, in[0].src ? e->g_in[0] : nullptr, in[1].src ? e->g_in[1] : nullptr, e->g_out);
        }, &graph)) return rc;
    trim_graphs(e);
    e->graphs.emplace(key, graph);
  } else {
    for (int i = 0; i < 2; ++i)
      if (in[i].src) PLIP_CUDA_CHECK(cudaMemcpyAsync(e->g_in[i], in[i].src, in[i].bytes, cudaMemcpyDeviceToDevice, st));
    PLIP_CUDA_CHECK(cudaGraphLaunch(it->second.exec, st));
    PLIP_CUDA_CHECK(cudaMemcpyAsync(out, e->g_out, (size_t)key.n * kProj * 4, cudaMemcpyDeviceToDevice, st));
    g_launch_count.fetch_add(it->second.kernels, std::memory_order_relaxed);
  }
  PLIP_CUDA_CHECK(cudaEventRecord(e->ev_last, st));
  return 0;
}

// plip_dbg_hidden_states[_hw]: one pass of a tower's trunk (tower 0: height x width images, 1: 77-token captions) up
// to num_layers encoder layers, then its residual stream X [n * S, D] copied to hidden.
int dbg_hidden_states(const char* fn, plip_engine* e, int tower, const void* in, int fmt, const void* mask, int64_t n,
                      int height, int width, int num_layers, float* hidden, cudaStream_t st) {
  PLIP_REQUIRE(tower == 0 || tower == 1, "%s: tower %d out of range (0 vision, 1 text)", fn, tower);
  PLIP_REQUIRE(num_layers >= 0 && num_layers <= kLayers, "%s: num_layers %d out of range", fn, num_layers);
  if (int rc = tower == 0 ? check_pixels(fn, e, in, hidden, fmt, n, height, width)
                          : check_ids(fn, e, in, hidden, fmt, n, kTxtSeq, kTxtSeq)) return rc;
  const VisGeom geo = vis_geom(height, width);
  const int S = tower == 0 ? geo.S : kTxtSeq, D = tower == 0 ? kVisDim : kTxtDim;
  const int64_t per_pass = tower == 0 ? images_per_pass(e->max_mb, S) : e->max_mb;
  PLIP_REQUIRE(n <= per_pass, "%s: n=%lld sequences of %d tokens exceed one pass (%lld)", fn, (long long)n, S,
               (long long)per_pass);
  return micro_batches(e, n, n, st, [&](int64_t, int64_t) {
    if (int rc = tower == 0 ? vision_trunk(e, tiles(in, fmt), n, geo, num_layers, st)
                            : text_trunk(e, in, fmt, mask, n, kTxtSeq, kTxtSeq, num_layers, st)) return rc;
    PLIP_CUDA_CHECK(cudaMemcpyAsync(hidden, e->X, (size_t)n * S * D * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  });
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

PLIP_API const char* plip_last_error(void) { return plip::get_last_error(); }
PLIP_API int plip_abi_version(void) { return PLIP_B200_ABI_VERSION; }
PLIP_API uint64_t plip_launch_count(void) { return plip::g_launch_count.load(std::memory_order_relaxed); }

PLIP_API int plip_weights_num_tensors(void) { return (int)specs().size(); }

PLIP_API int plip_weights_tensor_info(int index, plip_tensor_info_t* info) {
  const auto& v = specs();
  PLIP_REQUIRE(info != nullptr && index >= 0 && index < (int)v.size(), "tensor_info: index %d out of range", index);
  memset(info, 0, sizeof(*info));
  strncpy(info->name, v[index].name.c_str(), sizeof(info->name) - 1);
  info->offset = v[index].offset;
  info->numel = v[index].numel;
  info->dtype = v[index].dtype;
  info->rows = v[index].rows;
  info->cols = v[index].cols;
  info->fused = v[index].fused;
  return 0;
}

PLIP_API uint64_t plip_weights_blob_bytes(void) { return blob_bytes(); }

PLIP_API uint64_t plip_workspace_bytes(int max_micro_batch) {
  return max_micro_batch > 0 ? ws_layout(max_micro_batch).total : 0;
}

PLIP_API int plip_create(const void* host_blob, uint64_t nbytes, float logit_scale_exp, int device,
                         int max_micro_batch, plip_engine_t** out) {
  return plip_create_ex(host_blob, nbytes, logit_scale_exp, device, max_micro_batch, PLIP_OPERAND_BF16, out);
}

PLIP_API int plip_create_ex(const void* host_blob, uint64_t nbytes, float logit_scale_exp, int device,
                            int max_micro_batch, int operand_format, plip_engine_t** out) {
  PLIP_REQUIRE(out != nullptr && host_blob != nullptr, "plip_create: null argument");
  PLIP_REQUIRE(operand_format == PLIP_OPERAND_BF16 || operand_format == PLIP_OPERAND_FP16,
               "plip_create: unknown operand format %d", operand_format);
  PLIP_REQUIRE(nbytes == blob_bytes(), "plip_create: blob is %llu bytes, expected %llu",
               (unsigned long long)nbytes, (unsigned long long)blob_bytes());
  PLIP_REQUIRE(max_micro_batch >= 1 && max_micro_batch <= 8192, "plip_create: max_micro_batch %d out of [1,8192]",
               max_micro_batch);
  int ndev = 0;
  PLIP_CUDA_CHECK(cudaGetDeviceCount(&ndev));
  PLIP_REQUIRE(device >= 0 && device < ndev, "plip_create: device %d not present (%d devices)", device, ndev);
  PLIP_CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  PLIP_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  PLIP_REQUIRE(prop.major == 9 && prop.minor == 0, "plip_create: device %d is sm_%d%d; this library is built for sm_90a only",
               device, prop.major, prop.minor);
  plip_engine* e = new plip_engine();
  e->device = device;
  e->max_mb = max_micro_batch;
  e->f16 = operand_format == PLIP_OPERAND_FP16 ? 1 : 0;
  if (const char* gm = getenv("PLIP_GRAPH_MAX")) e->graph_max_n = atoi(gm) < 0 ? 0 : (atoi(gm) > 1024 ? 1024 : atoi(gm));
  e->logit_scale_exp = logit_scale_exp;
  const WsLayout w = ws_layout(max_micro_batch);
  uint8_t* ws = nullptr;
  cudaError_t ce = cudaEventCreateWithFlags(&e->ev_last, cudaEventDisableTiming);
  if (ce == cudaSuccess) ce = cudaMalloc(&e->d_blob, nbytes);
  if (ce == cudaSuccess) ce = cudaMalloc(&ws, w.total);
  e->X = reinterpret_cast<float*>(ws);  // workspace base (w.x == 0): what plip_destroy frees
  if (ce != cudaSuccess) {
    set_last_error("plip_create: allocating %llu (weights) + %llu (workspace) bytes on device %d failed: %s",
                   (unsigned long long)nbytes, (unsigned long long)w.total, device, cudaGetErrorString(ce));
    cudaGetLastError();
    plip_destroy(e);
    return -1;
  }
  e->Xn = reinterpret_cast<__nv_bfloat16*>(ws + w.xn);
  e->AO = reinterpret_cast<__nv_bfloat16*>(ws + w.ao);
  e->stats = reinterpret_cast<float2*>(ws + w.stats);
  e->QKV = reinterpret_cast<__nv_bfloat16*>(ws + w.qkv);
  e->H = reinterpret_cast<__nv_bfloat16*>(ws + w.h);
  e->pooled = reinterpret_cast<__nv_bfloat16*>(ws + w.pooled);
  e->row_idx = reinterpret_cast<int32_t*>(ws + w.rowidx);
  e->kmask = reinterpret_cast<int32_t*>(ws + w.kmask);
  ce = cudaMemcpy(e->d_blob, host_blob, nbytes, cudaMemcpyHostToDevice);
  if (ce != cudaSuccess) {
    set_last_error("plip_create: weight upload failed: %s", cudaGetErrorString(ce));
    plip_destroy(e);
    return -1;
  }
  if (bind_weights(e) != 0) {
    plip_destroy(e);
    return -1;
  }
  *out = e;
  return 0;
}

PLIP_API int plip_destroy(plip_engine_t* e) {
  if (!e) return 0;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  if (e->d_blob) cudaFree(e->d_blob);
  if (e->X) cudaFree(e->X);  // base of the workspace allocation
  for (int i = 0; i < 2; ++i) {
    if (e->d_in[i]) cudaFree(e->d_in[i]);
    if (e->h_stage[i]) cudaFreeHost(e->h_stage[i]);
    if (e->ev_copied[i]) cudaEventDestroy(e->ev_copied[i]);
    if (e->ev_done[i]) cudaEventDestroy(e->ev_done[i]);
  }
  if (e->d_out) cudaFree(e->d_out);
  if (e->d_aux) cudaFree(e->d_aux);
  if (e->d_win) cudaFree(e->d_win);
  if (e->ev_last) cudaEventDestroy(e->ev_last);
  for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second.exec);
  for (void* p : e->g_in)
    if (p) cudaFree(p);
  if (e->g_out) cudaFree(e->g_out);
  if (e->s_cap) cudaStreamDestroy(e->s_cap);
  for (cudaEvent_t ev : e->prof_ev) cudaEventDestroy(ev);
  if (e->s_compute) cudaStreamDestroy(e->s_compute);
  if (e->s_copy) cudaStreamDestroy(e->s_copy);
  delete e;
  return 0;
}

PLIP_API int plip_profile_enable(plip_engine_t* e, int on) {
  PLIP_REQUIRE(e != nullptr, "plip_profile_enable: null engine");
  for (cudaEvent_t ev : e->prof_ev) cudaEventDestroy(ev);
  e->prof_ev.clear();
  e->prof_rec.clear();
  e->prof_on = on != 0;
  return 0;
}

PLIP_API int plip_profile_read(plip_engine_t* e, plip_kernel_time_t* out, int cap, int* count) {
  PLIP_REQUIRE(e && out && count && cap > 0, "plip_profile_read: bad argument");
  plip_kernel_time_t agg[2 * PK_COUNT];
  memset(agg, 0, sizeof(agg));
  for (size_t i = 0; i < e->prof_rec.size(); ++i) {
    PLIP_CUDA_CHECK(cudaEventSynchronize(e->prof_ev[2 * i + 1]));
    float ms = 0.f;
    PLIP_CUDA_CHECK(cudaEventElapsedTime(&ms, e->prof_ev[2 * i], e->prof_ev[2 * i + 1]));
    plip_kernel_time_t& a = agg[e->prof_rec[i].tower * PK_COUNT + e->prof_rec[i].kind];
    a.launches += 1;
    a.total_ms += ms;
    a.flops += e->prof_rec[i].flops;
    a.bytes += e->prof_rec[i].bytes;
  }
  int n = 0;
  for (int t = 0; t < 2; ++t)
    for (int k = 0; k < PK_COUNT; ++k) {
      const plip_kernel_time_t& a = agg[t * PK_COUNT + k];
      if (a.launches == 0) continue;
      if (n < cap) {
        out[n] = a;
        snprintf(out[n].name, sizeof(out[n].name), "%s/%s", t == 0 ? "vision" : "text", kProfNames[k]);
      }
      ++n;
    }
  *count = n;
  return 0;
}

PLIP_API float plip_logit_scale_exp(const plip_engine_t* e) { return e ? e->logit_scale_exp : 0.f; }
PLIP_API int plip_max_micro_batch(const plip_engine_t* e) { return e ? e->max_mb : 0; }
PLIP_API int plip_operand_format(const plip_engine_t* e) { return e ? e->f16 : -1; }
PLIP_API int plip_set_text_pooling(plip_engine_t* e, int no_eos_argmax) {
  PLIP_REQUIRE(e != nullptr, "plip_set_text_pooling: null engine");
  e->text_pool_argmax = no_eos_argmax != 0;
  return 0;
}

PLIP_API int plip_set_last_layer_pruning(plip_engine_t* e, int on) {
  PLIP_REQUIRE(e != nullptr, "plip_set_last_layer_pruning: null engine");
  e->prune_last = on != 0;
  return 0;
}
PLIP_API int plip_last_layer_pruning(const plip_engine_t* e) { return e ? e->prune_last : -1; }

PLIP_API int plip_encode_images(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n,
                                float* out_dev, int normalize, void* stream) {
  return plip_encode_images_hw(e, pixels_dev, pixel_format, n, kImage, kImage, out_dev, normalize, stream);
}

PLIP_API int plip_encode_images_hw(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n, int height,
                                   int width, float* out_dev, int normalize, void* stream) {
  if (int rc = check_pixels("plip_encode_images_hw", e, pixels_dev, out_dev, pixel_format, n, height, width)) return rc;
  const VisGeom geo = vis_geom(height, width);
  const size_t pb = pixel_bytes(pixel_format, height, width);
  const bool prune = e->prune_last != 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (height == kImage && width == kImage && graph_eligible(e, n)) {
    const GraphKey key{0, (int)n, pixel_format, normalize ? 1 : 0, 0, 0, 0, 0, e->prune_last};
    return graph_call(e, key, {{{pixels_dev, (size_t)n * pb}, {nullptr, 0}}}, out_dev, st,
                      [&](cudaStream_t s, const void* pixels, const void*, float* out) {
                        return vision_pass(e, tiles(pixels, pixel_format), n, geo, embeds_only(out, normalize), prune,
                                           s);
                      });
  }
  return micro_batches(e, n, images_per_pass(e->max_mb, geo.S), st, [&](int64_t i, int64_t mb) {
    return vision_pass(e, tiles(static_cast<const uint8_t*>(pixels_dev) + i * pb, pixel_format), mb, geo,
                       embeds_only(out_dev + i * kProj, normalize), prune, st);
  });
}

PLIP_API int plip_encode_windows(plip_engine_t* e, const void* region_dev, int height, int width,
                                 int64_t row_pitch_bytes, const int32_t* origins_host, int64_t n, float* out_dev,
                                 int normalize, void* stream) {
  if (int rc = check_windows("plip_encode_windows", region_dev, height, width, row_pitch_bytes, origins_host, n,
                             out_dev)) return rc;
  PLIP_REQUIRE(e != nullptr, "plip_encode_windows: null engine");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // the engine's origin buffer may still be read by the previous call (any stream): wait for it before the upload
  PLIP_CUDA_CHECK(cudaStreamWaitEvent(st, e->ev_last, 0));
  if (int rc = grow_dev(reinterpret_cast<void**>(&e->d_win), &e->d_win_bytes, (size_t)n * 2 * sizeof(int32_t)))
    return rc;
  PLIP_CUDA_CHECK(cudaMemcpyAsync(e->d_win, origins_host, (size_t)n * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  const bool prune = e->prune_last != 0;
  const uint8_t* region = static_cast<const uint8_t*>(region_dev);
  // the micro-batches of plip_encode_images on tiles (no graph replay: its staging buffers hold tiles)
  return micro_batches(e, n, images_per_pass(e->max_mb, kVisSeq), st, [&](int64_t i, int64_t mb) {
    const VisInput in{nullptr, PLIP_PIX_U8_NHWC, WindowSrc{region, row_pitch_bytes, e->d_win + 2 * i}};
    return vision_pass(e, in, mb, VisGeom(), embeds_only(out_dev + i * kProj, normalize), prune, st);
  });
}

PLIP_API int plip_window_background_counts(const void* region_dev, int height, int width, int64_t row_pitch_bytes,
                                           const int32_t* origins_host, int64_t n, int threshold, int32_t* counts_dev,
                                           void* stream) {
  if (int rc = check_windows("plip_window_background_counts", region_dev, height, width, row_pitch_bytes,
                             origins_host, n, counts_dev)) return rc;
  return launch_window_background(static_cast<const uint8_t*>(region_dev), row_pitch_bytes, origins_host, n, threshold,
                                  counts_dev, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_window_mask_counts(const void* mask_dev, int height, int width, int channels,
                                     int64_t row_pitch_bytes, const int32_t* origins_host, int64_t n, int threshold,
                                     int32_t* counts_dev, void* stream) {
  PLIP_REQUIRE(channels == 1 || channels == 3, "plip_window_mask_counts: channels must be 1 or 3 (got %d)", channels);
  if (int rc = check_windows("plip_window_mask_counts", mask_dev, height, width, row_pitch_bytes, origins_host, n,
                             counts_dev, channels)) return rc;
  return launch_window_mask(static_cast<const uint8_t*>(mask_dev), row_pitch_bytes, channels, origins_host, n,
                            threshold, counts_dev, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_encode_text(plip_engine_t* e, const void* ids_dev, int ids_dtype, const void* attention_mask_dev,
                              int64_t n, int seq_len, float* out_dev, int normalize, void* stream) {
  return plip_encode_text_prefix(e, ids_dev, ids_dtype, attention_mask_dev, n, seq_len, seq_len, out_dev, normalize,
                                 stream);
}

PLIP_API int plip_encode_text_prefix(plip_engine_t* e, const void* ids_dev, int ids_dtype,
                                     const void* attention_mask_dev, int64_t n, int seq_len, int prefix_len,
                                     float* out_dev, int normalize, void* stream) {
  if (int rc = check_ids("plip_encode_text", e, ids_dev, out_dev, ids_dtype, n, seq_len, prefix_len)) return rc;
  const size_t row = (size_t)seq_len * (ids_dtype == PLIP_IDS_I64 ? 8 : 4);
  const bool prune = e->prune_last != 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (graph_eligible(e, n)) {
    const GraphKey key{1, (int)n, ids_dtype, normalize ? 1 : 0, seq_len, prefix_len, attention_mask_dev ? 1 : 0,
                       e->text_pool_argmax, e->prune_last};
    return graph_call(e, key, {{{ids_dev, n * row}, {attention_mask_dev, n * row}}}, out_dev, st,
                      [&](cudaStream_t s, const void* ids, const void* mask, float* out) {
                        return text_pass(e, ids, ids_dtype, mask, n, prefix_len, seq_len, embeds_only(out, normalize),
                                         prune, s);
                      });
  }
  return micro_batches(e, n, e->max_mb, st, [&](int64_t i, int64_t mb) {
    const uint8_t* mask = attention_mask_dev ? static_cast<const uint8_t*>(attention_mask_dev) + i * row : nullptr;
    return text_pass(e, static_cast<const uint8_t*>(ids_dev) + i * row, ids_dtype, mask, mb, prefix_len, seq_len,
                     embeds_only(out_dev + i * kProj, normalize), prune, st);
  });
}

PLIP_API int plip_vision_outputs(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n, int height,
                                 int width, const plip_tower_outputs_t* outputs, void* stream) {
  if (int rc = check_outputs("plip_vision_outputs", outputs)) return rc;
  if (int rc = check_pixels("plip_vision_outputs", e, pixels_dev, outputs, pixel_format, n, height, width)) return rc;
  const VisGeom geo = vis_geom(height, width);
  const size_t pb = pixel_bytes(pixel_format, height, width);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return micro_batches(e, n, images_per_pass(e->max_mb, geo.S), st, [&](int64_t i, int64_t mb) {
    return vision_pass(e, tiles(static_cast<const uint8_t*>(pixels_dev) + i * pb, pixel_format), mb, geo,
                       pass_out(*outputs, n, i, geo.S, kVisDim, kVisHeads), false, st);
  });
}

PLIP_API int plip_text_outputs(plip_engine_t* e, const void* ids_dev, int ids_dtype, const void* attention_mask_dev,
                               int64_t n, int seq_len, const plip_tower_outputs_t* outputs, void* stream) {
  if (int rc = check_outputs("plip_text_outputs", outputs)) return rc;
  if (int rc = check_ids("plip_text_outputs", e, ids_dev, outputs, ids_dtype, n, seq_len, seq_len)) return rc;
  const size_t row = (size_t)seq_len * (ids_dtype == PLIP_IDS_I64 ? 8 : 4);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return micro_batches(e, n, e->max_mb, st, [&](int64_t i, int64_t mb) {
    const uint8_t* mask = attention_mask_dev ? static_cast<const uint8_t*>(attention_mask_dev) + i * row : nullptr;
    return text_pass(e, static_cast<const uint8_t*>(ids_dev) + i * row, ids_dtype, mask, mb, seq_len, seq_len,
                     pass_out(*outputs, n, i, seq_len, kTxtDim, kTxtHeads), false, st);
  });
}

PLIP_API int plip_similarity(const float* img_dev, int64_t n, const float* txt_dev, int64_t m, float scale,
                             int normalize_img, int normalize_txt, float* logits_dev, int64_t ld_logits,
                             void* stream) {
  PLIP_REQUIRE(img_dev && txt_dev && logits_dev, "plip_similarity: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t chunk = 65535LL * 64;  // grid.y limit
  for (int64_t i = 0; i < n; i += chunk) {
    const int64_t rows = n - i < chunk ? n - i : chunk;
    if (int rc = launch_similarity(img_dev + i * kProj, rows, txt_dev, m, scale, normalize_img != 0,
                                   normalize_txt != 0, logits_dev + i * ld_logits, ld_logits, st)) return rc;
  }
  return 0;
}

PLIP_API int plip_similarity_topk(const float* query_dev, int64_t n, const float* space_dev, int64_t m, float scale,
                                  int normalize_query, int normalize_space, int k, int32_t* idx_dev, float* val_dev,
                                  void* stream) {
  PLIP_REQUIRE(query_dev && space_dev && idx_dev, "plip_similarity_topk: null argument");
  return launch_similarity_topk(query_dev, n, space_dev, m, scale, normalize_query != 0, normalize_space != 0, k,
                                idx_dev, val_dev, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_l2_normalize(float* x_dev, int64_t n, int dim, void* stream) {
  PLIP_REQUIRE(x_dev, "plip_l2_normalize: null argument");
  return launch_l2_normalize(x_dev, n, dim, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_resize_crop_u8(const void* src_dev, uint64_t src_bytes, const plip_resize_desc_t* descs_host,
                                 int64_t n, void* tiles_dev, void* stream) {
  PLIP_REQUIRE(src_dev && descs_host && tiles_dev, "plip_resize_crop_u8: null argument");
  PLIP_REQUIRE(n > 0, "plip_resize_crop_u8: n must be positive (got %lld)", (long long)n);
  return launch_resize_crop(static_cast<const uint8_t*>(src_dev), (size_t)src_bytes, descs_host, n,
                            static_cast<uint8_t*>(tiles_dev), static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_resize_crop_bilinear_u8(const void* src_dev, uint64_t src_bytes, const plip_resize_desc_t* descs_host,
                                          int64_t n, void* tiles_dev, void* stream) {
  PLIP_REQUIRE(src_dev && descs_host && tiles_dev, "plip_resize_crop_bilinear_u8: null argument");
  PLIP_REQUIRE(n > 0, "plip_resize_crop_bilinear_u8: n must be positive (got %lld)", (long long)n);
  return launch_resize_crop(static_cast<const uint8_t*>(src_dev), (size_t)src_bytes, descs_host, n,
                            static_cast<uint8_t*>(tiles_dev), static_cast<cudaStream_t>(stream), true);
}

PLIP_API int plip_resize_region_workspace(int height, int width, int new_height, int new_width, int out_row0,
                                          int out_row1, uint64_t* bytes) {
  PLIP_REQUIRE(bytes, "plip_resize_region_workspace: null argument");
  return resize_region_workspace(height, width, new_height, new_width, out_row0, out_row1, bytes);
}

PLIP_API int plip_resize_region_u8(const void* src_dev, int64_t src_row_pitch, int src_row0, int src_rows, int height,
                                   int width, void* out_dev, int64_t out_row_pitch, int new_height, int new_width,
                                   int out_row0, int out_row1, void* workspace_dev, uint64_t workspace_bytes,
                                   void* stream) {
  PLIP_REQUIRE(src_dev && out_dev && workspace_dev, "plip_resize_region_u8: null argument");
  return launch_resize_region(static_cast<const uint8_t*>(src_dev), src_row_pitch, src_row0, src_rows, height, width,
                              static_cast<uint8_t*>(out_dev), out_row_pitch, new_height, new_width, out_row0, out_row1,
                              static_cast<uint8_t*>(workspace_dev), workspace_bytes, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_resize_filter_bounds(int in_size, int out_size, int32_t* bounds_host) {
  PLIP_REQUIRE(bounds_host, "plip_resize_filter_bounds: null argument");
  PLIP_REQUIRE(in_size >= 1 && out_size >= 1 && in_size <= 65536 && out_size <= 65536,
               "plip_resize_filter_bounds: sizes %d -> %d are outside 1..65536", in_size, out_size);
  return resize_filter_bounds(in_size, out_size, bounds_host);
}

PLIP_API int plip_sgd_shuffle_permutation(int64_t n, uint32_t seed, int32_t* sigma_host) {
  return sgd_shuffle_permutation(n, seed, sigma_host);
}

PLIP_API int plip_sgd_workspace_bytes(int64_t n, int n_sigma, int n_problems, uint64_t* bytes) {
  return sgd_workspace_bytes(n, n_sigma, n_problems, bytes);
}

PLIP_API int plip_sgd_fit(const float* x_dev, int64_t n, int dim, const int32_t* class_host, int n_classes,
                          const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host,
                          int n_sigma, int max_iter, double tol, int n_iter_no_change, float* coef_dev,
                          double* intercept_dev, int32_t* n_iter_dev, int32_t* overflow_dev, void* workspace_dev,
                          uint64_t workspace_bytes, void* stream) {
  return launch_sgd_fit(x_dev, n, dim, class_host, n_classes, problems_host, n_problems, sigma_host, n_sigma, max_iter,
                        tol, n_iter_no_change, coef_dev, intercept_dev, n_iter_dev, overflow_dev, workspace_dev,
                        workspace_bytes, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_linear_decision(const float* x_dev, int64_t n, int dim, const float* coef_dev,
                                  const double* intercept_dev, int n_out, float* scores_dev, int32_t* pred_dev,
                                  void* stream) {
  return launch_linear_decision(x_dev, n, dim, coef_dev, intercept_dev, n_out, scores_dev, pred_dev,
                                static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_resize_filter(int in_size, int out_size, int xx, int32_t* k_host, int k_cap, int* xmin,
                                    int* count) {
  PLIP_REQUIRE(k_host && xmin && count && in_size > 0 && out_size > 0 && xx >= 0 && xx < out_size,
               "plip_dbg_resize_filter: bad argument");
  return resize_filter_host(in_size, out_size, xx, k_host, k_cap, xmin, count);
}

PLIP_API int plip_dbg_resize_filter_bilinear(int in_size, int out_size, int xx, int32_t* k_host, int k_cap, int* xmin,
                                             int* count) {
  PLIP_REQUIRE(k_host && xmin && count && in_size > 0 && out_size > 0 && xx >= 0 && xx < out_size,
               "plip_dbg_resize_filter_bilinear: bad argument");
  return resize_filter_bilinear_host(in_size, out_size, xx, k_host, k_cap, xmin, count);
}

// ---- host-buffer path ---------------------------------------------------------------------------
PLIP_API int plip_encode_images_host(plip_engine_t* e, const void* pixels_host, int pixel_format, int64_t n,
                                     float* out_host, int normalize) {
  if (int rc = check_pixels("plip_encode_images_host", e, pixels_host, out_host, pixel_format, n, kImage, kImage))
    return rc;
  PLIP_CUDA_CHECK(cudaSetDevice(e->device));
  if (int rc = ensure_host_path(e)) return rc;
  PLIP_CUDA_CHECK(cudaStreamWaitEvent(e->s_compute, e->ev_last, 0));  // earlier device-API work owns the workspace
  const size_t pb = pixel_bytes(pixel_format);
  const int64_t chunk = e->max_mb;
  const size_t in_bytes = (size_t)(n < chunk ? n : chunk) * pb;
  if (e->d_in_bytes < in_bytes) {
    size_t have0 = e->d_in_bytes, have1 = e->d_in_bytes;
    if (int rc = grow_dev(&e->d_in[0], &have0, in_bytes)) return rc;
    if (int rc = grow_dev(&e->d_in[1], &have1, in_bytes)) return rc;
    e->d_in_bytes = in_bytes;
  }
  if (int rc = grow_dev(reinterpret_cast<void**>(&e->d_out), &e->d_out_bytes, (size_t)n * kProj * 4)) return rc;
  const bool pinned = is_pinned(pixels_host);
  if (!pinned && e->h_stage_bytes < in_bytes) {
    for (int i = 0; i < 2; ++i) {
      if (e->h_stage[i]) cudaFreeHost(e->h_stage[i]);
      e->h_stage[i] = nullptr;
      PLIP_CUDA_CHECK(cudaMallocHost(&e->h_stage[i], in_bytes));
    }
    e->h_stage_bytes = in_bytes;
  }
  int64_t ci = 0;
  for (int64_t i = 0; i < n; i += chunk, ++ci) {
    const int b = (int)(ci & 1);
    const int64_t mb = (n - i < chunk) ? (n - i) : chunk;
    const uint8_t* src = static_cast<const uint8_t*>(pixels_host) + (size_t)i * pb;
    if (ci >= 2) PLIP_CUDA_CHECK(cudaStreamWaitEvent(e->s_copy, e->ev_done[b], 0));  // device buffer b consumed
    if (!pinned) {
      if (ci >= 2) PLIP_CUDA_CHECK(cudaEventSynchronize(e->ev_copied[b]));  // staging buffer b drained
      memcpy(e->h_stage[b], src, (size_t)mb * pb);
      src = static_cast<const uint8_t*>(e->h_stage[b]);
    }
    PLIP_CUDA_CHECK(cudaMemcpyAsync(e->d_in[b], src, (size_t)mb * pb, cudaMemcpyHostToDevice, e->s_copy));
    PLIP_CUDA_CHECK(cudaEventRecord(e->ev_copied[b], e->s_copy));
    PLIP_CUDA_CHECK(cudaStreamWaitEvent(e->s_compute, e->ev_copied[b], 0));
    if (int rc = vision_pass(e, tiles(e->d_in[b], pixel_format), mb, VisGeom(),
                             embeds_only(e->d_out + i * kProj, normalize), e->prune_last != 0, e->s_compute)) return rc;
    PLIP_CUDA_CHECK(cudaEventRecord(e->ev_done[b], e->s_compute));
  }
  PLIP_CUDA_CHECK(cudaMemcpyAsync(out_host, e->d_out, (size_t)n * kProj * 4, cudaMemcpyDeviceToHost, e->s_compute));
  PLIP_CUDA_CHECK(cudaStreamSynchronize(e->s_compute));
  return 0;
}

PLIP_API int plip_encode_text_host(plip_engine_t* e, const void* ids_host, int ids_dtype, const void* attention_mask_host,
                                   int64_t n, int seq_len, float* out_host, int normalize) {
  if (int rc = check_ids("plip_encode_text_host", e, ids_host, out_host, ids_dtype, n, seq_len, seq_len)) return rc;
  PLIP_CUDA_CHECK(cudaSetDevice(e->device));
  if (int rc = ensure_host_path(e)) return rc;
  PLIP_CUDA_CHECK(cudaStreamWaitEvent(e->s_compute, e->ev_last, 0));
  const size_t isz = ids_dtype == PLIP_IDS_I64 ? 8 : 4;
  const size_t ib = (size_t)n * seq_len * isz;
  const size_t ib_al = (ib + 255) & ~(size_t)255;
  if (int rc = grow_dev(&e->d_aux, &e->d_aux_bytes, 2 * ib_al)) return rc;
  if (int rc = grow_dev(reinterpret_cast<void**>(&e->d_out), &e->d_out_bytes, (size_t)n * kProj * 4)) return rc;
  uint8_t* d_ids = static_cast<uint8_t*>(e->d_aux);
  uint8_t* d_mask = attention_mask_host ? d_ids + ib_al : nullptr;
  // Caption lengths (first EOS position + 1) scanned on the host: rows after the first EOS cannot influence the
  // pooled output (causal attention), so only that prefix of every row is processed — per length bucket when
  // the batch is large and its lengths differ enough to pay for extra passes (plan_text_buckets).
  PLIP_REQUIRE(n <= 0x7fffffff, "plip_encode_text_host: n too large");
  std::vector<int32_t> lens((size_t)n);
  for (int64_t b = 0; b < n; ++b) {
    int len = seq_len;
    for (int t = 0; t < seq_len; ++t) {
      const long long id = ids_dtype == PLIP_IDS_I64 ? static_cast<const long long*>(ids_host)[b * seq_len + t]
                                                     : (long long)static_cast<const int*>(ids_host)[b * seq_len + t];
      if (id == kEosId) { len = t + 1; break; }
    }
    lens[(size_t)b] = len;
  }
  std::vector<int32_t> perm((size_t)n);
  int32_t start[kMaxTextBuckets + 1], prefix[kMaxTextBuckets];
  const int nb = plan_text_buckets(lens.data(), n, seq_len, perm.data(), start, prefix, kMaxTextBuckets);
  if (nb == 1) {
    PLIP_CUDA_CHECK(cudaMemcpyAsync(d_ids, ids_host, ib, cudaMemcpyHostToDevice, e->s_compute));
    if (d_mask) PLIP_CUDA_CHECK(cudaMemcpyAsync(d_mask, attention_mask_host, ib, cudaMemcpyHostToDevice, e->s_compute));
    if (int rc = plip_encode_text_prefix(e, d_ids, ids_dtype, d_mask, n, seq_len, prefix[0], e->d_out, normalize,
                                         e->s_compute)) return rc;
    PLIP_CUDA_CHECK(cudaMemcpyAsync(out_host, e->d_out, (size_t)n * kProj * 4, cudaMemcpyDeviceToHost, e->s_compute));
    PLIP_CUDA_CHECK(cudaStreamSynchronize(e->s_compute));
    return 0;
  }
  // several buckets: upload the rows sorted by length, run each bucket with its own prefix, un-permute on the host
  const size_t row_bytes = (size_t)seq_len * isz;
  std::vector<uint8_t> sorted(ib);
  for (int64_t i = 0; i < n; ++i)
    memcpy(sorted.data() + (size_t)i * row_bytes, static_cast<const uint8_t*>(ids_host) + (size_t)perm[(size_t)i] * row_bytes,
           row_bytes);
  PLIP_CUDA_CHECK(cudaMemcpyAsync(d_ids, sorted.data(), ib, cudaMemcpyHostToDevice, e->s_compute));
  PLIP_CUDA_CHECK(cudaStreamSynchronize(e->s_compute));  // `sorted` is reused for the mask
  if (d_mask) {
    for (int64_t i = 0; i < n; ++i)
      memcpy(sorted.data() + (size_t)i * row_bytes,
             static_cast<const uint8_t*>(attention_mask_host) + (size_t)perm[(size_t)i] * row_bytes, row_bytes);
    PLIP_CUDA_CHECK(cudaMemcpyAsync(d_mask, sorted.data(), ib, cudaMemcpyHostToDevice, e->s_compute));
    PLIP_CUDA_CHECK(cudaStreamSynchronize(e->s_compute));
  }
  for (int k = 0; k < nb; ++k) {
    const int64_t r0 = start[k], cnt = start[k + 1] - start[k];
    if (cnt <= 0) continue;
    if (int rc = plip_encode_text_prefix(e, d_ids + (size_t)r0 * row_bytes, ids_dtype,
                                         d_mask ? d_mask + (size_t)r0 * row_bytes : nullptr, cnt, seq_len, prefix[k],
                                         e->d_out + r0 * kProj, normalize, e->s_compute)) return rc;
  }
  std::vector<float> tmp((size_t)n * kProj);
  PLIP_CUDA_CHECK(cudaMemcpyAsync(tmp.data(), e->d_out, (size_t)n * kProj * 4, cudaMemcpyDeviceToHost, e->s_compute));
  PLIP_CUDA_CHECK(cudaStreamSynchronize(e->s_compute));
  for (int64_t i = 0; i < n; ++i)
    memcpy(out_host + (size_t)perm[(size_t)i] * kProj, tmp.data() + (size_t)i * kProj, (size_t)kProj * 4);
  return 0;
}

PLIP_API int plip_dbg_text_bucket_plan(const int32_t* lens_host, int64_t n, int seq_len, int32_t* perm_host,
                                       int32_t* bucket_start_host, int32_t* bucket_prefix_host, int cap) {
  if (!lens_host || !bucket_start_host || !bucket_prefix_host || n <= 0 || seq_len < 1 || seq_len > kTxtSeq || cap < 1) {
    set_last_error("plip_dbg_text_bucket_plan: bad argument");
    return -2;
  }
  return plan_text_buckets(lens_host, n, seq_len, perm_host, bucket_start_host, bucket_prefix_host, cap);
}

// ---- per-kernel test hooks ------------------------------------------------------------------------
static int g_dbg_f16 = 0;  // operand format the handle-free hooks below run in
PLIP_API int plip_dbg_set_operand_format(int operand_format) {
  PLIP_REQUIRE(operand_format == PLIP_OPERAND_BF16 || operand_format == PLIP_OPERAND_FP16,
               "plip_dbg_set_operand_format: unknown operand format %d", operand_format);
  g_dbg_f16 = operand_format == PLIP_OPERAND_FP16 ? 1 : 0;
  return 0;
}

PLIP_API int plip_dbg_gemm(const void* A_bf16, int lda, const void* W_bf16, int ldw, int M, int N, int K,
                           const float* bias, void* out, int ldo, const float* pos, int epilogue, int cluster_size,
                           int block_n, const float* colsum, const float* stats_in, int n_partials, void* xb_out,
                           float* stats_out, void* stream) {
  GemmArgs g;
  g.A = static_cast<const __nv_bfloat16*>(A_bf16); g.lda = lda;
  g.W = static_cast<const __nv_bfloat16*>(W_bf16); g.ldw = ldw;
  g.M = M; g.N = N; g.K = K;
  g.bias = bias; g.out = out; g.ldo = ldo; g.pos = pos; g.epi = epilogue;
  g.colsum = colsum; g.stats_in = reinterpret_cast<const float2*>(stats_in); g.n_partials = n_partials;
  g.xb_out = static_cast<__nv_bfloat16*>(xb_out); g.stats_out = reinterpret_cast<float2*>(stats_out);
  g.force_cg = cluster_size; g.force_bn = block_n;
  g.f16 = g_dbg_f16;
  return launch_gemm(g, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_rowstats_cast(const float* x, int64_t rows, int dim, void* xb_bf16, float* stats, void* stream) {
  return launch_rowstats_cast(x, rows, dim, static_cast<__nv_bfloat16*>(xb_bf16), reinterpret_cast<float2*>(stats),
                              g_dbg_f16, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_layernorm(const float* x, int64_t rows, int dim, int64_t in_row_stride, const float* gamma,
                                const float* beta, float* out_f32, void* out_bf16, void* stream) {
  return launch_layernorm(x, nullptr, in_row_stride, rows, dim, gamma, beta, out_f32,
                          static_cast<__nv_bfloat16*>(out_bf16), g_dbg_f16, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_attention(const void* qkv_bf16, int64_t n_seq, int seq_len, int heads, int causal,
                                const int32_t* key_mask, void* out_bf16, void* stream) {
  return launch_attention(static_cast<const __nv_bfloat16*>(qkv_bf16), n_seq, seq_len, heads, causal != 0, key_mask,
                          static_cast<__nv_bfloat16*>(out_bf16), g_dbg_f16, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_attention_probs(const void* qkv_bf16, int64_t n_seq, int seq_len, int heads, int causal,
                                      const int32_t* key_mask, float* probs_dev, void* stream) {
  return launch_attention_probs(static_cast<const __nv_bfloat16*>(qkv_bf16), n_seq, seq_len, heads, causal != 0,
                                key_mask, probs_dev, g_dbg_f16, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_im2col(const void* pixels, int pixel_format, int64_t n, void* out_bf16, void* stream) {
  return launch_im2col(pixels, pixel_format, n, kImage, kImage, static_cast<__nv_bfloat16*>(out_bf16), g_dbg_f16,
                       static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_pos_interp(const float* pos_dev, int grid_h, int grid_w, float* out_dev, void* stream) {
  return launch_pos_interp(pos_dev, grid_h, grid_w, out_dev, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_hidden_states(plip_engine_t* e, int tower, const void* input_dev, int input_format,
                                    const void* attention_mask_dev, int64_t n, int num_layers, float* hidden_dev,
                                    void* stream) {
  return dbg_hidden_states("plip_dbg_hidden_states", e, tower, input_dev, input_format, attention_mask_dev, n, kImage,
                           kImage, num_layers, hidden_dev, static_cast<cudaStream_t>(stream));
}

PLIP_API int plip_dbg_hidden_states_hw(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n,
                                       int height, int width, int num_layers, float* hidden_dev, void* stream) {
  return dbg_hidden_states("plip_dbg_hidden_states_hw", e, 0, pixels_dev, pixel_format, nullptr, n, height, width,
                           num_layers, hidden_dev, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

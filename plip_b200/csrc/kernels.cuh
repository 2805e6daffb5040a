// plip_b200 — host-side launchers of the non-GEMM kernels.
#pragma once
#include "plip_b200.h"

#include "common.cuh"
#include "gemm.cuh"

namespace plip {

// elementwise.cu  (f16 = 1: 16-bit outputs are IEEE half instead of bfloat16; the pointer type stays a 16-bit tag)
// pixels: n images of height x width (224 x 224 unless the position table is interpolated) -> the patch matrix
// [n * gh * gw, 3072], gh = height / 32, gw = width / 32.
int launch_im2col(const void* pixels, int fmt, int64_t n, int height, int width, __nv_bfloat16* out, int f16,
                  cudaStream_t st);
// 224 x 224 windows of one uint8 RGB region [H, W, 3] with a row pitch in bytes.  origins: int32 (row, col) pairs, one
// per window, each window inside the region (the callers check that on the host).
struct WindowSrc {
  const uint8_t* region;
  int64_t pitch;
  const int32_t* origins;  // device memory, 8-byte aligned
};
// n windows -> the patch matrix [n * 49, 3072], bit-identical to launch_im2col of the same windows as u8 tiles.
int launch_window_im2col(const WindowSrc& win, int64_t n, __nv_bfloat16* out, int f16, cudaStream_t st);
// Per window, the pixels whose three channels are all >= threshold -> counts int32 [n].  origins_host: host memory,
// consumed before the call returns.
int launch_window_background(const uint8_t* region, int64_t pitch, const int32_t* origins_host, int64_t n,
                             int threshold, int32_t* counts, cudaStream_t st);
// Per window of a uint8 mask [H, W, channels] (channels 1 or 3), the elements > threshold -> counts int32 [n].
int launch_window_mask(const uint8_t* mask, int64_t pitch, int channels, const int32_t* origins_host, int64_t n,
                       int threshold, int32_t* counts, cudaStream_t st);
// The vision position table resized to a gh x gw patch grid: fp32 [1 + gh * gw, 768] (bicubic, as HF).
int launch_pos_interp(const float* pos, int gh, int gw, float* out, cudaStream_t st);
int launch_layernorm(const float* x, const int32_t* row_index, int64_t in_row_stride, int64_t rows, int dim,
                     const float* gamma, const float* beta, float* out_f32, __nv_bfloat16* out_bf16, int f16,
                     cudaStream_t st);
int launch_rowstats_cast(const float* x, int64_t rows, int dim, __nv_bfloat16* xb, float2* stats, int f16, cudaStream_t st);
int launch_text_embed(const void* ids, int ids_dtype, int64_t n, int seq_len, int ids_stride, const float* tok,
                      const float* pos, float* x, int32_t* eos_rows, int eos_id, int no_eos_argmax, cudaStream_t st);
int launch_mask_to_i32(const void* mask, int dtype, int64_t count, int seq_len, int stride, int32_t* out,
                       cudaStream_t st);
int launch_cls_rows(const float* cls, const float* pos, int64_t n, int seq, float* x, cudaStream_t st);
int launch_l2_normalize(float* x, int64_t rows, int dim, cudaStream_t st);
// rows idx(i) (= row_index[i], or i * row_stride) of a 16-bit [*, dim] and an fp32 [*, dim] matrix -> compact [n, dim]
int launch_gather_rows(const __nv_bfloat16* a16, const float* x32, const int32_t* row_index, int64_t row_stride,
                       int64_t n, int dim, __nv_bfloat16* a16_out, float* x32_out, cudaStream_t st);

// resize.cu: Pillow-exact bicubic resize + crop of packed RGB uint8 images into [n,224,224,3] tiles.
// bilinear: Pillow's triangle filter instead of its bicubic one (plip_resize_crop_bilinear_u8).
int launch_resize_crop(const uint8_t* src, size_t src_bytes, const plip_resize_desc_t* descs_host, int64_t n,
                       uint8_t* tiles, cudaStream_t st, bool bilinear = false);

int resize_filter_host(int in_size, int out_size, int xx, int32_t* k, int k_cap, int* xmin, int* count);
int resize_filter_bilinear_host(int in_size, int out_size, int xx, int32_t* k, int k_cap, int* xmin, int* count);
// The same resample over whole images at any shrink: output rows [o0, o1) of the new_h x new_w resize of an h x w RGB
// uint8 image, from the band of src_rows source rows starting at source row src_row0 (src points at that row).  out
// points at output row o0.  ws: a 16-byte aligned device workspace of resize_region_workspace bytes.  Every argument
// is checked before anything is launched.
int resize_region_workspace(int h, int w, int new_h, int new_w, int o0, int o1, uint64_t* bytes);
int launch_resize_region(const uint8_t* src, int64_t src_pitch, int src_row0, int src_rows, int h, int w, uint8_t* out,
                         int64_t out_pitch, int new_h, int new_w, int o0, int o1, uint8_t* ws, uint64_t ws_bytes,
                         cudaStream_t st);
// Per output index of one axis, its filter window: bounds[2 * xx] = first source index, bounds[2 * xx + 1] = count.
int resize_filter_bounds(int in_size, int out_size, int32_t* bounds);

// attention.cu: softmax(q k^T [+causal/padding mask]) v per (sequence, head); q pre-scaled by dh^-0.5.
// qkv: bf16 [n_seq*seq_len, 3*heads*64]; key_mask: optional int32 [n_seq, seq_len] (0 = masked key).
// seq_len > 128 (up to kMaxVisSeq) runs the long-sequence kernel: no causal mask, no key mask.
// f16 = 1: q, k, v, P and the output are IEEE half instead of bfloat16 (the engine's operand format).
int launch_attention(const __nv_bfloat16* qkv, int64_t n_seq, int seq_len, int heads, bool causal,
                     const int32_t* key_mask, __nv_bfloat16* out, int f16, cudaStream_t st);
// The softmax probabilities of the same call, fp32 [n_seq, heads, seq_len, seq_len] (output_attentions), for any
// seq_len <= kMaxVisSeq with any causal / key mask.  A row without a visible key is written as zeros.
int launch_attention_probs(const __nv_bfloat16* qkv, int64_t n_seq, int seq_len, int heads, bool causal,
                           const int32_t* key_mask, float* probs, int f16, cudaStream_t st);

// similarity.cu
int launch_similarity(const float* a, int64_t n, const float* b, int64_t m, float scale, bool norm_a, bool norm_b,
                      float* out, int64_t ldo, cudaStream_t st);
int launch_similarity_topk(const float* q, int64_t n, const float* s, int64_t m, float scale, bool norm_q,
                           bool norm_s, int k, int32_t* idx, float* val, cudaStream_t st);

// linear_probe.cu: sklearn's SGD logistic regression, one warp per binary problem, and the linear decision (the
// plip_sgd_* / plip_linear_decision contracts of plip_b200.h; every argument is checked before anything is launched).
int sgd_shuffle_permutation(int64_t n, uint32_t seed, int32_t* sigma);
int sgd_workspace_bytes(int64_t n, int n_sigma, int n_problems, uint64_t* bytes);
int launch_sgd_fit(const float* x, int64_t n, int dim, const int32_t* class_host, int n_classes,
                   const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host, int n_sigma,
                   int max_iter, double tol, int n_iter_no_change, float* coef, double* intercept, int32_t* n_iter,
                   int32_t* overflow, void* ws, uint64_t ws_bytes, cudaStream_t st);
int launch_linear_decision(const float* x, int64_t n, int dim, const float* coef, const double* intercept, int n_out,
                           float* scores, int32_t* pred, cudaStream_t st);

}  // namespace plip

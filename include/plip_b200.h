/*
 * plip_b200 — C ABI of the H100-native PLIP (CLIP ViT-B/32) inference engine.
 *
 * One shared library (libplip_b200.so, nvcc -gencode arch=compute_90a,code=sm_90a) exports
 * exactly the entry points below.  Plain pointers and sizes only: no torch / python types.
 *
 * The reference (PathologyFoundation/plip) has no FFI of its own — its hot path is the Python
 * call surface of a HuggingFace CLIPModel.  Each entry point therefore cites the reference /
 * transformers call it replaces ("TF:" = transformers/models/clip/modeling_clip.py, v5.5.0).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; plip_last_error() then holds a
 *     message (thread-local).  Nothing throws across the ABI.
 *   - *_dev pointers are device pointers owned by the caller; the engine owns packed weights and
 *     its workspace (allocated at plip_create, nothing is allocated on the hot path).
 *   - `stream` is a cudaStream_t passed as void*; all work is stream-ordered, the device-pointer
 *     entry points never synchronise the host.  One handle per device; calls on one handle share a
 *     workspace and are serialised on the device (each call waits, stream-side, for the previous one);
 *     a handle must not be used from two host threads at once.
 *   - device-pointer entry points launch on the CALLER'S current device: make the handle's device (or, for the
 *     handle-free functions, the device that owns the buffers) current first, as for any CUDA library call.  The
 *     *_host entry points select the handle's device themselves.
 */
#ifndef PLIP_B200_H_
#define PLIP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PLIP_API __attribute__((visibility("default")))

#define PLIP_B200_ABI_VERSION 5  /* 3: + plip_resize_crop_u8; 4: + plip_profile_*, plip_create_ex (operand format); 5: + plip_set_last_layer_pruning, later plip_*_hw, plip_*_outputs, plip_encode_windows, plip_window_background_counts, plip_window_mask_counts, plip_resize_region_*, plip_resize_filter_bounds, plip_sgd_*, plip_linear_decision, plip_densenet_*, plip_resize_crop_bilinear_u8, plip_warp_tiles_u8, plip_resize_crop_fill_u8, plip_mask_value_sets_u8, plip_encode_pair, plip_sgd_fit_f64, plip_linear_decision_f64, plip_dbg_layernorm_ex, plip_dbg_im2col_hw, plip_dbg_text_embed, plip_dbg_mask_to_i32, plip_dbg_cls_rows, plip_dbg_gather_rows, plip_weights_*_patch, plip_create_patch, plip_vision_patch, plip_dbg_im2col_patch, plip_dbg_window_im2col_patch, plip_dbg_pos_interp_patch (new symbols only) */

/* Model constants (TF:configuration_clip.py:47-64,97-109,160-161). */
#define PLIP_IMAGE_SIZE 224
#define PLIP_EMBED_DIM 512
#define PLIP_TEXT_SEQ 77
#define PLIP_VOCAB 49408

typedef struct plip_engine plip_engine_t;

/* ---- pixel formats accepted by plip_encode_images ------------------------------------------ */
enum plip_pixel_format {
  PLIP_PIX_F32_NCHW = 0, /* CLIPProcessor output: normalised float32 [n,3,224,224] (plip.py:35,49) */
  PLIP_PIX_BF16_NCHW = 1, /* same, bfloat16 */
  PLIP_PIX_U8_NHWC = 2   /* raw RGB tiles uint8 [n,224,224,3]; (x/255-mean)/std fused on device
                            (TF:image_processing_clip.py:50-62, embedders/transform.py:51) */
};

enum plip_id_dtype { PLIP_IDS_I32 = 0, PLIP_IDS_I64 = 1 };

/* 16-bit format of every GEMM / attention OPERAND (packed weights, activations between kernels).  Accumulation, the
 * residual stream, LayerNorm statistics, softmax and the similarity head are float32 in both.  wgmma
 * runs both at the same rate.  BF16 is the default (BASELINE.json's dtype).  FP16 keeps 3 more significand bits:
 * end-to-end |dlogits_per_image| is 6-8x smaller (tools/precision_study.py) — the reference's own OpenAI-clip
 * flavour runs fp16 weights on the GPU (scripts/extract_embedding.py:94-97) — at the price of a 65504 range. */
enum plip_operand_format { PLIP_OPERAND_BF16 = 0, PLIP_OPERAND_FP16 = 1 };

/* ---- errors / version ---------------------------------------------------------------------- */
PLIP_API const char* plip_last_error(void);
PLIP_API int plip_abi_version(void);
/* Kernel launches issued by the library so far (bench.py's gpu_launches accounting). */
PLIP_API uint64_t plip_launch_count(void);

/* ---- packed weights ------------------------------------------------------------------------ */
/* The engine consumes ONE contiguous host blob.  Its layout is defined by the library and
 * queried by the host-side packer (plip_b200/weights.py), which fills it from a HuggingFace
 * CLIPModel state dict (names listed in SURVEY.md §8a) or an OpenAI-clip state dict.
 * Replaces CLIPModel.from_pretrained / load_state_dict (plip.py:26, embedders/factory.py:21-25). */
typedef struct plip_tensor_info {
  char name[96];    /* HuggingFace-style name, e.g. "vision_model.encoder.layers.0.mlp.fc1.weight" */
  uint64_t offset;  /* byte offset inside the blob (256-byte aligned) */
  uint64_t numel;
  int32_t dtype;    /* 0 = float32, 1 = 16-bit operand (bfloat16, or IEEE half for a PLIP_OPERAND_FP16 engine) */
  int32_t rows;     /* logical 2-D shape (rows x cols), cols == 1 for vectors */
  int32_t cols;
  int32_t fused;    /* 0 = plain copy of the named tensor.
                       bit 0 (1): q/k/v rows concatenated — name holds the q tensor, k and v follow
                         ("...q_proj" -> k_proj, v_proj); the q rows are pre-scaled by head_dim^-0.5 = 0.125.
                       bit 1 (2): the preceding LayerNorm (layer_norm1 for q_proj, layer_norm2 for fc1;
                         TF:371,380) is folded in: weight' = bf16(gamma o W), bias' = bias + W beta, and the
                         pseudo-tensor "<...>.colsum"[n] = sum_k float(weight'[n,k]); the kernels then compute
                         rstd_r * (x_bf16 . weight'_n - mean_r * colsum_n) + bias'_n  ==  LN(x) . W_n + bias_n. */
} plip_tensor_info_t;

PLIP_API int plip_weights_num_tensors(void);
PLIP_API int plip_weights_tensor_info(int index, plip_tensor_info_t* info);
PLIP_API uint64_t plip_weights_blob_bytes(void);
/* The layout above is CLIP ViT-B/32's (PLIP).  The same for a vision patch size: 32 (the functions above) or 16
 * (CLIP ViT-B/16: the same tensors in the same order; only patch_embedding.weight [768, 768] and
 * position_embedding.weight [197, 768] differ, so every offset after the first differs too).
 * plip_weights_num_tensors() holds for both.  blob_bytes_patch returns 0 for another patch size. */
PLIP_API int plip_weights_tensor_info_patch(int patch, int index, plip_tensor_info_t* info);
PLIP_API uint64_t plip_weights_blob_bytes_patch(int patch);

/* ---- engine lifetime ----------------------------------------------------------------------- */
/* host_blob: packed weights (layout above), plus exp(logit_scale) passed separately.
 * max_micro_batch: largest number of images / captions processed per internal pass; larger calls
 * are looped in micro-batches.  Device memory: blob + plip_workspace_bytes(max_micro_batch), and from the first
 * plip_encode_pair call that runs both towers at once a second, text-only workspace (the text tower's activations
 * while the vision tower's occupy the first): about 0.87 MB per unit of max_micro_batch, 0.9 GB at 1024. */
PLIP_API int plip_create(const void* host_blob, uint64_t blob_bytes, float logit_scale_exp, int device,
                         int max_micro_batch, plip_engine_t** out);
/* Same with an explicit operand format: the 16-bit entries of host_blob must have been packed in that format. */
PLIP_API int plip_create_ex(const void* host_blob, uint64_t blob_bytes, float logit_scale_exp, int device,
                            int max_micro_batch, int operand_format, plip_engine_t** out);
/* Same for the vision patch size of the weights: 32 (ViT-B/32, = plip_create_ex) or 16 (ViT-B/16, blob in the
 * plip_weights_tensor_info_patch(16, ...) layout).  Every vision call of the engine uses that patch size: images of
 * H x W pixels have (H / P) * (W / P) patches (196 at 224 x 224 for P = 16, 197 tokens), at most 32 per side, and a
 * micro-batch holds floor(50 * max_micro_batch / S) images of S tokens (259 of 197 tokens at 1024), so a ViT-B/16
 * engine needs max_micro_batch >= 4. */
PLIP_API int plip_create_patch(const void* host_blob, uint64_t blob_bytes, float logit_scale_exp, int device,
                               int max_micro_batch, int operand_format, int vision_patch, plip_engine_t** out);
PLIP_API int plip_destroy(plip_engine_t* e);
PLIP_API uint64_t plip_workspace_bytes(int max_micro_batch);
PLIP_API float plip_logit_scale_exp(const plip_engine_t* e);
PLIP_API int plip_max_micro_batch(const plip_engine_t* e);
PLIP_API int plip_operand_format(const plip_engine_t* e);
/* The engine's vision patch size (32 or 16; 0 for a NULL handle). */
PLIP_API int plip_vision_patch(const plip_engine_t* e);
/* Pooled position of a caption WITHOUT an eos token (49407).  0 (default): position 0, as transformers does for
 * configs with eos_token_id == 49407 (TF:571-584: argmax of an all-zero match vector).  1: first position of the
 * largest id, as legacy configs (eos_token_id == 2 — what openai/clip-vit-base-patch32 ships) and OpenAI clip's
 * text.argmax(-1) do (TF:564-570).  Captions that contain an eos are pooled at its first position either way. */
PLIP_API int plip_set_text_pooling(plip_engine_t* e, int no_eos_argmax);
/* Last-layer pruning for the embedding calls (default 0 = off).  Only the pooled row of a sequence leaves a tower
 * (CLS: TF:685-686; first eos: TF:571-584), and after the last layer's attention rows no longer interact, so with
 * on != 0 plip_encode_* / plip_clip_forward* run that layer's out_proj, LayerNorm 2 and MLP on the n pooled rows
 * instead of all n*seq rows: the embeddings are the same (same per-row arithmetic), the step is ~5 % shorter at
 * batch 1024 and more for small batches.  plip_hidden_states is never pruned.  plip_last_layer_pruning reads it back. */
PLIP_API int plip_set_last_layer_pruning(plip_engine_t* e, int on);
PLIP_API int plip_last_layer_pruning(const plip_engine_t* e);

/* ---- the hot path -------------------------------------------------------------------------- */
/* Vision tower + visual_projection: replaces CLIPModel.get_image_features (TF:829-863, called at
 * plip.py:50) and OpenAI-clip model.encode_image (embedders/plip.py:48).
 * out_dev: float32 [n,512]; normalize != 0 divides each row by its L2 norm (TF:57-65,923). */
PLIP_API int plip_encode_images(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n,
                                float* out_dev, int normalize, void* stream);

/* Same at any image size: CLIPModel.get_image_features(pixel_values, interpolate_pos_encoding=True) (TF:161-218,
 * 832-856).  pixels_dev holds n images of height x width in pixel_format ([n,3,H,W] or [n,H,W,3] for u8).  The patch
 * grid is gh = height / 32 by gw = width / 32 (remainder pixels on the right and bottom are ignored, as by the
 * stride-32 conv), S = gh * gw + 1 tokens, and the 7 x 7 position table is resized to gh x gw bicubically (A = -0.75,
 * align_corners = False, as F.interpolate).  Requires 32 <= height, width and gh, gw <= 32 (up to 1024 pixels per side),
 * and S <= 50 * max_micro_batch (the workspace's token rows): a pass holds min(max_micro_batch,
 * floor(50 * max_micro_batch / S)) images.  A 7 x 7 grid uses the stored table, so 224 <= height, width <= 255 give
 * exactly the 224 x 224 result; 224 x 224 is plip_encode_images itself.  Sequences longer than 128 tokens (more than
 * 8 x 16 patches) run the long-sequence attention kernel (profile role "vision/attention[long]"). */
PLIP_API int plip_encode_images_hw(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n, int height,
                                   int width, float* out_dev, int normalize, void* stream);

/* ---- windows of a slide region --------------------------------------------------------------- */
/* region_dev: one uint8 RGB region [height, width, 3], rows row_pitch_bytes apart (>= 3 * width; a view into a wider
 * array is fine, no alignment is required).  origins_host: HOST int32 [n, 2] (row, col) of n 224 x 224 windows, each
 * inside the region (0 <= row <= height - 224, 0 <= col <= width - 224); all are checked before anything is launched and
 * the error names the first bad window.  The origins are consumed before the call returns (copied from pageable memory,
 * which may wait for the stream's earlier work, as cudaMemcpyAsync does).  This is the crop loop of the reference's
 * slide preprocessing (reproducibility/generate_validation_datasets/preprocess/preprocess_DigestPath.py:28-100) without
 * cutting the crops out: the windows are read in place.
 *
 * plip_encode_windows: out_dev float32 [n,512] in window order, exactly what plip_encode_images returns for the same
 * windows cut out as PLIP_PIX_U8_NHWC tiles in the same order (same micro-batches, same 67 launches per micro-batch,
 * bit for bit); normalize as there.  The window gather runs under the profile role "vision/im2col".  Never replayed
 * as a CUDA graph.
 * plip_window_background_counts (no engine): counts_dev int32 [n], per window the pixels whose three channels are all
 * >= threshold — the reference's background_ratio(window, threshold) times 224 * 224, exactly. */
PLIP_API int plip_encode_windows(plip_engine_t* e, const void* region_dev, int height, int width,
                                 int64_t row_pitch_bytes, const int32_t* origins_host, int64_t n, float* out_dev,
                                 int normalize, void* stream);
PLIP_API int plip_window_background_counts(const void* region_dev, int height, int width, int64_t row_pitch_bytes,
                                           const int32_t* origins_host, int64_t n, int threshold, int32_t* counts_dev,
                                           void* stream);
/* plip_window_mask_counts (no engine): mask_dev is a uint8 mask [height, width] (channels = 1) or [height, width, 3]
 * (channels = 3), rows row_pitch_bytes apart (>= channels * width); origins as above.  counts_dev int32 [n]: per
 * window, the mask elements > threshold, every channel counted — the reference's (msk_np > 10) followed by
 * np.sum(msk_patch_np > 0).  Its tumour ratios divide by 224 * 224 whatever the channel count, so an RGB mask can give
 * a ratio above 1; that is kept. */
PLIP_API int plip_window_mask_counts(const void* mask_dev, int height, int width, int channels,
                                     int64_t row_pitch_bytes, const int32_t* origins_host, int64_t n, int threshold,
                                     int32_t* counts_dev, void* stream);

/* Text tower + text_projection: replaces CLIPModel.get_text_features (TF:793-825, called at
 * plip.py:68) and model.encode_text (embedders/plip.py:66).
 * ids_dev: [n,seq_len] token ids (seq_len <= 77); attention_mask_dev: optional [n,seq_len] of the
 * same dtype (0 = padded key), NULL = no padding mask.  Pooling takes the row of the first
 * eos_token_id (49407), as TF:571-584. */
PLIP_API int plip_encode_text(plip_engine_t* e, const void* ids_dev, int ids_dtype,
                              const void* attention_mask_dev, int64_t n, int seq_len, float* out_dev,
                              int normalize, void* stream);

/* Same, processing only the first prefix_len (<= seq_len) positions of every row.  The pooled output of a
 * caption depends only on positions up to its first eos (causal attention, TF:546-557,571-584), so with
 * prefix_len >= (longest first-eos position + 1) the result equals plip_encode_text at prefix_len/seq_len of
 * the work — what typical prompts ("An H&E image patch of ...", ~12 of 77 tokens) need. */
PLIP_API int plip_encode_text_prefix(plip_engine_t* e, const void* ids_dev, int ids_dtype,
                                     const void* attention_mask_dev, int64_t n, int seq_len, int prefix_len,
                                     float* out_dev, int normalize, void* stream);

/* Both towers: n_img 224 x 224 images (plip_encode_images' formats) -> img_out_dev [n_img,512] and n_txt captions
 * (plip_encode_text's arguments) -> txt_out_dev [n_txt,512], bit for bit what those two calls return.  When each side
 * fits one micro-batch and is larger than the graph-replayed small batches (PLIP_GRAPH_MAX), the text tower runs on
 * the engine's own stream and workspace at the same time as the vision tower on `stream`, so each tower's kernels fill
 * the SMs the other's leave idle at kernel tails and between launches; `stream` waits for both.  Otherwise it makes
 * the two calls, text first. */
PLIP_API int plip_encode_pair(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n_img,
                              const void* ids_dev, int ids_dtype, const void* attention_mask_dev, int64_t n_txt,
                              int seq_len, float* img_out_dev, float* txt_out_dev, int normalize, void* stream);

/* ---- per-token outputs: output_hidden_states / output_attentions ------------------------------ */
/* Device buffers (float32, caller-owned) filled by ONE pass of a tower: CLIPModel.vision_model(...) /
 * text_model(..., output_hidden_states=True, output_attentions=True) (TF:modeling_clip.py:477-507, 531-589, 667-691).
 * Every pointer is optional (NULL = not computed), but at least one must be set.  S is the sequence length (vision:
 * (height / 32) * (width / 32) + 1; text: seq_len), D the tower width (768 / 512), heads 12 / 8.
 *   embeds       [n,512]  projected pooled row (what plip_encode_* returns); normalize != 0 L2-normalises it
 *   pooled       [n,D]    pooler_output: vision post_layernorm(CLS row); text final_layer_norm(pooled row)
 *   last_hidden  [n,S,D]  vision: residual stream after the last layer (before post_layernorm);
 *                         text: final_layer_norm of every row
 *   hidden       [13,n,S,D]  hidden_states: [0] the encoder input (vision: after pre_layrnorm; text: token + position
 *                         embeddings), [l] the residual stream after layer l
 *   attn         [12,n,heads,S,S]  attentions: softmax(q k^T / 8 + mask) in fp32; masked keys are exactly 0, and a row
 *                         without any visible key (text whose position 0 is padded) is all zeros
 * These calls never replay CUDA graphs and never prune the last layer; the embeds equal plip_encode_* with pruning
 * off bit for bit.  attn is large: heads * S^2 * 4 bytes per sequence and layer (120 KB at 224 x 224, 50 MB at
 * 1024 x 1024).  Profile role of the probabilities kernel: "<tower>/attention[probs]". */
typedef struct plip_tower_outputs {
  float* embeds;
  float* pooled;
  float* last_hidden;
  float* hidden;
  float* attn;
  int32_t normalize;
} plip_tower_outputs_t;
/* Vision at any size accepted by plip_encode_images_hw (224 x 224 included), micro-batched the same way. */
PLIP_API int plip_vision_outputs(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n, int height,
                                 int width, const plip_tower_outputs_t* outputs, void* stream);
/* Text: ids / mask as plip_encode_text; all seq_len positions are processed. */
PLIP_API int plip_text_outputs(plip_engine_t* e, const void* ids_dev, int ids_dtype, const void* attention_mask_dev,
                               int64_t n, int seq_len, const plip_tower_outputs_t* outputs, void* stream);

/* Similarity head: logits_per_image[n,m] = scale * norm(img)[n,512] . norm(txt)[m,512]^T
 * (TF:923-930; numpy versions at plip.py:73-76, evaluation/zero_shot/zero_shot.py:12,
 * evaluation/retrieval/retrieval.py:14).  normalize_img / normalize_txt select which side is
 * L2-normalised on the fly (PLIP._cosine_similarity normalises only the key side). */
PLIP_API int plip_similarity(const float* img_dev, int64_t n, const float* txt_dev, int64_t m, float scale,
                             int normalize_img, int normalize_txt, float* logits_dev, int64_t ld_logits,
                             void* stream);

/* Fused similarity + top-k over the second operand (k <= 64), never materialising [n,m]:
 * idx_dev int32 [n,k] (descending score), val_dev float32 [n,k] (may be NULL).
 * Replaces np.argmax (plip.py:102, zero_shot.py:13) and argsort()[:, -k:][:, ::-1]
 * (plip.py:85, retrieval.py:16). */
PLIP_API int plip_similarity_topk(const float* query_dev, int64_t n, const float* space_dev, int64_t m,
                                  float scale, int normalize_query, int normalize_space, int k,
                                  int32_t* idx_dev, float* val_dev, void* stream);

/* L2-normalise rows in place (embedders/plip.py:53,73). */
PLIP_API int plip_l2_normalize(float* x_dev, int64_t n, int dim, void* stream);

/* Image preparation on the device: n variable-size RGB uint8 images (HWC, rows packed, image i at byte
 * descs[i].offset of src_dev) -> tiles_dev uint8 [n,224,224,3] (the PLIP_PIX_U8_NHWC input of
 * plip_encode_images).  Image i is resized to new_width x new_height with Pillow's antialiased bicubic filter
 * and the 224x224 window at (left, top) of the resized image is kept — bit-identical to
 * PIL.Image.resize((new_width,new_height), BICUBIC).crop(...), i.e. to what CLIPProcessor's resize +
 * center_crop (plip.py:35; TF:models/clip/image_processing_clip.py:50-62) and torchvision's
 * Resize(224, BICUBIC) + CenterCrop(224) (reproducibility/embedders/transform.py:45-52) produce before their
 * float conversion.  descs_host is a HOST array (the caller knows the sizes from decoding); it is consumed
 * before the call returns.  src_dev / tiles_dev are device pointers; stream-ordered, no synchronisation. */
typedef struct plip_resize_desc {
  int64_t offset;                 /* byte offset of the image in src_dev */
  int32_t width, height;          /* source size */
  int32_t new_width, new_height;  /* size after the resize (each >= 224) */
  int32_t left, top;              /* crop origin in the resized image */
} plip_resize_desc_t;
PLIP_API int plip_resize_crop_u8(const void* src_dev, uint64_t src_bytes, const plip_resize_desc_t* descs_host,
                                 int64_t n, void* tiles_dev, void* stream);
/* Same with Pillow's bilinear filter (triangle, support 1; the same ImagingResample): bit-identical to
 * PIL.Image.resize((new_width,new_height), BILINEAR).crop(...), i.e. torchvision's Resize(224) (BILINEAR, its default)
 * + CenterCrop(224) on a PIL image, the MuDiPath transform (reproducibility/embedders/factory.py:41-46) before ToTensor.
 * Accepts exactly the descriptors plip_resize_crop_u8 accepts. */
PLIP_API int plip_resize_crop_bilinear_u8(const void* src_dev, uint64_t src_bytes, const plip_resize_desc_t* descs_host,
                                          int64_t n, void* tiles_dev, void* stream);
/* The bicubic resize with the crop window anywhere: new_width / new_height may be 1..65536 and left / top any int32.
 * Tile pixel (x, y) is the resized image's pixel (left + x, top + y) when that lies inside it, else (0, 0, 0) —
 * bit-identical to PIL.Image.resize((new_width,new_height), BICUBIC).crop((left, top, left + 224, top + 224)), which is
 * what the reference's evaluation-tile resize (generate_validation_datasets/prepare_dataset_to_csv.py:40-63,
 * resizeimg) saves for an RGB image.  Rows of the tile entirely outside the resized image read no source.  A
 * descriptor whose filter tables and strip do not fit the kernel's 200 KB shared-memory plan (shrinks of roughly 25x
 * and more; the error names the image and its sizes) is rejected, like every other invalid argument, before anything
 * is launched.  Same call shape and stream semantics as plip_resize_crop_u8. */
PLIP_API int plip_resize_crop_fill_u8(const void* src_dev, uint64_t src_bytes, const plip_resize_desc_t* descs_host,
                                      int64_t n, void* tiles_dev, void* stream);

/* The distinct byte values of every (image, channel) of a device uint8 array masks_dev [n, height, width, channels]
 * (C order, channels 1..8, height * width * channels < 2^31, 16-byte aligned): sets_dev uint32 [n, channels, 8], bit
 * (v & 31) of word (v >> 5) set iff value v occurs in that channel of that image.  The call zeroes sets_dev itself.
 * len(np.unique(masks[i, ..., j])) is the set's popcount, and masks[i, ..., j] is all zero iff the set is exactly {0}
 * (the reference's PanNuke labelling, generate_validation_datasets/preprocess/preprocess_PanNuke.py:39,56-59).  One
 * pass over the array, which is read once; every argument is checked before anything is launched.  Stream-ordered,
 * allocates nothing. */
PLIP_API int plip_mask_value_sets_u8(const void* masks_dev, int64_t n, int height, int width, int channels,
                                     uint32_t* sets_dev, void* stream);

/* The geometric steps of torchvision's RandomHorizontalFlip, RandomAffine(BILINEAR, fill) and
 * RandomPerspective(BILINEAR, fill) on PIL images, the train-time transform of the reference
 * (reproducibility/embedders/transform.py:18-42), on n RGB uint8 tiles [n,224,224,3]: tile i is mirrored
 * left-right when descs[i].flip, then warped with PIL.Image.transform((224,224), AFFINE, affine, BILINEAR,
 * fillcolor=(fill,)*3), then, when descs[i].apply_perspective, with Image.transform(..., PERSPECTIVE, perspective,
 * BILINEAR, fillcolor=(fill,)*3) of that uint8 result — bit-identical to Pillow (IEEE double without FMA, results
 * truncated to uint8).  The coefficients are Pillow's: the map from an output pixel centre to the source point
 * (torchvision's inverse affine matrix and its float32 perspective coefficients).  src_dev / dst_dev: device tiles,
 * 16-byte aligned, the same buffer (in place) or not overlapping.  descs_host: HOST array, consumed before the call
 * returns.  Every argument is checked before anything is launched (n > 0, pointers, flags 0 / 1, fill 0..255, finite
 * coefficients; the perspective ones when applied); an error names the offending value.  Stream-ordered. */
typedef struct plip_warp_desc {
  double affine[6];           /* source x = a0*x + a1*y + a2, y = a3*x + a4*y + a5 at pixel centres (x+0.5, y+0.5) */
  double perspective[8];      /* x = (a0*x + a1*y + a2) / (a6*x + a7*y + 1), y = (a3*x + a4*y + a5) / (same) */
  int32_t flip;               /* 1: mirror the columns before the affine warp */
  int32_t apply_perspective;  /* 1: run the perspective warp after the affine one */
  int32_t fill;               /* 0..255: every channel of a pixel whose source point lies outside the tile */
  int32_t reserved;           /* 0 */
} plip_warp_desc_t;
PLIP_API int plip_warp_tiles_u8(const void* src_dev, void* dst_dev, const plip_warp_desc_t* descs_host, int64_t n,
                                void* stream);

/* Whole-image resize on the device, bit-identical to PIL.Image.fromarray(src).resize((new_width, new_height)) (BICUBIC,
 * no reducing_gap) for any ratio from upscaling to shrinks of over 64x (the horizontal filter must fit 64 columns in
 * 200 KB of shared memory: about 200x).  The source is a height x width RGB uint8 image, the output new_height x
 * new_width; sizes 1..65536.  The call writes output rows [out_row0, out_row1) and reads only the source rows their
 * vertical filter windows cover; the filters are always those of the full image, so ranges stitched together equal
 * the whole image.
 *   src_dev: source row src_row0 of the image; src_rows rows are readable from there, src_row_pitch bytes apart
 *            (>= 3 * width, no alignment needed): a band of a larger image, or the whole image (0, height).
 *   out_dev: output row out_row0, rows out_row_pitch bytes apart (>= 3 * new_width).
 *   workspace_dev: 16-byte aligned device memory of at least plip_resize_region_workspace(...) bytes (filter tables
 *            and the uint8 intermediate image of Pillow's horizontal pass); the call allocates nothing.
 * Every argument is checked before anything is launched, including that the band holds the source rows the output
 * rows read; an error names the offending value.  Stream-ordered, three launches. */
PLIP_API int plip_resize_region_workspace(int height, int width, int new_height, int new_width, int out_row0,
                                          int out_row1, uint64_t* bytes);
PLIP_API int plip_resize_region_u8(const void* src_dev, int64_t src_row_pitch, int src_row0, int src_rows, int height,
                                   int width, void* out_dev, int64_t out_row_pitch, int new_height, int new_width,
                                   int out_row0, int out_row1, void* workspace_dev, uint64_t workspace_bytes,
                                   void* stream);
/* Host-only: the filter window of every output index of one resize axis (in_size -> out_size, 1..65536), as the
 * kernels compute it: bounds_host int32 [out_size][2] = (first source index, count).  Output index i reads source
 * indices [first, first + count). */
PLIP_API int plip_resize_filter_bounds(int in_size, int out_size, int32_t* bounds_host);

/* ---- linear probe: scikit-learn's SGD logistic regression (no engine) ------------------------- */
/* The reference's linear probe (reproducibility/evaluation/linear_probing/linear_classifier.py) fits
 * SGDClassifier(loss="log_loss", penalty="l2", class_weight="balanced", learning_rate="optimal") on [n,512] (PLIP,
 * CLIP; float16 when the reference embeds on a GPU) or [n,1024] (MuDiPath's DenseNet-121) embeddings: one-vs-rest
 * binary problems, each a sequential pass of sklearn 1.9's _plain_sgd over a shuffled order per epoch.  plip_sgd_fit
 * runs its 32-bit instantiation (float32 input), plip_sgd_fit_f64 its 64-bit one (float16 / float64 input), cast for
 * cast, for many binary problems at once (every class of a fit, every alpha of a sweep): one warp per problem runs all
 * its epochs on the device.  The results equal sklearn's up to the order of the D-term double
 * sums (D = dim) and CUDA's exp / log1p against the C library's.
 *
 * One binary problem: labels y = (class_host[i] == pos_class), positive / negative sample weight pos_weight /
 * neg_weight (rounded to float by plip_sgd_fit, kept in double by plip_sgd_fit_f64, as sklearn's class_weight
 * local), regularisation alpha (> 0, finite), t starting at 1,
 * and the epoch order order_e[i] = order_{e-1}[sigma[i]] (order_0 = identity) with sigma row sigma_index of
 * sigma_host: the permutation sklearn's dataset.shuffle(seed) applies every epoch (plip_sgd_shuffle_permutation). */
typedef struct plip_sgd_problem {
  double alpha;
  double pos_weight;
  double neg_weight;
  int32_t pos_class;
  int32_t sigma_index;
} plip_sgd_problem_t;
/* Host-only: sklearn's Fisher-Yates shuffle (utils/_seq_dataset.pyx.tp, our_rand_r xorshift, j = i + r % (n - i))
 * applied to the identity: sigma_host int32 [n].  1 <= n < 2^31; seed 0 behaves as our_rand_r's default 1. */
PLIP_API int plip_sgd_shuffle_permutation(int64_t n, uint32_t seed, int32_t* sigma_host);
/* Device workspace bytes of plip_sgd_fit and plip_sgd_fit_f64 (problem table, labels, sigma rows and two epoch orders
 * per problem); one size serves both precisions. */
PLIP_API int plip_sgd_workspace_bytes(int64_t n, int n_sigma, int n_problems, uint64_t* bytes);
/* x_dev: device float32 [n,dim], dim = 512 or 1024, rows contiguous, 16-byte aligned; 2 <= n < 2^31.  class_host:
 * HOST int32 [n] class ids in 0..n_classes-1.  problems_host: HOST [n_problems].  sigma_host: HOST int32 [n_sigma, n], every entry in 0..n-1.
 * Host arrays are consumed before the call returns.  max_iter >= 1 epochs; an epoch whose mean objective exceeds the
 * best so far minus tol counts towards n_iter_no_change (>= 1) epochs without improvement, which stop the problem
 * (tol = -INFINITY disables the test).  Outputs (device): coef_dev float32 [n_problems,dim], intercept_dev float64
 * [n_problems], n_iter_dev int32 [n_problems] (epochs run), overflow_dev int32 [n_problems]: 1 if the weights or the
 * intercept were not finite at the end of epoch n_iter (sklearn raises there; coef / intercept are then undefined).
 * workspace_dev: 16-byte aligned device memory of at least plip_sgd_workspace_bytes(n, n_sigma, n_problems); the call
 * allocates nothing.  Every argument is checked before anything is launched; an error names the offending value.
 * Stream-ordered, one launch. */
PLIP_API int plip_sgd_fit(const float* x_dev, int64_t n, int dim, const int32_t* class_host, int n_classes,
                          const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host,
                          int n_sigma, int max_iter, double tol, int n_iter_no_change, float* coef_dev,
                          double* intercept_dev, int32_t* n_iter_dev, int32_t* overflow_dev, void* workspace_dev,
                          uint64_t workspace_bytes, void* stream);
/* decision_function and predict of a fitted linear classifier: scores_dev float32 [n, n_out] = x . coef^T + intercept
 * (products and sums in double, rounded once), pred_dev int32 [n]: n_out > 1, the first index of the largest score;
 * n_out == 1, 1 where the score is > 0, else 0.  x_dev float32 [n,dim] and coef_dev float32 [n_out,dim] (dim =
 * 512 or 1024) 16-byte aligned, intercept_dev float64 [n_out].  Stream-ordered, one launch. */
PLIP_API int plip_linear_decision(const float* x_dev, int64_t n, int dim, const float* coef_dev,
                                  const double* intercept_dev, int n_out, float* scores_dev, int32_t* pred_dev,
                                  void* stream);
/* The 64-bit instantiation of _plain_sgd, which sklearn runs on float64 input and on float16 input (its check_array
 * widens anything that is not float32 to float64): WeightVector64's double weights, dot returning the double
 * sum * wscale unrounded, scale and add taking double coefficients, the wscale reset below 1e-9 (not 1e-6), and
 * pos_weight / neg_weight kept in double.  Same arguments and contract as plip_sgd_fit, with x_dev float64 [n,dim]
 * (float16 embeddings widened exactly by the caller) and coef_dev float64 [n_problems,dim]; the same workspace
 * (plip_sgd_workspace_bytes).  The results equal sklearn's up to the order of the D-term double sums (dot and sum(w^2)
 * are reduced per lane, then across the warp; sklearn sums in index order) and CUDA's exp / log1p. */
PLIP_API int plip_sgd_fit_f64(const double* x_dev, int64_t n, int dim, const int32_t* class_host, int n_classes,
                              const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host,
                              int n_sigma, int max_iter, double tol, int n_iter_no_change, double* coef_dev,
                              double* intercept_dev, int32_t* n_iter_dev, int32_t* overflow_dev, void* workspace_dev,
                              uint64_t workspace_bytes, void* stream);
/* decision_function and predict in float64: scores_dev float64 [n, n_out] = x . coef^T + intercept (double products and
 * sums), pred_dev int32 [n] by plip_linear_decision's rule.  x_dev float64 [n,dim] and coef_dev float64 [n_out,dim]
 * (dim = 512 or 1024) 16-byte aligned, intercept_dev float64 [n_out].  Stream-ordered, one launch. */
PLIP_API int plip_linear_decision_f64(const double* x_dev, int64_t n, int dim, const double* coef_dev,
                                      const double* intercept_dev, int n_out, double* scores_dev, int32_t* pred_dev,
                                      void* stream);

/* ---- MuDiPath DenseNet-121 image embedder (separate handle) ----------------------------------- */
/* The reference's third embedder (reproducibility/embedders/factory.py:34-47, mudipath.py:125-130,205-215): torchvision's
 * DenseNet-121 features (growth 32, bottleneck 128, blocks 6/12/24/16) in eval mode, then a global average pool; no
 * final ReLU, no classifier.  Output: the un-normalised pooled features, float32 [n,1024].
 * Weights: ONE host blob whose layout the library defines (plip_densenet_tensor_info, same struct as the CLIP blob,
 * fused always 0): "<torchvision name>.weight" entries are bfloat16 (dtype 1), conv0 [64,160] with K = (ky,kx,c) and
 * columns 147..159 zero, conv1 [128,C_in], conv2 [32,1152] with K = (ky,kx,c), transition conv [C/2,C];
 * "<bn name>.scale" / ".shift" are float32 [C]: the eval BatchNorm as y = x * scale + shift
 * (scale = gamma / sqrt(running_var + 1e-5), shift = beta - running_mean * scale).
 * Device memory: blob + plip_densenet_workspace_bytes(max_micro_batch) (about 5.3 MB per image). */
typedef struct plip_densenet plip_densenet_t;
PLIP_API int plip_densenet_num_tensors(void);
PLIP_API int plip_densenet_tensor_info(int index, plip_tensor_info_t* info);
PLIP_API uint64_t plip_densenet_blob_bytes(void);
PLIP_API uint64_t plip_densenet_workspace_bytes(int max_micro_batch);
/* 1 <= max_micro_batch <= 4096; device must be an sm_90 GPU. */
PLIP_API int plip_densenet_create(const void* host_blob, uint64_t blob_bytes, int device, int max_micro_batch,
                                  plip_densenet_t** out);
PLIP_API int plip_densenet_destroy(plip_densenet_t* e);
PLIP_API int plip_densenet_max_micro_batch(const plip_densenet_t* e);
/* tiles_dev: uint8 RGB [n,224,224,3] (what Resize(224) + CenterCrop(224) produce before ToTensor; ToTensor + the
 * ImageNet Normalize are fused into the first convolution); out_dev float32 [n,1024].  Micro-batches of at most
 * max_micro_batch images, 122 launches each, on `stream`; calls on one handle are serialised on the device. */
PLIP_API int plip_densenet_encode(plip_densenet_t* e, const void* tiles_dev, int64_t n, float* out_dev, void* stream);

/* ---- host-buffer convenience (end-to-end path; copies are inside the call) ------------------- */
/* pixels_host / ids_host / out_host are host pointers (pinned or pageable).  The call stages
 * micro-batches through pinned buffers on two streams (H2D overlapped with compute), writes the
 * float32 [n,512] result to out_host and returns after the last D2H completed.
 * plip_encode_text_host scans the ids for the caption lengths (first eos) and uses plip_encode_text_prefix: one
 * pass up to the longest caption, or — for large batches of mixed lengths — the captions sorted by length and
 * processed in up to 8 length buckets, each only up to its own longest caption (results are returned in the
 * caller's order). */
PLIP_API int plip_encode_images_host(plip_engine_t* e, const void* pixels_host, int pixel_format, int64_t n,
                                     float* out_host, int normalize);
PLIP_API int plip_encode_text_host(plip_engine_t* e, const void* ids_host, int ids_dtype,
                                   const void* attention_mask_host, int64_t n, int seq_len,
                                   float* out_host, int normalize);

/* ---- in-step kernel timing (measurement support for bench.py; SURVEY.md §8d) --------------------- */
/* While enabled, every kernel launch of plip_encode_images / plip_encode_text* on this handle is bracketed by a
 * CUDA event pair recorded on the launch stream.  plip_profile_read waits for the recorded events and returns one
 * aggregated row per (tower, kernel role): launches, summed device time, and the ALGORITHMIC flops / HBM bytes of
 * those launches (DESIGN.md §4) — i.e. each kernel's average duration inside the step it belongs to, under the
 * step's own clocks and cache state.  Event pairs serialise nothing but cost a few microseconds of launch gap
 * each, so bench.py profiles separate, untimed steps.  enable(on) always clears what was recorded. */
typedef struct plip_kernel_time {
  char name[48];     /* "<tower>/<role>", e.g. "vision/gemm[fc2+resid]", "text/attention" */
  int32_t launches;
  float total_ms;
  double flops;      /* algorithmic FLOPs of the recorded launches (0 for memory-bound helpers) */
  double bytes;      /* algorithmic HBM bytes of the recorded launches */
} plip_kernel_time_t;
PLIP_API int plip_profile_enable(plip_engine_t* e, int on);
PLIP_API int plip_profile_read(plip_engine_t* e, plip_kernel_time_t* out, int cap, int* count);

/* ---- per-kernel test hooks (used by tests/ only; stream-ordered, device pointers) ------------ */
/* The handle-free hooks below interpret / produce 16-bit data in the format set here (default PLIP_OPERAND_BF16). */
PLIP_API int plip_dbg_set_operand_format(int operand_format);
/* epilogue: 0 bias->bf16, 1 bias+QuickGELU->bf16, 2 x_f32 += acc+bias (optionally also xb_out bf16 copy +
 * stats_out [M,8,2] row statistics), 3 patch scatter + pos, 4 plain f32, 5/6 = 0/1 with the LayerNorm fold
 * (colsum [N], stats_in [M,8,2] with n_partials valid slots).  cluster_size: 0 = auto, 1 / 2 = CTAs per cluster (2 = the
 * pair shares the W tile through TMA multicast); block_n: 0 = auto, 128 / 192 / 256 = N tile. */
PLIP_API int plip_dbg_gemm(const void* A_bf16, int lda, const void* W_bf16, int ldw, int M, int N, int K,
                           const float* bias, void* out, int ldo, const float* pos, int epilogue, int cluster_size,
                           int block_n, const float* colsum, const float* stats_in, int n_partials, void* xb_out,
                           float* stats_out, void* stream);
/* Host-only: fixed-point filter row of output index xx for one axis of plip_resize_crop_u8 (the same code the
 * kernel runs).  Returns the filter bank width ksize (or -ksize if k_cap is too small). */
PLIP_API int plip_dbg_resize_filter(int in_size, int out_size, int xx, int32_t* k_host, int k_cap, int* xmin,
                                    int* count);
/* The same for plip_resize_crop_bilinear_u8's triangle filter. */
PLIP_API int plip_dbg_resize_filter_bilinear(int in_size, int out_size, int xx, int32_t* k_host, int k_cap, int* xmin,
                                             int* count);
/* Host-only: the length-bucket plan plip_encode_text_host uses (lens = first-eos position + 1 per caption).
 * perm_host[i] = original index of the caption at sorted position i (may be NULL); bucket k covers sorted positions
 * [bucket_start[k], bucket_start[k+1]) and is processed with prefix bucket_prefix[k].  Arrays hold cap+1 / cap
 * entries (cap <= 8).  Returns the number of buckets. */
PLIP_API int plip_dbg_text_bucket_plan(const int32_t* lens_host, int64_t n, int seq_len, int32_t* perm_host,
                                       int32_t* bucket_start_host, int32_t* bucket_prefix_host, int cap);
PLIP_API int plip_dbg_rowstats_cast(const float* x, int64_t rows, int dim, void* xb_bf16, float* stats, void* stream);
PLIP_API int plip_dbg_layernorm(const float* x, int64_t rows, int dim, int64_t in_row_stride,
                                const float* gamma, const float* beta, float* out_f32, void* out_bf16,
                                void* stream);
/* The whole LayerNorm launcher: row r of the output is LayerNorm(x + row_index[r] * in_row_stride) (row_index NULL:
 * r * in_row_stride); out_f32 [rows, dim] and / or out16 [rows, dim] (either may be NULL; x == out_f32 is allowed).
 * x, gamma, beta, out_f32 16-byte aligned, out16 8-byte aligned; dim 768 or 512. */
PLIP_API int plip_dbg_layernorm_ex(const float* x, const int32_t* row_index, int64_t in_row_stride, int64_t rows,
                                   int dim, const float* gamma, const float* beta, float* out_f32, void* out16,
                                   void* stream);
/* seq_len <= 128: any causal / key_mask; 128 < seq_len <= 1025 (long-sequence kernel): causal = 0, key_mask = NULL. */
PLIP_API int plip_dbg_attention(const void* qkv_bf16, int64_t n_seq, int seq_len, int heads, int causal,
                                const int32_t* key_mask, void* out_bf16, void* stream);
/* The attention probabilities of plip_dbg_attention's input: probs_dev float32 [n_seq, heads, seq_len, seq_len], any
 * causal / key_mask, 1 <= seq_len <= 1025. */
PLIP_API int plip_dbg_attention_probs(const void* qkv_bf16, int64_t n_seq, int seq_len, int heads, int causal,
                                      const int32_t* key_mask, float* probs_dev, void* stream);
/* One DenseNet kernel on caller buffers (bf16 activations NHWC, pixel stride lda / ldo elements, 16-byte aligned):
 * op 0 stem conv0 + norm0 + ReLU (in: uint8 tiles [n,224,224,3]; out [n*112*112, ldo]); 1 3x3/s2/p1 max pool
 * (in [n,112,112,64]; out channels [0,64) of [n*56*56, ldo]); 2 conv1: relu(x*a_scale+a_shift) of the first c_in
 * channels . W^T, then relu(*e_scale+e_shift) (out [n*side^2, ldo], 128 channels); 3 conv2: 3x3/p1 over a dense
 * [n,side,side,128] (out 32 channels); 4 transition: 2x2 average pool of relu(x*a_scale+a_shift) over
 * [n,2*side,2*side,lda], then . W^T (out c_in/2 channels); 5 tail: fp32 out [n,1024] = mean over 49 positions of
 * in [n,49,1024], *e_scale+e_shift. */
PLIP_API int plip_dbg_densenet_op(int op, const void* in_dev, int lda, int64_t n, int side, int c_in, const void* w_dev,
                                  const float* a_scale, const float* a_shift, const float* e_scale,
                                  const float* e_shift, void* out_dev, int ldo, void* stream);
PLIP_API int plip_dbg_im2col(const void* pixels, int pixel_format, int64_t n, void* out_bf16, void* stream);
/* plip_dbg_im2col at any image size plip_encode_images_hw accepts: out16 [n * (height/32) * (width/32), 3072]. */
PLIP_API int plip_dbg_im2col_hw(const void* pixels, int pixel_format, int64_t n, int height, int width, void* out16,
                                void* stream);
/* plip_dbg_im2col_hw for a patch size of 32 or 16: out16 [n * (height/patch) * (width/patch), 3 * patch^2], row
 * b * gh * gw + py * gw + px, column c * patch^2 + ky * patch + kx. */
PLIP_API int plip_dbg_im2col_patch(const void* pixels, int pixel_format, int64_t n, int height, int width, int patch,
                                   void* out16, void* stream);
/* The patch matrix plip_encode_windows builds: n 224 x 224 windows of a uint8 RGB region (rows row_pitch_bytes apart)
 * at device int32 (row, col) origins_dev [n, 2] (8-byte aligned, each window inside the region; not checked here),
 * in the layout of plip_dbg_im2col_patch. */
PLIP_API int plip_dbg_window_im2col_patch(const void* region_dev, int64_t row_pitch_bytes, const int32_t* origins_dev,
                                          int64_t n, int patch, void* out16, void* stream);
/* Text embeddings of n captions (the first seq_len of ids_stride ids per row) with caller tables tok float32
 * [49408, 512] and pos float32 [>= seq_len, 512]: x_out [n * seq_len, 512] and the pooled row b * seq_len + t of each
 * caption in eos_rows_out int32 [n] (t = first eos 49407, else 0, or with no_eos_argmax the first largest id). */
PLIP_API int plip_dbg_text_embed(const void* ids, int ids_dtype, int64_t n, int seq_len, int ids_stride,
                                 const float* tok, const float* pos, float* x_out, int32_t* eos_rows_out,
                                 int no_eos_argmax, void* stream);
/* out[i] = mask[(i / seq_len) * stride + i % seq_len] != 0 for i < count (mask_dtype PLIP_IDS_I32 / I64). */
PLIP_API int plip_dbg_mask_to_i32(const void* mask, int mask_dtype, int64_t count, int seq_len, int stride,
                                  int32_t* out, void* stream);
/* x[b * seq * 768 + c] = cls[c] + pos[c] for b < n: the class rows of n sequences of seq rows. */
PLIP_API int plip_dbg_cls_rows(const float* cls, const float* pos, int64_t n, int seq, float* x, void* stream);
/* Rows idx(i) = row_index[i] (or i * row_stride when row_index is NULL) of a16 [*, dim] (16-bit) and x32 [*, dim]
 * (float32) copied to rows i of a16_out and x32_out, i < n; every pointer 16-byte aligned, dim % 8 == 0. */
PLIP_API int plip_dbg_gather_rows(const void* a16, const float* x32, const int32_t* row_index, int64_t row_stride,
                                  int64_t n, int dim, void* a16_out, float* x32_out, void* stream);
/* The vision position table pos_dev (float32 [50,768]) resized to a grid_h x grid_w patch grid as
 * plip_encode_images_hw does it: out_dev float32 [1 + grid_h * grid_w, 768]; 1 <= grid_h, grid_w <= 32. */
PLIP_API int plip_dbg_pos_interp(const float* pos_dev, int grid_h, int grid_w, float* out_dev, void* stream);
/* The same for the stored table of a patch size: 32 (pos_dev [50, 768], a 7 x 7 grid) or 16 ([197, 768], 14 x 14). */
PLIP_API int plip_dbg_pos_interp_patch(const float* pos_dev, int patch, int grid_h, int grid_w, float* out_dev,
                                       void* stream);
/* Vision tower at any image size (plip_encode_images_hw geometry): the fp32 residual stream [n*S, 768] after
 * `num_layers` layers; n must fit one pass. */
PLIP_API int plip_dbg_hidden_states_hw(plip_engine_t* e, const void* pixels_dev, int pixel_format, int64_t n,
                                       int height, int width, int num_layers, float* hidden_dev, void* stream);
/* Run one tower and copy the fp32 residual stream [n*S, D] after `num_layers` encoder layers
 * (0 = after embeddings / pre-LN) into hidden_dev.  tower: 0 = vision (input pixels), 1 = text. */
PLIP_API int plip_dbg_hidden_states(plip_engine_t* e, int tower, const void* input_dev, int input_format,
                                    const void* attention_mask_dev, int64_t n, int num_layers,
                                    float* hidden_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PLIP_B200_H_ */

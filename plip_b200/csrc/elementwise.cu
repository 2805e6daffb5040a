// plip_b200 — HBM-bound helper kernels around the GEMMs: patch im2col (+ uint8 preprocessing),
// LayerNorm, token/position embedding gather, class-token rows, EOS search, L2 normalisation.
//
// All are pure streaming kernels (roofline: HBM); accesses are 16-byte vectorised and coalesced.
#include "kernels.cuh"

#include <string.h>

namespace plip {

namespace {

constexpr int kEwThreads = 256;

__device__ __forceinline__ uint4 pack8(const float (&f)[8], int f16) {
  uint4 u;
  u.x = pack_op2_rt(f[0], f[1], f16);
  u.y = pack_op2_rt(f[2], f[3], f16);
  u.z = pack_op2_rt(f[4], f[5], f16);
  u.w = pack_op2_rt(f[6], f[7], f16);
  return u;
}

// ------------------------------------------------------------------------------------------------
// im2col of non-overlapping P x P patches (P = 32: ViT-B/32, 16: ViT-B/16):
// pixels -> A0[b*patches + py*gw + px][c*P*P + ky*P + kx] (bf16), i.e. [b*49 + py*7 + px][c*1024 + ky*32 + kx] at 32.
// Restates nn.Conv2d(3,768,P,P,bias=False) input gathering (TF:modeling_clip.py:148-154,209-210);
// the uint8 path fuses CLIPImageProcessor's rescale + normalise (TF:image_processing_clip.py:50-62).
// One thread moves 8 consecutive x of one image row (a patch row is 4 or 2 such groups).
// Any image size (interpolated position table): the image is H x W, the patch grid gh x gw (the H % P bottom rows
// and W % P right columns are never read, as with the stride-P conv).  FIXED = the 224 x 224 geometry as
// compile-time constants.  vec = 0 (rows whose start is not aligned for the vector loads, e.g. W = 250): the same
// pixels read one value at a time.
// ------------------------------------------------------------------------------------------------
struct ImGeom {
  int H, W, gh, gw;
};

template <int P>
struct PatchShift;  // log2 of the patch size: patch coordinates by shifts and masks
template <>
struct PatchShift<32> { static constexpr int value = 5; };
template <>
struct PatchShift<16> { static constexpr int value = 4; };

// 8 consecutive RGB pixels of one image row (24 bytes, interleaved) -> the three channel rows of one patch-matrix row
// at dst (channel c at dst + c * CS, CS = P * P).  Shared by the tile and the window im2col, so both produce the same
// bits.
template <int CS>
__device__ __forceinline__ void store_u8_patch_row(const uint8_t (&bytes)[24], __nv_bfloat16* dst, int f16) {
  const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
  const float istd[3] = {1.0f / 0.26862954f, 1.0f / 0.26130258f, 1.0f / 0.27577711f};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = (bytes[j * 3 + c] * (1.0f / 255.0f) - mean[c]) * istd[c];
    *reinterpret_cast<uint4*>(dst + c * CS) = pack8(f, f16);
  }
}

template <int FMT, bool FIXED, int P>
__global__ void __launch_bounds__(kEwThreads) im2col_kernel(const void* __restrict__ pixels,
                                                            __nv_bfloat16* __restrict__ out, int64_t n, int f16,
                                                            ImGeom geo, int vec) {
  constexpr int SH = PatchShift<P>::value, CS = P * P, K = 3 * CS;
  const int H = FIXED ? kImage : geo.H, W = FIXED ? kImage : geo.W;
  const int gw = FIXED ? vis_grid(P) : geo.gw, patches = FIXED ? vis_grid(P) * vis_grid(P) : geo.gh * geo.gw;
  const int rows = FIXED ? kImage : geo.gh * P;  // image rows that reach a patch
  const int kX8 = FIXED ? kImage / 8 : geo.gw * (P / 8);  // groups of 8 pixels per image row (28 at 224)
  const bool vload = FIXED || vec != 0;
  const int64_t total = (FMT == PLIP_PIX_U8_NHWC) ? n * rows * kX8 : n * 3 * rows * kX8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int x8 = (int)(i % kX8);
    int64_t r = i / kX8;
    const int y = (int)(r % rows);
    r /= rows;
    const int x = x8 * 8;
    const int py = y >> SH, ky = y & (P - 1), px = x >> SH, kx = x & (P - 1);
    if constexpr (FMT == PLIP_PIX_U8_NHWC) {
      const int64_t b = r;
      const uint8_t* src = static_cast<const uint8_t*>(pixels) + ((b * H + y) * W + x) * 3;
      uint8_t bytes[24];
      if (vload) {
        const uint2* s2 = reinterpret_cast<const uint2*>(src);  // 24 bytes, 8-byte aligned
        uint2 w0 = __ldg(s2), w1 = __ldg(s2 + 1), w2 = __ldg(s2 + 2);
        *reinterpret_cast<uint2*>(bytes) = w0;
        *reinterpret_cast<uint2*>(bytes + 8) = w1;
        *reinterpret_cast<uint2*>(bytes + 16) = w2;
      } else {
#pragma unroll
        for (int j = 0; j < 24; ++j) bytes[j] = __ldg(src + j);
      }
      store_u8_patch_row<CS>(bytes, out + (b * patches + py * gw + px) * (int64_t)K + ky * P + kx, f16);
    } else {
      const int c = (int)(r % 3);
      const int64_t b = r / 3;
      const int64_t src_off = ((b * 3 + c) * H + y) * W + x;
      __nv_bfloat16* dst =
          out + (b * patches + py * gw + px) * (int64_t)K + c * CS + ky * P + kx;
      if constexpr (FMT == PLIP_PIX_F32_NCHW) {
        const float* s = static_cast<const float*>(pixels) + src_off;
        float f[8];
        if (vload) {
          const float4* s4 = reinterpret_cast<const float4*>(s);
          const float4 a = __ldg(s4), bq = __ldg(s4 + 1);
          f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = bq.x; f[5] = bq.y; f[6] = bq.z; f[7] = bq.w;
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = __ldg(s + j);
        }
        *reinterpret_cast<uint4*>(dst) = pack8(f, f16);
      } else {  // bf16 NCHW: straight 16-byte copy (re-rounded to half for the fp16 operand format)
        const __nv_bfloat16* s = static_cast<const __nv_bfloat16*>(pixels) + src_off;
        uint4 w;
        if (vload) {
          w = __ldg(reinterpret_cast<const uint4*>(s));
        } else {
          const unsigned short* s16 = reinterpret_cast<const unsigned short*>(s);
          uint32_t u[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) u[j] = (uint32_t)__ldg(s16 + 2 * j) | ((uint32_t)__ldg(s16 + 2 * j + 1) << 16);
          w = make_uint4(u[0], u[1], u[2], u[3]);
        }
        if (f16) {
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&w);
          float f[8];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 t = __bfloat1622float2(h2[j]);
            f[2 * j] = t.x;
            f[2 * j + 1] = t.y;
          }
          w = pack8(f, 1);
        }
        *reinterpret_cast<uint4*>(dst) = w;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Windows of a slide region: 224 x 224 crops of one uint8 RGB region [H, W, 3] (row pitch in bytes, may be a view into a
// wider array) at arbitrary (row, col) origins, read in place instead of being cut out into tiles first.
//
// A window row starts at byte row * pitch + 3 * col, which is 8-byte aligned for few origins (the reference's grid
// steps by 201 pixels), so the 8-byte loads of im2col_kernel do not apply.  load24 reads the 6 or 7 aligned 32-bit
// words that hold the 24 bytes of an 8-pixel group and realigns them with __byte_perm, one selector for the whole
// group since the misalignment (address & 3) is the same for every word.  Versus staging each window row through shared
// memory this needs no barrier and no second pass, and the loads of a warp's 28 active lanes fall in one 672-byte row,
// so L1 merges them into the same sectors the aligned loads would touch.  Only words holding at least one of the 24
// bytes are read, never one past the end of the region.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load24(const uint8_t* src, uint8_t (&bytes)[24]) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(src);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
  const unsigned off = (unsigned)(a & 3);
  uint32_t v[7];
#pragma unroll
  for (int k = 0; k < 6; ++k) v[k] = __ldg(w + k);
  v[6] = off ? __ldg(w + 6) : 0u;
  const unsigned sel = 0x3210u + off * 0x1111u;  // bytes off .. off + 3 of the pair (v[k], v[k + 1])
  uint32_t* out = reinterpret_cast<uint32_t*>(bytes);
#pragma unroll
  for (int k = 0; k < 6; ++k) out[k] = __byte_perm(v[k], v[k + 1], sel);
}

// Window im2col: the matrix im2col_kernel<PLIP_PIX_U8_NHWC, true, P> builds from the same windows cut out as
// [n,224,224,3] tiles, bit for bit (same store_u8_patch_row).  origins: device int32 (row, col) pairs, one per window.
template <int P>
__global__ void __launch_bounds__(kEwThreads) window_im2col_kernel(const uint8_t* __restrict__ region, int64_t pitch,
                                                                   const int2* __restrict__ origins, int64_t n,
                                                                   __nv_bfloat16* __restrict__ out, int f16) {
  constexpr int SH = PatchShift<P>::value, CS = P * P, K = 3 * CS, G = vis_grid(P);
  constexpr int kX8 = kImage / 8;
  const int64_t total = n * kImage * kX8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int x8 = (int)(i % kX8);
    const int64_t r = i / kX8;
    const int y = (int)(r % kImage);
    const int64_t b = r / kImage;
    const int x = x8 * 8;
    const int2 o = __ldg(origins + b);
    alignas(16) uint8_t bytes[24];
    load24(region + (int64_t)(o.x + y) * pitch + (int64_t)(o.y + x) * 3, bytes);
    const int py = y >> SH, ky = y & (P - 1), px = x >> SH, kx = x & (P - 1);
    store_u8_patch_row<CS>(bytes, out + (b * (G * G) + py * G + px) * (int64_t)K + ky * P + kx, f16);
  }
}

// The sum of `cnt` over the block, stored by thread 0 at dst.
__device__ __forceinline__ void store_block_sum(int cnt, int32_t* dst) {
  __shared__ int part[kEwThreads / 32];
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
#pragma unroll
    for (int k = 0; k < kEwThreads / 32; ++k) s += part[k];
    *dst = s;
  }
}

// Background pixels of each window: those whose three channels are all >= threshold (the reference's background_ratio,
// preprocess_DigestPath.py:28-34, times 224 * 224), as exact int32 counts.  One block per window, blocks in window
// order: for window_grid's row-major origins the blocks resident at once cover neighbouring windows of one band of
// rows, so the overlap of two windows is read from HBM once and hit in L2 the second time.  The origins of a launch
// travel as kernel parameters (16 KB), so the call needs no device buffer of its own.
constexpr int kBgBatch = 2048;
struct WindowBatch {
  int2 org[kBgBatch];
};

__global__ void __launch_bounds__(kEwThreads) window_background_kernel(const uint8_t* __restrict__ region, int64_t pitch,
                                                                       const __grid_constant__ WindowBatch batch,
                                                                       int threshold, int32_t* __restrict__ counts) {
  constexpr int kX8 = kImage / 8;
  const int2 o = batch.org[blockIdx.x];
  int cnt = 0;
  for (int i = threadIdx.x; i < kImage * kX8; i += blockDim.x) {
    const int y = i / kX8, x = (i % kX8) * 8;
    alignas(16) uint8_t bytes[24];
    load24(region + (int64_t)(o.x + y) * pitch + (int64_t)(o.y + x) * 3, bytes);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      cnt += (bytes[3 * j] >= threshold) & (bytes[3 * j + 1] >= threshold) & (bytes[3 * j + 2] >= threshold);
  }
  store_block_sum(cnt, counts + blockIdx.x);
}

// Mask elements > threshold in each window of a uint8 mask [H, W, C] (C = 1 or 3), as exact int32 counts: the
// reference's (msk_np > 10) then np.sum(msk_patch_np > 0) (preprocess_DigestPath.py:58-62, 83-84), which counts every
// channel of an RGB mask.  Same launch shape as window_background_kernel; level-sized masks are small, so plain byte
// loads (coalesced along the window row) suffice.
template <int C>
__global__ void __launch_bounds__(kEwThreads) window_mask_kernel(const uint8_t* __restrict__ mask, int64_t pitch,
                                                                 const __grid_constant__ WindowBatch batch,
                                                                 int threshold, int32_t* __restrict__ counts) {
  constexpr int kRow = kImage * C;
  const int2 o = batch.org[blockIdx.x];
  const uint8_t* base = mask + (int64_t)o.x * pitch + (int64_t)o.y * C;
  int cnt = 0;
  for (int i = threadIdx.x; i < kImage * kRow; i += blockDim.x) {
    const int y = i / kRow, x = i - y * kRow;
    cnt += (int)__ldg(base + (int64_t)y * pitch + x) > threshold;
  }
  store_block_sum(cnt, counts + blockIdx.x);
}

// One launch of `kernel` per kBgBatch windows, the origins passed by value.
template <typename K>
int launch_window_batches(K kernel, const uint8_t* src, int64_t pitch, const int32_t* origins_host, int64_t n,
                          int threshold, int32_t* counts, cudaStream_t st) {
  static thread_local WindowBatch b;  // 16 KB: kept off the stack
  for (int64_t base = 0; base < n; base += kBgBatch) {
    const int cnt = (int)(n - base < kBgBatch ? n - base : kBgBatch);
    memcpy(b.org, origins_host + 2 * base, (size_t)cnt * sizeof(int2));
    PLIP_CUDA_CHECK(launch_kernel(kernel, dim3(cnt), dim3(kEwThreads), 0, st, 1, src, pitch, b, threshold,
                                  counts + base));
  }
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (eps 1e-5, affine), one warp per row, fp32 statistics (two-pass in
// registers).  TF:modeling_clip.py:371,380 (layer_norm1/2), :677 (pre_layrnorm), :686 (post_layernorm
// on the CLS row), :562 (final_layer_norm; only the pooled EOS row is needed downstream).
// Rows are addressed as x + row_index[r] * in_row_stride (row_index == nullptr -> r).
// ------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kEwThreads) layernorm_kernel(const float* __restrict__ x,
                                                               const int32_t* __restrict__ row_index,
                                                               int64_t in_row_stride, int64_t rows,
                                                               const float* __restrict__ gamma,
                                                               const float* __restrict__ beta,
                                                               float* __restrict__ out_f32,
                                                               __nv_bfloat16* __restrict__ out_bf16, int f16) {
  constexpr int V = D / 128;  // float4 per lane
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const int64_t src_row = row_index ? (int64_t)row_index[r] : r;
    const float4* xr = reinterpret_cast<const float4*>(x + src_row * in_row_stride);
    float4 v[V];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < V; ++j) {
      v[j] = xr[lane + 32 * j];
      s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
    }
    const float mean = warp_sum(s) * (1.0f / D);
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + kLnEps);
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * j);
      const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32 * j);
      float4 y;
      y.x = (v[j].x - mean) * rstd * g.x + b.x;
      y.y = (v[j].y - mean) * rstd * g.y + b.y;
      y.z = (v[j].z - mean) * rstd * g.z + b.z;
      y.w = (v[j].w - mean) * rstd * g.w + b.w;
      if (out_f32) reinterpret_cast<float4*>(out_f32 + r * D)[lane + 32 * j] = y;
      if (out_bf16) {
        uint2 u;
        u.x = pack_op2_rt(y.x, y.y, f16);
        u.y = pack_op2_rt(y.z, y.w, f16);
        reinterpret_cast<uint2*>(out_bf16 + r * D)[lane + 32 * j] = u;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// bf16 copy + per-row (sum, sum of squares) of the fp32 residual stream: the A operand and the
// statistics a LayerNorm-folded GEMM needs (EPI_LN_*), for rows that were not produced by a residual
// GEMM epilogue (start of a tower).  One warp per row; slot 0 of the statistics row is written.
// ------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kEwThreads) rowstats_cast_kernel(const float* __restrict__ x, int64_t rows,
                                                                   __nv_bfloat16* __restrict__ xb,
                                                                   float2* __restrict__ stats, int f16) {
  constexpr int V = D / 128;
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float4* xr = reinterpret_cast<const float4*>(x + r * D);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const float4 v = xr[lane + 32 * j];
      s1 += (v.x + v.y) + (v.z + v.w);
      s2 += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
      uint2 u;
      u.x = pack_op2_rt(v.x, v.y, f16);
      u.y = pack_op2_rt(v.z, v.w, f16);
      reinterpret_cast<uint2*>(xb + r * D)[lane + 32 * j] = u;
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) stats[r * kStatSlots] = make_float2(s1, s2);
  }
}

// ------------------------------------------------------------------------------------------------
// Text embeddings: x[b*S + t] = token_embedding[ids[b,t]] + position_embedding[t]   (TF:253-256).
// One warp per token row (512 fp32 = 4 float4 per lane).  Ids are clamped into the vocabulary for
// memory safety (the reference would raise an IndexError on out-of-range ids).
// ------------------------------------------------------------------------------------------------
template <typename IdT>
__global__ void __launch_bounds__(kEwThreads) text_embed_kernel(const IdT* __restrict__ ids, int64_t n,
                                                                int seq_len, int ids_stride,
                                                                const float* __restrict__ tok,
                                                                const float* __restrict__ pos,
                                                                float* __restrict__ x) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t rows = n * seq_len;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const int t = (int)(r % seq_len);
    long long id = (long long)ids[(r / seq_len) * ids_stride + t];  // rows may be a prefix of longer id rows
    id = id < 0 ? 0 : (id >= kVocab ? kVocab - 1 : id);
    const float4* e = reinterpret_cast<const float4*>(tok + id * kTxtDim);
    const float4* p = reinterpret_cast<const float4*>(pos + (int64_t)t * kTxtDim);
    float4* o = reinterpret_cast<float4*>(x + r * kTxtDim);
#pragma unroll
    for (int j = 0; j < kTxtDim / 128; ++j) {
      const float4 a = __ldg(e + lane + 32 * j), b = __ldg(p + lane + 32 * j);
      o[lane + 32 * j] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
  }
}

// Pooling row of each caption: b*S + (first t with ids[b,t] == eos, else 0) — the semantics of
// (input_ids == eos_token_id).int().argmax(-1) (TF:571-584).  One warp per caption.
template <typename IdT>
__global__ void __launch_bounds__(kEwThreads) eos_row_kernel(const IdT* __restrict__ ids, int64_t n,
                                                             int seq_len, int ids_stride, int eos_id,
                                                             int no_eos_argmax, int32_t* __restrict__ row_index) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t b = warp; b < n; b += nwarps) {
    int first = seq_len;
    for (int t0 = 0; t0 < seq_len && first == seq_len; t0 += 32) {
      const int t = t0 + lane;
      const bool hit = t < seq_len && (long long)ids[b * ids_stride + t] == (long long)eos_id;
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (m) first = t0 + __ffs(m) - 1;
    }
    if (first == seq_len) {
      // no eos in the row.  HF with eos_token_id == 49407 pools position 0 here ((ids == eos).argmax() of all zeros,
      // TF:571-584); legacy configs (eos_token_id == 2, what openai/clip-vit-base-patch32 ships) and OpenAI clip pool
      // the first position of the largest id (TF:564-570) — selected by plip_set_text_pooling.
      first = 0;
      if (no_eos_argmax) {
        long long best = -(1ll << 62);
        int best_t = 0;
        for (int t = lane; t < seq_len; t += 32) {
          const long long v = (long long)ids[b * ids_stride + t];
          if (v > best) { best = v; best_t = t; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const long long ov = __shfl_xor_sync(0xffffffffu, best, o);
          const int ot = __shfl_xor_sync(0xffffffffu, best_t, o);
          if (ov > best || (ov == best && ot < best_t)) { best = ov; best_t = ot; }
        }
        first = best_t;
      }
    }
    if (lane == 0) row_index[b] = (int32_t)(b * seq_len + first);
  }
}

// Key-padding mask -> int32 (1 = attend, 0 = padded key).
template <typename IdT>
__global__ void __launch_bounds__(kEwThreads) mask_to_i32_kernel(const IdT* __restrict__ m, int64_t count,
                                                                 int seq_len, int stride,
                                                                 int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count;
       i += (int64_t)gridDim.x * blockDim.x)
    out[i] = m[(i / seq_len) * stride + (i % seq_len)] != 0 ? 1 : 0;
}

// Class-token rows: x[b*S] = class_embedding + position_embedding[0]   (TF:212-217), S = 50 at 224 x 224.
__global__ void __launch_bounds__(kEwThreads) cls_rows_kernel(const float* __restrict__ cls,
                                                              const float* __restrict__ pos, int64_t n, int seq,
                                                              float* __restrict__ x) {
  constexpr int V = kVisDim / 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n * V;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / V;
    const int j = (int)(i % V);
    const float4 c = __ldg(reinterpret_cast<const float4*>(cls) + j);
    const float4 p = __ldg(reinterpret_cast<const float4*>(pos) + j);
    reinterpret_cast<float4*>(x + b * seq * kVisDim)[j] =
        make_float4(c.x + p.x, c.y + p.y, c.z + p.z, c.w + p.w);
  }
}

// Position table of a gh x gw patch grid (TF:modeling_clip.py:161-200, interpolate_pos_encoding): row 0 (class) is
// copied; rows 1..SRC^2 of the stored table (SRC = 7 for ViT-B/32, 14 for ViT-B/16), viewed as [768, SRC, SRC], are
// resized to [768, gh, gw] the way F.interpolate(mode="bicubic", align_corners=False) does it: cubic convolution with
// A = -0.75, source coordinate (i + 0.5) * SRC / g - 0.5, taps clamped to [0, SRC - 1], no antialias; out row
// 1 + y * gw + x.  One thread per output value.
template <int SRC>
__device__ __forceinline__ void cubic_taps(int g, int i, int (&idx)[4], float (&w)[4]) {
  constexpr float A = -0.75f;
  const float scale = (float)SRC / (float)g;
  const float real = scale * ((float)i + 0.5f) - 0.5f;
  const float fl = floorf(real);
  const float t = real - fl;
  const float t1 = t + 1.f, t2 = 1.f - t, t3 = 2.f - t;
  w[0] = ((A * t1 - 5.f * A) * t1 + 8.f * A) * t1 - 4.f * A;
  w[1] = ((A + 2.f) * t - (A + 3.f)) * t * t + 1.f;
  w[2] = ((A + 2.f) * t2 - (A + 3.f)) * t2 * t2 + 1.f;
  w[3] = ((A * t3 - 5.f * A) * t3 + 8.f * A) * t3 - 4.f * A;
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[k] = min(max((int)fl - 1 + k, 0), SRC - 1);
}

template <int SRC>
__global__ void __launch_bounds__(kEwThreads) pos_interp_kernel(const float* __restrict__ pos, int gh, int gw,
                                                                float* __restrict__ out) {
  const int total = (1 + gh * gw) * kVisDim;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int row = i / kVisDim, c = i - row * kVisDim;
    if (row == 0) {
      out[i] = __ldg(pos + c);
      continue;
    }
    const int y = (row - 1) / gw, x = (row - 1) - y * gw;
    int iy[4], ix[4];
    float wy[4], wx[4];
    cubic_taps<SRC>(gh, y, iy, wy);
    cubic_taps<SRC>(gw, x, ix, wx);
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float t = 0.f;
#pragma unroll
      for (int b = 0; b < 4; ++b) t += __ldg(pos + (size_t)(1 + iy[a] * SRC + ix[b]) * kVisDim + c) * wx[b];
      acc += t * wy[a];
    }
    out[i] = acc;
  }
}

// Pooled-row gather for the pruned last layer (engine.cu run_layers): copies row idx(i) of the 16-bit attention
// output and of the fp32 residual stream into compact [n, dim] buffers.  idx(i) = row_index[i], or i * row_stride
// when row_index is null (the vision CLS rows).  16-byte pieces, one per thread.
__global__ void __launch_bounds__(kEwThreads) gather_rows_kernel(const uint4* __restrict__ a16, const uint4* __restrict__ x32,
                                                                 const int32_t* __restrict__ row_index, int64_t row_stride,
                                                                 int64_t n, int dim, uint4* __restrict__ a16_out,
                                                                 uint4* __restrict__ x32_out) {
  const int v16 = dim / 8, v32 = dim / 4, per_row = v16 + v32;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n * per_row;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / per_row;
    const int j = (int)(i % per_row);
    const int64_t src = row_index ? (int64_t)row_index[r] : r * row_stride;
    if (j < v16) a16_out[r * v16 + j] = a16[src * v16 + j];
    else x32_out[r * v32 + (j - v16)] = x32[src * v32 + (j - v16)];
  }
}

// x[r] /= sqrt(sum x[r]^2): _get_vector_norm, no epsilon (TF:57-65,923-924). One warp per row.
__global__ void __launch_bounds__(kEwThreads) l2_normalize_kernel(float* __restrict__ x, int64_t rows,
                                                                  int dim) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    float* xr = x + r * dim;
    float s = 0.f;
    for (int j = lane; j < dim; j += 32) s += xr[j] * xr[j];
    const float inv = 1.0f / sqrtf(warp_sum(s));
    for (int j = lane; j < dim; j += 32) xr[j] *= inv;
  }
}

// p is a multiple of `bytes` (a power of two); null passes (optional outputs are checked where they are required).
inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

inline int grid_for(int64_t work_items, int per_block) {
  int64_t blocks = (work_items + per_block - 1) / per_block;
  const int64_t cap = 16LL * sm_count();
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace

int launch_im2col(const void* pixels, int fmt, int64_t n, int height, int width, __nv_bfloat16* out, int f16,
                  cudaStream_t st, int patch) {
  PLIP_REQUIRE(patch == kPatch || patch == kPatch16, "im2col: patch size %d (32 or 16)", patch);
  PLIP_REQUIRE(n > 0, "im2col: n must be positive");
  PLIP_REQUIRE(height >= patch && width >= patch && height / patch <= kMaxGrid && width / patch <= kMaxGrid,
               "im2col: image size %dx%d out of range", height, width);
  const bool fixed = height == kImage && width == kImage;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(pixels);
  PLIP_REQUIRE(pixels && out, "im2col: null argument");
  PLIP_REQUIRE(!fixed || (addr & 15) == 0, "im2col: pixels must be 16-byte aligned");
  PLIP_REQUIRE(aligned(pixels, fmt == PLIP_PIX_F32_NCHW ? 4 : fmt == PLIP_PIX_BF16_NCHW ? 2 : 1),
               "im2col: pixels not aligned to their element size");
  PLIP_REQUIRE(aligned(out, 16), "im2col: out must be 16-byte aligned");
  // vector loads need every row start aligned: f32 16 B (W % 4 == 0), bf16 16 B (W % 8), u8 8 B (3 W % 8)
  const bool aligned = (addr & (fmt == PLIP_PIX_U8_NHWC ? 7 : 15)) == 0;
  const int vec = aligned && width % (fmt == PLIP_PIX_F32_NCHW ? 4 : 8) == 0 ? 1 : 0;
  const ImGeom geo{height, width, height / patch, width / patch};
  const int64_t items = (fmt == PLIP_PIX_U8_NHWC ? 1 : 3) * n * (geo.gh * patch) * (geo.gw * (patch / 8));
  const int grid = grid_for(items, kEwThreads);
#define PLIP_IM2COL(F, P)                                                                                              \
  PLIP_CUDA_CHECK(fixed ? launch_kernel(im2col_kernel<F, true, P>, dim3(grid), dim3(kEwThreads), 0, st, 1, pixels, out, \
                                        n, f16, geo, vec)                                                              \
                        : launch_kernel(im2col_kernel<F, false, P>, dim3(grid), dim3(kEwThreads), 0, st, 1, pixels,    \
                                        out, n, f16, geo, vec))
#define PLIP_IM2COL_FMT(P)                                                                                             \
  switch (fmt) {                                                                                                       \
    case PLIP_PIX_F32_NCHW: PLIP_IM2COL(PLIP_PIX_F32_NCHW, P); break;                                                  \
    case PLIP_PIX_BF16_NCHW: PLIP_IM2COL(PLIP_PIX_BF16_NCHW, P); break;                                                \
    case PLIP_PIX_U8_NHWC: PLIP_IM2COL(PLIP_PIX_U8_NHWC, P); break;                                                    \
    default: set_last_error("im2col: unknown pixel format %d", fmt); return -2;                                        \
  }
  if (patch == kPatch) {
    PLIP_IM2COL_FMT(kPatch)
  } else {
    PLIP_IM2COL_FMT(kPatch16)
  }
#undef PLIP_IM2COL_FMT
#undef PLIP_IM2COL
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_window_im2col(const WindowSrc& win, int64_t n, __nv_bfloat16* out, int f16, cudaStream_t st, int patch) {
  PLIP_REQUIRE(n > 0 && win.region && win.origins && out, "window_im2col: bad argument");
  PLIP_REQUIRE(patch == kPatch || patch == kPatch16, "window_im2col: patch size %d (32 or 16)", patch);
  PLIP_REQUIRE((reinterpret_cast<uintptr_t>(win.origins) & 7) == 0, "window_im2col: origins must be 8-byte aligned");
  const int grid = grid_for(n * kImage * (kImage / 8), kEwThreads);
  PLIP_CUDA_CHECK(launch_kernel(patch == kPatch ? window_im2col_kernel<kPatch> : window_im2col_kernel<kPatch16>,
                                dim3(grid), dim3(kEwThreads), 0, st, 1, win.region, win.pitch,
                                reinterpret_cast<const int2*>(win.origins), n, out, f16));
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_window_background(const uint8_t* region, int64_t pitch, const int32_t* origins_host, int64_t n,
                             int threshold, int32_t* counts, cudaStream_t st) {
  PLIP_REQUIRE(n > 0 && region && origins_host && counts, "window_background: bad argument");
  return launch_window_batches(window_background_kernel, region, pitch, origins_host, n, threshold, counts, st);
}

int launch_window_mask(const uint8_t* mask, int64_t pitch, int channels, const int32_t* origins_host, int64_t n,
                       int threshold, int32_t* counts, cudaStream_t st) {
  PLIP_REQUIRE(n > 0 && mask && origins_host && counts, "window_mask: bad argument");
  PLIP_REQUIRE(channels == 1 || channels == 3, "window_mask: channels must be 1 or 3 (got %d)", channels);
  return launch_window_batches(channels == 1 ? window_mask_kernel<1> : window_mask_kernel<3>, mask, pitch,
                               origins_host, n, threshold, counts, st);
}

int launch_pos_interp(const float* pos, int src_grid, int gh, int gw, float* out, cudaStream_t st) {
  PLIP_REQUIRE(pos && out, "pos_interp: null argument");
  PLIP_REQUIRE(src_grid == vis_grid(kPatch) || src_grid == vis_grid(kPatch16),
               "pos_interp: stored grid %d (7 or 14)", src_grid);
  PLIP_REQUIRE(gh >= 1 && gw >= 1 && gh <= kMaxGrid && gw <= kMaxGrid, "pos_interp: grid %dx%d out of [1,%d]", gh, gw,
               kMaxGrid);
  const int64_t items = (int64_t)(1 + gh * gw) * kVisDim;
  PLIP_CUDA_CHECK(launch_kernel(src_grid == kGrid ? pos_interp_kernel<vis_grid(kPatch)>
                                                  : pos_interp_kernel<vis_grid(kPatch16)>,
                                dim3(grid_for(items, kEwThreads)), dim3(kEwThreads), 0, st, 1, pos, gh, gw, out));
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_layernorm(const float* x, const int32_t* row_index, int64_t in_row_stride, int64_t rows, int dim,
                     const float* gamma, const float* beta, float* out_f32, __nv_bfloat16* out_bf16, int f16,
                     cudaStream_t st) {
  PLIP_REQUIRE(rows > 0, "layernorm: rows must be positive");
  PLIP_REQUIRE(in_row_stride % 4 == 0, "layernorm: row stride must be a multiple of 4 floats");
  PLIP_REQUIRE(x && gamma && beta, "layernorm: null argument");
  // float4 loads of x, gamma, beta and stores of out_f32; 8-byte stores of the 16-bit output
  PLIP_REQUIRE(aligned(x, 16) && aligned(gamma, 16) && aligned(beta, 16) && aligned(out_f32, 16) && aligned(out_bf16, 8),
               "layernorm: x, gamma, beta and out_f32 must be 16-byte aligned, the 16-bit output 8-byte aligned");
  const int grid = grid_for(rows, kEwThreads / 32);
  if (dim == kVisDim)
    PLIP_CUDA_CHECK(launch_kernel(layernorm_kernel<kVisDim>, dim3(grid), dim3(kEwThreads), 0, st, 1, x, row_index, in_row_stride, rows, gamma, beta, out_f32, out_bf16, f16));
  else if (dim == kTxtDim)
    PLIP_CUDA_CHECK(launch_kernel(layernorm_kernel<kTxtDim>, dim3(grid), dim3(kEwThreads), 0, st, 1, x, row_index, in_row_stride, rows, gamma, beta, out_f32, out_bf16, f16));
  else {
    set_last_error("layernorm: unsupported dim %d (768 or 512)", dim);
    return -2;
  }
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_rowstats_cast(const float* x, int64_t rows, int dim, __nv_bfloat16* xb, float2* stats, int f16, cudaStream_t st) {
  PLIP_REQUIRE(rows > 0, "rowstats_cast: rows must be positive");
  PLIP_REQUIRE(x && xb && stats, "rowstats_cast: null argument");
  PLIP_REQUIRE(aligned(x, 16) && aligned(xb, 8) && aligned(stats, 8),
               "rowstats_cast: x must be 16-byte aligned, xb and stats 8-byte aligned");
  const int grid = grid_for(rows, kEwThreads / 32);
  if (dim == kVisDim)
    PLIP_CUDA_CHECK(launch_kernel(rowstats_cast_kernel<kVisDim>, dim3(grid), dim3(kEwThreads), 0, st, 1, x, rows, xb, stats, f16));
  else if (dim == kTxtDim)
    PLIP_CUDA_CHECK(launch_kernel(rowstats_cast_kernel<kTxtDim>, dim3(grid), dim3(kEwThreads), 0, st, 1, x, rows, xb, stats, f16));
  else {
    set_last_error("rowstats_cast: unsupported dim %d", dim);
    return -2;
  }
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_text_embed(const void* ids, int ids_dtype, int64_t n, int seq_len, int ids_stride, const float* tok,
                      const float* pos, float* x, int32_t* eos_rows, int eos_id, int no_eos_argmax, cudaStream_t st) {
  PLIP_REQUIRE(ids_stride >= seq_len, "text_embed: ids row stride %d < seq_len %d", ids_stride, seq_len);
  PLIP_REQUIRE(n > 0 && seq_len > 0 && seq_len <= kTxtSeq, "text_embed: bad shape n=%lld seq_len=%d",
               (long long)n, seq_len);
  PLIP_REQUIRE(ids && tok && pos && x && eos_rows, "text_embed: null argument");
  PLIP_REQUIRE(aligned(ids, ids_dtype == PLIP_IDS_I64 ? 8 : 4) && aligned(tok, 16) && aligned(pos, 16) && aligned(x, 16) &&
                   aligned(eos_rows, 4),
               "text_embed: tok, pos and x must be 16-byte aligned, ids and eos_rows to their element size");
  const int grid = grid_for(n * seq_len, kEwThreads / 32);
  const int grid2 = grid_for(n, kEwThreads / 32);
  if (ids_dtype == PLIP_IDS_I64) {
    PLIP_CUDA_CHECK(launch_kernel(text_embed_kernel<long long>, dim3(grid), dim3(kEwThreads), 0, st, 1, static_cast<const long long*>(ids), n, seq_len, ids_stride, tok, pos, x));
    PLIP_CUDA_CHECK(launch_kernel(eos_row_kernel<long long>, dim3(grid2), dim3(kEwThreads), 0, st, 1, static_cast<const long long*>(ids), n, seq_len, ids_stride, eos_id, no_eos_argmax, eos_rows));
  } else if (ids_dtype == PLIP_IDS_I32) {
    PLIP_CUDA_CHECK(launch_kernel(text_embed_kernel<int>, dim3(grid), dim3(kEwThreads), 0, st, 1, static_cast<const int*>(ids), n, seq_len, ids_stride, tok, pos, x));
    PLIP_CUDA_CHECK(launch_kernel(eos_row_kernel<int>, dim3(grid2), dim3(kEwThreads), 0, st, 1, static_cast<const int*>(ids), n, seq_len, ids_stride, eos_id, no_eos_argmax, eos_rows));
  } else {
    set_last_error("text_embed: unknown ids dtype %d", ids_dtype);
    return -2;
  }
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_mask_to_i32(const void* mask, int dtype, int64_t count, int seq_len, int stride, int32_t* out,
                       cudaStream_t st) {
  PLIP_REQUIRE(mask && out, "mask_to_i32: null argument");
  PLIP_REQUIRE(dtype == PLIP_IDS_I32 || dtype == PLIP_IDS_I64, "mask_to_i32: unknown mask dtype %d", dtype);
  PLIP_REQUIRE(count > 0 && seq_len > 0 && stride >= seq_len && count % seq_len == 0,
               "mask_to_i32: bad shape count=%lld seq_len=%d stride=%d", (long long)count, seq_len, stride);
  PLIP_REQUIRE(aligned(mask, dtype == PLIP_IDS_I64 ? 8 : 4) && aligned(out, 4),
               "mask_to_i32: mask and out must be aligned to their element size");
  const int grid = grid_for(count, kEwThreads);
  if (dtype == PLIP_IDS_I64)
    PLIP_CUDA_CHECK(launch_kernel(mask_to_i32_kernel<long long>, dim3(grid), dim3(kEwThreads), 0, st, 1, static_cast<const long long*>(mask), count, seq_len, stride, out));
  else
    PLIP_CUDA_CHECK(launch_kernel(mask_to_i32_kernel<int>, dim3(grid), dim3(kEwThreads), 0, st, 1, static_cast<const int*>(mask), count, seq_len, stride, out));
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_cls_rows(const float* cls, const float* pos, int64_t n, int seq, float* x, cudaStream_t st) {
  PLIP_REQUIRE(cls && pos && x, "cls_rows: null argument");
  PLIP_REQUIRE(n > 0 && seq > 0, "cls_rows: bad shape n=%lld seq=%d", (long long)n, seq);
  PLIP_REQUIRE(aligned(cls, 16) && aligned(pos, 16) && aligned(x, 16), "cls_rows: cls, pos and x must be 16-byte aligned");
  PLIP_CUDA_CHECK(launch_kernel(cls_rows_kernel, dim3(grid_for(n * (kVisDim / 4), kEwThreads)), dim3(kEwThreads), 0, st, 1, cls, pos, n, seq, x));
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_gather_rows(const __nv_bfloat16* a16, const float* x32, const int32_t* row_index, int64_t row_stride,
                       int64_t n, int dim, __nv_bfloat16* a16_out, float* x32_out, cudaStream_t st) {
  PLIP_REQUIRE(n > 0 && dim > 0 && dim % 8 == 0, "gather_rows: bad shape");
  PLIP_REQUIRE(a16 && x32 && a16_out && x32_out, "gather_rows: null argument");
  PLIP_REQUIRE(row_index || row_stride >= 0, "gather_rows: negative row stride");
  PLIP_REQUIRE(aligned(a16, 16) && aligned(x32, 16) && aligned(a16_out, 16) && aligned(x32_out, 16) && aligned(row_index, 4),
               "gather_rows: a16, x32 and both outputs must be 16-byte aligned");
  const int64_t items = n * (dim / 8 + dim / 4);
  PLIP_CUDA_CHECK(launch_kernel(gather_rows_kernel, dim3(grid_for(items, kEwThreads)), dim3(kEwThreads), 0, st, 1,
                                reinterpret_cast<const uint4*>(a16), reinterpret_cast<const uint4*>(x32), row_index,
                                row_stride, n, dim, reinterpret_cast<uint4*>(a16_out), reinterpret_cast<uint4*>(x32_out)));
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_l2_normalize(float* x, int64_t rows, int dim, cudaStream_t st) {
  PLIP_REQUIRE(rows > 0 && dim > 0, "l2_normalize: bad shape");
  PLIP_CUDA_CHECK(launch_kernel(l2_normalize_kernel, dim3(grid_for(rows, kEwThreads / 32)), dim3(kEwThreads), 0, st, 1, x, rows, dim));
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace plip

// plip_b200 — the geometric part of the reference's train-time transform on the device: 224x224 RGB uint8 tiles ->
// optional horizontal flip, an affine warp and an optional perspective warp, each with Pillow's bilinear sampling.
//
// The reference's OpenPath preprocess (reproducibility/embedders/transform.py:18-42) runs torchvision's
// RandomHorizontalFlip, RandomAffine(BILINEAR, fill=127) and RandomPerspective(BILINEAR, fill=127) on PIL images,
// i.e. Image.transpose(FLIP_LEFT_RIGHT) followed by Image.transform(AFFINE) and Image.transform(PERSPECTIVE).
// Pillow's generic transform (Geometry.c) maps each output pixel centre (x + 0.5, y + 0.5) through the coefficients
// in IEEE double:
//   affine       xs = a0*x + a1*y + a2,                  ys = a3*x + a4*y + a5
//   perspective  xs = (a0*x + a1*y + a2) / (a6*x + a7*y + 1), ys = (a3*x + a4*y + a5) / (a6*x + a7*y + 1)
// A source point outside [0,224) x [0,224) keeps the fill colour.  Otherwise, with xs -= 0.5 and ys -= 0.5, it
// blends the pixels at floor(xs), floor(xs) + 1 (columns clamped to the image) of row floor(ys) (clamped) and of
// row floor(ys) + 1 (the first row again when that one is outside) as a + (b - a) * d in double, horizontally then
// vertically, and TRUNCATES the result to uint8.  Every operation here is an explicit _rn intrinsic, so nothing is
// contracted into an FMA and the tiles are bit-identical to Pillow's (tests/test_gpu_train_transform.py).
//
// The perspective reads the affine's uint8 output, so the two warps are two passes.  One CTA owns one tile: the
// affine pass reads the source tile from global memory (L2-resident, gathered bytes) into a 150,528-byte uint8 tile in
// shared memory; the second pass either runs the perspective out of shared memory or copies the tile out with
// 16-byte stores.  All reads of a tile precede all its writes, so the warp may run in place.  The flip is a column
// permutation of the source, folded into the affine pass's reads.
#include "kernels.cuh"

#include <math.h>

namespace plip {

namespace {

constexpr int kWpThreads = 512;
constexpr int kWpBatch = 128;                     // tiles per launch: descriptors travel as kernel parameters (16 KB)
constexpr int kWpTileBytes = kImage * kImage * 3;  // 150,528
constexpr int kWpPixels = kImage * kImage;

struct WarpBatch {
  plip_warp_desc_t d[kWpBatch];
};

// One bilinear sample of a 224x224 RGB uint8 image at the source point (xs, ys), Pillow's BILINEAR_HEAD / BODY.
// SRC reads byte `i` of the image; FLIP mirrors the columns first.  Returns false (fill) outside the image or for a
// point that is not a number.
template <bool FLIP, typename SRC>
__device__ __forceinline__ bool bilinear_rgb(double xs, double ys, SRC src, uint8_t (&px)[3]) {
  if (!(xs >= 0.0 && xs < (double)kImage && ys >= 0.0 && ys < (double)kImage)) return false;
  xs = __dsub_rn(xs, 0.5);
  ys = __dsub_rn(ys, 0.5);
  const int x = (int)floor(xs), y = (int)floor(ys);  // in [-1, 223]
  const double dx = __dsub_rn(xs, (double)x), dy = __dsub_rn(ys, (double)y);
  int x0 = x < 0 ? 0 : x;
  int x1 = x + 1 > kImage - 1 ? kImage - 1 : x + 1;
  if (FLIP) x0 = kImage - 1 - x0, x1 = kImage - 1 - x1;
  const int y0 = y < 0 ? 0 : y;
  const bool second = y + 1 < kImage;  // y + 1 >= 0 always holds
  const int r0 = y0 * kImage * 3, r1 = (second ? y + 1 : y0) * kImage * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double a0 = (double)src(r0 + x0 * 3 + c), b0 = (double)src(r0 + x1 * 3 + c);
    const double v1 = __dadd_rn(a0, __dmul_rn(__dsub_rn(b0, a0), dx));
    double v2 = v1;
    if (second) {
      const double a1 = (double)src(r1 + x0 * 3 + c), b1 = (double)src(r1 + x1 * 3 + c);
      v2 = __dadd_rn(a1, __dmul_rn(__dsub_rn(b1, a1), dx));
    }
    px[c] = (uint8_t)(int)__dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy));  // truncation, as Pillow's (UINT8) cast
  }
  return true;
}

__device__ __forceinline__ void store_rgb(uint8_t* p, const uint8_t (&px)[3]) {
  p[0] = px[0];
  p[1] = px[1];
  p[2] = px[2];
}

template <bool FLIP>
__device__ __forceinline__ void affine_pass(const uint8_t* src, const double* a, uint8_t fill, uint8_t* tile) {
  const auto rd = [src](int i) { return src[i]; };
  for (int p = threadIdx.x; p < kWpPixels; p += kWpThreads) {
    const int oy = p / kImage, ox = p - oy * kImage;
    const double x = (double)ox + 0.5, y = (double)oy + 0.5;
    const double xs = __dadd_rn(__dadd_rn(__dmul_rn(a[0], x), __dmul_rn(a[1], y)), a[2]);
    const double ys = __dadd_rn(__dadd_rn(__dmul_rn(a[3], x), __dmul_rn(a[4], y)), a[5]);
    uint8_t px[3] = {fill, fill, fill};
    bilinear_rgb<FLIP>(xs, ys, rd, px);
    store_rgb(tile + p * 3, px);
  }
}

// src and dst may be the same buffer (no __restrict__): a CTA reads its whole source tile before it writes.
__global__ void __launch_bounds__(kWpThreads) warp_tiles_kernel(const uint8_t* src, uint8_t* dst,
                                                                const WarpBatch batch, int64_t first_tile) {
  extern __shared__ __align__(16) uint8_t wp_smem[];
  const plip_warp_desc_t& d = batch.d[blockIdx.x];
  const int64_t t = first_tile + blockIdx.x;
  const uint8_t* in = src + t * kWpTileBytes;
  uint8_t* out = dst + t * kWpTileBytes;
  const uint8_t fill = (uint8_t)d.fill;
  if (d.flip)
    affine_pass<true>(in, d.affine, fill, wp_smem);
  else
    affine_pass<false>(in, d.affine, fill, wp_smem);
  __syncthreads();
  if (!d.apply_perspective) {
    const uint4* s4 = reinterpret_cast<const uint4*>(wp_smem);
    uint4* o4 = reinterpret_cast<uint4*>(out);
    for (int i = threadIdx.x; i < kWpTileBytes / 16; i += kWpThreads) o4[i] = s4[i];
    return;
  }
  const double* a = d.perspective;
  const auto rd = [](int i) { return wp_smem[i]; };
  for (int p = threadIdx.x; p < kWpPixels; p += kWpThreads) {
    const int oy = p / kImage, ox = p - oy * kImage;
    const double x = (double)ox + 0.5, y = (double)oy + 0.5;
    const double den = __dadd_rn(__dadd_rn(__dmul_rn(a[6], x), __dmul_rn(a[7], y)), 1.0);
    const double xs = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(a[0], x), __dmul_rn(a[1], y)), a[2]), den);
    const double ys = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(a[3], x), __dmul_rn(a[4], y)), a[5]), den);
    uint8_t px[3] = {fill, fill, fill};
    bilinear_rgb<false>(xs, ys, rd, px);
    store_rgb(out + p * 3, px);
  }
}

}  // namespace

int launch_warp_tiles(const uint8_t* src, uint8_t* dst, const plip_warp_desc_t* d, int64_t n, cudaStream_t st) {
  const char* fn = "plip_warp_tiles_u8";
  PLIP_REQUIRE(src && dst && d, "%s: null argument (src_dev %p, dst_dev %p, descs_host %p)", fn, (const void*)src,
               (const void*)dst, (const void*)d);
  PLIP_REQUIRE(n > 0, "%s: n must be positive (got %lld)", fn, (long long)n);
  PLIP_REQUIRE((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
               "%s: src_dev %p and dst_dev %p must be 16-byte aligned", fn, (const void*)src, (const void*)dst);
  {
    const uintptr_t s0 = reinterpret_cast<uintptr_t>(src), d0 = reinterpret_cast<uintptr_t>(dst);
    const uintptr_t bytes = (uintptr_t)n * kWpTileBytes;
    PLIP_REQUIRE(s0 == d0 || s0 + bytes <= d0 || d0 + bytes <= s0,
                 "%s: src_dev %p and dst_dev %p overlap without being the same buffer", fn, (const void*)src,
                 (const void*)dst);
  }
  // every descriptor is checked before anything is launched: a bad one leaves the output untouched
  for (int64_t i = 0; i < n; ++i) {
    const plip_warp_desc_t& w = d[i];
    PLIP_REQUIRE(w.flip == 0 || w.flip == 1, "%s: tile %lld: flip = %d (must be 0 or 1)", fn, (long long)i, w.flip);
    PLIP_REQUIRE(w.apply_perspective == 0 || w.apply_perspective == 1,
                 "%s: tile %lld: apply_perspective = %d (must be 0 or 1)", fn, (long long)i, w.apply_perspective);
    PLIP_REQUIRE(w.fill >= 0 && w.fill <= 255, "%s: tile %lld: fill = %d is outside 0..255", fn, (long long)i,
                 w.fill);
    for (int k = 0; k < 6; ++k)
      PLIP_REQUIRE(isfinite(w.affine[k]), "%s: tile %lld: affine[%d] = %g is not finite", fn, (long long)i, k,
                   w.affine[k]);
    if (w.apply_perspective)
      for (int k = 0; k < 8; ++k)
        PLIP_REQUIRE(isfinite(w.perspective[k]), "%s: tile %lld: perspective[%d] = %g is not finite", fn,
                     (long long)i, k, w.perspective[k]);
  }
  static unsigned long long configured = 0;
  if (first_use_on_device(configured))
    PLIP_CUDA_CHECK(cudaFuncSetAttribute(warp_tiles_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWpTileBytes));
  for (int64_t base = 0; base < n; base += kWpBatch) {
    const int cnt = (int)((n - base) < kWpBatch ? (n - base) : kWpBatch);
    static thread_local WarpBatch b;  // 16 KB: kept off the stack
    for (int i = 0; i < cnt; ++i) b.d[i] = d[base + i];
    PLIP_CUDA_CHECK(launch_kernel(warp_tiles_kernel, dim3(cnt), dim3(kWpThreads), (size_t)kWpTileBytes, st, 1, src,
                                  dst, b, base));
  }
  return 0;
}

}  // namespace plip

// plip_b200 — the distinct values of every (image, channel) of a uint8 [n, h, w, c] mask array, in one pass.
//
// The reference labels PanNuke images by counting nucleus instances per channel with
// len(np.unique(masks[i, ..., j])) - 1 (preprocess/preprocess_PanNuke.py:56-59), one np.unique per image and channel.
// Here the answer is a 256-bit set per (image, channel); everything the reference derives (instance counts, "channels
// 0..4 are all zero") is a popcount or a comparison of those sets on the host.
//
// A channel of byte `pos` of an image is pos % c (pixels are interleaved), and the image's bytes are contiguous, so
// the kernel streams the array as aligned 16-byte vectors.  A CTA owns a chunk of one image; each warp walks
// kIter x 32 consecutive vectors.  Masks are long runs of 0 and of one instance id, so a byte is only looked up when it
// differs from the byte c positions earlier (the same channel, one pixel before), which this warp has already
// inserted; the previous vector's last 8 bytes come from the neighbouring lane (or, for lane 0, from lane 31 of the
// previous step), and a vector's differing bytes are visited one set bit of a 16-bit mask at a time.  The first vector of a warp's range and the first two vectors of an image (whose predecessor bytes
// may belong to the image before) insert every byte.  An inserted byte tests its bit in the CTA's shared c x 8-word
// set before setting it, so each bit is written O(1) times per CTA; the CTA's non-zero words are then OR-ed into the
// global sets.  Roofline: HBM, each mask byte read once.
#include "kernels.cuh"

namespace plip {

namespace {

constexpr int kMsThreads = 256;
constexpr int kMsIter = 4;                                          // vectors per lane
constexpr int kMsWarpVecs = kMsIter * 32;                           // 2 KB per warp
constexpr int kMsCtaVecs = kMsWarpVecs * (kMsThreads / 32);         // 16 KB per CTA

__device__ __forceinline__ uint4 load_vec(const uint8_t* __restrict__ base, int64_t v, uint64_t total) {
  if ((uint64_t)v * 16 + 16 <= total) return __ldg(reinterpret_cast<const uint4*>(base) + v);
  uint32_t w[4] = {0, 0, 0, 0};  // the last vector of the array: only its bytes inside the array are read
  for (int i = 0; i < 16; ++i)
    if ((uint64_t)v * 16 + i < total) w[i >> 2] |= (uint32_t)base[v * 16 + i] << (8 * (i & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// blockIdx.x = image (relative to first_image) * chunks + chunk.
__global__ void __launch_bounds__(kMsThreads) mask_value_sets_kernel(const uint8_t* __restrict__ masks,
                                                                     uint64_t total_bytes, int64_t first_image,
                                                                     int image_bytes, int c, int chunks,
                                                                     uint32_t* __restrict__ sets) {
  __shared__ uint32_t set[8 * 8];
  __shared__ uint8_t chan_of[8 * 16];  // [channel of byte 0][b]: the channel of byte b of a vector
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t n = first_image + blockIdx.x / chunks;
  const int chunk = blockIdx.x % chunks;
  const int64_t img0 = n * image_bytes;                 // first byte of the image
  const int64_t v0 = img0 >> 4, v1 = (img0 + image_bytes + 15) >> 4;  // vectors touching the image
  const int64_t cta0 = v0 + (int64_t)chunk * kMsCtaVecs;
  if (t < 8 * c) set[t] = 0;
  if (t < 8 * 16) chan_of[t] = (uint8_t)((t / 16 + t % 16) % c);
  __syncthreads();
  if (cta0 < v1) {
    const int64_t wv = cta0 + warp * kMsWarpVecs;
    const int64_t vend = min(v1, cta0 + kMsCtaVecs);
    uint4 x[kMsIter];
#pragma unroll
    for (int i = 0; i < kMsIter; ++i) {
      const int64_t v = wv + i * 32 + lane;
      x[i] = v < vend ? load_vec(masks, v, total_bytes) : make_uint4(0, 0, 0, 0);
    }
    const int q = (8 - c) >> 2, sh = ((8 - c) & 3) * 8;  // byte i - c of [previous bytes 8..15 | current 0..15]
    uint32_t carry_z = 0, carry_w = 0;
#pragma unroll
    for (int i = 0; i < kMsIter; ++i) {
      const int64_t v = wv + i * 32 + lane;
      uint32_t pz = __shfl_up_sync(0xffffffffu, x[i].z, 1), pw = __shfl_up_sync(0xffffffffu, x[i].w, 1);
      if (lane == 0) pz = carry_z, pw = carry_w;
      carry_z = __shfl_sync(0xffffffffu, x[i].z, 31);
      carry_w = __shfl_sync(0xffffffffu, x[i].w, 31);
      if (v >= vend) continue;
      const uint32_t u[6] = {pz, pw, x[i].x, x[i].y, x[i].z, x[i].w};
      uint32_t ne[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t lo = q ? u[k + 1] : u[k], hi = q ? u[k + 2] : u[k + 1];
        ne[k] = __vcmpne4(u[k + 2], __funnelshift_r(lo, hi, sh));
      }
      uint32_t m = 0;  // bit b: byte b differs from the byte c positions earlier
#pragma unroll
      for (int k = 0; k < 4; ++k) m |= (((ne[k] & 0x01010101u) * 0x10204080u) >> 28) << (4 * k);
      if ((i == 0 && lane == 0) || v <= v0 + 1) m = 0xffffu;
      if (!m) continue;
      const int64_t pos0 = v * 16 - img0;             // image byte of the vector's first byte (may be negative)
      const int lo = pos0 < 0 ? (int)-pos0 : 0;
      const int hi = image_bytes - pos0 < 16 ? (int)(image_bytes - pos0) : 16;
      m &= (0xffffu >> (16 - hi)) & (0xffffu << lo);
      const uint8_t* chan = chan_of + ((pos0 % c) + c) % c * 16;
      while (m) {
        const int b = __ffs(m) - 1;
        m &= m - 1;
        const uint32_t word = b < 8 ? (b < 4 ? u[2] : u[3]) : (b < 12 ? u[4] : u[5]);
        const uint32_t val = (word >> (8 * (b & 3))) & 0xffu;
        uint32_t* wd = set + chan[b] * 8 + (val >> 5);
        const uint32_t bit = 1u << (val & 31);
        if (!(*reinterpret_cast<volatile uint32_t*>(wd) & bit)) atomicOr(wd, bit);
      }
    }
  }
  __syncthreads();
  if (t < 8 * c && set[t]) atomicOr(sets + n * 8 * c + t, set[t]);
}

}  // namespace

int launch_mask_value_sets(const uint8_t* masks, int64_t n, int h, int w, int c, uint32_t* sets, cudaStream_t st) {
  const char* fn = "plip_mask_value_sets_u8";
  PLIP_REQUIRE(masks && sets, "%s: null argument", fn);
  PLIP_REQUIRE(n > 0, "%s: n must be positive (got %lld)", fn, (long long)n);
  PLIP_REQUIRE(h > 0 && w > 0, "%s: image size %dx%d must be positive", fn, h, w);
  PLIP_REQUIRE(c >= 1 && c <= 8, "%s: channels must be 1..8 (got %d)", fn, c);
  const int64_t image_bytes = (int64_t)h * w * c;
  PLIP_REQUIRE(image_bytes <= 0x7fffffffLL, "%s: an image of %dx%dx%d bytes exceeds 2^31 - 1", fn, h, w, c);
  PLIP_REQUIRE(reinterpret_cast<uintptr_t>(masks) % 16 == 0, "%s: masks_dev must be 16-byte aligned", fn);
  PLIP_REQUIRE(reinterpret_cast<uintptr_t>(sets) % 4 == 0, "%s: sets_dev must be 4-byte aligned", fn);
  PLIP_CUDA_CHECK(cudaMemsetAsync(sets, 0, (size_t)n * c * 8 * sizeof(uint32_t), st));
  // an image touches at most image_bytes / 16 + 2 vectors
  const int chunks = (int)((image_bytes / 16 + 2 + kMsCtaVecs - 1) / kMsCtaVecs);
  const int64_t per_launch = 0x7fffffffLL / chunks;
  for (int64_t i = 0; i < n; i += per_launch) {
    const int64_t cnt = n - i < per_launch ? n - i : per_launch;
    PLIP_CUDA_CHECK(launch_kernel(mask_value_sets_kernel, dim3((unsigned)(cnt * chunks)), dim3(kMsThreads), 0, st, 1,
                                  masks, (uint64_t)(n * image_bytes), i, (int)image_bytes, c, chunks, sets));
  }
  return 0;
}

}  // namespace plip

// plip_b200 — image resize + crop on the device: variable-size RGB uint8 images -> 224x224 uint8 tiles.
//
// Replaces the PIL pass the reference runs on the host before every forward: CLIPProcessor's shortest-edge
// bicubic resize + centre crop (/root/reference/plip.py:35; TF:models/clip/image_processing_clip.py:50-62) and
// torchvision's Resize(n_px, BICUBIC) + CenterCrop (reproducibility/embedders/transform.py:45-52), both of which
// end in Pillow's ImagingResample: separable antialiased bicubic (a = -0.5), window half-width 2*max(scale,1),
// double-precision weights normalised per output pixel and quantised to 22-bit fixed point, int32 accumulation
// from 1<<21, >>22 and clamp, uint8 image between the horizontal and the vertical pass.  The result here is
// bit-identical to PIL.Image.resize(...).crop(...) (tests/test_resize.py): the weights are rebuilt on the device
// with the same sequence of IEEE double operations (explicit _rn intrinsics: no FMA contraction).
//
// One CTA produces 32 output rows of one tile (7 CTAs per image).  Its 256 threads first build the 224
// horizontal filter rows it needs (only the cropped columns) and its 32 vertical ones in shared memory, zero-padded
// to a multiple of 4 taps.  Then, for `rows_per_pass` output rows at a time, the horizontal pass runs over the
// source rows those outputs touch — one thread per output column walking down the rows, all 3 channels, source
// bytes fetched as aligned 32-bit words and re-aligned with funnel shifts (4 pixels = 3 words per step; weights in
// registers for filters of up to 7 taps, else 16-byte shared loads) — into a uint8 shared-memory strip, and the
// vertical pass runs out of that strip, one thread per 4 output bytes.
// Source pixels are read once per strip (strips overlap by the filter support; L2 absorbs the re-reads); the
// roofline is HBM (source bytes + 150,528 tile bytes per image) but the kernel is issue-bound: H_src x 224 x 3 x
// taps integer MACs per image with ~3 instructions each.
#include "kernels.cuh"

#include <math.h>
#include <stdlib.h>

namespace plip {

namespace {

constexpr int kRsThreads = 256;
constexpr int kRsRowsPerCta = 32;
constexpr int kRsBatch = 512;                // images per launch: descriptors travel as kernel parameters (20 KB;
                                             // CUDA >= 12.1 allows 32,764 bytes on sm_70+)
constexpr int kTileRowBytes = kImage * 3;    // 672
constexpr int kPrecisionBits = 32 - 8 - 2;   // Pillow's PRECISION_BITS for 8-bit channels

struct ResizeImg {
  long long src_off;   // byte offset of the image in the packed source buffer
  int w, h;            // source size
  int new_w, new_h;    // size after the resize
  int left, top;       // crop origin in the resized image
  int rows_per_pass;   // output rows per strip (32, 16, ... or 1)
  int strip_rows;      // capacity of the uint8 strip, in source rows
};

struct ResizeBatch {
  ResizeImg img[kRsBatch];
};

struct AxisFilter {
  double scale, support, ss;
  int ksize;
};

// IEEE double operations without FMA contraction: intrinsics on the device, plain operators on the host (x86-64
// gcc does not contract without -mfma).  The host instantiation only serves plip_dbg_resize_filter (CPU tests).
#ifdef __CUDA_ARCH__
#define RN_ADD(a, b) __dadd_rn((a), (b))
#define RN_SUB(a, b) __dsub_rn((a), (b))
#define RN_MUL(a, b) __dmul_rn((a), (b))
#define RN_DIV(a, b) __ddiv_rn((a), (b))
#else
#define RN_ADD(a, b) ((a) + (b))
#define RN_SUB(a, b) ((a) - (b))
#define RN_MUL(a, b) ((a) * (b))
#define RN_DIV(a, b) ((a) / (b))
#endif

// BILINEAR selects Pillow's triangle filter (support 1) instead of its bicubic one (support 2): the same
// ImagingResample, used by torchvision's Resize(BILINEAR) on PIL images.
template <bool BILINEAR = false>
__host__ __device__ inline int axis_ksize(int in_size, int out_size) {
  double fs = (double)in_size / (double)out_size;
  if (fs < 1.0) fs = 1.0;
  return (int)ceil((BILINEAR ? 1.0 : 2.0) * fs) * 2 + 1;
}

template <bool BILINEAR = false>
__host__ __device__ __forceinline__ AxisFilter make_axis(int in_size, int out_size) {
  AxisFilter f;
  f.scale = RN_DIV((double)in_size, (double)out_size);
  const double fs = f.scale < 1.0 ? 1.0 : f.scale;
  f.support = RN_MUL(BILINEAR ? 1.0 : 2.0, fs);
  f.ksize = (int)ceil(f.support) * 2 + 1;
  f.ss = RN_DIV(1.0, fs);
  return f;
}

__host__ __device__ __forceinline__ double bicubic_rn(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return RN_ADD(RN_MUL(RN_MUL(RN_SUB(RN_MUL(a + 2.0, x), a + 3.0), x), x), 1.0);
  if (x < 2.0) return RN_MUL(RN_SUB(RN_MUL(RN_ADD(RN_MUL(RN_SUB(x, 5.0), x), 8.0), x), 4.0), a);
  return 0.0;
}

__host__ __device__ __forceinline__ double triangle_rn(double x) {
  if (x < 0.0) x = -x;
  if (x < 1.0) return RN_SUB(1.0, x);
  return 0.0;
}

template <bool BILINEAR>
__host__ __device__ __forceinline__ double filter_rn(double x) {
  return BILINEAR ? triangle_rn(x) : bicubic_rn(x);
}

// Filter row of output index `xx`: window [xmin, xmin+count) and fixed-point weights k[0..count).
template <bool BILINEAR = false>
__host__ __device__ __forceinline__ void filter_row(const AxisFilter& f, int in_size, int xx, int* k,
                                                    int& xmin_out, int& count_out) {
  const double center = RN_MUL((double)xx + 0.5, f.scale);
  int xmin = (int)RN_ADD(RN_SUB(center, f.support), 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)RN_ADD(RN_ADD(center, f.support), 0.5);
  if (xmax > in_size) xmax = in_size;
  const int count = xmax - xmin;
  double ww = 0.0;
  for (int x = 0; x < count; ++x)
    ww = RN_ADD(ww, filter_rn<BILINEAR>(RN_MUL(RN_ADD(RN_SUB((double)(x + xmin), center), 0.5), f.ss)));
  const double one = (double)(1 << kPrecisionBits);
  for (int x = 0; x < count; ++x) {
    double w = filter_rn<BILINEAR>(RN_MUL(RN_ADD(RN_SUB((double)(x + xmin), center), 0.5), f.ss));
    if (ww != 0.0) w = RN_DIV(w, ww);
    k[x] = w < 0.0 ? (int)RN_ADD(-0.5, RN_MUL(w, one)) : (int)RN_ADD(0.5, RN_MUL(w, one));
  }
  xmin_out = xmin;
  count_out = count;
}

__device__ __forceinline__ uint32_t clip8(int acc) {
  const int v = acc >> kPrecisionBits;
  return (uint32_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__device__ __forceinline__ int byte_of(uint32_t w, int i) { return (int)__byte_perm(w, 0, 0x4440 + i); }

// Aligned 32-bit read of the source; the last (partial) word of the buffer is assembled from its valid bytes.
template <bool GUARD>
__device__ __forceinline__ uint32_t src_word(const uint32_t* q, const uint32_t* end_w, const uint8_t* end_b) {
  if (!GUARD || q < end_w) return __ldg(q);
  uint32_t w = 0;
  const uint8_t* b = reinterpret_cast<const uint8_t*>(q);
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (b + i < end_b) w |= (uint32_t)__ldg(b + i) << (8 * i);
  return w;
}

// Four taps of one output pixel of the horizontal pass, all 3 channels: the next 12 source bytes are fetched as
// aligned words and re-aligned with funnel shifts (`prev` carries the last word over to the next group).
template <bool GUARD>
__device__ __forceinline__ void hgroup(const uint32_t*& wp, uint32_t& prev, uint32_t sh, const int4 kk,
                                       const uint32_t* end_w, const uint8_t* end_b, int& a0, int& a1, int& a2) {
  const uint32_t w1 = src_word<GUARD>(wp + 1, end_w, end_b), w2 = src_word<GUARD>(wp + 2, end_w, end_b),
                 w3 = src_word<GUARD>(wp + 3, end_w, end_b);
  const uint32_t s0 = __funnelshift_r(prev, w1, sh), s1 = __funnelshift_r(w1, w2, sh),
                 s2 = __funnelshift_r(w2, w3, sh);
  prev = w3;
  wp += 3;
  a0 += byte_of(s0, 0) * kk.x + byte_of(s0, 3) * kk.y + byte_of(s1, 2) * kk.z + byte_of(s2, 1) * kk.w;
  a1 += byte_of(s0, 1) * kk.x + byte_of(s1, 0) * kk.y + byte_of(s1, 3) * kk.z + byte_of(s2, 2) * kk.w;
  a2 += byte_of(s0, 2) * kk.x + byte_of(s1, 1) * kk.y + byte_of(s2, 0) * kk.z + byte_of(s2, 3) * kk.w;
}

// One output pixel: `cnt4` taps (a multiple of 4; weights beyond the window are zero) from shared memory.
template <bool GUARD>
__device__ __forceinline__ void hpass_pixel(const uint8_t* p, const int* __restrict__ k, int cnt4,
                                            const uint32_t* end_w, const uint8_t* end_b, int& a0, int& a1, int& a2) {
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3);
  const uint32_t* wp = reinterpret_cast<const uint32_t*>(p - mis);
  uint32_t prev = src_word<GUARD>(wp, end_w, end_b);
  const int4* k4 = reinterpret_cast<const int4*>(k);
  for (int x = 0; x < cnt4; x += 4) hgroup<GUARD>(wp, prev, mis * 8, *k4++, end_w, end_b, a0, a1, a2);
}

// One output pixel with exactly 8 (zero-padded) taps held in registers: every filter up to 7 taps, i.e. any
// scale factor <= 1.5 and all upscaling.
template <bool GUARD>
__device__ __forceinline__ void hpass_pixel8(const uint8_t* p, const int4 k0, const int4 k1, const uint32_t* end_w,
                                             const uint8_t* end_b, int& a0, int& a1, int& a2) {
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3);
  const uint32_t* wp = reinterpret_cast<const uint32_t*>(p - mis);
  uint32_t prev = src_word<GUARD>(wp, end_w, end_b);
  hgroup<GUARD>(wp, prev, mis * 8, k0, end_w, end_b, a0, a1, a2);
  hgroup<GUARD>(wp, prev, mis * 8, k1, end_w, end_b, a0, a1, a2);
}

template <bool BILINEAR>
__device__ __forceinline__ void resize_crop_body(const uint8_t* __restrict__ src, uint64_t src_bytes,
                                                 uint8_t* __restrict__ tiles, const ResizeBatch& batch,
                                                 int64_t first_image) {
  extern __shared__ __align__(16) uint8_t rs_smem[];
  const ResizeImg& im = batch.img[blockIdx.y];
  const int row0 = blockIdx.x * kRsRowsPerCta;  // first output row of this CTA
  const AxisFilter fh = make_axis<BILINEAR>(im.w, im.new_w), fv = make_axis<BILINEAR>(im.h, im.new_h);
  const int ksh4 = (fh.ksize + 3) & ~3, ksv4 = (fv.ksize + 3) & ~3;  // filter rows zero-padded to 4 taps

  int* kh = reinterpret_cast<int*>(rs_smem);                 // [224][ksh4]
  int* kv = kh + kImage * ksh4;                              // [32][ksv4]
  int* bh = kv + kRsRowsPerCta * ksv4;                       // [224][2] (xmin, count)
  int* bv = bh + kImage * 2;                                 // [32][2]
  uint8_t* strip = reinterpret_cast<uint8_t*>(bv + kRsRowsPerCta * 2);  // [strip_rows + 3][224*3], 16-byte aligned

  const int t = threadIdx.x;
  {
    const bool horiz = t < kImage;
    const int j = horiz ? t : t - kImage;
    int* k = horiz ? kh + j * ksh4 : kv + j * ksv4;
    int lo, cnt;
    if (horiz)
      filter_row<BILINEAR>(fh, im.w, im.left + j, k, lo, cnt);
    else
      filter_row<BILINEAR>(fv, im.h, im.top + row0 + j, k, lo, cnt);
    for (int x = cnt; x < (horiz ? ksh4 : ksv4); ++x) k[x] = 0;
    int* bnd = horiz ? bh + 2 * j : bv + 2 * j;
    bnd[0] = lo;
    bnd[1] = cnt;
  }
  __syncthreads();

  const uint8_t* img = src + im.src_off;
  const int64_t src_row_bytes = (int64_t)im.w * 3;
  const uint8_t* end_b = src + src_bytes;
  const uint32_t* end_w = reinterpret_cast<const uint32_t*>(src + (src_bytes & ~(uint64_t)3));  // src is 4-aligned
  uint8_t* out = tiles + ((first_image + blockIdx.y) * kImage + row0) * (int64_t)kTileRowBytes;
  const int rp = im.rows_per_pass;
  constexpr int kRowWords = kTileRowBytes / 4;  // 168
  for (int sub = 0; sub < kRsRowsPerCta; sub += rp) {
    const int s0 = bv[2 * sub];
    const int s1 = bv[2 * (sub + rp - 1)] + bv[2 * (sub + rp - 1) + 1];
    const int nrows = s1 - s0;
    if (nrows > im.strip_rows) __trap();  // host sizing bug: never expected
    // horizontal pass: strip[r][xx][0..2] for the source rows [s0, s1).  Thread t owns output column t (window,
    // weights and pointers are then loop invariants) and walks down the rows; threads 224..255 sit this out.
    if (t < kImage) {
      const uint8_t* p = img + (int64_t)s0 * src_row_bytes + (int64_t)bh[2 * t] * 3;
      const uint8_t* lim = reinterpret_cast<const uint8_t*>(end_w);
      uint8_t* d = strip + t * 3;
      if (ksh4 == 8) {
        const int4 k0 = reinterpret_cast<const int4*>(kh + t * 8)[0], k1 = reinterpret_cast<const int4*>(kh + t * 8)[1];
        for (int r = 0; r < nrows; ++r, p += src_row_bytes, d += kTileRowBytes) {
          int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
          // words read: [p & ~3, ... + 28) bytes; only the very end of the source buffer needs the guard
          if (p + 32 <= lim)
            hpass_pixel8<false>(p, k0, k1, end_w, end_b, a0, a1, a2);
          else
            hpass_pixel8<true>(p, k0, k1, end_w, end_b, a0, a1, a2);
          d[0] = (uint8_t)clip8(a0);
          d[1] = (uint8_t)clip8(a1);
          d[2] = (uint8_t)clip8(a2);
        }
      } else {
        const int cnt4 = (bh[2 * t + 1] + 3) & ~3;
        const int* k = kh + t * ksh4;
        for (int r = 0; r < nrows; ++r, p += src_row_bytes, d += kTileRowBytes) {
          int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
          if (p + 3 * cnt4 + 8 <= lim)  // words read: [p & ~3, ... + 3*cnt4 + 4) bytes
            hpass_pixel<false>(p, k, cnt4, end_w, end_b, a0, a1, a2);
          else
            hpass_pixel<true>(p, k, cnt4, end_w, end_b, a0, a1, a2);
          d[0] = (uint8_t)clip8(a0);
          d[1] = (uint8_t)clip8(a1);
          d[2] = (uint8_t)clip8(a2);
        }
      }
    }
    __syncthreads();
    // vertical pass: rp output rows out of the strip; one thread per 4 output bytes
    for (int idx = t; idx < rp * kRowWords; idx += kRsThreads) {
      const int j = idx / kRowWords, e = idx - j * kRowWords;
      const int ymin = bv[2 * (sub + j)], cnt4 = (bv[2 * (sub + j) + 1] + 3) & ~3;
      const uint32_t* sp = reinterpret_cast<const uint32_t*>(strip + (ymin - s0) * kTileRowBytes) + e;
      const int4* k4 = reinterpret_cast<const int4*>(kv + (sub + j) * ksv4);
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0, a3 = a0;
      for (int y = 0; y < cnt4; y += 4) {   // taps beyond the window have zero weight (rows exist: strip has +3)
        const int4 kk = *k4++;
        const uint32_t w0 = sp[0], w1 = sp[kRowWords], w2 = sp[2 * kRowWords], w3 = sp[3 * kRowWords];
        sp += 4 * kRowWords;
        a0 += byte_of(w0, 0) * kk.x + byte_of(w1, 0) * kk.y + byte_of(w2, 0) * kk.z + byte_of(w3, 0) * kk.w;
        a1 += byte_of(w0, 1) * kk.x + byte_of(w1, 1) * kk.y + byte_of(w2, 1) * kk.z + byte_of(w3, 1) * kk.w;
        a2 += byte_of(w0, 2) * kk.x + byte_of(w1, 2) * kk.y + byte_of(w2, 2) * kk.z + byte_of(w3, 2) * kk.w;
        a3 += byte_of(w0, 3) * kk.x + byte_of(w1, 3) * kk.y + byte_of(w2, 3) * kk.z + byte_of(w3, 3) * kk.w;
      }
      reinterpret_cast<uint32_t*>(out + (sub + j) * kTileRowBytes)[e] =
          clip8(a0) | (clip8(a1) << 8) | (clip8(a2) << 16) | (clip8(a3) << 24);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kRsThreads) resize_crop_kernel(const uint8_t* __restrict__ src, uint64_t src_bytes,
                                                                 uint8_t* __restrict__ tiles, const ResizeBatch batch,
                                                                 int64_t first_image) {
  resize_crop_body<false>(src, src_bytes, tiles, batch, first_image);
}

// The same with Pillow's bilinear (triangle) filter: torchvision's Resize(n, BILINEAR) + CenterCrop on PIL images.
__global__ void __launch_bounds__(kRsThreads) resize_crop_bilinear_kernel(const uint8_t* __restrict__ src,
                                                                          uint64_t src_bytes,
                                                                          uint8_t* __restrict__ tiles,
                                                                          const ResizeBatch batch,
                                                                          int64_t first_image) {
  resize_crop_body<true>(src, src_bytes, tiles, batch, first_image);
}

constexpr size_t kRsSmemHard = 200 * 1024;

size_t table_bytes(int ksh, int ksv) {
  const size_t ksh4 = (ksh + 3) & ~3, ksv4 = (ksv + 3) & ~3;
  return ((size_t)kImage * ksh4 + (size_t)kRsRowsPerCta * ksv4 + (kImage + kRsRowsPerCta) * 2) * sizeof(int);
}

// Source rows one strip of `rp` output rows can touch: (rp-1)*scale + 2*support + rounding slack.
int strip_rows_for(int in_h, int out_h, int rp) {
  const double scale = (double)in_h / (double)out_h;
  const double support = 2.0 * (scale < 1.0 ? 1.0 : scale);
  int rows = (int)ceil((rp - 1) * scale + 2.0 * support) + 3;
  return rows > in_h ? in_h : rows;
}

constexpr int kStripPadRows = 3;  // the vertical pass reads whole groups of 4 rows

}  // namespace

int resize_filter_host(int in_size, int out_size, int xx, int32_t* k, int k_cap, int* xmin, int* count) {
  const AxisFilter f = make_axis(in_size, out_size);
  if (k_cap < f.ksize) return -f.ksize;
  filter_row(f, in_size, xx, k, *xmin, *count);
  return f.ksize;
}

int resize_filter_bilinear_host(int in_size, int out_size, int xx, int32_t* k, int k_cap, int* xmin, int* count) {
  const AxisFilter f = make_axis<true>(in_size, out_size);
  if (k_cap < f.ksize) return -f.ksize;
  filter_row<true>(f, in_size, xx, k, *xmin, *count);
  return f.ksize;
}

// Validates descriptor `idx` and fills the kernel-side plan (strip height, shared memory need).
// Tables and strips are sized for the bicubic filter; the bilinear one's windows lie inside the bicubic ones, so the
// same plan also holds it (with some shared memory to spare).  `fn` names the entry point in errors.
static int plan_image(const char* fn, const plip_resize_desc_t& s, long long idx, size_t src_bytes, ResizeImg& o,
                      size_t& need_out) {
  PLIP_REQUIRE(s.width > 0 && s.height > 0 && s.width <= 65536 && s.height <= 65536,
               "%s: image %lld has invalid size %dx%d", fn, idx, s.width, s.height);
  PLIP_REQUIRE(s.offset >= 0 && (uint64_t)s.offset + (uint64_t)s.width * s.height * 3 <= src_bytes,
               "%s: image %lld (%dx%d at byte %lld) exceeds the %llu-byte source buffer", fn, idx,
               s.width, s.height, (long long)s.offset, (unsigned long long)src_bytes);
  PLIP_REQUIRE(s.new_width >= kImage && s.new_height >= kImage && s.new_width <= 65536 && s.new_height <= 65536,
               "%s: image %lld: resized size %dx%d is smaller than the %dx%d tile", fn, idx,
               s.new_width, s.new_height, kImage, kImage);
  PLIP_REQUIRE(s.left >= 0 && s.top >= 0 && s.left + kImage <= s.new_width && s.top + kImage <= s.new_height,
               "%s: image %lld: crop origin (%d,%d) leaves the %dx%d resized image", fn, idx, s.left,
               s.top, s.new_width, s.new_height);
  const int ksh = axis_ksize(s.width, s.new_width), ksv = axis_ksize(s.height, s.new_height);
  const size_t tb = table_bytes(ksh, ksv);
  // Strip height: taller strips re-read fewer source rows (adjacent strips overlap by the filter support),
  // shorter ones need less shared memory and keep more CTAs per SM.  Relative throughput by resident CTAs
  // (tools/resize_probe.py measures it; these weights have not been re-measured on H100); registers cap residency at 5.
  static const double kThroughput[6] = {0.0, 1.0, 1.12, 1.21, 1.57, 1.70};
  const double vscale = (double)s.height / (double)s.new_height, fs = vscale < 1.0 ? 1.0 : vscale;
  int rp = 0, rows = 0;
  double best = 0.0;
  for (int cand = kRsRowsPerCta; cand >= 1; cand >>= 1) {
    const int r = strip_rows_for(s.height, s.new_height, cand);
    const size_t need = tb + (size_t)(r + kStripPadRows) * kTileRowBytes;
    if (need > kRsSmemHard) continue;
    int resident = (int)((size_t)227 * 1024 / (need + 1024));
    resident = resident > 5 ? 5 : resident;
    const double reread = ((cand - 1) * vscale + 4.0 * fs + 1.0) / (cand * vscale);
    const double score = kThroughput[resident] / reread;
    if (score > best) best = score, rp = cand, rows = r;
  }
  PLIP_REQUIRE(rp, "%s: image %lld (%dx%d -> %dx%d) shrinks too much for the on-device "
               "resize (filter tables need %zu bytes of shared memory); reduce it on the host first",
               fn, idx, s.width, s.height, s.new_width, s.new_height, tb);
  o.src_off = s.offset;
  o.w = s.width, o.h = s.height, o.new_w = s.new_width, o.new_h = s.new_height;
  o.left = s.left, o.top = s.top, o.rows_per_pass = rp, o.strip_rows = rows;
  need_out = tb + (size_t)(rows + kStripPadRows) * kTileRowBytes;
  return 0;
}

int launch_resize_crop(const uint8_t* src, size_t src_bytes, const plip_resize_desc_t* d, int64_t n, uint8_t* tiles,
                       cudaStream_t st, bool bilinear) {
  const char* fn = bilinear ? "plip_resize_crop_bilinear_u8" : "plip_resize_crop_u8";
  PLIP_REQUIRE(reinterpret_cast<uintptr_t>(src) % 4 == 0 && reinterpret_cast<uintptr_t>(tiles) % 4 == 0,
               "%s: src_dev and tiles_dev must be 4-byte aligned", fn);
  // every descriptor is checked before anything is launched: a bad one leaves the output untouched
  {
    ResizeImg scratch;
    size_t need;
    for (int64_t i = 0; i < n; ++i)
      if (int rc = plan_image(fn, d[i], (long long)i, src_bytes, scratch, need)) return rc;
  }
  auto kernel = bilinear ? resize_crop_bilinear_kernel : resize_crop_kernel;
  static unsigned long long configured[2] = {0, 0};
  if (first_use_on_device(configured[bilinear]))
    PLIP_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRsSmemHard));
  for (int64_t base = 0; base < n; base += kRsBatch) {
    const int cnt = (int)((n - base) < kRsBatch ? (n - base) : kRsBatch);
    static thread_local ResizeBatch b;  // 20 KB: kept off the stack
    size_t smem = 0;
    for (int i = 0; i < cnt; ++i) {
      size_t need = 0;
      if (int rc = plan_image(fn, d[base + i], (long long)(base + i), src_bytes, b.img[i], need)) return rc;
      smem = need > smem ? need : smem;
    }
    PLIP_CUDA_CHECK(launch_kernel(kernel, dim3(kImage / kRsRowsPerCta, cnt), dim3(kRsThreads), smem, st, 1,
                               src, (uint64_t)src_bytes, tiles, b, base));
  }
  return 0;
}

// ---- whole-image resize (plip_resize_region_u8) --------------------------------------------------------------------
// The same resample at any shrink, whole output rows instead of a 224 x 224 crop: Pillow's own two passes through a
// uint8 intermediate in global memory, so no filter table or strip has to fit in shared memory at once.
//   1. resize_filters_kernel: the filter rows of every output column and of the requested output rows, one thread
//      each (make_axis + filter_row, as above), zero-padded to a multiple of 4 taps.
//   2. resize_rows_h_kernel: CTAs of 64 output columns x 64 source rows; the columns' filter rows are staged in shared
//      memory and each thread walks down rows of one column (hpass_pixel) into the intermediate
//      [s1 - s0 + 3][new_w * 3 rounded up to 4 bytes] (source rows [s0, s1) that the requested output rows touch).
//   3. resize_rows_v_kernel: one CTA row per output row, one thread per 4 output bytes; the row's filter is read
//      through the read-only cache (the same address in every lane).
// Roofline: HBM, source + 2 x intermediate + output bytes.  An output-row range [o0, o1) uses the filters of the full
// image, so ranges stitched together are the whole image bit for bit.
namespace {

constexpr int kRgCols = 64;                         // output columns per horizontal-pass CTA
constexpr int kRgRowLanes = kRsThreads / kRgCols;   // threads per column
constexpr int kRgRowsPerCta = 64;                   // source rows per horizontal-pass CTA
constexpr size_t kRgSmemHard = 200 * 1024;

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

struct RegionPlan {
  int ksh4, ksv4;
  int s0, s1;                // source rows the vertical windows of the output rows cover
  int64_t tmp_pitch;         // intermediate row pitch in bytes (a multiple of 4)
  size_t kh, bh, kv, bv, tmp, total;  // workspace offsets (16-byte aligned) and size
};

__global__ void __launch_bounds__(kRsThreads) resize_filters_kernel(int w, int new_w, int h, int new_h, int o0, int nv,
                                                                    int ksh4, int ksv4, int* __restrict__ kh,
                                                                    int2* __restrict__ bh, int* __restrict__ kv,
                                                                    int2* __restrict__ bv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= new_w + nv) return;
  const bool horiz = i < new_w;
  const int j = horiz ? i : i - new_w, k4 = horiz ? ksh4 : ksv4;
  int* k = (horiz ? kh : kv) + (size_t)j * k4;
  int lo, cnt;
  if (horiz)
    filter_row(make_axis(w, new_w), w, j, k, lo, cnt);
  else
    filter_row(make_axis(h, new_h), h, o0 + j, k, lo, cnt);
  for (int x = cnt; x < k4; ++x) k[x] = 0;
  (horiz ? bh : bv)[j] = make_int2(lo, cnt);
}

// src: the first of `rows` source rows to filter (the band's row s0); src_bytes: readable bytes from src on.
__global__ void __launch_bounds__(kRsThreads) resize_rows_h_kernel(const uint8_t* __restrict__ src, int64_t pitch,
                                                                   uint64_t src_bytes, int rows, int new_w, int ksh4,
                                                                   const int* __restrict__ kh,
                                                                   const int2* __restrict__ bh,
                                                                   uint8_t* __restrict__ tmp, int64_t tmp_pitch) {
  extern __shared__ __align__(16) uint8_t rs_smem[];
  int* ks = reinterpret_cast<int*>(rs_smem);  // [kRgCols][ksh4]
  const int c0 = blockIdx.x * kRgCols;
  const int ncols = min(kRgCols, new_w - c0);
  const int4* g4 = reinterpret_cast<const int4*>(kh + (size_t)c0 * ksh4);
  for (int i = threadIdx.x; i < ncols * ksh4 / 4; i += kRsThreads) reinterpret_cast<int4*>(ks)[i] = g4[i];
  __syncthreads();
  const int c = threadIdx.x % kRgCols, lane = threadIdx.x / kRgCols;
  if (c >= ncols) return;
  const int2 b = bh[c0 + c];
  const int cnt4 = (b.y + 3) & ~3;
  const int* k = ks + c * ksh4;
  const uint8_t* end_b = src + src_bytes;
  const uint32_t* end_w = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(end_b) & ~(uintptr_t)3);
  const uint8_t* lim = reinterpret_cast<const uint8_t*>(end_w);
  const int r1 = min(rows, (int)(blockIdx.y + 1) * kRgRowsPerCta);
  for (int r = blockIdx.y * kRgRowsPerCta + lane; r < r1; r += kRgRowLanes) {
    const uint8_t* p = src + (int64_t)r * pitch + (int64_t)b.x * 3;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    if (p + 3 * cnt4 + 8 <= lim)  // words read: [p & ~3, ... + 3*cnt4 + 4) bytes
      hpass_pixel<false>(p, k, cnt4, end_w, end_b, a0, a1, a2);
    else
      hpass_pixel<true>(p, k, cnt4, end_w, end_b, a0, a1, a2);
    uint8_t* d = tmp + (int64_t)r * tmp_pitch + (c0 + c) * 3;
    d[0] = (uint8_t)clip8(a0);
    d[1] = (uint8_t)clip8(a1);
    d[2] = (uint8_t)clip8(a2);
  }
}

// tmp row 0 is source row s0; out: output row o0 (blockIdx.x = 0); row_bytes = new_w * 3.
__global__ void __launch_bounds__(kRsThreads) resize_rows_v_kernel(const uint8_t* __restrict__ tmp, int64_t tmp_pitch,
                                                                   int s0, const int* __restrict__ kv,
                                                                   const int2* __restrict__ bv, int ksv4,
                                                                   uint8_t* __restrict__ out, int64_t out_pitch,
                                                                   int row_bytes) {
  const int j = blockIdx.x;
  const int e = blockIdx.y * kRsThreads + threadIdx.x;  // 32-bit word of the row
  if (4 * e >= row_bytes) return;
  const int2 b = __ldg(bv + j);
  const int cnt4 = (b.y + 3) & ~3;
  const int tw = (int)(tmp_pitch / 4);
  const uint32_t* sp = reinterpret_cast<const uint32_t*>(tmp + (int64_t)(b.x - s0) * tmp_pitch) + e;
  const int4* k4 = reinterpret_cast<const int4*>(kv + (size_t)j * ksv4);
  int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0, a3 = a0;
  for (int y = 0; y < cnt4; y += 4) {  // taps beyond the window have zero weight (the intermediate has 3 spare rows)
    const int4 kk = __ldg(k4++);
    const uint32_t w0 = __ldg(sp), w1 = __ldg(sp + tw), w2 = __ldg(sp + 2 * tw), w3 = __ldg(sp + 3 * tw);
    sp += 4 * tw;
    a0 += byte_of(w0, 0) * kk.x + byte_of(w1, 0) * kk.y + byte_of(w2, 0) * kk.z + byte_of(w3, 0) * kk.w;
    a1 += byte_of(w0, 1) * kk.x + byte_of(w1, 1) * kk.y + byte_of(w2, 1) * kk.z + byte_of(w3, 1) * kk.w;
    a2 += byte_of(w0, 2) * kk.x + byte_of(w1, 2) * kk.y + byte_of(w2, 2) * kk.z + byte_of(w3, 2) * kk.w;
    a3 += byte_of(w0, 3) * kk.x + byte_of(w1, 3) * kk.y + byte_of(w2, 3) * kk.z + byte_of(w3, 3) * kk.w;
  }
  const uint32_t v = clip8(a0) | (clip8(a1) << 8) | (clip8(a2) << 16) | (clip8(a3) << 24);
  uint8_t* d = out + (int64_t)j * out_pitch + 4 * e;
  if ((reinterpret_cast<uintptr_t>(d) & 3) == 0 && 4 * e + 4 <= row_bytes) {
    *reinterpret_cast<uint32_t*>(d) = v;
  } else {
    for (int i = 0; i < 4 && 4 * e + i < row_bytes; ++i) d[i] = (uint8_t)(v >> (8 * i));
  }
}

// Window [first, first + count) of output index xx of one axis, from the same filter_row the kernels run.
void filter_window(int in_size, int out_size, int xx, int& first, int& count) {
  const AxisFilter f = make_axis(in_size, out_size);
  int* k = static_cast<int*>(malloc(sizeof(int) * (size_t)f.ksize));
  filter_row(f, in_size, xx, k, first, count);
  free(k);
}

int plan_region(const char* fn, int h, int w, int new_h, int new_w, int o0, int o1, RegionPlan& p) {
  PLIP_REQUIRE(h >= 1 && w >= 1 && h <= 65536 && w <= 65536, "%s: source size %dx%d is outside 1..65536", fn, h, w);
  PLIP_REQUIRE(new_h >= 1 && new_w >= 1 && new_h <= 65536 && new_w <= 65536,
               "%s: output size %dx%d is outside 1..65536", fn, new_h, new_w);
  PLIP_REQUIRE(o0 >= 0 && o0 < o1 && o1 <= new_h, "%s: output rows [%d, %d) are not a non-empty range of 0..%d", fn,
               o0, o1, new_h);
  p.ksh4 = (axis_ksize(w, new_w) + 3) & ~3;
  p.ksv4 = (axis_ksize(h, new_h) + 3) & ~3;
  PLIP_REQUIRE((size_t)kRgCols * p.ksh4 * sizeof(int) <= kRgSmemHard,
               "%s: width %d -> %d shrinks too much (horizontal filter of %d taps; at most %d)", fn, w, new_w,
               axis_ksize(w, new_w), (int)(kRgSmemHard / (kRgCols * sizeof(int))));
  int f0, n0, f1, n1;
  filter_window(h, new_h, o0, f0, n0);
  filter_window(h, new_h, o1 - 1, f1, n1);
  p.s0 = f0, p.s1 = f1 + n1;
  p.tmp_pitch = ((int64_t)new_w * 3 + 3) & ~(int64_t)3;
  const int nv = o1 - o0;
  p.kh = 0;
  p.bh = align16(p.kh + (size_t)new_w * p.ksh4 * sizeof(int));
  p.kv = align16(p.bh + (size_t)new_w * sizeof(int2));
  p.bv = align16(p.kv + (size_t)nv * p.ksv4 * sizeof(int));
  p.tmp = align16(p.bv + (size_t)nv * sizeof(int2));
  p.total = align16(p.tmp + (size_t)(p.s1 - p.s0 + kStripPadRows) * p.tmp_pitch);
  return 0;
}

}  // namespace

int resize_region_workspace(int h, int w, int new_h, int new_w, int o0, int o1, uint64_t* bytes) {
  RegionPlan p;
  if (int rc = plan_region("plip_resize_region_workspace", h, w, new_h, new_w, o0, o1, p)) return rc;
  *bytes = p.total;
  return 0;
}

int resize_filter_bounds(int in_size, int out_size, int32_t* bounds) {
  for (int xx = 0; xx < out_size; ++xx) filter_window(in_size, out_size, xx, bounds[2 * xx], bounds[2 * xx + 1]);
  return 0;
}

int launch_resize_region(const uint8_t* src, int64_t src_pitch, int src_row0, int src_rows, int h, int w, uint8_t* out,
                         int64_t out_pitch, int new_h, int new_w, int o0, int o1, uint8_t* ws, uint64_t ws_bytes,
                         cudaStream_t st) {
  const char* fn = "plip_resize_region_u8";
  RegionPlan p;
  if (int rc = plan_region(fn, h, w, new_h, new_w, o0, o1, p)) return rc;
  PLIP_REQUIRE(src_pitch >= 3LL * w, "%s: source row pitch %lld bytes < 3 * width = %lld", fn, (long long)src_pitch,
               3LL * w);
  PLIP_REQUIRE(out_pitch >= 3LL * new_w, "%s: output row pitch %lld bytes < 3 * new_width = %lld", fn,
               (long long)out_pitch, 3LL * new_w);
  PLIP_REQUIRE(src_row0 >= 0 && src_rows >= 1 && (int64_t)src_row0 + src_rows <= h,
               "%s: source band of %d rows at row %d is not inside the %d source rows", fn, src_rows, src_row0, h);
  PLIP_REQUIRE(p.s0 >= src_row0 && p.s1 <= src_row0 + src_rows,
               "%s: output rows [%d, %d) read source rows [%d, %d), the band holds rows [%d, %d)", fn, o0, o1, p.s0,
               p.s1, src_row0, src_row0 + src_rows);
  PLIP_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "%s: the workspace must be 16-byte aligned", fn);
  PLIP_REQUIRE(ws_bytes >= p.total, "%s: workspace of %llu bytes, %llu needed (plip_resize_region_workspace)", fn,
               (unsigned long long)ws_bytes, (unsigned long long)p.total);
  static unsigned long long configured = 0;
  if (first_use_on_device(configured))
    PLIP_CUDA_CHECK(cudaFuncSetAttribute(resize_rows_h_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)kRgSmemHard));
  int* kh = reinterpret_cast<int*>(ws + p.kh);
  int2* bh = reinterpret_cast<int2*>(ws + p.bh);
  int* kv = reinterpret_cast<int*>(ws + p.kv);
  int2* bv = reinterpret_cast<int2*>(ws + p.bv);
  uint8_t* tmp = ws + p.tmp;
  const int nv = o1 - o0, rows = p.s1 - p.s0;
  PLIP_CUDA_CHECK(launch_kernel(resize_filters_kernel, dim3((new_w + nv + kRsThreads - 1) / kRsThreads),
                                dim3(kRsThreads), 0, st, 1, w, new_w, h, new_h, o0, nv, p.ksh4, p.ksv4, kh, bh, kv, bv));
  const uint8_t* band = src + (int64_t)(p.s0 - src_row0) * src_pitch;
  const uint64_t band_bytes = (uint64_t)(src_row0 + src_rows - 1 - p.s0) * src_pitch + 3ULL * w;
  PLIP_CUDA_CHECK(launch_kernel(resize_rows_h_kernel,
                                dim3((new_w + kRgCols - 1) / kRgCols, (rows + kRgRowsPerCta - 1) / kRgRowsPerCta),
                                dim3(kRsThreads), (size_t)kRgCols * p.ksh4 * sizeof(int), st, 1, band, src_pitch,
                                band_bytes, rows, new_w, p.ksh4, kh, bh, tmp, p.tmp_pitch));
  const int row_bytes = new_w * 3;
  PLIP_CUDA_CHECK(launch_kernel(resize_rows_v_kernel,
                                dim3(nv, ((row_bytes + 3) / 4 + kRsThreads - 1) / kRsThreads), dim3(kRsThreads), 0, st, 1,
                                tmp, p.tmp_pitch, p.s0, kv, bv, p.ksv4, out, out_pitch, row_bytes));
  PLIP_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace plip

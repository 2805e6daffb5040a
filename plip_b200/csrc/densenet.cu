// plip_b200 — the reference's MuDiPath baseline on the device: torchvision's DenseNet-121 features (growth 32,
// bottleneck 128, blocks 6 / 12 / 24 / 16, 64 stem features) followed by a global average pool, the
// NoHeadDenseNet.forward of reproducibility/embedders/mudipath.py (F.adaptive_avg_pool2d(features(x), (1, 1))), in
// eval mode.  Inference only; a separate handle from the CLIP engine.
//
// Layout: NHWC bf16 activations, fp32 accumulation.  Each dense block owns one [n, H, W, C_block] buffer: a layer
// reads the channel prefix [0, C_in) and writes its 32 new channels to [C_in, C_in + 32), so nothing is
// concatenated and the A operand of a 1x1 convolution is a strided prefix of the block buffer.
//
// Every convolution is one implicit GEMM, out[m, n] = sum_k A[m, k] W[n, k] (m = output pixel), run by
// dn_conv_kernel<MODE, EPI, BN>: 128 x BN x 32 tiles, 8 warps of mma.sync m16n8k16 bf16 -> fp32, operands staged
// through a register double buffer into shared memory.  MODE is how the A tile is formed from the activations, on
// the way into shared memory, so no layer needs a separate elementwise pass:
//   kAStem    conv0 (7x7 / s2 / p3): K = (ky, kx, c) = 147, zero-padded to 160.  The uint8 pixel is normalised
//             ((u8 / 255 - mean) / std, ToTensor + Normalize) and rounded to bf16; out-of-image taps are exactly 0,
//             i.e. the zero padding comes after the normalisation, as in the reference.
//   kAPreact  conv1 (1x1, C_in -> 128): A = bf16(relu(x * s1 + b1)) per K column.  norm1 sits between two
//             non-linear steps (the previous ReLU and this one), so it cannot fold into the weights, and every layer
//             has its own norm1 over the whole prefix: it is applied here, to the raw bf16 tile.
//   kATap3    conv2 (3x3 / p1, 128 -> 32): K = (ky, kx, c) = 1152 over the stored bottleneck.  The bottleneck is
//             post-ReLU, so the padding is exactly zero: out-of-image taps load zeros.
//   kAPool    transition: BN, ReLU, 2x2 average pool, then the 1x1 conv.  Pool and conv are both linear, so the pool
//             runs first, in the loader (4x fewer multiply-adds): A = bf16(((r00 + r01) + r10) + r11) * 0.25) with
//             r = relu(x * s + b) in fp32.
// EPI: kEpiBnRelu applies the next BN + ReLU per output channel (norm0 after conv0, norm2 after conv1) before the
// bf16 store; kEpiStore stores the accumulator as bf16 (conv2 into the layer's 32-channel slice, the transition
// into channels [0, C/2) of the next block buffer).
// The loaders multiply and add with __fmul_rn / __fadd_rn, so x * s + b is rounded twice, as PyTorch computes it
// (tests/densenet_oracle.py restates every rounding point).
//
// The 3x3 / s2 / p1 max pool after the stem and the tail are small kernels of their own.  Tail: norm5 is affine
// with no ReLU, so avgpool(norm5(x)) = norm5(avgpool(x)): the 7 x 7 positions are averaged in fp32, then the BN is
// applied.  A micro-batch is 122 launches.
#include "kernels.cuh"

#include <math.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

namespace plip {

namespace {

constexpr int kDnGrowth = 32;
constexpr int kDnBottleneck = 128;
constexpr int kDnStemC = 64;
constexpr int kDnOut = 1024;
constexpr int kDnLayers[4] = {6, 12, 24, 16};
constexpr int kDnBlockIn[4] = {64, 128, 256, 512};     // channels entering each block
constexpr int kDnBlockC[4] = {256, 512, 1024, 1024};   // channels leaving each block
constexpr int kDnSide[4] = {56, 28, 14, 7};
constexpr int kDnStemSide = 112;
constexpr int kDnStemK = 147;
constexpr int kDnStemKPad = 160;
constexpr int kDnTap3K = 9 * kDnBottleneck;
constexpr int kDnMaxMicroBatch = 4096;

enum { kAStem = 0, kAPreact = 1, kATap3 = 2, kAPool = 3 };
enum { kEpiBnRelu = 0, kEpiStore = 1 };

constexpr int kBM = 128;
constexpr int kBK = 32;
constexpr int kLdS = kBK + 8;   // shared row stride (80 bytes): the 8 rows of an ldmatrix hit distinct bank quads
constexpr int kDnThreads = 256;

struct ConvArgs {
  const __nv_bfloat16* a;   // activations, pixel p at a + p * lda (kAPreact / kATap3 / kAPool)
  const uint8_t* img;       // kAStem: uint8 tiles [n, 224, 224, 3]
  int lda;
  const float* a_scale;     // kAPreact / kAPool: BN of the input, per K column
  const float* a_shift;
  const __nv_bfloat16* w;   // [N, K], rows contiguous
  int M, N, K;
  int side;                 // output grid side (images are square at every stage)
  const float* e_scale;     // kEpiBnRelu: BN of the output, per N column
  const float* e_shift;
  __nv_bfloat16* out;       // output pixel m, channel c at out + m * ldo + c
  int ldo;
};

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf2(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

__device__ __forceinline__ float bn_relu(float x, float s, float b) { return fmaxf(__fadd_rn(__fmul_rn(x, s), b), 0.f); }

// relu(x * s + b) of 8 bf16 values, fp32 out.
__device__ __forceinline__ void preact8(const uint4 raw, const float4 s0, const float4 s1, const float4 b0,
                                        const float4 b1, float (&v)[8]) {
  v[0] = bn_relu(bf_lo(raw.x), s0.x, b0.x);
  v[1] = bn_relu(bf_hi(raw.x), s0.y, b0.y);
  v[2] = bn_relu(bf_lo(raw.y), s0.z, b0.z);
  v[3] = bn_relu(bf_hi(raw.y), s0.w, b0.w);
  v[4] = bn_relu(bf_lo(raw.z), s1.x, b1.x);
  v[5] = bn_relu(bf_hi(raw.z), s1.y, b1.y);
  v[6] = bn_relu(bf_lo(raw.w), s1.z, b1.z);
  v[7] = bn_relu(bf_hi(raw.w), s1.w, b1.w);
}

__device__ __forceinline__ uint4 pack8(const float (&v)[8]) {
  return make_uint4(pack_bf2(v[0], v[1]), pack_bf2(v[2], v[3]), pack_bf2(v[4], v[5]), pack_bf2(v[6], v[7]));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ImageNet statistics of the reference's Normalize (factory.py:45), as float32 like torch's tensors of them.
__device__ __forceinline__ float stem_pixel(uint8_t u, int c) {
  const float mean = c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f);
  const float stdv = c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f);
  return __fdiv_rn(__fsub_rn(__fdiv_rn((float)u, 255.f), mean), stdv);
}

// The transition's pooled loader holds four input pixels' worth of BN in flight: it runs at one CTA per SM (3 launches
// per micro-batch) rather than spill at two.
template <int MODE, int EPI, int BN>
__global__ void __launch_bounds__(kDnThreads, MODE == kAPool ? 1 : 2) dn_conv_kernel(const ConvArgs p) {
  constexpr int kWM = 4, kWN = 2;                    // warp grid: 32-row x BN/2-column warp tiles
  constexpr int kWarpN = BN / kWN;
  constexpr int kNF = kWarpN / 8;                    // n8 fragments per warp
  constexpr int kBChunks = BN * kBK / 8;             // 16-byte chunks of a W tile
  constexpr int kBPer = (kBChunks + kDnThreads - 1) / kDnThreads;
  static_assert(kNF % 2 == 0, "B fragments are loaded in pairs");
  __shared__ __align__(16) __nv_bfloat16 sA[2][kBM * kLdS];
  __shared__ __align__(16) __nv_bfloat16 sB[2][BN * kLdS];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp % kWM, wn = warp / kWM;
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
  const int side = p.side, plane = side * side;

  // This thread stages A rows tid / 4 and tid / 4 + 64, columns (tid % 4) * 8 .. + 8 of every K tile.
  const int kc = (tid & 3) * 8;
  long long base[2];   // kAPreact / kATap3: the row's pixel; kAPool: its top-left input pixel; kAStem: image index
  int ry[2], rx[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m0 + (tid >> 2) + 64 * i;
    const int im = m / plane, rem = m - im * plane, y = rem / side, x = rem - y * side;
    if (m >= p.M) {
      base[i] = -1;
    } else if (MODE == kAPool) {
      base[i] = (long long)im * 4 * plane + (long long)(2 * y) * (2 * side) + 2 * x;
    } else if (MODE == kAStem) {
      base[i] = im;
    } else {
      base[i] = m;
    }
    ry[i] = MODE == kAStem ? 2 * y - 3 : y;
    rx[i] = MODE == kAStem ? 2 * x - 3 : x;
  }

  auto load_a = [&](int kt, uint4 (&ra)[2]) {
    const int k = kt * kBK + kc;
    float4 s0, s1, b0, b1;
    if (MODE == kAPreact || MODE == kAPool) {
      s0 = __ldg(reinterpret_cast<const float4*>(p.a_scale + k));
      s1 = __ldg(reinterpret_cast<const float4*>(p.a_scale + k + 4));
      b0 = __ldg(reinterpret_cast<const float4*>(p.a_shift + k));
      b1 = __ldg(reinterpret_cast<const float4*>(p.a_shift + k + 4));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      ra[i] = make_uint4(0u, 0u, 0u, 0u);
      if (base[i] < 0) continue;
      if (MODE == kAPreact) {
        float v[8];
        preact8(__ldg(reinterpret_cast<const uint4*>(p.a + base[i] * p.lda + k)), s0, s1, b0, b1, v);
        ra[i] = pack8(v);
      } else if (MODE == kAPool) {
        // ((r00 + r01) + r10) + r11, then * 0.25: one input pixel at a time keeps the register footprint small
        float v[8], r[8];
        preact8(__ldg(reinterpret_cast<const uint4*>(p.a + base[i] * p.lda + k)), s0, s1, b0, b1, v);
#pragma unroll
        for (int t = 1; t < 4; ++t) {
          const long long q = base[i] + (t & 1) + (t >> 1) * 2 * side;
          preact8(__ldg(reinterpret_cast<const uint4*>(p.a + q * p.lda + k)), s0, s1, b0, b1, r);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = __fadd_rn(v[j], r[j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = __fmul_rn(v[j], 0.25f);
        ra[i] = pack8(v);
      } else if (MODE == kATap3) {
        const int tap = k / kDnBottleneck, c = k - tap * kDnBottleneck;
        const int dy = tap / 3 - 1, dx = tap - (tap / 3) * 3 - 1;
        const int yy = ry[i] + dy, xx = rx[i] + dx;
        if (yy >= 0 && yy < side && xx >= 0 && xx < side)
          ra[i] = __ldg(reinterpret_cast<const uint4*>(p.a + (base[i] + dy * side + dx) * kDnBottleneck + c));
      } else {  // kAStem
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          v[j] = 0.f;
          const int kk = k + j;
          if (kk < kDnStemK) {
            const int tap = kk / 3, c = kk - tap * 3, ky = tap / 7, kx = tap - ky * 7;
            const int iy = ry[i] + ky, ix = rx[i] + kx;
            if (iy >= 0 && iy < kImage && ix >= 0 && ix < kImage)
              v[j] = stem_pixel(__ldg(p.img + ((base[i] * kImage + iy) * kImage + ix) * 3 + c), c);
          }
        }
        ra[i] = pack8(v);
      }
    }
  };
  auto load_b = [&](int kt, uint4 (&rb)[kBPer]) {
#pragma unroll
    for (int i = 0; i < kBPer; ++i) {
      const int q = tid + i * kDnThreads;
      if (q < kBChunks)
        rb[i] = __ldg(reinterpret_cast<const uint4*>(p.w + (long long)(n0 + q / 4) * p.K + kt * kBK + (q & 3) * 8));
    }
  };
  auto store = [&](int buf, const uint4 (&ra)[2], const uint4 (&rb)[kBPer]) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
      *reinterpret_cast<uint4*>(&sA[buf][((tid >> 2) + 64 * i) * kLdS + kc]) = ra[i];
#pragma unroll
    for (int i = 0; i < kBPer; ++i) {
      const int q = tid + i * kDnThreads;
      if (q < kBChunks) *reinterpret_cast<uint4*>(&sB[buf][(q / 4) * kLdS + (q & 3) * 8]) = rb[i];
    }
  };

  float acc[2][kNF][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < kNF; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;

  const int KT = p.K / kBK;
  uint4 ra[2], rb[kBPer];
  load_a(0, ra);
  load_b(0, rb);
  store(0, ra, rb);
  __syncthreads();
  for (int kt = 0; kt < KT; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < KT) {
      load_a(kt + 1, ra);
      load_b(kt + 1, rb);
    }
#pragma unroll
    for (int kk = 0; kk < kBK; kk += 16) {
      uint32_t af[2][4];
#pragma unroll
      for (int mf = 0; mf < 2; ++mf)
        ldmatrix_x4(af[mf], &sA[buf][(wm * 32 + mf * 16 + (lane & 15)) * kLdS + kk + (lane >> 4) * 8]);
#pragma unroll
      for (int np = 0; np < kNF / 2; ++np) {
        uint32_t bf[4];
        ldmatrix_x4(bf, &sB[buf][(wn * kWarpN + np * 16 + (lane & 7) + (lane >> 4) * 8) * kLdS + kk +
                                 ((lane >> 3) & 1) * 8]);
#pragma unroll
        for (int mf = 0; mf < 2; ++mf) {
          mma_bf16_16816(acc[mf][2 * np], af[mf], bf[0], bf[1]);
          mma_bf16_16816(acc[mf][2 * np + 1], af[mf], bf[2], bf[3]);
        }
      }
    }
    if (kt + 1 < KT) store(buf ^ 1, ra, rb);
    __syncthreads();
  }

#pragma unroll
  for (int mf = 0; mf < 2; ++mf)
#pragma unroll
    for (int nf = 0; nf < kNF; ++nf) {
      const int col = n0 + wn * kWarpN + nf * 8 + (lane & 3) * 2;
      float s0 = 1.f, s1 = 1.f, b0 = 0.f, b1 = 0.f;
      if (EPI == kEpiBnRelu) {
        s0 = __ldg(p.e_scale + col);
        s1 = __ldg(p.e_scale + col + 1);
        b0 = __ldg(p.e_shift + col);
        b1 = __ldg(p.e_shift + col + 1);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m0 + wm * 32 + mf * 16 + (lane >> 2) + 8 * h;
        if (row >= p.M) continue;
        float v0 = acc[mf][nf][2 * h], v1 = acc[mf][nf][2 * h + 1];
        if (EPI == kEpiBnRelu) {
          v0 = bn_relu(v0, s0, b0);
          v1 = bn_relu(v1, s1, b1);
        }
        *reinterpret_cast<uint32_t*>(p.out + (long long)row * p.ldo + col) = pack_bf2(v0, v1);
      }
    }
}

// 3x3 / s2 / p1 max pool of the stem output [n, 112, 112, 64] into channels [0, 64) of block 1 ([n, 56, 56, ldo]).
// One thread per output pixel and 8 channels; the centre tap is always inside the image.
__global__ void __launch_bounds__(256) dn_maxpool_kernel(const __nv_bfloat16* __restrict__ in, long long n,
                                                         __nv_bfloat16* __restrict__ out, int ldo) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  constexpr int kOut = kDnStemSide / 2;
  if (t >= n * kOut * kOut * (kDnStemC / 8)) return;
  const int g = (int)(t & 7);
  const long long pix = t >> 3;
  const long long im = pix / (kOut * kOut);
  const int rem = (int)(pix - im * kOut * kOut), oy = rem / kOut, ox = rem - oy * kOut;
  const __nv_bfloat16* src = in + im * kDnStemSide * kDnStemSide * kDnStemC + g * 8;
  uint4 best = __ldg(reinterpret_cast<const uint4*>(src + ((long long)(2 * oy) * kDnStemSide + 2 * ox) * kDnStemC));
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int iy = 2 * oy - 1 + ky, ix = 2 * ox - 1 + kx;
      if (iy < 0 || iy >= kDnStemSide || ix < 0 || ix >= kDnStemSide) continue;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + ((long long)iy * kDnStemSide + ix) * kDnStemC));
      uint32_t* b = reinterpret_cast<uint32_t*>(&best);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        __nv_bfloat162 m = __hmax2(*reinterpret_cast<const __nv_bfloat162*>(&b[j]),
                                   *reinterpret_cast<const __nv_bfloat162*>(&w[j]));
        b[j] = *reinterpret_cast<uint32_t*>(&m);
      }
    }
  *reinterpret_cast<uint4*>(out + pix * ldo + g * 8) = best;
}

// Tail: out[i, c] = mean_p(x[i, p, c]) * s5[c] + b5[c], p over the 7 x 7 positions in order, fp32.
__global__ void __launch_bounds__(256) dn_tail_kernel(const __nv_bfloat16* __restrict__ x, long long n,
                                                      const float* __restrict__ scale,
                                                      const float* __restrict__ shift, float* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * kDnOut) return;
  const long long im = t / kDnOut;
  const int c = (int)(t - im * kDnOut);
  constexpr int kPos = 7 * 7;
  const __nv_bfloat16* src = x + im * kPos * kDnOut + c;
  float s = 0.f;
#pragma unroll 7
  for (int q = 0; q < kPos; ++q) s = __fadd_rn(s, __bfloat162float(src[(long long)q * kDnOut]));
  const float mean = __fdiv_rn(s, (float)kPos);
  out[t] = __fadd_rn(__fmul_rn(mean, __ldg(scale + c)), __ldg(shift + c));
}

template <int MODE, int EPI, int BN>
int launch_conv(const ConvArgs& p, cudaStream_t st) {
  if (p.M == 0) return 0;
  const dim3 grid((unsigned)((p.M + kBM - 1) / kBM), (unsigned)(p.N / BN));
  PLIP_CUDA_CHECK(launch_kernel(dn_conv_kernel<MODE, EPI, BN>, grid, dim3(kDnThreads), 0, st, 1u, p));
  return 0;
}

// ---- packed weights -------------------------------------------------------------------------------------------
struct DnSpec {
  std::string name;
  uint64_t offset, numel;
  int dtype, rows, cols;   // dtype 0 float32, 1 bfloat16
};

struct DnLayout {
  std::vector<DnSpec> specs;
  uint64_t bytes = 0;
  void add(const std::string& name, int dtype, int rows, int cols) {
    const uint64_t off = (bytes + 255) / 256 * 256;
    specs.push_back({name, off, (uint64_t)rows * cols, dtype, rows, cols});
    bytes = off + (uint64_t)rows * cols * (dtype ? 2 : 4);
  }
  void bn(const std::string& name, int c) {
    add(name + ".scale", 0, c, 1);
    add(name + ".shift", 0, c, 1);
  }
};

// Walk order of the blob: the order in which plip_densenet_encode uses the tensors.
const DnLayout& dn_layout() {
  static const DnLayout L = [] {
    DnLayout l;
    l.add("features.conv0.weight", 1, kDnStemC, kDnStemKPad);
    l.bn("features.norm0", kDnStemC);
    for (int b = 0; b < 4; ++b) {
      for (int j = 0; j < kDnLayers[b]; ++j) {
        const int cin = kDnBlockIn[b] + kDnGrowth * j;
        const std::string pre = "features.denseblock" + std::to_string(b + 1) + ".denselayer" + std::to_string(j + 1);
        l.bn(pre + ".norm1", cin);
        l.add(pre + ".conv1.weight", 1, kDnBottleneck, cin);
        l.bn(pre + ".norm2", kDnBottleneck);
        l.add(pre + ".conv2.weight", 1, kDnGrowth, kDnTap3K);
      }
      if (b < 3) {
        const std::string pre = "features.transition" + std::to_string(b + 1);
        l.bn(pre + ".norm", kDnBlockC[b]);
        l.add(pre + ".conv.weight", 1, kDnBlockC[b] / 2, kDnBlockC[b]);
      }
    }
    l.bn("features.norm5", kDnOut);
    l.bytes = (l.bytes + 255) / 256 * 256;
    return l;
  }();
  return L;
}

// Activation buffers per image, in elements: stem output, the bottleneck, the four block buffers.
constexpr long long kWsStem = (long long)kDnStemSide * kDnStemSide * kDnStemC;
constexpr long long kWsNeck = (long long)kDnSide[0] * kDnSide[0] * kDnBottleneck;
constexpr long long kWsBlock(int b) { return (long long)kDnSide[b] * kDnSide[b] * kDnBlockC[b]; }
constexpr long long kWsPerImage = kWsStem + kWsNeck + kWsBlock(0) + kWsBlock(1) + kWsBlock(2) + kWsBlock(3);

}  // namespace

}  // namespace plip

using namespace plip;

struct plip_densenet {
  int device = 0;
  int max_mb = 0;
  uint8_t* d_blob = nullptr;
  __nv_bfloat16* ws = nullptr;
  cudaEvent_t done = nullptr;   // end of the previous call: calls on one handle share the workspace
  const uint8_t* ptr(int index) const { return d_blob + dn_layout().specs[index].offset; }
};

namespace {

// One micro-batch: tiles [n, 224, 224, 3] -> out [n, 1024].
int dn_forward(const plip_densenet* e, const uint8_t* tiles, int n, float* out, cudaStream_t st) {
  const auto& specs = dn_layout().specs;
  __nv_bfloat16* stem = e->ws;
  __nv_bfloat16* neck = stem + kWsStem * e->max_mb;
  __nv_bfloat16* blk[4];
  blk[0] = neck + kWsNeck * e->max_mb;
  for (int b = 1; b < 4; ++b) blk[b] = blk[b - 1] + kWsBlock(b - 1) * e->max_mb;
  int t = 0;   // next tensor of the walk
  auto bf = [&](int i) { return reinterpret_cast<const __nv_bfloat16*>(e->ptr(i)); };
  auto f32 = [&](int i) { return reinterpret_cast<const float*>(e->ptr(i)); };

  ConvArgs p = {};
  p.img = tiles;
  p.w = bf(t);
  p.e_scale = f32(t + 1);
  p.e_shift = f32(t + 2);
  t += 3;
  p.M = n * kDnStemSide * kDnStemSide;
  p.N = kDnStemC;
  p.K = kDnStemKPad;
  p.side = kDnStemSide;
  p.out = stem;
  p.ldo = kDnStemC;
  if (launch_conv<kAStem, kEpiBnRelu, 64>(p, st)) return -1;
  const long long mp_threads = (long long)n * kDnSide[0] * kDnSide[0] * (kDnStemC / 8);
  PLIP_CUDA_CHECK(launch_kernel(dn_maxpool_kernel, dim3((unsigned)((mp_threads + 255) / 256)), dim3(256), 0, st, 1u,
                                (const __nv_bfloat16*)stem, (long long)n, blk[0], kDnBlockC[0]));
  for (int b = 0; b < 4; ++b) {
    const int side = kDnSide[b], M = n * side * side;
    for (int j = 0; j < kDnLayers[b]; ++j) {
      const int cin = kDnBlockIn[b] + kDnGrowth * j;
      ConvArgs c1 = {};
      c1.a = blk[b];
      c1.lda = kDnBlockC[b];
      c1.a_scale = f32(t);
      c1.a_shift = f32(t + 1);
      c1.w = bf(t + 2);
      c1.e_scale = f32(t + 3);
      c1.e_shift = f32(t + 4);
      c1.M = M;
      c1.N = kDnBottleneck;
      c1.K = cin;
      c1.side = side;
      c1.out = neck;
      c1.ldo = kDnBottleneck;
      if (launch_conv<kAPreact, kEpiBnRelu, 128>(c1, st)) return -1;
      ConvArgs c2 = {};
      c2.a = neck;
      c2.lda = kDnBottleneck;
      c2.w = bf(t + 5);
      c2.M = M;
      c2.N = kDnGrowth;
      c2.K = kDnTap3K;
      c2.side = side;
      c2.out = blk[b] + cin;
      c2.ldo = kDnBlockC[b];
      if (launch_conv<kATap3, kEpiStore, 32>(c2, st)) return -1;
      t += 6;
    }
    if (b < 3) {
      ConvArgs tr = {};
      tr.a = blk[b];
      tr.lda = kDnBlockC[b];
      tr.a_scale = f32(t);
      tr.a_shift = f32(t + 1);
      tr.w = bf(t + 2);
      tr.M = n * kDnSide[b + 1] * kDnSide[b + 1];
      tr.N = kDnBlockC[b] / 2;
      tr.K = kDnBlockC[b];
      tr.side = kDnSide[b + 1];
      tr.out = blk[b + 1];
      tr.ldo = kDnBlockC[b + 1];
      if (launch_conv<kAPool, kEpiStore, 128>(tr, st)) return -1;
      t += 3;
    }
  }
  const long long tail_threads = (long long)n * kDnOut;
  PLIP_CUDA_CHECK(launch_kernel(dn_tail_kernel, dim3((unsigned)((tail_threads + 255) / 256)), dim3(256), 0, st, 1u,
                                (const __nv_bfloat16*)blk[3], (long long)n, f32(t), f32(t + 1), out));
  t += 2;
  PLIP_REQUIRE(t == (int)specs.size(), "densenet: internal error: %d of %d tensors used", t, (int)specs.size());
  return 0;
}

bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

}  // namespace

extern "C" {

PLIP_API int plip_densenet_num_tensors(void) { return (int)dn_layout().specs.size(); }

PLIP_API int plip_densenet_tensor_info(int index, plip_tensor_info_t* info) {
  const auto& v = dn_layout().specs;
  PLIP_REQUIRE(info != nullptr, "plip_densenet_tensor_info: null argument");
  PLIP_REQUIRE(index >= 0 && index < (int)v.size(), "plip_densenet_tensor_info: index %d out of range [0, %d)", index,
               (int)v.size());
  memset(info, 0, sizeof(*info));
  strncpy(info->name, v[index].name.c_str(), sizeof(info->name) - 1);
  info->offset = v[index].offset;
  info->numel = v[index].numel;
  info->dtype = v[index].dtype;
  info->rows = v[index].rows;
  info->cols = v[index].cols;
  return 0;
}

PLIP_API uint64_t plip_densenet_blob_bytes(void) { return dn_layout().bytes; }

PLIP_API uint64_t plip_densenet_workspace_bytes(int max_micro_batch) {
  return max_micro_batch > 0 ? (uint64_t)kWsPerImage * 2 * (uint64_t)max_micro_batch : 0;
}

PLIP_API int plip_densenet_destroy(plip_densenet_t* e) {
  if (e == nullptr) return 0;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(e->device);
  if (e->done) cudaEventDestroy(e->done);
  cudaFree(e->d_blob);
  cudaFree(e->ws);
  cudaSetDevice(prev);
  delete e;
  return 0;
}

PLIP_API int plip_densenet_create(const void* host_blob, uint64_t blob_bytes, int device, int max_micro_batch,
                                  plip_densenet_t** out) {
  PLIP_REQUIRE(out != nullptr && host_blob != nullptr, "plip_densenet_create: null argument");
  PLIP_REQUIRE(blob_bytes == dn_layout().bytes, "plip_densenet_create: blob is %llu bytes, expected %llu",
               (unsigned long long)blob_bytes, (unsigned long long)dn_layout().bytes);
  PLIP_REQUIRE(max_micro_batch >= 1 && max_micro_batch <= kDnMaxMicroBatch,
               "plip_densenet_create: max_micro_batch %d out of [1, %d]", max_micro_batch, kDnMaxMicroBatch);
  int ndev = 0;
  PLIP_CUDA_CHECK(cudaGetDeviceCount(&ndev));
  PLIP_REQUIRE(device >= 0 && device < ndev, "plip_densenet_create: device %d not present (%d devices)", device, ndev);
  cudaDeviceProp prop;
  PLIP_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  PLIP_REQUIRE(prop.major == 9 && prop.minor == 0,
               "plip_densenet_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major,
               prop.minor);
  int prev = 0;
  PLIP_CUDA_CHECK(cudaGetDevice(&prev));
  PLIP_CUDA_CHECK(cudaSetDevice(device));
  plip_densenet* e = new plip_densenet();
  e->device = device;
  e->max_mb = max_micro_batch;
  const uint64_t ws = plip_densenet_workspace_bytes(max_micro_batch);
  cudaError_t ce = cudaMalloc(&e->d_blob, blob_bytes);
  if (ce == cudaSuccess) ce = cudaMalloc(&e->ws, ws);
  if (ce == cudaSuccess) ce = cudaMemcpy(e->d_blob, host_blob, blob_bytes, cudaMemcpyHostToDevice);
  if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&e->done, cudaEventDisableTiming);
  cudaSetDevice(prev);
  if (ce != cudaSuccess) {
    set_last_error("plip_densenet_create: %llu (weights) + %llu (workspace) bytes on device %d: %s",
                   (unsigned long long)blob_bytes, (unsigned long long)ws, device, cudaGetErrorString(ce));
    cudaGetLastError();
    plip_densenet_destroy(e);
    return -1;
  }
  *out = e;
  return 0;
}

PLIP_API int plip_densenet_max_micro_batch(const plip_densenet_t* e) { return e ? e->max_mb : 0; }

PLIP_API int plip_densenet_encode(plip_densenet_t* e, const void* tiles_dev, int64_t n, float* out_dev,
                                  void* stream) {
  PLIP_REQUIRE(e != nullptr, "plip_densenet_encode: null handle");
  PLIP_REQUIRE(n >= 0, "plip_densenet_encode: n = %lld is negative", (long long)n);
  if (n == 0) return 0;
  PLIP_REQUIRE(tiles_dev != nullptr && out_dev != nullptr, "plip_densenet_encode: null argument");
  PLIP_REQUIRE((reinterpret_cast<uintptr_t>(out_dev) & 3) == 0, "plip_densenet_encode: out_dev %p is not 4-byte aligned",
               (void*)out_dev);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PLIP_CUDA_CHECK(cudaStreamWaitEvent(st, e->done, 0));
  const uint8_t* tiles = static_cast<const uint8_t*>(tiles_dev);
  for (int64_t i = 0; i < n; i += e->max_mb) {
    const int nb = (int)(n - i < e->max_mb ? n - i : e->max_mb);
    if (dn_forward(e, tiles + i * (int64_t)kImage * kImage * 3, nb, out_dev + i * kDnOut, st)) return -1;
  }
  PLIP_CUDA_CHECK(cudaEventRecord(e->done, st));
  return 0;
}

PLIP_API int plip_dbg_densenet_op(int op, const void* in_dev, int lda, int64_t n, int side, int c_in,
                                  const void* w_dev, const float* a_scale, const float* a_shift, const float* e_scale,
                                  const float* e_shift, void* out_dev, int ldo, void* stream) {
  PLIP_REQUIRE(op >= 0 && op <= 5, "plip_dbg_densenet_op: op = %d out of [0, 5]", op);
  PLIP_REQUIRE(n >= 1 && n <= kDnMaxMicroBatch, "plip_dbg_densenet_op: n = %lld out of [1, %d]", (long long)n,
               kDnMaxMicroBatch);
  PLIP_REQUIRE(in_dev != nullptr && out_dev != nullptr, "plip_dbg_densenet_op: null argument");
  PLIP_REQUIRE(aligned16(in_dev) && aligned16(out_dev) && (!w_dev || aligned16(w_dev)) &&
                   (!a_scale || aligned16(a_scale)) && (!a_shift || aligned16(a_shift)),
               "plip_dbg_densenet_op: device pointers must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ConvArgs p = {};
  p.a = static_cast<const __nv_bfloat16*>(in_dev);
  p.img = static_cast<const uint8_t*>(in_dev);
  p.lda = lda;
  p.a_scale = a_scale;
  p.a_shift = a_shift;
  p.w = static_cast<const __nv_bfloat16*>(w_dev);
  p.e_scale = e_scale;
  p.e_shift = e_shift;
  p.out = static_cast<__nv_bfloat16*>(out_dev);
  p.ldo = ldo;
  p.side = side;
  const bool conv = op == 0 || op == 2 || op == 3 || op == 4;
  PLIP_REQUIRE(!conv || w_dev != nullptr, "plip_dbg_densenet_op: op %d needs w_dev", op);
  PLIP_REQUIRE(!(op == 0 || op == 2 || op == 5) || (e_scale && e_shift), "plip_dbg_densenet_op: op %d needs e_scale / e_shift", op);
  PLIP_REQUIRE(!(op == 2 || op == 4) || (a_scale && a_shift), "plip_dbg_densenet_op: op %d needs a_scale / a_shift", op);
  switch (op) {
    case 0:   // stem conv + norm0 + relu: u8 tiles -> [n * 112 * 112, ldo]
      PLIP_REQUIRE(ldo >= kDnStemC && ldo % 8 == 0, "plip_dbg_densenet_op: ldo = %d", ldo);
      p.M = (int)n * kDnStemSide * kDnStemSide;
      p.N = kDnStemC;
      p.K = kDnStemKPad;
      p.side = kDnStemSide;
      return launch_conv<kAStem, kEpiBnRelu, 64>(p, st);
    case 1: {  // max pool: [n, 112, 112, 64] -> channels [0, 64) of [n * 56 * 56, ldo]
      PLIP_REQUIRE(ldo >= kDnStemC && ldo % 8 == 0, "plip_dbg_densenet_op: ldo = %d", ldo);
      const long long th = n * kDnSide[0] * kDnSide[0] * (kDnStemC / 8);
      PLIP_CUDA_CHECK(launch_kernel(dn_maxpool_kernel, dim3((unsigned)((th + 255) / 256)), dim3(256), 0, st, 1u,
                                    p.a, (long long)n, p.out, ldo));
      return 0;
    }
    case 2:   // conv1: relu(norm1(x[:, :c_in])) . W^T -> relu(norm2) -> [M, ldo] channels [0, 128)
      PLIP_REQUIRE(c_in >= 32 && c_in % 32 == 0 && lda >= c_in && lda % 8 == 0 && ldo >= kDnBottleneck && ldo % 8 == 0,
                   "plip_dbg_densenet_op: conv1 c_in = %d, lda = %d, ldo = %d", c_in, lda, ldo);
      PLIP_REQUIRE(side >= 1 && side <= kDnSide[0], "plip_dbg_densenet_op: side = %d", side);
      p.M = (int)n * side * side;
      p.N = kDnBottleneck;
      p.K = c_in;
      return launch_conv<kAPreact, kEpiBnRelu, 128>(p, st);
    case 3:   // conv2: 3x3 / p1 over a dense [n, side, side, 128] bottleneck -> [M, ldo] channels [0, 32)
      PLIP_REQUIRE(ldo >= kDnGrowth && ldo % 8 == 0, "plip_dbg_densenet_op: ldo = %d", ldo);
      PLIP_REQUIRE(side >= 1 && side <= kDnSide[0], "plip_dbg_densenet_op: side = %d", side);
      p.lda = kDnBottleneck;
      p.M = (int)n * side * side;
      p.N = kDnGrowth;
      p.K = kDnTap3K;
      return launch_conv<kATap3, kEpiStore, 32>(p, st);
    case 4:   // transition: avgpool2(relu(norm(x))) . W^T, input [n, 2 side, 2 side, lda] -> [n side^2, ldo]
      PLIP_REQUIRE(c_in >= 128 && c_in % 256 == 0 && lda >= c_in && lda % 8 == 0 && ldo >= c_in / 2 && ldo % 8 == 0,
                   "plip_dbg_densenet_op: transition c_in = %d, lda = %d, ldo = %d", c_in, lda, ldo);
      PLIP_REQUIRE(side >= 1 && side <= kDnSide[1], "plip_dbg_densenet_op: side = %d", side);
      p.M = (int)n * side * side;
      p.N = c_in / 2;
      p.K = c_in;
      return launch_conv<kAPool, kEpiStore, 128>(p, st);
    default: {  // tail: [n, 49, 1024] -> fp32 [n, 1024]
      const long long th = n * kDnOut;
      PLIP_CUDA_CHECK(launch_kernel(dn_tail_kernel, dim3((unsigned)((th + 255) / 256)), dim3(256), 0, st, 1u, p.a,
                                    (long long)n, e_scale, e_shift, static_cast<float*>(out_dev)));
      return 0;
    }
  }
}

}  // extern "C"

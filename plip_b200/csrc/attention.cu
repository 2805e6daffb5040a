// plip_b200 — fused attention core on wgmma: S = Q K^T -> masked softmax -> O = P V, one kernel.
//
// Replaces F.scaled_dot_product_attention / eager_attention_forward for the CLIP towers
// (TF:integrations/sdpa_attention.py:92-101, TF:modeling_clip.py:261-279): per (sequence, head)
//     softmax(q k^T * dh^-0.5 + mask, fp32) v,   dh = 64,
// vision S = 50 without mask, text S <= 77 with the causal (+ key padding) mask (TF:546-557).
// The dh^-0.5 = 0.125 scale is folded into the q rows of the packed QKV weights (exact: power of 2).
//
// Sequences are short, so G = 128 / slot sequences of one head share a 128-row tile, slot = 32 / 64 / 128 rows
// (the power of two >= S), and attention between different sequences is masked out (block-diagonal: exact):
//   TMA      per sequence a [slot x 64] box of the Q, K, V head slices of the QKV activation -> smem (128B swizzle)
//   MMA 1    each of the two warpgroups owns 64 query rows: S[64 x NK] (registers, fp32) = Q (smem) x K^T (smem),
//            NK = 64 keys (the 64-key half that holds the rows' own sequences) when slot <= 64, else all 128
//   softmax  on the accumulator registers: mask, row max / sum over the 4 lanes of a row, exp2; the 16-bit P values
//            are already laid out as the A fragments of MMA 2
//   MMA 2    O[64 x 64] (registers, fp32) = P (registers) x V (smem, MN-major)
//   epilogue O / rowsum -> 16 bit -> the warpgroup's own Q rows (free once MMA 1 retired) -> one TMA bulk store per
//            sequence
// One CTA runs this chain serially per tile; with 48 KB of operands several CTAs co-reside per SM and hide each
// other's load -> MMA -> softmax -> MMA -> store latency.
// Sequences longer than 128 (vision at more than 256 x 256 pixels) go to attention_long_kernel below.
#include <cfloat>

#include "kernels.cuh"
#include "wgmma.cuh"

namespace plip {

namespace {

constexpr int kAttThreads = 256;
constexpr uint32_t kTileBytes = 128 * 64 * 2;  // one [128 x 64] bf16 operand tile
constexpr uint32_t kStageBytes = 3 * kTileBytes;
constexpr uint32_t kAttSmem = kStageBytes + 1024 + 64;

// 2^x, flush-to-zero, no range fix-ups: one MUFU op (inputs are <= 0 here, -inf -> +0).
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kLog2e = 1.4426950408889634f;

// ---- Per-block steps shared by the three kernels.  A thread's scores are its part of a wgmma accumulator
// (wgmma.cuh): a row pair, s[4 j + e] in row 0 and s[4 j + 2 + e] in row 1 (8 rows further), both at column
// 8 j + 2 q4 + e.  Each step is written once, so the kernels that use it share its masks, fp32 operations and order.

// S = Q K^T for one warpgroup: 64 query rows (qdesc) x NK keys (kdesc), K-major SWIZZLE_128B tiles, dh = 64.
template <bool F16, int NK>
__device__ __forceinline__ void qk_scores(float (&s)[NK / 2], uint64_t qdesc, uint64_t kdesc) {
  wgmma_pin(s);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kHeadDim / 16; ++k) {
    if constexpr (NK == 64) wgmma_ss_n64<F16>(s, qdesc + 2 * k, kdesc + 2 * k, k != 0 ? 1u : 0u);
    else wgmma_ss_n128<F16>(s, qdesc + 2 * k, kdesc + 2 * k, k != 0 ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_pin(s);
}

// Row max / row sum of a row pair over the 4 lanes that share its accumulator rows.
__device__ __forceinline__ void quad_max(float& a, float& b) {
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
}
__device__ __forceinline__ void quad_sum(float& a, float& b) {
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
}

// Last key a query row sees: itself under the causal mask, else the last key; -1 for a row past the sequence's end.
__device__ __forceinline__ int last_visible_key(int row, int S, int causal) {
  return row < S ? (causal ? row : S - 1) : -1;
}

// Key `key` (column (j, e)) is visible to a row when it exists and is not padding (ok) and is not past the row's last
// visible key; an invisible score becomes -inf, so its exp2 is 0.
template <int N>
__device__ __forceinline__ void mask_column(float (&s)[N], int j, int e, bool ok, int key, int lim0, int lim1) {
  if (!(ok && key <= lim0)) s[4 * j + e] = -INFINITY;
  if (!(ok && key <= lim1)) s[4 * j + 2 + e] = -INFINITY;
}

// The empty-row rule: a row without a visible key has max -inf and only -inf scores.  Its shift is clamped to a
// finite value, so every exp2 is 0 (not NaN from -inf + inf), l = 0 and row_inv(l) = 0: the row comes out as zeros.
__device__ __forceinline__ float row_shift(float m) { return fmaxf(m * kLog2e, -FLT_MAX); }
__device__ __forceinline__ float row_inv(float l) { return l > 0.f ? 1.0f / l : 0.f; }

// exp2(s log2e - m log2e) of one score, ms = row_shift(m).
__device__ __forceinline__ float softmax_exp(float s, float ms) { return fast_exp2(fmaf(s, kLog2e, -ms)); }

// Online softmax over key blocks: m <- max(m, the block's row max), l <- l * alpha with alpha = 2^(m_old - m_new)
// (m_old = -inf: alpha = 0 and l stays 0).  Returns alpha; the block's exps then use row_shift(m).
__device__ __forceinline__ float2 fold_row_max(const float (&s)[32], float& m0, float& m1, float& l0, float& l1) {
  float mx0 = m0, mx1 = m1;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mx0 = fmaxf(mx0, fmaxf(s[4 * j + 0], s[4 * j + 1]));
    mx1 = fmaxf(mx1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
  }
  quad_max(mx0, mx1);
  const float alpha0 = softmax_exp(m0, row_shift(mx0)), alpha1 = softmax_exp(m1, row_shift(mx1));
  m0 = mx0;
  m1 = mx1;
  l0 *= alpha0;
  l1 *= alpha1;
  return make_float2(alpha0, alpha1);
}

// The exps of a row pair: l += this thread's share of the row sums, in column order, and P in 16 bit as the A
// fragments of O = P V (k-step kk covers keys 16 kk .. 16 kk + 15).  One loop over the column pairs: written as three
// passes over s, it compiles to a different schedule of the long kernel that ran 1-2 % slower on an H100.
template <bool F16, int N>
__device__ __forceinline__ void exp_sum_pack(const float (&s)[N], float ms0, float ms1, float& l0, float& l1,
                                             uint32_t (&pa)[N / 8][4]) {
#pragma unroll
  for (int j = 0; j < N / 4; ++j) {
    const float e00 = softmax_exp(s[4 * j + 0], ms0), e01 = softmax_exp(s[4 * j + 1], ms0);
    const float e10 = softmax_exp(s[4 * j + 2], ms1), e11 = softmax_exp(s[4 * j + 3], ms1);
    l0 += e00 + e01;
    l1 += e10 + e11;
    pa[j >> 1][2 * (j & 1) + 0] = pack_op2<F16>(e00, e01);
    pa[j >> 1][2 * (j & 1) + 1] = pack_op2<F16>(e10, e11);
  }
}

// O / l -> 16 bit -> this thread's rows row0 and row0 + 8 of a [rows x 64] tile, swizzled like a SWIZZLE_128B TMA box.
template <bool F16>
__device__ __forceinline__ void stage_rows(uint32_t row0, const float (&o)[32], float inv0, float inv1, int rr, int q4) {
  const uint32_t row1 = row0 + 8u * 128u;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    st_shared_b32(row0 + ((j ^ rr) << 4) + q4 * 4, pack_op2<F16>(o[4 * j + 0] * inv0, o[4 * j + 1] * inv0));
    st_shared_b32(row1 + ((j ^ rr) << 4) + q4 * 4, pack_op2<F16>(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1));
  }
}

struct AttParams {
  int64_t n_seq;
  int seq_len;          // S
  int slot;             // rows reserved per sequence inside a tile: 32, 64 or 128
  int group;            // G = 128 / slot sequences per tile
  int heads;
  int64_t seq_tiles;    // ceil(n_seq / G)
  int causal;
  const int32_t* key_mask;  // [n_seq, S] or nullptr
};

template <bool F16, int NK>
__global__ void __launch_bounds__(kAttThreads, NK == 64 ? 3 : 2)
attention_kernel(const __grid_constant__ CUtensorMap tmLoad, const __grid_constant__ CUtensorMap tmStore,
                 const AttParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar = smem_base + kStageBytes;
  const uint32_t sq = smem_base, sk = smem_base + kTileBytes, sv = smem_base + 2 * kTileBytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int hf = warp >> 2;                       // warpgroup == 64-row half of the tile
  const int D = p.heads * kHeadDim;
  const int S = p.seq_len, G = p.group, slot = p.slot;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmLoad);
    tma_prefetch_desc(&tmStore);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int ntiles = (int)(p.seq_tiles * p.heads);
  const uint32_t slot_bytes = static_cast<uint32_t>(slot) * 128u;
  auto issue_loads = [&](int tile) {
    const int64_t st = tile / p.heads;
    const int h = (int)(tile - st * p.heads);
    mbar_arrive_expect_tx(bar, 3 * kTileBytes);
    for (int g = 0; g < G; ++g) {
      const int32_t row = (int32_t)((st * G + g) * S);  // past the last sequence: zero fill
      tma_load_2d(sq + g * slot_bytes, &tmLoad, bar, h * kHeadDim, row);
      tma_load_2d(sk + g * slot_bytes, &tmLoad, bar, D + h * kHeadDim, row);
      tma_load_2d(sv + g * slot_bytes, &tmLoad, bar, 2 * D + h * kHeadDim, row);
    }
  };
  if (threadIdx.x == 0 && (int)blockIdx.x < ntiles) issue_loads(blockIdx.x);

  // this thread's two tile rows, their sequence slot, and the keys its accumulator columns stand for
  const int q4 = lane & 3, rr = lane >> 2;
  const int R0 = 64 * hf + 16 * (warp & 3) + rr;  // second row: R0 + 8 (same sequence: slots are multiples of 32)
  const int g = R0 / slot;
  const int r_in0 = R0 - g * slot, r_in1 = r_in0 + 8;
  const int kbase = (NK == 64) ? 64 * hf : 0;     // first key of the tile this warpgroup multiplies with
  const int k_in_base = kbase - g * slot + 2 * q4; // + 8 j + e = index inside the sequence of column (j, e)
  const int lim0 = last_visible_key(r_in0, S, p.causal), lim1 = last_visible_key(r_in1, S, p.causal);

  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const int st = tile / p.heads;
    const int h = tile - st * p.heads;
    const int64_t seq = (int64_t)st * G + g;

    // keys of the sequence that exist (and are not padding): one bit per accumulator column of this thread, read
    // before the wait so that the key-mask loads overlap the TMA loads
    uint32_t kv = 0;
#pragma unroll
    for (int c = 0; c < NK / 4; ++c) {
      const int k_in = k_in_base + 8 * (c >> 1) + (c & 1);
      bool ok = k_in >= 0 && k_in < S;
      if (ok && p.key_mask != nullptr) ok = seq < p.n_seq && p.key_mask[seq * S + k_in] != 0;
      kv |= (ok ? 1u : 0u) << c;
    }

    mbar_wait(bar, it & 1u);

    // ---- S = Q K^T
    float s[NK / 2];
    qk_scores<F16, NK>(s, make_smem_desc_sw128(sq + hf * (64 * 128), 1024, 16),
                       make_smem_desc_sw128(sk + kbase * 128, 1024, 16));

    // ---- masked softmax on the registers; one key block, so the row max folds in column by column as it is masked
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int c = 0; c < NK / 4; ++c) {
      const int j = c >> 1, e = c & 1;
      mask_column(s, j, e, (kv >> c) & 1u, k_in_base + 8 * j + e, lim0, lim1);
      mx0 = fmaxf(mx0, s[4 * j + e]);
      mx1 = fmaxf(mx1, s[4 * j + 2 + e]);
    }
    quad_max(mx0, mx1);
    float sum0 = 0.f, sum1 = 0.f;
    uint32_t pa[NK / 16][4];
    exp_sum_pack<F16>(s, row_shift(mx0), row_shift(mx1), sum0, sum1, pa);
    quad_sum(sum0, sum1);

    // ---- O = P V   (V tile [keys][64 dh]: advancing 16 keys = 16 rows of 128 B)
    float o[32];
    wgmma_pin(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < NK / 16; ++kk) {
      const uint64_t vdesc = make_smem_desc_sw128(sv + (kbase + 16 * kk) * 128, 1024, 1024);
      wgmma_rs_n64<F16>(o, pa[kk], vdesc, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(o);

    // ---- epilogue: O / rowsum -> 16 bit -> this thread's Q rows -> one bulk store per sequence of the tile
    stage_rows<F16>(sq + static_cast<uint32_t>(R0) * 128u, o, row_inv(sum0), row_inv(sum1), rr, q4);
    fence_proxy_async_smem();
    __syncthreads();  // the output tile is complete, and both warpgroups are done with K and V
    if (threadIdx.x == 0) {  // persistent: the CTA's next tile is loaded once the stores have read the Q buffer
      for (int gg = 0; gg < G; ++gg) {
        const int64_t sq_idx = (int64_t)st * G + gg;
        if (sq_idx < p.n_seq)
          tma_store_2d(&tmStore, sq + static_cast<uint32_t>(gg * slot) * 128u, h * kHeadDim, (int32_t)(sq_idx * S));
      }
      tma_store_commit();
      tma_store_wait_read();   // the Q buffer may be refilled
      if (tile + (int)gridDim.x < ntiles) issue_loads(tile + gridDim.x);
    }
  }
  if (threadIdx.x == 0) tma_store_wait_all();
}

template <bool F16, int NK>
int launch_attention_inst(const CUtensorMap& tmL, const CUtensorMap& tmS, const AttParams& p, cudaStream_t st) {
  auto kern = attention_kernel<F16, NK>;
  static unsigned long long configured = 0;
  static int grid_cap = 0;
  if (first_use_on_device(configured)) {
    PLIP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttSmem));
    int dev = 0, sms = 0, per_sm = 0;
    PLIP_CUDA_CHECK(cudaGetDevice(&dev));
    PLIP_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PLIP_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kAttThreads, kAttSmem));
    grid_cap = (per_sm > 0 ? per_sm : 1) * sms;
  }
  const int64_t tiles = p.seq_tiles * p.heads;
  const int grid = (int)(tiles < grid_cap ? tiles : grid_cap);
  PLIP_CUDA_CHECK(launch_kernel(kern, dim3(grid), dim3(kAttThreads), kAttSmem, st, 1, tmL, tmS, p));
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Long sequences (S > 128: vision at more than 256 x 256 pixels, interpolated position table), non-causal and
// unmasked only.  Flash-style online softmax over blocks of 64 keys, one CTA per (sequence, head, 128-query block):
//   warp 8       producer: TMA of the Q block (once) and of the K / V blocks into a two-stage ring (full / empty
//                mbarriers), so block j + 1 lands while block j is multiplied
//   warpgroups   each owns 64 query rows:  S = Q K^T (wgmma m64n64k16, ss) -> keys >= S masked to -inf -> running
//   0 - 1        row max / sum in fp32 (O rescaled by 2^(m_old - m_new)) -> P packed straight into the A fragments
//                of O += P V (wgmma rs, P never leaves the registers) -> after the last block O / l -> 16 bit -> the
//                warpgroup's own Q rows -> one TMA store
// The 3-D tensor maps ([n_seq][S][cols], box {64, rows, 1}) zero-fill rows past a sequence's end on load and clip
// them on store: no tail code, and no row of the next sequence is read or written.  Key blocks are consumed in a
// fixed order: the result is bitwise reproducible.
constexpr int kLongThreads = 288;                 // two consumer warpgroups + one producer warp
constexpr int kLongKeys = 64;                     // keys per block
constexpr uint32_t kLongQBytes = 128 * 64 * 2;    // [128 queries x 64 dh]
constexpr uint32_t kLongKVBytes = kLongKeys * 64 * 2;
constexpr int kLongStages = 2;
constexpr uint32_t kLongSmem = kLongQBytes + kLongStages * 2 * kLongKVBytes + 1024 + 64;

struct LongAttParams {
  int seq_len;
  int heads;
  int q_blocks;  // ceil(S / 128)
};

template <bool F16>
__global__ void __launch_bounds__(kLongThreads, 2)
attention_long_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmO,
                      const LongAttParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sq = smem_base;
  auto sk = [&](int s) { return smem_base + kLongQBytes + (uint32_t)s * 2u * kLongKVBytes; };
  auto sv = [&](int s) { return sk(s) + kLongKVBytes; };
  const uint32_t bar = smem_base + kLongQBytes + kLongStages * 2 * kLongKVBytes;
  const uint32_t q_bar = bar;
  auto full_bar = [&](int s) { return bar + 8u * (1 + s); };
  auto empty_bar = [&](int s) { return bar + 8u * (1 + kLongStages + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int S = p.seq_len, D = p.heads * kHeadDim;
  const int qb = blockIdx.x % p.q_blocks;
  const int bh = blockIdx.x / p.q_blocks;
  const int h = bh % p.heads;
  const int seq = bh / p.heads;
  const int q0 = qb * 128;
  const int n_kb = (S + kLongKeys - 1) / kLongKeys;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmO);
    mbar_init(q_bar, 1);
    for (int s = 0; s < kLongStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 2) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_bar, kLongQBytes);
      tma_load_3d(sq, &tmQKV, q_bar, h * kHeadDim, q0, seq);
      tma_load_3d(sq + kLongQBytes / 2, &tmQKV, q_bar, h * kHeadDim, q0 + 64, seq);
      for (int kb = 0; kb < n_kb; ++kb) {
        const int s = kb % kLongStages;
        if (kb >= kLongStages) mbar_wait(empty_bar(s), (uint32_t)((kb / kLongStages - 1) & 1));
        mbar_arrive_expect_tx(full_bar(s), 2 * kLongKVBytes);
        tma_load_3d(sk(s), &tmQKV, full_bar(s), D + h * kHeadDim, kb * kLongKeys, seq);
        tma_load_3d(sv(s), &tmQKV, full_bar(s), 2 * D + h * kHeadDim, kb * kLongKeys, seq);
      }
    }
    return;
  }

  // ===================== consumers =====================
  const int q4 = lane & 3, rr = lane >> 2;
  const int R0 = 64 * wg + 16 * (warp & 3) + rr;  // this thread's tile rows R0 and R0 + 8
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY;  // running row max (raw scores)
  float l0 = 0.f, l1 = 0.f;              // this thread's share of the running row sum
  const uint64_t qdesc = make_smem_desc_sw128(sq + wg * (64 * 128), 1024, 16);
  mbar_wait(q_bar, 0);

  for (int kb = 0; kb < n_kb; ++kb) {
    const int s = kb % kLongStages;
    mbar_wait(full_bar(s), (uint32_t)((kb / kLongStages) & 1));

    // ---- S = Q K^T
    float sc[32];
    qk_scores<F16, 64>(sc, qdesc, make_smem_desc_sw128(sk(s), 1024, 16));

    // ---- online softmax on the registers; no causal or key mask (vision only): keys >= S exist in the last block only
    const int kbase = kb * kLongKeys + 2 * q4;  // + 8 j + e = key of column (j, e)
    if (kb * kLongKeys + kLongKeys > S) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * j + e >= S) {
            sc[4 * j + e] = -INFINITY;
            sc[4 * j + 2 + e] = -INFINITY;
          }
    }
    // Every block holds at least one real key, and zero-filled query rows still score 0 against real keys, so the
    // row max is finite and row_shift's empty-row case never occurs here.
    const float2 alpha = fold_row_max(sc, m0, m1, l0, l1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j + 0] *= alpha.x; o[4 * j + 1] *= alpha.x;
      o[4 * j + 2] *= alpha.y; o[4 * j + 3] *= alpha.y;
    }
    uint32_t pa[4][4];
    exp_sum_pack<F16>(sc, row_shift(m0), row_shift(m1), l0, l1, pa);

    // ---- O += P V   (V block [keys][64 dh]: advancing 16 keys = 16 rows of 128 B)
    wgmma_pin(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kLongKeys / 16; ++kk) {
      const uint64_t vdesc = make_smem_desc_sw128(sv(s) + 16 * kk * 128, 1024, 1024);
      wgmma_rs_n64<F16>(o, pa[kk], vdesc, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(o);
    if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar(s));  // this warpgroup is done with K / V of the stage
  }

  // ---- epilogue: O / l -> 16 bit -> this warpgroup's Q rows -> one TMA store
  quad_sum(l0, l1);
  stage_rows<F16>(sq + static_cast<uint32_t>(R0) * 128u, o, row_inv(l0), row_inv(l1), rr, q4);
  fence_proxy_async_smem();
  if (wg == 0) named_barrier_sync<1, 128>();  // the warpgroup's 64 output rows are staged
  else named_barrier_sync<2, 128>();
  if ((threadIdx.x & 127) == 0 && q0 + 64 * wg < S) {
    tma_store_3d(&tmO, sq + wg * (64 * 128), h * kHeadDim, q0 + 64 * wg, seq);
    tma_store_commit();
    tma_store_wait_all();
  }
}

// ------------------------------------------------------------------------------------------------
// Attention probabilities (output_attentions): P = softmax(q k^T + mask) in fp32, written as [n_seq, heads, S, S], for
// any 1 <= S <= kMaxVisSeq with the masks of the kernels above.  It reads the QKV buffer the layer's attention has just
// read and leaves that kernel alone.  One CTA (one warpgroup) per (sequence, head, block of 64 queries):
//   TMA      the [64 x 64] Q block once, then 64-key K blocks through a two-stage ring; the 3-D tensor maps
//            ([n_seq][S][3D], as the long kernel's) zero-fill rows past the sequence's end
//   pass 1   per key block S = Q K^T (wgmma m64n64k16, ss) -> mask -> running row max m and row sum l (l rescaled by
//            2^(m_old - m_new)), in fp32 and in a fixed block order
//   pass 2   S recomputed per key block -> exp2(s log2e - m log2e) / l -> the warp's 16 rows of a padded fp32 staging
//            tile -> global: each warp store instruction writes 32 consecutive floats of the output (128 B), walking
//            the block's rows x columns in output order, so with one key block (S <= 64) a warp's rows are one
//            contiguous run.  Streaming stores: the probabilities are not read again.
// When S <= 128 both key blocks stay in the ring and pass 2 loads nothing.  A row without a visible key (text with a
// padded first position) has l = 0 and is written as zeros, like the zero output row of the attention kernel.
// The output rows are S * 4 bytes and not 16-byte aligned for odd S: no TMA store can write them.
constexpr int kProbThreads = 128;
constexpr int kProbStages = 2;
constexpr int kProbLd = 72;                                    // staging row stride in floats: conflict-free float2 writes
constexpr uint32_t kProbTileBytes = 64 * 64 * 2;               // one [64 x 64] 16-bit operand block
constexpr uint32_t kProbStageOff = kProbTileBytes;             // K ring after the Q block
constexpr uint32_t kProbStagingOff = kProbStageOff + kProbStages * kProbTileBytes;
constexpr uint32_t kProbBarOff = kProbStagingOff + 64 * kProbLd * 4;
constexpr uint32_t kProbSmem = kProbBarOff + 8 * (1 + kProbStages) + 1024;

struct ProbParams {
  int seq_len;
  int heads;
  int q_blocks;  // ceil(S / 64)
  int causal;
  const int32_t* key_mask;  // [n_seq, S] or nullptr
  float* probs;             // [n_seq, heads, S, S]
};

template <bool F16>
__global__ void __launch_bounds__(kProbThreads)
attention_probs_kernel(const __grid_constant__ CUtensorMap tmQKV, const ProbParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  float* staging = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)) + kProbStagingOff);
  const uint32_t sq = smem_base;
  auto sk = [&](int s) { return smem_base + kProbStageOff + (uint32_t)s * kProbTileBytes; };
  const uint32_t q_bar = smem_base + kProbBarOff;
  auto full_bar = [&](int s) { return q_bar + 8u * (1 + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int S = p.seq_len, D = p.heads * kHeadDim;
  const int qb = blockIdx.x % p.q_blocks;
  const int64_t bh = blockIdx.x / p.q_blocks;
  const int h = (int)(bh % p.heads);
  const int64_t seq = bh / p.heads;
  const int q0 = qb * 64;
  const int n_kb = (S + 63) / 64;
  const bool resident = n_kb <= kProbStages;        // every key block fits the ring: pass 2 reuses them
  const int n_loads = resident ? n_kb : 2 * n_kb;   // load i: key block i % n_kb into stage i % kProbStages

  auto issue_k = [&](int i) {
    const int s = i % kProbStages;
    mbar_arrive_expect_tx(full_bar(s), kProbTileBytes);
    tma_load_3d(sk(s), &tmQKV, full_bar(s), D + h * kHeadDim, (i % n_kb) * 64, (int32_t)seq);
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    mbar_init(q_bar, 1);
    for (int s = 0; s < kProbStages; ++s) mbar_init(full_bar(s), 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(q_bar, kProbTileBytes);
    tma_load_3d(sq, &tmQKV, q_bar, h * kHeadDim, q0, (int32_t)seq);
    for (int i = 0; i < kProbStages && i < n_loads; ++i) issue_k(i);
  }
  __syncthreads();

  const int q4 = lane & 3, rr = lane >> 2;
  const int r0 = 16 * warp + rr;                    // this thread's block rows r0 and r0 + 8
  const int qa = q0 + r0, qc = qa + 8;              // their queries
  const int lim0 = last_visible_key(qa, S, p.causal), lim1 = last_visible_key(qc, S, p.causal);
  const int32_t* km = p.key_mask ? p.key_mask + seq * S : nullptr;
  const uint64_t qdesc = make_smem_desc_sw128(sq, 1024, 16);
  mbar_wait(q_bar, 0);

  // S = Q K^T for use u (key block u % n_kb), masked entries -> -inf
  float sc[32];
  auto scores = [&](int u) {
    const int li = resident ? u % n_kb : u;
    const int s = li % kProbStages;
    mbar_wait(full_bar(s), (uint32_t)((li / kProbStages) & 1));
    qk_scores<F16, 64>(sc, qdesc, make_smem_desc_sw128(sk(s), 1024, 16));
    if (!resident) {
      __syncthreads();  // every warp is done with the stage: refill it
      if (threadIdx.x == 0 && li + kProbStages < n_loads) issue_k(li + kProbStages);
    }
    const int kbase = (u % n_kb) * 64 + 2 * q4;     // + 8 j + e = key of column (j, e)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {  // one warpgroup per CTA: the key mask is read per column, after the wait
        const int key = kbase + 8 * j + e;
        mask_column(sc, j, e, key < S && (km == nullptr || km[key] != 0), key, lim0, lim1);
      }
  };

  // ---- pass 1: running row max / sum
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int kb = 0; kb < n_kb; ++kb) {
    scores(kb);
    fold_row_max(sc, m0, m1, l0, l1);
    const float ms0 = row_shift(m0), ms1 = row_shift(m1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      l0 += softmax_exp(sc[4 * j + 0], ms0) + softmax_exp(sc[4 * j + 1], ms0);
      l1 += softmax_exp(sc[4 * j + 2], ms1) + softmax_exp(sc[4 * j + 3], ms1);
    }
  }
  quad_sum(l0, l1);
  const float ms0 = row_shift(m0), ms1 = row_shift(m1);
  const float inv0 = row_inv(l0), inv1 = row_inv(l1);

  // ---- pass 2: probabilities -> staging rows of this warp -> global
  float* wst = staging + 16 * warp * kProbLd;       // the warp's 16 staging rows
  const int rows = S - (q0 + 16 * warp) < 16 ? S - (q0 + 16 * warp) : 16;  // its rows that are queries (may be <= 0)
  float* out_base = p.probs + ((seq * p.heads + h) * (int64_t)S + q0 + 16 * warp) * S;
  for (int kb = 0; kb < n_kb; ++kb) {
    scores(n_kb + kb);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<float2*>(wst + rr * kProbLd + 8 * j + 2 * q4) =
          make_float2(softmax_exp(sc[4 * j + 0], ms0) * inv0, softmax_exp(sc[4 * j + 1], ms0) * inv0);
      *reinterpret_cast<float2*>(wst + (rr + 8) * kProbLd + 8 * j + 2 * q4) =
          make_float2(softmax_exp(sc[4 * j + 2], ms1) * inv1, softmax_exp(sc[4 * j + 3], ms1) * inv1);
    }
    __syncwarp();
    const int k0 = kb * 64;
    const int nc = S - k0 < 64 ? S - k0 : 64;       // columns of this key block
    const int total = rows > 0 ? rows * nc : 0;
    int r = 0, c = lane;                            // element lane of the block's rows x columns, in output order
    while (c >= nc) { c -= nc; ++r; }
    for (int i = lane; i < total; i += 32) {
      __stcs(out_base + (int64_t)r * S + k0 + c, wst[r * kProbLd + c]);
      c += 32;
      while (c >= nc) { c -= nc; ++r; }
    }
    __syncwarp();  // the staging rows are rewritten by the next block
  }
}

// Launches `blocks` CTAs of the long or the probabilities kernel; its shared-memory limit is raised once per device.
template <auto Kern, int Threads, uint32_t Smem, typename... Args>
int launch_blocks(int64_t blocks, cudaStream_t st, const Args&... args) {
  static unsigned long long configured = 0;
  if (first_use_on_device(configured))
    PLIP_CUDA_CHECK(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Smem));
  PLIP_CUDA_CHECK(launch_kernel(Kern, dim3((unsigned)blocks), dim3(Threads), Smem, st, 1, args...));
  return 0;
}

// The argument checks of launch_attention and launch_attention_probs; `fn` prefixes the messages.
int check_attention_args(const char* fn, const void* qkv, const void* out, int64_t n_seq, int seq_len, int heads) {
  PLIP_REQUIRE(qkv && out, "%s: null argument", fn);
  PLIP_REQUIRE(n_seq > 0 && seq_len > 0 && seq_len <= kMaxVisSeq, "%s: bad shape n_seq=%lld seq_len=%d", fn,
               (long long)n_seq, seq_len);
  PLIP_REQUIRE(heads > 0 && heads <= 16, "%s: bad head count %d", fn, heads);
  return 0;
}

// [n_seq][S][cols] view of a 16-bit activation with a {64, 64, 1} box: rows past a sequence's end are zero-filled on
// load and clipped on store.
int make_seq_tmap(CUtensorMap* tm, const void* base, int64_t n_seq, int seq_len, int cols) {
  return make_tmap_bf16_3d(tm, base, (uint64_t)n_seq, (uint64_t)seq_len, (uint64_t)cols, (uint64_t)cols * 2,
                           (uint64_t)seq_len * cols * 2, 64, 64);
}

}  // namespace

int launch_attention(const __nv_bfloat16* qkv, int64_t n_seq, int seq_len, int heads, bool causal,
                     const int32_t* key_mask, __nv_bfloat16* out, int f16, cudaStream_t st) {
  if (int rc = check_attention_args("attention", qkv, out, n_seq, seq_len, heads)) return rc;
  const int D = heads * kHeadDim;
  if (seq_len > 128) {
    PLIP_REQUIRE(!causal && key_mask == nullptr,
                 "attention: seq_len %d > 128 is supported without causal or key mask only", seq_len);
    LongAttParams p;
    p.seq_len = seq_len;
    p.heads = heads;
    p.q_blocks = (seq_len + 127) / 128;
    const int64_t blocks = n_seq * heads * p.q_blocks;
    PLIP_REQUIRE(blocks < 0x7fffffff && n_seq < 0x7fffffff, "attention: too many sequences");
    CUtensorMap tmQKV, tmO;
    if (int rc = make_seq_tmap(&tmQKV, qkv, n_seq, seq_len, 3 * D)) return rc;
    if (int rc = make_seq_tmap(&tmO, out, n_seq, seq_len, D)) return rc;
    return f16 ? launch_blocks<attention_long_kernel<true>, kLongThreads, kLongSmem>(blocks, st, tmQKV, tmO, p)
               : launch_blocks<attention_long_kernel<false>, kLongThreads, kLongSmem>(blocks, st, tmQKV, tmO, p);
  }
  const int64_t rows = n_seq * seq_len;
  PLIP_REQUIRE(rows + 128 < 0x7fffffff, "attention: too many token rows");
  AttParams p;
  p.n_seq = n_seq;
  p.seq_len = seq_len;
  p.slot = seq_len <= 32 ? 32 : (seq_len <= 64 ? 64 : 128);
  p.group = 128 / p.slot;
  p.heads = heads;
  p.seq_tiles = (n_seq + p.group - 1) / p.group;
  p.causal = causal ? 1 : 0;
  p.key_mask = key_mask;
  CUtensorMap tmL, tmS;
  if (int rc = make_tmap_bf16_2d(&tmL, qkv, (uint64_t)rows, (uint64_t)3 * D, (uint64_t)3 * D * 2, (uint32_t)p.slot, 64)) return rc;
  if (int rc = make_tmap_bf16_2d(&tmS, out, (uint64_t)rows, (uint64_t)D, (uint64_t)D * 2, (uint32_t)seq_len, 64)) return rc;
  PLIP_REQUIRE(p.seq_tiles * heads < 0x7fffffff, "attention: too many tiles");
  if (p.slot == 128) return f16 ? launch_attention_inst<true, 128>(tmL, tmS, p, st) : launch_attention_inst<false, 128>(tmL, tmS, p, st);
  return f16 ? launch_attention_inst<true, 64>(tmL, tmS, p, st) : launch_attention_inst<false, 64>(tmL, tmS, p, st);
}

int launch_attention_probs(const __nv_bfloat16* qkv, int64_t n_seq, int seq_len, int heads, bool causal,
                           const int32_t* key_mask, float* probs, int f16, cudaStream_t st) {
  if (int rc = check_attention_args("attention_probs", qkv, probs, n_seq, seq_len, heads)) return rc;
  ProbParams p;
  p.seq_len = seq_len;
  p.heads = heads;
  p.q_blocks = (seq_len + 63) / 64;
  p.causal = causal ? 1 : 0;
  p.key_mask = key_mask;
  p.probs = probs;
  const int64_t blocks = n_seq * heads * p.q_blocks;
  PLIP_REQUIRE(blocks < 0x7fffffff && n_seq < 0x7fffffff, "attention_probs: too many sequences");
  const int D = heads * kHeadDim;
  CUtensorMap tm;
  if (int rc = make_seq_tmap(&tm, qkv, n_seq, seq_len, 3 * D)) return rc;
  return f16 ? launch_blocks<attention_probs_kernel<true>, kProbThreads, kProbSmem>(blocks, st, tm, p)
             : launch_blocks<attention_probs_kernel<false>, kProbThreads, kProbSmem>(blocks, st, tm, p);
}

}  // namespace plip

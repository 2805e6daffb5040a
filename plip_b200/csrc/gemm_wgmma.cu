// plip_b200 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   acc[M,N] = A[M,K] (bf16, K-major) x W[N,K]^T (bf16, K-major), fp32 accumulation in registers,
//   fused epilogue (bias / QuickGELU / fp32 residual add / patch-embedding scatter).
//
// Replaces, for the PLIP (CLIP ViT-B/32) hot path, the cuBLAS/cuDNN calls behind
//   nn.Conv2d patch embedding   TF:modeling_clip.py:148-154,209
//   q/k/v_proj, out_proj        TF:modeling_clip.py:310-312,334
//   fc1 + QuickGELU, fc2        TF:modeling_clip.py:347-351, TF:activations.py:117-123
//   visual/text_projection      TF:modeling_clip.py:861,823
//
// Structure (one CTA per SM, 288 threads, persistent over 64 x BN output tiles):
//   warpgroups 0-1  consumers, ping-pong: warpgroup w takes the CTA's tiles i with i % 2 == w, each a whole
//                   64 x BN tile, issues wgmma m64nBNk16 on the staged operands and runs the fused epilogue on its
//                   accumulator registers.  The main loops run one at a time, in tile order (two named barriers pass
//                   the turn): a warpgroup hands the turn over once its last k-block is issued, so its epilogue runs
//                   while the other warpgroup's MMAs keep the tensor cores busy.
//   warp 8          producer: one thread feeds the shared-memory ring with TMA, A / W k-blocks of 64 bf16 (one
//                   128B-swizzle atom wide), in the same tile order.  A single warp instead of a register-donating
//                   warpgroup: with 288 threads the compile-time register bound fits the 128-register accumulator
//                   without a spill in any main loop (a 384-thread CTA with setmaxnreg 40 / 232 compiled to the same
//                   168-register bound with more epilogue spills)
// CG == 2 launches clusters of two CTAs on neighbouring 64-row blocks of the same N block: each CTA loads its own A
// rows and one half of the W tile, which TMA multicasts into both CTAs, halving the L2 -> smem W traffic.  Both CTAs
// walk the same tile sequence, so their warpgroups consume each ring stage in lockstep.
#include "gemm.cuh"
#include "wgmma.cuh"

#include <stdio.h>
#include <stdlib.h>

namespace plip {

namespace {

constexpr int BM = 64;   // rows per tile: one consumer warpgroup's wgmma m64
constexpr int BK = 64;   // k-block: 64 bf16 = 128 B = one swizzle atom
constexpr int kThreads = 288;
constexpr int kConsumerWarps = 8;
constexpr uint32_t A_STAGE = BM * BK * 2;
constexpr uint32_t kStoreStageBytes = 16 * 128;  // one [16 rows x 64 bf16] TMA store box

// Staging blocks (2 KB each) per consumer warp.  The 16-bit epilogues alternate two store boxes.  The fp32 residual
// epilogue streams x in and y out through them, one box per block in flight: two blocks at BN 256 and 128, three at
// BN 192 (which still leaves 5 ring stages).  Each count divides the tile's BN / 32 boxes, so every tile starts at
// block 0.  Four blocks at BN 256 would cost a ring stage and measured slower with 128-row tiles
// (tools/gemm_epilogue_probe.py: out_proj 378 vs 351 us, fc2 638 vs 581 us on an H100 80GB HBM3 at 700 W).
constexpr int x_boxes(int BN, int EPI) {
  return EPI != EPI_BIAS_RESID_F32 ? 2 : BN == 192 ? 3 : 2;
}

template <int BN, int EPI>
struct Cfg {
  static constexpr uint32_t B_STAGE = BN * BK * 2;
  static constexpr uint32_t STAGE = A_STAGE + B_STAGE;
  static constexpr int XBOXES = x_boxes(BN, EPI);
  static constexpr uint32_t EPI_BYTES = kConsumerWarps * XBOXES * kStoreStageBytes;
  static constexpr uint32_t BAR_BYTES = EPI == EPI_BIAS_RESID_F32 ? 512 : 256;
  static constexpr uint32_t ALIGN_SLACK = 1024;  // SWIZZLE_128B tiles need a 1024-byte aligned base
  static constexpr int kMaxStages = (227 * 1024 - BAR_BYTES - EPI_BYTES - ALIGN_SLACK) / STAGE;
  static constexpr int STAGES = kMaxStages > 8 ? 8 : kMaxStages;
  static constexpr uint32_t SMEM_BYTES = STAGES * STAGE + EPI_BYTES + BAR_BYTES + ALIGN_SLACK;
};

struct GemmDev {
  int M, N, K;
  const float* bias;
  const float* rowscale;
  void* out;
  int ldo;
  const float* pos;
  int patches, seq;
  const float* colsum;
  const float2* stats_in;
  int n_partials;
  __nv_bfloat16* xb_out;
  float2* stats_out;
};

template <bool F16, int BN>
__device__ __forceinline__ void wgmma_ss(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  if constexpr (BN == 128) wgmma_ss_n128<F16>(d, adesc, bdesc, scale_d);
  else if constexpr (BN == 192) wgmma_ss_n192<F16>(d, adesc, bdesc, scale_d);
  else wgmma_ss_n256<F16>(d, adesc, bdesc, scale_d);
}

// LayerNorm statistics of one row from the partials the producing GEMM left, summed in a fixed order (bitwise
// reproducible); var = E[x^2] - mean^2 in fp32, eps = 1e-5 (TF:371,380).  Returns (-rstd * mean, rstd).
__device__ __forceinline__ float2 ln_row_terms(const GemmDev& p, int grow) {
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j = 0; j < kStatSlots; ++j) {
    const float2 t = (grow < p.M && j < p.n_partials) ? __ldg(p.stats_in + static_cast<size_t>(grow) * kStatSlots + j)
                                                      : make_float2(0.f, 0.f);
    s1 += t.x;
    s2 += t.y;
  }
  const float inv_k = 1.0f / static_cast<float>(p.K);
  const float mean = s1 * inv_k;
  const float rstd = rsqrtf(fmaxf(s2 * inv_k - mean * mean, 0.f) + kLnEps);
  return make_float2(-rstd * mean, rstd);
}

// ---- epilogue ---------------------------------------------------------------------------------
// One warp's [16 rows x BN] slice of the accumulator tile -> global memory.  Lane l owns rows l / 4 and l / 4 + 8 of
// the slice and the column pairs 8 j + 2 (l % 4) of every 8-column block j (wgmma.cuh).
//   fp32 outputs: the four lanes of a row write one full 32-byte sector per block, straight from registers.
//   16-bit outputs: a [16 x 64] block is staged in shared memory in the SWIZZLE_128B pattern (conflict-free: the 8
//   rows of a store instruction hit 8 different 16-byte chunks) and leaves with one TMA bulk store; two staging
//   blocks per warp alternate, so the math of a block overlaps the store of the previous one.
//   The fp32 residual (EPI_BIAS_RESID_F32) reads x through the same two blocks, see there.
template <int BN, int EPI, bool F16>
__device__ __forceinline__ void epilogue_warp(const GemmDev& p, const CUtensorMap* tmC, float (&d)[BN / 2], uint32_t stage_smem,
                                              uint32_t& stage_sel, uint32_t xbar, int row_base, int col_base, int n_blk, int lane,
                                              float2 ln0, float2 ln1) {
  constexpr bool LN_FOLD = (EPI == EPI_LN_BIAS_BF16 || EPI == EPI_LN_BIAS_GELU_BF16);
  constexpr bool GELU = (EPI == EPI_BIAS_GELU_BF16 || EPI == EPI_LN_BIAS_GELU_BF16);
  constexpr bool HAS_BIAS = (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16 || EPI == EPI_BIAS_RESID_F32 || LN_FOLD);
  constexpr bool OUT_BF16 = (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16 || LN_FOLD);
  const int q = lane & 3, rr = lane >> 2;
  const int row0 = row_base + rr, row1 = row0 + 8;

  if constexpr (EPI == EPI_NULL) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc += d[i];
    if (acc == 1.2345e30f && p.M < 0) reinterpret_cast<float*>(p.out)[0] = acc;  // keep the accumulators alive
  } else if constexpr (OUT_BF16) {
    // LN_FOLD: rstd * acc + (bias' - (rstd * mean) * colsum)  ==  rstd * (acc - mean * colsum) + bias'
    // (ln0 / ln1 = the (-rstd * mean, rstd) terms of the two rows, fetched by the caller before the main loop)
#pragma unroll
    for (int blk = 0; blk < BN / 64; ++blk) {
      const uint32_t buf = stage_smem + (stage_sel & 1u) * kStoreStageBytes;
      ++stage_sel;
      if (lane == 0) tma_store_wait_read_but_one();  // the store that last used this block has read it
      __syncwarp();
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = blk * 8 + jj;
        const int col = col_base + 8 * j + 2 * q;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        float v00 = d[4 * j + 0], v01 = d[4 * j + 1], v10 = d[4 * j + 2], v11 = d[4 * j + 3];
        if constexpr (LN_FOLD) {
          const float2 cs = __ldg(reinterpret_cast<const float2*>(p.colsum + col));
          v00 = fmaf(ln0.y, v00, fmaf(ln0.x, cs.x, b.x));
          v01 = fmaf(ln0.y, v01, fmaf(ln0.x, cs.y, b.y));
          v10 = fmaf(ln1.y, v10, fmaf(ln1.x, cs.x, b.x));
          v11 = fmaf(ln1.y, v11, fmaf(ln1.x, cs.y, b.y));
        } else {
          v00 += b.x; v01 += b.y; v10 += b.x; v11 += b.y;
        }
        if constexpr (GELU) {
          v00 = quick_gelu(v00); v01 = quick_gelu(v01); v10 = quick_gelu(v10); v11 = quick_gelu(v11);
        }
        st_shared_b32(buf + rr * 128 + ((jj ^ rr) << 4) + q * 4, pack_op2<F16>(v00, v01));
        st_shared_b32(buf + (rr + 8) * 128 + ((jj ^ rr) << 4) + q * 4, pack_op2<F16>(v10, v11));
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {  // rows past M are clipped by the tensor map
        tma_store_2d(tmC, buf, col_base + blk * 64, row_base);
        tma_store_commit();
      }
    }
  } else if constexpr (EPI == EPI_BIAS_RESID_F32) {
    // x += acc + bias in place; with xb_out, also the 16-bit copy of the new rows (A operand of the next,
    // LayerNorm-folded GEMM) and the (sum, sum of squares) of the fp32 rows, one partial per half of the tile's columns.
    // x is not read straight into registers: the compiler has to assume that out, xb_out and stats_out alias, so
    // every load of x would wait for the stores before it (one 8-byte load per lane in flight), and the accumulator
    // leaves no registers to batch them.  Instead x streams through the warp's NB staging blocks as TMA boxes of
    // [16 rows x 32 fp32] (tmC: the fp32 rows seen as 16-bit pairs, SWIZZLE_128B, rows past M zero-filled): box c
    // lands in block c % NB and completes a phase of that block's barrier (xbar + 8 (c % NB)).  Each lane overwrites
    // the x it read with y, and y leaves with one TMA store of the box (rows past M clipped): full 128-byte lines
    // instead of 32-byte pieces of 8 rows per store instruction.  Once that store has read the block, the load of box
    // c + NB goes into it, so NB boxes are always in flight.  (An L2 prefetch of the tile's rows by the producer during
    // the main loop measured slower: the extra requests delay the A / W feed more than they save here.)
    // In the swizzled box row r holds its eight 16-byte pieces at (piece ^ r % 8): the reads below (8 rows x 2 pieces
    // per instruction) are conflict-free.
    constexpr int kChunkCols = 32;
    constexpr int kChunks = BN / kChunkCols;
    constexpr int NB = x_boxes(BN, EPI);
    static_assert(kChunks % NB == 0, "every tile must start at staging block 0");
    constexpr int kUses = kChunks / NB;  // barrier phases each block completes per tile
    const bool ok0 = row0 < p.M, ok1 = row1 < p.M;
    const bool emit = p.xb_out != nullptr;
    // element offsets of the lane's first column in its two rows (row1 is only touched when row0 < M as well)
    const size_t o0 = static_cast<size_t>(ok0 ? row0 : 0) * p.ldo + col_base + 2 * q;
    const size_t o1 = o0 + 8 * static_cast<size_t>(p.ldo);
    // parity of the phases the blocks completed in earlier tiles: always even (no state) when kUses is even
    uint32_t ph0 = 0;
    if constexpr (kUses % 2 != 0) ph0 = stage_sel++ & 1u;
    auto fetch = [&](int c) {
      if (lane == 0) {
        const uint32_t bar = xbar + 8u * (c % NB);
        mbar_arrive_expect_tx(bar, kStoreStageBytes);
        tma_load_2d(stage_smem + (c % NB) * kStoreStageBytes, tmC, bar, 2 * (col_base + c * kChunkCols), row_base);
      }
    };
    // Refilling a block: lane 0 waits until its TMA store has read the block (the lanes' own accesses to it were
    // ordered before that store by the proxy fence and __syncwarp), then issues the load.
    if (lane == 0) tma_store_wait_read();  // the previous tile's stores out of every block
    __syncwarp();
#pragma unroll
    for (int c = 0; c < NB; ++c) fetch(c);
    float st[2][2] = {};  // (sum, sum of squares) of the lane's two rows over the current half of the tile's columns
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      const int h = c < kChunks / 2 ? 0 : 1;
      mbar_wait(xbar + 8u * (c % NB), ph0 ^ ((c / NB) & 1u));
      const uint32_t buf = stage_smem + (c % NB) * kStoreStageBytes;
#pragma unroll
      for (int jj = 0; jj < kChunkCols / 8; ++jj) {
        const int j = c * (kChunkCols / 8) + jj;
        const int col = col_base + 8 * j + 2 * q;
        const uint32_t xoff = (((2 * jj + (q >> 1)) ^ rr) << 4) + (q & 1) * 8;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        const float2 v0 = make_float2(d[4 * j + 0] + b.x, d[4 * j + 1] + b.y);
        const float2 v1 = make_float2(d[4 * j + 2] + b.x, d[4 * j + 3] + b.y);
        if (ok0) {
          const float2 x = ld_shared_f32x2(buf + rr * 128 + xoff);
          const float2 y = make_float2(x.x + v0.x, x.y + v0.y);
          st_shared_f32x2(buf + rr * 128 + xoff, y);
          if (emit) {
            *reinterpret_cast<uint32_t*>(p.xb_out + o0 + 8 * j) = pack_op2<F16>(y.x, y.y);
            st[0][0] += y.x + y.y;
            st[0][1] = fmaf(y.x, y.x, fmaf(y.y, y.y, st[0][1]));
          }
        }
        if (ok1) {
          const float2 x = ld_shared_f32x2(buf + (rr + 8) * 128 + xoff);
          const float2 y = make_float2(x.x + v1.x, x.y + v1.y);
          st_shared_f32x2(buf + (rr + 8) * 128 + xoff, y);
          if (emit) {
            *reinterpret_cast<uint32_t*>(p.xb_out + o1 + 8 * j) = pack_op2<F16>(y.x, y.y);
            st[1][0] += y.x + y.y;
            st[1][1] = fmaf(y.x, y.x, fmaf(y.y, y.y, st[1][1]));
          }
        }
      }
      fence_proxy_async_smem();  // y in the block -> visible to the TMA store
      __syncwarp();
      if (lane == 0) {
        tma_store_2d(tmC, buf, 2 * (col_base + c * kChunkCols), row_base);
        tma_store_commit();
      }
      if (c + NB < kChunks) {
        if (lane == 0) tma_store_wait_read();
        fetch(c + NB);
      }
      if (emit && (c + 1) % (kChunks / 2) == 0) {  // a half is complete: its partials leave, freeing the registers
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float a = st[r][0], b = st[r][1];
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {  // the 4 lanes that share a row
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
          }
          if (q == 0 && (r == 0 ? ok0 : ok1))
            p.stats_out[static_cast<size_t>(row0 + 8 * r) * kStatSlots + 2 * n_blk + h] = make_float2(a, b);
          st[r][0] = 0.f;
          st[r][1] = 0.f;
        }
      }
    }
  } else {
    float* out = reinterpret_cast<float*>(p.out);
    const bool ok0 = row0 < p.M, ok1 = row1 < p.M;
    float rs0 = 1.f, rs1 = 1.f;
    size_t o0 = static_cast<size_t>(ok0 ? row0 : 0) * p.ldo, o1 = static_cast<size_t>(ok1 ? row1 : 0) * p.ldo;
    if constexpr (EPI == EPI_SIM_F32) {
      rs0 = ok0 ? __ldg(p.rowscale + row0) : 0.f;
      rs1 = ok1 ? __ldg(p.rowscale + row1) : 0.f;
    }
    size_t q0 = 0, q1 = 0;  // EPI_PATCH_F32: rows of the position embedding
    if constexpr (EPI == EPI_PATCH_F32) {
      const int r0 = ok0 ? row0 : 0, r1 = ok1 ? row1 : 0;
      const int b0 = r0 / p.patches, b1 = r1 / p.patches;
      o0 = static_cast<size_t>(b0 * p.seq + 1 + (r0 - b0 * p.patches)) * p.ldo;
      o1 = static_cast<size_t>(b1 * p.seq + 1 + (r1 - b1 * p.patches)) * p.ldo;
      q0 = static_cast<size_t>(1 + (r0 - b0 * p.patches)) * p.N;
      q1 = static_cast<size_t>(1 + (r1 - b1 * p.patches)) * p.N;
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = col_base + 8 * j + 2 * q;
      float2 v0 = make_float2(d[4 * j + 0], d[4 * j + 1]), v1 = make_float2(d[4 * j + 2], d[4 * j + 3]);
      if constexpr (HAS_BIAS) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        v0.x += b.x; v0.y += b.y; v1.x += b.x; v1.y += b.y;
      }
      if constexpr (EPI == EPI_SIM_F32) {
        const float2 cs = __ldg(reinterpret_cast<const float2*>(p.bias + col));  // the column scales
        if (ok0) *reinterpret_cast<float2*>(out + o0 + col) = make_float2(v0.x * rs0 * cs.x, v0.y * rs0 * cs.y);
        if (ok1) *reinterpret_cast<float2*>(out + o1 + col) = make_float2(v1.x * rs1 * cs.x, v1.y * rs1 * cs.y);
      } else if constexpr (EPI == EPI_PATCH_F32) {
        if (ok0) {
          const float2 e = __ldg(reinterpret_cast<const float2*>(p.pos + q0 + col));
          *reinterpret_cast<float2*>(out + o0 + col) = make_float2(v0.x + e.x, v0.y + e.y);
        }
        if (ok1) {
          const float2 e = __ldg(reinterpret_cast<const float2*>(p.pos + q1 + col));
          *reinterpret_cast<float2*>(out + o1 + col) = make_float2(v1.x + e.x, v1.y + e.y);
        }
      } else {
        if (ok0) *reinterpret_cast<float2*>(out + o0 + col) = v0;
        if (ok1) *reinterpret_cast<float2*>(out + o1 + col) = v1;
      }
    }
  }
}

template <int CG, int BN, int EPI, bool F16>
__global__ void __launch_bounds__(kThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmC, const GemmDev p) {
  using C = Cfg<BN, EPI>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t epi_base = smem_base + STAGES * C::STAGE;   // 1024-aligned: 2 KB store boxes
  const uint32_t bar_base = epi_base + C::EPI_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t resid_bar = bar_base + 8u * (2 * STAGES);  // EPI_BIAS_RESID_F32: one per staging block
  static_assert(8 * (2 * STAGES + (EPI == EPI_BIAS_RESID_F32 ? C::XBOXES * kConsumerWarps : 0)) <= C::BAR_BYTES,
                "barrier area too small");

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const uint32_t cta_rank = (CG > 1) ? cluster_ctarank() : 0u;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);        // the producer's arrive.expect_tx
      mbar_init(empty_bar(s), CG);      // one arrive from the consuming warpgroup of every CTA that reads the slot's W tile
    }
    if constexpr (EPI == EPI_BIAS_RESID_F32) {
      tma_prefetch_desc(&tmC);
      for (int i = 0; i < C::XBOXES * kConsumerWarps; ++i) mbar_init(resid_bar + 8u * i, 1);  // lane 0's arrive.expect_tx
    }
    fence_mbar_init();
  }
  if constexpr (CG > 1) cluster_sync_all(); else __syncthreads();

  const int num_n_blk = p.N / BN;
  const int num_m_blk = (p.M + BM * CG - 1) / (BM * CG);  // CG == 2: an odd block count leaves the second CTA of the
  const int num_tiles = num_m_blk * num_n_blk;            // last cluster with rows past M only (zero fill, no stores)
  const int num_kb = p.K / BK;
  const int tile0 = blockIdx.x / CG;
  const int tile_step = gridDim.x / CG;
  const int my_tiles = (num_tiles - tile0 + tile_step - 1) / tile_step;  // >= 1: the grid has at most num_tiles groups

  if (wg == 2) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int t = tile0; t < num_tiles; t += tile_step) {
        const int m0 = ((t / num_n_blk) * CG + cta_rank) * BM;
        const int n0 = (t % num_n_blk) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar(s), ph ^ 1u);
          const uint32_t sa = smem_base + s * C::STAGE;
          const uint32_t sb = sa + A_STAGE;
          mbar_arrive_expect_tx(full_bar(s), C::STAGE);
          tma_load_2d(sa, &tmA, full_bar(s), kb * BK, m0);
          if constexpr (CG == 1) {
            tma_load_2d(sb, &tmB, full_bar(s), kb * BK, n0);
          } else {
            // this CTA's half of the W tile, delivered to the same slot of both CTAs
            tma_load_2d_mc(sb + cta_rank * (C::B_STAGE / 2), &tmB, full_bar(s), kb * BK, n0 + cta_rank * (BN / 2), 0x3);
          }
          if (++s == STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== MMA + epilogue, two warpgroups taking turns =====================
    // Named barrier 1 + w completes when warpgroup w may start its next main loop: warpgroup w syncs on it (128
    // threads) and the other warpgroup arrives on it (128) once its own main loop is issued.  The turn order also
    // keeps each warpgroup's ring waits within one phase of the barriers it waits on.  Both warpgroups run the same
    // number of rounds; every arrive is matched by one sync: warpgroup 1 waits for its turn even in a last round
    // without a tile, and does not pass the turn after its last round (warpgroup 0 has nothing left to start).
    const int wtid = threadIdx.x & 127;
    auto release = [&](int s) {  // the warpgroup's wgmmas on slot s have retired
      if (wtid == 0) mbar_arrive(empty_bar(s));
      if constexpr (CG > 1) {
        if (wtid == 32) mbar_arrive_cluster(mapa_shared(empty_bar(s), cta_rank ^ 1u));
      }
    };
    float d[BN / 2];
    int s = 0;
    uint32_t ph = 0;
    auto skip_tile = [&]() {  // the other warpgroup's k-blocks in the ring
      s += num_kb;
      ph ^= static_cast<uint32_t>(s / STAGES) & 1u;
      s %= STAGES;
    };
    uint32_t stage_sel = 0;
    const uint32_t my_turn = 1u + wg, other_turn = 2u - wg;
    const int rounds = (my_tiles + 1) / 2;
    if (wg == 1) skip_tile();
    for (int r = 0; r < rounds; ++r) {
      const int i = 2 * r + wg;
      const int t = tile0 + i * tile_step;
      const int n_blk = t % num_n_blk;
      const int m0 = ((t / num_n_blk) * CG + cta_rank) * BM;
      const int wrow = m0 + (warp & 3) * 16;  // first of this warp's 16 rows
      float2 ln0 = make_float2(0.f, 1.f), ln1 = make_float2(0.f, 1.f);
      if constexpr (EPI == EPI_LN_BIAS_BF16 || EPI == EPI_LN_BIAS_GELU_BF16) {
        // the row statistics are fetched before the main loop: the loads overlap the MMAs and need no registers next
        // to the full accumulator
        if (i < my_tiles) {
          ln0 = ln_row_terms(p, wrow + (lane >> 2));
          ln1 = ln_row_terms(p, wrow + (lane >> 2) + 8);
        }
      }
      if (wg == 1 || r > 0) named_barrier_sync<256>(my_turn);
      if (i >= my_tiles) break;  // warpgroup 1 in the last round of an odd tile count
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(full_bar(s), ph);
        const uint32_t sa = smem_base + s * C::STAGE;
        const uint64_t adesc = make_smem_desc_sw128(sa, 1024, 16);
        const uint64_t bdesc = make_smem_desc_sw128(sa + A_STAGE, 1024, 16);
        wgmma_pin(d);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_ss<F16, BN>(d, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's group has retired: hand its slot back
        if (prev >= 0) release(prev);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1u; }
      }
      if (wg == 0 || r + 1 < rounds) named_barrier_arrive<256>(other_turn);
      wgmma_wait<0>();
      wgmma_pin(d);
      release(prev);
      skip_tile();
      epilogue_warp<BN, EPI, F16>(p, &tmC, d, epi_base + warp * C::XBOXES * kStoreStageBytes, stage_sel,
                                  resid_bar + 8u * C::XBOXES * warp, wrow,
                                  n_blk * BN, n_blk, lane, ln0, ln1);
    }
    if (lane == 0) tma_store_wait_all();
    __syncwarp();
  }
  // no CTA may leave while its peer still multicasts into its shared memory or arrives on its barriers
  if constexpr (CG > 1) cluster_sync_all();
}

int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

template <int CG, int BN, int EPI, bool F16>
int launch_inst(const GemmArgs& g, cudaStream_t stream) {
  using C = Cfg<BN, EPI>;
  auto kern = gemm_kernel<CG, BN, EPI, F16>;
  static unsigned long long configured = 0;
  static int max_groups = 0;  // co-resident clusters (CTAs for CG == 1)
  if (first_use_on_device(configured)) {
    PLIP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    int dev = 0, sms = 0;
    PLIP_CUDA_CHECK(cudaGetDevice(&dev));
    PLIP_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    max_groups = sms / CG;
    if (CG >= 2) {
      // the SMs of a cluster share a GPC, so fewer than sms / 2 clusters may fit at once
      cudaLaunchConfig_t q = {};
      q.gridDim = dim3(sms / CG * CG);
      q.blockDim = dim3(kThreads);
      q.dynamicSmemBytes = C::SMEM_BYTES;
      cudaLaunchAttribute qa[1];
      qa[0].id = cudaLaunchAttributeClusterDimension;
      qa[0].val.clusterDim.x = CG; qa[0].val.clusterDim.y = 1; qa[0].val.clusterDim.z = 1;
      q.attrs = qa; q.numAttrs = 1;
      int n_clusters = 0;
      PLIP_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&n_clusters, kern, &q));
      if (n_clusters > 0 && n_clusters < max_groups) max_groups = n_clusters;
    }
    PLIP_REQUIRE(max_groups > 0, "launch_gemm: no resident CTA fits (cg=%d bn=%d)", CG, BN);
  }
  CUtensorMap tmA, tmB;
  if (int rc = make_tmap_bf16_2d(&tmA, g.A, g.M, g.K, (uint64_t)g.lda * 2, BM, BK)) return rc;
  if (int rc = make_tmap_bf16_2d(&tmB, g.W, g.N, g.K, (uint64_t)g.ldw * 2, BN / CG, BK)) return rc;
  constexpr bool kOutBf16 = (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16 || EPI == EPI_LN_BIAS_BF16 ||
                             EPI == EPI_LN_BIAS_GELU_BF16);
  CUtensorMap tmC = tmA;  // placeholder when unused
  if (kOutBf16)
    if (int rc = make_tmap_bf16_2d(&tmC, g.out, g.M, g.N, (uint64_t)g.ldo * 2, 16, 64)) return rc;
  // the residual epilogue loads [16 x 32] fp32 boxes of x: the same bytes as [16 x 64] 16-bit elements, so the fp32
  // rows are described as rows of 2 N 16-bit elements (a plain copy: the element type only sets the unit of the box)
  if (EPI == EPI_BIAS_RESID_F32)
    if (int rc = make_tmap_bf16_2d(&tmC, g.out, g.M, 2 * (uint64_t)g.N, (uint64_t)g.ldo * 4, 16, 64)) return rc;

  GemmDev p;
  p.M = g.M; p.N = g.N; p.K = g.K;
  p.bias = g.bias; p.rowscale = g.rowscale; p.out = g.out; p.ldo = g.ldo; p.pos = g.pos;
  p.patches = g.patches; p.seq = g.seq;
  p.colsum = g.colsum; p.stats_in = g.stats_in; p.n_partials = g.n_partials;
  p.xb_out = g.xb_out; p.stats_out = g.stats_out;
  if (g.n_tiles_used) *g.n_tiles_used = 2 * (g.N / BN);

  // With fewer tiles than resident groups each CTA takes one tile and its second warpgroup idles: two tiles on one SM
  // would run their main loops one after the other, one tile on each of two SMs runs them side by side.
  const int num_tiles = ((g.M + BM * CG - 1) / (BM * CG)) * (g.N / BN);
  const int groups = max_groups < num_tiles ? max_groups : num_tiles;
  PLIP_CUDA_CHECK(launch_kernel(kern, dim3(groups * CG), dim3(kThreads), C::SMEM_BYTES, stream, CG, tmA, tmB, tmC, p));
  return 0;
}

template <int CG, int BN, bool F16>
int launch_epi_fmt(const GemmArgs& g, cudaStream_t stream) {
  switch (g.epi) {
    case EPI_BIAS_BF16: return launch_inst<CG, BN, EPI_BIAS_BF16, F16>(g, stream);
    case EPI_BIAS_GELU_BF16: return launch_inst<CG, BN, EPI_BIAS_GELU_BF16, F16>(g, stream);
    case EPI_BIAS_RESID_F32: return launch_inst<CG, BN, EPI_BIAS_RESID_F32, F16>(g, stream);
    case EPI_PATCH_F32: return launch_inst<CG, BN, EPI_PATCH_F32, F16>(g, stream);
    case EPI_F32: return launch_inst<CG, BN, EPI_F32, F16>(g, stream);
    case EPI_LN_BIAS_BF16: return launch_inst<CG, BN, EPI_LN_BIAS_BF16, F16>(g, stream);
    case EPI_LN_BIAS_GELU_BF16: return launch_inst<CG, BN, EPI_LN_BIAS_GELU_BF16, F16>(g, stream);
    case EPI_NULL: return launch_inst<CG, BN, EPI_NULL, F16>(g, stream);
    case EPI_SIM_F32: return launch_inst<CG, BN, EPI_SIM_F32, F16>(g, stream);
    default: set_last_error("launch_gemm: bad epilogue %d", g.epi); return -2;
  }
}
template <int CG, int BN>
int launch_epi(const GemmArgs& g, cudaStream_t stream) {
  return g.f16 ? launch_epi_fmt<CG, BN, true>(g, stream) : launch_epi_fmt<CG, BN, false>(g, stream);
}

}  // namespace

int launch_gemm(const GemmArgs& g, cudaStream_t stream) {
  PLIP_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0, "launch_gemm: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
  PLIP_REQUIRE(g.K % BK == 0, "launch_gemm: K=%d must be a multiple of %d", g.K, BK);
  PLIP_REQUIRE(g.N % 128 == 0 || g.N % 192 == 0, "launch_gemm: N=%d must be a multiple of 128 or 192", g.N);
  PLIP_REQUIRE((g.lda % 8) == 0 && (g.ldw % 8) == 0 && (g.ldo % 8) == 0,
               "launch_gemm: leading dimensions must be multiples of 8 elements");
  PLIP_REQUIRE((reinterpret_cast<uintptr_t>(g.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.W) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(g.out) & 15) == 0,
               "launch_gemm: operands must be 16-byte aligned");
  if (g.epi == EPI_LN_BIAS_BF16 || g.epi == EPI_LN_BIAS_GELU_BF16)
    PLIP_REQUIRE(g.colsum && g.stats_in && g.bias && g.n_partials >= 1 && g.n_partials <= kStatSlots,
                 "launch_gemm: LayerNorm-folded epilogue needs colsum, stats and 1..%d partials", kStatSlots);
  if (g.epi == EPI_SIM_F32)
    PLIP_REQUIRE(g.bias && g.rowscale, "launch_gemm: the similarity epilogue needs row and column scales");
  if (g.epi == EPI_PATCH_F32)
    PLIP_REQUIRE(g.patches >= 1 && g.seq == g.patches + 1, "launch_gemm: patch epilogue with %d patches, %d rows",
                 g.patches, g.seq);
  if (g.xb_out || g.stats_out)
    PLIP_REQUIRE(g.epi == EPI_BIAS_RESID_F32 && g.xb_out && g.stats_out,
                 "launch_gemm: xb/stats outputs belong to the residual epilogue");
  static const int env_cg = env_int("PLIP_GEMM_CG", 0);
  static const int env_bn = env_int("PLIP_GEMM_BN", 0);
  int cg = g.force_cg ? g.force_cg : (env_cg ? env_cg : 2);
  int bn = g.force_bn ? g.force_bn : (env_bn ? env_bn : 256);
  if (g.N % bn != 0) bn = 128;
  // a residual GEMM that emits row statistics has two slots per N tile: a narrow PLIP_GEMM_BN yields to 256 there
  if (!g.force_bn && g.stats_out && 2 * (g.N / bn) > kStatSlots && g.N % 256 == 0) bn = 256;
  PLIP_REQUIRE((cg == 1 || cg == 2) && (bn == 128 || bn == 256 || (bn == 192 && cg == 2)),
               "launch_gemm: bad config cg=%d bn=%d", cg, bn);
  PLIP_REQUIRE(!g.stats_out || 2 * (g.N / bn) <= kStatSlots, "launch_gemm: N=%d / BN=%d exceeds %d statistics slots",
               g.N, bn, kStatSlots);
  if (cg == 1) return bn == 256 ? launch_epi<1, 256>(g, stream) : launch_epi<1, 128>(g, stream);
  if (bn == 192) return launch_epi<2, 192>(g, stream);
  return bn == 256 ? launch_epi<2, 256>(g, stream) : launch_epi<2, 128>(g, stream);
}

}  // namespace plip

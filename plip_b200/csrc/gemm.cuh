// plip_b200 — wgmma GEMM interface (host side).
#pragma once
#include "common.cuh"

namespace plip {

// Fused epilogues.  All GEMMs compute acc[M,N] = A[M,K] (bf16) x W[N,K]^T (bf16), fp32 accumulate.
enum GemmEpilogue : int {
  EPI_BIAS_BF16 = 0,       // out_bf16 = acc + bias                     (QKV projection, TF:modeling_clip.py:310-312)
  EPI_BIAS_GELU_BF16 = 1,  // out_bf16 = quick_gelu(acc + bias)         (fc1, TF:modeling_clip.py:348-349)
  EPI_BIAS_RESID_F32 = 2,  // x_f32   += acc + bias  (in place)         (out_proj / fc2 + residual, :334,:377,:350,:382)
  EPI_PATCH_F32 = 3,       // x_f32[b*S+1+p] = acc + pos[1+p]           (patch conv + position embedding, :209-217)
  EPI_F32 = 4,             // out_f32 = acc                             (visual/text projection, :861,:823)
  // LayerNorm folded into the consuming GEMM (DESIGN.md §4.1): A holds bf16(x) (un-normalised), W holds
  // bf16(gamma o W), colsum[n] = sum_k W'[n,k], bias' = bias + W beta, and per-row (sum, sum of squares)
  // partials of x come from the producing residual GEMM:  out = rstd_r (acc - mean_r colsum_n) + bias'_n.
  EPI_LN_BIAS_BF16 = 5,       // layer_norm1 + q/k/v projection            (TF:371, 310-312)
  EPI_LN_BIAS_GELU_BF16 = 6,  // layer_norm2 + fc1 + QuickGELU             (TF:380, 348-349)
  EPI_NULL = 7,               // (diagnostic) accumulators are dropped: main-loop-only rate
  // Similarity head on the tensor cores (similarity.cu): out_f32[r,c] = acc * rowscale[r] * colscale[c].  The operands
  // are fp16 hi/lo splits of power-of-two-scaled embeddings ([hi|lo|hi] x [hi|hi|lo], K = 3 x 512), the scales undo
  // the power of two and carry logit_scale and the optional 1/|x| normalisation.   (TF:modeling_clip.py:923-930)
  EPI_SIM_F32 = 8,
  EPI_COUNT = 9
};

constexpr int kStatSlots = 8;  // per-row partial statistics slots (two per N tile of the producing GEMM: one per half of the tile's columns)

struct GemmArgs {
  const __nv_bfloat16* A = nullptr;  // [M, K] row-major, row stride lda elements
  int lda = 0;
  const __nv_bfloat16* W = nullptr;  // [N, K] row-major (nn.Linear weight layout), row stride ldw
  int ldw = 0;
  int M = 0, N = 0, K = 0;
  const float* bias = nullptr;       // [N]   (EPI_SIM_F32: the column scales)
  const float* rowscale = nullptr;   // [M]   EPI_SIM_F32 only
  void* out = nullptr;               // bf16 or fp32 depending on epilogue; row stride ldo elements
  int ldo = 0;
  const float* pos = nullptr;        // EPI_PATCH_F32: vision position embedding [seq, N]
  int patches = kPatches;            // EPI_PATCH_F32: patches per image (A row r = patch r % patches of image r / patches)
  int seq = kVisSeq;                 // EPI_PATCH_F32: rows per image in out (class row + patches)
  const float* colsum = nullptr;     // EPI_LN_*: [N] row sums of the folded bf16 weight
  const float2* stats_in = nullptr;  // EPI_LN_*: [M, kStatSlots] partial (sum, sumsq) of the fp32 rows behind A
  int n_partials = 0;                // EPI_LN_*: valid slots in stats_in
  __nv_bfloat16* xb_out = nullptr;   // EPI_BIAS_RESID_F32 (optional): bf16 copy of the updated rows, stride ldo
  float2* stats_out = nullptr;       // EPI_BIAS_RESID_F32 (optional): [M, kStatSlots], slot = N-tile index
  int* n_tiles_used = nullptr;       // out (host): number of statistics slots written (2 per N tile)
  int epi = EPI_F32;
  int f16 = 0;                       // 16-bit operand format of A, W and the bf16-typed outputs: 0 = bfloat16, 1 = IEEE half
  int force_cg = 0;                  // 0 = auto; 1 / 2 = CTAs per cluster (test hook)
  int force_bn = 0;                  // 0 = auto; 128 / 192 / 256 = N tile (test hook)
};

// Enqueue the GEMM on `stream`.  Returns 0 on success (see last_error otherwise).
int launch_gemm(const GemmArgs& g, cudaStream_t stream);

}  // namespace plip

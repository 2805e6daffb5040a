// plip_b200 — similarity head: L2-normalise + scale * A . B^T in one fp32 kernel, and a fused top-k.
//
// Replaces   x / _get_vector_norm(x);  text @ image.T * exp(logit_scale);  .t()   (TF:modeling_clip.py:57-65,923-930)
// and the numpy heads  key.dot(space.T) + argmax / argsort top-k
//   (plip.py:73-87,99-102; evaluation/zero_shot/zero_shot.py:12-13; evaluation/retrieval/retrieval.py:13-16).
//
// The [n,512] x [m,512]^T product needs fp32-class accuracy: the |dlogits| <= 1e-3 bar at logit scales up to 100
// rules out plain 16-bit operands (SURVEY.md §7).  Wide score matrices and big top-k problems run it on the tensor
// cores with operands split into fp16 hi + lo parts; the other cases use fp32 FMA kernels that accumulate the row
// norms from the same operand tiles that feed the product, so each input is read once per tile.
#include "kernels.cuh"

#include <cuda_fp16.h>

#include <mutex>

namespace plip {

namespace {

constexpr int kSimThreads = 256;
constexpr int TM = 64, TN = 64, TK = 16;

__global__ void __launch_bounds__(kSimThreads)
similarity_kernel(const float* __restrict__ A, int64_t n, const float* __restrict__ B, int64_t m, int K,
                  float scale, int norm_a, int norm_b, float* __restrict__ C, int64_t ldc) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  __shared__ float inv_a[TM], inv_b[TN];

  const int t = threadIdx.x;
  const int64_t row0 = (int64_t)blockIdx.y * TM;
  const int64_t col0 = (int64_t)blockIdx.x * TN;
  const int lr = t >> 2;         // tile row loaded by this thread (0..63)
  const int lk = (t & 3) * 4;    // k offset inside the TK slab
  const int ty = t >> 4, tx = t & 15;

  float acc[4][4] = {};
  float ssa = 0.f, ssb = 0.f;
  const bool a_ok = row0 + lr < n, b_ok = col0 + lr < m;
  const float* ap = A + (row0 + lr) * K + lk;
  const float* bp = B + (col0 + lr) * K + lk;

  for (int k0 = 0; k0 < K; k0 += TK) {
    float4 av = a_ok ? __ldg(reinterpret_cast<const float4*>(ap + k0)) : make_float4(0, 0, 0, 0);
    float4 bv = b_ok ? __ldg(reinterpret_cast<const float4*>(bp + k0)) : make_float4(0, 0, 0, 0);
    ssa += av.x * av.x + av.y * av.y + av.z * av.z + av.w * av.w;
    ssb += bv.x * bv.x + bv.y * bv.y + bv.z * bv.z + bv.w * bv.w;
    __syncthreads();
    As[lk + 0][lr] = av.x; As[lk + 1][lr] = av.y; As[lk + 2][lr] = av.z; As[lk + 3][lr] = av.w;
    Bs[lk + 0][lr] = bv.x; Bs[lk + 1][lr] = bv.y; Bs[lk + 2][lr] = bv.z; Bs[lk + 3][lr] = bv.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float ar[4] = {a.x, a.y, a.z, a.w};
      const float br[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
  }
  // the 4 threads that loaded one row are adjacent lanes
  ssa += __shfl_xor_sync(0xffffffffu, ssa, 1);
  ssa += __shfl_xor_sync(0xffffffffu, ssa, 2);
  ssb += __shfl_xor_sync(0xffffffffu, ssb, 1);
  ssb += __shfl_xor_sync(0xffffffffu, ssb, 2);
  if ((t & 3) == 0) {
    inv_a[lr] = norm_a ? 1.0f / sqrtf(ssa) : 1.0f;
    inv_b[lr] = norm_b ? 1.0f / sqrtf(ssb) : 1.0f;
  }
  __syncthreads();

  const bool vec_ok = (ldc % 4 == 0) && (col0 + tx * 4 + 3 < m);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = row0 + ty * 4 + i;
    if (r >= n) continue;
    const float sa = scale * inv_a[ty * 4 + i];
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = acc[i][j] * sa * inv_b[tx * 4 + j];
    float* cp = C + r * ldc + col0 + tx * 4;
    if (vec_ok) {
      *reinterpret_cast<float4*>(cp) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (col0 + tx * 4 + j < m) cp[j] = o[j];
    }
  }
}

// ---- fused similarity + top-k (round-1 version: one CTA per query, streaming the space) ---------
constexpr int kTopkThreads = 128;
constexpr int kTopkMax = 64;

__device__ __forceinline__ bool better(float s, int i, float s2, int i2) {
  return s > s2 || (s == s2 && i < i2);
}

__global__ void __launch_bounds__(kTopkThreads)
similarity_topk_kernel(const float* __restrict__ Q, int64_t n, const float* __restrict__ Sp, int64_t m, int K,
                       float scale, int norm_q, int norm_s, int k, int32_t* __restrict__ idx,
                       float* __restrict__ val) {
  __shared__ float q[kProj];
  __shared__ float ls[4][kTopkMax];
  __shared__ int li[4][kTopkMax];
  __shared__ float red[4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x;

  float ss = 0.f;
  for (int j = threadIdx.x; j < K; j += kTopkThreads) {
    const float v = Q[row * K + j];
    q[j] = v;
    ss += v * v;
  }
  ss = warp_sum(ss);
  if (lane == 0) red[warp] = ss;
  for (int j = lane; j < k; j += 32) {
    ls[warp][j] = -INFINITY;
    li[warp][j] = 0x7fffffff;
  }
  __syncthreads();
  const float qs = scale * (norm_q ? 1.0f / sqrtf(red[0] + red[1] + red[2] + red[3]) : 1.0f);

  for (int64_t c = warp; c < m; c += 4) {
    const float* sp = Sp + c * K;
    float dot = 0.f, s2 = 0.f;
    for (int j = lane * 4; j < K; j += 128) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(sp + j));
      const float4 w = *reinterpret_cast<const float4*>(&q[j]);
      dot = fmaf(v.x, w.x, fmaf(v.y, w.y, fmaf(v.z, w.z, fmaf(v.w, w.w, dot))));
      s2 += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    dot = warp_sum(dot);
    s2 = warp_sum(s2);
    const float score = dot * qs * (norm_s ? 1.0f / sqrtf(s2) : 1.0f);
    if (lane == 0 && better(score, (int)c, ls[warp][k - 1], li[warp][k - 1])) {
      int pos = k - 1;  // insertion into the warp's descending list
      while (pos > 0 && better(score, (int)c, ls[warp][pos - 1], li[warp][pos - 1])) {
        ls[warp][pos] = ls[warp][pos - 1];
        li[warp][pos] = li[warp][pos - 1];
        --pos;
      }
      ls[warp][pos] = score;
      li[warp][pos] = (int)c;
    }
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int head[4] = {0, 0, 0, 0};
    for (int o = 0; o < k; ++o) {
      int bw = -1;
      for (int w = 0; w < 4; ++w) {
        if (head[w] >= k) continue;
        if (bw < 0 || better(ls[w][head[w]], li[w][head[w]], ls[bw][head[bw]], li[bw][head[bw]])) bw = w;
      }
      const int id = li[bw][head[bw]];
      idx[row * k + o] = (id == 0x7fffffff) ? -1 : id;
      if (val) val[row * k + o] = ls[bw][head[bw]];
      ++head[bw];
    }
  }
}

// ---- fused similarity + top-k, GEMM-shaped: 64 queries x a slice of the space per CTA ---------------
// The score tile is produced exactly like similarity_kernel (fp32 FMA, norms folded in) but stays in
// shared memory; each warp then folds 8 rows into per-row sorted top-k lists (also in smem).  Candidates
// below the current k-th best are rejected with one compare, so insertions are rare after warm-up.
// The space is split over gridDim.y CTAs per query tile; the last CTA to finish merges the partial lists
// (threadfence + atomic ticket).  Ordering: higher score first, ties by lower index (deterministic).
constexpr int kTkThreads = 256;
constexpr int kTkSmemFloats = 2 * TK * (TM + 4) + TM + TN + TM * (TN + 1) + TM * kTopkMax;  // + int lists

struct TopkLists {
  float* v;  // [TM][kTopkMax]
  int* i;    // [TM][kTopkMax]
};

// Insert (s, id) into the sorted list of `row` (one warp, k <= 64: lane holds entries lane and lane + 32).
__device__ __forceinline__ void topk_insert(const TopkLists& L, int row, int k, float s, int id, int lane) {
  float* lv = L.v + row * kTopkMax;
  int* li = L.i + row * kTopkMax;
  const float v0 = lane < k ? lv[lane] : -INFINITY, v1 = lane + 32 < k ? lv[lane + 32] : -INFINITY;
  const int i0 = lane < k ? li[lane] : 0x7fffffff, i1 = lane + 32 < k ? li[lane + 32] : 0x7fffffff;
  const unsigned b0 = __ballot_sync(0xffffffffu, lane < k && better(v0, i0, s, id));
  const unsigned b1 = __ballot_sync(0xffffffffu, lane + 32 < k && better(v1, i1, s, id));
  const int pos = __popc(b0) + __popc(b1);  // entries that stay ahead of the candidate
  if (pos >= k) return;
  __syncwarp();
  if (lane >= pos && lane + 1 < k) { lv[lane + 1] = v0; li[lane + 1] = i0; }
  if (lane + 32 >= pos && lane + 33 < k) { lv[lane + 33] = v1; li[lane + 33] = i1; }
  __syncwarp();
  if (lane == 0) { lv[pos] = s; li[pos] = id; }
  __syncwarp();
}

__global__ void __launch_bounds__(kTkThreads)
similarity_topk_tiled_kernel(const float* __restrict__ Q, int64_t n, const float* __restrict__ Sp, int64_t m, int K,
                             float scale, int norm_q, int norm_s, int k, int tiles_per_split,
                             float* __restrict__ scratch_v, int* __restrict__ scratch_i,
                             unsigned* __restrict__ tickets, int32_t* __restrict__ idx, float* __restrict__ val) {
  extern __shared__ float tk_smem[];
  float (*As)[TM + 4] = reinterpret_cast<float (*)[TM + 4]>(tk_smem);
  float (*Bs)[TN + 4] = reinterpret_cast<float (*)[TN + 4]>(tk_smem + TK * (TM + 4));
  float* inv_a = tk_smem + 2 * TK * (TM + 4);
  float* inv_b = inv_a + TM;
  float (*Sc)[TN + 1] = reinterpret_cast<float (*)[TN + 1]>(inv_b + TN);
  TopkLists L;
  L.v = inv_b + TN + TM * (TN + 1);
  L.i = reinterpret_cast<int*>(L.v + TM * kTopkMax);
  __shared__ unsigned last_flag;

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int64_t row0 = (int64_t)blockIdx.x * TM;
  const int lr = t >> 2, lk = (t & 3) * 4, ty = t >> 4, tx = t & 15;
  const int64_t total_tiles = (m + TN - 1) / TN;
  const int64_t tile_lo = (int64_t)blockIdx.y * tiles_per_split;
  const int64_t tile_hi = min(total_tiles, tile_lo + tiles_per_split);

  for (int j = t; j < TM * kTopkMax; j += kTkThreads) { L.v[j] = -INFINITY; L.i[j] = 0x7fffffff; }
  const bool a_ok = row0 + lr < n;
  const float* ap = Q + (row0 + lr) * K + lk;
  bool have_inv_a = false;

  for (int64_t tile = tile_lo; tile < tile_hi; ++tile) {
    const int64_t col0 = tile * TN;
    const bool b_ok = col0 + lr < m;
    const float* bp = Sp + (col0 + lr) * K + lk;
    float acc[4][4] = {};
    float ssa = 0.f, ssb = 0.f;
    for (int k0 = 0; k0 < K; k0 += TK) {
      const float4 av = a_ok ? __ldg(reinterpret_cast<const float4*>(ap + k0)) : make_float4(0, 0, 0, 0);
      const float4 bv = b_ok ? __ldg(reinterpret_cast<const float4*>(bp + k0)) : make_float4(0, 0, 0, 0);
      ssa += av.x * av.x + av.y * av.y + av.z * av.z + av.w * av.w;
      ssb += bv.x * bv.x + bv.y * bv.y + bv.z * bv.z + bv.w * bv.w;
      __syncthreads();
      As[lk + 0][lr] = av.x; As[lk + 1][lr] = av.y; As[lk + 2][lr] = av.z; As[lk + 3][lr] = av.w;
      Bs[lk + 0][lr] = bv.x; Bs[lk + 1][lr] = bv.y; Bs[lk + 2][lr] = bv.z; Bs[lk + 3][lr] = bv.w;
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < TK; ++kk) {
        const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        const float ar[4] = {a.x, a.y, a.z, a.w};
        const float br[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
      }
    }
    ssa += __shfl_xor_sync(0xffffffffu, ssa, 1);
    ssa += __shfl_xor_sync(0xffffffffu, ssa, 2);
    ssb += __shfl_xor_sync(0xffffffffu, ssb, 1);
    ssb += __shfl_xor_sync(0xffffffffu, ssb, 2);
    if ((t & 3) == 0) {
      if (!have_inv_a) inv_a[lr] = norm_q ? 1.0f / sqrtf(ssa) : 1.0f;
      inv_b[lr] = norm_s ? 1.0f / sqrtf(ssb) : 1.0f;
    }
    have_inv_a = true;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool ok = (row0 + ty * 4 + i < n) && (col0 + tx * 4 + j < m);
        Sc[ty * 4 + i][tx * 4 + j] = ok ? acc[i][j] * scale * inv_a[ty * 4 + i] * inv_b[tx * 4 + j] : -INFINITY;
      }
    __syncthreads();
    // fold the tile into the per-row lists: warp w owns rows 8w .. 8w+7
    for (int r = warp * 8; r < warp * 8 + 8; ++r) {
#pragma unroll
      for (int hb = 0; hb < 2; ++hb) {
        const float s = Sc[r][lane + 32 * hb];
        const int id = (int)(col0 + lane + 32 * hb);
        const float thr = L.v[r * kTopkMax + k - 1];
        const int thr_i = L.i[r * kTopkMax + k - 1];
        unsigned pass = __ballot_sync(0xffffffffu, s > -INFINITY && better(s, id, thr, thr_i));
        while (pass) {
          const int b = __ffs(pass) - 1;
          pass &= pass - 1;
          topk_insert(L, r, k, __shfl_sync(0xffffffffu, s, b), __shfl_sync(0xffffffffu, id, b), lane);
        }
      }
    }
    // (the next tile's first __syncthreads orders these list updates before Sc is overwritten)
  }
  __syncthreads();

  const int splits = gridDim.y;
  if (splits == 1) {
    for (int j = t; j < TM * k; j += kTkThreads) {
      const int r = j / k, c = j - r * k;
      if (row0 + r < n) {
        const int id = L.i[r * kTopkMax + c];
        idx[(row0 + r) * k + c] = id == 0x7fffffff ? -1 : id;
        if (val) val[(row0 + r) * k + c] = L.v[r * kTopkMax + c];
      }
    }
    return;
  }
  // publish the partial lists, take a ticket; the last CTA of this query tile merges them
  for (int j = t; j < TM * k; j += kTkThreads) {
    const int r = j / k, c = j - r * k;
    const int64_t o = (((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * TM + r) * k + c;
    scratch_v[o] = L.v[r * kTopkMax + c];
    scratch_i[o] = L.i[r * kTopkMax + c];
  }
  __threadfence();
  __syncthreads();
  if (t == 0) last_flag = (atomicAdd(&tickets[blockIdx.x], 1u) == (unsigned)(splits - 1)) ? 1u : 0u;
  __syncthreads();
  if (!last_flag) return;
  __threadfence();
  for (int sp = 0; sp < splits; ++sp) {
    if (sp == (int)blockIdx.y) continue;  // our own partial lists are already in smem
    for (int r = warp * 8; r < warp * 8 + 8; ++r) {
      const int64_t o = (((int64_t)sp * gridDim.x + blockIdx.x) * TM + r) * k;
      for (int c = 0; c < k; ++c) {
        const float s = __ldcg(scratch_v + o + c);
        const int id = __ldcg(scratch_i + o + c);
        if (id == 0x7fffffff) break;  // sorted: the rest of this partial list is empty
        if (!better(s, id, L.v[r * kTopkMax + k - 1], L.i[r * kTopkMax + k - 1])) break;  // sorted: nothing better follows
        topk_insert(L, r, k, s, id, lane);
      }
    }
  }
  __syncthreads();
  for (int j = t; j < TM * k; j += kTkThreads) {
    const int r = j / k, c = j - r * k;
    if (row0 + r < n) {
      const int id = L.i[r * kTopkMax + c];
      idx[(row0 + r) * k + c] = id == 0x7fffffff ? -1 : id;
      if (val) val[(row0 + r) * k + c] = L.v[r * kTopkMax + c];
    }
  }
}


// ---- similarity on the tensor cores ------------------------------------------------------------------------------
// scale * norm(a) . norm(b)^T as ONE wgmma GEMM with fp32-class accuracy: every embedding row is scaled by a power
// of two to max|x| in [32, 64) and split into fp16 hi + lo (22 significand bits, every fp16 x fp16 product exact in the
// fp32 accumulator); with A' = [hi | lo | hi] and B' = [hi | hi | lo] (K = 3 x 512) the GEMM sums hi.hi + lo.hi + hi.lo
// (the dropped lo.lo term is 2^-22 relative).  Row / column scale vectors undo the powers of two and carry logit_scale
// and the optional 1/|x|; they are applied by the GEMM's EPI_SIM_F32 epilogue.  Error vs fp64: ~1e-6 relative, i.e.
// |dlogits| ~1e-4 at scale 100 — the fp32 SIMT kernel above stays as the fallback for outputs whose leading dimension
// cannot take the 128-column padding.  [125000 x 10000] (cfg5, one rank): 1.28 TFLOP of fp32 FMAs -> 3.9 TFLOP of MMAs.
constexpr int kSplitK = 3 * kProj;

__global__ void __launch_bounds__(256)
split_embed_kernel(const float* __restrict__ x, int64_t n, int64_t n_pad, int normalize, int role_b, float scale,
                   __half* __restrict__ out, float* __restrict__ vec_scale) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n_pad; r += nwarps) {
    __half* o = out + r * kSplitK;
    if (r >= n) {  // padding rows of the B operand: zeros, unit scale
      for (int j = lane; j < kSplitK / 8; j += 32) reinterpret_cast<uint4*>(o)[j] = make_uint4(0u, 0u, 0u, 0u);
      if (lane == 0) vec_scale[r] = 0.f;
      continue;
    }
    const float4* xr = reinterpret_cast<const float4*>(x + r * kProj);
    float4 v[kProj / 128];
    float ss = 0.f, mx = 0.f;
#pragma unroll
    for (int j = 0; j < kProj / 128; ++j) {
      v[j] = __ldg(xr + lane + 32 * j);
      ss += (v[j].x * v[j].x + v[j].y * v[j].y) + (v[j].z * v[j].z + v[j].w * v[j].w);
      mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v[j].x), fabsf(v[j].y))), fmaxf(fabsf(v[j].z), fabsf(v[j].w)));
    }
    ss = warp_sum(ss);
    mx = warp_max(mx);
    // power of two that brings max|x| into [32, 64): exact scaling, no fp16 subnormals in the lo parts that matter
    int e = 0;
    frexpf(mx, &e);                                   // mx = m * 2^e, m in [0.5, 1)
    const float p2 = (mx > 0.f) ? exp2f((float)(6 - e)) : 1.0f;
    const float undo = 1.0f / p2;                     // exact
    if (lane == 0) vec_scale[r] = undo * (normalize ? rsqrtf(ss) : 1.0f) * scale;
#pragma unroll
    for (int j = 0; j < kProj / 128; ++j) {
      const float f[4] = {v[j].x * p2, v[j].y * p2, v[j].z * p2, v[j].w * p2};
      __half hi[4], lo[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        hi[q] = __float2half_rn(f[q]);
        lo[q] = __float2half_rn(f[q] - __half2float(hi[q]));
      }
      const uint2 uh = make_uint2(*reinterpret_cast<uint32_t*>(&hi[0]), *reinterpret_cast<uint32_t*>(&hi[2]));
      const uint2 ul = make_uint2(*reinterpret_cast<uint32_t*>(&lo[0]), *reinterpret_cast<uint32_t*>(&lo[2]));
      const int c = lane + 32 * j;                    // 4-element group inside the 512-wide block
      reinterpret_cast<uint2*>(o)[c] = uh;                                  // block 0: hi
      reinterpret_cast<uint2*>(o + kProj)[c] = role_b ? uh : ul;            // block 1: A lo / B hi
      reinterpret_cast<uint2*>(o + 2 * kProj)[c] = role_b ? ul : uh;        // block 2: A hi / B lo
    }
  }
}

// Grow-only per-device scratch: these entry points have no engine handle to hang a workspace on, and nothing is
// allocated once the buffers are warm.  A lease holds its slot's lock for the whole call, so concurrent calls on
// different streams take turns; the stream waits for the previous user's kernels, and the lease records the slot's
// event for the next one when it ends.  Each pool has its own lock, so one lease may enclose a lease of another pool.
struct ScratchSlot {
  std::mutex mu;
  void* p = nullptr;
  size_t bytes = 0;
  cudaEvent_t ev = nullptr;
};
using ScratchPool = ScratchSlot[64];

class ScratchLease {
 public:
  ScratchLease(ScratchPool& pool, cudaStream_t st) : st_(st) {
    int dev = 0;
    cudaGetDevice(&dev);
    slot_ = &pool[dev & 63];
    slot_->mu.lock();
  }
  ~ScratchLease() {
    if (acquired_) cudaEventRecord(slot_->ev, st_);
    slot_->mu.unlock();
  }
  ScratchLease(const ScratchLease&) = delete;
  ScratchLease& operator=(const ScratchLease&) = delete;

  // At least `bytes` of scratch at *out; a buffer that is too small is replaced (by one 1.5x as large with `slack`)
  // once its last user has finished.
  int acquire(size_t bytes, void** out, bool slack = false) {
    ScratchSlot& s = *slot_;
    if (!s.ev) PLIP_CUDA_CHECK(cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming));
    if (s.bytes < bytes) {
      if (s.p) {
        PLIP_CUDA_CHECK(cudaEventSynchronize(s.ev));
        PLIP_CUDA_CHECK(cudaFree(s.p));
        s.p = nullptr; s.bytes = 0;
      }
      const size_t want = slack ? bytes + bytes / 2 : bytes;
      PLIP_CUDA_CHECK(cudaMalloc(&s.p, want));
      s.bytes = want;
    }
    PLIP_CUDA_CHECK(cudaStreamWaitEvent(st_, s.ev, 0));
    acquired_ = true;
    *out = s.p;
    return 0;
  }

 private:
  ScratchSlot* slot_ = nullptr;
  cudaStream_t st_;
  bool acquired_ = false;
};

ScratchPool g_sim_pool, g_topk_tc_pool, g_topk_tiled_pool;

constexpr int64_t kSimRowChunk = 131072;  // A rows split + multiplied per pass (403 MB of fp16 operand scratch)

int launch_similarity_tc(const float* a, int64_t n, const float* b, int64_t m, float scale, bool norm_a, bool norm_b,
                         float* out, int64_t ldo, cudaStream_t st) {
  const int64_t m_pad = (m + 127) / 128 * 128;
  const int64_t rows = n < kSimRowChunk ? n : kSimRowChunk;
  const size_t bytes_b = (size_t)m_pad * kSplitK * 2, bytes_a = (size_t)rows * kSplitK * 2;
  ScratchLease lease(g_sim_pool, st);
  void* scratch = nullptr;
  if (int rc = lease.acquire(bytes_b + bytes_a + (size_t)(m_pad + rows) * 4 + 1024, &scratch)) return rc;
  uint8_t* base = static_cast<uint8_t*>(scratch);
  __half* bsplit = reinterpret_cast<__half*>(base);
  __half* asplit = reinterpret_cast<__half*>(base + bytes_b);
  float* cscale = reinterpret_cast<float*>(base + bytes_b + bytes_a);
  float* rscale = cscale + m_pad;
  const int64_t row_grid_cap = 8LL * sm_count();
  auto grid_for_rows = [row_grid_cap](int64_t r) { int64_t g = (r + 7) / 8; return (int)(g < 1 ? 1 : (g > row_grid_cap ? row_grid_cap : g)); };
  PLIP_CUDA_CHECK(launch_kernel(split_embed_kernel, dim3(grid_for_rows(m_pad)), dim3(256), 0, st, 1, b, m, m_pad,
                                norm_b ? 1 : 0, 1, 1.0f, bsplit, cscale));
  for (int64_t i = 0; i < n; i += rows) {
    const int64_t cnt = n - i < rows ? n - i : rows;
    PLIP_CUDA_CHECK(launch_kernel(split_embed_kernel, dim3(grid_for_rows(cnt)), dim3(256), 0, st, 1, a + i * kProj, cnt, cnt,
                                  norm_a ? 1 : 0, 0, scale, asplit, rscale));
    GemmArgs g;
    g.f16 = 1;
    g.A = reinterpret_cast<const __nv_bfloat16*>(asplit); g.lda = kSplitK;
    g.W = reinterpret_cast<const __nv_bfloat16*>(bsplit); g.ldw = kSplitK;
    g.M = (int)cnt; g.N = (int)m_pad; g.K = kSplitK;
    g.bias = cscale; g.rowscale = rscale;
    g.out = out + i * ldo; g.ldo = (int)ldo; g.epi = EPI_SIM_F32;
    if (int rc = launch_gemm(g, st)) return rc;
  }
  return 0;
}


// ---- top-k on the tensor cores: score chunks from the split-fp16 GEMM, folded row by row ---------------------------
// For big retrieval problems (cfg5: 10,000 queries x 125,000 gallery rows per rank) the fused fp32 SIMT kernel above
// spends its time on FMAs (1.28 TFLOP -> ~88 ms).  Here the scores of all queries against a CHUNK of the space come
// from launch_similarity_tc (0.5 ms per 16 k columns) into a scratch block, and one warp per query folds its row
// into the query's running sorted top-k list (global memory, k <= 64): every lane tests 4 scores per iteration against
// the current k-th best, survivors are inserted with the same warp-cooperative topk_insert — ~k ln(m / k) insertions
// per row in total, so the pass is a streaming read of the chunk.  Ordering: score, then lower index (deterministic).
constexpr int kMergeWarps = 8;

__global__ void __launch_bounds__(kMergeWarps * 32)
rowwise_topk_merge_kernel(const float* __restrict__ S, int64_t n, int64_t cols, int64_t ld, int64_t col0, int k,
                          int first, int32_t* __restrict__ idx, float* __restrict__ val) {
  __shared__ float lv[kMergeWarps][kTopkMax];
  __shared__ int li[kMergeWarps][kTopkMax];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kMergeWarps + warp;
  if (row >= n) return;
  TopkLists L;
  L.v = &lv[0][0];
  L.i = &li[0][0];
  for (int j = lane; j < kTopkMax; j += 32) {
    const bool have = !first && j < k;
    const int id = have ? idx[row * k + j] : -1;
    lv[warp][j] = (have && id >= 0) ? val[row * k + j] : -INFINITY;
    li[warp][j] = (have && id >= 0) ? id : 0x7fffffff;
  }
  __syncwarp();
  const float* sr = S + row * ld;
  for (int64_t c0 = 0; c0 < cols; c0 += 128) {
    const int64_t c = c0 + lane * 4;
    float4 v = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    if (c + 3 < cols) v = __ldg(reinterpret_cast<const float4*>(sr + c));
    else {
      if (c < cols) v.x = sr[c];
      if (c + 1 < cols) v.y = sr[c + 1];
      if (c + 2 < cols) v.z = sr[c + 2];
    }
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float s = vv[q];
      const int id = (int)(col0 + c + q);
      const float thr = lv[warp][k - 1];
      const int thr_i = li[warp][k - 1];
      unsigned pass = __ballot_sync(0xffffffffu, s > -INFINITY && better(s, id, thr, thr_i));
      while (pass) {
        const int b = __ffs(pass) - 1;
        pass &= pass - 1;
        topk_insert(L, warp, k, __shfl_sync(0xffffffffu, s, b), __shfl_sync(0xffffffffu, id, b), lane);
      }
    }
  }
  __syncwarp();
  for (int j = lane; j < k; j += 32) {
    const int id = li[warp][j];
    idx[row * k + j] = id == 0x7fffffff ? -1 : id;
    val[row * k + j] = lv[warp][j];
  }
}

int launch_similarity_topk_tc(const float* q, int64_t n, const float* s, int64_t m, float scale, bool norm_q,
                              bool norm_s, int k, int32_t* idx, float* val, cudaStream_t st) {
  // chunk of the space: <= 256 MB of fp32 scores for all n queries, a multiple of 256 columns
  int64_t gc = ((int64_t)256 << 20) / (4 * n) / 256 * 256;
  if (gc < 256) gc = 256;
  if (gc > 32768) gc = 32768;
  if (gc > (m + 255) / 256 * 256) gc = (m + 255) / 256 * 256;
  const size_t score_bytes = (size_t)n * gc * 4, val_bytes = val ? 0 : (size_t)n * k * 4;
  ScratchLease lease(g_topk_tc_pool, st);
  void* scratch = nullptr;
  if (int rc = lease.acquire(score_bytes + val_bytes + 256, &scratch)) return rc;
  float* scores = static_cast<float*>(scratch);
  float* vals = val ? val : reinterpret_cast<float*>(static_cast<uint8_t*>(scratch) + score_bytes);
  const unsigned grid = (unsigned)((n + kMergeWarps - 1) / kMergeWarps);
  for (int64_t c0 = 0; c0 < m; c0 += gc) {
    const int64_t cols = m - c0 < gc ? m - c0 : gc;
    if (int rc = launch_similarity_tc(q, n, s + c0 * kProj, cols, scale, norm_q, norm_s, scores, gc, st)) return rc;
    PLIP_CUDA_CHECK(launch_kernel(rowwise_topk_merge_kernel, dim3(grid), dim3(kMergeWarps * 32), 0, st, 1, scores, n, cols,
                                  gc, c0, k, c0 == 0 ? 1 : 0, idx, vals));
  }
  return 0;
}

}  // namespace

int launch_similarity(const float* a, int64_t n, const float* b, int64_t m, float scale, bool norm_a, bool norm_b,
                      float* out, int64_t ldo, cudaStream_t st) {
  PLIP_REQUIRE(n > 0 && m > 0, "similarity: empty operand n=%lld m=%lld", (long long)n, (long long)m);
  PLIP_REQUIRE(ldo >= m, "similarity: ld_logits %lld < m %lld", (long long)ldo, (long long)m);
  PLIP_REQUIRE((reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(b) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(out) & 15) == 0, "similarity: operands must be 16-byte aligned");
  // Tensor-core path for wide score matrices (>= 256 columns) whenever the output rows can take the 128-column
  // padding of the GEMM tile (plip_b200's own callers allocate ld_logits that way) and the GEMM's row stride
  // (a multiple of 8 floats).
  const int64_t m_pad = (m + 127) / 128 * 128;
  // (the choice depends on m only, so a row-sharded call computes bit-identical rows to the unsharded one)
  if (m >= 256 && ldo >= m_pad && ldo % 8 == 0 && ldo < 0x7fffffff)
    return launch_similarity_tc(a, n, b, m, scale, norm_a, norm_b, out, ldo, st);
  const int64_t gy = (n + TM - 1) / TM, gx = (m + TN - 1) / TN;
  PLIP_REQUIRE(gy <= 65535, "similarity: n=%lld too large for one launch (chunk rows)", (long long)n);
  dim3 grid((unsigned)gx, (unsigned)gy);
  PLIP_CUDA_CHECK(launch_kernel(similarity_kernel, grid, dim3(kSimThreads), 0, st, 1, a, n, b, m, (int)kProj, scale,
                             norm_a ? 1 : 0, norm_b ? 1 : 0, out, ldo));
  return 0;
}

int launch_similarity_topk(const float* q, int64_t n, const float* s, int64_t m, float scale, bool norm_q,
                           bool norm_s, int k, int32_t* idx, float* val, cudaStream_t st) {
  PLIP_REQUIRE(n > 0 && m > 0, "similarity_topk: empty operand");
  PLIP_REQUIRE(k >= 1 && k <= kTopkMax, "similarity_topk: k=%d out of range [1,%d]", k, kTopkMax);
  PLIP_REQUIRE(n <= 0x7fffffff && m <= 0x7fffffff, "similarity_topk: operand too large");
  if (n >= 256 && m >= 8192)  // big retrieval problems: scores from the tensor cores, chunk by chunk
    return launch_similarity_topk_tc(q, n, s, m, scale, norm_q, norm_s, k, idx, val, st);
  if (n * m < (int64_t)1 << 16) {
    // tiny problems (e.g. a handful of class prompts): one CTA per query streaming the space
    PLIP_CUDA_CHECK(launch_kernel(similarity_topk_kernel, dim3((unsigned)n), dim3(kTopkThreads), 0, st, 1, q, n, s, m,
                               (int)kProj, scale, norm_q ? 1 : 0, norm_s ? 1 : 0, k, idx, val));
    return 0;
  }
  static unsigned long long configured = 0;
  const size_t smem = (size_t)(kTkSmemFloats + TM * kTopkMax) * 4;
  if (first_use_on_device(configured)) {
    PLIP_CUDA_CHECK(cudaFuncSetAttribute(similarity_topk_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
  }
  const int64_t row_tiles = (n + TM - 1) / TM, space_tiles = (m + TN - 1) / TN;
  PLIP_REQUIRE(row_tiles <= 0x7fffffff, "similarity_topk: too many queries");
  int64_t splits = (2 * sm_count() + row_tiles - 1) / row_tiles;  // aim at ~2 CTAs per SM
  if (splits > space_tiles) splits = space_tiles;
  if (splits > 64) splits = 64;
  if (splits < 1) splits = 1;
  const int tiles_per_split = (int)((space_tiles + splits - 1) / splits);
  splits = (space_tiles + tiles_per_split - 1) / tiles_per_split;
  float* scratch_v = nullptr;
  int* scratch_i = nullptr;
  unsigned* tickets = nullptr;
  ScratchLease lease(g_topk_tiled_pool, st);
  if (splits > 1) {  // partial lists of the space splits + one merge ticket per query tile
    const size_t ent = (size_t)splits * row_tiles * TM * k;
    void* scratch = nullptr;
    if (int rc = lease.acquire(ent * 8 + (size_t)row_tiles * 4, &scratch, true)) return rc;
    scratch_v = static_cast<float*>(scratch);
    scratch_i = reinterpret_cast<int*>(scratch_v + ent);
    tickets = reinterpret_cast<unsigned*>(scratch_i + ent);
    PLIP_CUDA_CHECK(cudaMemsetAsync(tickets, 0, (size_t)row_tiles * 4, st));
  }
  dim3 grid((unsigned)row_tiles, (unsigned)splits);
  PLIP_CUDA_CHECK(launch_kernel(similarity_topk_tiled_kernel, grid, dim3(kTkThreads), smem, st, 1, q, n, s, m, (int)kProj,
                             scale, norm_q ? 1 : 0, norm_s ? 1 : 0, k, tiles_per_split, scratch_v, scratch_i, tickets,
                             idx, val));
  return 0;
}

}  // namespace plip

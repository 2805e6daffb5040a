// plip_b200 — shared device/host helpers for the sm_90a kernels.
//
// Thin inline-PTX wrappers for the Hopper primitives the engine uses: mbarrier, TMA (cp.async.bulk.tensor),
// cluster addressing.  The warpgroup MMA wrappers live in wgmma.cuh.  No CUTLASS/CuTe dependency.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

namespace plip {

// ---------------------------------------------------------------------------
// Model constants (CLIP ViT-B/32 == PLIP; TF:configuration_clip.py:47-64,97-109)
// ---------------------------------------------------------------------------
constexpr int kImage = 224;
constexpr int kPatch = 32;
constexpr int kGrid = 7;           // 224 / 32
constexpr int kPatches = 49;
constexpr int kVisSeq = 50;        // 49 patches + class token
// Inputs other than 224 x 224 (interpolated position table): patch grid gh x gw up to kMaxGrid per side.
constexpr int kMaxGrid = 32;       // 1024 pixels
constexpr int kMaxVisSeq = kMaxGrid * kMaxGrid + 1;
constexpr int kVisDim = 768;
constexpr int kVisHeads = 12;
constexpr int kVisFF = 3072;
constexpr int kPatchK = 3072;      // 3 * 32 * 32
// CLIP ViT-B/16: the same towers behind a 16-pixel patch.  An engine's patch size (32 or 16) comes from its weights;
// the k* constants above are the ViT-B/32 geometry, these give any accepted patch size's.
constexpr int kPatch16 = 16;
constexpr int vis_grid(int patch) { return kImage / patch; }                      // 7 or 14 patches per side at 224
constexpr int vis_seq(int patch) { return vis_grid(patch) * vis_grid(patch) + 1; }  // 50 or 197 tokens at 224
constexpr int patch_k(int patch) { return 3 * patch * patch; }                    // 3072 or 768
constexpr int kTxtSeq = 77;
constexpr int kTxtDim = 512;
constexpr int kTxtHeads = 8;
constexpr int kTxtFF = 2048;
constexpr int kVocab = 49408;
constexpr int kLayers = 12;
constexpr int kHeadDim = 64;
constexpr int kProj = 512;
constexpr float kLnEps = 1e-5f;

// ---------------------------------------------------------------------------
// Host-side error plumbing: C-ABI functions return int, never throw.
// ---------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);

#define PLIP_CUDA_CHECK(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::plip::set_last_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,      \
                             cudaGetErrorString(_e));                                \
      return -1;                                                                     \
    }                                                                                \
  } while (0)

#define PLIP_REQUIRE(cond, ...)                                                      \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      ::plip::set_last_error(__VA_ARGS__);                                           \
      return -2;                                                                     \
    }                                                                                \
  } while (0)

// Kernels enqueued for execution since load (plip_launch_count): launch_kernel counts each launch, a stream capture
// takes back the kernels it recorded (nothing runs), and a graph replay adds its kernel nodes.
inline std::atomic<unsigned long long> g_launch_count{0};

// cudaFuncSetAttribute is per device: returns true the first time it is called for the current device with
// a given per-kernel mask (a process that drives several GPUs configures each kernel once per GPU).
inline bool first_use_on_device(unsigned long long& mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (mask & bit) return false;
  mask |= bit;
  return true;
}

// SMs of the current device (grid caps of the streaming kernels).
inline int sm_count() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

// Encode a 2-D bf16 row-major tensor map with 128-byte swizzle.
// dims: inner (contiguous) extent `cols`, outer extent `rows`, row stride in bytes.
// box: box_cols (must be 64 bf16 == 128 B for SWIZZLE_128B) x box_rows (<=256).
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols);
// Encode a 3-D bf16 tensor map [mats][rows][cols] with 128-byte swizzle and a {box_cols, box_rows, 1} box: a box
// that reaches past `rows` is zero-filled on load and clipped on store inside its own matrix, never spilling into the
// next one.
int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t mats, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint64_t mat_stride_bytes, uint32_t box_rows, uint32_t box_cols);

#ifdef __CUDACC__

// ---------------------------------------------------------------------------
// Kernel launch helper (cluster dimension as a launch attribute); counts the launch in g_launch_count.
// ---------------------------------------------------------------------------
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                 unsigned cluster_x, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (cluster_x > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster_x;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  const cudaError_t err = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  if (err == cudaSuccess) g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return err;
}

// ---------------------------------------------------------------------------
// Small device utilities
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// Map a CTA-local shared address to the same offset in CTA `rank` of the cluster.
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}

// ---------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
// Arrive on a barrier that may live in another CTA of the cluster (shared::cluster address).
// Plain (CTA-scope release) form: the signals sent this way only order wgmma reads against TMA writes of an
// operand slot, and a .release.cluster arrive would drain every outstanding global store of the thread.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Blocking wait with a watchdog: a protocol bug traps (launch error on the host) instead of hanging the GPU.
// ~2^31 cycles (> 1 s) is far beyond any legal wait.  No printf here: a function call inside a kernel that issues
// wgmma makes ptxas serialise every wgmma.mma_async (warning C7510).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ff) == 0 && clock64() - t0 > (1ll << 31)) __trap();
  }
}

// ---------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// Pull a 2-D tile into L2 only (no smem destination, no completion signal).
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* tm, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(tm)),
               "r"(c0), "r"(c1)
               : "memory");
}

__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float2 v) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}

// 2-D tile load, completion on an mbarrier of the executing CTA.
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* tm, uint32_t bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// 2-D tile load, multicast: the tile lands at the same shared-memory offset of every CTA in `cta_mask` (cluster
// ranks), and each destination CTA's barrier at `bar`'s offset is credited with the bytes.
__device__ __forceinline__ void tma_load_2d_mc(uint32_t smem_dst, const CUtensorMap* tm, uint32_t bar, int32_t c0,
                                               int32_t c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}

// 2-D tile store smem -> global (bulk async group); rows / columns outside the tensor are clipped.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, uint32_t smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tm)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
// 3-D tile load / store (make_tmap_bf16_3d maps): c0 column, c1 row inside matrix c2.
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const CUtensorMap* tm, uint32_t bar, int32_t c0,
                                            int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, uint32_t smem_src, int32_t c0, int32_t c1,
                                             int32_t c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tm)),
               "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// Barrier over THREADS threads of the CTA (a warpgroup), ID 1..15 (0 is __syncthreads).
template <int ID, int THREADS>
__device__ __forceinline__ void named_barrier_sync() {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(THREADS) : "memory");
}
// The same with a run-time ID, and its non-waiting half: bar.arrive counts the calling warps towards the THREADS of
// barrier ID and returns at once; the threads that complete the count with bar.sync wait for it.
template <int THREADS>
__device__ __forceinline__ void named_barrier_sync(uint32_t id) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(THREADS) : "memory");
}
template <int THREADS>
__device__ __forceinline__ void named_barrier_arrive(uint32_t id) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "n"(THREADS) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed store groups have finished READING their shared-memory source
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// all committed store groups but the most recent one have finished reading their shared-memory source
__device__ __forceinline__ void tma_store_wait_read_but_one() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
// all committed store groups are complete (global writes performed)
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------
// Packing / math
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
// two fp32 -> one 32-bit word of the engine's 16-bit operand format
template <bool F16>
__device__ __forceinline__ uint32_t pack_op2(float lo, float hi) {
  if constexpr (F16) return pack_f16x2(lo, hi);
  else return pack_bf16x2(lo, hi);
}
__device__ __forceinline__ uint32_t pack_op2_rt(float lo, float hi, int f16) {  // memory-bound kernels: runtime format
  return f16 ? pack_f16x2(lo, hi) : pack_bf16x2(lo, hi);
}
// QuickGELU: x * sigmoid(1.702 x)   (TF:activations.py:117-123)
// sigmoid(y) = 0.5 * (1 + tanh(y / 2)): one MUFU op (tanh.approx.f32, max rel. error 2^-11) instead of
// ex2 + rcp; the absolute error (<= 2.5e-4 |x|) is ~10x below the bf16 rounding of the result.
__device__ __forceinline__ float quick_gelu(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.851f * x));
  const float h = 0.5f * x;
  return fmaf(h, t, h);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

#endif  // __CUDACC__

}  // namespace plip

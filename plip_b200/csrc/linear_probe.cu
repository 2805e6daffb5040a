// plip_b200 — the reference's linear probe on the device: scikit-learn's SGD logistic regression
// (SGDClassifier(loss="log_loss", penalty="l2", learning_rate="optimal"), sklearn 1.9 _plain_sgd, 32-bit
// instantiation), every one-vs-rest problem of a fit and every alpha of a sweep at once, plus the linear decision.
//
// sgd_fit_kernel: one warp per binary problem, all epochs on the device.  A problem is one dependent chain of n
// sample steps per epoch (each step's update feeds the next step's dot product), so the kernel is bound by the latency
// of that chain, not by HBM or the tensor cores: one warp per problem, one problem per block so that problems spread
// over SMs.  Per step the warp
//   - reads row x of X from a shared-memory ring that cp.async fills kRing samples ahead along the epoch order (the
//     order and the class ids are loaded a 32-sample chunk or two ahead), so no global-memory latency is on the chain;
//   - reduces w.x and sum(w^2) in one warp-shuffle pass (the objective needs |w|^2 of the previous add; sklearn's add
//     recomputes it right away, here it is taken at the start of the next step, from the same weights);
//   - runs sklearn's scalar step in fp64, lane-uniform (every lane holds the bit-identical reduced sums: a butterfly
//     reduction adds the same two values in every lane);
//   - applies scale / add to its D / 32 weights (lane l holds elements 4 * (l + 32 k) .. + 3, k = 0..D/128-1) with
//     sklearn's casts: scale takes a float, add takes a float coefficient and divides it by a float copy of wscale.
// Both kernels are instantiated for the two embedding widths the reference probes, D = 512 (CLIP) and D = 1024
// (MuDiPath's DenseNet-121); at 1024 the cp.async ring holds 8 x 4 KB rows, 32 KB of static shared memory.
// The weights never leave registers until the problem stops.  At the end of an epoch the warp gathers the next order
// through sigma into its own buffer, checks for non-finite values and runs the stop test itself.
//
// Every multiply that feeds an add is written with __dmul_rn / __fmul_rn: nvcc would otherwise contract it into an
// FMA, which sklearn's C code (x86-64, no FMA) does not do.
#include "kernels.cuh"

#include <math.h>

#include <vector>

namespace plip {

namespace {

// The embedding widths a fit runs at: 512 (the CLIP projection) and 1024 (MuDiPath's DenseNet-121 features).
constexpr int kSgdDimClip = kProj;
constexpr int kSgdDimDenseNet = 1024;
constexpr int kRing = 8;                      // rows in flight per problem
constexpr double kResetWscale = 1e-6;         // WeightVector32
constexpr double kMaxDloss = 1e12;
constexpr unsigned kFull = 0xffffffffu;

struct SgdProblem {
  double alpha;
  double optimal_init;   // computed on the host with the C library's exp, as sklearn does in Python
  float weight_pos;
  float weight_neg;
  int32_t pos_class;
  int32_t sigma_index;
};
static_assert(sizeof(SgdProblem) == 32, "SgdProblem layout");

__device__ __forceinline__ void cp_async_16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// CyHalfBinomialLoss (sklearn/_loss/_loss.pyx.tp: log1pexp, closs / cgradient_half_binomial).
__device__ __forceinline__ double log1pexp(double x) {
  if (x <= -37) return exp(x);
  if (x <= -2) return log1p(exp(x));
  if (x <= 18) return log(__dadd_rn(1.0, exp(x)));
  if (x <= 33.3) return __dadd_rn(x, exp(-x));
  return x;
}
__device__ __forceinline__ double half_binomial_loss(double y, double p) {
  return __dsub_rn(log1pexp(p), __dmul_rn(y, p));
}
__device__ __forceinline__ double half_binomial_gradient(double y, double p) {
  if (p > -37) {
    const double e = exp(-p);
    return __dsub_rn(__dsub_rn(1.0, y), __dmul_rn(y, e)) / __dadd_rn(1.0, e);
  }
  return __dsub_rn(exp(p), y);
}

__device__ __forceinline__ float& comp(float4& v, int c) { return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w; }

template <int D>
__global__ void __launch_bounds__(32) sgd_fit_kernel(const float* __restrict__ X, int n, const int32_t* __restrict__ cls,
                                                    const SgdProblem* __restrict__ problems,
                                                    const int32_t* __restrict__ sigma, int32_t* orders, int max_iter,
                                                    double tol, int n_iter_no_change, float* __restrict__ coef,
                                                    double* __restrict__ intercept_out, int32_t* __restrict__ n_iter_out,
                                                    int32_t* __restrict__ overflow_out) {
  constexpr int kSgdVec = D / (32 * 4);  // float4 per lane
  __shared__ __align__(16) float4 ring[kRing][D / 4];
  const int lane = threadIdx.x;
  const int pid = blockIdx.x;
  const SgdProblem pr = problems[pid];
  const int32_t* sig = sigma + (size_t)pr.sigma_index * n;
  int32_t* own = orders + (size_t)pid * 2 * n;  // two epoch orders, used in turn
  const float4* X4 = reinterpret_cast<const float4*>(X);

  float4 w[kSgdVec];
#pragma unroll
  for (int j = 0; j < kSgdVec; ++j) w[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  double wscale = 1.0, sq_norm = 0.0, intercept = 0.0, t = 1.0;
  bool sq_pending = false;  // the last step added to w: sq_norm = sum(w^2) * sq_factor at the next step
  float sq_factor = 1.f;
  double best = INFINITY;
  int no_improvement = 0, iters = max_iter;
  bool overflow = false;
  const int32_t* ord = sig;  // epoch 0 applies sigma to the identity

  for (int epoch = 0; epoch < max_iter; ++epoch) {
    if (epoch > 0) {  // order_e[i] = order_{e-1}[sigma[i]]
      int32_t* dst = own + (epoch & 1) * (size_t)n;
      constexpr int kU = 8;
      for (int base = 0; base < n; base += 32 * kU) {
        int32_t v[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int i = base + u * 32 + lane;
          v[u] = i < n ? sig[i] : 0;
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) v[u] = ord[v[u]];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int i = base + u * 32 + lane;
          if (i < n) dst[i] = v[u];
        }
      }
      __syncwarp();
      ord = dst;
    }
    // order / class id registers: chunk c (samples 32c..32c+31) of the current step, chunk c+1, and the order of c+2
    auto order_at = [&](int i) { return i < n ? ord[i] : 0; };
    int a_idx = order_at(lane), b_idx = order_at(32 + lane), c_idx = order_at(64 + lane);
    int a_cls = cls[a_idx], b_cls = cls[b_idx];
    auto issue = [&](int s, int k) {  // prefetch the row of sample s into its ring slot (an empty group past the end)
      const int v = ((s >> 5) == (k >> 5)) ? a_idx : b_idx;
      const int row = __shfl_sync(kFull, v, s & 31);
      if (s < n) {
        float4* slot = ring[s % kRing];
#pragma unroll
        for (int j = 0; j < kSgdVec; ++j) cp_async_16(slot + lane + 32 * j, X4 + (size_t)row * (D / 4) + lane + 32 * j);
      }
      cp_async_commit();
    };
#pragma unroll
    for (int s = 0; s < kRing; ++s) issue(s, 0);

    double objective = 0.0;
    for (int k = 0; k < n; ++k) {
      if ((k & 31) == 0 && k > 0) {
        a_idx = b_idx;
        a_cls = b_cls;
        b_idx = c_idx;
        b_cls = cls[b_idx];
        c_idx = order_at(k + 64 + lane);
      }
      const float y = __shfl_sync(kFull, a_cls, k & 31) == pr.pos_class ? 1.f : 0.f;
      cp_async_wait<kRing - 1>();  // this lane's copies of sample k have landed (each lane reads only its own)
      float4 x[kSgdVec];
      const float4* slot = ring[k % kRing];
#pragma unroll
      for (int j = 0; j < kSgdVec; ++j) x[j] = slot[lane + 32 * j];

      double dot = 0.0, sq = 0.0;
#pragma unroll
      for (int j = 0; j < kSgdVec; ++j)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          dot = __dadd_rn(dot, (double)__fmul_rn(comp(w[j], c), comp(x[j], c)));
          sq = __dadd_rn(sq, (double)__fmul_rn(comp(w[j], c), comp(w[j], c)));
        }
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        dot = __dadd_rn(dot, __shfl_xor_sync(kFull, dot, m));
        sq = __dadd_rn(sq, __shfl_xor_sync(kFull, sq, m));
      }
      issue(k + kRing, k);  // the slot's row is in registers now

      if (sq_pending) sq_norm = __dmul_rn(sq, (double)sq_factor);
      sq_pending = false;
      const double yd = (double)y;
      const double p = __dadd_rn((double)__double2float_rn(__dmul_rn(dot, wscale)), intercept);
      const double eta = 1.0 / __dmul_rn(pr.alpha, __dsub_rn(__dadd_rn(pr.optimal_init, t), 1.0));
      objective = __dadd_rn(objective, half_binomial_loss(yd, p));
      const float norm = __double2float_rn(sqrt(sq_norm));
      objective = __dadd_rn(objective, __dmul_rn(__dmul_rn(0.5, (double)__fmul_rn(norm, norm)), pr.alpha));
      const double dloss = fmin(fmax(half_binomial_gradient(yd, p), -kMaxDloss), kMaxDloss);
      const double update = __dmul_rn(__dmul_rn(-eta, dloss), (double)(y > 0.f ? pr.weight_pos : pr.weight_neg));

      const float c = __double2float_rn(fmax(0.0, __dsub_rn(1.0, __dmul_rn(eta, pr.alpha))));  // w.scale
      wscale = __dmul_rn(wscale, (double)c);
      sq_norm = __dmul_rn(sq_norm, (double)__fmul_rn(c, c));
      if (wscale < kResetWscale) {
        const float s = __double2float_rn(wscale);
#pragma unroll
        for (int j = 0; j < kSgdVec; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) comp(w[j], q) = __fmul_rn(comp(w[j], q), s);
        wscale = 1.0;
      }
      if (update != 0.0) {  // w.add
        const float wsf = __double2float_rn(wscale);
        const double coeff = (double)__fdiv_rn(__double2float_rn(update), wsf);
#pragma unroll
        for (int j = 0; j < kSgdVec; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q)
            comp(w[j], q) = __double2float_rn(__dadd_rn((double)comp(w[j], q), __dmul_rn((double)comp(x[j], q), coeff)));
        sq_pending = true;
        sq_factor = __fmul_rn(wsf, wsf);
      }
      intercept = __dadd_rn(intercept, update);
      t = __dadd_rn(t, 1.0);
    }

    bool finite = isfinite(intercept);
#pragma unroll
    for (int j = 0; j < kSgdVec; ++j)
      finite = finite && isfinite(w[j].x) && isfinite(w[j].y) && isfinite(w[j].z) && isfinite(w[j].w);
    if (!__all_sync(kFull, finite)) {
      overflow = true;
      iters = epoch + 1;
      break;
    }
    const double mean = objective / (double)n;
    if (tol > -INFINITY && mean > __dsub_rn(best, tol)) ++no_improvement;
    else no_improvement = 0;
    if (mean < best) best = mean;
    if (no_improvement >= n_iter_no_change) {
      iters = epoch + 1;
      break;
    }
  }

  const float s = __double2float_rn(wscale);  // w.reset_wscale
  float4* out = reinterpret_cast<float4*>(coef + (size_t)pid * D);
#pragma unroll
  for (int j = 0; j < kSgdVec; ++j)
    out[lane + 32 * j] = make_float4(__fmul_rn(w[j].x, s), __fmul_rn(w[j].y, s), __fmul_rn(w[j].z, s),
                                     __fmul_rn(w[j].w, s));
  if (lane == 0) {
    intercept_out[pid] = intercept;
    n_iter_out[pid] = iters;
    overflow_out[pid] = overflow ? 1 : 0;
  }
}

constexpr int kDecWarps = 8;

// One warp per row: scores[row, c] = x . coef_c + intercept_c (exact float products, double sums, one rounding), the
// first arg-max (n_out > 1) or score > 0 (n_out == 1).
template <int D>
__global__ void __launch_bounds__(kDecWarps * 32) linear_decision_kernel(const float* __restrict__ X, int64_t n,
                                                                         const float* __restrict__ coef,
                                                                         const double* __restrict__ intercept,
                                                                         int n_out, float* __restrict__ scores,
                                                                         int32_t* __restrict__ pred) {
  constexpr int kSgdVec = D / (32 * 4);
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kDecWarps + (threadIdx.x >> 5);
  if (row >= n) return;
  const float4* x4 = reinterpret_cast<const float4*>(X) + row * (D / 4);
  float4 x[kSgdVec];
#pragma unroll
  for (int j = 0; j < kSgdVec; ++j) x[j] = __ldg(x4 + lane + 32 * j);
  float best = -INFINITY, score = 0.f;
  int arg = 0;
  for (int c = 0; c < n_out; ++c) {
    const float4* w4 = reinterpret_cast<const float4*>(coef) + (size_t)c * (D / 4);
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < kSgdVec; ++j) {
      const float4 w = __ldg(w4 + lane + 32 * j);
      acc = __dadd_rn(acc, __dmul_rn((double)x[j].x, (double)w.x));
      acc = __dadd_rn(acc, __dmul_rn((double)x[j].y, (double)w.y));
      acc = __dadd_rn(acc, __dmul_rn((double)x[j].z, (double)w.z));
      acc = __dadd_rn(acc, __dmul_rn((double)x[j].w, (double)w.w));
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(kFull, acc, m));
    score = __double2float_rn(__dadd_rn(acc, intercept[c]));
    if (lane == 0) scores[row * n_out + c] = score;
    if (score > best || c == 0) {
      best = score;
      arg = c;
    }
  }
  if (lane == 0) pred[row] = n_out == 1 ? (score > 0.f ? 1 : 0) : arg;
}

// Workspace sections, each 256-byte aligned: problem table, class ids, sigma rows, two orders per problem.
struct SgdLayout {
  size_t problems, classes, sigma, orders, total;
};
SgdLayout sgd_layout(int64_t n, int n_sigma, int n_problems) {
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  SgdLayout l;
  l.problems = 0;
  l.classes = up(sizeof(SgdProblem) * (size_t)n_problems);
  l.sigma = l.classes + up(sizeof(int32_t) * (size_t)n);
  l.orders = l.sigma + up(sizeof(int32_t) * (size_t)n * n_sigma);
  l.total = l.orders + up(sizeof(int32_t) * (size_t)n * 2 * n_problems);
  return l;
}

uint32_t our_rand_r(uint32_t* seed) {  // sklearn/utils/_random.pxd
  if (*seed == 0) *seed = 1;
  *seed ^= (uint32_t)(*seed << 13);
  *seed ^= (uint32_t)(*seed >> 17);
  *seed ^= (uint32_t)(*seed << 5);
  return *seed % ((uint32_t)2147483647 + 1);
}

// sklearn's cgradient_half_binomial, on the host (the C library's exp, like sklearn's Cython)
double host_half_binomial_gradient(double y, double p) {
  if (p > -37) {
    const double e = exp(-p);
    return ((1 - y) - y * e) / (1 + e);
  }
  return exp(p) - y;
}

}  // namespace

int sgd_shuffle_permutation(int64_t n, uint32_t seed, int32_t* sigma) {
  PLIP_REQUIRE(sigma, "plip_sgd_shuffle_permutation: null argument");
  PLIP_REQUIRE(n >= 1 && n <= INT32_MAX, "plip_sgd_shuffle_permutation: n = %lld is outside 1..2^31-1", (long long)n);
  for (int64_t i = 0; i < n; ++i) sigma[i] = (int32_t)i;
  const int nn = (int)n;
  for (unsigned i = 0; i + 1 < (unsigned)nn; ++i) {  // dataset.shuffle: int n, unsigned i, j
    const unsigned j = i + our_rand_r(&seed) % (nn - i);
    const int32_t tmp = sigma[i];
    sigma[i] = sigma[j];
    sigma[j] = tmp;
  }
  return 0;
}

int sgd_workspace_bytes(int64_t n, int n_sigma, int n_problems, uint64_t* bytes) {
  PLIP_REQUIRE(bytes, "plip_sgd_workspace_bytes: null argument");
  PLIP_REQUIRE(n >= 2 && n <= INT32_MAX, "plip_sgd_workspace_bytes: n = %lld is outside 2..2^31-1", (long long)n);
  PLIP_REQUIRE(n_sigma >= 1 && n_problems >= 1, "plip_sgd_workspace_bytes: n_sigma = %d and n_problems = %d must be >= 1",
               n_sigma, n_problems);
  *bytes = sgd_layout(n, n_sigma, n_problems).total;
  return 0;
}

int launch_sgd_fit(const float* x, int64_t n, int dim, const int32_t* class_host, int n_classes,
                   const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host, int n_sigma,
                   int max_iter, double tol, int n_iter_no_change, float* coef, double* intercept, int32_t* n_iter,
                   int32_t* overflow, void* ws, uint64_t ws_bytes, cudaStream_t st) {
  PLIP_REQUIRE(x && class_host && problems_host && sigma_host && coef && intercept && n_iter && overflow && ws,
               "plip_sgd_fit: null argument");
  PLIP_REQUIRE(n >= 2 && n <= INT32_MAX, "plip_sgd_fit: n = %lld samples; a fit needs 2..2^31-1", (long long)n);
  PLIP_REQUIRE(dim == kSgdDimClip || dim == kSgdDimDenseNet,
               "plip_sgd_fit: dim = %d; the embeddings must be %d or %d wide", dim, kSgdDimClip, kSgdDimDenseNet);
  PLIP_REQUIRE(n_classes >= 2, "plip_sgd_fit: n_classes = %d; a fit needs at least 2", n_classes);
  PLIP_REQUIRE(n_problems >= 1 && n_sigma >= 1, "plip_sgd_fit: n_problems = %d and n_sigma = %d must be >= 1",
               n_problems, n_sigma);
  PLIP_REQUIRE(max_iter >= 1, "plip_sgd_fit: max_iter = %d must be >= 1", max_iter);
  PLIP_REQUIRE(n_iter_no_change >= 1, "plip_sgd_fit: n_iter_no_change = %d must be >= 1", n_iter_no_change);
  PLIP_REQUIRE(!isnan(tol), "plip_sgd_fit: tol is NaN");
  PLIP_REQUIRE(((uintptr_t)x & 15) == 0, "plip_sgd_fit: x_dev %p is not 16-byte aligned", (const void*)x);
  PLIP_REQUIRE(((uintptr_t)coef & 15) == 0, "plip_sgd_fit: coef_dev %p is not 16-byte aligned", (void*)coef);
  PLIP_REQUIRE(((uintptr_t)ws & 15) == 0, "plip_sgd_fit: workspace_dev %p is not 16-byte aligned", ws);
  const SgdLayout lay = sgd_layout(n, n_sigma, n_problems);
  PLIP_REQUIRE(ws_bytes >= lay.total, "plip_sgd_fit: workspace of %llu bytes, %llu needed",
               (unsigned long long)ws_bytes, (unsigned long long)lay.total);
  std::vector<SgdProblem> table((size_t)n_problems);
  for (int i = 0; i < n_problems; ++i) {
    const plip_sgd_problem_t& p = problems_host[i];
    PLIP_REQUIRE(isfinite(p.alpha) && p.alpha > 0, "plip_sgd_fit: problem %d: alpha = %g must be finite and > 0", i,
                 p.alpha);
    PLIP_REQUIRE(p.pos_class >= 0 && p.pos_class < n_classes,
                 "plip_sgd_fit: problem %d: pos_class = %d is outside 0..%d", i, p.pos_class, n_classes - 1);
    PLIP_REQUIRE(p.sigma_index >= 0 && p.sigma_index < n_sigma,
                 "plip_sgd_fit: problem %d: sigma_index = %d is outside 0..%d", i, p.sigma_index, n_sigma - 1);
    PLIP_REQUIRE(isfinite(p.pos_weight) && isfinite(p.neg_weight) && p.pos_weight > 0 && p.neg_weight > 0,
                 "plip_sgd_fit: problem %d: weights %g / %g must be finite and > 0", i, p.pos_weight, p.neg_weight);
    // plain_sgd's learning_rate == OPTIMAL set-up, as sklearn evaluates it in Python
    const double typw = sqrt(1.0 / sqrt(p.alpha));
    const double g = host_half_binomial_gradient(1.0, -typw);
    const double initial_eta0 = typw / (g > 1.0 ? g : 1.0);
    table[i] = SgdProblem{p.alpha, 1.0 / (initial_eta0 * p.alpha), (float)p.pos_weight, (float)p.neg_weight,
                          p.pos_class, p.sigma_index};
  }
  for (int64_t i = 0; i < n; ++i)
    PLIP_REQUIRE(class_host[i] >= 0 && class_host[i] < n_classes,
                 "plip_sgd_fit: class id %d of sample %lld is outside 0..%d", class_host[i], (long long)i,
                 n_classes - 1);
  for (int64_t i = 0; i < n * n_sigma; ++i)
    PLIP_REQUIRE(sigma_host[i] >= 0 && sigma_host[i] < n, "plip_sgd_fit: sigma[%lld][%lld] = %d is outside 0..%lld",
                 (long long)(i / n), (long long)(i % n), sigma_host[i], (long long)(n - 1));

  uint8_t* base = static_cast<uint8_t*>(ws);
  PLIP_CUDA_CHECK(cudaMemcpyAsync(base + lay.problems, table.data(), sizeof(SgdProblem) * table.size(),
                                  cudaMemcpyHostToDevice, st));
  PLIP_CUDA_CHECK(cudaMemcpyAsync(base + lay.classes, class_host, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice,
                                  st));
  PLIP_CUDA_CHECK(cudaMemcpyAsync(base + lay.sigma, sigma_host, sizeof(int32_t) * (size_t)n * n_sigma,
                                  cudaMemcpyHostToDevice, st));
  auto* kernel = dim == kSgdDimClip ? sgd_fit_kernel<kSgdDimClip> : sgd_fit_kernel<kSgdDimDenseNet>;
  PLIP_CUDA_CHECK(launch_kernel(kernel, dim3((unsigned)n_problems), dim3(32), 0, st, 1, x, (int)n,
                                reinterpret_cast<const int32_t*>(base + lay.classes),
                                reinterpret_cast<const SgdProblem*>(base + lay.problems),
                                reinterpret_cast<const int32_t*>(base + lay.sigma),
                                reinterpret_cast<int32_t*>(base + lay.orders), max_iter, tol, n_iter_no_change, coef,
                                intercept, n_iter, overflow));
  return 0;
}

int launch_linear_decision(const float* x, int64_t n, int dim, const float* coef, const double* intercept, int n_out,
                           float* scores, int32_t* pred, cudaStream_t st) {
  PLIP_REQUIRE(x && coef && intercept && scores && pred, "plip_linear_decision: null argument");
  PLIP_REQUIRE(dim == kSgdDimClip || dim == kSgdDimDenseNet,
               "plip_linear_decision: dim = %d; the embeddings must be %d or %d wide", dim, kSgdDimClip, kSgdDimDenseNet);
  PLIP_REQUIRE(n >= 0, "plip_linear_decision: n = %lld is negative", (long long)n);
  PLIP_REQUIRE(n_out >= 1, "plip_linear_decision: n_out = %d must be >= 1", n_out);
  PLIP_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)coef & 15) == 0,
               "plip_linear_decision: x_dev %p and coef_dev %p must be 16-byte aligned", (const void*)x,
               (const void*)coef);
  if (n == 0) return 0;
  auto* kernel = dim == kSgdDimClip ? linear_decision_kernel<kSgdDimClip> : linear_decision_kernel<kSgdDimDenseNet>;
  PLIP_CUDA_CHECK(launch_kernel(kernel, dim3((unsigned)((n + kDecWarps - 1) / kDecWarps)),
                                dim3(kDecWarps * 32), 0, st, 1, x, n, coef, intercept, n_out, scores, pred));
  return 0;
}

}  // namespace plip

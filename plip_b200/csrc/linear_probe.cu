// plip_b200 — the reference's linear probe on the device: scikit-learn's SGD logistic regression
// (SGDClassifier(loss="log_loss", penalty="l2", learning_rate="optimal"), sklearn 1.9 _plain_sgd in both of its
// instantiations: 32-bit for float32 input, 64-bit for float16 / float64 input), every one-vs-rest problem of a fit and
// every alpha of a sweep at once, plus the linear decision.
//
// sgd_fit_kernel<T, D>: one warp per binary problem, all epochs on the device.  A problem is one dependent chain of n
// sample steps per epoch (each step's update feeds the next step's dot product), so the kernel is bound by the latency
// of that chain, not by HBM or the tensor cores: one warp per problem, one problem per block so that problems spread
// over SMs.  Per step the warp
//   - reads row x of X from a shared-memory ring that cp.async fills kRing samples ahead along the epoch order (the
//     order and the class ids are loaded a 32-sample chunk or two ahead), so no global-memory latency is on the chain;
//   - reduces w.x and sum(w^2) in one warp-shuffle pass (the objective needs |w|^2 of the previous add; sklearn's add
//     recomputes it right away, here it is taken at the start of the next step, from the same weights);
//   - runs sklearn's scalar step in fp64, lane-uniform (every lane holds the bit-identical reduced sums: a butterfly
//     reduction adds the same two values in every lane);
//   - applies scale / add to its D / 32 weights (lane l holds the 16-byte chunks l + 32 k of the row: 4 floats or
//     2 doubles) with the casts of sklearn's WeightVector32 / WeightVector64 (SgdReal<T>, from_double<T>).
// T = float (WeightVector32) and T = double (WeightVector64) are instantiated for the two embedding widths the
// reference probes, D = 512 (CLIP) and D = 1024 (MuDiPath's DenseNet-121).  The ring stays within 32 KB of static
// shared memory: 8 rows, except 4 rows of 8 KB for double at 1024 (a shallower ring rather than an opt-in to more
// than 48 KB of dynamic shared memory; a row is still issued 4 dependent steps before it is read).
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
constexpr double kMaxDloss = 1e12;
constexpr unsigned kFull = 0xffffffffu;

// The weight type T of sklearn's two instantiations: WeightVector32 (float weights, reset below 1e-6) and
// WeightVector64 (double weights, reset below 1e-9).  X, the weights and the class weights are T; wscale, sq_norm, p,
// eta, update and the objective are double in both.  Each lane moves 16-byte chunks (Vec) of a row: 4 floats or
// 2 doubles.  The cp.async ring holds kRing rows of at most 32 KB in all (static shared memory): 8 rows in float at both
// widths and in double at 512, 4 rows of 8 KB in double at 1024.
template <typename T>
struct SgdReal;
template <>
struct SgdReal<float> {
  using Vec = float4;
  static constexpr double kResetWscale = 1e-6;
};
template <>
struct SgdReal<double> {
  using Vec = double2;
  static constexpr double kResetWscale = 1e-9;
};
template <typename T, int D>
struct SgdShape {
  static constexpr int kPerVec = 16 / (int)sizeof(T);
  static constexpr int kRowVecs = D / kPerVec;       // 16-byte chunks per row
  static constexpr int kVec = kRowVecs / 32;          // chunks per lane
  static constexpr int kRing = 32768 / (D * (int)sizeof(T)) < 8 ? 32768 / (D * (int)sizeof(T)) : 8;
  static_assert(kVec * 32 == kRowVecs && kRing >= 2, "SgdShape");
};

// T arithmetic with one rounding and no FMA contraction (sklearn's C code runs on x86-64 without FMA).
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
template <typename T>
__device__ __forceinline__ T from_double(double v);
template <>
__device__ __forceinline__ float from_double<float>(double v) { return __double2float_rn(v); }
template <>
__device__ __forceinline__ double from_double<double>(double v) { return v; }

// One binary problem; pos / neg weights are T, as sklearn's class_weight local (32 or 40 bytes).
template <typename T>
struct SgdProblem {
  double alpha;
  double optimal_init;   // computed on the host with the C library's exp, as sklearn does in Python
  T weight_pos;
  T weight_neg;
  int32_t pos_class;
  int32_t sigma_index;
};
static_assert(sizeof(SgdProblem<float>) == 32 && sizeof(SgdProblem<double>) == 40, "SgdProblem layout");
constexpr size_t kSgdProblemSlot = sizeof(SgdProblem<double>);  // the workspace holds either table

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

// sklearn's clip of dloss to +-MAX_DLOSS (`if dloss < -MAX_DLOSS: ... elif dloss > MAX_DLOSS: ...`) lets a NaN through:
// float64 rows near 1e200 overflow w.x to inf - inf, the NaN update makes the weights NaN and the fit raises.  The
// 32-bit instantiation keeps its fmin / fmax form, so its kernels compile to what they were (there fmax maps a NaN to
// -MAX_DLOSS).
template <typename T>
__device__ __forceinline__ double clip_dloss(double d);
template <>
__device__ __forceinline__ double clip_dloss<float>(double d) { return fmin(fmax(d, -kMaxDloss), kMaxDloss); }
template <>
__device__ __forceinline__ double clip_dloss<double>(double d) {
  return d < -kMaxDloss ? -kMaxDloss : d > kMaxDloss ? kMaxDloss : d;
}

__device__ __forceinline__ float& comp(float4& v, int c) { return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w; }
__device__ __forceinline__ double& comp(double2& v, int c) { return c == 0 ? v.x : v.y; }

// sklearn's _plain_sgd in the instantiation of T.  The casts of WeightVector32 / 64 fall out of T: dot returns T
// (rounded to float, or the double sum * wscale as is), scale takes a T, add takes a T coefficient and divides it by a T
// copy of wscale, and the objective squares a T norm.  In double every from_double is the identity.
template <typename T, int D>
__global__ void __launch_bounds__(32) sgd_fit_kernel(const T* __restrict__ X, int n, const int32_t* __restrict__ cls,
                                                    const SgdProblem<T>* __restrict__ problems,
                                                    const int32_t* __restrict__ sigma, int32_t* orders, int max_iter,
                                                    double tol, int n_iter_no_change, T* __restrict__ coef,
                                                    double* __restrict__ intercept_out, int32_t* __restrict__ n_iter_out,
                                                    int32_t* __restrict__ overflow_out) {
  using Vec = typename SgdReal<T>::Vec;
  using S = SgdShape<T, D>;
  constexpr int kVec = S::kVec, kPer = S::kPerVec, kRing = S::kRing;
  __shared__ __align__(16) Vec ring[kRing][S::kRowVecs];
  const int lane = threadIdx.x;
  const int pid = blockIdx.x;
  const SgdProblem<T> pr = problems[pid];
  const int32_t* sig = sigma + (size_t)pr.sigma_index * n;
  int32_t* own = orders + (size_t)pid * 2 * n;  // two epoch orders, used in turn
  const Vec* Xv = reinterpret_cast<const Vec*>(X);

  Vec w[kVec];
#pragma unroll
  for (int j = 0; j < kVec; ++j)
#pragma unroll
    for (int q = 0; q < kPer; ++q) comp(w[j], q) = T(0);
  double wscale = 1.0, sq_norm = 0.0, intercept = 0.0, t = 1.0;
  bool sq_pending = false;  // the last step added to w: sq_norm = sum(w^2) * sq_factor at the next step
  T sq_factor = T(1);
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
        Vec* slot = ring[s % kRing];
#pragma unroll
        for (int j = 0; j < kVec; ++j)
          cp_async_16(slot + lane + 32 * j, Xv + (size_t)row * S::kRowVecs + lane + 32 * j);
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
      const T y = __shfl_sync(kFull, a_cls, k & 31) == pr.pos_class ? T(1) : T(0);
      cp_async_wait<kRing - 1>();  // this lane's copies of sample k have landed (each lane reads only its own)
      Vec x[kVec];
      const Vec* slot = ring[k % kRing];
#pragma unroll
      for (int j = 0; j < kVec; ++j) x[j] = slot[lane + 32 * j];

      double dot = 0.0, sq = 0.0;
#pragma unroll
      for (int j = 0; j < kVec; ++j)
#pragma unroll
        for (int c = 0; c < kPer; ++c) {
          dot = __dadd_rn(dot, (double)mul_rn(comp(w[j], c), comp(x[j], c)));
          sq = __dadd_rn(sq, (double)mul_rn(comp(w[j], c), comp(w[j], c)));
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
      const double p = __dadd_rn((double)from_double<T>(__dmul_rn(dot, wscale)), intercept);
      const double eta = 1.0 / __dmul_rn(pr.alpha, __dsub_rn(__dadd_rn(pr.optimal_init, t), 1.0));
      objective = __dadd_rn(objective, half_binomial_loss(yd, p));
      // alpha * ((1 - l1_ratio) * 0.5 * norm ** 2 + l1_ratio * l1norm) with l1_ratio = 0
      const T norm = from_double<T>(sqrt(sq_norm));
      objective = __dadd_rn(objective, __dmul_rn(__dmul_rn(0.5, (double)mul_rn(norm, norm)), pr.alpha));
      const double dloss = clip_dloss<T>(half_binomial_gradient(yd, p));
      const double update = __dmul_rn(__dmul_rn(-eta, dloss), (double)(y > T(0) ? pr.weight_pos : pr.weight_neg));

      const T c = from_double<T>(fmax(0.0, __dsub_rn(1.0, __dmul_rn(eta, pr.alpha))));  // w.scale
      wscale = __dmul_rn(wscale, (double)c);
      sq_norm = __dmul_rn(sq_norm, (double)mul_rn(c, c));
      if (wscale < SgdReal<T>::kResetWscale) {
        const T s = from_double<T>(wscale);
#pragma unroll
        for (int j = 0; j < kVec; ++j)
#pragma unroll
          for (int q = 0; q < kPer; ++q) comp(w[j], q) = mul_rn(comp(w[j], q), s);
        wscale = 1.0;
      }
      if (update != 0.0) {  // w.add
        const T wsf = from_double<T>(wscale);
        const double coeff = (double)div_rn(from_double<T>(update), wsf);
#pragma unroll
        for (int j = 0; j < kVec; ++j)
#pragma unroll
          for (int q = 0; q < kPer; ++q)
            comp(w[j], q) = from_double<T>(__dadd_rn((double)comp(w[j], q), __dmul_rn((double)comp(x[j], q), coeff)));
        sq_pending = true;
        sq_factor = mul_rn(wsf, wsf);
      }
      intercept = __dadd_rn(intercept, update);
      t = __dadd_rn(t, 1.0);
    }

    bool finite = isfinite(intercept);
#pragma unroll
    for (int j = 0; j < kVec; ++j)
#pragma unroll
      for (int q = 0; q < kPer; ++q) finite = finite && isfinite(comp(w[j], q));
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

  const T s = from_double<T>(wscale);  // w.reset_wscale
  Vec* out = reinterpret_cast<Vec*>(coef + (size_t)pid * D);
#pragma unroll
  for (int j = 0; j < kVec; ++j) {
    Vec v = w[j];
#pragma unroll
    for (int q = 0; q < kPer; ++q) comp(v, q) = mul_rn(comp(v, q), s);
    out[lane + 32 * j] = v;
  }
  if (lane == 0) {
    intercept_out[pid] = intercept;
    n_iter_out[pid] = iters;
    overflow_out[pid] = overflow ? 1 : 0;
  }
}

constexpr int kDecWarps = 8;

// One warp per row: scores[row, c] = x . coef_c + intercept_c (exact widening of x and coef, double products and sums,
// one rounding to T), the first arg-max (n_out > 1) or score > 0 (n_out == 1).
template <typename T, int D>
__global__ void __launch_bounds__(kDecWarps * 32) linear_decision_kernel(const T* __restrict__ X, int64_t n,
                                                                         const T* __restrict__ coef,
                                                                         const double* __restrict__ intercept,
                                                                         int n_out, T* __restrict__ scores,
                                                                         int32_t* __restrict__ pred) {
  using Vec = typename SgdReal<T>::Vec;
  using S = SgdShape<T, D>;
  constexpr int kVec = S::kVec, kPer = S::kPerVec;
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kDecWarps + (threadIdx.x >> 5);
  if (row >= n) return;
  const Vec* xv = reinterpret_cast<const Vec*>(X) + row * S::kRowVecs;
  Vec x[kVec];
#pragma unroll
  for (int j = 0; j < kVec; ++j) x[j] = __ldg(xv + lane + 32 * j);
  T best = -INFINITY, score = T(0);
  int arg = 0;
  for (int c = 0; c < n_out; ++c) {
    const Vec* wv = reinterpret_cast<const Vec*>(coef) + (size_t)c * S::kRowVecs;
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
      Vec w = __ldg(wv + lane + 32 * j);
#pragma unroll
      for (int q = 0; q < kPer; ++q) acc = __dadd_rn(acc, __dmul_rn((double)comp(x[j], q), (double)comp(w, q)));
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(kFull, acc, m));
    score = from_double<T>(__dadd_rn(acc, intercept[c]));
    if (lane == 0) scores[row * n_out + c] = score;
    if (score > best || c == 0) {
      best = score;
      arg = c;
    }
  }
  if (lane == 0) pred[row] = n_out == 1 ? (score > T(0) ? 1 : 0) : arg;
}

// Workspace sections, each 256-byte aligned: problem table, class ids, sigma rows, two orders per problem.
struct SgdLayout {
  size_t problems, classes, sigma, orders, total;
};
SgdLayout sgd_layout(int64_t n, int n_sigma, int n_problems) {
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  SgdLayout l;
  l.problems = 0;
  l.classes = up(kSgdProblemSlot * (size_t)n_problems);
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

namespace {

// plip_sgd_fit / plip_sgd_fit_f64: the checks and the launch are shared; `name` prefixes every error.
template <typename T>
int sgd_fit_impl(const char* name, const T* x, int64_t n, int dim, const int32_t* class_host, int n_classes,
                 const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host, int n_sigma,
                 int max_iter, double tol, int n_iter_no_change, T* coef, double* intercept, int32_t* n_iter,
                 int32_t* overflow, void* ws, uint64_t ws_bytes, cudaStream_t st) {
  PLIP_REQUIRE(x && class_host && problems_host && sigma_host && coef && intercept && n_iter && overflow && ws,
               "%s: null argument", name);
  PLIP_REQUIRE(n >= 2 && n <= INT32_MAX, "%s: n = %lld samples; a fit needs 2..2^31-1", name, (long long)n);
  PLIP_REQUIRE(dim == kSgdDimClip || dim == kSgdDimDenseNet, "%s: dim = %d; the embeddings must be %d or %d wide",
               name, dim, kSgdDimClip, kSgdDimDenseNet);
  PLIP_REQUIRE(n_classes >= 2, "%s: n_classes = %d; a fit needs at least 2", name, n_classes);
  PLIP_REQUIRE(n_problems >= 1 && n_sigma >= 1, "%s: n_problems = %d and n_sigma = %d must be >= 1", name,
               n_problems, n_sigma);
  PLIP_REQUIRE(max_iter >= 1, "%s: max_iter = %d must be >= 1", name, max_iter);
  PLIP_REQUIRE(n_iter_no_change >= 1, "%s: n_iter_no_change = %d must be >= 1", name, n_iter_no_change);
  PLIP_REQUIRE(!isnan(tol), "%s: tol is NaN", name);
  PLIP_REQUIRE(((uintptr_t)x & 15) == 0, "%s: x_dev %p is not 16-byte aligned", name, (const void*)x);
  PLIP_REQUIRE(((uintptr_t)coef & 15) == 0, "%s: coef_dev %p is not 16-byte aligned", name, (void*)coef);
  PLIP_REQUIRE(((uintptr_t)ws & 15) == 0, "%s: workspace_dev %p is not 16-byte aligned", name, ws);
  const SgdLayout lay = sgd_layout(n, n_sigma, n_problems);
  PLIP_REQUIRE(ws_bytes >= lay.total, "%s: workspace of %llu bytes, %llu needed", name, (unsigned long long)ws_bytes,
               (unsigned long long)lay.total);
  std::vector<SgdProblem<T>> table((size_t)n_problems);
  for (int i = 0; i < n_problems; ++i) {
    const plip_sgd_problem_t& p = problems_host[i];
    PLIP_REQUIRE(isfinite(p.alpha) && p.alpha > 0, "%s: problem %d: alpha = %g must be finite and > 0", name, i,
                 p.alpha);
    PLIP_REQUIRE(p.pos_class >= 0 && p.pos_class < n_classes, "%s: problem %d: pos_class = %d is outside 0..%d", name,
                 i, p.pos_class, n_classes - 1);
    PLIP_REQUIRE(p.sigma_index >= 0 && p.sigma_index < n_sigma, "%s: problem %d: sigma_index = %d is outside 0..%d",
                 name, i, p.sigma_index, n_sigma - 1);
    PLIP_REQUIRE(isfinite(p.pos_weight) && isfinite(p.neg_weight) && p.pos_weight > 0 && p.neg_weight > 0,
                 "%s: problem %d: weights %g / %g must be finite and > 0", name, i, p.pos_weight, p.neg_weight);
    // plain_sgd's learning_rate == OPTIMAL set-up, as sklearn evaluates it in Python
    const double typw = sqrt(1.0 / sqrt(p.alpha));
    const double g = host_half_binomial_gradient(1.0, -typw);
    const double initial_eta0 = typw / (g > 1.0 ? g : 1.0);
    table[i] = SgdProblem<T>{p.alpha, 1.0 / (initial_eta0 * p.alpha), (T)p.pos_weight, (T)p.neg_weight, p.pos_class,
                             p.sigma_index};
  }
  for (int64_t i = 0; i < n; ++i)
    PLIP_REQUIRE(class_host[i] >= 0 && class_host[i] < n_classes, "%s: class id %d of sample %lld is outside 0..%d",
                 name, class_host[i], (long long)i, n_classes - 1);
  for (int64_t i = 0; i < n * n_sigma; ++i)
    PLIP_REQUIRE(sigma_host[i] >= 0 && sigma_host[i] < n, "%s: sigma[%lld][%lld] = %d is outside 0..%lld", name,
                 (long long)(i / n), (long long)(i % n), sigma_host[i], (long long)(n - 1));

  uint8_t* base = static_cast<uint8_t*>(ws);
  PLIP_CUDA_CHECK(cudaMemcpyAsync(base + lay.problems, table.data(), sizeof(SgdProblem<T>) * table.size(),
                                  cudaMemcpyHostToDevice, st));
  PLIP_CUDA_CHECK(cudaMemcpyAsync(base + lay.classes, class_host, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice,
                                  st));
  PLIP_CUDA_CHECK(cudaMemcpyAsync(base + lay.sigma, sigma_host, sizeof(int32_t) * (size_t)n * n_sigma,
                                  cudaMemcpyHostToDevice, st));
  auto* kernel = dim == kSgdDimClip ? sgd_fit_kernel<T, kSgdDimClip> : sgd_fit_kernel<T, kSgdDimDenseNet>;
  PLIP_CUDA_CHECK(launch_kernel(kernel, dim3((unsigned)n_problems), dim3(32), 0, st, 1, x, (int)n,
                                reinterpret_cast<const int32_t*>(base + lay.classes),
                                reinterpret_cast<const SgdProblem<T>*>(base + lay.problems),
                                reinterpret_cast<const int32_t*>(base + lay.sigma),
                                reinterpret_cast<int32_t*>(base + lay.orders), max_iter, tol, n_iter_no_change, coef,
                                intercept, n_iter, overflow));
  return 0;
}

template <typename T>
int linear_decision_impl(const char* name, const T* x, int64_t n, int dim, const T* coef, const double* intercept,
                         int n_out, T* scores, int32_t* pred, cudaStream_t st) {
  PLIP_REQUIRE(x && coef && intercept && scores && pred, "%s: null argument", name);
  PLIP_REQUIRE(dim == kSgdDimClip || dim == kSgdDimDenseNet, "%s: dim = %d; the embeddings must be %d or %d wide",
               name, dim, kSgdDimClip, kSgdDimDenseNet);
  PLIP_REQUIRE(n >= 0, "%s: n = %lld is negative", name, (long long)n);
  PLIP_REQUIRE(n_out >= 1, "%s: n_out = %d must be >= 1", name, n_out);
  PLIP_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)coef & 15) == 0,
               "%s: x_dev %p and coef_dev %p must be 16-byte aligned", name, (const void*)x, (const void*)coef);
  if (n == 0) return 0;
  auto* kernel = dim == kSgdDimClip ? linear_decision_kernel<T, kSgdDimClip> : linear_decision_kernel<T, kSgdDimDenseNet>;
  PLIP_CUDA_CHECK(launch_kernel(kernel, dim3((unsigned)((n + kDecWarps - 1) / kDecWarps)), dim3(kDecWarps * 32), 0,
                                st, 1, x, n, coef, intercept, n_out, scores, pred));
  return 0;
}

}  // namespace

int launch_sgd_fit(const float* x, int64_t n, int dim, const int32_t* class_host, int n_classes,
                   const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host, int n_sigma,
                   int max_iter, double tol, int n_iter_no_change, float* coef, double* intercept, int32_t* n_iter,
                   int32_t* overflow, void* ws, uint64_t ws_bytes, cudaStream_t st) {
  return sgd_fit_impl("plip_sgd_fit", x, n, dim, class_host, n_classes, problems_host, n_problems, sigma_host,
                      n_sigma, max_iter, tol, n_iter_no_change, coef, intercept, n_iter, overflow, ws, ws_bytes, st);
}

int launch_sgd_fit_f64(const double* x, int64_t n, int dim, const int32_t* class_host, int n_classes,
                       const plip_sgd_problem_t* problems_host, int n_problems, const int32_t* sigma_host, int n_sigma,
                       int max_iter, double tol, int n_iter_no_change, double* coef, double* intercept,
                       int32_t* n_iter, int32_t* overflow, void* ws, uint64_t ws_bytes, cudaStream_t st) {
  return sgd_fit_impl("plip_sgd_fit_f64", x, n, dim, class_host, n_classes, problems_host, n_problems, sigma_host,
                      n_sigma, max_iter, tol, n_iter_no_change, coef, intercept, n_iter, overflow, ws, ws_bytes, st);
}

int launch_linear_decision(const float* x, int64_t n, int dim, const float* coef, const double* intercept, int n_out,
                           float* scores, int32_t* pred, cudaStream_t st) {
  return linear_decision_impl("plip_linear_decision", x, n, dim, coef, intercept, n_out, scores, pred, st);
}

int launch_linear_decision_f64(const double* x, int64_t n, int dim, const double* coef, const double* intercept,
                               int n_out, double* scores, int32_t* pred, cudaStream_t st) {
  return linear_decision_impl("plip_linear_decision_f64", x, n, dim, coef, intercept, n_out, scores, pred, st);
}

}  // namespace plip

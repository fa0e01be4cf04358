// SGDClassifier(loss="log") of the reference's eval scripts (eval_scripts/*_eval.py): scikit-learn's plain SGD
// (sklearn/linear_model/_sgd_fast.pyx.tp, _plain_sgd) for L2 / alpha / "optimal" learning rate / no averaging, in fp64,
// for P independent binary problems over one X.  Contract: oracle/sgd.py; semantics: include/graphsage_b200.h.
#include "common.cuh"

namespace gs {

// ---- epoch orders ----------------------------------------------------------------------------
// our_rand_r (sklearn/utils/_random.pxd): xorshift32, a zero state becomes 1, result modulo 2^31
__device__ __forceinline__ uint32_t sgd_rand(uint32_t& s) {
  if (s == 0u) s = 1u;
  s ^= s << 13;
  s ^= s >> 17;
  s ^= s << 5;
  return s & 0x7fffffffu;
}

// One CTA per problem: the CTA writes arange(n) into epoch 0's slice, then thread 0 runs the n - 1 Fisher-Yates swaps
// (SequentialDataset.shuffle) on it.  The chain is sequential by definition.
__global__ void __launch_bounds__(256) sgd_sigma_kernel(const uint32_t* __restrict__ seeds, int64_t n, int32_t epochs,
                                                        int32_t* __restrict__ orders) {
  int32_t* ind = orders + (int64_t)blockIdx.x * epochs * n;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) ind[i] = (int32_t)i;
  __syncthreads();
  if (threadIdx.x != 0) return;
  uint32_t s = seeds[blockIdx.x];
  const uint32_t nn = (uint32_t)n;
  for (uint32_t i = 0; i + 1 < nn; ++i) {
    const uint32_t j = i + sgd_rand(s) % (nn - i);
    const int32_t a = ind[i], b = ind[j];
    ind[i] = b;
    ind[j] = a;
  }
}

// orders[p, e, k] = sigma[orders[p, e - 1, k]]: every epoch re-applies the same swaps to the previous order.
__global__ void sgd_epochs_kernel(int64_t n, int32_t epochs, int32_t* __restrict__ orders) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  int32_t* o = orders + (int64_t)blockIdx.y * epochs * n;
  int32_t cur = o[k];
  for (int32_t e = 1; e < epochs; ++e) {
    cur = o[cur];
    o[(int64_t)e * n + k] = cur;
  }
}

// ---- fit ---------------------------------------------------------------------------------------
constexpr int kSgdStages = 8;   // rows in flight ahead of the step that consumes them

struct SgdFitArgs {
  const void* x;
  int64_t n, ldx, ldy, ldc;
  int32_t d, epochs;
  const int32_t* labels;
  const int32_t* orders;
  double alpha, optimal_init;
  double* coef;
  double* intercept;
};

__device__ __forceinline__ void cp_async(void* smem, const void* g, int bytes) {
  if (bytes == 8)
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem)), "l"(g) : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// One warp (= one CTA) per problem.  Lane l owns columns j = k*32 + l (k < K): w in registers, its x elements copied by
// the lane itself into a shared ring of kSgdStages rows.  Lane 0 streams the step's row index (two rings ahead) and label.
// Products and sums are separately rounded (__dmul_rn / __dadd_rn): no FMA contraction, so the order below is the whole
// rounding contract of the dot product and the update.
template <typename T, int K>
__global__ void __launch_bounds__(32) sgd_fit_kernel(SgdFitArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  T* xring = reinterpret_cast<T*>(smem);                                        // [kSgdStages][K * 32]
  int32_t* lring = reinterpret_cast<int32_t*>(xring + kSgdStages * K * 32);     // [kSgdStages] labels
  int32_t* iring = lring + kSgdStages;                                          // [2 * kSgdStages] row indices
  const int lane = threadIdx.x;
  const int64_t p = blockIdx.x;
  const int64_t steps = (int64_t)a.epochs * a.n;
  const int32_t* ord = a.orders + p * steps;
  const int32_t* lab = a.labels + p * a.ldy;
  const T* X = static_cast<const T*>(a.x);

  // the row of step s + kSgdStages: x and label; the index of step s + 2 kSgdStages (an empty group past the end)
  auto issue = [&](int64_t s, bool with_index) {
    const int64_t t = s + kSgdStages;
    if (t < steps) {
      const int32_t row = iring[t % (2 * kSgdStages)];
      const T* src = X + (int64_t)row * a.ldx;
      T* dst = xring + (t % kSgdStages) * (K * 32);
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int j = k * 32 + lane;
        if (j < a.d) cp_async(dst + j, src + j, (int)sizeof(T));
      }
      if (lane == 0) cp_async(lring + t % kSgdStages, lab + row, 4);
    }
    if (with_index && lane == 0 && t + kSgdStages < steps)
      cp_async(iring + (t + kSgdStages) % (2 * kSgdStages), ord + t + kSgdStages, 4);
    cp_async_commit();
  };

  // prologue: indices of steps 0 .. 2 kSgdStages - 1, then the rows of steps 0 .. kSgdStages - 1
  if (lane < 2 * kSgdStages && lane < steps) cp_async(iring + lane, ord + lane, 4);
  cp_async_commit();
  cp_async_wait<0>();
  __syncwarp();
  for (int s = -kSgdStages; s < 0; ++s) issue(s, false);

  double w[K];
#pragma unroll
  for (int k = 0; k < K; ++k) w[k] = 0.0;
  double wscale = 1.0, intercept = 0.0, t = 1.0;
  const double alpha = a.alpha, optimal_init = a.optimal_init;

  for (int64_t s = 0; s < steps; ++s) {
    cp_async_wait<kSgdStages - 1>();     // the group of step s (and the index of step s + kSgdStages) has landed
    __syncwarp();
    const T* xs = xring + (s % kSgdStages) * (K * 32);
    double xv[K];
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int j = k * 32 + lane;
      xv[k] = j < a.d ? (double)xs[j] : 0.0;
      if (j < a.d) acc = __dadd_rn(acc, __dmul_rn(w[k], xv[k]));
    }
    const double y = lring[s % kSgdStages] > 0 ? 1.0 : 0.0;
    __syncwarp();                        // every lane has read its slots before they are refilled
    issue(s, true);

#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, off));
    const double pred = __dadd_rn(__dmul_rn(acc, wscale), intercept);              // w.dot() + intercept  (:484)
    const double eta = 1.0 / (alpha * __dsub_rn(__dadd_rn(optimal_init, t), 1.0)); // (:486)
    double dloss;                                                                   // CyHalfBinomialLoss.cy_gradient
    if (pred > -37.0) {
      const double e = exp(-pred);
      dloss = __dsub_rn(1.0 - y, __dmul_rn(y, e)) / __dadd_rn(1.0, e);
    } else {
      dloss = __dsub_rn(exp(pred), y);
    }
    if (dloss < -1e12) dloss = -1e12;                                               // (:526-529)
    else if (dloss > 1e12) dloss = 1e12;
    const double update = -eta * dloss;                                             // (:530)
    double c = __dsub_rn(1.0, __dmul_rn(eta, alpha));                               // w.scale(max(0, ...)) (:545)
    c = c > 0.0 ? c : 0.0;
    wscale = __dmul_rn(wscale, c);
    if (wscale < 1e-9) {                                                            // reset_wscale
#pragma unroll
      for (int k = 0; k < K; ++k) w[k] = __dmul_rn(wscale, w[k]);
      wscale = 1.0;
    }
    if (update != 0.0) {                                                            // w.add (:547-548)
      const double cw = update / wscale;
#pragma unroll
      for (int k = 0; k < K; ++k) w[k] = __dadd_rn(w[k], __dmul_rn(xv[k], cw));
      intercept = __dadd_rn(intercept, update);                                     // (:549-554)
    }
    t = __dadd_rn(t, 1.0);
  }
  cp_async_wait<0>();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int j = k * 32 + lane;
    if (j < a.d) a.coef[p * a.ldc + j] = __dmul_rn(wscale, w[k]);                  // w.reset_wscale() (:635)
  }
  if (lane == 0) a.intercept[p] = intercept;
}

template <typename T, int K>
int32_t launch_fit(const SgdFitArgs& a, int32_t P, cudaStream_t st) {
  const int smem = kSgdStages * K * 32 * (int)sizeof(T) + 3 * kSgdStages * 4;
  int32_t rc = ensure_dyn_smem((const void*)sgd_fit_kernel<T, K>, smem);
  if (rc != GS_OK) return rc;
  sgd_fit_kernel<T, K><<<(unsigned)P, 32, smem, st>>>(a);
  return launch_check("sgd_fit_kernel");
}

template <typename T>
int32_t dispatch_fit(const SgdFitArgs& a, int32_t P, cudaStream_t st) {
  const int slots = (a.d + 31) / 32;
  if (slots <= 1) return launch_fit<T, 1>(a, P, st);
  if (slots <= 2) return launch_fit<T, 2>(a, P, st);
  if (slots <= 4) return launch_fit<T, 4>(a, P, st);
  if (slots <= 8) return launch_fit<T, 8>(a, P, st);
  if (slots <= 16) return launch_fit<T, 16>(a, P, st);
  return launch_fit<T, 32>(a, P, st);
}

}  // namespace gs

extern "C" {

int32_t gs_sgd_orders(const uint32_t* seeds, int32_t P, int64_t n, int32_t epochs, int32_t* orders, void* stream) {
  GS_REQUIRE(seeds && orders, "gs_sgd_orders: NULL pointer");
  GS_REQUIRE(P >= 1 && epochs >= 1, "gs_sgd_orders: need P >= 1 and epochs >= 1");
  if (P > GS_SGD_MAX_PROBLEMS || epochs > GS_SGD_MAX_EPOCHS || n < 1 || n > 0x7fffffffLL) {
    gs::set_error("gs_sgd_orders: need P <= %d, epochs <= %d, 1 <= n < 2^31 (got P=%d, epochs=%d, n=%lld)",
                  GS_SGD_MAX_PROBLEMS, GS_SGD_MAX_EPOCHS, P, epochs, (long long)n);
    return GS_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  gs::sgd_sigma_kernel<<<(unsigned)P, 256, 0, st>>>(seeds, n, epochs, orders);
  int32_t rc = gs::launch_check("sgd_sigma_kernel");
  if (rc != GS_OK || epochs == 1) return rc;
  gs::sgd_epochs_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)P), 256, 0, st>>>(n, epochs, orders);
  return gs::launch_check("sgd_epochs_kernel");
}

int32_t gs_sgd_fit(const void* x, int32_t dtype, int64_t n, int32_t d, int64_t ldx, const int32_t* labels, int64_t ldy,
                   const int32_t* orders, int32_t P, int32_t epochs, double alpha, double optimal_init, double* coef,
                   int64_t ldc, double* intercept, void* stream) {
  GS_REQUIRE(x && labels && orders && coef && intercept, "gs_sgd_fit: NULL pointer");
  GS_REQUIRE(P >= 1 && epochs >= 1 && n >= 1 && d >= 1, "gs_sgd_fit: need P, epochs, n, d >= 1");
  GS_REQUIRE(ldx >= d && ldy >= n && ldc >= d, "gs_sgd_fit: need ldx >= d, ldy >= n, ldc >= d");
  GS_REQUIRE(alpha > 0.0 && optimal_init >= 1.0, "gs_sgd_fit: need alpha > 0 and optimal_init >= 1");
  if ((dtype != GS_F32 && dtype != GS_F64) || d > GS_SGD_MAX_D || P > GS_SGD_MAX_PROBLEMS ||
      epochs > GS_SGD_MAX_EPOCHS || n > 0x7fffffffLL) {
    gs::set_error("gs_sgd_fit: need an fp32 or fp64 X, d <= %d, P <= %d, epochs <= %d, n < 2^31 (got dtype=%d, d=%d, "
                  "P=%d, epochs=%d, n=%lld)", GS_SGD_MAX_D, GS_SGD_MAX_PROBLEMS, GS_SGD_MAX_EPOCHS, dtype, d, P, epochs,
                  (long long)n);
    return GS_ERR_UNSUPPORTED;
  }
  gs::SgdFitArgs a;
  a.x = x; a.n = n; a.ldx = ldx; a.ldy = ldy; a.ldc = ldc; a.d = d; a.epochs = epochs;
  a.labels = labels; a.orders = orders; a.alpha = alpha; a.optimal_init = optimal_init;
  a.coef = coef; a.intercept = intercept;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == GS_F64 ? gs::dispatch_fit<double>(a, P, st) : gs::dispatch_fit<float>(a, P, st);
}

}  // extern "C"

// Backward of the full-neighbourhood reductions (SupervisedGraphsage.full_neighbor_train_step; contract in
// oracle/full_neighbor_grad.py):
//   gs_csr_transpose     the effective forward CSR (clamped entries, {N} for empty rows and the dummy, optionally the row's
//                        own id) transposed on the device: per-row entry counts -> CUB exclusive scan (slots) -> one warp
//                        per row writes its (destination, source row) pairs in (row, position) order -> CUB stable radix
//                        sort by destination -> t_indptr[j] = lower_bound(sorted destinations, j).  Integer work only;
//                        the entry count never leaves the device.
//   gs_csr_max_backward  TensorFlow's reduce_max gradient over whole CSR rows in two launches of one kernel template:
//                        (a) per forward row, the tie count and the scale s = dm / count; (b) per transposed row, the
//                        masked sum of s, then the ReLU mask of the Dense layer.
//                        kW (gs_csr_max_backward_weighted; oracle/weighted.py): m = max fl(w_e * z_e), so (a) counts the
//                        entries with fl(w_e * z_e) == m (forward weights, 1 for the dummy entry) and (b) adds fl(w * s)
//                        where fl(w * z_j) == m (w: the transposed entry's forward weight).
// Each output element of (a) and (b) is ONE sequential chain over its row's entries in order, run on the hub / short row
// schedule of csr_rows.cuh; the hub rows here include the in-degree hubs of the transpose.
#include "csr_rows.cuh"

#define CUB_WRAPPED_NAMESPACE gs_cub
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace gs {

constexpr int kTransposeThreads = 256;

// ---------------------------------------------------------------- transpose

struct TransposePlan {
  int64_t rows = 0, cap = 0;          // N + 1 effective rows; slots for their entries
  int end_bit = 1;
  size_t off_cnt = 0, off_slot = 0, off_kin = 0, off_kout = 0, off_vin = 0, off_cub = 0;
  size_t cub_bytes = 0, bytes = 0;
};

// cnt[i] = entries of effective row i (i <= N); cnt[N + 1] = 0 so the exclusive scan's last element is the total
__global__ void __launch_bounds__(kTransposeThreads) eff_count_kernel(const int64_t* __restrict__ indptr, int64_t n_nodes,
                                                                int32_t with_self, int64_t* __restrict__ cnt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_nodes + 1) return;
  int64_t c = 0;
  if (i < n_nodes) {
    c = indptr[i + 1] - indptr[i];
    c = c > 0 ? c : 1;
  } else if (i == n_nodes) {
    c = 1;
  }
  cnt[i] = i <= n_nodes ? c + with_self : 0;
}

// one warp per effective row: its (destination, source row) pairs at its scanned slots, in CSR order, the self entry last.
// kSlots: the value is the slot itself, from which slot_rows_kernel derives both the source row and the entry offset.
template <bool kSlots>
__global__ void __launch_bounds__(kTransposeThreads) eff_fill_kernel(const int64_t* __restrict__ indptr,
                                                               const int32_t* __restrict__ indices, int64_t n_nodes,
                                                               int32_t with_self, const int64_t* __restrict__ slot,
                                                               int64_t cap, uint32_t* __restrict__ keys,
                                                               int32_t* __restrict__ vals) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kTransposeThreads / 32);
  for (int64_t i = (int64_t)blockIdx.x * (kTransposeThreads / 32) + (threadIdx.x >> 5); i <= n_nodes; i += warps) {
    const int64_t base = slot[i];
    int64_t c = 0, lo = 0;
    if (i < n_nodes) {
      lo = indptr[i];
      c = indptr[i + 1] - lo;
    }
    if (c > 0) {
      for (int64_t e = lane; e < c; e += 32) {
        int64_t d = indices[lo + e];
        d = (d < 0 || d > n_nodes) ? n_nodes : d;
        if (base + e < cap) {
          keys[base + e] = (uint32_t)d;
          vals[base + e] = kSlots ? (int32_t)(base + e) : (int32_t)i;
        }
      }
    } else if (lane == 0 && base < cap) {        // an empty row and the dummy row: {N}
      keys[base] = (uint32_t)n_nodes;
      vals[base] = kSlots ? (int32_t)base : (int32_t)i;
    }
    const int64_t at = base + (c > 0 ? c : 1);
    if (with_self && lane == 0 && at < cap) {
      keys[at] = (uint32_t)i;
      vals[at] = kSlots ? (int32_t)at : (int32_t)i;
    }
  }
}

// t_indptr[j] = #{sorted destinations < j}, j = 0 .. N + 1 (unused slots hold 0xFFFFFFFF and sort last)
__global__ void __launch_bounds__(kTransposeThreads) t_indptr_kernel(const uint32_t* __restrict__ keys, int64_t cap,
                                                               int64_t n_nodes, int64_t* __restrict__ t_indptr) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j > n_nodes + 1) return;
  int64_t lo = 0, hi = cap;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)keys[mid] < j) lo = mid + 1;
    else hi = mid;
  }
  t_indptr[j] = lo;
}

// after a kSlots sort: t_indices[k] holds the effective slot s of transposed entry k; write its source row i (the row
// whose scanned slots hold s) to t_indices[k] and its offset in that row to t_slot[k]: j for entry j of the row's CSR
// entries, -1 for the implicit {N} entry of an empty row or the dummy row, -2 for the with_self entry.  The unused tail
// holds slot 0, so it becomes row 0 as without t_slot.
__global__ void __launch_bounds__(kTransposeThreads) slot_rows_kernel(const int64_t* __restrict__ slot,
                                                                const int64_t* __restrict__ indptr, int64_t n_nodes,
                                                                int64_t cap, int32_t* __restrict__ t_indices,
                                                                int32_t* __restrict__ t_slot) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < cap; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = t_indices[k];
    int64_t lo = 0, hi = n_nodes;               // the last row i <= N with slot[i] <= s (every row has >= 1 entry)
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (slot[mid] <= s) lo = mid;
      else hi = mid - 1;
    }
    const int64_t j = s - slot[lo];
    const int64_t c = lo < n_nodes ? indptr[lo + 1] - indptr[lo] : 0;
    t_indices[k] = (int32_t)lo;
    t_slot[k] = j >= (c > 0 ? c : 1) ? -2 : c > 0 ? (int32_t)j : -1;
  }
}

static int32_t make_transpose_plan(int64_t n_nodes, int64_t nnz, int32_t with_self, TransposePlan& P, const char* who) {
  GS_REQUIRE(n_nodes >= 0 && n_nodes < 0x7fffffffLL - 2, "%s: n_nodes must be in [0, 2^31 - 2)", who);
  GS_REQUIRE(nnz >= 0 && (with_self == 0 || with_self == 1), "%s: bad nnz or with_self", who);
  P.rows = n_nodes + 1;
  P.cap = nnz + P.rows * (1 + with_self);
  GS_REQUIRE(P.cap < 0x7fffffffLL, "%s: nnz + (N + 1) * (1 + with_self) = %lld must be < 2^31", who, (long long)P.cap);
  P.end_bit = 1;
  while ((1LL << P.end_bit) <= P.rows) ++P.end_bit;          // 2^end_bit > N + 1: a sentinel's low bits exceed every id
  size_t scan_bytes = 0, sort_bytes = 0;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                        (int)(P.rows + 1));
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveSum (size query)");
  e = gs_cub::cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                              (const int32_t*)nullptr, (int32_t*)nullptr, (int)P.cap, 0, P.end_bit);
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceRadixSort::SortPairs (size query)");
  P.cub_bytes = std::max(scan_bytes, sort_bytes);
  size_t off = 0;
  P.off_cnt = off;  off += align256((size_t)(P.rows + 1) * 8);
  P.off_slot = off; off += align256((size_t)(P.rows + 1) * 8);
  P.off_kin = off;  off += align256((size_t)P.cap * 4);
  P.off_kout = off; off += align256((size_t)P.cap * 4);
  P.off_vin = off;  off += align256((size_t)P.cap * 4);
  P.off_cub = off;  off += align256(P.cub_bytes);
  P.bytes = off;
  return GS_OK;
}

// ---------------------------------------------------------------- max backward

struct BwdArgs {
  const float* z;  int64_t ldz;
  const float* m;  int64_t ldm;
  const float* dm; int64_t lddm;
  float* s;        int64_t lds;
  float* dz;       int64_t lddz;
  int32_t F;
  const int64_t* indptr;      // the phase's rows: the forward CSR (a) or its transpose (b)
  const int32_t* indices;
  int64_t n_nodes;            // N; the phase has N + 1 rows
  int32_t slices;             // ceil(F / 32)
  int64_t hub_items, hub_blocks;
  const float* w;             // kW only: one weight per entry of the phase's indices
};

// the max backward on the csr_rows.cuh schedule: the N + 1 rows of the phase, one column per lane, written up to F
template <int PHASE, bool kW = false>
struct MaxBackwardRows {
  static constexpr bool kFromFirst = false;
  static constexpr bool kEmptyIsDummy = false;     // row() already gives (a)'s empty rows their {N} entry
  const BwdArgs& a;

  struct Row {
    int64_t lo, cnt;
    bool dummy;
    float rv;                 // the row's fixed operand of the lane's column: m[i][c] (a) or z[j][c] (b)
  };

  __device__ __forceinline__ int64_t rows() const { return a.n_nodes + 1; }
  __device__ __forceinline__ int32_t hub_slices() const { return a.slices; }
  __device__ __forceinline__ int32_t slices() const { return a.slices; }
  __device__ __forceinline__ int32_t out_cols() const { return a.F; }

  // (a): the forward rows - an empty row and the dummy row N are {N} (cnt = 1, dummy); (b): the transposed rows, whose
  // entries are in range and may be none
  __device__ __forceinline__ Row row(int64_t i) const {
    Row r;
    r.lo = 0;
    r.cnt = 0;
    r.dummy = false;
    if (PHASE == 1 || i < a.n_nodes) {
      r.lo = __ldg(a.indptr + i);
      r.cnt = __ldg(a.indptr + i + 1) - r.lo;
      if (r.cnt < 0) r.cnt = 0;
    }
    if (PHASE == 0 && r.cnt == 0) {
      r.dummy = true;
      r.cnt = 1;
    }
    return r;
  }

  __device__ __forceinline__ void begin(Row& r, int64_t i, int c, bool col_ok) const {
    r.rv = col_ok ? (PHASE == 0 ? __ldg(a.m + i * a.ldm + c) : __ldg(a.z + i * a.ldz + c)) : 0.f;
  }

  __device__ __forceinline__ int64_t entry(const Row& r, int64_t e) const {
    if (PHASE == 0) {
      if (r.dummy) return a.n_nodes;
      const int64_t d = __ldg(a.indices + r.lo + e);
      return (d < 0 || d > a.n_nodes) ? a.n_nodes : d;
    }
    return __ldg(a.indices + r.lo + e);
  }

  // the term entry e adds: (a) 1 for a tie with the max; (b) s[k][c] where z[j][c] attains the max of forward row k
  // kW: the weighted term of (a), fl(w_e * z[k][c]) against m, and the routing of (b), fl(w_e * s) where fl(w_e * z) == m
  __device__ __forceinline__ float value(const Row& r, int64_t e, int c) const {
    const int64_t k = entry(r, e);
    if constexpr (kW) {
      const float w = (PHASE == 0 && r.dummy) ? 1.f : __ldg(a.w + r.lo + e);
      if (PHASE == 0) return __fmul_rn(w, __ldg(a.z + k * a.ldz + c)) == r.rv ? 1.f : 0.f;
      return __ldg(a.m + k * a.ldm + c) == __fmul_rn(w, r.rv) ? __fmul_rn(w, __ldg(a.s + k * a.lds + c)) : 0.f;
    }
    if (PHASE == 0) return __ldg(a.z + k * a.ldz + c) == r.rv ? 1.f : 0.f;
    return __ldg(a.m + k * a.ldm + c) == r.rv ? __ldg(a.s + k * a.lds + c) : 0.f;
  }

  __device__ __forceinline__ void load(const Row& r, int64_t e, int c, bool ok, float (&x)[1]) const {
    x[0] = ok ? value(r, e, c) : 0.f;
  }
  __device__ __forceinline__ void mask(const Row&, int64_t, int, float (&)[1]) const {}
  __device__ __forceinline__ float weight(const Row&, int64_t, bool) const { return 1.f; }
  __device__ __forceinline__ void scale(float, float (&)[1]) const {}
  __device__ __forceinline__ void hub_mask(const Row&, int64_t, int, float (&)[kHubPerWarp]) const {}
  __device__ __forceinline__ float step(float acc, float x) const { return acc + x; }
  __device__ __forceinline__ void finish(const Row&, int, int64_t, float (&)[1]) const {}

  __device__ __forceinline__ void store(const Row& r, int64_t i, int c, const float (&acc)[1]) const {
    if (PHASE == 0) a.s[i * a.lds + c] = __ldg(a.dm + i * a.lddm + c) / acc[0];
    else a.dz[i * a.lddz + c] = r.rv > 0.f ? acc[0] : 0.f;
  }
};

template <int PHASE, bool kW = false>
__global__ void __launch_bounds__(kCsrThreads, 3) csr_max_backward_kernel(const __grid_constant__ BwdArgs a) {
  __shared__ __align__(16) float tile[2][kHubRows][kHubCols];
  csr_rows<1, 8>(MaxBackwardRows<PHASE, kW>{a}, tile);
}

// gs_csr_max_backward, or with weights (w forward, t_w transposed) gs_csr_max_backward_weighted
static int32_t csr_max_backward(const float* z, int64_t ldz, const float* m, int64_t ldm, const float* dm, int64_t lddm,
                                int32_t F, const int64_t* indptr, const int32_t* indices, const float* w,
                                const int64_t* t_indptr, const int32_t* t_indices, const float* t_w, int64_t n_nodes,
                                float* s, int64_t lds, float* dz, int64_t lddz, void* stream, const char* who) {
  GS_REQUIRE(F >= 1 && n_nodes >= 0 && ldz >= F && ldm >= F && lddm >= F && lds >= F && lddz >= F, "%s: bad sizes", who);
  GS_REQUIRE(z && m && dm && s && dz && t_indptr && t_indices && (n_nodes == 0 || (indptr && indices)),
             "%s: NULL pointer", who);
  BwdArgs a{z, ldz, m, ldm, dm, lddm, s, lds, dz, lddz, F, indptr, indices, n_nodes, 0, 0, 0, w};
  a.slices = (F + kHubCols - 1) / kHubCols;
  const unsigned blocks = csr_grid(n_nodes + 1, a.slices, a.slices, a.hub_items, a.hub_blocks);
  cudaStream_t st = (cudaStream_t)stream;
  if (t_w) csr_max_backward_kernel<0, true><<<blocks, kCsrThreads, 0, st>>>(a);
  else csr_max_backward_kernel<0><<<blocks, kCsrThreads, 0, st>>>(a);         // (a) tie counts -> s
  int32_t rc = launch_check("csr_max_backward_kernel<0>");
  if (rc != GS_OK) return rc;
  a.indptr = t_indptr;
  a.indices = t_indices;
  a.w = t_w;
  if (t_w) csr_max_backward_kernel<1, true><<<blocks, kCsrThreads, 0, st>>>(a);
  else csr_max_backward_kernel<1><<<blocks, kCsrThreads, 0, st>>>(a);         // (b) masked sums over the transpose -> dz
  return launch_check("csr_max_backward_kernel<1>");
}

}  // namespace gs

extern "C" {

int64_t gs_csr_transpose_workspace_bytes(int64_t n_nodes, int64_t nnz, int32_t with_self) {
  gs::TransposePlan P;
  if (gs::make_transpose_plan(n_nodes, nnz, with_self, P, "gs_csr_transpose_workspace_bytes") != GS_OK) return -1;
  return (int64_t)P.bytes;
}

int32_t gs_csr_transpose(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz, int32_t with_self,
                         int64_t* t_indptr, int32_t* t_indices, int32_t* t_slot, void* workspace, int64_t workspace_bytes,
                         void* stream) {
  const char* who = "gs_csr_transpose";
  gs::TransposePlan P;
  int32_t rc = gs::make_transpose_plan(n_nodes, nnz, with_self, P, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(indptr && t_indptr && t_indices && (nnz == 0 || indices), "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)P.bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)P.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  int64_t* cnt = (int64_t*)(ws + P.off_cnt);
  int64_t* slot = (int64_t*)(ws + P.off_slot);
  uint32_t* kin = (uint32_t*)(ws + P.off_kin);
  uint32_t* kout = (uint32_t*)(ws + P.off_kout);
  int32_t* vin = (int32_t*)(ws + P.off_vin);
  const unsigned row_blocks = (unsigned)((P.rows + 1 + gs::kTransposeThreads - 1) / gs::kTransposeThreads);
  gs::eff_count_kernel<<<row_blocks, gs::kTransposeThreads, 0, st>>>(indptr, n_nodes, with_self, cnt);
  rc = gs::launch_check("eff_count_kernel");
  if (rc != GS_OK) return rc;
  size_t cub_bytes = P.cub_bytes;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(ws + P.off_cub, cub_bytes, (const int64_t*)cnt, slot,
                                                        (int)(P.rows + 1), st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceScan::ExclusiveSum");
  GS_CUDA(cudaMemsetAsync(kin, 0xFF, (size_t)P.cap * 4, st));       // unused slots: destination 0xFFFFFFFF, sorted last
  GS_CUDA(cudaMemsetAsync(vin, 0, (size_t)P.cap * 4, st));
  const int64_t fill_blocks = std::min<int64_t>((P.rows + 7) / 8, (int64_t)gs::sm_count() * 8 * 16);
  if (t_slot)
    gs::eff_fill_kernel<true><<<(unsigned)fill_blocks, gs::kTransposeThreads, 0, st>>>(indptr, indices, n_nodes, with_self, slot,
                                                                               P.cap, kin, vin);
  else
    gs::eff_fill_kernel<false><<<(unsigned)fill_blocks, gs::kTransposeThreads, 0, st>>>(indptr, indices, n_nodes, with_self, slot,
                                                                                P.cap, kin, vin);
  rc = gs::launch_check("eff_fill_kernel");
  if (rc != GS_OK) return rc;
  cub_bytes = P.cub_bytes;
  e = gs_cub::cub::DeviceRadixSort::SortPairs(ws + P.off_cub, cub_bytes, (const uint32_t*)kin, kout, (const int32_t*)vin,
                                              t_indices, (int)P.cap, 0, P.end_bit, st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceRadixSort::SortPairs");
  gs::t_indptr_kernel<<<row_blocks, gs::kTransposeThreads, 0, st>>>(kout, P.cap, n_nodes, t_indptr);
  rc = gs::launch_check("t_indptr_kernel");
  if (rc != GS_OK || !t_slot) return rc;
  const int64_t slot_blocks = std::min<int64_t>((P.cap + gs::kTransposeThreads - 1) / gs::kTransposeThreads, (int64_t)gs::sm_count() * 16);
  gs::slot_rows_kernel<<<(unsigned)slot_blocks, gs::kTransposeThreads, 0, st>>>(slot, indptr, n_nodes, P.cap, t_indices, t_slot);
  return gs::launch_check("slot_rows_kernel");
}

int32_t gs_csr_max_backward(const float* z, int64_t ldz, const float* m, int64_t ldm, const float* dm, int64_t lddm,
                            int32_t F, const int64_t* indptr, const int32_t* indices, const int64_t* t_indptr,
                            const int32_t* t_indices, int64_t n_nodes, float* s, int64_t lds, float* dz, int64_t lddz,
                            void* stream) {
  return gs::csr_max_backward(z, ldz, m, ldm, dm, lddm, F, indptr, indices, nullptr, t_indptr, t_indices, nullptr, n_nodes,
                              s, lds, dz, lddz, stream, "gs_csr_max_backward");
}

int32_t gs_csr_max_backward_weighted(const float* z, int64_t ldz, const float* m, int64_t ldm, const float* dm,
                                     int64_t lddm, int32_t F, const int64_t* indptr, const int32_t* indices,
                                     const float* weight, const int64_t* t_indptr, const int32_t* t_indices,
                                     const float* t_weight, int64_t n_nodes, float* s, int64_t lds, float* dz,
                                     int64_t lddz, void* stream) {
  const char* who = "gs_csr_max_backward_weighted";
  GS_REQUIRE(t_weight && (n_nodes == 0 || weight), "%s: NULL weight or t_weight", who);
  return gs::csr_max_backward(z, ldz, m, ldm, dm, lddm, F, indptr, indices, weight, t_indptr, t_indices, t_weight,
                              n_nodes, s, lds, dz, lddz, stream, who);
}

}  // extern "C"

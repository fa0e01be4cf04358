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
// Each output element of (a) and (b) is ONE sequential chain over its row's entries in order.  The two roles of
// gs_csr_aggregate share each launch: rows with more than kBwdLong entries (in-degree hubs of the transpose) go to hub
// CTAs, 32-column slices each, whose 8 warps stage 64 entries' terms in a double-buffered shared tile while warp 0 adds
// them in order; every other row gets one warp per 32-column slice with kBwdUnroll entries' loads in flight.
#include <algorithm>

#include "common.cuh"

#define CUB_WRAPPED_NAMESPACE gs_cub
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace gs {

constexpr int kBwdThreads = 256;
constexpr int64_t kBwdLong = 256;     // rows with more entries go to the hub role
constexpr int kBwdChunk = 256;        // rows scanned per hub work item (one per thread)
constexpr int kBwdCols = 32;          // columns per work item (one per lane)
constexpr int kBwdPerWarp = 8;        // entries each warp stages per hub round
constexpr int kBwdRows = kBwdPerWarp * (kBwdThreads / 32);   // entries per hub round: 64
constexpr int kBwdUnroll = 8;         // short role: entries' loads in flight per lane

static size_t bwd_align256(size_t x) { return (x + 255) & ~(size_t)255; }

// ---------------------------------------------------------------- transpose

struct TransposePlan {
  int64_t rows = 0, cap = 0;          // N + 1 effective rows; slots for their entries
  int end_bit = 1;
  size_t off_cnt = 0, off_slot = 0, off_kin = 0, off_kout = 0, off_vin = 0, off_cub = 0;
  size_t cub_bytes = 0, bytes = 0;
};

// cnt[i] = entries of effective row i (i <= N); cnt[N + 1] = 0 so the exclusive scan's last element is the total
__global__ void __launch_bounds__(kBwdThreads) eff_count_kernel(const int64_t* __restrict__ indptr, int64_t n_nodes,
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
__global__ void __launch_bounds__(kBwdThreads) eff_fill_kernel(const int64_t* __restrict__ indptr,
                                                               const int32_t* __restrict__ indices, int64_t n_nodes,
                                                               int32_t with_self, const int64_t* __restrict__ slot,
                                                               int64_t cap, uint32_t* __restrict__ keys,
                                                               int32_t* __restrict__ vals) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kBwdThreads / 32);
  for (int64_t i = (int64_t)blockIdx.x * (kBwdThreads / 32) + (threadIdx.x >> 5); i <= n_nodes; i += warps) {
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
__global__ void __launch_bounds__(kBwdThreads) t_indptr_kernel(const uint32_t* __restrict__ keys, int64_t cap,
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
__global__ void __launch_bounds__(kBwdThreads) slot_rows_kernel(const int64_t* __restrict__ slot,
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
  P.off_cnt = off;  off += bwd_align256((size_t)(P.rows + 1) * 8);
  P.off_slot = off; off += bwd_align256((size_t)(P.rows + 1) * 8);
  P.off_kin = off;  off += bwd_align256((size_t)P.cap * 4);
  P.off_kout = off; off += bwd_align256((size_t)P.cap * 4);
  P.off_vin = off;  off += bwd_align256((size_t)P.cap * 4);
  P.off_cub = off;  off += bwd_align256(P.cub_bytes);
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
};

// entry range of row i of the phase.  (a): the forward rows - an empty row and the dummy row N are {N} (cnt = 1, read
// through bwd_entry); (b): the transposed rows, N + 1 of them, whose entries are in range and may be none.
template <int PHASE>
__device__ __forceinline__ void bwd_row(const BwdArgs& a, int64_t i, int64_t& lo, int64_t& cnt, bool& dummy) {
  lo = 0;
  cnt = 0;
  dummy = false;
  if (PHASE == 1 || i < a.n_nodes) {
    lo = __ldg(a.indptr + i);
    cnt = __ldg(a.indptr + i + 1) - lo;
    if (cnt < 0) cnt = 0;
  }
  if (PHASE == 0 && cnt == 0) {
    dummy = true;
    cnt = 1;
  }
}

template <int PHASE>
__device__ __forceinline__ int64_t bwd_entry(const BwdArgs& a, int64_t lo, bool dummy, int64_t e) {
  if (PHASE == 0) {
    if (dummy) return a.n_nodes;
    const int64_t d = __ldg(a.indices + lo + e);
    return (d < 0 || d > a.n_nodes) ? a.n_nodes : d;
  }
  return __ldg(a.indices + lo + e);
}

// the row's fixed operand of column c: m[i][c] (a) or z[j][c] (b)
template <int PHASE>
__device__ __forceinline__ float bwd_row_value(const BwdArgs& a, int64_t i, int c) {
  return PHASE == 0 ? __ldg(a.m + i * a.ldm + c) : __ldg(a.z + i * a.ldz + c);
}

// the term entry r adds: (a) 1 for a tie with the max; (b) s[r][c] where z[j][c] attains row r's max
template <int PHASE>
__device__ __forceinline__ float bwd_term(const BwdArgs& a, int64_t r, int c, float rv) {
  if (PHASE == 0) return __ldg(a.z + r * a.ldz + c) == rv ? 1.f : 0.f;
  return __ldg(a.m + r * a.ldm + c) == rv ? __ldg(a.s + r * a.lds + c) : 0.f;
}

template <int PHASE>
__device__ __forceinline__ void bwd_store(const BwdArgs& a, int64_t i, int c, float acc, float rv) {
  if (PHASE == 0) a.s[i * a.lds + c] = __ldg(a.dm + i * a.lddm + c) / acc;
  else a.dz[i * a.lddz + c] = rv > 0.f ? acc : 0.f;
}

template <int PHASE>
__device__ void bwd_hub_role(const BwdArgs& a, float (*tile)[kBwdRows][kBwdCols]) {
  __shared__ int32_t list[kBwdChunk];
  __shared__ int32_t warp_count[kBwdThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t rows = a.n_nodes + 1;
  for (int64_t item = blockIdx.x; item < a.hub_items; item += a.hub_blocks) {
    const int64_t chunk = item / a.slices;
    const int c = (int)(item % a.slices) * kBwdCols + lane;
    const bool col_ok = c < a.F;
    const int64_t i0 = chunk * kBwdChunk + threadIdx.x;
    int64_t lo, cnt = 0;
    bool dummy;
    if (i0 < rows) bwd_row<PHASE>(a, i0, lo, cnt, dummy);
    const bool is_long = cnt > kBwdLong;
    const uint32_t ballot = __ballot_sync(0xffffffffu, is_long);
    if (lane == 0) warp_count[warp] = __popc(ballot);
    __syncthreads();
    int off = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kBwdThreads / 32; ++w) {
      off += w < warp ? warp_count[w] : 0;
      total += warp_count[w];
    }
    if (is_long) list[off + __popc(ballot & ((1u << lane) - 1u))] = (int32_t)threadIdx.x;
    __syncthreads();
    for (int q = 0; q < total; ++q) {
      const int64_t i = chunk * kBwdChunk + list[q];
      bwd_row<PHASE>(a, i, lo, cnt, dummy);
      const float rv = col_ok ? bwd_row_value<PHASE>(a, i, c) : 0.f;
      float r[kBwdPerWarp];
#pragma unroll
      for (int u = 0; u < kBwdPerWarp; ++u) {
        const int e = warp * kBwdPerWarp + u;                                   // cnt > kBwdRows
        r[u] = col_ok ? bwd_term<PHASE>(a, bwd_entry<PHASE>(a, lo, dummy, e), c, rv) : 0.f;
      }
      float acc = 0.f;
      int buf = 0;
      for (int64_t base = 0; base < cnt; base += kBwdRows, buf ^= 1) {
#pragma unroll
        for (int u = 0; u < kBwdPerWarp; ++u) tile[buf][warp * kBwdPerWarp + u][lane] = r[u];
        __syncthreads();
        const int64_t next = base + kBwdRows + warp * kBwdPerWarp;
#pragma unroll
        for (int u = 0; u < kBwdPerWarp; ++u)                 // the next round's loads are in flight during the sum
          r[u] = (col_ok && next + u < cnt) ? bwd_term<PHASE>(a, bwd_entry<PHASE>(a, lo, dummy, next + u), c, rv) : 0.f;
        if (warp == 0) {
          const int mm = (int)min((int64_t)kBwdRows, cnt - base);
          for (int t = 0; t < mm; ++t) acc += tile[buf][t][lane];
        }
      }
      if (warp == 0 && col_ok) bwd_store<PHASE>(a, i, c, acc, rv);
      __syncthreads();      // the tiles are reused by the next row
    }
    __syncthreads();        // `list` and `warp_count` are rewritten by the next item
  }
}

template <int PHASE>
__device__ void bwd_short_role(const BwdArgs& a, int64_t block) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t items = (a.n_nodes + 1) * a.slices;
  const int64_t stride = ((int64_t)gridDim.x - a.hub_blocks) * (kBwdThreads / 32);
  for (int64_t item = block * (kBwdThreads / 32) + warp; item < items; item += stride) {
    const int64_t i = item / a.slices;
    const int c = (int)(item % a.slices) * kBwdCols + lane;
    int64_t lo, cnt;
    bool dummy;
    bwd_row<PHASE>(a, i, lo, cnt, dummy);
    if (cnt > kBwdLong || c >= a.F) continue;        // a hub row (hub role), or past the last column
    const float rv = bwd_row_value<PHASE>(a, i, c);
    float acc = 0.f;
    for (int64_t e = 0; e < cnt; e += kBwdUnroll) {
      float x[kBwdUnroll];
#pragma unroll
      for (int u = 0; u < kBwdUnroll; ++u)
        x[u] = e + u < cnt ? bwd_term<PHASE>(a, bwd_entry<PHASE>(a, lo, dummy, e + u), c, rv) : 0.f;
#pragma unroll
      for (int u = 0; u < kBwdUnroll; ++u)
        if (e + u < cnt) acc += x[u];
    }
    bwd_store<PHASE>(a, i, c, acc, rv);
  }
}

template <int PHASE>
__global__ void __launch_bounds__(kBwdThreads, 3) csr_max_backward_kernel(const __grid_constant__ BwdArgs a) {
  __shared__ __align__(16) float tile[2][kBwdRows][kBwdCols];
  if (blockIdx.x < a.hub_blocks) bwd_hub_role<PHASE>(a, tile);
  else bwd_short_role<PHASE>(a, (int64_t)blockIdx.x - a.hub_blocks);
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
  const unsigned row_blocks = (unsigned)((P.rows + 1 + gs::kBwdThreads - 1) / gs::kBwdThreads);
  gs::eff_count_kernel<<<row_blocks, gs::kBwdThreads, 0, st>>>(indptr, n_nodes, with_self, cnt);
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
    gs::eff_fill_kernel<true><<<(unsigned)fill_blocks, gs::kBwdThreads, 0, st>>>(indptr, indices, n_nodes, with_self, slot,
                                                                               P.cap, kin, vin);
  else
    gs::eff_fill_kernel<false><<<(unsigned)fill_blocks, gs::kBwdThreads, 0, st>>>(indptr, indices, n_nodes, with_self, slot,
                                                                                P.cap, kin, vin);
  rc = gs::launch_check("eff_fill_kernel");
  if (rc != GS_OK) return rc;
  cub_bytes = P.cub_bytes;
  e = gs_cub::cub::DeviceRadixSort::SortPairs(ws + P.off_cub, cub_bytes, (const uint32_t*)kin, kout, (const int32_t*)vin,
                                              t_indices, (int)P.cap, 0, P.end_bit, st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceRadixSort::SortPairs");
  gs::t_indptr_kernel<<<row_blocks, gs::kBwdThreads, 0, st>>>(kout, P.cap, n_nodes, t_indptr);
  rc = gs::launch_check("t_indptr_kernel");
  if (rc != GS_OK || !t_slot) return rc;
  const int64_t slot_blocks = std::min<int64_t>((P.cap + gs::kBwdThreads - 1) / gs::kBwdThreads, (int64_t)gs::sm_count() * 16);
  gs::slot_rows_kernel<<<(unsigned)slot_blocks, gs::kBwdThreads, 0, st>>>(slot, indptr, n_nodes, P.cap, t_indices, t_slot);
  return gs::launch_check("slot_rows_kernel");
}

int32_t gs_csr_max_backward(const float* z, int64_t ldz, const float* m, int64_t ldm, const float* dm, int64_t lddm,
                            int32_t F, const int64_t* indptr, const int32_t* indices, const int64_t* t_indptr,
                            const int32_t* t_indices, int64_t n_nodes, float* s, int64_t lds, float* dz, int64_t lddz,
                            void* stream) {
  const char* who = "gs_csr_max_backward";
  GS_REQUIRE(F >= 1 && n_nodes >= 0 && ldz >= F && ldm >= F && lddm >= F && lds >= F && lddz >= F, "%s: bad sizes", who);
  GS_REQUIRE(z && m && dm && s && dz && t_indptr && t_indices && (n_nodes == 0 || (indptr && indices)),
             "%s: NULL pointer", who);
  gs::BwdArgs a{z, ldz, m, ldm, dm, lddm, s, lds, dz, lddz, F, indptr, indices, n_nodes, 0, 0, 0};
  a.slices = (F + gs::kBwdCols - 1) / gs::kBwdCols;
  const int64_t rows = n_nodes + 1;
  a.hub_items = (rows + gs::kBwdChunk - 1) / gs::kBwdChunk * a.slices;
  a.hub_blocks = std::min<int64_t>(a.hub_items, (int64_t)gs::sm_count() * 4);
  const int64_t short_blocks = std::min<int64_t>((rows * a.slices + 7) / 8, (int64_t)gs::sm_count() * 8 * 64);
  const unsigned blocks = (unsigned)(a.hub_blocks + short_blocks);
  cudaStream_t st = (cudaStream_t)stream;
  gs::csr_max_backward_kernel<0><<<blocks, gs::kBwdThreads, 0, st>>>(a);       // (a) tie counts -> s
  int32_t rc = gs::launch_check("csr_max_backward_kernel<0>");
  if (rc != GS_OK) return rc;
  a.indptr = t_indptr;
  a.indices = t_indices;
  gs::csr_max_backward_kernel<1><<<blocks, gs::kBwdThreads, 0, st>>>(a);       // (b) masked sums over the transpose -> dz
  return gs::launch_check("csr_max_backward_kernel<1>");
}

}  // extern "C"

// Random-walk co-occurrence pairs (reference graphsage/utils.py:77-92, run_random_walks), contract in oracle/walks.py.
//   random_walk_kernel   one thread per walk: the walk's visited ids (start excluded) into a column-major [L-1, walks]
//                        buffer and its pair count into counts[walk]
//   (CUB exclusive scan) counts -> int64 offsets; offsets[walks] is the pair count
//   walk_emit_kernel     one thread per walk: copies its visited ids to out[offsets[walk] + j] = (start, visited)
// The visited ids are stored rather than recomputed in the emit pass: a walk is L - 1 dependent pairs of random reads
// (the indptr pair, then one indices entry), while storing it costs 4 (L - 1) coalesced bytes per walk written once and
// read once - far less than repeating the gather chain.
// node2vec's second-order (p, q) walk (contract in oracle/biased_walks.py) reuses the plan, the scan and the emit pass:
//   gs_csr_sort_rows        a copy of indices sorted within each row (CUB segmented sort): the membership test's input
//   biased_walk_kernel      one thread per walk, as random_walk_kernel; each move after the first draws a candidate
//                           uniformly from the current row and accepts it with probability thr(class) / 2^32, the class
//                           ("is x an entry of the previous node's row") found by binary search in the sorted copy
#include "common.cuh"

#define CUB_WRAPPED_NAMESPACE gs_cub
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

namespace gs {

constexpr int kWalkThreads = 256;

struct WalkPlan {
  int64_t walks = 0;                 // n * num_walks
  size_t off_visited = 0, off_counts = 0, off_offsets = 0, off_cub = 0;
  size_t cub_bytes = 0, bytes = 0;
};

// Walk g = t * num_walks + w starts at starts[t] (global start position i = start_offset + t).  Draw s of the walk is
// word s % 4 of philox4x32_10((counter_lo, counter_hi, i, kStreamWalk + w * nblk + s / 4), seed), nblk = ceil((L-1)/4).
__global__ void __launch_bounds__(kWalkThreads, 8) random_walk_kernel(const int64_t* __restrict__ indptr,
                                                                      const int32_t* __restrict__ indices, int64_t n_nodes,
                                                                      const int32_t* __restrict__ starts, int64_t walks,
                                                                      int32_t num_walks, int32_t walk_len, uint64_t seed,
                                                                      uint64_t counter, int64_t start_offset,
                                                                      int32_t* __restrict__ visited,
                                                                      uint8_t* __restrict__ counts) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g == 0) counts[walks] = 0;                     // the scan's extra element: offsets[walks] becomes the total
  if (g >= walks) return;
  const int64_t t = g / num_walks;
  const uint32_t w = (uint32_t)(g - t * num_walks);
  const int32_t node = starts[t];
  int cnt = 0;
  if (node >= 0 && node < n_nodes) {
    const uint32_t nblk = (uint32_t)(walk_len + 2) >> 2;           // ceil((L - 1) / 4)
    const uint32_t i = (uint32_t)(start_offset + t);
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    int64_t curr = node;
    u32x4 r{0, 0, 0, 0};
    // step j: emit curr unless it is the start, then move on with draw j (the L-th move of the reference is never used)
    for (int j = 0; j < walk_len; ++j) {
      if (curr != node) visited[(int64_t)cnt++ * walks + g] = (int32_t)curr;
      if (j == walk_len - 1) break;
      if (curr < 0 || curr >= n_nodes) break;      // an out-of-range neighbour id has no neighbours
      const int64_t row = indptr[curr];
      const int64_t deg = indptr[curr + 1] - row;
      if (deg <= 0) break;                         // a start without neighbours emits nothing; a sink ends the walk
      if ((j & 3) == 0) {
        u32x4 c{(uint32_t)counter, (uint32_t)(counter >> 32), i, kStreamWalk + w * nblk + (uint32_t)(j >> 2)};
        r = philox4x32_10(c, k0, k1);
      }
      curr = indices[row + (int64_t)mulhi32(pick(r, j & 3), (uint32_t)deg)];
    }
  }
  counts[g] = (uint8_t)cnt;
}

__global__ void __launch_bounds__(kWalkThreads) walk_emit_kernel(const int32_t* __restrict__ starts, int64_t walks,
                                                                 int32_t num_walks, const int32_t* __restrict__ visited,
                                                                 const uint8_t* __restrict__ counts,
                                                                 const int64_t* __restrict__ offsets,
                                                                 int32_t* __restrict__ out) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= walks) return;
  const int cnt = counts[g];
  if (cnt == 0) return;
  const int32_t node = starts[g / num_walks];
  int2* dst = reinterpret_cast<int2*>(out) + offsets[g];
  for (int j = 0; j < cnt; ++j) dst[j] = make_int2(node, visited[(int64_t)j * walks + g]);
}

// ---- the biased walk ----------------------------------------------------------------------------------------------
struct WalkBias {
  uint64_t ret, in, out;  // thr of the return / in / out classes, each in [1, 2^32]
  uint64_t lo, hi;        // min and max of (in, out): an acceptance word below lo accepts and one at or above hi rejects
                          // any candidate other than t without the membership search
};

// is x an entry of sorted[lo, lo + n)?  The last entry <= x, by a halving search with no early exit.
__device__ __forceinline__ bool row_has(const int32_t* __restrict__ sorted, int64_t lo, uint32_t n, int32_t x) {
  if (n == 0) return false;
  while (n > 1) {
    const uint32_t h = n >> 1;
    if (__ldg(sorted + lo + h) <= x) lo += h;
    n -= h;
  }
  return __ldg(sorted + lo) == x;
}

// thr of candidate x from current node v reached from t (t's sorted row at [trow, trow + tdeg))
__device__ __forceinline__ uint64_t class_thr(const WalkBias& b, const int32_t* __restrict__ sorted, int64_t t,
                                              int64_t trow, uint32_t tdeg, int32_t x) {
  if (x == t) return b.ret;
  return row_has(sorted, trow, tdeg, x) ? b.in : b.out;
}

__device__ __forceinline__ bool accept(const WalkBias& b, const int32_t* __restrict__ sorted, int64_t t, int64_t trow,
                                       uint32_t tdeg, int32_t x, uint32_t acc) {
  if (x == t) return acc < b.ret;
  if (acc < b.lo) return true;
  if (acc >= b.hi) return false;
  return acc < (row_has(sorted, trow, tdeg, x) ? b.in : b.out);
}

// Walk g = t * num_walks + w as random_walk_kernel; move s draws from philox4x32_10((counter_lo, counter_hi, i,
// kStreamWalkBiased + ((w * 32 + s) << 3) + call), seed): call 0 word 0 is the first move's pick; from s = 1, calls 0..6
// are attempts (cand, acc, cand, acc) and call 7's words 0, 1 are the fallback's u (oracle/biased_walks.py).
__global__ void __launch_bounds__(kWalkThreads) biased_walk_kernel(
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const int32_t* __restrict__ sorted,
    int64_t n_nodes, const int32_t* __restrict__ starts, int64_t walks, int32_t num_walks, int32_t walk_len, WalkBias b,
    uint64_t seed, uint64_t counter, int64_t start_offset, int32_t* __restrict__ visited, uint8_t* __restrict__ counts) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g == 0) counts[walks] = 0;
  if (g >= walks) return;
  const int64_t t = g / num_walks;
  const uint32_t w = (uint32_t)(g - t * num_walks);
  const int32_t node = starts[t];
  int cnt = 0;
  if (node >= 0 && node < n_nodes) {
    const uint32_t i = (uint32_t)(start_offset + t);
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    int64_t curr = node, prev = -1, prow = 0;    // prev's row [prow, prow + pdeg) stays in registers for the next move
    uint32_t pdeg = 0;
    for (int j = 0; j < walk_len; ++j) {
      if (curr != node) visited[(int64_t)cnt++ * walks + g] = (int32_t)curr;
      if (j == walk_len - 1) break;
      if (curr < 0 || curr >= n_nodes) break;
      const int64_t row = indptr[curr];
      const int64_t deg64 = indptr[curr + 1] - row;
      if (deg64 <= 0) break;
      const uint32_t deg = (uint32_t)deg64;
      const uint32_t tag = kStreamWalkBiased + ((w * 32u + (uint32_t)j) << 3);
      u32x4 c{(uint32_t)counter, (uint32_t)(counter >> 32), i, tag};
      int32_t nxt = 0;
      bool done = false;
      if (j == 0) {
        nxt = indices[row + (int64_t)mulhi32(philox4x32_10(c, k0, k1).x, deg)];
        done = true;
      }
      for (uint32_t call = 0; !done && call < GS_WALK_BIASED_ATTEMPTS / 2; ++call) {
        c.w = tag + call;
        const u32x4 r = philox4x32_10(c, k0, k1);
        nxt = indices[row + (int64_t)mulhi32(r.x, deg)];
        done = accept(b, sorted, prev, prow, pdeg, nxt, r.y);
        if (!done) {
          nxt = indices[row + (int64_t)mulhi32(r.z, deg)];
          done = accept(b, sorted, prev, prow, pdeg, nxt, r.w);
        }
      }
      if (!done) {                               // exact inverse-CDF draw over the row: target = floor(u * S / 2^64)
        c.w = tag + 7u;
        const u32x4 r = philox4x32_10(c, k0, k1);
        const uint64_t u = (uint64_t)r.x | ((uint64_t)r.y << 32);
        uint64_t total = 0;
        for (uint32_t k = 0; k < deg; ++k) total += class_thr(b, sorted, prev, prow, pdeg, indices[row + k]);
        const uint64_t target = __umul64hi(u, total);
        uint64_t acc = 0;
        for (uint32_t k = 0; k < deg; ++k) {
          nxt = indices[row + k];
          acc += class_thr(b, sorted, prev, prow, pdeg, nxt);
          if (acc > target) break;
        }
      }
      prev = curr;
      prow = row;
      pdeg = deg;
      curr = nxt;
    }
  }
  counts[g] = (uint8_t)cnt;
}

// float64, as oracle/biased_walks.py:thresholds
static WalkBias make_walk_bias(double p, double q) {
  const double a[3] = {1.0 / p, 1.0, 1.0 / q};
  const double amax = fmax(a[0], fmax(a[1], a[2]));
  uint64_t thr[3];
  for (int c = 0; c < 3; ++c) thr[c] = a[c] == amax ? (1ull << 32) : (uint64_t)floor(a[c] / amax * 4294967296.0);
  WalkBias b;
  b.ret = thr[0];
  b.in = thr[1];
  b.out = thr[2];
  b.lo = thr[1] < thr[2] ? thr[1] : thr[2];
  b.hi = thr[1] < thr[2] ? thr[2] : thr[1];
  return b;
}

static int32_t make_walk_plan(int64_t n, int32_t num_walks, int32_t walk_len, WalkPlan& P, const char* who) {
  GS_REQUIRE(n >= 0, "%s: n must be >= 0 (got %lld)", who, (long long)n);
  GS_REQUIRE(num_walks >= 1 && num_walks <= GS_WALK_MAX_WALKS, "%s: num_walks must be in [1, %d] (got %d)", who,
             GS_WALK_MAX_WALKS, num_walks);
  GS_REQUIRE(walk_len >= 2 && walk_len <= GS_WALK_MAX_LEN, "%s: walk_len must be in [2, %d] (got %d)", who,
             GS_WALK_MAX_LEN, walk_len);
  P.walks = n * (int64_t)num_walks;
  GS_REQUIRE(P.walks < 0x7fffffffLL, "%s: n * num_walks = %lld must be < 2^31 - 1 (walk the starts in chunks)", who,
             (long long)P.walks);
  if (P.walks == 0) return GS_OK;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveScan(nullptr, P.cub_bytes, (const uint8_t*)nullptr,
                                                         (int64_t*)nullptr, ::cuda::std::plus<>{}, (int64_t)0,
                                                         (int)(P.walks + 1));
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveScan (size query)");
  size_t off = 0;
  P.off_visited = off; off += align256((size_t)P.walks * (size_t)(walk_len - 1) * 4);
  P.off_counts = off;  off += align256((size_t)P.walks + 1);
  P.off_offsets = off; off += align256(((size_t)P.walks + 1) * 8);
  P.off_cub = off;     off += align256(P.cub_bytes);
  P.bytes = off;
  return GS_OK;
}

// the per-walk counts -> int64 offsets (offsets[walks] = P), and P to the device word n_pairs
static int32_t scan_walk_counts(const WalkPlan& P, char* ws, int64_t* n_pairs, cudaStream_t st) {
  const uint8_t* counts = (const uint8_t*)(ws + P.off_counts);
  int64_t* offsets = (int64_t*)(ws + P.off_offsets);
  size_t cub_bytes = P.cub_bytes;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveScan(ws + P.off_cub, cub_bytes, counts, offsets,
                                                         ::cuda::std::plus<>{}, (int64_t)0, (int)(P.walks + 1), st);
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveScan");
  GS_CUDA(cudaMemcpyAsync(n_pairs, offsets + P.walks, 8, cudaMemcpyDeviceToDevice, st));
  return GS_OK;
}

static int32_t sort_rows_bytes(int64_t n_nodes, int64_t nnz, size_t& bytes, const char* who) {
  GS_REQUIRE(n_nodes >= 0 && n_nodes < 0x7fffffffLL, "%s: n_nodes must be in [0, 2^31 - 1) (got %lld)", who,
             (long long)n_nodes);
  GS_REQUIRE(nnz >= 0 && nnz < 0x7fffffffLL, "%s: nnz must be in [0, 2^31 - 1) (got %lld)", who, (long long)nnz);
  bytes = 0;
  if (n_nodes == 0 || nnz == 0) return GS_OK;
  cudaError_t e = gs_cub::cub::DeviceSegmentedSort::SortKeys(nullptr, bytes, (const int32_t*)nullptr, (int32_t*)nullptr,
                                                             (int)nnz, (int)n_nodes, (const int64_t*)nullptr,
                                                             (const int64_t*)nullptr);
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceSegmentedSort::SortKeys (size query)");
  bytes = align256(bytes);
  return GS_OK;
}

}  // namespace gs

extern "C" {

int64_t gs_csr_sort_rows_workspace_bytes(int64_t n_nodes, int64_t nnz) {
  size_t bytes = 0;
  if (gs::sort_rows_bytes(n_nodes, nnz, bytes, "gs_csr_sort_rows_workspace_bytes") != GS_OK) return -1;
  return (int64_t)bytes;
}

int32_t gs_csr_sort_rows(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                         int32_t* sorted_indices, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "gs_csr_sort_rows";
  size_t bytes = 0;
  int32_t rc = gs::sort_rows_bytes(n_nodes, nnz, bytes, who);
  if (rc != GS_OK) return rc;
  if (nnz == 0) return GS_OK;
  GS_REQUIRE(indptr && indices && sorted_indices, "%s: NULL pointer", who);
  cudaStream_t st = (cudaStream_t)stream;
  // entries outside every row, and rows CUB leaves alone (one entry), keep their bytes
  GS_CUDA(cudaMemcpyAsync(sorted_indices, indices, (size_t)nnz * 4, cudaMemcpyDeviceToDevice, st));
  if (n_nodes == 0) return GS_OK;
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)bytes);
  cudaError_t e = gs_cub::cub::DeviceSegmentedSort::SortKeys(workspace, bytes, indices, sorted_indices, (int)nnz,
                                                             (int)n_nodes, indptr, indptr + 1, st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceSegmentedSort::SortKeys");
  return GS_OK;
}

int64_t gs_random_walks_workspace_bytes(int64_t n, int32_t num_walks, int32_t walk_len) {
  gs::WalkPlan P;
  if (gs::make_walk_plan(n, num_walks, walk_len, P, "gs_random_walks_workspace_bytes") != GS_OK) return -1;
  return (int64_t)P.bytes;
}

int32_t gs_random_walks(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, const int32_t* starts, int64_t n,
                        int32_t num_walks, int32_t walk_len, uint64_t seed, uint64_t counter, int64_t start_offset,
                        void* workspace, int64_t workspace_bytes, int64_t* n_pairs, void* stream) {
  const char* who = "gs_random_walks";
  gs::WalkPlan P;
  int32_t rc = gs::make_walk_plan(n, num_walks, walk_len, P, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(n_nodes >= 0 && n_nodes < 0x7fffffffLL, "%s: n_nodes must be in [0, 2^31 - 1)", who);
  GS_REQUIRE(start_offset >= 0 && start_offset + n <= (1LL << 32),
             "%s: start_offset + n must be <= 2^32 (start positions are a 32-bit counter word)", who);
  GS_REQUIRE(n_pairs != nullptr, "%s: n_pairs is NULL", who);
  cudaStream_t st = (cudaStream_t)stream;
  if (P.walks == 0) {
    GS_CUDA(cudaMemsetAsync(n_pairs, 0, 8, st));
    return GS_OK;
  }
  GS_REQUIRE(indptr && indices && starts, "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)P.bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)P.bytes);
  char* ws = (char*)workspace;
  int32_t* visited = (int32_t*)(ws + P.off_visited);
  uint8_t* counts = (uint8_t*)(ws + P.off_counts);
  const int64_t blocks = (P.walks + gs::kWalkThreads - 1) / gs::kWalkThreads;
  gs::random_walk_kernel<<<(unsigned)blocks, gs::kWalkThreads, 0, st>>>(indptr, indices, n_nodes, starts, P.walks,
                                                                        num_walks, walk_len, seed, counter, start_offset,
                                                                        visited, counts);
  rc = gs::launch_check("random_walk_kernel");
  if (rc != GS_OK) return rc;
  return gs::scan_walk_counts(P, ws, n_pairs, st);
}

int32_t gs_random_walks_biased(const int64_t* indptr, const int32_t* indices, const int32_t* sorted_indices,
                               int64_t n_nodes, const int32_t* starts, int64_t n, int32_t num_walks, int32_t walk_len,
                               double p, double q, uint64_t seed, uint64_t counter, int64_t start_offset, void* workspace,
                               int64_t workspace_bytes, int64_t* n_pairs, void* stream) {
  const char* who = "gs_random_walks_biased";
  GS_REQUIRE(isfinite(p) && p >= GS_WALK_PQ_MIN && p <= GS_WALK_PQ_MAX, "%s: p must be finite and in [%g, %g] (got %g)",
             who, GS_WALK_PQ_MIN, GS_WALK_PQ_MAX, p);
  GS_REQUIRE(isfinite(q) && q >= GS_WALK_PQ_MIN && q <= GS_WALK_PQ_MAX, "%s: q must be finite and in [%g, %g] (got %g)",
             who, GS_WALK_PQ_MIN, GS_WALK_PQ_MAX, q);
  if (p == 1.0 && q == 1.0)
    return gs_random_walks(indptr, indices, n_nodes, starts, n, num_walks, walk_len, seed, counter, start_offset,
                           workspace, workspace_bytes, n_pairs, stream);
  gs::WalkPlan P;
  int32_t rc = gs::make_walk_plan(n, num_walks, walk_len, P, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(n_nodes >= 0 && n_nodes < 0x7fffffffLL, "%s: n_nodes must be in [0, 2^31 - 1)", who);
  GS_REQUIRE(start_offset >= 0 && start_offset + n <= (1LL << 32),
             "%s: start_offset + n must be <= 2^32 (start positions are a 32-bit counter word)", who);
  GS_REQUIRE(n_pairs != nullptr, "%s: n_pairs is NULL", who);
  cudaStream_t st = (cudaStream_t)stream;
  if (P.walks == 0) {
    GS_CUDA(cudaMemsetAsync(n_pairs, 0, 8, st));
    return GS_OK;
  }
  GS_REQUIRE(indptr && indices && sorted_indices && starts, "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)P.bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)P.bytes);
  char* ws = (char*)workspace;
  const int64_t blocks = (P.walks + gs::kWalkThreads - 1) / gs::kWalkThreads;
  gs::biased_walk_kernel<<<(unsigned)blocks, gs::kWalkThreads, 0, st>>>(
      indptr, indices, sorted_indices, n_nodes, starts, P.walks, num_walks, walk_len, gs::make_walk_bias(p, q), seed,
      counter, start_offset, (int32_t*)(ws + P.off_visited), (uint8_t*)(ws + P.off_counts));
  rc = gs::launch_check("biased_walk_kernel");
  if (rc != GS_OK) return rc;
  return gs::scan_walk_counts(P, ws, n_pairs, st);
}

int32_t gs_random_walks_emit(const int32_t* starts, int64_t n, int32_t num_walks, int32_t walk_len, const void* workspace,
                             int64_t workspace_bytes, int32_t* out, void* stream) {
  const char* who = "gs_random_walks_emit";
  gs::WalkPlan P;
  int32_t rc = gs::make_walk_plan(n, num_walks, walk_len, P, who);
  if (rc != GS_OK) return rc;
  if (P.walks == 0) return GS_OK;
  GS_REQUIRE(starts && workspace && workspace_bytes >= (int64_t)P.bytes, "%s: NULL pointer or short workspace", who);
  const char* ws = (const char*)workspace;
  const int64_t blocks = (P.walks + gs::kWalkThreads - 1) / gs::kWalkThreads;
  gs::walk_emit_kernel<<<(unsigned)blocks, gs::kWalkThreads, 0, (cudaStream_t)stream>>>(
      starts, P.walks, num_walks, (const int32_t*)(ws + P.off_visited), (const uint8_t*)(ws + P.off_counts),
      (const int64_t*)(ws + P.off_offsets), out);
  return gs::launch_check("walk_emit_kernel");
}

}  // extern "C"

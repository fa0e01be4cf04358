// Random-walk co-occurrence pairs (reference graphsage/utils.py:77-92, run_random_walks), contract in oracle/walks.py.
//   random_walk_kernel   one thread per walk: the walk's visited ids (start excluded) into a column-major [L-1, walks]
//                        buffer and its pair count into counts[walk]
//   (CUB exclusive scan) counts -> int64 offsets; offsets[walks] is the pair count
//   walk_emit_kernel     one thread per walk: copies its visited ids to out[offsets[walk] + j] = (start, visited)
// The visited ids are stored rather than recomputed in the emit pass: a walk is L - 1 dependent pairs of random reads
// (the indptr pair, then one indices entry), while storing it costs 4 (L - 1) coalesced bytes per walk written once and
// read once - far less than repeating the gather chain.
#include "common.cuh"

#define CUB_WRAPPED_NAMESPACE gs_cub
#include <cub/device/device_scan.cuh>

namespace gs {

constexpr int kWalkThreads = 256;

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

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

}  // namespace gs

extern "C" {

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
  int64_t* offsets = (int64_t*)(ws + P.off_offsets);
  const int64_t blocks = (P.walks + gs::kWalkThreads - 1) / gs::kWalkThreads;
  gs::random_walk_kernel<<<(unsigned)blocks, gs::kWalkThreads, 0, st>>>(indptr, indices, n_nodes, starts, P.walks,
                                                                        num_walks, walk_len, seed, counter, start_offset,
                                                                        visited, counts);
  rc = gs::launch_check("random_walk_kernel");
  if (rc != GS_OK) return rc;
  size_t cub_bytes = P.cub_bytes;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveScan(ws + P.off_cub, cub_bytes, (const uint8_t*)counts, offsets,
                                                         ::cuda::std::plus<>{}, (int64_t)0, (int)(P.walks + 1), st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceScan::ExclusiveScan");
  GS_CUDA(cudaMemcpyAsync(n_pairs, offsets + P.walks, 8, cudaMemcpyDeviceToDevice, st));
  return GS_OK;
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

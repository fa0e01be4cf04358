// Per-layer receptive-field blocks of a minibatch over whole neighbourhoods (full_neighbor_minibatch_*; contract in
// oracle/full_neighbor_blocks.py).  Two entry points sharing one workspace:
//   gs_csr_blocks_plan  device only.  Level L is the seed set; then for l = L-1 .. 0: clear a [N+2] flag array, mark
//                       V_{l+1}, every (clamped) entry of its rows and N (one warp per node, idempotent stores: a hub
//                       row's entries spread over 32 lanes), CUB exclusive scan -> the position map pos_l [N+2]
//                       (pos_l[N+1] = |V_l|), compact V_l in ascending order, and sum V_{l+1}'s degrees (CUB reduce,
//                       integer) -> the block's entry count.  The kernels read |V_{l+1}| from its device word and
//                       grid-stride over a capacity, so nothing returns to the host between layers; the 2L counts land
//                       in one small device array for the caller's single read.
//   gs_csr_blocks_fill  with the host-known sizes: per block, src_ids (a copy of V_l), indptr (V_{l+1} members' degrees
//                       at their local positions, zero elsewhere, CUB exclusive scan), indices (one warp per local row,
//                       entries in CSR order relabelled through pos_l) and rows.
// Integer work only and no atomics: two calls give the same bytes.
#include <algorithm>

#include "common.cuh"

#define CUB_WRAPPED_NAMESPACE gs_cub
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

namespace gs {

constexpr int kBlkThreads = 256;
constexpr int kBlkWarps = kBlkThreads / 32;

struct BlocksPlan {
  int64_t n_nodes = 0, cap = 0;       // N; cap = N + 2 (the flags, positions and degrees of nodes 0 .. N, plus a 0)
  int32_t levels = 0;                 // L + 1: level l < L is V_l, level L the distinct seeds
  size_t off_flag = 0, off_pos = 0, off_ids = 0, off_deg = 0, off_cub = 0;
  size_t cub_bytes = 0, bytes = 0;
};

__device__ __forceinline__ int64_t blk_clamp(int64_t v, int64_t n_nodes) { return (v < 0 || v >= n_nodes) ? n_nodes : v; }

// the raw CSR row of node v < N: [lo, lo + cnt), cnt >= 0
__device__ __forceinline__ void blk_row(const int64_t* __restrict__ indptr, int64_t v, int64_t& lo, int64_t& cnt) {
  lo = indptr[v];
  cnt = indptr[v + 1] - lo;
  if (cnt < 0) cnt = 0;
}

// the i-th node of level l + 1: the clamped seed (level L is built from the seeds) or V_{l+1}[i]
__device__ __forceinline__ int64_t blk_node(const int32_t* __restrict__ seeds, const int32_t* __restrict__ ids, int64_t i,
                                            int64_t n_nodes) {
  return seeds ? blk_clamp(seeds[i], n_nodes) : (int64_t)ids[i];
}

// one warp per node of the previous level (count: *count_dev, or n when count_dev is NULL): flag the node and, with
// expand, its row's clamped entries; the dummy N too with expand.  Stores of 1 only: the order of racing stores is moot.
__global__ void __launch_bounds__(kBlkThreads) blk_mark_kernel(const int64_t* __restrict__ indptr,
                                                               const int32_t* __restrict__ indices, int64_t n_nodes,
                                                               const int32_t* __restrict__ seeds,
                                                               const int32_t* __restrict__ ids,
                                                               const int32_t* __restrict__ count_dev, int64_t n,
                                                               int32_t expand, int32_t* __restrict__ flag) {
  const int lane = threadIdx.x & 31;
  const int64_t count = count_dev ? (int64_t)*count_dev : n;
  const int64_t warps = (int64_t)gridDim.x * kBlkWarps;
  if (expand && blockIdx.x == 0 && threadIdx.x == 0) flag[n_nodes] = 1;
  for (int64_t i = (int64_t)blockIdx.x * kBlkWarps + (threadIdx.x >> 5); i < count; i += warps) {
    const int64_t v = blk_node(seeds, ids, i, n_nodes);
    if (lane == 0) flag[v] = 1;
    if (!expand || v >= n_nodes) continue;
    int64_t lo, cnt;
    blk_row(indptr, v, lo, cnt);
    for (int64_t e = lane; e < cnt; e += 32) flag[blk_clamp(indices[lo + e], n_nodes)] = 1;
  }
}

// ids[pos[v]] = v for every flagged v (pos[v + 1] - pos[v] is v's flag), ascending
__global__ void __launch_bounds__(kBlkThreads) blk_compact_kernel(const int32_t* __restrict__ pos, int64_t n_nodes,
                                                                  int32_t* __restrict__ ids) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v <= n_nodes && pos[v + 1] != pos[v]) ids[pos[v]] = (int32_t)v;
}

// deg[i] = the raw degree of the i-th node of V_{l+1} (0 for the dummy), for i < cap (0 past |V_{l+1}|)
__global__ void __launch_bounds__(kBlkThreads) blk_member_degree_kernel(const int64_t* __restrict__ indptr,
                                                                        int64_t n_nodes, const int32_t* __restrict__ ids,
                                                                        const int32_t* __restrict__ count_dev,
                                                                        int64_t cap, int64_t* __restrict__ deg) {
  const int64_t count = *count_dev;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t c = 0;
    if (i < count && ids[i] < n_nodes) {
      int64_t lo;
      blk_row(indptr, ids[i], lo, c);
    }
    deg[i] = c;
  }
}

// counts[2l] = |V_l| (from its position map)
__global__ void blk_size_kernel(const int32_t* __restrict__ pos_end, int64_t* __restrict__ count) { *count = *pos_end; }

// deg[p] for the n_local - 1 CSR rows of a block: V_l[p]'s raw degree when it is in V_{l+1} (member: next_pos steps at
// it), else 0; deg[n_local - 1] = 0 so the exclusive scan's last element is the entry count
__global__ void __launch_bounds__(kBlkThreads) blk_local_degree_kernel(const int64_t* __restrict__ indptr,
                                                                       int64_t n_nodes, const int32_t* __restrict__ ids,
                                                                       const int32_t* __restrict__ next_pos,
                                                                       int64_t n_local, int64_t* __restrict__ deg) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_local) return;
  int64_t c = 0;
  const int64_t v = ids[p];
  if (p < n_local - 1 && v < n_nodes && next_pos[v + 1] != next_pos[v]) {
    int64_t lo;
    blk_row(indptr, v, lo, c);
  }
  deg[p] = c;
}

// one warp per local row: its raw entries, clamped, relabelled through pos, in CSR order
__global__ void __launch_bounds__(kBlkThreads) blk_fill_kernel(const int64_t* __restrict__ indptr,
                                                               const int32_t* __restrict__ indices, int64_t n_nodes,
                                                               const int32_t* __restrict__ ids,
                                                               const int32_t* __restrict__ pos,
                                                               const int64_t* __restrict__ b_indptr, int64_t n_rows,
                                                               int32_t* __restrict__ b_indices) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * kBlkWarps;
  for (int64_t p = (int64_t)blockIdx.x * kBlkWarps + (threadIdx.x >> 5); p < n_rows; p += warps) {
    const int64_t at = b_indptr[p], cnt = b_indptr[p + 1] - at;
    if (cnt == 0) continue;
    const int64_t lo = indptr[ids[p]];
    for (int64_t e = lane; e < cnt; e += 32) b_indices[at + e] = pos[blk_clamp(indices[lo + e], n_nodes)];
  }
}

// rows[i] = pos[the i-th node of the next level]: V_{l+1}[i], or the clamped seed i for the last block
__global__ void __launch_bounds__(kBlkThreads) blk_rows_kernel(const int32_t* __restrict__ seeds,
                                                               const int32_t* __restrict__ ids, int64_t n,
                                                               int64_t n_nodes, const int32_t* __restrict__ pos,
                                                               int32_t* __restrict__ rows) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rows[i] = pos[blk_node(seeds, ids, i, n_nodes)];
}

static int32_t make_blocks_plan(int64_t n_nodes, int64_t nnz, int64_t n_seeds, int32_t n_layers, BlocksPlan& P,
                                const char* who) {
  GS_REQUIRE(n_nodes >= 0 && n_nodes < 0x7fffffffLL - 2, "%s: n_nodes must be in [0, 2^31 - 3)", who);
  GS_REQUIRE(nnz >= 0 && n_seeds >= 0 && n_seeds < 0x7fffffffLL, "%s: bad nnz or n_seeds", who);
  GS_REQUIRE(n_layers >= 1 && n_layers <= GS_MAX_BLOCK_LAYERS, "%s: n_layers must be in [1, %d]", who,
             GS_MAX_BLOCK_LAYERS);
  P.n_nodes = n_nodes;
  P.cap = n_nodes + 2;
  P.levels = n_layers + 1;
  size_t scan32 = 0, scan64 = 0, reduce64 = 0;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(nullptr, scan32, (const int32_t*)nullptr, (int32_t*)nullptr,
                                                        (int)P.cap);
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveSum (size query)");
  e = gs_cub::cub::DeviceScan::ExclusiveSum(nullptr, scan64, (const int64_t*)nullptr, (int64_t*)nullptr, (int)P.cap);
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveSum (size query)");
  e = gs_cub::cub::DeviceReduce::Sum(nullptr, reduce64, (const int64_t*)nullptr, (int64_t*)nullptr, (int)P.cap);
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceReduce::Sum (size query)");
  P.cub_bytes = std::max(std::max(scan32, scan64), reduce64);
  size_t off = 0;
  P.off_flag = off; off += align256((size_t)P.cap * 4);
  P.off_pos = off;  off += (size_t)P.levels * align256((size_t)P.cap * 4);
  P.off_ids = off;  off += (size_t)P.levels * align256((size_t)P.cap * 4);
  P.off_deg = off;  off += align256((size_t)P.cap * 8);
  P.off_cub = off;  off += align256(P.cub_bytes);
  P.bytes = off;
  return GS_OK;
}

struct BlocksWs {
  int32_t* flag;
  char* pos0;
  char* ids0;
  int64_t* deg;
  void* cub;
  size_t stride;
  int32_t* pos(int l) const { return (int32_t*)(pos0 + (size_t)l * stride); }
  int32_t* ids(int l) const { return (int32_t*)(ids0 + (size_t)l * stride); }
};

static BlocksWs blocks_ws(const BlocksPlan& P, void* workspace) {
  char* ws = (char*)workspace;
  return BlocksWs{(int32_t*)(ws + P.off_flag), ws + P.off_pos, ws + P.off_ids, (int64_t*)(ws + P.off_deg),
                  ws + P.off_cub, align256((size_t)P.cap * 4)};
}

static unsigned blk_grid(int64_t items, int64_t per_block, int64_t max_blocks) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((items + per_block - 1) / per_block, max_blocks));
}

}  // namespace gs

extern "C" {

int64_t gs_csr_blocks_workspace_bytes(int64_t n_nodes, int64_t nnz, int64_t n_seeds, int32_t n_layers) {
  gs::BlocksPlan P;
  if (gs::make_blocks_plan(n_nodes, nnz, n_seeds, n_layers, P, "gs_csr_blocks_workspace_bytes") != GS_OK) return -1;
  return (int64_t)P.bytes;
}

int32_t gs_csr_blocks_plan(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers, void* workspace,
                           int64_t workspace_bytes, int64_t* counts_dev, void* stream) {
  const char* who = "gs_csr_blocks_plan";
  gs::BlocksPlan P;
  int32_t rc = gs::make_blocks_plan(n_nodes, nnz, n_seeds, n_layers, P, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(indptr && counts_dev && (nnz == 0 || indices) && (n_seeds == 0 || seeds), "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)P.bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)P.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const gs::BlocksWs W = gs::blocks_ws(P, workspace);
  const int64_t max_warp_blocks = (int64_t)gs::sm_count() * 16;
  const unsigned node_blocks = gs::blk_grid(P.cap, gs::kBlkThreads, INT32_MAX);
  for (int l = n_layers; l >= 0; --l) {
    const bool seed_level = l == n_layers;             // level L: the distinct seeds, rows not expanded
    const int32_t* prev_ids = seed_level ? nullptr : W.ids(l + 1);
    const int32_t* prev_count = seed_level ? nullptr : W.pos(l + 1) + (P.cap - 1);
    const int64_t prev_cap = seed_level ? n_seeds : P.cap - 1;
    GS_CUDA(cudaMemsetAsync(W.flag, 0, (size_t)P.cap * 4, st));
    gs::blk_mark_kernel<<<gs::blk_grid(prev_cap, gs::kBlkWarps, max_warp_blocks), gs::kBlkThreads, 0, st>>>(
        indptr, indices, n_nodes, seed_level ? seeds : nullptr, prev_ids, prev_count, n_seeds, seed_level ? 0 : 1,
        W.flag);
    rc = gs::launch_check("blk_mark_kernel");
    if (rc != GS_OK) return rc;
    size_t cub_bytes = P.cub_bytes;
    cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(W.cub, cub_bytes, (const int32_t*)W.flag, W.pos(l), (int)P.cap,
                                                          st);
    if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceScan::ExclusiveSum");
    gs::blk_compact_kernel<<<node_blocks, gs::kBlkThreads, 0, st>>>(W.pos(l), n_nodes, W.ids(l));
    rc = gs::launch_check("blk_compact_kernel");
    if (rc != GS_OK) return rc;
    if (seed_level) continue;
    gs::blk_size_kernel<<<1, 1, 0, st>>>(W.pos(l) + (P.cap - 1), counts_dev + 2 * l);
    rc = gs::launch_check("blk_size_kernel");
    if (rc != GS_OK) return rc;
    // the entry count of block l: the degrees of V_{l+1}'s (distinct) nodes
    gs::blk_member_degree_kernel<<<gs::blk_grid(P.cap, gs::kBlkThreads, (int64_t)gs::sm_count() * 8), gs::kBlkThreads, 0,
                                   st>>>(indptr, n_nodes, W.ids(l + 1), W.pos(l + 1) + (P.cap - 1), P.cap, W.deg);
    rc = gs::launch_check("blk_member_degree_kernel");
    if (rc != GS_OK) return rc;
    cub_bytes = P.cub_bytes;
    e = gs_cub::cub::DeviceReduce::Sum(W.cub, cub_bytes, (const int64_t*)W.deg, counts_dev + 2 * l + 1, (int)P.cap, st);
    if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceReduce::Sum");
  }
  return GS_OK;
}

int32_t gs_csr_blocks_fill(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers, void* workspace,
                           int64_t workspace_bytes, const int64_t* counts, int32_t* const* src_ids,
                           int64_t* const* b_indptr, int32_t* const* b_indices, int32_t* const* b_rows, void* stream) {
  const char* who = "gs_csr_blocks_fill";
  gs::BlocksPlan P;
  int32_t rc = gs::make_blocks_plan(n_nodes, nnz, n_seeds, n_layers, P, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(indptr && counts && src_ids && b_indptr && b_indices && b_rows && (nnz == 0 || indices) &&
                 (n_seeds == 0 || seeds),
             "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)P.bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)P.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const gs::BlocksWs W = gs::blocks_ws(P, workspace);
  const int64_t max_warp_blocks = (int64_t)gs::sm_count() * 16;
  for (int l = 0; l < n_layers; ++l) {
    const int64_t n_local = counts[2 * l], entries = counts[2 * l + 1];
    const bool last = l == n_layers - 1;
    const int64_t n_out = last ? n_seeds : counts[2 * l + 2];
    GS_REQUIRE(n_local >= 1 && n_local <= n_nodes + 1 && entries >= 0 && n_out >= 0, "%s: bad counts for block %d", who,
               l);
    GS_REQUIRE(src_ids[l] && b_indptr[l] && (entries == 0 || b_indices[l]) && (n_out == 0 || b_rows[l]),
               "%s: NULL output of block %d", who, l);
    GS_CUDA(cudaMemcpyAsync(src_ids[l], W.ids(l), (size_t)n_local * 4, cudaMemcpyDeviceToDevice, st));
    gs::blk_local_degree_kernel<<<gs::blk_grid(n_local, gs::kBlkThreads, INT32_MAX), gs::kBlkThreads, 0, st>>>(
        indptr, n_nodes, W.ids(l), W.pos(l + 1), n_local, W.deg);
    rc = gs::launch_check("blk_local_degree_kernel");
    if (rc != GS_OK) return rc;
    size_t cub_bytes = P.cub_bytes;
    cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(W.cub, cub_bytes, (const int64_t*)W.deg, b_indptr[l],
                                                          (int)n_local, st);
    if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceScan::ExclusiveSum");
    if (entries > 0) {
      gs::blk_fill_kernel<<<gs::blk_grid(n_local - 1, gs::kBlkWarps, max_warp_blocks), gs::kBlkThreads, 0, st>>>(
          indptr, indices, n_nodes, W.ids(l), W.pos(l), b_indptr[l], n_local - 1, b_indices[l]);
      rc = gs::launch_check("blk_fill_kernel");
      if (rc != GS_OK) return rc;
    }
    if (n_out > 0) {
      gs::blk_rows_kernel<<<gs::blk_grid(n_out, gs::kBlkThreads, INT32_MAX), gs::kBlkThreads, 0, st>>>(
          last ? seeds : nullptr, W.ids(l + 1), n_out, n_nodes, W.pos(l), b_rows[l]);
      rc = gs::launch_check("blk_rows_kernel");
      if (rc != GS_OK) return rc;
    }
  }
  return GS_OK;
}

}  // extern "C"

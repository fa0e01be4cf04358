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
//
// Sampled blocks (gs_csr_sampled_blocks_plan / _fill, gs_csr_sample_rows; contract in oracle/sampled_blocks.py): the same
// kernels, instantiated with kSample = true, read S_l(v) - at most k_l entries of v's row, drawn without replacement by
// Floyd's algorithm - instead of the whole row.  One warp per node: the draws u_i are spread over the lanes (lane i % 32,
// slot i / 32), the k held positions too; each of Floyd's k steps broadcasts u_i, tests membership with one ballot and
// stores the taken position at its owner.  The fill ranks the held positions (each lane counts the smaller ones over the
// warp) to write them in ascending order.  The plan and the fill recompute the same draws; nothing is stored between
// them.  A hub row is never walked: with d > k a warp touches only the k drawn entries.  kSample = false is the code
// above, instruction for instruction (the draw arguments are appended and unused).
// gs_csr_sampled_blocks_fill_offsets runs the fill with kOff = true: where it writes an entry it also writes the entry's
// offset in its node's raw row (the held Floyd position, or e), which the training masks name it by
// (oracle/sampled_blocks_dropout.py).  No other kernel changes, and the other arrays are the same bytes.
//
// Weighted blocks (gs_csr_weighted_blocks_plan / _fill / _fill_offsets, gs_csr_sample_rows_weighted; contract in
// oracle/weighted_sampling.py): the same plan and fill, with S_l^w(v) - the k eligible (w > 0) entries with the smallest
// fp64 keys E / w - in place of Floyd's sample.  wblk_degree_kernel gives min(d+, k) where the uniform path takes
// min(d, k), and wblk_select_kernel replaces the mark and the fill (one warp per row, a row of kHubRow entries or more
// over the whole CTA).  The kernels above are not touched.
#include <algorithm>

#include "common.cuh"

#define CUB_WRAPPED_NAMESPACE gs_cub
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

namespace gs {

constexpr int kBlkThreads = 256;
constexpr int kBlkWarps = kBlkThreads / 32;

constexpr int kMaxFanout = GS_MAX_FANOUT;
constexpr int kSlots = kMaxFanout / 32;   // held positions per lane

// the draws of one sampled layer: S_l(v) takes min(d, k) entries; u_i = word 0 of
// philox4x32_10((i, v, call, kStreamSampledBlocks | layer), key = seed)
struct SampleArgs {
  uint32_t k0, k1, call, tag;
  int32_t k;
};

static SampleArgs make_sample_args(int32_t k, uint64_t seed, uint64_t call, int32_t layer) {
  return SampleArgs{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)call, kStreamSampledBlocks | (uint32_t)layer, k};
}

// Floyd's sample of k of the d > k positions of node v's row, in draw order: position i of the sample sits in slot i / 32
// of lane i % 32; unused slots hold INT32_MAX.  Step i: j = d - k + i, t = mulhi(u_i, j + 1); t unless already held, else j.
__device__ __forceinline__ void floyd_sample(const SampleArgs& sa, int64_t v, int64_t d, int lane,
                                             int32_t (&held)[kSlots]) {
  const int k = sa.k;
  uint32_t u[kSlots];
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    held[s] = INT32_MAX;
    u[s] = 0;
    const int i = s * 32 + lane;
    if (s * 32 < k && i < k) u[s] = philox4x32_10(u32x4{(uint32_t)i, (uint32_t)v, sa.call, sa.tag}, sa.k0, sa.k1).x;
  }
  for (int i = 0; i < k; ++i) {
    const int slot = i >> 5, owner = i & 31;
    uint32_t mine = 0;
#pragma unroll
    for (int s = 0; s < kSlots; ++s)
      if (s == slot) mine = u[s];
    const uint32_t ui = __shfl_sync(0xffffffffu, mine, owner);
    const int64_t j = d - k + i;
    const int32_t t = (int32_t)(((uint64_t)ui * (uint64_t)(j + 1)) >> 32);
    bool hit = false;
#pragma unroll
    for (int s = 0; s < kSlots; ++s)
      if (s * 32 < k) hit |= held[s] == t;
    const int32_t take = __any_sync(0xffffffffu, hit) ? (int32_t)j : t;
#pragma unroll
    for (int s = 0; s < kSlots; ++s)
      if (s == slot && lane == owner) held[s] = take;
  }
}

// rank[s] = the number of held positions below held[s] (they are distinct): the slot's place in ascending order
__device__ __forceinline__ void warp_ranks(const int32_t (&held)[kSlots], int k, int32_t (&rank)[kSlots]) {
#pragma unroll
  for (int s = 0; s < kSlots; ++s) rank[s] = 0;
#pragma unroll
  for (int s2 = 0; s2 < kSlots; ++s2) {
    if (s2 * 32 >= k) break;
    for (int src = 0; src < 32; ++src) {
      const int32_t x = __shfl_sync(0xffffffffu, held[s2], src);
#pragma unroll
      for (int s = 0; s < kSlots; ++s)
        if (s * 32 < k) rank[s] += x < held[s];
    }
  }
}

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

// ---- weighted draws (contract: oracle/weighted_sampling.py) ----------------------------------------------------------
// S_l^w(v): the min(d+, k) eligible (w > 0) entries with the smallest (key_j, j); key_j = E_j / w_j in fp64, E_j =
// ws_neg_log(U_j), U_j = (2m + 1) 2^-53 from words (0, 1) (j even) or (2, 3) (j odd) of
// philox4x32_10((j >> 1, v, call, kStreamWeightedBlocks | layer), key = seed).
struct WeightArgs {
  const float* w;
  uint32_t k0, k1, call, tag;
  int32_t k;
};

static WeightArgs make_weight_args(const float* w, int32_t k, uint64_t seed, uint64_t call, int32_t layer) {
  return WeightArgs{w, (uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)call, kStreamWeightedBlocks | (uint32_t)layer, k};
}

constexpr int kHubRow = 4096;   // a row at least this long is split over the CTA's warps, then merged by warp 0

// -ln(u), u in (0, 1) normal: the oracle's sequence of IEEE fp64 operations (never contracted into FMAs)
__device__ __forceinline__ double ws_neg_log(double u) {
  const unsigned long long bits = (unsigned long long)__double_as_longlong(u);
  int e = (int)((bits >> 52) & 0x7ff) - 1023;
  double f = __longlong_as_double((long long)((bits & 0x000fffffffffffffULL) | 0x3ff0000000000000ULL));
  if (f > 0x1.6a09e667f3bcdp+0) {
    f = __dmul_rn(f, 0.5);
    e += 1;
  }
  const double s = __ddiv_rn(__dsub_rn(f, 1.0), __dadd_rn(f, 1.0));
  const double z = __dmul_rn(s, s);
  double p = 0x1.8618618618618p-5;                            // 1/21, then Horner down to 1/3
  p = __dadd_rn(__dmul_rn(p, z), 0x1.af286bca1af28p-5);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.e1e1e1e1e1e1ep-5);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.1111111111111p-4);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.3b13b13b13b14p-4);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.745d1745d1746p-4);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.c71c71c71c71cp-4);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.2492492492492p-3);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.999999999999ap-3);
  p = __dadd_rn(__dmul_rn(p, z), 0x1.5555555555555p-2);
  const double t = __dadd_rn(s, s);
  const double lnf = __dadd_rn(t, __dmul_rn(t, __dmul_rn(z, p)));
  const double ed = (double)e;
  return -__dadd_rn(__dmul_rn(ed, 0x1.62e42fee00000p-1), __dadd_rn(__dmul_rn(ed, 0x1.a39ef35793c76p-33), lnf));
}

// the key bits of weight w > 0 from words (a, b): E / w >= 0, so the bits order as the values do
__device__ __forceinline__ uint64_t ws_key(uint32_t a, uint32_t b, float w) {
  const uint64_t m = ((uint64_t)a << 20) | (b >> 12);
  const double u = __dmul_rn((double)(2 * m + 1), 0x1p-53);
  return (uint64_t)__double_as_longlong(__ddiv_rn(ws_neg_log(u), (double)w));
}

__device__ __forceinline__ bool ws_less(uint64_t ka, int32_t pa, uint64_t kb, int32_t pb) {
  return ka < kb || (ka == kb && pa < pb);
}

// one warp's candidates in shared memory: n (warp-uniform) held (key, position) pairs in [0, cap), cap = 2k + 32, and a
// threshold (tk, tp): once n has exceeded 2k, the k-th smallest held pair - nothing above it can be among the k smallest
struct WarpSel {
  uint64_t* key;
  int32_t* pos;
  uint64_t* t_key;   // the warp's shared slot for a threshold
  int32_t* t_pos;
  int n, cap;
  uint64_t tk;
  int32_t tp;
};

// keep the `keep` < n smallest held pairs, in buffer order, and make the largest of them the threshold.  Ranks by
// counting over the whole buffer (pairs are distinct: positions are); compaction moves pairs down only.
__device__ __forceinline__ void ws_compact(WarpSel& s, int keep, int lane) {
  __syncwarp();
  for (int i = lane; i < s.n; i += 32) {
    const uint64_t ki = s.key[i];
    const int32_t pi = s.pos[i];
    int r = 0;
    for (int j = 0; j < s.n; ++j) r += ws_less(s.key[j], s.pos[j], ki, pi);
    if (r == keep - 1) {
      *s.t_key = ki;
      *s.t_pos = pi;
    }
  }
  __syncwarp();
  s.tk = *s.t_key;
  s.tp = *s.t_pos;
  int base = 0;
  for (int i0 = 0; i0 < s.n; i0 += 32) {
    const int i = i0 + lane;
    uint64_t ki = 0;
    int32_t pi = 0;
    bool in = false;
    if (i < s.n) {
      ki = s.key[i];
      pi = s.pos[i];
      in = !ws_less(s.tk, s.tp, ki, pi);
    }
    const unsigned m = __ballot_sync(0xffffffffu, in);
    __syncwarp();
    if (in) {
      const int at = base + __popc(m & ((1u << lane) - 1u));
      s.key[at] = ki;
      s.pos[at] = pi;
    }
    base += __popc(m);
  }
  __syncwarp();
  s.n = base;
}

// offer one pair per lane (ok: the lane has one); room for 32 is made first
__device__ __forceinline__ void ws_insert(WarpSel& s, int k, uint64_t key, int32_t pos, bool ok, int lane) {
  if (s.n + 32 > s.cap) ws_compact(s, k, lane);
  const bool in = ok && ws_less(key, pos, s.tk, s.tp);
  const unsigned m = __ballot_sync(0xffffffffu, in);
  if (in) {
    const int at = s.n + __popc(m & ((1u << lane) - 1u));
    s.key[at] = key;
    s.pos[at] = pos;
  }
  s.n += __popc(m);
}

// offer the entries [begin + stride * i, + 64) of node v's row [lo, lo + d): each lane takes the pair (j, j + 1), j even,
// and one Philox call.  keys = false (d <= k: every eligible entry is kept) skips the words.
__device__ __forceinline__ void ws_scan(WarpSel& s, const WeightArgs& a, int64_t v, int64_t lo, int64_t d, int64_t begin,
                                        int64_t stride, bool keys, int lane) {
  for (int64_t c = begin; c < d; c += stride) {
    const int64_t j = c + 2 * lane;
    const float w0 = j < d ? a.w[lo + j] : 0.f, w1 = j + 1 < d ? a.w[lo + j + 1] : 0.f;
    const bool ok0 = w0 > 0.f, ok1 = w1 > 0.f;                  // false for NaN, zero and negative weights
    uint64_t key0 = 0, key1 = 0;
    if (keys && (ok0 || ok1)) {
      const u32x4 r = philox4x32_10(u32x4{(uint32_t)(j >> 1), (uint32_t)v, a.call, a.tag}, a.k0, a.k1);
      if (ok0) key0 = ws_key(r.x, r.y, w0);
      if (ok1) key1 = ws_key(r.z, r.w, w1);
    }
    ws_insert(s, a.k, key0, (int32_t)j, ok0, lane);
    ws_insert(s, a.k, key1, (int32_t)(j + 1), ok1, lane);
  }
}

// where a sampled row's entries go: flag them (the plan's mark) or write them, ascending, into a block (the fill)
struct WSelRows {
  const int64_t* indptr;
  const int32_t* indices;
  int64_t n_nodes;
  const int32_t* ids;          // row p is node ids[p] (NULL: node p, fill only)
  const int32_t* count_dev;    // mark: the number of rows, on the device
  int32_t* flag;               // mark
  const int32_t* pos;          // fill: the relabelling (NULL: entries as stored)
  const int64_t* b_indptr;     // fill
  int32_t* b_indices;          // fill
  int32_t* b_off;              // fill with offsets (kOff)
  int64_t n_rows;              // fill: the number of rows
};

// the k smallest of the n held pairs, emitted: the mark flags each entry; the fill writes entry q at at + its rank
// among the held positions, so the row keeps CSR order
template <bool kFill, bool kOff>
__device__ __forceinline__ void ws_emit(WarpSel& s, const WSelRows& r, int k, int64_t lo, int64_t at, int lane) {
  if (s.n > k) ws_compact(s, k, lane);
  __syncwarp();
  for (int i = lane; i < s.n; i += 32) {
    const int32_t q = s.pos[i];
    const int32_t x = r.indices[lo + q];
    if (!kFill) {
      r.flag[blk_clamp(x, r.n_nodes)] = 1;
      continue;
    }
    int rank = 0;
    for (int j = 0; j < s.n; ++j) rank += s.pos[j] < q;
    r.b_indices[at + rank] = r.pos ? r.pos[blk_clamp(x, r.n_nodes)] : x;
    if (kOff) r.b_off[at + rank] = q;
  }
  __syncwarp();
}

// one warp per node of the previous level (count: *count_dev, or n when count_dev is NULL): flag the node and, with
// expand, its row's clamped entries (kSample: those of S_l(v)); the dummy N too with expand.  Stores of 1 only: the order
// of racing stores is moot.
template <bool kSample>
__global__ void __launch_bounds__(kBlkThreads) blk_mark_kernel(const int64_t* __restrict__ indptr,
                                                               const int32_t* __restrict__ indices, int64_t n_nodes,
                                                               const int32_t* __restrict__ seeds,
                                                               const int32_t* __restrict__ ids,
                                                               const int32_t* __restrict__ count_dev, int64_t n,
                                                               int32_t expand, int32_t* __restrict__ flag,
                                                               SampleArgs sa) {
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
    if (kSample && cnt > sa.k) {
      int32_t held[kSlots];
      floyd_sample(sa, v, cnt, lane, held);
#pragma unroll
      for (int s = 0; s < kSlots; ++s)
        if (held[s] != INT32_MAX) flag[blk_clamp(indices[lo + held[s]], n_nodes)] = 1;
      continue;
    }
    for (int64_t e = lane; e < cnt; e += 32) flag[blk_clamp(indices[lo + e], n_nodes)] = 1;
  }
}

// ids[pos[v]] = v for every flagged v (pos[v + 1] - pos[v] is v's flag), ascending
__global__ void __launch_bounds__(kBlkThreads) blk_compact_kernel(const int32_t* __restrict__ pos, int64_t n_nodes,
                                                                  int32_t* __restrict__ ids) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v <= n_nodes && pos[v + 1] != pos[v]) ids[pos[v]] = (int32_t)v;
}

// deg[i] = the raw degree of the i-th node of V_{l+1} (kSample: min(degree, k); 0 for the dummy), for i < cap (0 past
// |V_{l+1}|)
template <bool kSample>
__global__ void __launch_bounds__(kBlkThreads) blk_member_degree_kernel(const int64_t* __restrict__ indptr,
                                                                        int64_t n_nodes, const int32_t* __restrict__ ids,
                                                                        const int32_t* __restrict__ count_dev,
                                                                        int64_t cap, int64_t* __restrict__ deg,
                                                                        SampleArgs sa) {
  const int64_t count = *count_dev;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t c = 0;
    if (i < count && ids[i] < n_nodes) {
      int64_t lo;
      blk_row(indptr, ids[i], lo, c);
    }
    deg[i] = kSample ? min(c, (int64_t)sa.k) : c;
  }
}

// counts[2l] = |V_l| (from its position map)
__global__ void blk_size_kernel(const int32_t* __restrict__ pos_end, int64_t* __restrict__ count) { *count = *pos_end; }

// deg[p] for the n_local - 1 CSR rows of a block: V_l[p]'s raw degree (kSample: min(degree, k)) when it is in V_{l+1}
// (member: next_pos steps at it), else 0; deg[n_local - 1] = 0 so the exclusive scan's last element is the entry count.
// kSample with ids == NULL: row p is node p and every row is a member (gs_csr_sample_rows, S_l over all nodes).
template <bool kSample>
__global__ void __launch_bounds__(kBlkThreads) blk_local_degree_kernel(const int64_t* __restrict__ indptr,
                                                                       int64_t n_nodes, const int32_t* __restrict__ ids,
                                                                       const int32_t* __restrict__ next_pos,
                                                                       int64_t n_local, int64_t* __restrict__ deg,
                                                                       SampleArgs sa) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_local) return;
  int64_t c = 0;
  if (kSample && ids == nullptr) {
    if (p < n_local - 1) {
      int64_t lo;
      blk_row(indptr, p, lo, c);
    }
    deg[p] = min(c, (int64_t)sa.k);
    return;
  }
  const int64_t v = ids[p];
  if (p < n_local - 1 && v < n_nodes && next_pos[v + 1] != next_pos[v]) {
    int64_t lo;
    blk_row(indptr, v, lo, c);
  }
  deg[p] = kSample ? min(c, (int64_t)sa.k) : c;
}

// one warp per local row: its raw entries, clamped, relabelled through pos, in CSR order.  kSample: the entries of
// S_l(v) (a row with more than k entries: Floyd's draws again, written in ascending position order); ids == NULL: row p
// is node p; pos == NULL: the entries are copied as they are (gs_csr_sample_rows).  kOff (kSample only): b_off[at + .]
// = the entry's offset in v's raw row, beside b_indices
template <bool kSample, bool kOff = false>
__global__ void __launch_bounds__(kBlkThreads) blk_fill_kernel(const int64_t* __restrict__ indptr,
                                                               const int32_t* __restrict__ indices, int64_t n_nodes,
                                                               const int32_t* __restrict__ ids,
                                                               const int32_t* __restrict__ pos,
                                                               const int64_t* __restrict__ b_indptr, int64_t n_rows,
                                                               int32_t* __restrict__ b_indices, SampleArgs sa,
                                                               int32_t* __restrict__ b_off = nullptr) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * kBlkWarps;
  for (int64_t p = (int64_t)blockIdx.x * kBlkWarps + (threadIdx.x >> 5); p < n_rows; p += warps) {
    const int64_t at = b_indptr[p], cnt = b_indptr[p + 1] - at;
    if (cnt == 0) continue;
    if (kSample) {
      const int64_t v = ids ? (int64_t)ids[p] : p;
      int64_t lo, d;
      blk_row(indptr, v, lo, d);
      if (d > cnt) {                                   // cnt = k < d: the sample, ascending
        int32_t held[kSlots], rank[kSlots];
        floyd_sample(sa, v, d, lane, held);
        warp_ranks(held, sa.k, rank);
#pragma unroll
        for (int s = 0; s < kSlots; ++s) {
          if (held[s] == INT32_MAX) continue;
          const int32_t x = indices[lo + held[s]];
          b_indices[at + rank[s]] = pos ? pos[blk_clamp(x, n_nodes)] : x;
          if (kOff) b_off[at + rank[s]] = held[s];
        }
      } else {
        for (int64_t e = lane; e < cnt; e += 32) {
          const int32_t x = indices[lo + e];
          b_indices[at + e] = pos ? pos[blk_clamp(x, n_nodes)] : x;
          if (kOff) b_off[at + e] = (int32_t)e;
        }
      }
      continue;
    }
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

// deg[i] = min(d+, k) for i < n, one warp per item (a hub row's weights spread over the lanes; the count stops at k):
//   ids == NULL                 row i is node i for i < n - 1, deg[n - 1] = 0 (gs_csr_sample_rows_weighted);
//   next_pos == NULL            the members V_{l+1}[i], i < *count_dev (the plan's entry count; 0 past it);
//   else                        local row i of a block, node ids[i], when it is in V_{l+1} (next_pos steps at it).
// The dummy and rows outside V_{l+1} give 0.
__global__ void __launch_bounds__(kBlkThreads) wblk_degree_kernel(const int64_t* __restrict__ indptr,
                                                                  const float* __restrict__ w, int64_t n_nodes,
                                                                  const int32_t* __restrict__ ids,
                                                                  const int32_t* __restrict__ count_dev,
                                                                  const int32_t* __restrict__ next_pos, int64_t n,
                                                                  int64_t* __restrict__ deg, int32_t k) {
  const int lane = threadIdx.x & 31;
  const int64_t count = count_dev ? (int64_t)*count_dev : n;
  const int64_t warps = (int64_t)gridDim.x * kBlkWarps;
  for (int64_t i = (int64_t)blockIdx.x * kBlkWarps + (threadIdx.x >> 5); i < n; i += warps) {
    int64_t v = -1;
    if (ids == nullptr) {
      if (i < n - 1) v = i;
    } else if (next_pos == nullptr) {
      if (i < count && ids[i] < n_nodes) v = ids[i];
    } else {
      const int64_t u = ids[i];
      if (i < n - 1 && u < n_nodes && next_pos[u + 1] != next_pos[u]) v = u;
    }
    int64_t c = 0;
    if (v >= 0) {
      int64_t lo, d;
      blk_row(indptr, v, lo, d);
      for (int64_t e0 = 0; e0 < d && c < k; e0 += 32) {
        const int64_t e = e0 + lane;
        c += __popc(__ballot_sync(0xffffffffu, e < d && w[lo + e] > 0.f));
      }
    }
    if (lane == 0) deg[i] = min(c, (int64_t)k);
  }
}

// The weighted selection, one group of kBlkWarps rows per CTA at a time: warp i takes row i of the group when it is
// shorter than kHubRow; then every hub row of the group is split over all the warps (warp i offers the 64-entry chunks
// i, i + kBlkWarps, ...), each warp keeps its k smallest, and warp 0 merges them.  The result is the set of the k
// smallest (key, position) pairs, whatever the schedule: no atomics, the same bytes every call.
// kFill = false: the plan's mark (rows V_{l+1}[p], p < *count_dev; flags each node, its sample's clamped entries and
// N).  kFill: the fill (rows p < n_rows with b_indptr[p + 1] > b_indptr[p]), kOff also writing the raw-row offsets.
// Dynamic shared memory: kBlkWarps * (2k + 32) * 12 bytes.
template <bool kFill, bool kOff>
__global__ void __launch_bounds__(kBlkThreads) wblk_select_kernel(WSelRows r, WeightArgs a) {
  extern __shared__ __align__(16) unsigned char ws_smem[];
  __shared__ uint64_t t_key[kBlkWarps];
  __shared__ int32_t t_pos[kBlkWarps], held[kBlkWarps];
  __shared__ int64_t hub_v[kBlkWarps], hub_lo[kBlkWarps], hub_d[kBlkWarps], hub_at[kBlkWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cap = 2 * a.k + 32;
  uint64_t* keys = (uint64_t*)ws_smem;
  int32_t* poss = (int32_t*)(ws_smem + (size_t)kBlkWarps * cap * 8);
  const WarpSel init{keys + warp * cap, poss + warp * cap, t_key + warp, t_pos + warp, 0, cap, ~0ULL, INT32_MAX};
  const int64_t n_rows = kFill ? r.n_rows : (int64_t)*r.count_dev;
  if (!kFill && blockIdx.x == 0 && threadIdx.x == 0) r.flag[r.n_nodes] = 1;
  for (int64_t g0 = (int64_t)blockIdx.x * kBlkWarps; g0 < n_rows; g0 += (int64_t)gridDim.x * kBlkWarps) {
    const int64_t p = g0 + warp;
    int64_t v = -1, lo = 0, d = 0, at = 0;
    if (p < n_rows) {
      if (kFill) {
        at = r.b_indptr[p];
        if (r.b_indptr[p + 1] != at) v = r.ids ? (int64_t)r.ids[p] : p;
      } else {
        v = r.ids[p];
        if (lane == 0) r.flag[v] = 1;
        if (v >= r.n_nodes) v = -1;
      }
      if (v >= 0) blk_row(r.indptr, v, lo, d);
    }
    if (d > 0 && d < kHubRow) {
      WarpSel s = init;
      ws_scan(s, a, v, lo, d, 0, 64, d > a.k, lane);
      ws_emit<kFill, kOff>(s, r, a.k, lo, at, lane);
    }
    if (lane == 0) {
      hub_d[warp] = d >= kHubRow ? d : 0;
      hub_v[warp] = v;
      hub_lo[warp] = lo;
      hub_at[warp] = at;
    }
    __syncthreads();
    for (int h = 0; h < kBlkWarps; ++h) {
      const int64_t hd = hub_d[h];
      if (hd == 0) continue;                                      // CTA-uniform
      WarpSel s = init;
      ws_scan(s, a, hub_v[h], hub_lo[h], hd, (int64_t)warp * 64, (int64_t)kBlkWarps * 64, true, lane);
      if (s.n > a.k) ws_compact(s, a.k, lane);
      if (lane == 0) held[warp] = s.n;
      __syncthreads();
      if (warp == 0) {
        for (int o = 1; o < kBlkWarps; ++o) {
          const uint64_t* ok_ = keys + o * cap;
          const int32_t* op_ = poss + o * cap;
          for (int i0 = 0; i0 < held[o]; i0 += 32) {
            const int i = i0 + lane;
            const bool ok = i < held[o];
            ws_insert(s, a.k, ok ? ok_[i] : 0, ok ? op_[i] : 0, ok, lane);
          }
        }
        ws_emit<kFill, kOff>(s, r, a.k, hub_lo[h], hub_at[h], lane);
      }
      __syncthreads();
    }
    __syncthreads();
  }
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

static size_t wblk_smem_bytes(int32_t k) { return (size_t)kBlkWarps * (size_t)(2 * k + 32) * 12; }

template <bool kFill, bool kOff>
static int32_t launch_wblk_select(const WSelRows& r, const WeightArgs& a, int64_t max_rows, cudaStream_t st) {
  auto kern = wblk_select_kernel<kFill, kOff>;
  GS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wblk_smem_bytes(kMaxFanout)));
  kern<<<blk_grid(max_rows, kBlkWarps, (int64_t)sm_count() * 16), kBlkThreads, wblk_smem_bytes(a.k), st>>>(r, a);
  return launch_check("wblk_select_kernel");
}

static int32_t check_fanouts(const int32_t* fanouts, int32_t n_layers, int64_t nnz, const char* who) {
  GS_REQUIRE(fanouts != nullptr, "%s: NULL fanouts", who);
  GS_REQUIRE(nnz <= INT32_MAX, "%s: sampled rows need nnz < 2^31 (got %lld)", who, (long long)nnz);
  for (int l = 0; l < n_layers; ++l)
    GS_REQUIRE(fanouts[l] >= 1 && fanouts[l] <= kMaxFanout, "%s: fanout %d of layer %d outside [1, %d]", who, fanouts[l], l,
               kMaxFanout);
  return GS_OK;
}

// gs_csr_blocks_plan, or with fanouts (host, one per layer) gs_csr_sampled_blocks_plan, and with weighted
// gs_csr_weighted_blocks_plan (sw: the sample weights, NULL only when nnz = 0)
static int32_t blocks_plan(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers, const int32_t* fanouts, uint64_t seed,
                           uint64_t call, void* workspace, int64_t workspace_bytes, int64_t* counts_dev, void* stream,
                           const char* who, bool weighted = false, const float* sw = nullptr) {
  BlocksPlan P;
  int32_t rc = make_blocks_plan(n_nodes, nnz, n_seeds, n_layers, P, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(indptr && counts_dev && (nnz == 0 || indices) && (n_seeds == 0 || seeds), "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)P.bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)P.bytes);
  if (fanouts && (rc = check_fanouts(fanouts, n_layers, nnz, who)) != GS_OK) return rc;
  GS_REQUIRE(!weighted || (fanouts && (nnz == 0 || sw)), "%s: NULL fanouts or sample weights", who);
  auto mark = fanouts ? blk_mark_kernel<true> : blk_mark_kernel<false>;
  auto member_degree = fanouts ? blk_member_degree_kernel<true> : blk_member_degree_kernel<false>;
  cudaStream_t st = (cudaStream_t)stream;
  const BlocksWs W = blocks_ws(P, workspace);
  const int64_t max_warp_blocks = (int64_t)sm_count() * 16;
  const unsigned node_blocks = blk_grid(P.cap, kBlkThreads, INT32_MAX);
  for (int l = n_layers; l >= 0; --l) {
    const bool seed_level = l == n_layers;             // level L: the distinct seeds, rows not expanded
    const int32_t* prev_ids = seed_level ? nullptr : W.ids(l + 1);
    const int32_t* prev_count = seed_level ? nullptr : W.pos(l + 1) + (P.cap - 1);
    const int64_t prev_cap = seed_level ? n_seeds : P.cap - 1;
    const SampleArgs sa = fanouts && !seed_level ? make_sample_args(fanouts[l], seed, call, l) : SampleArgs{};
    GS_CUDA(cudaMemsetAsync(W.flag, 0, (size_t)P.cap * 4, st));
    if (weighted && !seed_level) {
      const WSelRows r{indptr, indices, n_nodes, prev_ids, prev_count, W.flag, nullptr, nullptr, nullptr, nullptr, 0};
      rc = launch_wblk_select<false, false>(r, make_weight_args(sw, fanouts[l], seed, call, l), prev_cap, st);
    } else {
      mark<<<blk_grid(prev_cap, kBlkWarps, max_warp_blocks), kBlkThreads, 0, st>>>(
          indptr, indices, n_nodes, seed_level ? seeds : nullptr, prev_ids, prev_count, n_seeds, seed_level ? 0 : 1,
          W.flag, sa);
      rc = launch_check("blk_mark_kernel");
    }
    if (rc != GS_OK) return rc;
    size_t cub_bytes = P.cub_bytes;
    cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(W.cub, cub_bytes, (const int32_t*)W.flag, W.pos(l), (int)P.cap,
                                                          st);
    if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveSum");
    blk_compact_kernel<<<node_blocks, kBlkThreads, 0, st>>>(W.pos(l), n_nodes, W.ids(l));
    rc = launch_check("blk_compact_kernel");
    if (rc != GS_OK) return rc;
    if (seed_level) continue;
    blk_size_kernel<<<1, 1, 0, st>>>(W.pos(l) + (P.cap - 1), counts_dev + 2 * l);
    rc = launch_check("blk_size_kernel");
    if (rc != GS_OK) return rc;
    // the entry count of block l: the degrees (sampled: min(degree, k_l); weighted: min(d+, k_l)) of V_{l+1}'s
    // (distinct) nodes
    if (weighted) {
      wblk_degree_kernel<<<blk_grid(P.cap, kBlkWarps, max_warp_blocks), kBlkThreads, 0, st>>>(
          indptr, sw, n_nodes, W.ids(l + 1), W.pos(l + 1) + (P.cap - 1), nullptr, P.cap, W.deg, fanouts[l]);
      rc = launch_check("wblk_degree_kernel");
    } else {
      member_degree<<<blk_grid(P.cap, kBlkThreads, (int64_t)sm_count() * 8), kBlkThreads, 0, st>>>(
          indptr, n_nodes, W.ids(l + 1), W.pos(l + 1) + (P.cap - 1), P.cap, W.deg, sa);
      rc = launch_check("blk_member_degree_kernel");
    }
    if (rc != GS_OK) return rc;
    cub_bytes = P.cub_bytes;
    e = gs_cub::cub::DeviceReduce::Sum(W.cub, cub_bytes, (const int64_t*)W.deg, counts_dev + 2 * l + 1, (int)P.cap, st);
    if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceReduce::Sum");
  }
  return GS_OK;
}

// gs_csr_blocks_fill, or with fanouts gs_csr_sampled_blocks_fill (and with b_off, _fill_offsets); with weighted the
// gs_csr_weighted_blocks_fill counterparts
static int32_t blocks_fill(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers, const int32_t* fanouts, uint64_t seed,
                           uint64_t call, void* workspace, int64_t workspace_bytes, const int64_t* counts,
                           int32_t* const* src_ids, int64_t* const* b_indptr, int32_t* const* b_indices,
                           int32_t* const* b_rows, int32_t* const* b_off, void* stream, const char* who,
                           bool weighted = false, const float* sw = nullptr) {
  BlocksPlan P;
  int32_t rc = make_blocks_plan(n_nodes, nnz, n_seeds, n_layers, P, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(indptr && counts && src_ids && b_indptr && b_indices && b_rows && (nnz == 0 || indices) &&
                 (n_seeds == 0 || seeds),
             "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)P.bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)P.bytes);
  if (fanouts && (rc = check_fanouts(fanouts, n_layers, nnz, who)) != GS_OK) return rc;
  GS_REQUIRE(!weighted || (fanouts && (nnz == 0 || sw)), "%s: NULL fanouts or sample weights", who);
  auto local_degree = fanouts ? blk_local_degree_kernel<true> : blk_local_degree_kernel<false>;
  auto fill = b_off ? blk_fill_kernel<true, true> : fanouts ? blk_fill_kernel<true> : blk_fill_kernel<false>;
  cudaStream_t st = (cudaStream_t)stream;
  const BlocksWs W = blocks_ws(P, workspace);
  const int64_t max_warp_blocks = (int64_t)sm_count() * 16;
  for (int l = 0; l < n_layers; ++l) {
    const int64_t n_local = counts[2 * l], entries = counts[2 * l + 1];
    const bool last = l == n_layers - 1;
    const int64_t n_out = last ? n_seeds : counts[2 * l + 2];
    const SampleArgs sa = fanouts ? make_sample_args(fanouts[l], seed, call, l) : SampleArgs{};
    GS_REQUIRE(n_local >= 1 && n_local <= n_nodes + 1 && entries >= 0 && n_out >= 0, "%s: bad counts for block %d", who,
               l);
    GS_REQUIRE(src_ids[l] && b_indptr[l] && (entries == 0 || (b_indices[l] && (!b_off || b_off[l]))) &&
                   (n_out == 0 || b_rows[l]),
               "%s: NULL output of block %d", who, l);
    GS_CUDA(cudaMemcpyAsync(src_ids[l], W.ids(l), (size_t)n_local * 4, cudaMemcpyDeviceToDevice, st));
    if (weighted) {
      wblk_degree_kernel<<<blk_grid(n_local, kBlkWarps, max_warp_blocks), kBlkThreads, 0, st>>>(
          indptr, sw, n_nodes, W.ids(l), nullptr, W.pos(l + 1), n_local, W.deg, fanouts[l]);
      rc = launch_check("wblk_degree_kernel");
    } else {
      local_degree<<<blk_grid(n_local, kBlkThreads, INT32_MAX), kBlkThreads, 0, st>>>(indptr, n_nodes, W.ids(l),
                                                                                      W.pos(l + 1), n_local, W.deg, sa);
      rc = launch_check("blk_local_degree_kernel");
    }
    if (rc != GS_OK) return rc;
    size_t cub_bytes = P.cub_bytes;
    cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(W.cub, cub_bytes, (const int64_t*)W.deg, b_indptr[l],
                                                          (int)n_local, st);
    if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveSum");
    if (entries > 0 && weighted) {
      const WSelRows r{indptr, indices, n_nodes, W.ids(l), nullptr, nullptr, W.pos(l), b_indptr[l], b_indices[l],
                       b_off ? b_off[l] : nullptr, n_local - 1};
      const WeightArgs wa = make_weight_args(sw, fanouts[l], seed, call, l);
      rc = b_off ? launch_wblk_select<true, true>(r, wa, n_local - 1, st)
                 : launch_wblk_select<true, false>(r, wa, n_local - 1, st);
      if (rc != GS_OK) return rc;
    } else if (entries > 0) {
      fill<<<blk_grid(n_local - 1, kBlkWarps, max_warp_blocks), kBlkThreads, 0, st>>>(
          indptr, indices, n_nodes, W.ids(l), W.pos(l), b_indptr[l], n_local - 1, b_indices[l], sa,
          b_off ? b_off[l] : nullptr);
      rc = launch_check("blk_fill_kernel");
      if (rc != GS_OK) return rc;
    }
    if (n_out > 0) {
      blk_rows_kernel<<<blk_grid(n_out, kBlkThreads, INT32_MAX), kBlkThreads, 0, st>>>(
          last ? seeds : nullptr, W.ids(l + 1), n_out, n_nodes, W.pos(l), b_rows[l]);
      rc = launch_check("blk_rows_kernel");
      if (rc != GS_OK) return rc;
    }
  }
  return GS_OK;
}

static int32_t sample_rows_plan(int64_t n_nodes, int64_t nnz, size_t& cub_bytes, size_t& bytes, const char* who) {
  GS_REQUIRE(n_nodes >= 0 && n_nodes < 0x7fffffffLL - 2, "%s: n_nodes must be in [0, 2^31 - 3)", who);
  GS_REQUIRE(nnz >= 0 && nnz <= INT32_MAX, "%s: sampled rows need 0 <= nnz < 2^31", who);
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                        (int)(n_nodes + 1));
  if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceScan::ExclusiveSum (size query)");
  bytes = align256((size_t)(n_nodes + 1) * 8) + align256(cub_bytes);
  return GS_OK;
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
  return gs::blocks_plan(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, nullptr, 0, 0, workspace,
                         workspace_bytes, counts_dev, stream, "gs_csr_blocks_plan");
}

int32_t gs_csr_blocks_fill(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers, void* workspace,
                           int64_t workspace_bytes, const int64_t* counts, int32_t* const* src_ids,
                           int64_t* const* b_indptr, int32_t* const* b_indices, int32_t* const* b_rows, void* stream) {
  return gs::blocks_fill(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, nullptr, 0, 0, workspace,
                         workspace_bytes, counts, src_ids, b_indptr, b_indices, b_rows, nullptr, stream,
                         "gs_csr_blocks_fill");
}

int32_t gs_csr_sampled_blocks_plan(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                                   const int32_t* seeds, int64_t n_seeds, int32_t n_layers, const int32_t* fanouts,
                                   uint64_t seed, uint64_t call, void* workspace, int64_t workspace_bytes,
                                   int64_t* counts_dev, void* stream) {
  const char* who = "gs_csr_sampled_blocks_plan";
  GS_REQUIRE(fanouts != nullptr, "%s: NULL fanouts", who);
  return gs::blocks_plan(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, fanouts, seed, call, workspace,
                         workspace_bytes, counts_dev, stream, who);
}

int32_t gs_csr_sampled_blocks_fill(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                                   const int32_t* seeds, int64_t n_seeds, int32_t n_layers, const int32_t* fanouts,
                                   uint64_t seed, uint64_t call, void* workspace, int64_t workspace_bytes,
                                   const int64_t* counts, int32_t* const* src_ids, int64_t* const* b_indptr,
                                   int32_t* const* b_indices, int32_t* const* b_rows, void* stream) {
  const char* who = "gs_csr_sampled_blocks_fill";
  GS_REQUIRE(fanouts != nullptr, "%s: NULL fanouts", who);
  return gs::blocks_fill(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, fanouts, seed, call, workspace,
                         workspace_bytes, counts, src_ids, b_indptr, b_indices, b_rows, nullptr, stream, who);
}

int32_t gs_csr_sampled_blocks_fill_offsets(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers,
                                           const int32_t* fanouts, uint64_t seed, uint64_t call, void* workspace,
                                           int64_t workspace_bytes, const int64_t* counts, int32_t* const* src_ids,
                                           int64_t* const* b_indptr, int32_t* const* b_indices, int32_t* const* b_rows,
                                           int32_t* const* b_off, void* stream) {
  const char* who = "gs_csr_sampled_blocks_fill_offsets";
  GS_REQUIRE(fanouts != nullptr && b_off != nullptr, "%s: NULL fanouts or offsets", who);
  return gs::blocks_fill(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, fanouts, seed, call, workspace,
                         workspace_bytes, counts, src_ids, b_indptr, b_indices, b_rows, b_off, stream, who);
}

int32_t gs_csr_weighted_blocks_plan(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                    int64_t n_nodes, int64_t nnz, const int32_t* seeds, int64_t n_seeds, int32_t n_layers,
                                    const int32_t* fanouts, uint64_t seed, uint64_t call, void* workspace,
                                    int64_t workspace_bytes, int64_t* counts_dev, void* stream) {
  const char* who = "gs_csr_weighted_blocks_plan";
  GS_REQUIRE(fanouts != nullptr, "%s: NULL fanouts", who);
  return gs::blocks_plan(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, fanouts, seed, call, workspace,
                         workspace_bytes, counts_dev, stream, who, true, sample_weight);
}

int32_t gs_csr_weighted_blocks_fill(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                    int64_t n_nodes, int64_t nnz, const int32_t* seeds, int64_t n_seeds, int32_t n_layers,
                                    const int32_t* fanouts, uint64_t seed, uint64_t call, void* workspace,
                                    int64_t workspace_bytes, const int64_t* counts, int32_t* const* src_ids,
                                    int64_t* const* b_indptr, int32_t* const* b_indices, int32_t* const* b_rows,
                                    void* stream) {
  const char* who = "gs_csr_weighted_blocks_fill";
  GS_REQUIRE(fanouts != nullptr, "%s: NULL fanouts", who);
  return gs::blocks_fill(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, fanouts, seed, call, workspace,
                         workspace_bytes, counts, src_ids, b_indptr, b_indices, b_rows, nullptr, stream, who, true,
                         sample_weight);
}

int32_t gs_csr_weighted_blocks_fill_offsets(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                            int64_t n_nodes, int64_t nnz, const int32_t* seeds, int64_t n_seeds,
                                            int32_t n_layers, const int32_t* fanouts, uint64_t seed, uint64_t call,
                                            void* workspace, int64_t workspace_bytes, const int64_t* counts,
                                            int32_t* const* src_ids, int64_t* const* b_indptr,
                                            int32_t* const* b_indices, int32_t* const* b_rows, int32_t* const* b_off,
                                            void* stream) {
  const char* who = "gs_csr_weighted_blocks_fill_offsets";
  GS_REQUIRE(fanouts != nullptr && b_off != nullptr, "%s: NULL fanouts or offsets", who);
  return gs::blocks_fill(indptr, indices, n_nodes, nnz, seeds, n_seeds, n_layers, fanouts, seed, call, workspace,
                         workspace_bytes, counts, src_ids, b_indptr, b_indices, b_rows, b_off, stream, who, true,
                         sample_weight);
}

int64_t gs_csr_sample_rows_workspace_bytes(int64_t n_nodes, int64_t nnz) {
  size_t cub_bytes = 0, bytes = 0;
  if (gs::sample_rows_plan(n_nodes, nnz, cub_bytes, bytes, "gs_csr_sample_rows_workspace_bytes") != GS_OK) return -1;
  return (int64_t)bytes;
}

int32_t gs_csr_sample_rows(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz, int32_t k,
                           uint64_t seed, uint64_t call, int32_t layer, void* workspace, int64_t workspace_bytes,
                           int64_t* out_indptr, int32_t* out_indices, void* stream) {
  const char* who = "gs_csr_sample_rows";
  size_t cub_bytes = 0, bytes = 0;
  int32_t rc = gs::sample_rows_plan(n_nodes, nnz, cub_bytes, bytes, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(k >= 1 && k <= gs::kMaxFanout, "%s: fanout %d outside [1, %d]", who, k, gs::kMaxFanout);
  GS_REQUIRE(layer >= 0 && layer < GS_MAX_BLOCK_LAYERS, "%s: layer %d outside [0, %d)", who, layer, GS_MAX_BLOCK_LAYERS);
  GS_REQUIRE(indptr && out_indptr && (nnz == 0 || indices), "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)bytes);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* deg = (int64_t*)workspace;
  void* cub = (char*)workspace + gs::align256((size_t)(n_nodes + 1) * 8);
  const gs::SampleArgs sa = gs::make_sample_args(k, seed, call, layer);
  gs::blk_local_degree_kernel<true><<<gs::blk_grid(n_nodes + 1, gs::kBlkThreads, INT32_MAX), gs::kBlkThreads, 0, st>>>(
      indptr, n_nodes, nullptr, nullptr, n_nodes + 1, deg, sa);
  rc = gs::launch_check("blk_local_degree_kernel");
  if (rc != GS_OK) return rc;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(cub, cub_bytes, (const int64_t*)deg, out_indptr,
                                                        (int)(n_nodes + 1), st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceScan::ExclusiveSum");
  if (out_indices == nullptr || n_nodes == 0) return GS_OK;
  gs::blk_fill_kernel<true><<<gs::blk_grid(n_nodes, gs::kBlkWarps, (int64_t)gs::sm_count() * 16), gs::kBlkThreads, 0,
                              st>>>(indptr, indices, n_nodes, nullptr, nullptr, out_indptr, n_nodes, out_indices, sa);
  return gs::launch_check("blk_fill_kernel");
}

int32_t gs_csr_sample_rows_weighted(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                    int64_t n_nodes, int64_t nnz, int32_t k, uint64_t seed, uint64_t call, int32_t layer,
                                    void* workspace, int64_t workspace_bytes, int64_t* out_indptr, int32_t* out_indices,
                                    void* stream) {
  const char* who = "gs_csr_sample_rows_weighted";
  size_t cub_bytes = 0, bytes = 0;
  int32_t rc = gs::sample_rows_plan(n_nodes, nnz, cub_bytes, bytes, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(k >= 1 && k <= gs::kMaxFanout, "%s: fanout %d outside [1, %d]", who, k, gs::kMaxFanout);
  GS_REQUIRE(layer >= 0 && layer < GS_MAX_BLOCK_LAYERS, "%s: layer %d outside [0, %d)", who, layer, GS_MAX_BLOCK_LAYERS);
  GS_REQUIRE(indptr && out_indptr && (nnz == 0 || (indices && sample_weight)), "%s: NULL pointer", who);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)bytes, "%s: workspace of %lld bytes, %lld needed", who,
             (long long)workspace_bytes, (long long)bytes);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* deg = (int64_t*)workspace;
  void* cub = (char*)workspace + gs::align256((size_t)(n_nodes + 1) * 8);
  gs::wblk_degree_kernel<<<gs::blk_grid(n_nodes + 1, gs::kBlkWarps, (int64_t)gs::sm_count() * 16), gs::kBlkThreads, 0,
                           st>>>(indptr, sample_weight, n_nodes, nullptr, nullptr, nullptr, n_nodes + 1, deg, k);
  rc = gs::launch_check("wblk_degree_kernel");
  if (rc != GS_OK) return rc;
  cudaError_t e = gs_cub::cub::DeviceScan::ExclusiveSum(cub, cub_bytes, (const int64_t*)deg, out_indptr,
                                                        (int)(n_nodes + 1), st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceScan::ExclusiveSum");
  if (out_indices == nullptr || n_nodes == 0) return GS_OK;
  const gs::WSelRows r{indptr, indices, n_nodes, nullptr, nullptr, nullptr, nullptr, out_indptr, out_indices, nullptr,
                       n_nodes};
  return gs::launch_wblk_select<true, false>(r, gs::make_weight_args(sample_weight, k, seed, call, layer), n_nodes, st);
}

}  // extern "C"

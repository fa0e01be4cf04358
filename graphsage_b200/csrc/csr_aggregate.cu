// Full-neighbourhood reduction over variable-length CSR rows: the neighbour branch of layer-wise inference
// (SampleAndAggregate.full_neighbor_embeddings; contract in oracle/full_neighbor.py).
//   reference: tf.reduce_mean(neigh_vecs, axis=1)              graphsage/aggregators.py:48
//              mean(concat([neigh, self]), 1)  (GCN)           graphsage/aggregators.py:106-107
//              tf.reduce_max(neigh_h, axis=1)                  graphsage/aggregators.py:182
// with the fanout k made per row, and the plain sum GS_CSR_SUM, the backward of the means over the transposed graph
// (SupervisedGraphsage.full_neighbor_train_step; contract in oracle/full_neighbor_grad.py).  Every output element is ONE sequential chain over the row's entries in CSR order
// (the order of gs_gather_mean / gs_segment_max), so no work split may cut a row along its entries.  Two roles share
// one launch of 256-thread CTAs:
//   hub role (the first hub_blocks CTAs): rows with more than kCsrLong entries.  Work item = (chunk of 256 rows, slice of
//     32 columns); the CTA finds the long rows of its chunk and, per row, its 8 warps load 64 entries' slices into a
//     double-buffered shared tile while warp 0 sums the previous 64 in order.  A hub is spread over out_pitch / 32 CTAs
//     and keeps 64 rows in flight in each, instead of one warp walking 10^5 dependent steps.
//   short role (the rest): one warp per (row, slice of 32 * V columns), V columns per lane (float4 / 8 x bf16 loads),
//     kUnroll entries' loads in flight before they are summed in order.
// Hub CTAs come first in the grid, so the long rows start before the short ones fill the machine.
// kDrop (gs_csr_aggregate_dropout; contract in oracle/full_neighbor_dropout.py): every entry is masked where it is
// loaded - per entry and 4 columns one Philox call in the short role (the float4 / 8 x bf16 loads), in the hub role's
// loading warps before the tile is written, a quad of lanes sharing its 4 columns' calls through shuffles - so warp 0's
// ordered sum does no extra work.  The kDrop = false instantiations are the plain kernel.
#include <algorithm>

#include "common.cuh"

namespace gs {

constexpr int kCsrThreads = 256;
constexpr int64_t kCsrLong = 256;     // rows with more entries go to the hub role
constexpr int kHubChunk = 256;        // rows scanned per hub work item (one per thread)
constexpr int kHubCols = 32;          // columns per hub work item (one per lane of the summing warp)
constexpr int kHubPerWarp = 8;        // entries each warp loads per round
constexpr int kHubRows = kHubPerWarp * (kCsrThreads / 32);   // entries per round: 64

struct CsrArgs {
  const void* src;
  int64_t n_src_rows;
  int32_t F;
  int64_t pitch;
  const int64_t* indptr;
  const int32_t* indices;
  int64_t n_nodes;
  const int32_t* rows;
  int64_t n;
  float* out;
  int64_t out_pitch;
  int32_t n_slices;          // short role: ceil(out_pitch / (32 V))
  int32_t hub_slices;        // ceil(out_pitch / 32)
  int64_t hub_items;         // ceil(n / kHubChunk) * hub_slices
  int64_t hub_blocks;
  // kDrop only: the neighbour and self sites, the position map and (GS_CSR_SUM) the transposed entries' slots
  DropSite neigh, self;
  const int64_t* pos_indptr;
  const int32_t* pos_ids;
  int64_t pos_nnz;
  const int32_t* t_slot;
};

__device__ __forceinline__ int64_t csr_clamp(int64_t id, int64_t n_rows) { return (id < 0 || id >= n_rows) ? n_rows - 1 : id; }

// node of output row i and its entry range; cnt = 0 for an empty row or a node outside [0, n_nodes)
__device__ __forceinline__ int64_t csr_row(const CsrArgs& a, int64_t i, int64_t& lo, int64_t& cnt) {
  const int64_t v = a.rows ? (int64_t)__ldg(a.rows + i) : i;
  lo = 0;
  cnt = 0;
  if (v >= 0 && v < a.n_nodes) {
    lo = __ldg(a.indptr + v);
    cnt = __ldg(a.indptr + v + 1) - lo;
    if (cnt < 0) cnt = 0;
  }
  return v;
}

// source row of entry e; an empty row reduces over the dummy row (n_src_rows - 1) alone
__device__ __forceinline__ int64_t csr_entry(const CsrArgs& a, int64_t lo, int64_t cnt, int64_t e) {
  return cnt == 0 ? a.n_src_rows - 1 : csr_clamp((int64_t)__ldg(a.indices + lo + e), a.n_src_rows);
}

template <typename T, int V>
struct Loader;

template <>
struct Loader<float, 4> {
  static __device__ __forceinline__ void load(const CsrArgs& a, int64_t r, int c0, float (&x)[4]) {
    const float4 v = ldg_nc_f4(reinterpret_cast<const float4*>(static_cast<const float*>(a.src) + r * a.pitch + c0));
    x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
  }
};

template <>
struct Loader<float, 1> {
  static __device__ __forceinline__ void load(const CsrArgs& a, int64_t r, int c0, float (&x)[1]) {
    x[0] = __ldg(static_cast<const float*>(a.src) + r * a.pitch + c0);
  }
};

__device__ __forceinline__ float bf16_bits_to_f32(uint32_t b) { return __uint_as_float(b << 16); }

template <>
struct Loader<uint16_t, 8> {
  static __device__ __forceinline__ void load(const CsrArgs& a, int64_t r, int c0, float (&x)[8]) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(a.src) + r * a.pitch + c0));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      x[2 * q] = bf16_bits_to_f32(w[q] & 0xFFFFu);
      x[2 * q + 1] = bf16_bits_to_f32(w[q] >> 16);
    }
  }
};

template <typename T>
__device__ __forceinline__ float load_scalar(const CsrArgs& a, int64_t r, int c) {
  if constexpr (sizeof(T) == 2) return bf16_bits_to_f32(__ldg(static_cast<const uint16_t*>(a.src) + r * a.pitch + c));
  else return __ldg(static_cast<const float*>(a.src) + r * a.pitch + c);
}

// one step of the chain after its first entry (the max starts from x_0 itself, the means and the sum from +0)
template <int OP>
__device__ __forceinline__ float csr_step(float acc, float x) {
  if constexpr (OP == GS_CSR_MAX) return fmaxf(acc, x);
  else return acc + x;
}

// the chain's end: the mean's division (after the self row for GS_CSR_MEAN_SELF); the max and the sum end as they are
template <int OP>
__device__ __forceinline__ float csr_final(float acc, int64_t count, float self) {
  if constexpr (OP == GS_CSR_MAX || OP == GS_CSR_SUM) return acc;
  if constexpr (OP == GS_CSR_MEAN_SELF) return (acc + self) / (float)(count + 1);
  return acc / (float)count;
}

// ---- masks (kDrop) ----
// global node of local row v: v clamped to the dummy row n_nodes, then mapped through pos_ids
__device__ __forceinline__ int64_t drop_node(const CsrArgs& a, int64_t v) {
  const int64_t vc = (v < 0 || v >= a.n_nodes) ? a.n_nodes : v;
  return a.pos_ids ? (int64_t)__ldg(a.pos_ids + vc) : vc;
}

// position of a forward row's entry 0: its node's global CSR position, or nnz + node for the implicit dummy entry
__device__ __forceinline__ int64_t drop_row_base(const CsrArgs& a, int64_t node, int64_t cnt) {
  return cnt > 0 ? __ldg(a.pos_indptr + node) : a.pos_nnz + node;
}

struct DropEntry {
  int64_t pos;
  bool self;
};

// site and position of entry e of a row: a forward row's entries follow their node's row (base = drop_row_base); a
// transposed row's (GS_CSR_SUM) come from forward row i = indices[lo + e] at slot t_slot[lo + e] - entry j of i's row,
// -1 its implicit dummy entry, -2 its self entry (the self site at pos = node)
template <int OP>
__device__ __forceinline__ DropEntry drop_entry(const CsrArgs& a, int64_t lo, int64_t base, int64_t e) {
  if constexpr (OP != GS_CSR_SUM) {
    return {base + e, false};
  } else {
    const int64_t node = drop_node(a, __ldg(a.indices + lo + e));
    const int32_t s = __ldg(a.t_slot + lo + e);
    return {s >= 0 ? __ldg(a.pos_indptr + node) + s : s == -1 ? a.pos_nnz + node : node, s == -2};
  }
}

// x[q] = drop(x[q]) for columns c0 .. c0 + V - 1 at pos (one Philox call per 4 columns; c0 % 4 == 0 unless V == 1)
template <int V>
__device__ __forceinline__ void drop_vec(const DropSite& s, int64_t pos, int c0, float (&x)[V]) {
#pragma unroll
  for (int q = 0; q < V; q += 4) {
    const u32x4 w = drop_words(s, pos, (uint32_t)(c0 + q) >> 2);
#pragma unroll
    for (int e = 0; e < (V < 4 ? V : 4); ++e) x[q + e] = drop_one(s, pick(w, V == 1 ? (c0 & 3) : e), x[q + e]);
  }
}

// a quad of lanes (4 consecutive columns) computed the Philox blocks of 4 entries, entry u's in lane u of the quad: lane
// j gets word j of each, m[u] of entry u (a 4 x 4 transpose in 4 shuffles; every lane of the warp takes part)
__device__ __forceinline__ void quad_transpose(const u32x4& w, uint32_t (&m)[4]) {
  const int lane = threadIdx.x & 31, j = lane & 3;
  u32x4 got;
  got.x = __shfl_sync(0xffffffffu, pick(w, j), lane);
  got.y = __shfl_sync(0xffffffffu, pick(w, (j + 3) & 3), (lane & ~3) | ((j + 1) & 3));
  got.z = __shfl_sync(0xffffffffu, pick(w, (j + 2) & 3), (lane & ~3) | ((j + 2) & 3));
  got.w = __shfl_sync(0xffffffffu, pick(w, (j + 1) & 3), (lane & ~3) | ((j + 3) & 3));
#pragma unroll
  for (int u = 0; u < 4; ++u) m[u] = pick(got, (u - j) & 3);
}

// the hub role's masks of the warp's entries e0 .. e0 + kHubPerWarp - 1 of a row (cnt > kHubRows), loaded into r at
// column c; entries past the row are computed on its last entry and multiply a loaded 0
template <int OP>
__device__ __forceinline__ void hub_mask(const CsrArgs& a, int64_t lo, int64_t cnt, int64_t base, int64_t e0, int c,
                                         const DropSite& sn, const DropSite& ss, float (&r)[kHubPerWarp]) {
  const int j = threadIdx.x & 3;
#pragma unroll
  for (int h = 0; h < kHubPerWarp / 4; ++h) {
    const DropEntry mine = drop_entry<OP>(a, lo, base, min(e0 + 4 * h + j, cnt - 1));
    uint32_t m[4];
    quad_transpose(drop_words(mine.self ? ss : sn, mine.pos, (uint32_t)c >> 2), m);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int u = 4 * h + q;
      const bool self = OP == GS_CSR_SUM && drop_entry<OP>(a, lo, base, min(e0 + u, cnt - 1)).self;
      r[u] = drop_one(self ? ss : sn, m[q], r[u]);
    }
  }
}

template <typename T, int OP, bool kDrop>
__device__ void hub_role(const CsrArgs& a, float (*tile)[kHubRows][kHubCols], const DropSite& sn, const DropSite& ss) {
  __shared__ int32_t list[kHubChunk];
  __shared__ int32_t warp_count[kCsrThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t item = blockIdx.x; item < a.hub_items; item += a.hub_blocks) {
    const int64_t chunk = item / a.hub_slices;
    const int c = (int)(item % a.hub_slices) * kHubCols + lane;
    // the chunk's long rows, in row order (ballot + per-warp offsets: no atomics)
    const int64_t i0 = chunk * kHubChunk + threadIdx.x;
    int64_t lo, cnt = 0;
    if (i0 < a.n) csr_row(a, i0, lo, cnt);
    const bool is_long = cnt > kCsrLong;
    const uint32_t ballot = __ballot_sync(0xffffffffu, is_long);
    if (lane == 0) warp_count[warp] = __popc(ballot);
    __syncthreads();
    int off = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kCsrThreads / 32; ++w) {
      off += w < warp ? warp_count[w] : 0;
      total += warp_count[w];
    }
    if (is_long) list[off + __popc(ballot & ((1u << lane) - 1u))] = (int32_t)threadIdx.x;
    __syncthreads();
    for (int q = 0; q < total; ++q) {
      const int64_t i = chunk * kHubChunk + list[q];
      const int64_t v = csr_row(a, i, lo, cnt);
      const bool col_ok = c < a.F;
      float r[kHubPerWarp];
#pragma unroll
      for (int u = 0; u < kHubPerWarp; ++u) {
        const int e = warp * kHubPerWarp + u;
        r[u] = col_ok ? load_scalar<T>(a, csr_entry(a, lo, cnt, e), c) : 0.f;     // cnt > kHubRows
      }
      int64_t node = 0, pbase = 0;
      if constexpr (kDrop) {
        node = drop_node(a, v);
        if (OP != GS_CSR_SUM) pbase = drop_row_base(a, node, cnt);
        hub_mask<OP>(a, lo, cnt, pbase, warp * kHubPerWarp, c, sn, ss, r);
      }
      float acc = 0.f;
      int buf = 0;
      for (int64_t base = 0; base < cnt; base += kHubRows, buf ^= 1) {
#pragma unroll
        for (int u = 0; u < kHubPerWarp; ++u) tile[buf][warp * kHubPerWarp + u][lane] = r[u];
        __syncthreads();
        const int64_t next = base + kHubRows + warp * kHubPerWarp;
#pragma unroll
        for (int u = 0; u < kHubPerWarp; ++u)                 // the next round's loads are in flight during the sum
          r[u] = (col_ok && next + u < cnt) ? load_scalar<T>(a, csr_entry(a, lo, cnt, next + u), c) : 0.f;
        if constexpr (kDrop) hub_mask<OP>(a, lo, cnt, pbase, next, c, sn, ss, r);
        if (warp == 0) {
          const int m = (int)min((int64_t)kHubRows, cnt - base);
          int t = 0;
          if (OP == GS_CSR_MAX && base == 0) acc = tile[buf][t++][lane];
          for (; t < m; ++t) acc = csr_step<OP>(acc, tile[buf][t][lane]);
        }
      }
      if (warp == 0 && c < a.out_pitch) {
        float y = 0.f;
        if (col_ok) {
          float self = OP == GS_CSR_MEAN_SELF ? load_scalar<T>(a, csr_clamp(v, a.n_src_rows), c) : 0.f;
          if constexpr (kDrop && OP == GS_CSR_MEAN_SELF) self = drop_col(ss, node, c, self);
          y = csr_final<OP>(acc, cnt, self);
        }
        a.out[i * a.out_pitch + c] = y;
      }
      __syncthreads();      // the tiles are reused by the next row
    }
    __syncthreads();        // `list` and `warp_count` are rewritten by the next item
  }
}

template <typename T, int V, int OP, bool kDrop>
__device__ void short_role(const CsrArgs& a, int64_t block, const DropSite& sn, const DropSite& ss) {
  constexpr int kUnroll = V == 8 ? 4 : 8;      // 16-byte loads in flight per lane: 4 (bf16) or 8 (fp32 float4)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t items = a.n * a.n_slices;
  const int64_t stride = ((int64_t)gridDim.x - a.hub_blocks) * (kCsrThreads / 32);
  for (int64_t item = block * (kCsrThreads / 32) + warp; item < items; item += stride) {
    const int64_t i = item / a.n_slices;
    const int c0 = ((int)(item % a.n_slices) * 32 + lane) * V;
    int64_t lo, cnt;
    const int64_t v = csr_row(a, i, lo, cnt);
    if (cnt > kCsrLong || c0 >= a.out_pitch) continue;       // a hub row (hub role), or past the row's last column
    float acc[V];
#pragma unroll
    for (int q = 0; q < V; ++q) acc[q] = 0.f;
    if (c0 < a.F) {
      // an empty row: the dummy row alone, except for the sum, whose empty row is +0 (a node nobody points to)
      const int64_t count = OP == GS_CSR_SUM ? cnt : cnt > 0 ? cnt : 1;
      int64_t node = 0, pbase = 0;
      if constexpr (kDrop) {
        node = drop_node(a, v);
        if (OP != GS_CSR_SUM) pbase = drop_row_base(a, node, cnt);
      }
      int64_t e = 0;
      if constexpr (OP == GS_CSR_MAX) {
        float x0[V];
        Loader<T, V>::load(a, csr_entry(a, lo, cnt, e++), c0, x0);
#pragma unroll
        for (int q = 0; q < V; ++q) acc[q] = x0[q];
      }
      for (; e < count; e += kUnroll) {
        float x[kUnroll][V];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
          if (e + u < count) Loader<T, V>::load(a, csr_entry(a, lo, cnt, e + u), c0, x[u]);
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
          if (e + u < count) {
            if constexpr (kDrop) {
              const DropEntry d = drop_entry<OP>(a, lo, pbase, e + u);
              drop_vec<V>(d.self ? ss : sn, d.pos, c0, x[u]);
            }
#pragma unroll
            for (int q = 0; q < V; ++q) acc[q] = csr_step<OP>(acc[q], x[u][q]);
          }
      }
      float self[V];
#pragma unroll
      for (int q = 0; q < V; ++q) self[q] = 0.f;
      if (OP == GS_CSR_MEAN_SELF) Loader<T, V>::load(a, csr_clamp(v, a.n_src_rows), c0, self);
      if constexpr (kDrop && OP == GS_CSR_MEAN_SELF) drop_vec<V>(ss, node, c0, self);
#pragma unroll
      for (int q = 0; q < V; ++q) acc[q] = c0 + q < a.F ? csr_final<OP>(acc[q], count, self[q]) : 0.f;
    }
    float* dst = a.out + i * a.out_pitch + c0;
    if constexpr (V == 1) {
      dst[0] = acc[0];
    } else {
#pragma unroll
      for (int q = 0; q < V; q += 4) *reinterpret_cast<float4*>(dst + q) = make_float4(acc[q], acc[q + 1], acc[q + 2], acc[q + 3]);
    }
  }
}

template <typename T, int V, int OP, bool kDrop>
__global__ void __launch_bounds__(kCsrThreads, 3) csr_aggregate_kernel(const __grid_constant__ CsrArgs a) {
  __shared__ __align__(16) float tile[2][kHubRows][kHubCols];
  DropSite sn = a.neigh, ss = a.self;
  if constexpr (kDrop) {
    sn.call += drop_call_offset(sn);
    ss.call += drop_call_offset(ss);
  }
  if (blockIdx.x < a.hub_blocks) hub_role<T, OP, kDrop>(a, tile, sn, ss);
  else short_role<T, V, OP, kDrop>(a, (int64_t)blockIdx.x - a.hub_blocks, sn, ss);
}

template <typename T, int V>
static void launch_csr(int32_t op, unsigned blocks, const CsrArgs& a, cudaStream_t st) {
  if (op == GS_CSR_MEAN) csr_aggregate_kernel<T, V, GS_CSR_MEAN, false><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MEAN_SELF) csr_aggregate_kernel<T, V, GS_CSR_MEAN_SELF, false><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MAX) csr_aggregate_kernel<T, V, GS_CSR_MAX, false><<<blocks, kCsrThreads, 0, st>>>(a);
  else if constexpr (sizeof(T) == 4) csr_aggregate_kernel<T, V, GS_CSR_SUM, false><<<blocks, kCsrThreads, 0, st>>>(a);
}

// the masked instantiations: the means, and the sum over fp32 sources
template <typename T, int V>
static void launch_csr_drop(int32_t op, unsigned blocks, const CsrArgs& a, cudaStream_t st) {
  if (op == GS_CSR_MEAN) csr_aggregate_kernel<T, V, GS_CSR_MEAN, true><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MEAN_SELF) csr_aggregate_kernel<T, V, GS_CSR_MEAN_SELF, true><<<blocks, kCsrThreads, 0, st>>>(a);
  else if constexpr (sizeof(T) == 4) csr_aggregate_kernel<T, V, GS_CSR_SUM, true><<<blocks, kCsrThreads, 0, st>>>(a);
}

struct CsrDrop {
  gs_dropout_site neigh, self;
  const int64_t* pos_indptr;
  const int32_t* pos_ids;
  int64_t pos_nnz;
  const int32_t* t_slot;
};

static int32_t csr_aggregate(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                             const int64_t* indptr, const int32_t* indices, int64_t n_nodes, const int32_t* rows, int64_t n,
                             int32_t op, float* out, int64_t out_pitch, void* stream, const CsrDrop* drop, const char* who) {
  GS_REQUIRE(op == GS_CSR_MEAN || op == GS_CSR_MEAN_SELF || op == GS_CSR_MAX || op == GS_CSR_SUM, "%s: unknown op %d", who,
             (int)op);
  GS_REQUIRE(dtype == GS_F32 || dtype == GS_BF16, "%s: dtype must be GS_F32 or GS_BF16", who);
  GS_REQUIRE(op != GS_CSR_SUM || dtype == GS_F32, "%s: GS_CSR_SUM reads fp32 sources only", who);
  GS_REQUIRE(n >= 0 && n_nodes >= 0 && F >= 1 && pitch >= F && out_pitch >= F, "%s: bad sizes", who);
  GS_REQUIRE(out_pitch < (1LL << 30), "%s: out_pitch must be < 2^30", who);
  if (n == 0) return GS_OK;
  GS_REQUIRE(n_src_rows >= 1, "%s: the source table needs at least its dummy row", who);
  GS_REQUIRE(src && out, "%s: NULL src or out", who);
  GS_REQUIRE(n_nodes == 0 || (indptr && indices), "%s: NULL indptr or indices", who);
  const uintptr_t sa = (uintptr_t)src, oa = (uintptr_t)out;
  int V = 1;
  if (dtype == GS_BF16) {
    GS_REQUIRE(pitch % 8 == 0 && out_pitch % 8 == 0 && sa % 16 == 0 && oa % 16 == 0,
               "%s: a bfloat16 table needs 16-byte rows and pointers (pitch %% 8 == 0, out_pitch %% 8 == 0)", who);
    V = 8;
  } else if (pitch % 4 == 0 && out_pitch % 4 == 0 && sa % 16 == 0 && oa % 16 == 0) {
    V = 4;
  }
  CsrArgs a{src, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, out, out_pitch, 0, 0, 0, 0};
  memset(&a.neigh, 0, sizeof(a.neigh));
  memset(&a.self, 0, sizeof(a.self));
  a.pos_indptr = nullptr;
  a.pos_ids = a.t_slot = nullptr;
  a.pos_nnz = 0;
  if (drop) {
    a.neigh = make_drop_site(drop->neigh);
    a.self = make_drop_site(drop->self);
    a.pos_indptr = drop->pos_indptr;
    a.pos_ids = drop->pos_ids;
    a.pos_nnz = drop->pos_nnz;
    a.t_slot = drop->t_slot;
  }
  a.n_slices = (int32_t)((out_pitch + 32 * V - 1) / (32 * V));
  a.hub_slices = (int32_t)((out_pitch + kHubCols - 1) / kHubCols);
  a.hub_items = (n + kHubChunk - 1) / kHubChunk * a.hub_slices;
  a.hub_blocks = std::min<int64_t>(a.hub_items, (int64_t)sm_count() * 4);
  const int64_t short_items = n * a.n_slices;
  const int64_t short_blocks = std::min<int64_t>((short_items + 7) / 8, (int64_t)sm_count() * 8 * 64);
  const unsigned blocks = (unsigned)(a.hub_blocks + short_blocks);
  cudaStream_t st = (cudaStream_t)stream;
  if (drop) {
    if (dtype == GS_BF16) launch_csr_drop<uint16_t, 8>(op, blocks, a, st);
    else if (V == 4) launch_csr_drop<float, 4>(op, blocks, a, st);
    else launch_csr_drop<float, 1>(op, blocks, a, st);
    return launch_check("csr_aggregate_kernel<drop>");
  }
  if (dtype == GS_BF16) launch_csr<uint16_t, 8>(op, blocks, a, st);
  else if (V == 4) launch_csr<float, 4>(op, blocks, a, st);
  else launch_csr<float, 1>(op, blocks, a, st);
  return launch_check("csr_aggregate_kernel");
}

static int32_t check_site(const gs_dropout_site& s, const char* who) {
  GS_REQUIRE(s.rate >= 0.f && s.rate < 1.f, "%s: dropout rate %g outside [0, 1)", who, (double)s.rate);
  return GS_OK;
}

}  // namespace gs

extern "C" {

int32_t gs_csr_aggregate(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch, const int64_t* indptr,
                         const int32_t* indices, int64_t n_nodes, const int32_t* rows, int64_t n, int32_t op, float* out,
                         int64_t out_pitch, void* stream) {
  return gs::csr_aggregate(src, dtype, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, op, out, out_pitch, stream,
                           nullptr, "gs_csr_aggregate");
}

int32_t gs_csr_aggregate_dropout(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                 const int64_t* indptr, const int32_t* indices, const int32_t* t_slot, int64_t n_nodes,
                                 const int32_t* rows, int64_t n, int32_t op, gs_dropout_site neigh_site,
                                 gs_dropout_site self_site, const int64_t* pos_indptr, const int32_t* pos_ids,
                                 int64_t pos_nnz, float* out, int64_t out_pitch, void* stream) {
  const char* who = "gs_csr_aggregate_dropout";
  GS_REQUIRE(op == GS_CSR_MEAN || op == GS_CSR_MEAN_SELF || op == GS_CSR_SUM, "%s: op must be GS_CSR_MEAN, "
             "GS_CSR_MEAN_SELF or GS_CSR_SUM (got %d)", who, (int)op);
  int32_t rc = gs::check_site(neigh_site, who);
  if (rc == GS_OK) rc = gs::check_site(self_site, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(pos_nnz >= 0, "%s: pos_nnz < 0", who);
  if (neigh_site.rate == 0.f && self_site.rate == 0.f)      // every mask keeps and divides by 1: the plain kernel
    return gs::csr_aggregate(src, dtype, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, op, out, out_pitch, stream,
                             nullptr, who);
  GS_REQUIRE(n == 0 || pos_indptr, "%s: NULL pos_indptr", who);
  GS_REQUIRE(op != GS_CSR_SUM || n == 0 || t_slot, "%s: GS_CSR_SUM needs t_slot", who);
  const gs::CsrDrop drop{neigh_site, self_site, pos_indptr, pos_ids, pos_nnz, op == GS_CSR_SUM ? t_slot : nullptr};
  return gs::csr_aggregate(src, dtype, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, op, out, out_pitch, stream,
                           &drop, who);
}

}  // extern "C"

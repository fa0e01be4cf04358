// Full-neighbourhood reduction over variable-length CSR rows: the neighbour branch of layer-wise inference
// (SampleAndAggregate.full_neighbor_embeddings; contract in oracle/full_neighbor.py).
//   reference: tf.reduce_mean(neigh_vecs, axis=1)              graphsage/aggregators.py:48
//              mean(concat([neigh, self]), 1)  (GCN)           graphsage/aggregators.py:106-107
//              tf.reduce_max(neigh_h, axis=1)                  graphsage/aggregators.py:182
// with the fanout k made per row, and the plain sum GS_CSR_SUM, the backward of the means over the transposed graph
// (SupervisedGraphsage.full_neighbor_train_step; contract in oracle/full_neighbor_grad.py).  Every output element is ONE
// sequential chain over the row's entries in CSR order (the order of gs_gather_mean / gs_segment_max), run on the hub /
// short row schedule of csr_rows.cuh; the short role reads V columns per lane (float4 / 8 x bf16 loads).
// kDrop (gs_csr_aggregate_dropout; contract in oracle/full_neighbor_dropout.py): every entry is masked where it is
// loaded - per entry and 4 columns one Philox call in the short role (the float4 / 8 x bf16 loads), in the hub role's
// loading warps before the tile is written, a quad of lanes sharing its 4 columns' calls through shuffles - so warp 0's
// ordered sum does no extra work.  The kDrop = false instantiations are the plain kernel.
// kOff (gs_csr_aggregate_dropout_offsets; contract in oracle/sampled_blocks_dropout.py): a sampled block's row keeps
// only some entries of its node's raw row, so entry e is masked at pos_indptr[g] + pos_off[lo + e] (its offset in the raw
// row) instead of + e; the implicit dummy entry of an empty row keeps pos_nnz + g.  The means only: the transposed sum
// of a sampled block reads t_slot already mapped through the offsets.
// kW (gs_csr_aggregate_weighted; contract in oracle/weighted.py): entry e's term is fl(weight[lo + e] * x), rounded to
// fp32 before it joins the chain (__fmul_rn: never contracted into the sum), 1 for an empty row's dummy entry.  The short
// role loads the weight beside the entry's index and columns (weight()) and scales where the term is consumed (scale()),
// so all kUnroll entries' loads stay in flight; the hub role's loading warps scale their terms in hub_mask(), after the
// round's loads are issued and before the tile is written, so warp 0's ordered sum is unchanged.  All four ops; the
// sum's weights are aligned with its own (transposed) indices.
#include "csr_rows.cuh"

namespace gs {

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
  const int32_t* pos_off;    // kOff only: each entry's offset in its node's raw CSR row
  const float* weight;       // kW only: one weight per entry of indices
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

template <>
struct Loader<uint16_t, 1> {
  static __device__ __forceinline__ void load(const CsrArgs& a, int64_t r, int c0, float (&x)[1]) {
    x[0] = bf16_bits_to_f32(__ldg(static_cast<const uint16_t*>(a.src) + r * a.pitch + c0));
  }
};

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

// the aggregate on the csr_rows.cuh schedule: the rows of `rows` (or 0 .. n - 1), entries read from src, written up to
// out_pitch with columns F .. out_pitch - 1 zero-filled
template <typename T, int OP, bool kDrop, bool kOff = false, bool kW = false>
struct AggregateRows {
  static constexpr bool kFromFirst = OP == GS_CSR_MAX;
  static constexpr bool kEmptyIsDummy = OP != GS_CSR_SUM;   // the sum's empty row is +0 (a node nobody points to)
  const CsrArgs& a;
  const DropSite& sn;                                  // kDrop: the neighbour and self sites
  const DropSite& ss;

  struct Row {
    int64_t v, lo, cnt;
    int64_t node = 0, pbase = 0;                       // kDrop: global node, position of entry 0 (drop_row_base)
  };

  __device__ __forceinline__ int64_t rows() const { return a.n; }
  __device__ __forceinline__ int32_t hub_slices() const { return a.hub_slices; }
  __device__ __forceinline__ int32_t slices() const { return a.n_slices; }
  __device__ __forceinline__ int64_t out_cols() const { return a.out_pitch; }

  __device__ __forceinline__ Row row(int64_t i) const {
    Row r;
    r.v = csr_row(a, i, r.lo, r.cnt);
    return r;
  }

  __device__ __forceinline__ void begin(Row& r, int64_t, int, bool) const {
    if constexpr (kDrop) {
      r.node = drop_node(a, r.v);
      if (OP != GS_CSR_SUM) r.pbase = drop_row_base(a, r.node, r.cnt);
    }
  }

  template <int W>
  __device__ __forceinline__ void load(const Row& r, int64_t e, int c0, bool ok, float (&x)[W]) const {
    if (ok) Loader<T, W>::load(a, csr_entry(a, r.lo, r.cnt, e), c0, x);
  }

  // kW: entry e's weight (an empty row's one entry is its dummy, of weight 1), and its scaling of the loaded columns
  __device__ __forceinline__ float weight(const Row& r, int64_t e, bool ok) const {
    if constexpr (kW) return (ok && r.cnt > 0) ? __ldg(a.weight + r.lo + e) : 1.f;
    else return 1.f;
  }

  template <int W>
  __device__ __forceinline__ void scale(float w, float (&x)[W]) const {
    if constexpr (kW) {
#pragma unroll
      for (int q = 0; q < W; ++q) x[q] = __fmul_rn(w, x[q]);
    }
  }

  __device__ __forceinline__ float value(const Row& r, int64_t e, int c) const {
    float x[1];
    load(r, e, c, true, x);
    return x[0];
  }

  // site and position of entry e of row r (kOff: entry 0's position plus the entry's raw-row offset; an empty row's
  // one entry is its dummy, at pbase itself)
  __device__ __forceinline__ DropEntry entry(const Row& r, int64_t e) const {
    if constexpr (kOff) return {r.pbase + (r.cnt > 0 ? (int64_t)__ldg(a.pos_off + r.lo + e) : 0), false};
    else return drop_entry<OP>(a, r.lo, r.pbase, e);
  }

  template <int W>
  __device__ __forceinline__ void mask(const Row& r, int64_t e, int c0, float (&x)[W]) const {
    if constexpr (kDrop) {
      const DropEntry d = entry(r, e);
      drop_vec<W>(d.self ? ss : sn, d.pos, c0, x);
    }
  }

  // the masks (kDrop) or weights (kW) of the warp's entries e0 .. e0 + kHubPerWarp - 1 of a hub row (cnt > kHubRows) at
  // column c; entries past the row are computed on its last entry and multiply a loaded 0
  __device__ __forceinline__ void hub_mask(const Row& r, int64_t e0, int c, float (&x)[kHubPerWarp]) const {
    if constexpr (kW) {
      float w[kHubPerWarp];
#pragma unroll
      for (int u = 0; u < kHubPerWarp; ++u) w[u] = __ldg(a.weight + r.lo + min(e0 + u, r.cnt - 1));
#pragma unroll
      for (int u = 0; u < kHubPerWarp; ++u) x[u] = __fmul_rn(w[u], x[u]);
    }
    if constexpr (kDrop) {
      const int j = threadIdx.x & 3;
#pragma unroll
      for (int h = 0; h < kHubPerWarp / 4; ++h) {
        const DropEntry mine = entry(r, min(e0 + 4 * h + j, r.cnt - 1));
        uint32_t m[4];
        quad_transpose(drop_words(mine.self ? ss : sn, mine.pos, (uint32_t)c >> 2), m);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int u = 4 * h + q;
          const bool self = OP == GS_CSR_SUM && drop_entry<OP>(a, r.lo, r.pbase, min(e0 + u, r.cnt - 1)).self;
          x[u] = drop_one(self ? ss : sn, m[q], x[u]);
        }
      }
    }
  }

  __device__ __forceinline__ float step(float acc, float x) const {
    if constexpr (OP == GS_CSR_MAX) return fmaxf(acc, x);
    else return acc + x;
  }

  template <int W>
  __device__ __forceinline__ void finish(const Row& r, int c0, int64_t count, float (&acc)[W]) const {
    float self[W];
#pragma unroll
    for (int q = 0; q < W; ++q) self[q] = 0.f;
    if (OP == GS_CSR_MEAN_SELF) Loader<T, W>::load(a, csr_clamp(r.v, a.n_src_rows), c0, self);
    if constexpr (kDrop && OP == GS_CSR_MEAN_SELF) drop_vec<W>(ss, r.node, c0, self);
#pragma unroll
    for (int q = 0; q < W; ++q) acc[q] = c0 + q < a.F ? csr_final<OP>(acc[q], count, self[q]) : 0.f;
  }

  template <int W>
  __device__ __forceinline__ void store(const Row&, int64_t i, int c0, const float (&acc)[W]) const {
    float* dst = a.out + i * a.out_pitch + c0;
    if constexpr (W == 1) {
      dst[0] = acc[0];
    } else {
#pragma unroll
      for (int q = 0; q < W; q += 4) *reinterpret_cast<float4*>(dst + q) = make_float4(acc[q], acc[q + 1], acc[q + 2], acc[q + 3]);
    }
  }
};

template <typename T, int V, int OP, bool kDrop, bool kOff = false, bool kW = false>
__global__ void __launch_bounds__(kCsrThreads, 3) csr_aggregate_kernel(const __grid_constant__ CsrArgs a) {
  __shared__ __align__(16) float tile[2][kHubRows][kHubCols];
  DropSite sn = a.neigh, ss = a.self;
  if constexpr (kDrop) {
    sn.call += drop_call_offset(sn);
    ss.call += drop_call_offset(ss);
  }
  // short role: 16-byte loads in flight per lane: 4 (bf16) or 8 (fp32 float4)
  csr_rows<V, V == 8 ? 4 : 8>(AggregateRows<T, OP, kDrop, kOff, kW>{a, sn, ss}, tile);
}

template <typename T, int V>
static void launch_csr(int32_t op, unsigned blocks, const CsrArgs& a, cudaStream_t st) {
  if (op == GS_CSR_MEAN) csr_aggregate_kernel<T, V, GS_CSR_MEAN, false><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MEAN_SELF) csr_aggregate_kernel<T, V, GS_CSR_MEAN_SELF, false><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MAX) csr_aggregate_kernel<T, V, GS_CSR_MAX, false><<<blocks, kCsrThreads, 0, st>>>(a);
  else if constexpr (sizeof(T) == 4) csr_aggregate_kernel<T, V, GS_CSR_SUM, false><<<blocks, kCsrThreads, 0, st>>>(a);
}

// the weighted instantiations: every op, the sum over fp32 sources only
template <typename T, int V>
static void launch_csr_weighted(int32_t op, unsigned blocks, const CsrArgs& a, cudaStream_t st) {
  if (op == GS_CSR_MEAN) csr_aggregate_kernel<T, V, GS_CSR_MEAN, false, false, true><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MEAN_SELF) csr_aggregate_kernel<T, V, GS_CSR_MEAN_SELF, false, false, true><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MAX) csr_aggregate_kernel<T, V, GS_CSR_MAX, false, false, true><<<blocks, kCsrThreads, 0, st>>>(a);
  else if constexpr (sizeof(T) == 4) csr_aggregate_kernel<T, V, GS_CSR_SUM, false, false, true><<<blocks, kCsrThreads, 0, st>>>(a);
}

// the masked instantiations: the means, and the sum over fp32 sources; with per-entry offsets (kOff), the means only
template <typename T, int V, bool kOff>
static void launch_csr_drop(int32_t op, unsigned blocks, const CsrArgs& a, cudaStream_t st) {
  if (op == GS_CSR_MEAN) csr_aggregate_kernel<T, V, GS_CSR_MEAN, true, kOff><<<blocks, kCsrThreads, 0, st>>>(a);
  else if (op == GS_CSR_MEAN_SELF) csr_aggregate_kernel<T, V, GS_CSR_MEAN_SELF, true, kOff><<<blocks, kCsrThreads, 0, st>>>(a);
  else if constexpr (sizeof(T) == 4 && !kOff) csr_aggregate_kernel<T, V, GS_CSR_SUM, true><<<blocks, kCsrThreads, 0, st>>>(a);
}

struct CsrDrop {
  gs_dropout_site neigh, self;
  const int64_t* pos_indptr;
  const int32_t* pos_ids;
  int64_t pos_nnz;
  const int32_t* t_slot;
  const int32_t* pos_off;
};

static int32_t csr_aggregate(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                             const int64_t* indptr, const int32_t* indices, int64_t n_nodes, const int32_t* rows, int64_t n,
                             int32_t op, float* out, int64_t out_pitch, void* stream, const CsrDrop* drop, const char* who,
                             const float* weight = nullptr) {
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
  a.pos_ids = a.t_slot = a.pos_off = nullptr;
  a.pos_nnz = 0;
  a.weight = weight;
  if (drop) {
    a.neigh = make_drop_site(drop->neigh);
    a.self = make_drop_site(drop->self);
    a.pos_indptr = drop->pos_indptr;
    a.pos_ids = drop->pos_ids;
    a.pos_nnz = drop->pos_nnz;
    a.t_slot = drop->t_slot;
    a.pos_off = drop->pos_off;
  }
  a.n_slices = (int32_t)((out_pitch + 32 * V - 1) / (32 * V));
  a.hub_slices = (int32_t)((out_pitch + kHubCols - 1) / kHubCols);
  const unsigned blocks = csr_grid(n, a.hub_slices, a.n_slices, a.hub_items, a.hub_blocks);
  cudaStream_t st = (cudaStream_t)stream;
  if (weight) {
    if (dtype == GS_BF16) launch_csr_weighted<uint16_t, 8>(op, blocks, a, st);
    else if (V == 4) launch_csr_weighted<float, 4>(op, blocks, a, st);
    else launch_csr_weighted<float, 1>(op, blocks, a, st);
    return launch_check("csr_aggregate_kernel<weighted>");
  }
  if (drop && drop->pos_off) {
    if (dtype == GS_BF16) launch_csr_drop<uint16_t, 8, true>(op, blocks, a, st);
    else if (V == 4) launch_csr_drop<float, 4, true>(op, blocks, a, st);
    else launch_csr_drop<float, 1, true>(op, blocks, a, st);
    return launch_check("csr_aggregate_kernel<drop, offsets>");
  }
  if (drop) {
    if (dtype == GS_BF16) launch_csr_drop<uint16_t, 8, false>(op, blocks, a, st);
    else if (V == 4) launch_csr_drop<float, 4, false>(op, blocks, a, st);
    else launch_csr_drop<float, 1, false>(op, blocks, a, st);
    return launch_check("csr_aggregate_kernel<drop>");
  }
  if (dtype == GS_BF16) launch_csr<uint16_t, 8>(op, blocks, a, st);
  else if (V == 4) launch_csr<float, 4>(op, blocks, a, st);
  else launch_csr<float, 1>(op, blocks, a, st);
  return launch_check("csr_aggregate_kernel");
}

}  // namespace gs

extern "C" {

int32_t gs_csr_aggregate(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch, const int64_t* indptr,
                         const int32_t* indices, int64_t n_nodes, const int32_t* rows, int64_t n, int32_t op, float* out,
                         int64_t out_pitch, void* stream) {
  return gs::csr_aggregate(src, dtype, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, op, out, out_pitch, stream,
                           nullptr, "gs_csr_aggregate");
}

int32_t gs_csr_aggregate_weighted(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                  const int64_t* indptr, const int32_t* indices, const float* weight, int64_t n_nodes,
                                  const int32_t* rows, int64_t n, int32_t op, float* out, int64_t out_pitch,
                                  void* stream) {
  const char* who = "gs_csr_aggregate_weighted";
  GS_REQUIRE(weight || n == 0 || n_nodes == 0, "%s: NULL weight", who);
  // with no node, every row reduces over the dummy entry alone (weight 1): the plain kernel
  return gs::csr_aggregate(src, dtype, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, op, out, out_pitch, stream,
                           nullptr, who, n_nodes == 0 ? nullptr : weight);
}

}  // extern "C"

namespace gs {

// gs_csr_aggregate_dropout, or with pos_off (the means only) gs_csr_aggregate_dropout_offsets
static int32_t csr_aggregate_dropout(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                     const int64_t* indptr, const int32_t* indices, const int32_t* t_slot,
                                     int64_t n_nodes, const int32_t* rows, int64_t n, int32_t op,
                                     gs_dropout_site neigh_site, gs_dropout_site self_site, const int64_t* pos_indptr,
                                     const int32_t* pos_ids, int64_t pos_nnz, const int32_t* pos_off, float* out,
                                     int64_t out_pitch, void* stream, const char* who) {
  int32_t rc = check_site(neigh_site, who);
  if (rc == GS_OK) rc = check_site(self_site, who);
  if (rc != GS_OK) return rc;
  GS_REQUIRE(pos_nnz >= 0, "%s: pos_nnz < 0", who);
  if (neigh_site.rate == 0.f && self_site.rate == 0.f)      // every mask keeps and divides by 1: the plain kernel
    return csr_aggregate(src, dtype, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, op, out, out_pitch, stream,
                         nullptr, who);
  GS_REQUIRE(n == 0 || pos_indptr, "%s: NULL pos_indptr", who);
  GS_REQUIRE(op != GS_CSR_SUM || n == 0 || t_slot, "%s: GS_CSR_SUM needs t_slot", who);
  const CsrDrop drop{neigh_site, self_site, pos_indptr, pos_ids, pos_nnz, op == GS_CSR_SUM ? t_slot : nullptr, pos_off};
  return csr_aggregate(src, dtype, n_src_rows, F, pitch, indptr, indices, n_nodes, rows, n, op, out, out_pitch, stream,
                       &drop, who);
}

}  // namespace gs

extern "C" {

int32_t gs_csr_aggregate_dropout(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                 const int64_t* indptr, const int32_t* indices, const int32_t* t_slot, int64_t n_nodes,
                                 const int32_t* rows, int64_t n, int32_t op, gs_dropout_site neigh_site,
                                 gs_dropout_site self_site, const int64_t* pos_indptr, const int32_t* pos_ids,
                                 int64_t pos_nnz, float* out, int64_t out_pitch, void* stream) {
  const char* who = "gs_csr_aggregate_dropout";
  GS_REQUIRE(op == GS_CSR_MEAN || op == GS_CSR_MEAN_SELF || op == GS_CSR_SUM, "%s: op must be GS_CSR_MEAN, "
             "GS_CSR_MEAN_SELF or GS_CSR_SUM (got %d)", who, (int)op);
  return gs::csr_aggregate_dropout(src, dtype, n_src_rows, F, pitch, indptr, indices, t_slot, n_nodes, rows, n, op,
                                   neigh_site, self_site, pos_indptr, pos_ids, pos_nnz, nullptr, out, out_pitch, stream,
                                   who);
}

int32_t gs_csr_aggregate_dropout_offsets(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                         const int64_t* indptr, const int32_t* indices, int64_t n_nodes,
                                         const int32_t* rows, int64_t n, int32_t op, gs_dropout_site neigh_site,
                                         gs_dropout_site self_site, const int64_t* pos_indptr, const int32_t* pos_ids,
                                         int64_t pos_nnz, const int32_t* pos_off, float* out, int64_t out_pitch,
                                         void* stream) {
  const char* who = "gs_csr_aggregate_dropout_offsets";
  GS_REQUIRE(op == GS_CSR_MEAN || op == GS_CSR_MEAN_SELF, "%s: op must be GS_CSR_MEAN or GS_CSR_MEAN_SELF (got %d)",
             who, (int)op);
  GS_REQUIRE(n == 0 || pos_off, "%s: NULL pos_off", who);
  return gs::csr_aggregate_dropout(src, dtype, n_src_rows, F, pitch, indptr, indices, nullptr, n_nodes, rows, n, op,
                                   neigh_site, self_site, pos_indptr, pos_ids, pos_nnz, pos_off, out, out_pitch, stream,
                                   who);
}

}  // extern "C"

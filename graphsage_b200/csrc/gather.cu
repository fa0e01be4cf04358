// K2 / K3a: K-hop feature-row gather and the fused gather + fixed-fanout segmented mean.
//   reference: tf.nn.embedding_lookup(features, samples[h])      graphsage/models.py:299
//              tf.reduce_mean(neigh_vecs, axis=1)                graphsage/aggregators.py:48
//              mean(concat([neigh, self]), 1)  (GCN)             graphsage/aggregators.py:106-107
//              tf.reduce_max(neigh_h, axis=1)                    graphsage/aggregators.py:182
//              tf.nn.l2_normalize(x, 1)                          graphsage/models.py:368
// HBM-bound byte movement: rows are 2.4 KB (F=602 fp32), fetched whole.  Two data paths:
//   variant 1 (default when rows are 16-B multiples): the TMA bulk-copy engine
//     (cp.async.bulk global->shared, mbarrier complete_tx) stages whole rows in shared memory;
//   variant 0: 128-bit ld.global.nc loads, k independent loads in flight per thread.
#include "common.cuh"

namespace gs {

struct SegTable {
  gs_segment s[GS_MAX_SEGMENTS];
  int32_t n_segments;
  int64_t total_rows;
};

// segment of flattened row r: the last segment whose cumulative start is <= r.  The comparison is against the cumulative end
// of segment q, which never decreases, so a later shorter (or empty) segment cannot claim a row an earlier one holds.
__device__ __forceinline__ int find_segment(const SegTable& t, int64_t r, int64_t& local) {
  int si = 0;
  int64_t base = 0, end = 0;
#pragma unroll
  for (int q = 0; q < GS_MAX_SEGMENTS - 1; ++q) {
    if (q < t.n_segments - 1) {
      end += t.s[q].n;
      if (r >= end) {
        base = end;
        si = q + 1;
      }
    }
  }
  local = r - base;
  return si;
}

__device__ __forceinline__ int64_t clamp_row(int64_t id, int64_t n_rows) {
  return (id < 0 || id >= n_rows) ? n_rows - 1 : id;
}

__device__ __forceinline__ float4 mask_tail(float4 v, int col0, int F) {
  if (col0 + 1 >= F) v.y = 0.f;
  if (col0 + 2 >= F) v.z = 0.f;
  if (col0 + 3 >= F) v.w = 0.f;
  return v;
}

// ------------------------------------------------------------------------------------------
// gather + mean, LDG variant.  One block per output row (grid-stride); thread c owns float4
// column c; the k neighbour rows are summed in j order with kUnroll loads in flight.
// ------------------------------------------------------------------------------------------
template <int kUnroll>
__global__ void __launch_bounds__(256) gather_mean_ldg_kernel(const float* __restrict__ src, int64_t n_src_rows, int F,
                                                              int64_t pitch, const __grid_constant__ SegTable tab, int include_self,
                                                              float* __restrict__ out_self,
                                                              float* __restrict__ out_mean, int64_t out_pitch) {
  const int ncol4 = (int)(out_pitch >> 2);
  for (int64_t r = blockIdx.x; r < tab.total_rows; r += gridDim.x) {
    int64_t i;
    const gs_segment& sg = tab.s[find_segment(tab, r, i)];
    const int k = sg.k;
    const int64_t orow = sg.out_row0 + i;
    const int64_t srow = clamp_row(sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i, n_src_rows);
    for (int c = threadIdx.x; c < ncol4; c += blockDim.x) {
      const int col0 = c * 4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 sv = acc;
      if (col0 < F) {
        int j = 0;
        for (; j + kUnroll <= k; j += kUnroll) {
          float4 v[kUnroll];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            int64_t nr = clamp_row(sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j + u] : sg.neigh_row0 + i * k + j + u,
                                   n_src_rows);
            v[u] = ldg_nc_f4(reinterpret_cast<const float4*>(src + nr * pitch) + c);
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w;
          }
        }
        for (; j < k; ++j) {
          int64_t nr = clamp_row(sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j] : sg.neigh_row0 + i * k + j, n_src_rows);
          float4 v = ldg_nc_f4(reinterpret_cast<const float4*>(src + nr * pitch) + c);
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        if (include_self || out_self) sv = ldg_nc_f4(reinterpret_cast<const float4*>(src + srow * pitch) + c);
        float div = (float)(k + (include_self ? 1 : 0));
        if (include_self) { acc.x += sv.x; acc.y += sv.y; acc.z += sv.z; acc.w += sv.w; }
        acc.x /= div; acc.y /= div; acc.z /= div; acc.w /= div;
        acc = mask_tail(acc, col0, F);
        sv = mask_tail(sv, col0, F);
      }
      reinterpret_cast<float4*>(out_mean + orow * out_pitch)[c] = acc;
      if (out_self) reinterpret_cast<float4*>(out_self + orow * out_pitch)[c] = sv;
    }
  }
}

// dropout sites of a gs_gather_mean_dropout call: one neighbour and one self site per segment
struct DropTab {
  DropSite neigh[GS_MAX_SEGMENTS];
  DropSite self[GS_MAX_SEGMENTS];
};

// scalar fallback for tables whose pitch / alignment rules out 128-bit access (kDrop: gs_gather_mean_dropout's masks)
template <bool kDrop>
__global__ void __launch_bounds__(256) gather_mean_scalar_kernel(const float* __restrict__ src, int64_t n_src_rows, int F,
                                                                 int64_t pitch, const __grid_constant__ SegTable tab, int include_self,
                                                                 float* __restrict__ out_self,
                                                                 float* __restrict__ out_mean, int64_t out_pitch,
                                                                 const __grid_constant__ DropTab drop) {
  __shared__ uint32_t drop_off[2 * GS_MAX_SEGMENTS];      // kDrop: the device-side call offsets, neighbour sites then self
  if constexpr (kDrop) {
    if (threadIdx.x < 2 * GS_MAX_SEGMENTS) {
      const int s = threadIdx.x % GS_MAX_SEGMENTS;
      drop_off[threadIdx.x] = drop_call_offset(threadIdx.x < GS_MAX_SEGMENTS ? drop.neigh[s] : drop.self[s]);
    }
    __syncthreads();
  }
  for (int64_t r = blockIdx.x; r < tab.total_rows; r += gridDim.x) {
    int64_t i;
    const int si = find_segment(tab, r, i);
    const gs_segment& sg = tab.s[si];
    const int k = sg.k;
    const int64_t orow = sg.out_row0 + i;
    const int64_t srow = clamp_row(sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i, n_src_rows);
    DropSite nsite{}, ssite{};
    if constexpr (kDrop) {
      nsite = with_call_offset(drop.neigh[si], drop_off[si]);
      ssite = with_call_offset(drop.self[si], drop_off[GS_MAX_SEGMENTS + si]);
    }
    for (int c = threadIdx.x; c < (int)out_pitch; c += blockDim.x) {
      float acc = 0.f, sv = 0.f;
      if (c < F) {
        for (int j = 0; j < k; ++j) {
          int64_t nr = clamp_row(sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j] : sg.neigh_row0 + i * k + j, n_src_rows);
          if constexpr (kDrop) acc += drop_col(nsite, i * k + j, c, src[nr * pitch + c]);
          else acc += src[nr * pitch + c];
        }
        sv = src[srow * pitch + c];
        if constexpr (kDrop) sv = drop_col(ssite, i, c, sv);
        if (include_self) acc += sv;
        acc /= (float)(k + (include_self ? 1 : 0));
      }
      out_mean[orow * out_pitch + c] = acc;
      if (out_self) out_self[orow * out_pitch + c] = sv;
    }
  }
}

// ------------------------------------------------------------------------------------------
// gather + mean, TMA bulk variant.  Per output row, one elected thread posts k+1 whole-row
// bulk copies (UBLKCP) into shared memory against one mbarrier; the block then sums the rows
// column-parallel out of shared memory.  Several CTAs are resident per SM so one CTA's
// reduction overlaps the others' copies (row buffers of all resident CTAs = bytes in flight).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(192) gather_mean_tma_kernel(const float* __restrict__ src, int64_t n_src_rows, int F,
                                                              int64_t pitch, const __grid_constant__ SegTable tab, int include_self,
                                                              float* __restrict__ out_self,
                                                              float* __restrict__ out_mean, int64_t out_pitch,
                                                              int row_bytes) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bar;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int ncol4 = (int)(out_pitch >> 2);
  const int row_f4 = row_bytes >> 4;
  uint32_t phase = 0;
  for (int64_t r = blockIdx.x; r < tab.total_rows; r += gridDim.x) {
    int64_t i;
    const gs_segment& sg = tab.s[find_segment(tab, r, i)];
    const int k = sg.k;
    const int64_t orow = sg.out_row0 + i;
    if (threadIdx.x < 32) {
      // warp 0 posts the copies: lane l takes rows l, l+32, ... (row k = self)
      if (threadIdx.x == 0) mbar_expect_tx(&bar, (uint32_t)((k + 1) * row_bytes));
      __syncwarp();
      for (int j = threadIdx.x; j <= k; j += 32) {
        int64_t id;
        if (j < k) id = sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j] : sg.neigh_row0 + i * k + j;
        else id = sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i;
        id = clamp_row(id, n_src_rows);
        bulk_g2s(smem + (size_t)j * row_bytes, src + id * pitch, (uint32_t)row_bytes, &bar);
      }
    }
    mbar_wait(&bar, phase);
    phase ^= 1u;
    const float4* rows = reinterpret_cast<const float4*>(smem);
    for (int c = threadIdx.x; c < ncol4; c += blockDim.x) {
      const int col0 = c * 4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 sv = acc;
      if (col0 < F) {
#pragma unroll 5
        for (int j = 0; j < k; ++j) {
          float4 v = rows[j * row_f4 + c];
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        sv = rows[k * row_f4 + c];
        float div = (float)(k + (include_self ? 1 : 0));
        if (include_self) { acc.x += sv.x; acc.y += sv.y; acc.z += sv.z; acc.w += sv.w; }
        acc.x /= div; acc.y /= div; acc.z /= div; acc.w /= div;
        acc = mask_tail(acc, col0, F);
        sv = mask_tail(sv, col0, F);
      }
      reinterpret_cast<float4*>(out_mean + orow * out_pitch)[c] = acc;
      if (out_self) reinterpret_cast<float4*>(out_self + orow * out_pitch)[c] = sv;
    }
    __syncthreads();  // all generic-proxy reads of the row buffer are done before it is refilled
  }
}

// ------------------------------------------------------------------------------------------
// Row resolvers: where the feature row of a node id lives.
//   DenseRows : one table in this GPU's HBM.
//   ShardRows : node-partitioned table (multi-GPU).  Shard o owns the ids [row_start[o], row_start[o+1]) at
//     base[o] (peer-mapped over NVLink for o != my_shard); this GPU additionally holds REPLICAS of the remote rows
//     it reads most, addressed through `remap` (remap[id] >= 0: local row index inside base[my_shard]; -1: not
//     held locally).  Ids outside [0, N) - the dummy id N included - read the local zero row.
//     Remote rows are pulled by the consuming kernel itself: the halo exchange IS the gather.
// ------------------------------------------------------------------------------------------
struct DenseRows {
  const float* src;
  int64_t n_rows, pitch;
  __device__ __forceinline__ const float* row(int64_t id) const { return src + clamp_row(id, n_rows) * pitch; }
};

struct ShardTab {
  const float* base[GS_MAX_SHARDS];
  int64_t row_start[GS_MAX_SHARDS + 1];
  int32_t n_shards, my_shard;
  int64_t n_global_rows;      // N + 1
  int64_t zero_row;           // local row index of this GPU's all-zero row
  const int32_t* remap;       // [N + 1] or NULL
};

struct ShardRows {
  ShardTab t;
  int64_t pitch;
  int32_t locators;           // 0: global ids; 1: gs_translate_ids locators (>= 0 local row index, < 0 -> -(global id) - 1);
                              // 2: gs_halo_translate locators (>= 0 local row index, < 0 -> row -(loc) - 1 of `staging`)
  const float* staging;       // this step's halo rows, fetched once each by gs_halo_fetch (locators == 2)
  __device__ __forceinline__ const float* row(int64_t id) const {
    const float* mine = t.base[t.my_shard];
    if (locators) {
      if (id >= 0) return mine + id * pitch;
      if (locators == 2) return staging + (-id - 1) * pitch;
      id = -id - 1;                                  // a remote row: owner found below
    } else if (id < 0 || id >= t.n_global_rows - 1) {
      return mine + t.zero_row * pitch;
    } else if (t.remap) {
      const int32_t s = __ldg(t.remap + id);
      if (s >= 0) return mine + (int64_t)s * pitch;
    } else if (id >= t.row_start[t.my_shard] && id < t.row_start[t.my_shard + 1]) {
      return mine + (id - t.row_start[t.my_shard]) * pitch;
    }
    int o = 0;
#pragma unroll
    for (int q = 1; q < GS_MAX_SHARDS; ++q)
      if (q < t.n_shards && id >= t.row_start[q]) o = q;
    return t.base[o] + (id - t.row_start[o]) * pitch;
  }
};

// ------------------------------------------------------------------------------------------
// gather + mean, TMA bulk variant 2: the rows of an output node are fetched in GROUPS of up to
// kGroupRows rows through a two-buffer ring, so the bulk copies of group t+1 are in flight while the
// CTA sums group t (variant 1 alternates copy and sum inside a CTA and relies on co-resident CTAs
// for overlap).  Per-thread accumulators persist across the groups of a node.
// ------------------------------------------------------------------------------------------
constexpr int kGroupRows = 13;

// kDrop: every gathered row is dropped in registers before it is summed (gs_gather_mean_dropout); the kDrop = false
// instantiation is the plain gather.
// min 3 CTAs per SM: what the two-buffer ring's shared memory allows at F = 602 (2 x 13 rows x 2,432 B); without the hint
// ptxas caps the kernel at 64 registers and spills
template <class Rows, bool kDrop>
__global__ void __launch_bounds__(192, 3) gather_mean_tma2_kernel(const __grid_constant__ Rows rows_of, int F,
                                                               const __grid_constant__ SegTable tab,
                                                               int include_self, float* __restrict__ out_self,
                                                               float* __restrict__ out_mean, int64_t out_pitch,
                                                               int row_bytes, const __grid_constant__ DropTab drop) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bar[2];
  __shared__ uint32_t drop_off[2 * GS_MAX_SEGMENTS];      // kDrop: the device-side call offsets, neighbour sites then self
  if (threadIdx.x == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_mbar_init();
  }
  if constexpr (kDrop) {
    if (threadIdx.x < 2 * GS_MAX_SEGMENTS) {
      const int s = threadIdx.x % GS_MAX_SEGMENTS;
      drop_off[threadIdx.x] = drop_call_offset(threadIdx.x < GS_MAX_SEGMENTS ? drop.neigh[s] : drop.self[s]);
    }
  }
  __syncthreads();
  const int ncol4 = (int)(out_pitch >> 2);
  const int row_f4 = row_bytes >> 4;
  const size_t buf_bytes = (size_t)kGroupRows * row_bytes;
  // a node's self row is fetched only when something reads it: the GCN sum or out_self.  The mean layer whose GEMM reads
  // the self rows by id (gs_sage_gemm_rows) asks for neither and so moves k rows per node, not k + 1.
  const int self_rows = (include_self || out_self) ? 1 : 0;

  // work items of this CTA: (node r, group g); enumerate lazily
  int64_t r_issue = blockIdx.x;      // node whose groups are being issued
  int g_issue = 0;
  auto issue = [&](int buf) -> bool {   // post the copies of the next (node, group) into `buf`; false if none left
    if (r_issue >= tab.total_rows) return false;
    int64_t i;
    const gs_segment& sg = tab.s[find_segment(tab, r_issue, i)];
    const int k = sg.k;
    const int rows_total = k + self_rows;                 // neighbours, then self
    const int first = g_issue * kGroupRows;
    const int cnt = min(kGroupRows, rows_total - first);
    if (threadIdx.x < 32) {
      if (threadIdx.x == 0) mbar_expect_tx(&bar[buf], (uint32_t)(cnt * row_bytes));
      __syncwarp();
      for (int j = threadIdx.x; j < cnt; j += 32) {
        const int jj = first + j;
        int64_t id;
        if (jj < k) id = sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + jj] : sg.neigh_row0 + i * k + jj;
        else id = sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i;
        bulk_g2s(smem + buf * buf_bytes + (size_t)j * row_bytes, rows_of.row(id), (uint32_t)row_bytes, &bar[buf]);
      }
    }
    if (first + cnt >= rows_total) { r_issue += gridDim.x; g_issue = 0; } else { ++g_issue; }
    return true;
  };

  uint32_t phase[2] = {0u, 0u};
  int buf = 0;
  bool have = issue(0);
  int64_t r = blockIdx.x;
  int g = 0;
  float4 acc[2];                                          // up to 2 float4 columns per thread (ncol4 <= 2 * blockDim)
  acc[0] = acc[1] = make_float4(0.f, 0.f, 0.f, 0.f);
  while (have) {
    const bool have_next = issue(buf ^ 1);                // prefetch the next group into the other buffer
    int64_t i;
    const int si = find_segment(tab, r, i);
    const gs_segment& sg = tab.s[si];
    const int k = sg.k;
    const int rows_total = k + self_rows;
    const int first = g * kGroupRows;
    const int cnt = min(kGroupRows, rows_total - first);
    const bool last = first + cnt >= rows_total;
    mbar_wait(&bar[buf], phase[buf]);
    phase[buf] ^= 1u;
    const float4* rows = reinterpret_cast<const float4*>(smem + buf * buf_bytes);
    const int nn = last ? cnt - self_rows : cnt;          // neighbour rows in this group (the self row is the node's last row)
    DropSite nsite{};
    if constexpr (kDrop) nsite = with_call_offset(drop.neigh[si], drop_off[si]);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int c = threadIdx.x + q * blockDim.x;
      if (c < ncol4 && c * 4 < F) {
        float4 a = acc[q];
        for (int j = 0; j < nn; ++j) {
          float4 v = rows[j * row_f4 + c];
          if constexpr (kDrop) v = drop4(nsite, i * k + first + j, (uint32_t)c, v);
          a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
        acc[q] = a;
      }
    }
    if (last) {
      const int64_t orow = sg.out_row0 + i;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int c = threadIdx.x + q * blockDim.x;
        if (c < ncol4) {
          float4 a = make_float4(0.f, 0.f, 0.f, 0.f), sv = a;
          if (c * 4 < F) {
            a = acc[q];
            if (self_rows) {
              sv = rows[(cnt - 1) * row_f4 + c];
              if constexpr (kDrop) sv = drop4(with_call_offset(drop.self[si], drop_off[GS_MAX_SEGMENTS + si]), i, (uint32_t)c, sv);
            }
            const float div = (float)(k + (include_self ? 1 : 0));
            if (include_self) { a.x += sv.x; a.y += sv.y; a.z += sv.z; a.w += sv.w; }
            a.x /= div; a.y /= div; a.z /= div; a.w /= div;
            a = mask_tail(a, c * 4, F);
            sv = mask_tail(sv, c * 4, F);
          }
          if (out_mean) reinterpret_cast<float4*>(out_mean + orow * out_pitch)[c] = a;
          if (out_self) reinterpret_cast<float4*>(out_self + orow * out_pitch)[c] = sv;
          acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      r += gridDim.x;
      g = 0;
    } else {
      ++g;
    }
    __syncthreads();                                       // buffer `buf` fully read before it is refilled
    buf ^= 1;
    have = have_next;
  }
}

// ------------------------------------------------------------------------------------------
// gather + mean over a BFLOAT16 table (BASELINE.md's 160.9 MB bf16 gather yardstick): the structure of
// gather_mean_tma2_kernel - whole rows (1,216 B at F = 602) fetched by cp.async.bulk in groups of kGroupRows through a
// two-buffer ring - with the rows widened to fp32 as they are summed (fp32 accumulate, j order, like the fp32 kernel), so
// the result equals the fp32 kernel's on the bf16-rounded table.  A thread owns 8 columns (one 128-bit shared load).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(192) gather_mean_bf16_tma2_kernel(const uint16_t* __restrict__ src, int64_t n_src_rows, int F,
                                                                    int64_t pitch, const __grid_constant__ SegTable tab,
                                                                    int include_self, float* __restrict__ out_self,
                                                                    float* __restrict__ out_mean, int64_t out_pitch,
                                                                    int row_bytes) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bar[2];
  if (threadIdx.x == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int ncol8 = (int)(out_pitch >> 3);
  const int row_u4 = row_bytes >> 4;
  const size_t buf_bytes = (size_t)kGroupRows * row_bytes;
  int64_t r_issue = blockIdx.x;
  int g_issue = 0;
  auto issue = [&](int buf) -> bool {
    if (r_issue >= tab.total_rows) return false;
    int64_t i;
    const gs_segment& sg = tab.s[find_segment(tab, r_issue, i)];
    const int k = sg.k;
    const int rows_total = k + 1;
    const int first = g_issue * kGroupRows;
    const int cnt = min(kGroupRows, rows_total - first);
    if (threadIdx.x < 32) {
      if (threadIdx.x == 0) mbar_expect_tx(&bar[buf], (uint32_t)(cnt * row_bytes));
      __syncwarp();
      for (int j = threadIdx.x; j < cnt; j += 32) {
        const int jj = first + j;
        int64_t id;
        if (jj < k) id = sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + jj] : sg.neigh_row0 + i * k + jj;
        else id = sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i;
        id = clamp_row(id, n_src_rows);
        bulk_g2s(smem + buf * buf_bytes + (size_t)j * row_bytes, src + id * pitch, (uint32_t)row_bytes, &bar[buf]);
      }
    }
    if (first + cnt >= rows_total) { r_issue += gridDim.x; g_issue = 0; } else { ++g_issue; }
    return true;
  };
  auto widen = [](uint4 u, float (&v)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      v[2 * e] = __uint_as_float(w[e] << 16);
      v[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u);
    }
  };
  uint32_t phase[2] = {0u, 0u};
  int buf = 0;
  bool have = issue(0);
  int64_t r = blockIdx.x;
  int g = 0;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  const int c = threadIdx.x;                                // this thread's 8-column chunk (ncol8 <= blockDim)
  while (have) {
    const bool have_next = issue(buf ^ 1);
    int64_t i;
    const gs_segment& sg = tab.s[find_segment(tab, r, i)];
    const int k = sg.k;
    const int rows_total = k + 1;
    const int first = g * kGroupRows;
    const int cnt = min(kGroupRows, rows_total - first);
    const bool last = first + cnt >= rows_total;
    mbar_wait(&bar[buf], phase[buf]);
    phase[buf] ^= 1u;
    const uint4* rows = reinterpret_cast<const uint4*>(smem + buf * buf_bytes);
    const int nn = last ? cnt - 1 : cnt;
    if (c < ncol8 && c * 8 < F) {
      for (int j = 0; j < nn; ++j) {
        float v[8];
        widen(rows[j * row_u4 + c], v);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += v[e];
      }
    }
    if (last) {
      const int64_t orow = sg.out_row0 + i;
      if (c < ncol8) {
        float a[8], sv[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) { a[e] = 0.f; sv[e] = 0.f; }
        if (c * 8 < F) {
          widen(rows[(cnt - 1) * row_u4 + c], sv);
          const float div = (float)(k + (include_self ? 1 : 0));
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            float t = acc[e];
            if (include_self) t += sv[e];
            a[e] = (c * 8 + e < F) ? t / div : 0.f;
            if (c * 8 + e >= F) sv[e] = 0.f;
          }
        }
        float4* om = reinterpret_cast<float4*>(out_mean + orow * out_pitch) + 2 * c;
        om[0] = make_float4(a[0], a[1], a[2], a[3]);
        om[1] = make_float4(a[4], a[5], a[6], a[7]);
        if (out_self) {
          float4* os = reinterpret_cast<float4*>(out_self + orow * out_pitch) + 2 * c;
          os[0] = make_float4(sv[0], sv[1], sv[2], sv[3]);
          os[1] = make_float4(sv[4], sv[5], sv[6], sv[7]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
      }
      r += gridDim.x;
      g = 0;
    } else {
      ++g;
    }
    __syncthreads();
    buf ^= 1;
    have = have_next;
  }
}

// ------------------------------------------------------------------------------------------
// plain row gather.  TMA variant: each lane of a one-warp CTA moves one row
// global -> shared -> global entirely with the bulk-copy engine (no register traffic).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) gather_rows_tma_kernel(const unsigned char* __restrict__ src, int64_t n_rows,
                                                             int64_t pitch_bytes, const int32_t* __restrict__ ids,
                                                             int64_t n, unsigned char* __restrict__ out,
                                                             int64_t out_pitch_bytes, int row_bytes) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bar;
  const int lane = threadIdx.x;
  if (lane == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncwarp();
  uint32_t phase = 0;
  for (int64_t base = (int64_t)blockIdx.x * 32; base < n; base += (int64_t)gridDim.x * 32) {
    int cnt = (int)((n - base) < 32 ? (n - base) : 32);
    if (lane == 0) mbar_expect_tx(&bar, (uint32_t)(cnt * row_bytes));
    __syncwarp();
    if (lane < cnt) {
      int64_t id = clamp_row(ids[base + lane], n_rows);
      bulk_g2s(smem + (size_t)lane * row_bytes, src + id * pitch_bytes, (uint32_t)row_bytes, &bar);
    }
    mbar_wait(&bar, phase);
    phase ^= 1u;
    if (lane < cnt) bulk_s2g(out + (base + lane) * out_pitch_bytes, smem + (size_t)lane * row_bytes, (uint32_t)row_bytes);
    bulk_commit();
    bulk_wait_read<0>();  // shared buffer may be overwritten once the stores have read it
    __syncwarp();
  }
  bulk_wait<0>();
}

// generic byte-row gather (any alignment): one warp per row, 4-byte or 2-byte units
template <typename T>
__global__ void __launch_bounds__(256) gather_rows_simple_kernel(const T* __restrict__ src, int64_t n_rows, int F,
                                                                 int64_t pitch, const int32_t* __restrict__ ids,
                                                                 int64_t n, T* __restrict__ out, int64_t out_pitch) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    int64_t id = clamp_row(ids[i], n_rows);
    for (int c = lane; c < F; c += 32) out[i * out_pitch + c] = src[id * pitch + c];
  }
}

// rows of a bf16 (or fp32) table gathered straight into an fp32 matrix - the self rows of the bf16 max-pool path
// (models.py:299 + the cast the fp32 self_weights contraction needs); one warp per row, pad columns zeroed
template <typename T>
__global__ void __launch_bounds__(256) gather_rows_to_f32_kernel(const T* __restrict__ src, int64_t n_rows, int F,
                                                                 int64_t pitch, const int32_t* __restrict__ ids, int64_t row0,
                                                                 int64_t n, float* __restrict__ out, int64_t out_pitch) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    const int64_t id = clamp_row(ids ? (int64_t)ids[i] : row0 + i, n_rows);
    for (int c = lane; c < (int)out_pitch; c += 32) {
      float v = 0.f;
      if (c < F) {
        if constexpr (sizeof(T) == 2) v = __uint_as_float(((uint32_t)src[id * pitch + c]) << 16);   // bf16 -> fp32 (exact)
        else v = src[id * pitch + c];
      }
      out[i * out_pitch + c] = v;
    }
  }
}

// the same for bf16 rows that are 16-byte multiples (pitch % 8 == 0, 16-byte aligned table and output, out_pitch % 8 == 0):
// a lane converts 8 values per step (one 128-bit load, two 128-bit stores)
__global__ void __launch_bounds__(256) gather_rows_bf16_to_f32_vec_kernel(const uint16_t* __restrict__ src, int64_t n_rows, int F,
                                                                          int64_t pitch, const int32_t* __restrict__ ids,
                                                                          int64_t row0, int64_t n, float* __restrict__ out,
                                                                          int64_t out_pitch) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int chunks = (int)(out_pitch >> 3);
  for (int64_t i = warp; i < n; i += nwarps) {
    const int64_t id = clamp_row(ids ? (int64_t)ids[i] : row0 + i, n_rows);
    const uint4* rp = reinterpret_cast<const uint4*>(src + id * pitch);
    float4* op = reinterpret_cast<float4*>(out + i * out_pitch);
    for (int c = lane; c < chunks; c += 32) {
      uint4 u = make_uint4(0u, 0u, 0u, 0u);
      if (c * 8 < F) u = __ldg(rp + c);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
      float v[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        v[2 * e] = (c * 8 + 2 * e < F) ? __uint_as_float(w[e] << 16) : 0.f;
        v[2 * e + 1] = (c * 8 + 2 * e + 1 < F) ? __uint_as_float(w[e] & 0xffff0000u) : 0.f;
      }
      op[2 * c] = make_float4(v[0], v[1], v[2], v[3]);
      op[2 * c + 1] = make_float4(v[4], v[5], v[6], v[7]);
    }
  }
}

__device__ __forceinline__ uint32_t f32_to_bf16_rne(float x) {
  const uint32_t u = __float_as_uint(x);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (u >> 16) | 0x40u;          // NaN stays NaN
  return (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;
}

// fp32 [n, F] -> bf16 [n, out_pitch] (round to nearest even, pad columns zeroed): the layer-(l+1) source of the
// bf16 max-pool path.  A thread produces 8 consecutive outputs (one 128-bit store); out_pitch % 8 == 0.
__global__ void __launch_bounds__(256) cast_rows_bf16_kernel(const float* __restrict__ x, int64_t n, int F, int64_t ldx,
                                                             uint16_t* __restrict__ out, int64_t out_pitch) {
  const int chunks = (int)(out_pitch >> 3);
  const int64_t total = n * chunks;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = q / chunks;
    const int c = (int)(q - i * chunks) * 8;
    const float* xp = x + i * ldx + c;
    uint32_t h[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = (c + e < F) ? f32_to_bf16_rne(xp[e]) : 0u;
    uint4 o;
    o.x = h[0] | (h[1] << 16); o.y = h[2] | (h[3] << 16); o.z = h[4] | (h[5] << 16); o.w = h[6] | (h[7] << 16);
    *reinterpret_cast<uint4*>(out + i * out_pitch + c) = o;
  }
}

// any out_pitch (scalar stores)
__global__ void __launch_bounds__(256) cast_rows_bf16_scalar_kernel(const float* __restrict__ x, int64_t n, int F, int64_t ldx,
                                                                    uint16_t* __restrict__ out, int64_t out_pitch) {
  const int64_t total = n * out_pitch;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = q / out_pitch;
    const int c = (int)(q - i * out_pitch);
    out[q] = c < F ? (uint16_t)f32_to_bf16_rne(x[i * ldx + c]) : (uint16_t)0;
  }
}

// out[r, c] (+)= keep(site, pos, c) ? (x[r / group, c] * scale) / keep : 0, pos = kIds ? pos_ids[r] : r - one thread per
// 4 columns of a row (one Philox block), so every element is read and written by one thread (out may alias x when
// group == 1)
template <bool kIds>
__global__ void __launch_bounds__(256) dropout_apply_kernel(const float* x, int64_t ldx, int64_t rows, int F, int group,
                                                            float scale, DropSite site, int accumulate, float* out,
                                                            int64_t ldo, const int32_t* pos_ids) {
  const int nc4 = (F + 3) >> 2;
  const int64_t total = rows * nc4;
  site.call += drop_call_offset(site);
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = q / nc4;
    const int c4 = (int)(q - r * nc4);
    const u32x4 w = drop_words(site, kIds ? (int64_t)__ldg(pos_ids + r) : r, (uint32_t)c4);
    const float* xr = x + (r / group) * ldx;
    float* orow = out + r * ldo;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c4 * 4 + e;
      if (c < F) {
        const float v = pick(w, e) >= site.threshold ? (xr[c] * scale) / site.keep : 0.f;
        orow[c] = accumulate ? orow[c] + v : v;
      }
    }
  }
}

// *counter += inc on the stream (the samplers' device-side call counter, advanced once per step)
__global__ void bump_counter_kernel(unsigned long long* counter, unsigned long long inc) { *counter += inc; }

__global__ void __launch_bounds__(256) segment_max_kernel(const float* __restrict__ x, int64_t n, int k, int C,
                                                          int64_t ldx, float* __restrict__ out, int64_t ldo) {
  for (int64_t i = blockIdx.x; i < n; i += gridDim.x) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float m = x[(i * k) * ldx + c];
      for (int j = 1; j < k; ++j) m = fmaxf(m, x[(i * k + j) * ldx + c]);
      out[i * ldo + c] = m;
    }
  }
}

// one warp per row: x *= rsqrt(max(sum x^2, 1e-12))
__global__ void __launch_bounds__(256) l2_normalize_kernel(float* __restrict__ x, int64_t n, int C, int64_t ldx) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) {
      float v = x[i * ldx + c];
      ss += v * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    float inv = 1.0f / sqrtf(fmaxf(ss, 1e-12f));
    for (int c = lane; c < C; c += 32) x[i * ldx + c] *= inv;
  }
}

// ------------------------------------------------------------------------------------------
// Node-partitioned table: the same fused gather+mean, with every row address resolved through the
// shard table (peer-mapped pointers).  Remote rows travel over NVLink as 128-bit loads issued by
// the consuming kernel itself - the halo exchange IS the gather.
// ------------------------------------------------------------------------------------------
// ids -> locators for a node-partitioned table with replicas: loc = remap[id] (row index inside this GPU's own buffer) when
// the row is held locally - own rows, replicas, and the zero row for ids outside [0, N) -, else -(id) - 1.  One thread per id:
// the dependent 4-byte lookup leaves the gather kernel's copy-issue path (where it cost 8 us per step).
__global__ void __launch_bounds__(256) translate_ids_kernel(const int32_t* __restrict__ remap, int64_t n_global_rows,
                                                            int32_t zero_row, const int32_t* __restrict__ ids, int64_t n,
                                                            int32_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t id = ids[i];
    int32_t loc;
    if (id < 0 || id >= n_global_rows - 1) loc = zero_row;
    else {
      loc = __ldg(remap + id);
      if (loc < 0) loc = -id - 1;
    }
    out[i] = loc;
  }
}

// ---- halo staging: every remote row a step needs is fetched ONCE into a local staging buffer --------------------------
// A step's frontier names the same remote node many times (one permutation per sampler call + hub nodes: ~25 % of the
// remote rows of a Reddit-shaped batch are repeats), and peer reads bypass the local L2, so the fused gather pulled each
// repeat over NVLink again.  Three small passes remove that:
//   claim     : thread per id; the first thread to see a remote id (atomicCAS on claim[id]) takes the next staging slot
//   fetch     : warp per claimed row, 128-bit loads from the owner (peer mapping) -> staging (local HBM)
//   translate : thread per id -> locator (>= 0: row of this GPU's own buffer; < 0: staging row -(loc) - 1)
// after which the gather kernel reads local memory only.  The passes of step i overlap the gathers of steps i +- 1 on the
// other streams: the NVLink transfer is no longer inside the HBM-bound kernel.
__device__ __forceinline__ bool halo_is_local(const ShardTab& t, int32_t id, int32_t& loc) {
  if (id < 0 || id >= t.n_global_rows - 1) { loc = (int32_t)t.zero_row; return true; }
  if (t.remap) {
    loc = __ldg(t.remap + id);
    return loc >= 0;
  }
  if (id >= t.row_start[t.my_shard] && id < t.row_start[t.my_shard + 1]) { loc = (int32_t)(id - t.row_start[t.my_shard]); return true; }
  return false;
}

__global__ void __launch_bounds__(256) halo_claim_kernel(const __grid_constant__ ShardTab t, const int32_t* __restrict__ ids,
                                                         int64_t n, int32_t* __restrict__ claim, int32_t* __restrict__ count,
                                                         int32_t* __restrict__ stage_ids, int64_t capacity) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t id = ids[i];
    int32_t loc;
    if (halo_is_local(t, id, loc)) continue;
    if (atomicCAS(claim + id, -1, -2) == -1) {             // first sighting of this remote id in the step
      const int32_t idx = atomicAdd(count, 1);
      if (idx < capacity) stage_ids[idx] = id;
      claim[id] = idx;                                     // read by the translate pass (a later launch)
    }
  }
}

// a staged id becomes miss_row0 + miss_step * claim[id]: -(slot) - 1 for the halo locators (-1, -1), the working-set row
// stage_row0 + slot for a host table (stage_row0, +1)
__global__ void __launch_bounds__(256) halo_translate_kernel(const __grid_constant__ ShardTab t, const int32_t* __restrict__ ids,
                                                             int64_t n, const int32_t* __restrict__ claim,
                                                             int32_t* __restrict__ out, int32_t miss_row0, int32_t miss_step) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t id = ids[i];
    int32_t loc;
    if (!halo_is_local(t, id, loc)) loc = miss_row0 + miss_step * claim[id];
    out[i] = loc;
  }
}

// warp per staged row; every lane keeps kHaloLoads 128-bit peer loads in flight before it stores
constexpr int kHaloLoads = 5;
__global__ void __launch_bounds__(256) halo_fetch_kernel(const __grid_constant__ ShardRows sr, int row_f4,
                                                         const int32_t* __restrict__ stage_ids, const int32_t* __restrict__ count,
                                                         int64_t capacity, float* __restrict__ staging, int64_t staging_pitch) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  int64_t n = *count;
  if (n > capacity) n = capacity;
  for (int64_t i = warp; i < n; i += nwarps) {
    const float4* src = reinterpret_cast<const float4*>(sr.row(stage_ids[i]));
    float4* dst = reinterpret_cast<float4*>(staging + i * staging_pitch);
    for (int c0 = lane; c0 < row_f4; c0 += 32 * kHaloLoads) {
      float4 v[kHaloLoads];
#pragma unroll
      for (int u = 0; u < kHaloLoads; ++u)
        if (c0 + 32 * u < row_f4) v[u] = ldg_nc_f4(src + c0 + 32 * u);
#pragma unroll
      for (int u = 0; u < kHaloLoads; ++u)
        if (c0 + 32 * u < row_f4) dst[c0 + 32 * u] = v[u];
    }
  }
}

template <int kUnroll>
__global__ void __launch_bounds__(256) gather_mean_sharded_kernel(const __grid_constant__ ShardRows st, int F,
                                                                  const __grid_constant__ SegTable tab, int include_self,
                                                                  float* __restrict__ out_self,
                                                                  float* __restrict__ out_mean, int64_t out_pitch) {
  const int ncol4 = (int)(out_pitch >> 2);
  for (int64_t r = blockIdx.x; r < tab.total_rows; r += gridDim.x) {
    int64_t i;
    const gs_segment& sg = tab.s[find_segment(tab, r, i)];
    const int k = sg.k;
    const int64_t orow = sg.out_row0 + i;
    const float* srow = st.row(sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i);
    for (int c = threadIdx.x; c < ncol4; c += blockDim.x) {
      const int col0 = c * 4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 sv = acc;
      if (col0 < F) {
        int j = 0;
        for (; j + kUnroll <= k; j += kUnroll) {
          float4 v[kUnroll];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const float* p = st.row(sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j + u] : sg.neigh_row0 + i * k + j + u);
            v[u] = ldg_nc_f4(reinterpret_cast<const float4*>(p) + c);
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w;
          }
        }
        for (; j < k; ++j) {
          const float* p = st.row(sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j] : sg.neigh_row0 + i * k + j);
          float4 v = ldg_nc_f4(reinterpret_cast<const float4*>(p) + c);
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        if (include_self || out_self) sv = ldg_nc_f4(reinterpret_cast<const float4*>(srow) + c);
        float div = (float)(k + (include_self ? 1 : 0));
        if (include_self) { acc.x += sv.x; acc.y += sv.y; acc.z += sv.z; acc.w += sv.w; }
        acc.x /= div; acc.y /= div; acc.z /= div; acc.w /= div;
        acc = mask_tail(acc, col0, F);
        sv = mask_tail(sv, col0, F);
      }
      reinterpret_cast<float4*>(out_mean + orow * out_pitch)[c] = acc;
      if (out_self) reinterpret_cast<float4*>(out_self + orow * out_pitch)[c] = sv;
    }
  }
}

// one warp per row, 128-bit loads through the shard table
__global__ void __launch_bounds__(256) gather_rows_sharded_kernel(const __grid_constant__ ShardRows st, int F,
                                                                  const int32_t* __restrict__ ids, int64_t n,
                                                                  float* __restrict__ out, int64_t out_pitch) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int ncol4 = (int)(out_pitch >> 2);
  for (int64_t i = warp; i < n; i += nwarps) {
    const float* p = st.row(ids[i]);
    for (int c = lane; c < ncol4; c += 32) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c * 4 < F) v = mask_tail(ldg_nc_f4(reinterpret_cast<const float4*>(p) + c), c * 4, F);
      reinterpret_cast<float4*>(out + i * out_pitch)[c] = v;
    }
  }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace gs


namespace gs {
// launch of the grouped double-buffered bulk-copy gather (dense or sharded resolver)
template <class Rows, bool kDrop = false>
static int32_t launch_gather_tma2(const Rows& rows_of, int F, const SegTable& tab, int include_self, float* out_self, float* out_mean,
                                  int64_t out_pitch, cudaStream_t st, const DropTab* drop = nullptr) {
  const int32_t rc_attr = ensure_dyn_smem((const void*)gather_mean_tma2_kernel<Rows, kDrop>, 200 * 1024);
  if (rc_attr != GS_OK) return rc_attr;
  const int ncol4 = (int)(out_pitch / 4);
  const int row_bytes = ((F + 3) / 4) * 16;
  const size_t smem2 = (size_t)2 * kGroupRows * row_bytes;
  int threads = ((ncol4 + 31) / 32) * 32;
  if (threads > 160) threads = 160;
  if (threads < 32) threads = 32;
  int per_sm = (int)((224 * 1024) / (smem2 + 1024));
  if (per_sm < 1) per_sm = 1;
  int lim = tuning("gather_ctas_per_sm", 8);
  if (per_sm > lim) per_sm = lim;
  int64_t blocks = tab.total_rows;
  int64_t cap = (int64_t)sm_count() * per_sm;
  if (blocks > cap) blocks = cap;
  DropTab no_drop;
  memset(&no_drop, 0, sizeof(no_drop));
  gather_mean_tma2_kernel<Rows, kDrop><<<(unsigned)blocks, threads, smem2, st>>>(rows_of, F, tab, include_self, out_self,
                                                                                 out_mean, out_pitch, row_bytes,
                                                                                 drop ? *drop : no_drop);
  return launch_check("gather_mean_tma2_kernel");
}
}  // namespace gs

// copies the caller's segments into `tab`, checks each one and sums total_rows; raises *kmax (if given) to the largest fanout
static int32_t fill_seg_table(const gs_segment* segments_host, int32_t n_segments, gs::SegTable& tab, const char* who,
                              int* kmax = nullptr) {
  memset(&tab, 0, sizeof(tab));
  tab.n_segments = n_segments;
  for (int s = 0; s < n_segments; ++s) {
    tab.s[s] = segments_host[s];
    GS_REQUIRE(tab.s[s].n >= 0 && tab.s[s].k >= 1, "%s: segment %d has n=%lld k=%d", who, s, (long long)tab.s[s].n, tab.s[s].k);
    tab.total_rows += tab.s[s].n;
    if (kmax && tab.s[s].k > *kmax) *kmax = tab.s[s].k;
  }
  return GS_OK;
}

extern "C" {

int32_t gs_gather_rows(const void* feats, int32_t dtype, int64_t n_rows, int32_t F, int64_t pitch, const int32_t* ids,
                       int64_t n, void* out, int64_t out_pitch, void* stream) {
  GS_REQUIRE(n >= 0 && F >= 0, "gs_gather_rows: negative size");
  if (n == 0 || F == 0) return GS_OK;
  GS_REQUIRE(feats && ids && out, "gs_gather_rows: NULL pointer");
  GS_REQUIRE(dtype == GS_F32 || dtype == GS_BF16, "gs_gather_rows: dtype %d", dtype);
  GS_REQUIRE(n_rows > 0 && pitch >= F && out_pitch >= F, "gs_gather_rows: pitch < F");
  const int es = dtype == GS_F32 ? 4 : 2;
  cudaStream_t st = (cudaStream_t)stream;
  const int row_bytes = ((F * es + 15) / 16) * 16;
  const bool tma_ok = gs::aligned16(feats) && gs::aligned16(out) && (pitch * es) % 16 == 0 && (out_pitch * es) % 16 == 0 &&
                      row_bytes <= pitch * es && row_bytes <= out_pitch * es && row_bytes * 32 <= 200 * 1024;
  if (tma_ok && gs::tuning("gather_variant", 2) != 0) {
    size_t smem = (size_t)row_bytes * 32;
    {
      const int32_t rc_attr = gs::ensure_dyn_smem((const void*)gs::gather_rows_tma_kernel, 200 * 1024);
      if (rc_attr != GS_OK) return rc_attr;
    }
    int per_sm = (int)((220 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 16) per_sm = 16;
    int64_t blocks = (n + 31) / 32;
    int64_t cap = (int64_t)gs::sm_count() * per_sm;
    if (blocks > cap) blocks = cap;
    gs::gather_rows_tma_kernel<<<(unsigned)blocks, 32, smem, st>>>((const unsigned char*)feats, n_rows, pitch * es, ids, n,
                                                                   (unsigned char*)out, out_pitch * es, row_bytes);
    return gs::launch_check("gather_rows_tma_kernel");
  }
  int64_t blocks = (n + 7) / 8;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (dtype == GS_F32)
    gs::gather_rows_simple_kernel<float><<<(unsigned)blocks, 256, 0, st>>>((const float*)feats, n_rows, F, pitch, ids, n,
                                                                           (float*)out, out_pitch);
  else
    gs::gather_rows_simple_kernel<uint16_t><<<(unsigned)blocks, 256, 0, st>>>((const uint16_t*)feats, n_rows, F, pitch, ids,
                                                                              n, (uint16_t*)out, out_pitch);
  return gs::launch_check("gather_rows_simple_kernel");
}

int32_t gs_gather_mean(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                       const gs_segment* segments_host, int32_t n_segments, int32_t include_self, void* out_self,
                       void* out_mean, int64_t out_pitch, void* stream) {
  GS_REQUIRE(dtype == GS_F32 || dtype == GS_BF16, "gs_gather_mean: dtype %d (GS_F32 or GS_BF16)", dtype);
  GS_REQUIRE(n_segments >= 0 && n_segments <= GS_MAX_SEGMENTS, "gs_gather_mean: n_segments=%d (max %d)", n_segments,
             GS_MAX_SEGMENTS);
  GS_REQUIRE(segments_host || n_segments == 0, "gs_gather_mean: segments_host is NULL");
  gs::SegTable tab;
  int kmax = 0;
  const int32_t rc = fill_seg_table(segments_host, n_segments, tab, "gs_gather_mean", &kmax);
  if (rc != GS_OK) return rc;
  if (tab.total_rows == 0) return GS_OK;
  GS_REQUIRE(src && out_mean, "gs_gather_mean: NULL pointer");
  GS_REQUIRE(F > 0 && pitch >= F && out_pitch >= F && n_src_rows > 0, "gs_gather_mean: bad F/pitch");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == GS_BF16) {
    // bf16 table -> fp32 means / self rows: the bulk-copy kernel only (rows must be 16-byte multiples)
    const int64_t f8 = ((int64_t)F + 7) / 8 * 8;
    if (!(gs::aligned16(src) && gs::aligned16(out_mean) && (!out_self || gs::aligned16(out_self)) && pitch % 8 == 0 &&
          out_pitch % 8 == 0 && f8 <= pitch && f8 <= out_pitch && f8 / 8 <= 192)) {
      gs::set_error("gs_gather_mean(GS_BF16): needs 16-byte aligned rows (pitch %% 8 == 0), out_pitch %% 8 == 0 and F <= 1536");
      return GS_ERR_UNSUPPORTED;
    }
    const int32_t rc_attr = gs::ensure_dyn_smem((const void*)gs::gather_mean_bf16_tma2_kernel, 200 * 1024);
    if (rc_attr != GS_OK) return rc_attr;
    const int row_bytes = (int)(f8 * 2);
    const size_t smem2 = (size_t)2 * gs::kGroupRows * row_bytes;
    const int ncol8 = (int)(out_pitch / 8);
    int threads = ((ncol8 + 31) / 32) * 32;
    if (threads < 32) threads = 32;
    GS_REQUIRE(threads <= 192, "gs_gather_mean(GS_BF16): out_pitch too wide");
    int per_sm = (int)((224 * 1024) / (smem2 + 1024));
    if (per_sm < 1) per_sm = 1;
    int lim = gs::tuning("gather_ctas_per_sm", 8);
    if (per_sm > lim) per_sm = lim;
    int64_t blocks = tab.total_rows;
    int64_t cap = (int64_t)gs::sm_count() * per_sm;
    if (blocks > cap) blocks = cap;
    gs::gather_mean_bf16_tma2_kernel<<<(unsigned)blocks, threads, smem2, st>>>((const uint16_t*)src, n_src_rows, F, pitch, tab,
                                                                              include_self, (float*)out_self, (float*)out_mean,
                                                                              out_pitch, row_bytes);
    return gs::launch_check("gather_mean_bf16_tma2_kernel");
  }
  const float* fsrc = (const float*)src;
  const bool vec_ok = gs::aligned16(src) && gs::aligned16(out_mean) && (!out_self || gs::aligned16(out_self)) &&
                      pitch % 4 == 0 && out_pitch % 4 == 0 && ((F + 3) / 4) * 4 <= pitch;
  if (!vec_ok) {
    int64_t blocks = tab.total_rows;
    int64_t cap = (int64_t)gs::sm_count() * 8;
    if (blocks > cap) blocks = cap;
    gs::DropTab no_drop;
    memset(&no_drop, 0, sizeof(no_drop));
    gs::gather_mean_scalar_kernel<false><<<(unsigned)blocks, 256, 0, st>>>(fsrc, n_src_rows, F, pitch, tab, include_self,
                                                                           (float*)out_self, (float*)out_mean, out_pitch,
                                                                           no_drop);
    return gs::launch_check("gather_mean_scalar_kernel");
  }
  const int ncol4 = (int)(out_pitch / 4);
  const int row_bytes = ((F + 3) / 4) * 16;
  const size_t smem = (size_t)row_bytes * (kmax + 1);
  const int variant = gs::tuning("gather_variant", 2);   // 2: grouped double-buffered TMA (default), 1: whole-node TMA, 0: LDG
  if (variant == 2 && ncol4 <= 2 * 160) {
    const gs::DenseRows rows_of{fsrc, n_src_rows, pitch};
    return gs::launch_gather_tma2(rows_of, F, tab, include_self, (float*)out_self, (float*)out_mean, out_pitch, st);
  }
  if (variant >= 1 && smem <= 200 * 1024) {
    {
      const int32_t rc_attr = gs::ensure_dyn_smem((const void*)gs::gather_mean_tma_kernel, 200 * 1024);
      if (rc_attr != GS_OK) return rc_attr;
    }
    int threads = ((ncol4 + 31) / 32) * 32;
    if (threads > 192) threads = 192;
    if (threads < 32) threads = 32;
    int per_sm = (int)((224 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    int lim = gs::tuning("gather_ctas_per_sm", 8);
    if (per_sm > lim) per_sm = lim;
    int64_t blocks = tab.total_rows;
    int64_t cap = (int64_t)gs::sm_count() * per_sm;
    if (blocks > cap) blocks = cap;
    gs::gather_mean_tma_kernel<<<(unsigned)blocks, threads, smem, st>>>(fsrc, n_src_rows, F, pitch, tab, include_self,
                                                                        (float*)out_self, (float*)out_mean, out_pitch,
                                                                        row_bytes);
    return gs::launch_check("gather_mean_tma_kernel");
  }
  int threads = ((ncol4 + 31) / 32) * 32;
  if (threads > 256) threads = 256;
  int64_t blocks = tab.total_rows;
  int64_t cap = (int64_t)gs::sm_count() * gs::tuning("gather_ctas_per_sm", 8);
  if (blocks > cap) blocks = cap;
  gs::gather_mean_ldg_kernel<5><<<(unsigned)blocks, threads, 0, st>>>(fsrc, n_src_rows, F, pitch, tab, include_self,
                                                                      (float*)out_self, (float*)out_mean, out_pitch);
  return gs::launch_check("gather_mean_ldg_kernel");
}

int32_t gs_gather_rows_f32(const void* feats, int32_t dtype, int64_t n_rows, int32_t F, int64_t pitch, const int32_t* ids,
                           int64_t row0, int64_t n, float* out, int64_t out_pitch, void* stream) {
  GS_REQUIRE(n >= 0 && F >= 0, "gs_gather_rows_f32: negative size");
  if (n == 0 || out_pitch == 0) return GS_OK;
  GS_REQUIRE(feats && out, "gs_gather_rows_f32: NULL pointer");
  GS_REQUIRE(dtype == GS_F32 || dtype == GS_BF16, "gs_gather_rows_f32: dtype %d", dtype);
  GS_REQUIRE(n_rows > 0 && pitch >= F && out_pitch >= F, "gs_gather_rows_f32: pitch < F");
  int64_t blocks = (n + 7) / 8;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (dtype == GS_F32)
    gs::gather_rows_to_f32_kernel<float><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        (const float*)feats, n_rows, F, pitch, ids, row0, n, out, out_pitch);
  else if (pitch % 8 == 0 && out_pitch % 8 == 0 && gs::aligned16(feats) && gs::aligned16(out) && out_pitch <= pitch)
    gs::gather_rows_bf16_to_f32_vec_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        (const uint16_t*)feats, n_rows, F, pitch, ids, row0, n, out, out_pitch);
  else
    gs::gather_rows_to_f32_kernel<uint16_t><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        (const uint16_t*)feats, n_rows, F, pitch, ids, row0, n, out, out_pitch);
  return gs::launch_check("gather_rows_to_f32_kernel");
}

int32_t gs_cast_rows_bf16(const float* x, int64_t n, int32_t F, int64_t ldx, void* out_bf16, int64_t out_pitch,
                          void* stream) {
  GS_REQUIRE(n >= 0 && F >= 0 && ldx >= F && out_pitch >= F, "gs_cast_rows_bf16: bad sizes");
  if (n == 0 || out_pitch == 0) return GS_OK;
  GS_REQUIRE(x && out_bf16, "gs_cast_rows_bf16: NULL pointer");
  const bool vec = out_pitch % 8 == 0 && gs::aligned16(out_bf16) && ldx >= ((F + 7) / 8) * 8;
  int64_t blocks = ((vec ? n * (out_pitch / 8) : n * out_pitch) + 255) / 256;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (vec)
    gs::cast_rows_bf16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, n, F, ldx, (uint16_t*)out_bf16, out_pitch);
  else
    gs::cast_rows_bf16_scalar_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, n, F, ldx, (uint16_t*)out_bf16,
                                                                                         out_pitch);
  return gs::launch_check("cast_rows_bf16_kernel");
}

int32_t gs_bump_counter(uint64_t* counter_dev, uint64_t inc, void* stream) {
  GS_REQUIRE(counter_dev != nullptr, "gs_bump_counter: NULL counter");
  gs::bump_counter_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((unsigned long long*)counter_dev, (unsigned long long)inc);
  return gs::launch_check("bump_counter_kernel");
}

int32_t gs_segment_max(const float* x, int64_t n, int32_t k, int32_t C, int64_t ldx, float* out, int64_t ldo,
                       void* stream) {
  GS_REQUIRE(n >= 0 && k >= 1 && C >= 0, "gs_segment_max: bad sizes");
  if (n == 0 || C == 0) return GS_OK;
  GS_REQUIRE(x && out, "gs_segment_max: NULL pointer");
  int64_t blocks = n;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::segment_max_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, n, k, C, ldx, out, ldo);
  return gs::launch_check("segment_max_kernel");
}

int32_t gs_gather_mean_dropout(const float* src, int64_t n_src_rows, int32_t F, int64_t pitch, const gs_segment* segments_host,
                               int32_t n_segments, const gs_dropout_site* neigh_sites_host,
                               const gs_dropout_site* self_sites_host, int32_t include_self, float* out_self,
                               float* out_mean, int64_t out_pitch, void* stream) {
  GS_REQUIRE(n_segments >= 0 && n_segments <= GS_MAX_SEGMENTS, "gs_gather_mean_dropout: n_segments=%d (max %d)", n_segments,
             GS_MAX_SEGMENTS);
  GS_REQUIRE((segments_host && neigh_sites_host && self_sites_host) || n_segments == 0,
             "gs_gather_mean_dropout: segments / sites are NULL");
  gs::SegTable tab;
  int32_t rc = fill_seg_table(segments_host, n_segments, tab, "gs_gather_mean_dropout");
  if (rc != GS_OK) return rc;
  gs::DropTab drop;
  memset(&drop, 0, sizeof(drop));
  for (int s = 0; s < n_segments; ++s) {
    rc = gs::check_site(neigh_sites_host[s], "gs_gather_mean_dropout");
    if (rc == GS_OK) rc = gs::check_site(self_sites_host[s], "gs_gather_mean_dropout");
    if (rc != GS_OK) return rc;
    drop.neigh[s] = gs::make_drop_site(neigh_sites_host[s]);
    drop.self[s] = gs::make_drop_site(self_sites_host[s]);
  }
  if (tab.total_rows == 0) return GS_OK;
  GS_REQUIRE(src && out_mean, "gs_gather_mean_dropout: NULL pointer");
  GS_REQUIRE(F > 0 && pitch >= F && out_pitch >= F && n_src_rows > 0, "gs_gather_mean_dropout: bad F/pitch");
  cudaStream_t st = (cudaStream_t)stream;
  const int ncol4 = (int)(out_pitch / 4);
  const bool vec_ok = gs::aligned16(src) && gs::aligned16(out_mean) && (!out_self || gs::aligned16(out_self)) &&
                      pitch % 4 == 0 && out_pitch % 4 == 0 && ((F + 3) / 4) * 4 <= pitch;
  if (vec_ok && ncol4 <= 2 * 160) {
    const gs::DenseRows rows_of{src, n_src_rows, pitch};
    return gs::launch_gather_tma2<gs::DenseRows, true>(rows_of, F, tab, include_self, out_self, out_mean, out_pitch, st, &drop);
  }
  int64_t blocks = tab.total_rows;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::gather_mean_scalar_kernel<true><<<(unsigned)blocks, 256, 0, st>>>(src, n_src_rows, F, pitch, tab, include_self, out_self,
                                                                        out_mean, out_pitch, drop);
  return gs::launch_check("gather_mean_scalar_kernel<drop>");
}

int32_t gs_dropout_apply(const float* x, int64_t ldx, int64_t rows, int32_t F, int32_t group, float scale,
                         gs_dropout_site site, int32_t accumulate, float* out, int64_t ldo, const int32_t* pos_ids,
                         void* stream) {
  int32_t rc = gs::check_site(site, "gs_dropout_apply");
  if (rc != GS_OK) return rc;
  GS_REQUIRE(rows >= 0 && F >= 0 && group >= 1, "gs_dropout_apply: bad sizes (rows=%lld F=%d group=%d)", (long long)rows, F,
             group);
  if (rows == 0 || F == 0) return GS_OK;
  GS_REQUIRE(x && out, "gs_dropout_apply: NULL pointer");
  GS_REQUIRE(ldx >= F && ldo >= F, "gs_dropout_apply: row stride < F");
  GS_REQUIRE(x != out || (group == 1 && ldx == ldo), "gs_dropout_apply: in place needs group == 1 and ldo == ldx");
  const int64_t total = rows * ((F + 3) / 4);
  int64_t blocks = (total + 255) / 256;
  int64_t cap = (int64_t)gs::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (pos_ids)
    gs::dropout_apply_kernel<true><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, ldx, rows, F, group, scale,
                                                                                      gs::make_drop_site(site), accumulate,
                                                                                      out, ldo, pos_ids);
  else
    gs::dropout_apply_kernel<false><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, ldx, rows, F, group, scale,
                                                                                       gs::make_drop_site(site), accumulate,
                                                                                       out, ldo, nullptr);
  return gs::launch_check("dropout_apply_kernel");
}

int32_t gs_l2_normalize_rows(float* x, int64_t n, int32_t C, int64_t ldx, void* stream) {
  GS_REQUIRE(n >= 0 && C >= 0, "gs_l2_normalize_rows: bad sizes");
  if (n == 0 || C == 0) return GS_OK;
  GS_REQUIRE(x, "gs_l2_normalize_rows: NULL pointer");
  int64_t blocks = (n + 7) / 8;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::l2_normalize_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, n, C, ldx);
  return gs::launch_check("l2_normalize_kernel");
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// node-partitioned table entry points
// ---------------------------------------------------------------------------------------------
static int32_t fill_shard_tab(const gs_sharded_table* t, gs::ShardRows& sr, int64_t pitch, const char* who) {
  GS_REQUIRE(t != nullptr, "%s: table is NULL", who);
  GS_REQUIRE(t->n_shards >= 1 && t->n_shards <= GS_MAX_SHARDS, "%s: n_shards=%d (max %d)", who, t->n_shards, GS_MAX_SHARDS);
  GS_REQUIRE(t->my_shard >= 0 && t->my_shard < t->n_shards, "%s: my_shard=%d", who, t->my_shard);
  GS_REQUIRE(t->n_global_rows > 0 && t->row_start[0] == 0 && t->row_start[t->n_shards] == t->n_global_rows - 1,
             "%s: row_start must run from 0 to n_global_rows - 1", who);
  for (int i = 0; i < t->n_shards; ++i)
    GS_REQUIRE(t->row_start[i] <= t->row_start[i + 1], "%s: row_start must be non-decreasing (shard %d)", who, i);
  GS_REQUIRE(t->zero_row >= 0, "%s: zero_row < 0", who);
  GS_REQUIRE(pitch % 4 == 0, "%s: pitch must be a multiple of 4 floats", who);
  memset(&sr, 0, sizeof(sr));
  gs::ShardTab& st = sr.t;
  for (int i = 0; i < t->n_shards; ++i) {
    GS_REQUIRE(t->base[i] != nullptr && gs::aligned16(t->base[i]), "%s: shard %d pointer NULL or not 16-byte aligned", who, i);
    st.base[i] = (const float*)t->base[i];
  }
  for (int i = 0; i <= t->n_shards; ++i) st.row_start[i] = t->row_start[i];
  for (int i = t->n_shards + 1; i <= GS_MAX_SHARDS; ++i) st.row_start[i] = t->row_start[t->n_shards];
  st.n_shards = t->n_shards;
  st.my_shard = t->my_shard;
  st.n_global_rows = t->n_global_rows;
  st.zero_row = t->zero_row;
  st.remap = t->remap;
  sr.pitch = pitch;
  return GS_OK;
}

extern "C" {

int32_t gs_translate_ids(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, int32_t* out, void* stream) {
  GS_REQUIRE(table_host && table_host->remap, "gs_translate_ids: the table has no remap (no replicas)");
  GS_REQUIRE(n >= 0, "gs_translate_ids: n < 0");
  if (n == 0) return GS_OK;
  GS_REQUIRE(ids && out, "gs_translate_ids: NULL pointer");
  GS_REQUIRE(table_host->zero_row >= 0 && table_host->zero_row < 0x7fffffffLL, "gs_translate_ids: zero_row out of range");
  int64_t blocks = (n + 255) / 256;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::translate_ids_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(table_host->remap, table_host->n_global_rows,
                                                                                (int32_t)table_host->zero_row, ids, n, out);
  return gs::launch_check("translate_ids_kernel");
}

int32_t gs_halo_begin(int32_t* claim, int64_t n_global_rows, int32_t* count, void* stream) {
  GS_REQUIRE(claim && count && n_global_rows > 0, "gs_halo_begin: bad arguments");
  GS_CUDA(cudaMemsetAsync(claim, 0xff, (size_t)n_global_rows * 4, (cudaStream_t)stream));     // every entry = -1
  GS_CUDA(cudaMemsetAsync(count, 0, 4, (cudaStream_t)stream));
  return GS_OK;
}

int32_t gs_halo_claim(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, int32_t* claim, int32_t* count,
                      int32_t* stage_ids, int64_t capacity, void* stream) {
  gs::ShardRows sr;
  int32_t rc = fill_shard_tab(table_host, sr, 4, "gs_halo_claim");
  if (rc != GS_OK) return rc;
  GS_REQUIRE(n >= 0 && capacity >= 0, "gs_halo_claim: negative size");
  if (n == 0) return GS_OK;
  GS_REQUIRE(ids && claim && count && stage_ids, "gs_halo_claim: NULL pointer");
  int64_t blocks = (n + 255) / 256;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::halo_claim_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(sr.t, ids, n, claim, count, stage_ids, capacity);
  return gs::launch_check("halo_claim_kernel");
}

int32_t gs_halo_translate(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, const int32_t* claim, int32_t* out,
                          void* stream) {
  gs::ShardRows sr;
  int32_t rc = fill_shard_tab(table_host, sr, 4, "gs_halo_translate");
  if (rc != GS_OK) return rc;
  GS_REQUIRE(n >= 0, "gs_halo_translate: n < 0");
  if (n == 0) return GS_OK;
  GS_REQUIRE(ids && claim && out, "gs_halo_translate: NULL pointer");
  int64_t blocks = (n + 255) / 256;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::halo_translate_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(sr.t, ids, n, claim, out, -1, -1);
  return gs::launch_check("halo_translate_kernel");
}

int32_t gs_host_translate(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, const int32_t* claim,
                          int64_t stage_row0, int32_t* out, void* stream) {
  gs::ShardRows sr;
  int32_t rc = fill_shard_tab(table_host, sr, 4, "gs_host_translate");
  if (rc != GS_OK) return rc;
  GS_REQUIRE(n >= 0, "gs_host_translate: n < 0");
  GS_REQUIRE(table_host->remap != nullptr, "gs_host_translate: the table needs its cache_slot array as remap");
  GS_REQUIRE(stage_row0 > table_host->zero_row && stage_row0 < 0x7fffffffLL,
             "gs_host_translate: stage_row0 must follow the zero row and fit int32");
  if (n == 0) return GS_OK;
  GS_REQUIRE(ids && claim && out, "gs_host_translate: NULL pointer");
  int64_t blocks = (n + 255) / 256;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::halo_translate_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(sr.t, ids, n, claim, out,
                                                                                 (int32_t)stage_row0, 1);
  return gs::launch_check("halo_translate_kernel");
}

int32_t gs_halo_fetch(const gs_sharded_table* table_host, int32_t F, int64_t pitch, const int32_t* stage_ids,
                      const int32_t* count, int64_t capacity, float* staging, int64_t staging_pitch, void* stream) {
  gs::ShardRows sr;
  int32_t rc = fill_shard_tab(table_host, sr, pitch, "gs_halo_fetch");
  if (rc != GS_OK) return rc;
  if (capacity == 0) return GS_OK;
  GS_REQUIRE(stage_ids && count && staging && gs::aligned16(staging) && staging_pitch % 4 == 0 && F > 0 &&
                 pitch >= ((F + 3) / 4) * 4 && staging_pitch >= ((F + 3) / 4) * 4,
             "gs_halo_fetch: bad arguments");
  sr.locators = 0;
  sr.staging = nullptr;
  sr.t.remap = nullptr;                        // staged ids are remote by construction: resolve them by owner only
  const int blocks = gs::sm_count() * gs::tuning("halo_fetch_ctas_per_sm", 2);
  gs::halo_fetch_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(sr, (F + 3) / 4, stage_ids, count, capacity, staging,
                                                                            staging_pitch);
  return gs::launch_check("halo_fetch_kernel");
}

int32_t gs_gather_mean_sharded(const gs_sharded_table* table_host, int32_t dtype, int32_t F, int64_t pitch,
                               const gs_segment* segments_host, int32_t n_segments, int32_t include_self,
                               int32_t ids_are_locators, const void* staging, void* out_self, void* out_mean,
                               int64_t out_pitch, void* stream) {
  GS_REQUIRE(dtype == GS_F32, "gs_gather_mean_sharded: only GS_F32 (dtype=%d)", dtype);
  GS_REQUIRE(n_segments >= 0 && n_segments <= GS_MAX_SEGMENTS && (segments_host || n_segments == 0),
             "gs_gather_mean_sharded: bad segments");
  gs::ShardRows sr;
  int32_t rc = fill_shard_tab(table_host, sr, pitch, "gs_gather_mean_sharded");
  if (rc != GS_OK) return rc;
  GS_REQUIRE(ids_are_locators >= 0 && ids_are_locators <= 2 && (ids_are_locators != 2 || staging != nullptr),
             "gs_gather_mean_sharded: ids_are_locators = 2 needs the staging buffer");
  sr.locators = ids_are_locators;
  sr.staging = (const float*)staging;
  gs::SegTable tab;
  rc = fill_seg_table(segments_host, n_segments, tab, "gs_gather_mean_sharded");
  if (rc != GS_OK) return rc;
  if (tab.total_rows == 0) return GS_OK;
  GS_REQUIRE(out_mean && gs::aligned16(out_mean) && (!out_self || gs::aligned16(out_self)) && out_pitch % 4 == 0 &&
                 F > 0 && pitch >= ((F + 3) / 4) * 4 && out_pitch >= F,
             "gs_gather_mean_sharded: bad output / pitch");
  const int ncol4 = (int)(out_pitch / 4);
  // default: the grouped double-buffered bulk-copy kernel of the dense table with peer-mapped row addresses - a
  // remote row is one cp.async.bulk over NVLink straight into this SM's shared memory (gather_variant=0: 128-bit loads)
  if (gs::tuning("gather_variant", 2) != 0 && ncol4 <= 2 * 160)
    return gs::launch_gather_tma2(sr, F, tab, include_self, (float*)out_self, (float*)out_mean, out_pitch, (cudaStream_t)stream);
  int threads = ((ncol4 + 31) / 32) * 32;
  if (threads > 256) threads = 256;
  int64_t blocks = tab.total_rows;
  int64_t cap = (int64_t)gs::sm_count() * gs::tuning("gather_ctas_per_sm", 8);
  if (blocks > cap) blocks = cap;
  gs::gather_mean_sharded_kernel<5><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      sr, F, tab, include_self, (float*)out_self, (float*)out_mean, out_pitch);
  return gs::launch_check("gather_mean_sharded_kernel");
}

int32_t gs_gather_rows_sharded(const gs_sharded_table* table_host, int32_t dtype, int32_t F, int64_t pitch,
                               const int32_t* ids, int64_t n, void* out, int64_t out_pitch, void* stream) {
  GS_REQUIRE(dtype == GS_F32, "gs_gather_rows_sharded: only GS_F32 (dtype=%d)", dtype);
  gs::ShardRows sr;
  int32_t rc = fill_shard_tab(table_host, sr, pitch, "gs_gather_rows_sharded");
  if (rc != GS_OK) return rc;
  if (n == 0) return GS_OK;
  GS_REQUIRE(ids && out && gs::aligned16(out) && out_pitch % 4 == 0 && F > 0 && pitch >= ((F + 3) / 4) * 4 && out_pitch >= F,
             "gs_gather_rows_sharded: bad arguments");
  int64_t blocks = (n + 7) / 8;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::gather_rows_sharded_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(sr, F, ids, n, (float*)out, out_pitch);
  return gs::launch_check("gather_rows_sharded_kernel");
}

int32_t gs_shard_alloc(int64_t bytes, void** dev_ptr_out) {
  GS_REQUIRE(bytes > 0 && dev_ptr_out, "gs_shard_alloc: bad arguments");
  GS_CUDA(cudaMalloc(dev_ptr_out, (size_t)bytes));
  return GS_OK;
}

int32_t gs_shard_free(void* dev_ptr) {
  if (dev_ptr) GS_CUDA(cudaFree(dev_ptr));
  return GS_OK;
}

int32_t gs_ipc_export(const void* dev_ptr, uint8_t* handle64_out_host) {
  GS_REQUIRE(dev_ptr && handle64_out_host, "gs_ipc_export: NULL argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  cudaIpcMemHandle_t h;
  GS_CUDA(cudaIpcGetMemHandle(&h, const_cast<void*>(dev_ptr)));
  memcpy(handle64_out_host, &h, 64);
  return GS_OK;
}

int32_t gs_ipc_import(const uint8_t* handle64_host, void** dev_ptr_out) {
  GS_REQUIRE(handle64_host && dev_ptr_out, "gs_ipc_import: NULL argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64_host, 64);
  GS_CUDA(cudaIpcOpenMemHandle(dev_ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  return GS_OK;
}

int32_t gs_ipc_close(void* dev_ptr) {
  if (dev_ptr) GS_CUDA(cudaIpcCloseMemHandle(dev_ptr));
  return GS_OK;
}

}  // extern "C"

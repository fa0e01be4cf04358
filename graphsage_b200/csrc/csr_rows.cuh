// One schedule for reductions over variable-length CSR rows, shared by gs_csr_aggregate (csr_aggregate.cu) and
// gs_csr_max_backward (csr_backward.cu).  Every output element is ONE sequential chain over its row's entries in order,
// so no work split may cut a row along its entries.  Two roles share one launch of kCsrThreads-thread CTAs:
//   hub role (the first hub_blocks CTAs): rows with more than kCsrLong entries.  Work item = (chunk of kHubChunk rows,
//     slice of kHubCols columns); the CTA finds the long rows of its chunk and, per row, its 8 warps load 64 entries'
//     terms into a double-buffered shared tile while warp 0 sums the previous 64 in order.  A hub is spread over
//     ceil(columns / 32) CTAs and keeps 64 entries in flight in each, instead of one warp walking 10^5 dependent steps.
//   short role (the rest): one warp per (row, slice of 32 * V columns), V columns per lane, kUnroll entries' loads in
//     flight before they are summed in order.
// Hub CTAs come first in the grid, so the long rows start before the short ones fill the machine.
//
// A kernel calls csr_rows<V, kUnroll>(p, tile) with a policy object p (inlined) for what differs between kernels: p.a
// (its arguments: F, hub_items, hub_blocks), kFromFirst (the chain starts from its first entry, as the max does, not
// from +0), kEmptyIsDummy (the short role reduces an empty row over one entry, the dummy row), the launch's rows(),
// hub_slices(), slices() and out_cols() (the columns written), row(i) (row i's entry range: Row::cnt entries), begin()
// (row state read before the entries; col_ok: c < F), value() (the term an entry adds at one column, hub role), load()
// and mask() (an entry's W columns, ok: inside the row; the loads, then what is applied before the sum), weight() and
// scale() (an entry's scale, loaded beside its columns, applied after mask() where the term is consumed - so no load
// waits on another; 1 and nothing where a kernel has no scale), hub_mask() (applied to the hub role's kHubPerWarp
// terms), step(), finish() (the chain's end on columns c0 .. c0 + W - 1 < F) and store().
#pragma once
#include <algorithm>

#include "common.cuh"

namespace gs {

constexpr int kCsrThreads = 256;
constexpr int64_t kCsrLong = 256;     // rows with more entries go to the hub role
constexpr int kHubChunk = 256;        // rows scanned per hub work item (one per thread)
constexpr int kHubCols = 32;          // columns per hub work item (one per lane of the summing warp)
constexpr int kHubPerWarp = 8;        // entries each warp loads per round
constexpr int kHubRows = kHubPerWarp * (kCsrThreads / 32);   // entries per round: 64

// host: the grid over `rows` rows in slices of 32 (hub role) and 32 * V (short role) columns; sets hub_items and
// hub_blocks, returns the CTA count
inline unsigned csr_grid(int64_t rows, int32_t hub_slices, int32_t slices, int64_t& hub_items, int64_t& hub_blocks) {
  hub_items = (rows + kHubChunk - 1) / kHubChunk * hub_slices;
  hub_blocks = std::min<int64_t>(hub_items, (int64_t)sm_count() * 4);
  const int64_t short_blocks = std::min<int64_t>((rows * slices + 7) / 8, (int64_t)sm_count() * 8 * 64);
  return (unsigned)(hub_blocks + short_blocks);
}

template <class P>
__device__ void csr_hub_role(const P& p, float (*tile)[kHubRows][kHubCols]) {
  __shared__ int32_t list[kHubChunk];
  __shared__ int32_t warp_count[kCsrThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t item = blockIdx.x; item < p.a.hub_items; item += p.a.hub_blocks) {
    const int64_t chunk = item / p.hub_slices();
    const int c = (int)(item % p.hub_slices()) * kHubCols + lane;
    const bool col_ok = c < p.a.F;
    // the chunk's long rows, in row order (ballot + per-warp offsets: no atomics)
    const int64_t i0 = chunk * kHubChunk + threadIdx.x;
    typename P::Row r;
    r.cnt = 0;
    if (i0 < p.rows()) r = p.row(i0);
    const bool is_long = r.cnt > kCsrLong;
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
      r = p.row(i);
      p.begin(r, i, c, col_ok);
      float x[kHubPerWarp];
#pragma unroll
      for (int u = 0; u < kHubPerWarp; ++u) {
        const int e = warp * kHubPerWarp + u;
        x[u] = col_ok ? p.value(r, e, c) : 0.f;                // cnt > kHubRows
      }
      p.hub_mask(r, warp * kHubPerWarp, c, x);
      float acc = 0.f;
      int buf = 0;
      for (int64_t base = 0; base < r.cnt; base += kHubRows, buf ^= 1) {
#pragma unroll
        for (int u = 0; u < kHubPerWarp; ++u) tile[buf][warp * kHubPerWarp + u][lane] = x[u];
        __syncthreads();
        const int64_t next = base + kHubRows + warp * kHubPerWarp;
#pragma unroll
        for (int u = 0; u < kHubPerWarp; ++u)                 // the next round's loads are in flight during the sum
          x[u] = (col_ok && next + u < r.cnt) ? p.value(r, next + u, c) : 0.f;
        p.hub_mask(r, next, c, x);
        if (warp == 0) {
          const int m = (int)min((int64_t)kHubRows, r.cnt - base);
          int t = 0;
          if (P::kFromFirst && base == 0) acc = tile[buf][t++][lane];
          for (; t < m; ++t) acc = p.step(acc, tile[buf][t][lane]);
        }
      }
      if (warp == 0 && c < p.out_cols()) {
        float y[1] = {0.f};
        if (col_ok) {
          y[0] = acc;
          p.finish(r, c, r.cnt, y);
        }
        p.store(r, i, c, y);
      }
      __syncthreads();      // the tiles are reused by the next row
    }
    __syncthreads();        // `list` and `warp_count` are rewritten by the next item
  }
}

template <int V, int kUnroll, class P>
__device__ void csr_short_role(const P& p, int64_t block) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t items = p.rows() * p.slices();
  const int64_t stride = ((int64_t)gridDim.x - p.a.hub_blocks) * (kCsrThreads / 32);
  for (int64_t item = block * (kCsrThreads / 32) + warp; item < items; item += stride) {
    const int64_t i = item / p.slices();
    const int c0 = ((int)(item % p.slices()) * 32 + lane) * V;
    typename P::Row r = p.row(i);
    if (r.cnt > kCsrLong || c0 >= p.out_cols()) continue;    // a hub row (hub role), or past the row's last column
    float acc[V];
#pragma unroll
    for (int q = 0; q < V; ++q) acc[q] = 0.f;
    if (c0 < p.a.F) {
      const int64_t count = P::kEmptyIsDummy ? (r.cnt > 0 ? r.cnt : 1) : r.cnt;
      p.begin(r, i, c0, true);
      int64_t e = 0;
      if constexpr (P::kFromFirst) {
        float x0[V];
        p.load(r, e, c0, true, x0);
        p.scale(p.weight(r, e++, true), x0);
#pragma unroll
        for (int q = 0; q < V; ++q) acc[q] = x0[q];
      }
      for (; e < count; e += kUnroll) {
        float x[kUnroll][V];
        float wt[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          p.load(r, e + u, c0, e + u < count, x[u]);
          wt[u] = p.weight(r, e + u, e + u < count);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
          if (e + u < count) {
            p.mask(r, e + u, c0, x[u]);
            p.scale(wt[u], x[u]);
#pragma unroll
            for (int q = 0; q < V; ++q) acc[q] = p.step(acc[q], x[u][q]);
          }
      }
      p.finish(r, c0, count, acc);
    }
    p.store(r, i, c0, acc);
  }
}

// the kernel body: hub CTAs first, then the short role with V columns per lane and kUnroll entries in flight
template <int V, int kUnroll, class P>
__device__ __forceinline__ void csr_rows(const P& p, float (*tile)[kHubRows][kHubCols]) {
  if (blockIdx.x < p.a.hub_blocks) csr_hub_role(p, tile);
  else csr_short_role<V, kUnroll>(p, (int64_t)blockIdx.x - p.a.hub_blocks);
}

}  // namespace gs

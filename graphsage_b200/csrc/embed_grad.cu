// Backward of the layer-0 embedding lookup (reference graphsage/models.py:299, tf.nn.embedding_lookup on the trainable
// node_embeddings table): the IndexedSlices gradient densified into [n_rows, d], deterministically.
//
//   1. keys/values: contribution c (lists concatenated in call order) -> (id, c); ids outside [0, n_rows) get the
//      sentinel key n_rows and contribute nothing.
//   2. CUB radix sort of (key, c).  The sort is stable and c starts ascending, so each id's contributions end up in
//      ascending c order.
//   3. chunk pass: the sorted array is cut into fixed chunks of kChunk entries, one warp per chunk.  The warp sums every
//      id run inside its chunk in sorted order; a run that lies wholly inside the chunk is written to out[id], a run
//      that crosses a chunk edge leaves its piece in a partial slot (first piece of chunk j -> slot 2j, last -> 2j+1).
//   4. combine pass: the chunk where a crossing run starts adds the run's pieces in a fixed lane / chunk order.
// No atomics anywhere: the result depends on the inputs only.
// gs_embedding_sgd is the same machinery with the stores turned into in-place updates of the touched rows,
// table[id] = fmaf(alpha, sum, table[id]) with one rounding (kApply); it clears nothing, so untouched rows are neither
// read nor written.  The chunk pass's products and sums and the update are written as __fmul_rn / __fadd_rn /
// __fmaf_rn so that no compiler contraction can change the rounding oracle/sparse_grad.py emulates.
#define CUB_WRAPPED_NAMESPACE gs_cub
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace gs {
namespace {

constexpr int kChunk = 32;           // sorted contributions per chunk (one warp)
constexpr int kColsPerLane = 4;      // chunk pass column tile = 128 columns
constexpr int kBatch = 8;            // gradient rows loaded ahead in the chunk pass
constexpr int kLanes = 8;            // combine pass: piece lanes x 32 columns = 256 threads
constexpr int kUnroll = 4;           // independent accumulators per piece lane

struct ListDev {
  const int32_t* ids;
  const float* grad;
  int64_t ldg;
  int64_t offset;       // first global contribution index of this list
  int32_t group;
  float scale;
  DropSite site;        // gs_embedding_grad_dropout only
};
struct Lists {
  ListDev l[GS_MAX_EMBED_LISTS];
  int32_t count;
};

__device__ __forceinline__ int find_list(const Lists& L, int64_t c) {
  int li = 0;
  while (li + 1 < L.count && c >= L.l[li + 1].offset) ++li;
  return li;
}

__global__ void embed_keys_kernel(Lists L, int64_t total, uint32_t n_rows, uint32_t* __restrict__ keys,
                                  int32_t* __restrict__ vals) {
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (int64_t)gridDim.x * blockDim.x) {
    const ListDev& l = L.l[find_list(L, c)];
    int32_t id = l.ids[c - l.offset];
    keys[c] = ((uint32_t)id < n_rows) ? (uint32_t)id : n_rows;
    vals[c] = (int32_t)c;
  }
}

// kDrop: every product scale * grad goes through its list's dropout mask at pos = index in the list (the masked entry)
// kApply: out is a table updated in place, out[id] += alpha * (row sum), instead of a gradient written with out[id] = sum
template <bool kDrop, bool kApply>
__global__ void __launch_bounds__(256) embed_chunk_kernel(Lists L, const uint32_t* __restrict__ keys,
                                                          const int32_t* __restrict__ vals, int64_t total,
                                                          uint32_t n_rows, int32_t d, float* __restrict__ out,
                                                          int64_t ldo, float* __restrict__ partial, float alpha) {
  const unsigned FULL = 0xffffffffu;
  __shared__ uint32_t call_off[GS_MAX_EMBED_LISTS];       // kDrop: each list's device-side call offset
  if constexpr (kDrop) {
    if (threadIdx.x < L.count) call_off[threadIdx.x] = drop_call_offset(L.l[threadIdx.x].site);
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  const int64_t nchunks = (total + kChunk - 1) / kChunk;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < nchunks; j += nwarps) {
    const int64_t s = j * kChunk;
    const int cnt = (int)min((int64_t)kChunk, total - s);
    // lane i resolves sorted entry s + i: its key, gradient row and scale
    uint32_t my_key = n_rows;
    const float* my_row = nullptr;
    float my_scale = 0.f;
    int64_t my_pos = 0;
    int my_list = 0;
    if (lane < cnt) {
      my_key = keys[s + lane];
      if (my_key < n_rows) {
        int64_t c = vals[s + lane];
        my_list = find_list(L, c);
        const ListDev& l = L.l[my_list];
        my_pos = c - l.offset;
        my_row = l.grad + (my_pos / l.group) * l.ldg;
        my_scale = l.scale;
      }
    }
    const uint32_t key_before = s > 0 ? keys[s - 1] : 0xffffffffu;
    const uint32_t key_after = s + cnt < total ? keys[s + cnt] : 0xffffffffu;
    const uint32_t next_key = __shfl_down_sync(FULL, my_key, 1);
    const unsigned piece_end = __ballot_sync(FULL, lane < cnt && (lane == cnt - 1 || next_key != my_key));
    for (int c0 = 0; c0 < d; c0 += 32 * kColsPerLane) {
      float acc[kColsPerLane];
#pragma unroll
      for (int q = 0; q < kColsPerLane; ++q) acc[q] = 0.f;
      int piece_start = 0;
      for (int b = 0; b < cnt; b += kBatch) {
        float v[kBatch][kColsPerLane];
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
          const int i = (b + u) & 31;
          const float* row = (const float*)__shfl_sync(FULL, (unsigned long long)my_row, i);
          const float sc = __shfl_sync(FULL, my_scale, i);
          int64_t pos = 0;
          int li = 0;
          if constexpr (kDrop) {
            pos = __shfl_sync(FULL, my_pos, i);
            li = __shfl_sync(FULL, my_list, i);
          }
#pragma unroll
          for (int q = 0; q < kColsPerLane; ++q) {
            const int col = c0 + lane + 32 * q;
            v[u][q] = (b + u < cnt && row != nullptr && col < d) ? __fmul_rn(sc, __ldg(row + col)) : 0.f;
            if constexpr (kDrop) v[u][q] = drop_col(with_call_offset(L.l[li].site, call_off[li]), pos, col, v[u][q]);
          }
        }
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
          const int i = b + u;
          if (i >= cnt) break;
#pragma unroll
          for (int q = 0; q < kColsPerLane; ++q) acc[q] = __fadd_rn(acc[q], v[u][q]);
          if ((piece_end >> i) & 1u) {
            const uint32_t key = __shfl_sync(FULL, my_key, i);
            if (key < n_rows) {
              const bool before = piece_start == 0 && key_before == key;
              const bool after = i == cnt - 1 && key_after == key;
              const bool whole = !before && !after;
              float* dst = whole ? out + (int64_t)key * ldo
                                 : partial + (2 * j + (piece_start == 0 ? 0 : 1)) * (int64_t)d;
#pragma unroll
              for (int q = 0; q < kColsPerLane; ++q) {
                const int col = c0 + lane + 32 * q;
                if constexpr (kApply) {
                  if (col < d) dst[col] = whole ? __fmaf_rn(alpha, acc[q], dst[col]) : acc[q];
                } else {
                  if (col < d) dst[col] = acc[q];
                }
              }
            }
#pragma unroll
            for (int q = 0; q < kColsPerLane; ++q) acc[q] = 0.f;
            piece_start = i + 1;
          }
        }
      }
    }
  }
}

template <bool kApply>
__global__ void __launch_bounds__(kLanes * 32) embed_combine_kernel(const uint32_t* __restrict__ keys, int64_t total,
                                                                    uint32_t n_rows, int32_t d,
                                                                    const float* __restrict__ partial,
                                                                    float* __restrict__ out, int64_t ldo, float alpha) {
  __shared__ float red[kLanes][32];
  __shared__ int64_t run_end;
  const int cl = threadIdx.x & 31, p = threadIdx.x >> 5;
  const int64_t nchunks = (total + kChunk - 1) / kChunk;
  for (int64_t j = blockIdx.x; j < nchunks; j += gridDim.x) {
    const int64_t s = j * kChunk, e = s + kChunk;
    if (e >= total) continue;                                    // nothing continues past the last entry
    const uint32_t X = keys[e - 1];
    if (X >= n_rows || keys[e] != X) continue;                  // the chunk's last run ends inside it
    if (s > 0 && keys[s - 1] == X) continue;                    // the run started in an earlier chunk
    if (threadIdx.x == 0) {
      int64_t lo = e, hi = total;                               // first sorted index past the run
      while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (keys[mid] == X) lo = mid + 1; else hi = mid;
      }
      run_end = lo;
    }
    __syncthreads();
    const int64_t npieces = (run_end - 1) / kChunk - j + 1;
    const int64_t first_slot = keys[s] == X ? 2 * j : 2 * j + 1;
    for (int c0 = 0; c0 < d; c0 += 32) {
      const int col = c0 + cl;
      float a[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) a[u] = 0.f;
      if (col < d) {
        // piece q = p + kLanes * (kUnroll * t + u) goes to accumulator u of lane p
        for (int64_t q0 = p; q0 < npieces; q0 += kLanes * kUnroll) {
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const int64_t q = q0 + (int64_t)kLanes * u;
            if (q < npieces) {
              const int64_t slot = q == 0 ? first_slot : 2 * (j + q);
              a[u] += partial[slot * d + col];
            }
          }
        }
      }
      float t = a[0];
#pragma unroll
      for (int u = 1; u < kUnroll; ++u) t += a[u];
      red[p][cl] = t;
      __syncthreads();
      if (p == 0 && col < d) {
        float r = red[0][cl];
#pragma unroll
        for (int pp = 1; pp < kLanes; ++pp) r += red[pp][cl];
        if constexpr (kApply)
          out[(int64_t)X * ldo + col] = __fmaf_rn(alpha, r, out[(int64_t)X * ldo + col]);
        else
          out[(int64_t)X * ldo + col] = r;
      }
      __syncthreads();
    }
  }
}

struct Plan {
  int64_t total = 0, nchunks = 0;
  int end_bit = 1;
  size_t off_keys_in = 0, off_keys_out = 0, off_vals_in = 0, off_vals_out = 0, off_partial = 0, off_cub = 0;
  size_t cub_bytes = 0, bytes = 0;
};

int32_t make_plan(const gs_embed_grad_list* lists, int32_t n_lists, int64_t n_rows, int32_t d, Plan& P,
                  const char* who) {
  GS_REQUIRE(n_lists >= 0 && n_lists <= GS_MAX_EMBED_LISTS, "%s: n_lists must be in [0, %d]", who,
             GS_MAX_EMBED_LISTS);
  GS_REQUIRE(n_lists == 0 || lists != nullptr, "%s: lists is NULL", who);
  GS_REQUIRE(n_rows >= 0 && n_rows < 0x7fffffffLL, "%s: n_rows must be in [0, 2^31 - 1)", who);
  GS_REQUIRE(d >= 0, "%s: d must be >= 0", who);
  for (int i = 0; i < n_lists; ++i) {
    const gs_embed_grad_list& l = lists[i];
    GS_REQUIRE(l.n >= 0, "%s: list %d has n < 0", who, i);
    if (l.n == 0) continue;
    GS_REQUIRE(l.group >= 1, "%s: list %d has group < 1", who, i);
    GS_REQUIRE(l.ids != nullptr && l.grad != nullptr, "%s: list %d has a NULL pointer", who, i);
    GS_REQUIRE(l.ldg >= d, "%s: list %d has ldg < d", who, i);
    P.total += l.n;
  }
  GS_REQUIRE(P.total < 0x7fffffffLL, "%s: more than 2^31 - 1 contributions", who);
  P.nchunks = (P.total + kChunk - 1) / kChunk;
  P.end_bit = 1;
  while (P.end_bit < 32 && ((uint64_t)n_rows >> P.end_bit) != 0) ++P.end_bit;   // keys are <= n_rows
  if (P.total > 0) {
    cudaError_t e = gs_cub::cub::DeviceRadixSort::SortPairs(nullptr, P.cub_bytes, (const uint32_t*)nullptr,
                                                            (uint32_t*)nullptr, (const int32_t*)nullptr,
                                                            (int32_t*)nullptr, (int)P.total, 0, P.end_bit);
    if (e != cudaSuccess) return cuda_fail(e, "cub::DeviceRadixSort::SortPairs (size query)");
  }
  size_t off = 0;
  const size_t n4 = align256((size_t)P.total * 4);
  P.off_keys_in = off;  off += n4;
  P.off_keys_out = off; off += n4;
  P.off_vals_in = off;  off += n4;
  P.off_vals_out = off; off += n4;
  P.off_partial = off;  off += align256((size_t)P.nchunks * 2 * (size_t)d * 4);
  P.off_cub = off;      off += align256(P.cub_bytes);
  P.bytes = P.total > 0 ? off : 0;
  return GS_OK;
}

}  // namespace
}  // namespace gs

extern "C" {

int64_t gs_embedding_grad_workspace_bytes(const gs_embed_grad_list* lists_host, int32_t n_lists, int64_t n_rows,
                                          int32_t d) {
  gs::Plan P;
  if (gs::make_plan(lists_host, n_lists, n_rows, d, P, "gs_embedding_grad_workspace_bytes") != GS_OK) return -1;
  return (int64_t)P.bytes;
}

static int32_t embedding_grad(const gs_embed_grad_list* lists_host, const gs_dropout_site* sites_host, int32_t n_lists,
                              int64_t n_rows, int32_t d, float* out, int64_t ldo, void* workspace, int64_t workspace_bytes,
                              void* stream, const char* who, bool apply = false, float alpha = 0.f) {
  gs::Plan P;
  int32_t rc = gs::make_plan(lists_host, n_lists, n_rows, d, P, who);
  if (rc != GS_OK) return rc;
  if (n_rows == 0 || d == 0) return GS_OK;
  GS_REQUIRE(out != nullptr, "%s: out is NULL", who);
  GS_REQUIRE(ldo >= d, "%s: ldo < d", who);
  GS_REQUIRE(workspace_bytes >= (int64_t)P.bytes && (P.bytes == 0 || workspace != nullptr),
             "%s: workspace of %lld bytes, %lld needed", who, (long long)workspace_bytes,
             (long long)P.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  if (!apply) GS_CUDA(cudaMemset2DAsync(out, (size_t)ldo * 4, 0, (size_t)d * 4, (size_t)n_rows, st));
  if (P.total == 0) return GS_OK;

  gs::Lists L{};
  int64_t off = 0;
  for (int i = 0; i < n_lists; ++i) {
    const gs_embed_grad_list& l = lists_host[i];
    if (l.n == 0) continue;
    L.l[L.count] = gs::ListDev{l.ids, l.grad, l.ldg, off, l.group, l.scale, gs::DropSite{}};
    if (sites_host) L.l[L.count].site = gs::make_drop_site(sites_host[i]);
    ++L.count;
    off += l.n;
  }
  char* ws = (char*)workspace;
  uint32_t* keys_in = (uint32_t*)(ws + P.off_keys_in);
  uint32_t* keys_out = (uint32_t*)(ws + P.off_keys_out);
  int32_t* vals_in = (int32_t*)(ws + P.off_vals_in);
  int32_t* vals_out = (int32_t*)(ws + P.off_vals_out);
  float* partial = (float*)(ws + P.off_partial);
  const int64_t cap = (int64_t)gs::sm_count() * 8;

  int64_t blocks = (P.total + 255) / 256;
  if (blocks > cap) blocks = cap;
  gs::embed_keys_kernel<<<(unsigned)blocks, 256, 0, st>>>(L, P.total, (uint32_t)n_rows, keys_in, vals_in);
  rc = gs::launch_check("embed_keys_kernel");
  if (rc != GS_OK) return rc;

  size_t cub_bytes = P.cub_bytes;
  cudaError_t e = gs_cub::cub::DeviceRadixSort::SortPairs(ws + P.off_cub, cub_bytes, keys_in, keys_out, vals_in,
                                                          vals_out, (int)P.total, 0, P.end_bit, st);
  if (e != cudaSuccess) return gs::cuda_fail(e, "cub::DeviceRadixSort::SortPairs");

  blocks = (P.nchunks * 32 + 255) / 256;
  if (blocks > cap * 2) blocks = cap * 2;
  if (apply)
    gs::embed_chunk_kernel<false, true><<<(unsigned)blocks, 256, 0, st>>>(L, keys_out, vals_out, P.total, (uint32_t)n_rows, d,
                                                                          out, ldo, partial, alpha);
  else if (sites_host)
    gs::embed_chunk_kernel<true, false><<<(unsigned)blocks, 256, 0, st>>>(L, keys_out, vals_out, P.total, (uint32_t)n_rows, d,
                                                                          out, ldo, partial, 0.f);
  else
    gs::embed_chunk_kernel<false, false><<<(unsigned)blocks, 256, 0, st>>>(L, keys_out, vals_out, P.total, (uint32_t)n_rows, d,
                                                                           out, ldo, partial, 0.f);
  rc = gs::launch_check("embed_chunk_kernel");
  if (rc != GS_OK) return rc;

  blocks = P.nchunks < cap ? P.nchunks : cap;
  if (apply)
    gs::embed_combine_kernel<true><<<(unsigned)blocks, gs::kLanes * 32, 0, st>>>(keys_out, P.total, (uint32_t)n_rows, d,
                                                                                partial, out, ldo, alpha);
  else
    gs::embed_combine_kernel<false><<<(unsigned)blocks, gs::kLanes * 32, 0, st>>>(keys_out, P.total, (uint32_t)n_rows, d,
                                                                                 partial, out, ldo, 0.f);
  return gs::launch_check("embed_combine_kernel");
}

int32_t gs_embedding_grad(const gs_embed_grad_list* lists_host, int32_t n_lists, int64_t n_rows, int32_t d, float* out,
                          int64_t ldo, void* workspace, int64_t workspace_bytes, void* stream) {
  return embedding_grad(lists_host, nullptr, n_lists, n_rows, d, out, ldo, workspace, workspace_bytes, stream,
                        "gs_embedding_grad");
}

int32_t gs_embedding_grad_dropout(const gs_embed_grad_list* lists_host, const gs_dropout_site* sites_host, int32_t n_lists,
                                  int64_t n_rows, int32_t d, float* out, int64_t ldo, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
  for (int i = 0; sites_host && i < n_lists; ++i)
    GS_REQUIRE(sites_host[i].rate >= 0.f && sites_host[i].rate < 1.f, "gs_embedding_grad_dropout: list %d has rate %g outside [0, 1)",
               i, (double)sites_host[i].rate);
  return embedding_grad(lists_host, sites_host, n_lists, n_rows, d, out, ldo, workspace, workspace_bytes, stream,
                        "gs_embedding_grad_dropout");
}

int32_t gs_embedding_sgd(const gs_embed_grad_list* lists_host, int32_t n_lists, int64_t n_rows, int32_t d, float alpha,
                         float* table, int64_t ldt, void* workspace, int64_t workspace_bytes, void* stream) {
  GS_REQUIRE(isfinite(alpha), "gs_embedding_sgd: alpha must be finite");
  return embedding_grad(lists_host, nullptr, n_lists, n_rows, d, table, ldt, workspace, workspace_bytes, stream,
                        "gs_embedding_sgd", true, alpha);
}

}  // extern "C"

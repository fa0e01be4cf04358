// K1: UniformNeighborSampler kernels.
//   padded mode  - reference graphsage/neigh_samplers.py:24-29 (one shared column permutation per call)
//   CSR mode     - warp-per-node per-node draws (north_star), semantics in oracle/sampler.py
#include "common.cuh"

namespace gs {

constexpr int kMaxDegSmem = 1024;  // permutation scratch (int16 entries) lives in static smem

// Each block recomputes the k-step Fisher-Yates prefix in shared memory (k <= 32 steps of a
// serial swap chain - ~1 us, cheaper than a separate launch), then threads stream
// out[i*k + j] = adj[ids[i]*MD + pi[j]].  Integer/byte work: bound by the 4-byte random reads
// of the adj table (k sectors per node), not by anything a tensor core could help with.
__global__ void __launch_bounds__(256) sample_padded_kernel(const int32_t* __restrict__ adj, int64_t n_rows,
                                                            int32_t max_deg, const int32_t* __restrict__ ids,
                                                            int64_t n, int32_t k,
                                                            const int32_t* __restrict__ col_perm, uint64_t seed,
                                                            uint64_t counter, const uint64_t* __restrict__ counter_dev,
                                                            int32_t* __restrict__ out) {
  __shared__ int16_t perm[kMaxDegSmem];
  __shared__ int32_t pi[kMaxDegSmem];
  if (col_perm != nullptr) {
    for (int j = threadIdx.x; j < k; j += blockDim.x) pi[j] = col_perm[j];
  } else {
    for (int j = threadIdx.x; j < max_deg; j += blockDim.x) perm[j] = (int16_t)j;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint64_t ctr = counter + (counter_dev ? *counter_dev : 0ull);
      u32x4 r{0, 0, 0, 0};
      for (int i = 0; i < k; ++i) {
        if ((i & 3) == 0) {
          u32x4 c{(uint32_t)ctr, (uint32_t)(ctr >> 32), 0u, kStreamPadded + (uint32_t)(i >> 2)};  // oracle/sampler.py:_draws
          r = philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
        }
        int j = i + (int)mulhi32(pick(r, i & 3), (uint32_t)(max_deg - i));
        int16_t t = perm[i];
        perm[i] = perm[j];
        perm[j] = t;
        pi[i] = perm[i];
      }
    }
  }
  __syncthreads();
  const int64_t total = n * (int64_t)k;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = e / k;
    int j = (int)(e - i * k);
    int64_t id = ids[i];
    if (id < 0 || id >= n_rows) id = n_rows - 1;  // out-of-range -> dummy row (TF GPU gather would return zeros)
    out[e] = adj[id * max_deg + pi[j]];
  }
}

// The whole frontier expansion (models.py:254-275) in one launch.  Warp t of each block builds hop
// t's permutation prefix; every output element re-walks its ancestor chain from the seed
// (hop-t element = t dependent 4-byte loads; siblings share all but the last, served by L1).
struct KhopParams {
  int32_t* out[GS_MAX_HOPS];
  int32_t fanout[GS_MAX_HOPS];
  int64_t count[GS_MAX_HOPS];     // elements of hop t+1 = n_seeds * prod(fanout[0..t])
  int32_t n_hops;
};

__global__ void __launch_bounds__(512) sample_padded_khop_kernel(const int32_t* __restrict__ adj, int64_t n_rows,
                                                                 int32_t max_deg, const int32_t* __restrict__ seeds,
                                                                 const __grid_constant__ KhopParams kp, uint64_t seed,
                                                                 uint64_t counter,
                                                                 const uint64_t* __restrict__ counter_dev) {
  __shared__ int16_t perm[GS_MAX_HOPS][kMaxDegSmem];
  __shared__ int32_t pi[GS_MAX_HOPS][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < kp.n_hops) {
    for (int j = lane; j < max_deg; j += 32) perm[warp][j] = (int16_t)j;
    __syncwarp();
    // the k draws are independent Philox blocks: lanes compute them in parallel (draw i = word i&3 of block i>>2),
    // then lane 0 runs the short serial swap chain
    const uint64_t ctr = counter + (counter_dev ? *counter_dev : 0ull) + (uint64_t)warp;
    const int k = kp.fanout[warp];
    for (int blk = lane; blk * 4 < k; blk += 32) {
      u32x4 c{(uint32_t)ctr, (uint32_t)(ctr >> 32), 0u, kStreamPadded + (uint32_t)blk};
      u32x4 r = philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
      pi[warp][blk * 4 + 0] = (int32_t)r.x;
      if (blk * 4 + 1 < 64) pi[warp][blk * 4 + 1] = (int32_t)r.y;
      if (blk * 4 + 2 < 64) pi[warp][blk * 4 + 2] = (int32_t)r.z;
      if (blk * 4 + 3 < 64) pi[warp][blk * 4 + 3] = (int32_t)r.w;
    }
    __syncwarp();
    if (lane == 0) {
      for (int i = 0; i < k; ++i) {
        int j = i + (int)mulhi32((uint32_t)pi[warp][i], (uint32_t)(max_deg - i));
        int16_t t = perm[warp][i];
        perm[warp][i] = perm[warp][j];
        perm[warp][j] = t;
        pi[warp][i] = perm[warp][i];
      }
    }
  }
  __syncthreads();
  int64_t total = 0;
  for (int t = 0; t < kp.n_hops; ++t) total += kp.count[t];
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int hop = 0;
    int64_t local = e;
    while (local >= kp.count[hop]) { local -= kp.count[hop]; ++hop; }
    // support size of this hop and the ancestor chain
    int64_t sup = 1;
    for (int t = 0; t <= hop; ++t) sup *= kp.fanout[t];
    int64_t id = seeds[local / sup];
    int64_t rem = local % sup;
    for (int t = 0; t <= hop; ++t) {
      sup /= kp.fanout[t];
      const int j = (int)(rem / sup);
      rem -= (int64_t)j * sup;
      if (id < 0 || id >= n_rows) id = n_rows - 1;
      id = adj[id * max_deg + pi[t][j]];
    }
    kp.out[hop][local] = (int32_t)id;
  }
}

// One warp per requested node; lane j owns draw j (k <= 32).
__global__ void __launch_bounds__(256) sample_csr_kernel(const int64_t* __restrict__ indptr,
                                                         const int32_t* __restrict__ indices, int64_t n_nodes,
                                                         const int32_t* __restrict__ ids, int64_t n, int32_t k,
                                                         int32_t replace_if_short, uint64_t seed, uint64_t counter,
                                                         const uint64_t* __restrict__ counter_dev, int32_t pad_id,
                                                         int32_t* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const uint64_t ctr = counter + (counter_dev ? *counter_dev : 0ull);
  for (int64_t t = warp; t < n; t += nwarps) {
    int64_t id = ids[t];
    int64_t start = 0, deg = 0;
    if (id >= 0 && id < n_nodes) {
      start = indptr[id];
      deg = indptr[id + 1] - start;
    }
    int32_t res = pad_id;
    uint32_t r = 0;
    if (lane < k && deg > 0) r = philox_draw(seed, ctr, (uint32_t)t, kStreamCsr, lane);
    if (deg >= k) {
      // Floyd: step j draws from [0, deg-k+j]; a repeat is replaced by deg-k+j itself
      int64_t mine = -1;
      for (int j = 0; j < k; ++j) {
        uint32_t rj = __shfl_sync(0xffffffffu, r, j);
        int64_t m = deg - k + j;
        int64_t tpos = (int64_t)mulhi32(rj, (uint32_t)(m + 1));
        unsigned dup = __ballot_sync(0xffffffffu, lane < j && mine == tpos);
        if (lane == j) mine = dup ? m : tpos;
      }
      if (lane < k) res = indices[start + mine];
    } else if (deg > 0) {
      if (replace_if_short) {
        if (lane < k) res = indices[start + (int64_t)mulhi32(r, (uint32_t)deg)];
      } else {
        if (lane < deg) res = indices[start + lane];
      }
    }
    if (lane < k) out[t * k + lane] = res;
  }
}

// negatives proportional to deg^0.75 (reference models.py:336-343): inverse-CDF lookup, one thread per draw
__global__ void __launch_bounds__(128) sample_unigram_kernel(const double* __restrict__ cdf, int64_t n, int32_t num,
                                                             uint64_t seed, uint64_t counter,
                                                             const uint64_t* __restrict__ counter_dev,
                                                             int32_t* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= num) return;
  const uint64_t ctr = counter + (counter_dev ? *counter_dev : 0ull);
  const uint32_t r = philox_draw(seed, ctr, 0u, kStreamUnigram, j);
  const double u = ((double)r + 0.5) * (1.0 / 4294967296.0) * cdf[n - 1];
  int64_t lo = 0, hi = n - 1;                       // first index with cdf[index] > u
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (cdf[mid] > u) hi = mid; else lo = mid + 1;
  }
  out[j] = (int32_t)lo;
}

// the u -> id rule of sample_unigram_kernel: first index whose inclusive prefix sum exceeds u
__device__ __forceinline__ int32_t unigram_lookup(const double* __restrict__ cdf, int64_t n, uint32_t r) {
  const double u = ((double)r + 0.5) * (1.0 / 4294967296.0) * cdf[n - 1];
  int64_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (cdf[mid] > u) hi = mid; else lo = mid + 1;
  }
  return (int32_t)lo;
}

// unique=True: ONE warp.  Round t draws candidates 32t .. 32t+31 (lane l owns draw 32t + l); a lane is accepted iff its id
// is not in the accepted set and no lower lane of the round holds the same id (__match_any_sync); a ballot prefix keeps
// draw order and the round is cut at num.  That is exactly "draw in sequence, reject ids already held".  The set is a
// linear list in shared memory (num <= kMaxUniqueSampled), scanned by every lane with broadcast reads.
__global__ void __launch_bounds__(32) sample_unigram_unique_kernel(const double* __restrict__ cdf, int64_t n, int32_t num,
                                                                   int64_t max_draws, uint64_t seed, uint64_t counter,
                                                                   const uint64_t* __restrict__ counter_dev,
                                                                   int32_t* __restrict__ out, int32_t* __restrict__ status) {
  __shared__ int32_t held[GS_MAX_UNIQUE_SAMPLED];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x;
  const unsigned lower = (1u << lane) - 1u;
  const uint64_t ctr = counter + (counter_dev ? *counter_dev : 0ull);
  int count = 0;
  int64_t j0 = 0;
  for (; count < num && j0 < max_draws; j0 += 32) {
    const int64_t j = j0 + lane;
    const bool live = j < max_draws;
      const int32_t id = live ? unigram_lookup(cdf, n, philox_draw(seed, ctr, 0u, kStreamUnigramUnique, (int)j)) : -1 - lane;
    bool fresh = live;
    for (int q = 0; q < count; ++q) fresh &= held[q] != id;
    const unsigned same = __match_any_sync(FULL, id);
    fresh &= (same & lower) == 0u;
    const unsigned acc = __ballot_sync(FULL, fresh);
    const int pos = count + __popc(acc & lower);
    if (fresh && pos < num) {
      held[pos] = id;
      out[pos] = id;
    }
    count = min(num, count + __popc(acc));
    __syncwarp();
  }
  // draw budget exhausted: the unfilled positions get -1 and the (sticky) status word says so
  for (int p = count + lane; p < num; p += 32) out[p] = -1;
  if (lane == 0 && status != nullptr && count < num) *status = 1;
}

// padded adjacency from CSR, one warp per node (start-up time, not per batch)
__global__ void __launch_bounds__(256) build_padded_adj_kernel(const int64_t* __restrict__ indptr,
                                                               const int32_t* __restrict__ indices, int64_t n_nodes,
                                                               int32_t max_deg, const uint8_t* __restrict__ skip,
                                                               uint64_t seed, uint64_t counter, int32_t* __restrict__ adj,
                                                               float* __restrict__ deg_out) {
  __shared__ int32_t sel[8][kMaxDegSmem];            // Floyd's selected positions, one row per warp
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t warp = (int64_t)blockIdx.x * 8 + w;
  const int64_t nwarps = (int64_t)gridDim.x * 8;
  for (int64_t u = warp; u <= n_nodes; u += nwarps) {
    int32_t* row = adj + u * max_deg;
    int64_t start = 0, deg = 0;
    if (u < n_nodes && !(skip && skip[u])) {
      start = indptr[u];
      deg = indptr[u + 1] - start;
    }
    if (u < n_nodes && deg_out && lane == 0) deg_out[u] = (float)deg;
    if (deg == 0) {
      for (int j = lane; j < max_deg; j += 32) row[j] = (int32_t)n_nodes;
    } else if (deg == max_deg) {
      for (int j = lane; j < max_deg; j += 32) row[j] = indices[start + j];
    } else if (deg < max_deg) {
      for (int j = lane; j < max_deg; j += 32) {
        const uint32_t r = philox_draw(seed, counter, (uint32_t)u, kStreamBuild, j);
        row[j] = indices[start + (int64_t)mulhi32(r, (uint32_t)deg)];
      }
    } else {
      // Floyd: step j draws t in [0, deg - max_deg + j]; a repeat is replaced by the upper bound itself
      for (int j = 0; j < max_deg; ++j) {
        const int64_t m = deg - max_deg + j;
        const uint32_t r = philox_draw(seed, counter, (uint32_t)u, kStreamBuild, j);   // same value in every lane
        const int32_t t = (int32_t)mulhi32(r, (uint32_t)(m + 1));
        bool dup = false;
        for (int q = lane; q < j; q += 32) dup |= (sel[w][q] == t);
        dup = __any_sync(0xffffffffu, dup);
        if (lane == 0) sel[w][j] = dup ? (int32_t)m : t;
        __syncwarp();
      }
      for (int j = lane; j < max_deg; j += 32) row[j] = indices[start + sel[w][j]];
      __syncwarp();
    }
  }
}

}  // namespace gs

extern "C" {

int32_t gs_sample_padded(const int32_t* adj, int64_t n_rows, int32_t max_deg, const int32_t* ids, int64_t n, int32_t k,
                         const int32_t* col_perm, uint64_t seed, uint64_t counter, const uint64_t* counter_dev,
                         int32_t* out, void* stream) {
  GS_REQUIRE(n >= 0 && k >= 0, "gs_sample_padded: negative size (n=%lld, k=%d)", (long long)n, k);
  if (n == 0 || k == 0) return GS_OK;
  GS_REQUIRE(adj && ids && out, "gs_sample_padded: NULL pointer");
  GS_REQUIRE(n_rows > 0 && max_deg > 0 && max_deg <= gs::kMaxDegSmem, "gs_sample_padded: need 0 < max_deg <= %d (got %d)",
             gs::kMaxDegSmem, max_deg);
  GS_REQUIRE(k <= max_deg, "gs_sample_padded: num_samples %d > max_degree %d", k, max_deg);
  int64_t total = n * (int64_t)k;
  int64_t blocks = (total + 255) / 256;
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::sample_padded_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(adj, n_rows, max_deg, ids, n, k, col_perm,
                                                                               seed, counter, counter_dev, out);
  return gs::launch_check("sample_padded_kernel");
}

int32_t gs_sample_padded_khop(const int32_t* adj, int64_t n_rows, int32_t max_deg, const int32_t* seeds, int64_t n_seeds,
                              const int32_t* fanout_host, int32_t n_hops, uint64_t seed, uint64_t counter,
                              const uint64_t* counter_dev, int32_t* const* out_host, void* stream) {
  GS_REQUIRE(n_hops >= 1 && n_hops <= GS_MAX_HOPS, "gs_sample_padded_khop: n_hops=%d (max %d)", n_hops, GS_MAX_HOPS);
  GS_REQUIRE(fanout_host && out_host, "gs_sample_padded_khop: NULL host array");
  GS_REQUIRE(n_seeds >= 0, "gs_sample_padded_khop: n_seeds < 0");
  if (n_seeds == 0) return GS_OK;
  GS_REQUIRE(adj && seeds, "gs_sample_padded_khop: NULL pointer");
  GS_REQUIRE(n_rows > 0 && max_deg > 0 && max_deg <= gs::kMaxDegSmem, "gs_sample_padded_khop: need 0 < max_deg <= %d",
             gs::kMaxDegSmem);
  gs::KhopParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.n_hops = n_hops;
  int64_t cnt = n_seeds, total = 0;
  for (int t = 0; t < n_hops; ++t) {
    GS_REQUIRE(fanout_host[t] >= 1 && fanout_host[t] <= max_deg && fanout_host[t] <= 64,
               "gs_sample_padded_khop: fanout[%d]=%d (need 1..min(64, max_degree))", t, fanout_host[t]);
    GS_REQUIRE(out_host[t] != nullptr, "gs_sample_padded_khop: out[%d] is NULL", t);
    cnt *= fanout_host[t];
    kp.fanout[t] = fanout_host[t];
    kp.count[t] = cnt;
    kp.out[t] = out_host[t];
    total += cnt;
  }
  int64_t blocks = (total + 511) / 512;
  int64_t cap = (int64_t)gs::sm_count() * 2;             // few, fat blocks: each block rebuilds the permutations once
  if (blocks > cap) blocks = cap;
  gs::sample_padded_khop_kernel<<<(unsigned)blocks, 512, 0, (cudaStream_t)stream>>>(adj, n_rows, max_deg, seeds, kp, seed,
                                                                                    counter, counter_dev);
  return gs::launch_check("sample_padded_khop_kernel");
}

int32_t gs_build_padded_adj(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int32_t max_deg,
                            const uint8_t* skip, uint64_t seed, uint64_t counter, int32_t* adj, float* deg, void* stream) {
  GS_REQUIRE(indptr && indices && adj && n_nodes >= 0, "gs_build_padded_adj: NULL pointer / bad size");
  GS_REQUIRE(max_deg >= 1 && max_deg <= gs::kMaxDegSmem, "gs_build_padded_adj: need 1 <= max_deg <= %d", gs::kMaxDegSmem);
  int64_t blocks = (n_nodes + 1 + 7) / 8;
  int64_t cap = (int64_t)gs::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  gs::build_padded_adj_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(indptr, indices, n_nodes, max_deg, skip,
                                                                                   seed, counter, adj, deg);
  return gs::launch_check("build_padded_adj_kernel");
}

int32_t gs_sample_unigram(const double* cdf, int64_t n, int32_t num_sampled, uint64_t seed, uint64_t counter,
                          const uint64_t* counter_dev, int32_t* out, void* stream) {
  GS_REQUIRE(num_sampled >= 0 && n >= 1, "gs_sample_unigram: bad sizes");
  if (num_sampled == 0) return GS_OK;
  GS_REQUIRE(cdf && out, "gs_sample_unigram: NULL pointer");
  gs::sample_unigram_kernel<<<(num_sampled + 127) / 128, 128, 0, (cudaStream_t)stream>>>(cdf, n, num_sampled, seed, counter,
                                                                                       counter_dev, out);
  return gs::launch_check("sample_unigram_kernel");
}

int32_t gs_sample_unigram_unique(const double* cdf, int64_t n, int32_t num_sampled, uint64_t seed, uint64_t counter,
                                 const uint64_t* counter_dev, int32_t* out, int32_t* status, void* stream) {
  GS_REQUIRE(n >= 1 && n < 0x7fffffffLL, "gs_sample_unigram_unique: need 1 <= n < 2^31 - 1 (got %lld)", (long long)n);
  GS_REQUIRE(num_sampled >= 0 && num_sampled <= GS_MAX_UNIQUE_SAMPLED && num_sampled <= n,
             "gs_sample_unigram_unique: num_sampled=%d must be in [0, min(%d, n=%lld)]", num_sampled, GS_MAX_UNIQUE_SAMPLED,
             (long long)n);
  if (num_sampled == 0) return GS_OK;
  GS_REQUIRE(cdf && out, "gs_sample_unigram_unique: NULL pointer");
  gs::sample_unigram_unique_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(cdf, n, num_sampled, GS_UNIQUE_DRAW_BUDGET, seed,
                                                                      counter, counter_dev, out, status);
  return gs::launch_check("sample_unigram_unique_kernel");
}

int32_t gs_sample_csr(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, const int32_t* ids, int64_t n,
                      int32_t k, int32_t replace_if_short, uint64_t seed, uint64_t counter, const uint64_t* counter_dev,
                      int32_t pad_id, int32_t* out, void* stream) {
  GS_REQUIRE(n >= 0 && k >= 0, "gs_sample_csr: negative size");
  if (n == 0 || k == 0) return GS_OK;
  GS_REQUIRE(indptr && indices && ids && out, "gs_sample_csr: NULL pointer");
  if (k > 32) {
    gs::set_error("gs_sample_csr: k=%d > 32 not supported (one lane per draw)", k);
    return GS_ERR_UNSUPPORTED;
  }
  int64_t blocks = (n + 7) / 8;  // 8 warps per block
  int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::sample_csr_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(indptr, indices, n_nodes, ids, n, k,
                                                                            replace_if_short, seed, counter, counter_dev,
                                                                            pad_id, out);
  return gs::launch_check("sample_csr_kernel");
}

}  // extern "C"

// WeightedNeighborSampler kernels: fixed-fanout draws with replacement in proportion to edge weight, from per-row alias
// tables (contract: oracle/alias_sampling.py, bit for bit).
//   alias_build_kernel        - the table, one thread per row (set-up work, run once per graph)
//   sample_alias_kernel       - one thread per draw: indptr[v], indptr[v+1] and one 16-byte record
//   sample_alias_khop_kernel  - every hop of SampleAndAggregate.sample in one launch
// No atomics, no allocation; the two sampling kernels read counter_dev, so they can be captured in CUDA graphs.
#include "common.cuh"

namespace gs {

constexpr uint64_t kAliasCap = 1ull << 32;

// (thr, id, alias, hi): hi is 0 in a finished table; while a row is built, (hi, thr) holds the entry's 64-bit mass,
// and hi != 0 (mass >= 2^32) marks a heavy entry for the whole sweep
struct AliasRec {
  uint32_t thr;
  int32_t id, alias;
  uint32_t hi;
};

__device__ __forceinline__ bool alias_eligible(float x, bool inf_row) {
  return inf_row ? (x == INFINITY) : (isfinite(x) && x > 0.f);
}

// One thread per row: the fp64 sum in CSR order, the masses (three passes), then the two-pointer sweep.  Rows are long
// enough in a power-law graph that the longest one sets the time; this runs once per graph.
__global__ void __launch_bounds__(128) alias_build_kernel(const int64_t* __restrict__ indptr,
                                                          const int32_t* __restrict__ indices,
                                                          const float* __restrict__ w, int64_t n_nodes,
                                                          AliasRec* __restrict__ tab) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_nodes; v += stride) {
    const int64_t a = indptr[v], d = indptr[v + 1] - a;
    if (d <= 0) continue;
    const float* wr = w + a;
    AliasRec* r = tab + a;
    bool inf_row = false;
    for (int64_t p = 0; p < d && !inf_row; ++p) inf_row = wr[p] == INFINITY;
    double S = 0.0;
    int64_t ne = 0;
    for (int64_t p = 0; p < d; ++p) {
      const float x = wr[p];
      if (alias_eligible(x, inf_row)) {
        S = __dadd_rn(S, inf_row ? 1.0 : (double)x);
        ++ne;
      }
    }
    if (ne == 0) {
      for (int64_t p = 0; p < d; ++p) r[p] = AliasRec{0u, (int32_t)n_nodes, (int32_t)n_nodes, 0u};
      continue;
    }
    const int64_t R = (int64_t)(((uint64_t)d << 32) - (uint64_t)ne);
    const double Rf = __ll2double_rn(R);
    int64_t sumb = 0;
    for (int64_t p = 0; p < d; ++p) {         // b_j = min(floor(min(fl(fl(w / S) * fl(R)), fl(R))), R)
      const float x = wr[p];
      int64_t b = 0;
      if (alias_eligible(x, inf_row)) {
        const double q = fmin(__dmul_rn(__ddiv_rn(inf_row ? 1.0 : (double)x, S), Rf), Rf);
        b = min((int64_t)__double2ll_rz(q), R);
      }
      sumb += b;
      r[p] = AliasRec{(uint32_t)b, indices[a + p], 0, (uint32_t)((uint64_t)b >> 32)};
    }
    const int64_t rem = R - sumb;
    const int64_t q = rem >= 0 ? rem / ne : 0, rr = rem >= 0 ? rem % ne : 0;
    int64_t rank = 0, pre = 0;
    for (int64_t p = 0; p < d; ++p) {         // the remainder: shared round-robin, or taken greedily in CSR order
      const AliasRec e = r[p];
      const int64_t b = (int64_t)(((uint64_t)e.hi << 32) | e.thr);
      int64_t m = 0;
      if (alias_eligible(wr[p], inf_row)) {
        m = rem >= 0 ? 1 + b + q + (rank < rr ? 1 : 0) : 1 + b - min(b, max((int64_t)0, -rem - pre));
        ++rank;
      }
      pre += b;
      r[p].thr = (uint32_t)m;
      r[p].hi = (uint32_t)((uint64_t)m >> 32);
    }
    // the sweep (oracle/alias_sampling.py:sweep): writes thr and alias only, so hi keeps every entry's class
    int64_t i = 0, j = 0;
    while (i < d && r[i].hi != 0u) ++i;
    while (j < d && r[j].hi == 0u) ++j;
    uint64_t wj = j < d ? (((uint64_t)r[j].hi << 32) | r[j].thr) : 0ull;
    while (j < d) {
      if (wj > kAliasCap) {
        if (i >= d) break;                    // unreachable: the masses sum to d 2^32
        const uint32_t mi = r[i].thr;
        r[i].alias = r[j].id;
        wj -= kAliasCap - mi;
        for (++i; i < d && r[i].hi != 0u; ++i) {
        }
      } else if (wj == kAliasCap) {
        r[j].thr = 0u;
        r[j].alias = r[j].id;
        for (++j; j < d && r[j].hi == 0u; ++j) {
        }
        wj = j < d ? (((uint64_t)r[j].hi << 32) | r[j].thr) : 0ull;
      } else {
        int64_t j2 = j + 1;
        while (j2 < d && r[j2].hi == 0u) ++j2;
        if (j2 >= d) break;                   // unreachable, as above
        r[j].thr = (uint32_t)wj;
        r[j].alias = r[j2].id;
        wj = (((uint64_t)r[j2].hi << 32) | r[j2].thr) - (kAliasCap - wj);
        j = j2;
      }
    }
    for (int64_t p = 0; p < d; ++p) r[p].hi = 0u;
  }
}

// draw j of output position t from row id (oracle/alias_sampling.py:sample); the dummy n_nodes for an id outside
// [0, n_nodes) or an empty row
__device__ __forceinline__ int32_t alias_draw(const int64_t* __restrict__ indptr, const int4* __restrict__ tab,
                                              int64_t n_nodes, int64_t id, uint64_t ctr, uint32_t t, int j,
                                              uint32_t k0, uint32_t k1) {
  if (id < 0 || id >= n_nodes) return (int32_t)n_nodes;
  const int64_t a = indptr[id], d = indptr[id + 1] - a;
  if (d <= 0) return (int32_t)n_nodes;
  const u32x4 c{(uint32_t)ctr, (uint32_t)(ctr >> 32), t, kStreamAlias + (uint32_t)(j >> 1)};
  const u32x4 r = philox4x32_10(c, k0, k1);
  const uint32_t wa = (j & 1) ? r.z : r.x, wb = (j & 1) ? r.w : r.y;
  const int4 rec = __ldg(tab + a + (int64_t)mulhi32(wa, (uint32_t)d));
  return wb < (uint32_t)rec.x ? rec.y : rec.z;
}

__global__ void __launch_bounds__(256) sample_alias_kernel(const int64_t* __restrict__ indptr,
                                                           const int4* __restrict__ tab, int64_t n_nodes,
                                                           const int32_t* __restrict__ ids, int64_t n, int32_t k,
                                                           uint64_t seed, uint64_t counter,
                                                           const uint64_t* __restrict__ counter_dev,
                                                           int32_t* __restrict__ out) {
  const uint64_t ctr = counter + (counter_dev ? *counter_dev : 0ull);
  const int64_t total = n * (int64_t)k;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = e / k;
    const int j = (int)(e - t * k);
    out[e] = alias_draw(indptr, tab, n_nodes, ids[t], ctr, (uint32_t)t, j, (uint32_t)seed, (uint32_t)(seed >> 32));
  }
}

struct AliasKhopParams {
  int32_t* out[GS_MAX_HOPS];
  int32_t fanout[GS_MAX_HOPS];
  int64_t count[GS_MAX_HOPS];     // elements of hop t+1 = n_seeds * prod(fanout[0..t])
  int32_t n_hops;
};

// Each element rewalks its ancestor chain from the seed, as sample_padded_khop_kernel does: hop t of the chain is draw
// (t-th call: counter + t, position = the ancestor's index in hop t's input, j); siblings share the ancestors' reads.
__global__ void __launch_bounds__(256) sample_alias_khop_kernel(const int64_t* __restrict__ indptr,
                                                                const int4* __restrict__ tab, int64_t n_nodes,
                                                                const int32_t* __restrict__ seeds,
                                                                const __grid_constant__ AliasKhopParams kp, uint64_t seed,
                                                                uint64_t counter,
                                                                const uint64_t* __restrict__ counter_dev) {
  const uint64_t ctr = counter + (counter_dev ? *counter_dev : 0ull);
  int64_t total = 0;
  for (int t = 0; t < kp.n_hops; ++t) total += kp.count[t];
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int hop = 0;
    int64_t local = e;
    while (local >= kp.count[hop]) { local -= kp.count[hop]; ++hop; }
    int64_t sup = 1;
    for (int t = 0; t <= hop; ++t) sup *= kp.fanout[t];
    int64_t pos = local / sup;
    int64_t rem = local - pos * sup;
    int64_t id = seeds[pos];
    for (int t = 0; t <= hop; ++t) {
      sup /= kp.fanout[t];
      const int j = (int)(rem / sup);
      rem -= (int64_t)j * sup;
      id = alias_draw(indptr, tab, n_nodes, id, ctr + (uint64_t)t, (uint32_t)pos, j, (uint32_t)seed,
                      (uint32_t)(seed >> 32));
      pos = pos * kp.fanout[t] + j;
    }
    kp.out[hop][local] = (int32_t)id;
  }
}

}  // namespace gs

extern "C" {

int32_t gs_csr_alias_build(const int64_t* indptr, const int32_t* indices, const float* weights, int64_t n_nodes,
                           int64_t n_entries, int32_t* table, void* stream) {
  GS_REQUIRE(n_nodes >= 0 && n_entries >= 0, "gs_csr_alias_build: negative size");
  GS_REQUIRE(n_nodes < 0x7fffffffLL, "gs_csr_alias_build: n_nodes=%lld must be < 2^31 - 1", (long long)n_nodes);
  if (n_nodes == 0 || n_entries == 0) return GS_OK;
  GS_REQUIRE(indptr && indices && weights && table, "gs_csr_alias_build: NULL pointer");
  if (n_entries >= (1LL << 31)) {
    // only a table this large can hold a row of 2^31 entries; d 2^32 must fit in 63 bits (set-up work: read indptr once)
    int64_t* h = (int64_t*)malloc((size_t)(n_nodes + 1) * sizeof(int64_t));
    GS_REQUIRE(h != nullptr, "gs_csr_alias_build: host allocation failed");
    cudaError_t e = cudaMemcpyAsync(h, indptr, (size_t)(n_nodes + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost,
                                    (cudaStream_t)stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) {
      free(h);
      return gs::cuda_fail(e, "gs_csr_alias_build: indptr read");
    }
    int64_t worst = -1, deg = 0;
    for (int64_t v = 0; v < n_nodes; ++v)
      if (h[v + 1] - h[v] >= (1LL << 31)) { worst = v; deg = h[v + 1] - h[v]; break; }
    free(h);
    if (worst >= 0) {
      gs::set_error("gs_csr_alias_build: row %lld has %lld entries (rows of 2^31 entries or more are not supported)",
                    (long long)worst, (long long)deg);
      return GS_ERR_UNSUPPORTED;
    }
  }
  int64_t blocks = (n_nodes + 127) / 128;
  const int64_t cap = (int64_t)gs::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  gs::alias_build_kernel<<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>(indptr, indices, weights, n_nodes,
                                                                              (gs::AliasRec*)table);
  return gs::launch_check("alias_build_kernel");
}

int32_t gs_sample_alias(const int64_t* indptr, const int32_t* table, int64_t n_nodes, const int32_t* ids, int64_t n,
                        int32_t k, uint64_t seed, uint64_t counter, const uint64_t* counter_dev, int32_t* out,
                        void* stream) {
  GS_REQUIRE(n >= 0 && k >= 0 && n_nodes >= 0, "gs_sample_alias: negative size (n=%lld, k=%d)", (long long)n, k);
  GS_REQUIRE(k <= GS_MAX_ALIAS_FANOUT, "gs_sample_alias: k=%d > %d", k, GS_MAX_ALIAS_FANOUT);
  if (n == 0 || k == 0) return GS_OK;
  GS_REQUIRE(indptr && ids && out, "gs_sample_alias: NULL pointer");
  const int64_t total = n * (int64_t)k;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::sample_alias_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      indptr, (const int4*)table, n_nodes, ids, n, k, seed, counter, counter_dev, out);
  return gs::launch_check("sample_alias_kernel");
}

int32_t gs_sample_alias_khop(const int64_t* indptr, const int32_t* table, int64_t n_nodes, const int32_t* seeds,
                             int64_t n_seeds, const int32_t* fanout_host, int32_t n_hops, uint64_t seed,
                             uint64_t counter, const uint64_t* counter_dev, int32_t* const* out_host, void* stream) {
  GS_REQUIRE(n_hops >= 1 && n_hops <= GS_MAX_HOPS, "gs_sample_alias_khop: n_hops=%d (max %d)", n_hops, GS_MAX_HOPS);
  GS_REQUIRE(fanout_host && out_host, "gs_sample_alias_khop: NULL host array");
  GS_REQUIRE(n_seeds >= 0 && n_nodes >= 0, "gs_sample_alias_khop: negative size");
  gs::AliasKhopParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.n_hops = n_hops;
  int64_t cnt = n_seeds, total = 0;
  for (int t = 0; t < n_hops; ++t) {
    GS_REQUIRE(fanout_host[t] >= 1 && fanout_host[t] <= 64, "gs_sample_alias_khop: fanout[%d]=%d (need 1..64)", t,
               fanout_host[t]);
    cnt *= fanout_host[t];
    kp.fanout[t] = fanout_host[t];
    kp.count[t] = cnt;
    kp.out[t] = out_host[t];
    total += cnt;
  }
  if (n_seeds == 0) return GS_OK;
  GS_REQUIRE(indptr && seeds, "gs_sample_alias_khop: NULL pointer");
  for (int t = 0; t < n_hops; ++t) GS_REQUIRE(out_host[t] != nullptr, "gs_sample_alias_khop: out[%d] is NULL", t);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::sample_alias_khop_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(indptr, (const int4*)table, n_nodes,
                                                                                   seeds, kp, seed, counter, counter_dev);
  return gs::launch_check("sample_alias_khop_kernel");
}

}  // extern "C"

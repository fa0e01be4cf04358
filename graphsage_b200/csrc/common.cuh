// Shared host/device helpers for libgraphsage_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/graphsage_b200.h"

namespace gs {

// ---- thread-local error string -------------------------------------------------------------
void set_error(const char* fmt, ...);
int32_t cuda_fail(cudaError_t e, const char* what);
int32_t tuning(const char* key, int32_t dflt);
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (current device, kernel); GS_OK or GS_ERR_CUDA
int32_t ensure_dyn_smem(const void* kernel, int bytes);

#define GS_REQUIRE(cond, ...)            \
  do {                                   \
    if (!(cond)) {                       \
      gs::set_error(__VA_ARGS__);        \
      return GS_ERR_INVALID_ARG;         \
    }                                    \
  } while (0)

#define GS_CUDA(expr)                                        \
  do {                                                       \
    cudaError_t _e = (expr);                                 \
    if (_e != cudaSuccess) return gs::cuda_fail(_e, #expr);  \
  } while (0)

inline int32_t launch_check(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, what);
  return GS_OK;
}

int sm_count();

// workspace carving: every region starts on a 256-byte boundary
inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

inline int32_t check_site(const gs_dropout_site& s, const char* who) {
  GS_REQUIRE(s.rate >= 0.f && s.rate < 1.f, "%s: dropout rate %g outside [0, 1)", who, (double)s.rate);
  return GS_OK;
}

// ---- Philox4x32-10 (contract: oracle/philox.py) --------------------------------------------
struct u32x4 { uint32_t x, y, z, w; };

__host__ __device__ inline uint32_t mulhi32(uint32_t a, uint32_t b) {
  return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
}

__host__ __device__ inline u32x4 philox4x32_10(u32x4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c.x;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c.z;
    u32x4 n;
    n.x = (uint32_t)(p1 >> 32) ^ c.y ^ k0;
    n.y = (uint32_t)p1;
    n.z = (uint32_t)(p0 >> 32) ^ c.w ^ k1;
    n.w = (uint32_t)p0;
    c = n;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

__host__ __device__ inline uint32_t pick(const u32x4& v, int i) {
  return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w;
}

// draw number i of stream position (c2, tag) - oracle/sampler.py:_draws
__host__ __device__ inline uint32_t philox_draw(uint64_t seed, uint64_t counter, uint32_t c2, uint32_t tag, int i) {
  u32x4 c{(uint32_t)counter, (uint32_t)(counter >> 32), c2, tag + (uint32_t)(i >> 2)};
  u32x4 r = philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  return pick(r, i & 3);
}

// ---- dropout masks (contract: oracle/dropout.py) --------------------------------------------
// A site (seed, call, rate) drops element (pos, c) of a logical [rows, F] tensor unless word c % 4 of
// philox4x32_10(ctr = (c / 4, pos_lo32, pos_hi32, call), key = split64(seed)) is >= T = floor(rate * 2^32) (float64).
// A kept element becomes x / keep with keep = fp32(1 - rate) (IEEE division), a dropped one 0.  rate = 0 keeps every
// element and divides by 1, so it is the identity.
// call_dev (optional, device) is added to call by the kernel: see drop_call_offset.
struct DropSite {
  uint32_t k0, k1, call, threshold;
  float keep;
  const uint64_t* call_dev;
};

__host__ inline DropSite make_drop_site(const gs_dropout_site& s) {
  DropSite d;
  d.k0 = (uint32_t)s.seed;
  d.k1 = (uint32_t)(s.seed >> 32);
  d.call = s.call;
  d.threshold = (uint32_t)floor((double)s.rate * 4294967296.0);
  d.keep = (float)(1.0 - (double)s.rate);
  d.call_dev = s.call_dev;
  return d;
}

#ifdef __CUDACC__
// what the device word adds to a site's call number (0 without one); a kernel reads it once, not per element
__device__ __forceinline__ uint32_t drop_call_offset(const DropSite& s) {
  return s.call_dev ? (uint32_t)*s.call_dev : 0u;
}
#endif

__host__ __device__ inline DropSite with_call_offset(DropSite s, uint32_t off) {
  s.call += off;
  return s;
}

// the four keep words of columns 4 * c4 .. 4 * c4 + 3 at position pos
__host__ __device__ inline u32x4 drop_words(const DropSite& s, int64_t pos, uint32_t c4) {
  u32x4 c{c4, (uint32_t)pos, (uint32_t)((uint64_t)pos >> 32), s.call};
  return philox4x32_10(c, s.k0, s.k1);
}

__host__ __device__ inline float drop_one(const DropSite& s, uint32_t word, float x) {
  return word >= s.threshold ? x / s.keep : 0.f;
}

__host__ __device__ inline float4 drop4(const DropSite& s, int64_t pos, uint32_t c4, float4 v) {
  const u32x4 w = drop_words(s, pos, c4);
  return make_float4(drop_one(s, w.x, v.x), drop_one(s, w.y, v.y), drop_one(s, w.z, v.z), drop_one(s, w.w, v.w));
}

__host__ __device__ inline float drop_col(const DropSite& s, int64_t pos, int c, float x) {
  return drop_one(s, pick(drop_words(s, pos, (uint32_t)c >> 2), c & 3), x);
}

constexpr uint32_t kStreamPadded = 0u;
constexpr uint32_t kStreamCsr = 0x40000000u;
constexpr uint32_t kStreamUnigram = 0x20000000u;
constexpr uint32_t kStreamBuild = 0x10000000u;
constexpr uint32_t kStreamUnigramUnique = 0x30000000u;
constexpr uint32_t kStreamWalk = 0x50000000u;
constexpr uint32_t kStreamWalkBiased = 0x60000000u;  // 2^28 words: ((w * 32 + move) << 3) + call
constexpr uint32_t kStreamSampledBlocks = 0x70000000u;  // GS_MAX_BLOCK_LAYERS words: | layer (counter (i, v, call, .))
// weighted blocks: [0x80000000, 0x80000008), | layer (counter (j >> 1, v, call, .)); past every range above
constexpr uint32_t kStreamWeightedBlocks = 0x80000000u;
// alias draws: [0x90000000, 0x90000000 + GS_MAX_ALIAS_FANOUT / 2), + (j >> 1) (counter (c_lo, c_hi, t, .))
constexpr uint32_t kStreamAlias = 0x90000000u;

// ---- PTX wrappers (mbarrier / bulk copy) ---------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// 1-D bulk async copy global -> shared::cta, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// 1-D bulk async copy shared::cta -> global (bulk-group completion)
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ float4 ldg_nc_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// the A row that operand row r of a GEMM part reads (gs_sage_gemm_rows): r itself for a dense part, else the clamped id
// its range holds; -1 = a zero row (r >= M, or no range covers r)
__device__ __forceinline__ int64_t gemm_a_row(const gs_gemm_row_ids& R, int64_t M, int64_t r) {
  if (r >= M) return -1;
  if (R.n_ranges == 0) return r;
#pragma unroll
  for (int s = 0; s < GS_MAX_SEGMENTS; ++s) {
    const gs_row_range& g = R.ranges[s];
    if (s < R.n_ranges && r >= g.row0 && r - g.row0 < g.n) {
      const int64_t id = g.ids[r - g.row0];
      return (id < 0 || id >= R.n_table_rows) ? R.n_table_rows - 1 : id;
    }
  }
  return -1;
}
#endif  // __CUDACC__

}  // namespace gs

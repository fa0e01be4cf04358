// Feature table in host memory (graphsage_b200.HostFeatures): registration of the page-locked rows and the fetch pass
// that copies a step's staged rows over the host link into the device working set.  Claim and translate are the halo
// passes of gather.cu (gs_halo_claim, gs_host_translate) with the working set described as a one-shard table.
#include "common.cuh"

namespace gs {

// Every thread walks the flat list of 16-byte units of the staged rows (unit u = row u / row_v, column u % row_v) and
// keeps kHostLoads loads in flight before it stores them: the loads of one warp touch kHostLoads rows a grid stride
// apart (and neighbouring lanes the neighbouring units of a row), so a warp has kHostLoads x 512 bytes outstanding
// however narrow the rows are.  A zero-copy read takes about a microsecond, so that depth, not the issue rate, is what
// fills the link.  Plain 16-byte loads: the bulk-copy engine is not used on the host mapping.
constexpr int kHostLoads = 8;

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

__global__ void __launch_bounds__(256) host_fetch_kernel(const uint4* __restrict__ host, int64_t row_v,
                                                         const int32_t* __restrict__ stage_ids,
                                                         const int32_t* __restrict__ count, int64_t capacity,
                                                         uint4* __restrict__ staging) {
  int64_t n = *count;
  if (n > capacity) n = capacity;
  const int64_t total = n * row_v;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u0 < total; u0 += stride * kHostLoads) {
    uint4 v[kHostLoads];
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const int64_t u = u0 + k * stride;
      if (u < total) {
        const int64_t i = u / row_v;
        v[k] = host[(int64_t)__ldg(stage_ids + i) * row_v + (u - i * row_v)];
      }
    }
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const int64_t u = u0 + k * stride;
      if (u < total) staging[u] = v[k];       // staging rows are packed at the same pitch: unit u is unit u
    }
  }
}

}  // namespace gs

extern "C" {

int32_t gs_host_register(void* host_ptr, int64_t bytes, void** dev_alias_out) {
  GS_REQUIRE(host_ptr && bytes > 0 && dev_alias_out, "gs_host_register: bad arguments");
  GS_CUDA(cudaHostRegister(host_ptr, (size_t)bytes, cudaHostRegisterMapped | cudaHostRegisterPortable));
  void* alias = nullptr;
  cudaError_t e = cudaHostGetDevicePointer(&alias, host_ptr, 0);
  if (e != cudaSuccess) {
    cudaHostUnregister(host_ptr);
    GS_CUDA(e);
  }
  GS_REQUIRE(gs::aligned16(alias), "gs_host_register: the device alias is not 16-byte aligned");
  *dev_alias_out = alias;
  return GS_OK;
}

int32_t gs_host_unregister(void* host_ptr) {
  if (host_ptr) GS_CUDA(cudaHostUnregister(host_ptr));
  return GS_OK;
}

int32_t gs_host_fetch(const void* host_alias, int64_t row_bytes, const int32_t* stage_ids, const int32_t* count,
                      int64_t capacity, void* staging, void* stream) {
  GS_REQUIRE(capacity >= 0, "gs_host_fetch: capacity < 0");
  if (capacity == 0) return GS_OK;
  GS_REQUIRE(host_alias && stage_ids && count && staging, "gs_host_fetch: NULL pointer");
  GS_REQUIRE(row_bytes > 0 && row_bytes % 16 == 0 && gs::aligned16(host_alias) && gs::aligned16(staging),
             "gs_host_fetch: rows must be 16-byte multiples at 16-byte aligned addresses (row_bytes=%lld)",
             (long long)row_bytes);
  const int blocks = gs::sm_count() * 3;       // 76 registers (ptxas, sm_90a): three 256-thread CTAs fit an SM
  gs::host_fetch_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)host_alias, row_bytes / 16, stage_ids, count, capacity, (uint4*)staging);
  return gs::launch_check("host_fetch_kernel");
}

}  // extern "C"

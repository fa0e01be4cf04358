// Feature table in host memory (graphsage_b200.HostFeatures): registration of the page-locked rows and the fetch pass
// that copies a step's staged rows over the host link into the device working set.  Claim and translate are the halo
// passes of gather.cu (gs_halo_claim, gs_host_translate) with the working set described as a one-shard table.  The
// sampled blocks' layer 0 reads its rows in one pass instead (gs_host_gather_rows_f32): from the cache or over the link,
// straight into fp32 rows.
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

// out[i, 0:out_pitch) = the fp32 row of ids[i], read from the cache (cache_slot[id] >= 0) or over the host link, pad
// columns (>= F) zeroed.  Same flat walk as host_fetch_kernel, over the 16-byte units of the OUTPUT's rows: unit c of a row
// holds source columns [c * W, c * W + W) (W = 4 fp32, 8 bf16 or 16 int8 values), so a thread still has kHostLoads loads in
// flight, a warp kHostLoads x 512 source bytes.  A unit wholly past F, and every unit of an id outside [0, N), reads
// nothing.  The fp32 and bf16 rows, and int8 rows too wide for host_gather_i8row_kernel: there an int8 unit also needs
// its row's scale (at byte P4), which each such thread loads beside its unit, in the same batch as the units.
template <int W>
__global__ void __launch_bounds__(256) host_gather_f32_kernel(const uint8_t* __restrict__ host,
                                                              const uint8_t* __restrict__ cache,
                                                              const int32_t* __restrict__ cache_slot, int64_t n_nodes,
                                                              int F, int64_t pitch_bytes, const int32_t* __restrict__ ids,
                                                              int64_t n, float* __restrict__ out, int64_t out_pitch) {
  const int64_t row_u = (out_pitch + W - 1) / W;       // output units per row
  const int64_t total = n * row_u;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int p4 = (F + 3) & ~3;
  for (int64_t u0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u0 < total; u0 += stride * kHostLoads) {
    // three batches - ids, cache slots, then the rows - so the two dependent device reads are paid once per batch, not
    // once per row, before the link reads go out
    int64_t id[kHostLoads];
    int32_t slot[kHostLoads];
    int col[kHostLoads];                       // each unit's place in its row, so no division sits between the row loads
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const int64_t u = u0 + k * stride;
      id[k] = -1;
      col[k] = 0;
      if (u < total) {
        const int64_t i = u / row_u;
        col[k] = (int)(u - i * row_u);
        if (col[k] * W < F) id[k] = __ldg(ids + i);
      }
    }
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) slot[k] = (id[k] >= 0 && id[k] < n_nodes) ? __ldg(cache_slot + id[k]) : -2;
    uint4 v[kHostLoads];
    float s[kHostLoads];
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      v[k] = make_uint4(0u, 0u, 0u, 0u);
      s[k] = 0.f;
      if (slot[k] != -2) {                     // -2: past F or an id outside [0, N) - the zero row, nothing read
        const uint8_t* row = slot[k] >= 0 ? cache + (int64_t)slot[k] * pitch_bytes : host + id[k] * pitch_bytes;
        v[k] = *reinterpret_cast<const uint4*>(row + (int64_t)col[k] * 16);
        if (W == 16) s[k] = *reinterpret_cast<const float*>(row + p4);
      }
    }
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const int64_t u = u0 + k * stride;
      if (u >= total) continue;
      const int64_t i = u / row_u;
      const int c = (int)(u - i * row_u);
      const uint32_t w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
      float f[W];
#pragma unroll
      for (int e = 0; e < W; ++e) {
        float x;
        if (W == 4) x = __uint_as_float(w[e]);
        else if (W == 8) x = __uint_as_float((e & 1) ? (w[e >> 1] & 0xffff0000u) : (w[e >> 1] << 16));
        else x = __fmul_rn((float)(int8_t)(w[e >> 2] >> (8 * (e & 3))), s[k]);
        f[e] = (c * W + e < F) ? x : 0.f;
      }
      float4* o = reinterpret_cast<float4*>(out + i * out_pitch + (int64_t)c * W);
#pragma unroll
      for (int q = 0; q < W / 4; ++q)
        if (c * W + 4 * q < out_pitch) o[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
    }
  }
}

// GS_I8ROW rows read the way whole-row copies read them, so the scale costs no request of its own.  One warp reads
// whole rows: the units [0, U) of a row, U = P4 / 16 + 1 (the data's and the scale's, = gs_i8row_pitch(F) / 16), take
// S = ceil(U / 32) of a thread's kHostLoads slots - unit c in slot c / 32 of lane c % 32 - and a warp reads R =
// kHostLoads / S rows per batch, all loads in flight before any is used.  The scale arrives inside unit P4 / 16 and
// reaches the row's other lanes by a shuffle.  For F <= kI8RowMaxF (S <= kHostLoads); wider rows take the flat walk.
constexpr int kI8RowMaxF = kHostLoads * 32 * 16 - 4;

__global__ void __launch_bounds__(256, 3) host_gather_i8row_kernel(const uint8_t* __restrict__ host,
                                                                const uint8_t* __restrict__ cache,
                                                                const int32_t* __restrict__ cache_slot, int64_t n_nodes,
                                                                int F, int64_t pitch_bytes,
                                                                const int32_t* __restrict__ ids, int64_t n,
                                                                float* __restrict__ out, int64_t out_pitch) {
  const int p4 = (F + 3) & ~3;
  const int cs = p4 >> 4;                    // the unit holding the scale, word (p4 & 15) / 4 of it
  const int units = cs + 1;
  const int S = (units + 31) >> 5;           // slots per row
  const int R = kHostLoads / S;              // rows per warp and batch
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r0 = warp * R; r0 < n; r0 += nwarps * R) {      // warp-uniform: every lane takes part in the shuffles
    int64_t id[kHostLoads];
    int32_t slot[kHostLoads];
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const int j = k / S;
      id[k] = (j < R && r0 + j < n) ? (int64_t)__ldg(ids + r0 + j) : -1;
    }
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) slot[k] = (id[k] >= 0 && id[k] < n_nodes) ? __ldg(cache_slot + id[k]) : -2;
    uint4 v[kHostLoads];
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const int c = (k - (k / S) * S) * 32 + lane;
      v[k] = make_uint4(0u, 0u, 0u, 0u);
      if (slot[k] != -2 && c < units) {      // -2: no row in this slot, or an id outside [0, N) - the zero row
        const uint8_t* row = slot[k] >= 0 ? cache + (int64_t)slot[k] * pitch_bytes : host + id[k] * pitch_bytes;
        v[k] = *reinterpret_cast<const uint4*>(row + (int64_t)c * 16);
      }
    }
    // every slot's word of the scale from the lane that holds unit cs; row j's scale is slot j * S + cs / 32's
    const int sw = (p4 & 15) >> 2;
    float sc[kHostLoads];
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const uint32_t w = sw == 0 ? v[k].x : sw == 1 ? v[k].y : sw == 2 ? v[k].z : v[k].w;
      sc[k] = __uint_as_float(__shfl_sync(0xffffffffu, w, cs & 31));
    }
#pragma unroll
    for (int k = 0; k < kHostLoads; ++k) {
      const int j = k / S;
      const int c = (k - j * S) * 32 + lane;
      if (j >= R || r0 + j >= n || c >= units) continue;
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < kHostLoads; ++q)
        if (q == j * S + (cs >> 5)) s = sc[q];
      const uint32_t w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
      float f[16];
#pragma unroll
      for (int e = 0; e < 16; ++e)
        f[e] = (c * 16 + e < F) ? __fmul_rn((float)(int8_t)(w[e >> 2] >> (8 * (e & 3))), s) : 0.f;
      float4* o = reinterpret_cast<float4*>(out + (r0 + j) * out_pitch + (int64_t)c * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (c * 16 + 4 * q < out_pitch) o[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
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

int32_t gs_host_gather_rows_f32(const void* host_alias, const void* cache, const int32_t* cache_slot, int32_t dtype,
                                int64_t n_nodes, int32_t F, int64_t pitch, const int32_t* ids, int64_t n, float* out,
                                int64_t out_pitch, void* stream) {
  GS_REQUIRE(n >= 0 && F >= 1 && n_nodes >= 0, "gs_host_gather_rows_f32: bad sizes (n=%lld F=%d)", (long long)n, F);
  if (n == 0) return GS_OK;
  GS_REQUIRE(host_alias && cache && cache_slot && ids && out, "gs_host_gather_rows_f32: NULL pointer");
  GS_REQUIRE(dtype == GS_F32 || dtype == GS_BF16 || dtype == GS_I8ROW, "gs_host_gather_rows_f32: dtype %d", dtype);
  const int W = dtype == GS_F32 ? 4 : dtype == GS_BF16 ? 8 : 16;          // values per 16-byte unit
  const int64_t pitch_bytes = dtype == GS_F32 ? pitch * 4 : dtype == GS_BF16 ? pitch * 2 : pitch;
  GS_REQUIRE(pitch_bytes % 16 == 0 && gs::aligned16(host_alias) && gs::aligned16(cache) &&
                 pitch_bytes >= (dtype == GS_I8ROW ? gs_i8row_pitch(F) : ((int64_t)F + W - 1) / W * 16),
             "gs_host_gather_rows_f32: rows must be 16-byte multiples at 16-byte aligned addresses, wide enough for F=%d "
             "(pitch=%lld)", F, (long long)pitch);
  GS_REQUIRE(out_pitch >= F && out_pitch % 4 == 0 && gs::aligned16(out) &&
                 (dtype != GS_I8ROW || out_pitch <= gs_i8row_pitch(F)),
             "gs_host_gather_rows_f32: out must be 16-byte aligned with out_pitch >= F, out_pitch %% 4 == 0 and, for "
             "int8 rows, out_pitch <= gs_i8row_pitch(F)");
  const int blocks = gs::sm_count() * 3;       // as host_fetch: three 256-thread CTAs per SM
  const uint8_t* h = (const uint8_t*)host_alias;
  const uint8_t* c = (const uint8_t*)cache;
  if (W == 4)
    gs::host_gather_f32_kernel<4><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(h, c, cache_slot, n_nodes, F,
                                                                                      pitch_bytes, ids, n, out, out_pitch);
  else if (W == 8)
    gs::host_gather_f32_kernel<8><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(h, c, cache_slot, n_nodes, F,
                                                                                      pitch_bytes, ids, n, out, out_pitch);
  else if (F <= gs::kI8RowMaxF) {
    gs::host_gather_i8row_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(h, c, cache_slot, n_nodes, F,
                                                                                   pitch_bytes, ids, n, out, out_pitch);
    return gs::launch_check("host_gather_i8row_kernel");
  } else
    gs::host_gather_f32_kernel<16><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(h, c, cache_slot, n_nodes, F,
                                                                                       pitch_bytes, ids, n, out, out_pitch);
  return gs::launch_check("host_gather_f32_kernel");
}

}  // extern "C"

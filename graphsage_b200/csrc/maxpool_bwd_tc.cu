// B2 / B3: the weight- and input-gradient GEMMs of the pooling branch's backward, on the dP^T tile images that B1
// (maxpool_mlp_kernel<..., kGrad>, maxpool_tc.cu) writes.  Notation for one hop: X = the n*k gathered bf16 rows [R, K],
// dP = dpre rounded to bf16 [R, hidden], Wm [K, hidden].
//
//   B2: dWm += X^T dP   (reduction over the gathered rows; X is re-gathered straight into shared memory, never HBM)
//   B3: dX   = dP Wm^T  (only the first Kd columns; fp32 out)
//
// Both are one kernel shape: a CTA owns a 128 x 128 fp32 output tile in two warpgroups (m64n128 each), and loops over a
// reduction in steps of 64 with a 3-stage cp.async ring of 32 KB stages:
//   [A of warpgroup 0: 8 KB][A of warpgroup 1: 8 KB][B: 16 KB].
// The A pieces are MN-major (wgmma transpose-A): 64 M values per 128-byte row, one row per reduction index, SW128.
//   B2: A = X^T: row r of the piece = gathered row r's 64 features of one K-block (byte-for-byte K4's rows image);
//       B = the dP^T image of (tile, slice, row half): 128 hidden units x 64 rows, K-major.
//   B3: A = dP^T: row n of the piece = hidden unit n's 64 rows of one half tile (half of a B1 image);
//       B = Wm image: 128 input columns x 64 hidden units, K-major (gs_pool_mlp_dx_pack).
// Row space: B1 tiles are 128 row slots; slot r of tile t is gathered row t*G*k + r when r < G*k (G = 128 / k groups),
// and padding otherwise (dP = 0 there, X zero-filled).
//
// Determinism: no atomics.  B2 splits the row blocks (64 slots) into at most PB_MAX_CHUNKS chunks of equal length (the
// last one shorter) of at least PB_MIN_RB_PER_CHUNK blocks, so their number is fixed by the shape; each chunk writes its
// own fp32 partial tile, and pool_chunk_sum_kernel adds the partials in chunk order, then adds the sum into the caller's
// dWm.  dbm: B1's per-tile partials are summed in tile order in groups
// of PB_DBM_GROUP tiles, then the group sums in order, then added into the caller's dbm.
#include "tc_common.cuh"

namespace gs {

constexpr int PB_THREADS = 256;
constexpr int PB_HALF = 64 * 128;               // one 64-row MN-major piece
constexpr int PB_IMG = 128 * 128;               // one 128 x 128 B image
constexpr int PB_STAGE = 2 * PB_HALF + PB_IMG;  // 32 KB
constexpr int PB_STAGES = 3;
constexpr int PB_SMEM = PB_STAGES * PB_STAGE + 1024;
constexpr int PB_MAX_CHUNKS = 32;
constexpr int PB_MIN_RB_PER_CHUNK = 8;          // 512 row slots: a chunk's K x hidden partial is worth its rows
constexpr int PB_DBM_GROUP = 32;

struct PbParams {
  const __nv_bfloat16* table;   // B2: bf16 [n_rows, pitch]
  int64_t n_rows, pitch;
  int32_t K;
  const int32_t* row_ids;       // B2: [n_groups * k] or NULL (row0 + flat)
  int64_t row0;
  int64_t n_groups;
  int32_t k, G, n_slices;
  int64_t n_tiles;
  const unsigned char* dp;      // B1's images
  int32_t rb_per_chunk, n_rb;   // B2: row blocks (2 per tile) per chunk, in all
  int32_t n_ftiles;             // B2: ceil(K / 128); B3: ceil(Kd / 128)
  float* part;                  // B2: [n_chunks][K][hidden]
  const unsigned char* wimg;    // B3: [n_ftiles][hidden / 64][16 KB]
  int32_t Kd;
  float* dx;                    // B3: [n_groups * k, ldx]
  int64_t ldx;
};

// Wm [K, hidden] fp32 -> bf16 images of Wm (rows = input columns f < Kd, K-major over hidden): image (fb, hb) holds
// columns 128 fb .. + 127 x hidden units 64 hb .. + 63
__global__ void __launch_bounds__(256) pool_dx_pack_kernel(const float* __restrict__ W, int64_t ldw, int Kd, int hidden,
                                                           unsigned char* __restrict__ img) {
  const int hbs = hidden / 64, fb = blockIdx.x / hbs, hb = blockIdx.x % hbs;
  unsigned char* dst = img + (int64_t)blockIdx.x * PB_IMG;
  for (int q = threadIdx.x; q < 128 * 8; q += blockDim.x) {
    const int n = q >> 3, c = q & 7;
    const int f = fb * 128 + n, h0 = hb * 64 + c * 8;
    __nv_bfloat162 h[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float a = f < Kd ? W[(int64_t)f * ldw + h0 + 2 * e] : 0.f;
      const float b = f < Kd ? W[(int64_t)f * ldw + h0 + 2 * e + 1] : 0.f;
      h[e] = __floats2bfloat162_rn(a, b);
    }
    *reinterpret_cast<uint4*>(dst + sw128_off(n, c)) = *reinterpret_cast<uint4*>(h);
  }
}

// kDW: B2 (grid: chunk x slice x feature tile, feature tile fastest); else B3 (grid: tile x column tile)
template <bool kDW>
__global__ void __launch_bounds__(PB_THREADS, 2) pool_bwd_gemm_kernel(const __grid_constant__ PbParams prm) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31, wq = (tid >> 5) & 3;
  const int ft = blockIdx.x % prm.n_ftiles;
  int slice = 0, it0 = 0, it1 = 0;
  int64_t t = 0;
  int chunk = 0;
  if constexpr (kDW) {
    const int rest = blockIdx.x / prm.n_ftiles;
    slice = rest % prm.n_slices;
    chunk = rest / prm.n_slices;
    it0 = chunk * prm.rb_per_chunk;
    it1 = min(it0 + prm.rb_per_chunk, prm.n_rb);
  } else {
    t = blockIdx.x / prm.n_ftiles;
    it1 = prm.n_slices * 2;                         // hidden in blocks of 64
  }
  const int rows_valid = prm.G * prm.k;
  const int64_t total_rows = prm.n_groups * prm.k;
  const int c = tid & 7, rl = tid >> 3;              // B2: this thread's 16-byte column c of rows rl and rl + 32

  auto issue = [&](int it) {
    if (it < it1) {
      unsigned char* st = smem + (size_t)(it % PB_STAGES) * PB_STAGE;
      if constexpr (kDW) {
        const int64_t tt = it >> 1;
        const int h = it & 1;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = rl + 32 * i, slot = h * 64 + r;
          const int64_t flat = tt * rows_valid + slot;
          const __nv_bfloat16* rowp = nullptr;
          if (slot < rows_valid && flat < total_rows) {
            int64_t id = prm.row_ids ? (int64_t)prm.row_ids[flat] : prm.row0 + flat;
            if (id < 0 || id >= prm.n_rows) id = prm.n_rows - 1;
            rowp = prm.table + id * prm.pitch;
          }
#pragma unroll
          for (int w = 0; w < 2; ++w) {
            const int col = (2 * ft + w) * 64 + c * 8;
            const int nbytes = (rowp != nullptr && col < prm.K) ? min(8, prm.K - col) * 2 : 0;
            cp_async16(st + w * PB_HALF + sw128_off(r, c), nbytes ? (const void*)(rowp + col) : (const void*)prm.table,
                       nbytes);
          }
        }
        const unsigned char* src = prm.dp + ((tt * prm.n_slices + slice) * 2 + h) * (int64_t)PB_IMG;
#pragma unroll
        for (int i = 0; i < PB_IMG / 16 / PB_THREADS; ++i) {
          const int q = tid + PB_THREADS * i;
          cp_async16(st + 2 * PB_HALF + q * 16, src + q * 16, 16);
        }
      } else {
        const int s = it >> 1, hoff = (it & 1) * PB_HALF;    // hidden units 64 it .. + 63 = rows hoff / 128 .. of the image
        const unsigned char* a0 = prm.dp + ((t * prm.n_slices + s) * 2) * (int64_t)PB_IMG + hoff;
        const unsigned char* b = prm.wimg + ((int64_t)ft * prm.n_slices * 2 + it) * PB_IMG;
#pragma unroll
        for (int i = 0; i < PB_STAGE / 16 / PB_THREADS; ++i) {
          const int q = tid + PB_THREADS * i;             // 16-byte piece of the stage
          const unsigned char* src = q < PB_HALF / 16       ? a0 + q * 16
                                     : q < PB_HALF / 8      ? a0 + PB_IMG + (q - PB_HALF / 16) * 16
                                                            : b + (q - PB_HALF / 8) * 16;
          cp_async16(st + q * 16, src, 16);
        }
      }
    }
    cp_async_commit();                               // empty groups keep the group count uniform
  };

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  issue(it0);
  issue(it0 + 1);
  for (int it = it0; it < it1; ++it) {
    unsigned char* st = smem + (size_t)(it % PB_STAGES) * PB_STAGE;
    cp_async_wait<1>();
    fence_proxy_async();
    __syncthreads();                                 // everyone's pieces are in; the stage of it - 1 is free
    issue(it + 2);
    const uint64_t adesc = make_smem_desc(smem_u32(st + wg * PB_HALF));
    const uint64_t bdesc = make_smem_desc(smem_u32(st + 2 * PB_HALF));
    acc_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)                      // 16 reduction rows = 2048 B of the MN-major piece, 32 B of the B rows
      wgmma_m64n128<true, 1>(acc, adesc + (uint64_t)(k * 128), bdesc + (uint64_t)(k * 2), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);
  }
  cp_async_wait<0>();

  const int hidden = prm.n_slices * 128;
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e2 = 0; e2 < 2; ++e2) {
      const int m = wq * 16 + (lane >> 2) + 8 * e2, n = 8 * j + 2 * (lane & 3);
      const float2 v = make_float2(acc[4 * j + 2 * e2], acc[4 * j + 2 * e2 + 1]);
      if constexpr (kDW) {
        const int f = ft * 128 + wg * 64 + m;
        if (f < prm.K)
          *reinterpret_cast<float2*>(prm.part + ((int64_t)chunk * prm.K + f) * hidden + slice * 128 + n) = v;
      } else {
        const int slot = wg * 64 + m, f = ft * 128 + n;
        const int64_t flat = t * rows_valid + slot;
        if (slot < rows_valid && flat < total_rows) {
          float* o = prm.dx + flat * prm.ldx;
          if (f < prm.Kd) o[f] = v.x;
          if (f + 1 < prm.Kd) o[f + 1] = v.y;
        }
      }
    }
}

// out[o * n + i] (+)= sum over p in [o * per_out, min((o + 1) * per_out, n_parts)) of part[p * n + i], p ascending
__global__ void pool_chunk_sum_kernel(const float* __restrict__ part, int64_t n_parts, int64_t per_out, int64_t n,
                                      float* __restrict__ out, int accumulate) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, o = blockIdx.y;
  if (i >= n) return;
  const int64_t p1 = min(n_parts, (o + 1) * per_out);
  float s = 0.f;
  for (int64_t p = o * per_out; p < p1; ++p) s += part[p * n + i];
  out[o * n + i] = accumulate ? out[o * n + i] + s : s;
}

static int32_t chunk_sum(const float* part, int64_t n_parts, int64_t per_out, int64_t n, float* out, int accumulate,
                         cudaStream_t st) {
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)((n_parts + per_out - 1) / per_out));
  pool_chunk_sum_kernel<<<grid, 256, 0, st>>>(part, n_parts, per_out, n, out, accumulate);
  return launch_check("pool_chunk_sum_kernel");
}

struct PbShape {
  int64_t n_tiles, n_rb, rb_per_chunk, n_chunks, dbm_groups;
};

static PbShape pb_shape(int64_t n_groups, int32_t k) {
  PbShape s;
  const int64_t G = 128 / k;
  s.n_tiles = (n_groups + G - 1) / G;
  s.n_rb = 2 * s.n_tiles;
  s.rb_per_chunk = (s.n_rb + PB_MAX_CHUNKS - 1) / PB_MAX_CHUNKS;
  if (s.rb_per_chunk < PB_MIN_RB_PER_CHUNK) s.rb_per_chunk = PB_MIN_RB_PER_CHUNK;
  s.n_chunks = (s.n_rb + s.rb_per_chunk - 1) / s.rb_per_chunk;
  s.dbm_groups = (s.n_tiles + PB_DBM_GROUP - 1) / PB_DBM_GROUP;
  return s;
}

}  // namespace gs

extern "C" {

// B2's scratch: the chunk partials of dWm [n_chunks][K][hidden] fp32, then the dbm group sums [groups][hidden] fp32
int64_t gs_pool_mlp_dw_workspace_bytes(int64_t n_groups, int32_t k, int32_t K, int32_t hidden) {
  if (n_groups < 0 || k < 1 || k > 128 || K < 1 || hidden < 128 || hidden % 128 != 0) return -1;
  const gs::PbShape s = gs::pb_shape(n_groups, k);
  return (s.n_chunks * K + s.dbm_groups) * (int64_t)hidden * 4;
}

int32_t gs_pool_mlp_backward_dw(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch, const int32_t* row_ids,
                                int64_t row0, int64_t n_groups, int32_t k, int32_t hidden, const void* dp, void* workspace,
                                int64_t workspace_bytes, float* dWm, int64_t ldw, float* dbm, void* stream) {
  GS_REQUIRE(n_groups >= 0 && k >= 1 && k <= 128, "gs_pool_mlp_backward_dw: bad n_groups / k (k <= 128)");
  if (n_groups == 0) return GS_OK;
  GS_REQUIRE(table_bf16 && dp && workspace && dWm && dbm, "gs_pool_mlp_backward_dw: NULL pointer");
  GS_REQUIRE(n_rows > 0 && n_rows < 0x7fffffffLL && K >= 1 && K <= 640 && pitch >= K,
             "gs_pool_mlp_backward_dw: bad table shape (K <= 640)");
  GS_REQUIRE((pitch * 2) % 16 == 0 && (reinterpret_cast<uintptr_t>(table_bf16) & 15u) == 0,
             "gs_pool_mlp_backward_dw: table rows must be 16-byte multiples and 16-byte aligned (pitch %% 8 == 0)");
  GS_REQUIRE(hidden >= 128 && hidden % 128 == 0 && ldw == hidden, "gs_pool_mlp_backward_dw: needs hidden %% 128 == 0 and ldw == hidden");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(dp) & 15u) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 15u) == 0,
             "gs_pool_mlp_backward_dw: dp / workspace misaligned");
  GS_REQUIRE(workspace_bytes >= gs_pool_mlp_dw_workspace_bytes(n_groups, k, K, hidden),
             "gs_pool_mlp_backward_dw: workspace too small");
  const gs::PbShape s = gs::pb_shape(n_groups, k);
  gs::PbParams prm;
  memset(&prm, 0, sizeof(prm));
  prm.table = (const __nv_bfloat16*)table_bf16; prm.n_rows = n_rows; prm.pitch = pitch; prm.K = K;
  prm.row_ids = row_ids; prm.row0 = row0; prm.n_groups = n_groups; prm.k = k; prm.G = 128 / k;
  prm.n_slices = hidden / 128; prm.n_tiles = s.n_tiles; prm.dp = (const unsigned char*)dp;
  prm.rb_per_chunk = (int32_t)s.rb_per_chunk; prm.n_rb = (int32_t)s.n_rb; prm.n_ftiles = (K + 127) / 128;
  prm.part = (float*)workspace;
  GS_REQUIRE(s.n_rb < 0x7fffffffLL, "gs_pool_mlp_backward_dw: too many groups (%lld)", (long long)n_groups);
  const void* fn = (const void*)gs::pool_bwd_gemm_kernel<true>;
  const int32_t rc_attr = gs::ensure_dyn_smem(fn, gs::PB_SMEM);
  if (rc_attr != GS_OK) return rc_attr;
  const cudaStream_t st = (cudaStream_t)stream;
  gs::pool_bwd_gemm_kernel<true><<<(unsigned)(s.n_chunks * prm.n_slices * prm.n_ftiles), gs::PB_THREADS, gs::PB_SMEM, st>>>(prm);
  int32_t rc = gs::launch_check("pool_bwd_gemm_kernel<dW>");
  if (rc != GS_OK) return rc;
  rc = gs::chunk_sum(prm.part, s.n_chunks, s.n_chunks, (int64_t)K * hidden, dWm, 1, st);
  if (rc != GS_OK) return rc;
  const float* dbm_part = reinterpret_cast<const float*>((const unsigned char*)dp + s.n_tiles * hidden * 256);
  float* groups = prm.part + s.n_chunks * (int64_t)K * hidden;
  rc = gs::chunk_sum(dbm_part, s.n_tiles, gs::PB_DBM_GROUP, hidden, groups, 0, st);
  if (rc != GS_OK) return rc;
  return gs::chunk_sum(groups, s.dbm_groups, s.dbm_groups, hidden, dbm, 1, st);
}

int64_t gs_pool_mlp_dx_pack_bytes(int32_t Kd, int32_t hidden) {
  if (Kd < 1 || hidden < 128 || hidden % 128 != 0) return -1;
  return (int64_t)((Kd + 127) / 128) * (hidden / 64) * gs::PB_IMG;
}

int32_t gs_pool_mlp_dx_pack(const float* Wm, int64_t ldw, int32_t Kd, int32_t hidden, void* packed, void* stream) {
  GS_REQUIRE(Wm && packed && Kd >= 1 && hidden >= 128 && hidden % 128 == 0 && ldw >= hidden,
             "gs_pool_mlp_dx_pack: bad arguments");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 15u) == 0, "gs_pool_mlp_dx_pack: packed must be 16-byte aligned");
  gs::pool_dx_pack_kernel<<<((Kd + 127) / 128) * (hidden / 64), 256, 0, (cudaStream_t)stream>>>(Wm, ldw, Kd, hidden,
                                                                                                 (unsigned char*)packed);
  return gs::launch_check("pool_dx_pack_kernel");
}

int32_t gs_pool_mlp_backward_dx(int64_t n_groups, int32_t k, int32_t hidden, const void* dp, const void* packed, int32_t Kd,
                                float* dx, int64_t ldx, void* stream) {
  GS_REQUIRE(n_groups >= 0 && k >= 1 && k <= 128, "gs_pool_mlp_backward_dx: bad n_groups / k (k <= 128)");
  if (n_groups == 0) return GS_OK;
  GS_REQUIRE(dp && packed && dx, "gs_pool_mlp_backward_dx: NULL pointer");
  GS_REQUIRE(hidden >= 128 && hidden % 128 == 0 && Kd >= 1 && ldx >= Kd, "gs_pool_mlp_backward_dx: bad shape");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(dp) & 15u) == 0 && (reinterpret_cast<uintptr_t>(packed) & 15u) == 0,
             "gs_pool_mlp_backward_dx: dp / packed misaligned");
  const gs::PbShape s = gs::pb_shape(n_groups, k);
  gs::PbParams prm;
  memset(&prm, 0, sizeof(prm));
  prm.n_groups = n_groups; prm.k = k; prm.G = 128 / k; prm.n_slices = hidden / 128; prm.n_tiles = s.n_tiles;
  prm.dp = (const unsigned char*)dp; prm.n_ftiles = (Kd + 127) / 128; prm.wimg = (const unsigned char*)packed;
  prm.Kd = Kd; prm.dx = dx; prm.ldx = ldx;
  GS_REQUIRE(s.n_tiles * prm.n_ftiles < 0x7fffffffLL, "gs_pool_mlp_backward_dx: too many groups (%lld)", (long long)n_groups);
  const void* fn = (const void*)gs::pool_bwd_gemm_kernel<false>;
  const int32_t rc_attr = gs::ensure_dyn_smem(fn, gs::PB_SMEM);
  if (rc_attr != GS_OK) return rc_attr;
  gs::pool_bwd_gemm_kernel<false>
      <<<(unsigned)(s.n_tiles * prm.n_ftiles), gs::PB_THREADS, gs::PB_SMEM, (cudaStream_t)stream>>>(prm);
  return gs::launch_check("pool_bwd_gemm_kernel<dX>");
}

}  // extern "C"

// K5: the two-layer max-pool aggregator's neighbour branch as ONE kernel on the Hopper tensor cores (wgmma, bf16
// operands, fp32 accumulate):
//   h1[r, :]  = bf16_rne(relu(table[row(g, j), :K] . W1 + b1))          (r = the gathered row of group g, fanout slot j)
//   out[g, u] = max_{j<k} relu(h1[r, :] . W2[:, u] + b2[u])
//   reference graphsage/aggregators.py:276-361 (reshape -> Dense -> Dense -> reshape -> reduce_max) with the feature
//   gather of graphsage/models.py:299 fused in front: neither the gathered rows nor h1 nor the second layer's
//   activations ever touch HBM.
//
// One CTA = one tile of 128 gathered rows (G = floor(128 / k) whole fanout groups, zero rows after them) x one 256-wide
// slice of h2; the h2 / 256 CTAs of a tile are adjacent in the grid and each recomputes layer 1 (the accumulators stay
// in registers).  Two consumer warpgroups of 64 rows.  The CTA walks h1 in 64-wide chunks:
//   layer 1: acc1 (64 x 64 per warpgroup) = X . W1[:, chunk] over the K-blocks, the gathered rows landing by cp.async
//            in a 3-stage ring beside the matching half (64 output rows) of the packed W1^T image, bulk-copied;
//   epilogue 1: + b1, ReLU, RNE to bf16 into a 128-row x 64-column SW128 tile - one K-block of layer 2's A operand;
//   layer 2: acc2 (64 x 256 per warpgroup, two m64n128) += h1_chunk . W2[chunk, slice], the two 128-wide W2^T images of
//            the chunk bulk-copied while layer 1 of the chunk runs.
// X is re-read (from L2) once per h1 chunk: the price of not holding the whole 128 x K row tile resident.
// Epilogue: raw acc2 -> staging tile in the operand ring ([128 columns][129] fp32, one 128-wide half at a time) -> max
// over each group's k rows -> + b2 -> ReLU -> coalesced store (bias and ReLU commute with the max).
// Both weights are packed by gs_maxpool_mlp_pack: W1 with K = F, W2 with K = h1.
#include "tc_common.cuh"

namespace gs {

constexpr int M2_KCOLS = 64;                      // bf16 columns per K-block (128 B of operand row)
constexpr int M2_IMG = 128 * 128;                 // one packed image: 128 output rows x 64 K columns, SW128
constexpr int M2_HALF = 64 * 128;                 // 64 output rows of it (one h1 chunk of W1^T)
constexpr int M2_MAX_KB = 10;                     // K <= 640
constexpr int M2_STAGES = 3;
constexpr int M2_LOOK = M2_STAGES - 1;            // K-blocks prefetched ahead of the one being multiplied
constexpr int M2_THREADS = 256;
constexpr int M2_ROWS_IMG = 128 * 128;            // 128 gathered rows x one K-block
constexpr int M2_STAGE = M2_ROWS_IMG + M2_HALF;   // rows image, then the W1 half image
constexpr int M2_H1 = 128 * 128;                  // h1 chunk: 128 rows x 64 bf16 columns
constexpr int M2_W2 = 2 * M2_IMG;                 // W2^T images of one chunk for the CTA's two 128-wide h2 halves
constexpr int M2_SMEM = M2_STAGES * M2_STAGE + M2_H1 + M2_W2;
constexpr int M2_LD = 129;                        // staging: [128 columns][128 + 1 rows]
static_assert(128 * M2_LD * 4 <= M2_STAGES * M2_STAGE, "epilogue staging must fit in the operand ring");

struct Mp2Params {
  const __nv_bfloat16* table;   // [n_rows, pitch]
  int64_t n_rows, pitch;
  int32_t K, kblocks;
  const int32_t* row_ids;       // [n_groups * k] or NULL
  int64_t row0;                 // used when row_ids == NULL: row(g, j) = row0 + g*k + j
  int64_t n_groups;
  int32_t k, G;                 // fanout, groups per tile
  int32_t n_chunks;             // h1 / 64
  int32_t n_slices;             // h2 / 256
  const unsigned char* w1img;   // packed W1^T: [h1 / 128][kblocks][16 KB]
  const unsigned char* w2img;   // packed W2^T: [h2 / 128][h1 / 64][16 KB]
  const float* b1;              // [h1] or NULL
  const float* b2;              // [h2] or NULL
  float* out;                   // [n_groups, h2]
  int64_t ldo;
};

__global__ void __launch_bounds__(M2_THREADS, 1) maxpool2_mlp_kernel(const __grid_constant__ Mp2Params prm) {
  constexpr int CPT = 128 / 32;                     // 16-byte row pieces per thread per K-block
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full_b[M2_STAGES];
  __shared__ __align__(8) uint64_t w2_b;
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* h1s = smem + M2_STAGES * M2_STAGE;
  unsigned char* w2s = h1s + M2_H1;
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31, wq = (tid >> 5) & 3;
  const int slice = blockIdx.x % prm.n_slices;
  const int64_t t = blockIdx.x / prm.n_slices;
  const int kblocks = prm.kblocks, n_chunks = prm.n_chunks, total = n_chunks * kblocks;

  if (tid == 0) {
    for (int s = 0; s < M2_STAGES; ++s) mbar_init(&full_b[s], 1);
    mbar_init(&w2_b, 1);
    fence_mbar_init();
  }
  __syncthreads();

  // this thread's 16-byte chunk column c of tile rows r0 + 32 i (padding rows and rows past the last group: zero-filled)
  const int c = tid & 7, r0 = tid >> 3;
  const int rows_valid = prm.G * prm.k;
  const __nv_bfloat16* rowp[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) {
    const int r = r0 + 32 * i;
    const int64_t flat = t * rows_valid + r;
    rowp[i] = nullptr;
    if (r < rows_valid && flat < prm.n_groups * prm.k) {
      int64_t id = prm.row_ids ? (int64_t)prm.row_ids[flat] : prm.row0 + flat;
      if (id < 0 || id >= prm.n_rows) id = prm.n_rows - 1;
      rowp[i] = prm.table + id * prm.pitch;
    }
  }
  // the CTA's two 128-wide W2^T slices (2 slice, 2 slice + 1), chunk ch at + ch * M2_IMG
  const unsigned char* w2src = prm.w2img + (int64_t)(2 * slice) * n_chunks * M2_IMG;
  auto issue_w2 = [&](int ch) {
    if (tid == 0) {
      mbar_expect_tx(&w2_b, M2_W2);
      bulk_g2s(w2s, w2src + (int64_t)ch * M2_IMG, M2_IMG, &w2_b);
      bulk_g2s(w2s + M2_IMG, w2src + (int64_t)(n_chunks + ch) * M2_IMG, M2_IMG, &w2_b);
    }
  };
  auto stage_of = [&](int it) { return smem + (size_t)(it % M2_STAGES) * M2_STAGE; };
  // step it = (chunk, K-block): the W1 half image by bulk copy, the row pieces by cp.async
  auto issue = [&](int it) {
    if (it < total) {
      const int ch = it / kblocks, kb = it - ch * kblocks;
      unsigned char* st = stage_of(it);
      if (tid == 0) {
        mbar_expect_tx(&full_b[it % M2_STAGES], M2_HALF);
        bulk_g2s(st + M2_ROWS_IMG, prm.w1img + ((int64_t)(ch >> 1) * kblocks + kb) * M2_IMG + (ch & 1) * M2_HALF, M2_HALF,
                 &full_b[it % M2_STAGES]);
      }
      const int col = kb * M2_KCOLS + c * 8;
#pragma unroll
      for (int i = 0; i < CPT; ++i) {
        int nbytes = 0;
        if (rowp[i] != nullptr && col < prm.K) nbytes = min(8, prm.K - col) * 2;
        const void* src = nbytes ? (const void*)(rowp[i] + col) : (const void*)prm.table;
        cp_async16(st + sw128_off(r0 + 32 * i, c), src, nbytes);
      }
    }
    cp_async_commit();                              // empty groups keep the group count uniform
  };

  issue_w2(0);
  for (int j = 0; j < M2_LOOK; ++j) issue(j);
  float acc1[32], acc2[2][64];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc1[i] = 0.f;
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc2[q][i] = 0.f;

  for (int it = 0; it < total; ++it) {
    const int ch = it / kblocks, kb = it - ch * kblocks;
    unsigned char* st = stage_of(it);
    cp_async_wait<M2_LOOK - 1>();                   // this thread's pieces of step it have landed
    fence_proxy_async();                            // generic-proxy writes -> visible to wgmma (async proxy)
    __syncthreads();                                // everyone's pieces are in; step it - 1's stage is free
    issue(it + M2_LOOK);
    mbar_wait(&full_b[it % M2_STAGES], (uint32_t)(it / M2_STAGES) & 1u);
    const uint32_t rows_s = smem_u32(st), w_s = smem_u32(st + M2_ROWS_IMG);
    acc_fence(acc1);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)                     // four K = 16 steps, 32 B apart inside the swizzle atom
      wgmma_m64n64_bf16(acc1, make_smem_desc(rows_s + (uint32_t)(wg * 64 * 128)) + (uint64_t)(k * 2),
                        make_smem_desc(w_s) + (uint64_t)(k * 2), (kb > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc1);
    if (kb != kblocks - 1) continue;

    // epilogue 1: h1 = bf16_rne(relu(acc1 + b1)) into this warpgroup's 64 rows of the h1 tile (SW128, K-major)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int m = wq * 16 + (lane >> 2) + 8 * p, n = 8 * j + 2 * (lane & 3);
        const int hc = ch * M2_KCOLS + n;
        const float v0 = fmaxf(acc1[4 * j + 2 * p] + (prm.b1 ? prm.b1[hc] : 0.f), 0.f);
        const float v1 = fmaxf(acc1[4 * j + 2 * p + 1] + (prm.b1 ? prm.b1[hc + 1] : 0.f), 0.f);
        *reinterpret_cast<__nv_bfloat162*>(h1s + sw128_off(wg * 64 + m, n >> 3) + (n & 7) * 2) =
            __floats2bfloat162_rn(v0, v1);
      }
    fence_proxy_async();
    __syncthreads();
    mbar_wait(&w2_b, (uint32_t)ch & 1u);
    const uint32_t h_s = smem_u32(h1s), v_s = smem_u32(w2s);
    acc_fence(acc2[0]);
    acc_fence(acc2[1]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int q = 0; q < 2; ++q)
        wgmma_m64n128<true>(acc2[q], make_smem_desc(h_s + (uint32_t)(wg * 64 * 128)) + (uint64_t)(k * 2),
                            make_smem_desc(v_s + (uint32_t)(q * M2_IMG)) + (uint64_t)(k * 2), (ch > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc2[0]);
    acc_fence(acc2[1]);
    __syncthreads();                                // both warpgroups are done with this chunk's h1 tile and W2 images
    if (ch + 1 < n_chunks) issue_w2(ch + 1);
  }
  cp_async_wait<0>();
  __syncthreads();                                  // the operand ring becomes the staging tile

  // =============================== epilogue ===============================
  // raw acc2 -> staging [column][row], one 128-wide half at a time; + b2 and ReLU after the max
  float* stage = reinterpret_cast<float*>(smem);
  const int k = prm.k, G = prm.G;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = wq * 16 + (lane >> 2) + 8 * (e >> 1);
        const int n = 8 * j + 2 * (lane & 3) + (e & 1);
        stage[n * M2_LD + wg * 64 + m] = acc2[q][4 * j + e];
      }
    __syncthreads();
    // thread = (column cc, group): consecutive threads take consecutive columns (conflict-free reads, coalesced stores)
    for (int u = tid; u < 128 * G; u += M2_THREADS) {
      const int cc = u & 127, g = u >> 7;
      const int64_t gg = t * G + g;
      if (gg >= prm.n_groups) break;
      const float* p = stage + cc * M2_LD + g * k;
      const int hcol = slice * 256 + q * 128 + cc;
      float mx = -3.0e38f;
      for (int j = 0; j < k; ++j) mx = fmaxf(mx, p[j]);
      prm.out[gg * prm.ldo + hcol] = fmaxf(mx + (prm.b2 ? prm.b2[hcol] : 0.f), 0.f);
    }
    __syncthreads();
  }
}

}  // namespace gs

extern "C" {

int32_t gs_maxpool2_mlp_fused(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch, const int32_t* row_ids,
                              int64_t row0, int64_t n_groups, int32_t k, const void* packed_w1, const float* b1,
                              int32_t h1, const void* packed_w2, const float* b2, int32_t h2, float* out, int64_t ldo,
                              void* stream) {
  GS_REQUIRE(n_groups >= 0 && k >= 1, "gs_maxpool2_mlp_fused: bad n_groups / k");
  if (n_groups == 0) return GS_OK;
  GS_REQUIRE(table_bf16 && packed_w1 && packed_w2 && out, "gs_maxpool2_mlp_fused: NULL pointer");
  GS_REQUIRE(n_rows > 0 && n_rows < 0x7fffffffLL && K >= 1 && pitch >= K, "gs_maxpool2_mlp_fused: bad table shape");
  GS_REQUIRE((pitch * 2) % 16 == 0 && (reinterpret_cast<uintptr_t>(table_bf16) & 15u) == 0,
             "gs_maxpool2_mlp_fused: table rows must be 16-byte multiples and 16-byte aligned (pitch %% 8 == 0)");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(packed_w1) & 127u) == 0 && (reinterpret_cast<uintptr_t>(packed_w2) & 127u) == 0,
             "gs_maxpool2_mlp_fused: packed weights misaligned");
  if (k > 128 || (K + gs::M2_KCOLS - 1) / gs::M2_KCOLS > gs::M2_MAX_KB || h1 < 128 || h1 % 128 != 0 || h2 < 256 ||
      h2 % 256 != 0) {
    gs::set_error("gs_maxpool2_mlp_fused: needs k <= 128, K <= %d, h1 %% 128 == 0, h2 %% 256 == 0 (k=%d K=%d h1=%d h2=%d)",
                  gs::M2_MAX_KB * gs::M2_KCOLS, k, K, h1, h2);
    return GS_ERR_UNSUPPORTED;
  }
  GS_REQUIRE(ldo >= h2, "gs_maxpool2_mlp_fused: ldo < h2");
  gs::Mp2Params prm;
  memset(&prm, 0, sizeof(prm));
  prm.table = (const __nv_bfloat16*)table_bf16;
  prm.n_rows = n_rows; prm.pitch = pitch; prm.K = K; prm.kblocks = (K + gs::M2_KCOLS - 1) / gs::M2_KCOLS;
  prm.row_ids = row_ids; prm.row0 = row0; prm.n_groups = n_groups; prm.k = k; prm.G = 128 / k;
  prm.n_chunks = h1 / gs::M2_KCOLS; prm.n_slices = h2 / 256;
  prm.w1img = (const unsigned char*)packed_w1; prm.w2img = (const unsigned char*)packed_w2;
  prm.b1 = b1; prm.b2 = b2; prm.out = out; prm.ldo = ldo;
  const int64_t n_tiles = (n_groups + prm.G - 1) / prm.G;
  GS_REQUIRE(n_tiles * prm.n_slices < 0x7fffffffLL, "gs_maxpool2_mlp_fused: too many groups (%lld)", (long long)n_groups);
  const void* fn = (const void*)gs::maxpool2_mlp_kernel;
  const int smem = gs::M2_SMEM + 1024;
  const int32_t rc_attr = gs::ensure_dyn_smem(fn, smem);
  if (rc_attr != GS_OK) return rc_attr;
  gs::maxpool2_mlp_kernel<<<(unsigned)(n_tiles * prm.n_slices), gs::M2_THREADS, smem, (cudaStream_t)stream>>>(prm);
  return gs::launch_check("maxpool2_mlp_kernel");
}

}  // extern "C"

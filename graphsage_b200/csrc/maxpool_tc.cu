// K4: the max-pool aggregator's neighbour branch as ONE kernel on the Hopper tensor cores (wgmma, bf16 operands,
// fp32 accumulate):
//   out[g, h] = max_{j<k} relu( table[row(g, j), :] . Wm[:, h] + bm[h] )
//   reference graphsage/aggregators.py:176-182 (reshape -> Dense(relu, bias) -> reshape -> reduce_max) with
//   graphsage/layers.py:104-116 and the feature gather of graphsage/models.py:299 fused in front of it:
//   neither the gathered [n*k, F] rows nor the [n*k, hidden] MLP activations ever touch HBM.
//
// One CTA = one tile of NT gathered rows (G = floor(NT / k) whole fanout groups, zero rows after them) x one 128-wide
// slice of the hidden dimension; the n_slices CTAs of a tile are adjacent in the grid, so the rows the first of them
// gathers are still in L2 for the others.  Two warpgroups.  K loop over 64-column K-blocks (128-byte operand rows,
// SWIZZLE_128B), MP_STAGES stages: the gathered rows land straight in a K-major tile (bf16 in the table = bf16 in the
// tile: no conversion), the slice's pre-swizzled Wm^T image comes by one cp.async.bulk on an mbarrier, then
// wgmma.m64n128k16 x 4 per K-block with the accumulators in registers.  Epilogue: raw accumulators -> staging tile in
// shared memory (reusing the operand ring, hidden-unit-major) -> max (or mean) over each group's k rows -> + bias ->
// ReLU -> coalesced store.
//
// Variants (template parameters, chosen at run time by tuning keys; every one is parity-tested):
//   kRowsA  (k4_operands = 1, the default): gathered rows = A operand (M = NT rows over the two warpgroups), Wm^T slice =
//           B (N = 128); 0: the roles swapped - the weight slice is A (M = 64 hidden units per warpgroup) and the
//           gathered rows are B (N = NT), so the weight image is read once per NT rows.
//   NT      (k4_tile): 128 rows per tile (two CTAs per SM, fanout <= 128) or 256 (fanout <= 256, one CTA per SM).
//   DEPTH   (k4_mma_depth): wgmma groups in flight; 2 lets the next K-block's MMAs queue behind the current ones at
//           the price of one stage of prefetch.
//   PROD    (k4_producer): 0 = cp.async 16-byte pieces; 1 = 128-bit register loads stored to the swizzled tile (the
//           loads of K-block kb + 1 fly under K-block kb's MMAs).
//   k4_cluster: launch the slices of a tile as a thread-block cluster (2 .. 8 CTAs; -1 = all slices of the tile) so
//           they are co-scheduled on one GPC and the tile's rows are fetched from HBM once for the whole cluster.
#include "tc_common.cuh"

namespace gs {

constexpr int MP_KCOLS = 64;                   // bf16 columns per K-block (128 B of operand row)
constexpr int MP_IMG = 128 * 128;              // one operand K-block image: 128 rows x 128 B
constexpr int MP_MAX_KB = 10;                  // K <= 640
constexpr int MP_STAGES = 3;
constexpr int MP_THREADS = 256;

struct MpParams {
  const __nv_bfloat16* table;   // [n_rows, pitch]
  int64_t n_rows, pitch;
  int32_t K, kblocks;
  const int32_t* row_ids;       // [n_groups * k] or NULL
  int64_t row0;                 // used when row_ids == NULL: row(g, j) = row0 + g*k + j
  int64_t n_groups;
  int32_t k, G;                 // fanout, groups per tile
  int32_t n_slices;
  const unsigned char* wimg;    // packed Wm^T: [n_slices][kblocks][16 KB]
  const float* bias;            // [hidden] or NULL
  int32_t pool_mean;            // 0: max over the fanout (MaxPoolingAggregator), 1: mean (MeanPoolingAggregator)
  float* out;                   // [n_groups, hidden]
  int64_t ldo;
  // B1 (kGrad, gs_pool_mlp_backward_dp) only
  const float* dhp;             // [n_groups, hidden] (row stride lddhp): gradient of the pooled output
  int64_t lddhp;
  unsigned char* dp;            // dP^T tile images: [n_tiles][n_slices][2 row halves][128 hidden x 64 rows, bf16, SW128]
  float* dbm_part;              // [n_tiles][hidden]: per-tile column sums of dpre
};

// Wm [K, hidden] row-major fp32 -> bf16 tile images of Wm^T (128 hidden rows x 64 k, K-major, SW128)
__global__ void __launch_bounds__(256) maxpool_pack_kernel(const float* __restrict__ W, int64_t ldw, int K, int hidden,
                                                           int kblocks, unsigned char* __restrict__ img) {
  const int slice = blockIdx.x / kblocks, kb = blockIdx.x % kblocks;
  unsigned char* dst = img + ((int64_t)slice * kblocks + kb) * MP_IMG;
  for (int q = threadIdx.x; q < 128 * 8; q += blockDim.x) {
    const int c = q >> 7, n = q & 127;
    const int gn = slice * 128 + n, k0 = kb * MP_KCOLS + c * 8;
    __nv_bfloat162 h[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float a = (gn < hidden && k0 + 2 * e < K) ? W[(int64_t)(k0 + 2 * e) * ldw + gn] : 0.f;
      float b = (gn < hidden && k0 + 2 * e + 1 < K) ? W[(int64_t)(k0 + 2 * e + 1) * ldw + gn] : 0.f;
      h[e] = __floats2bfloat162_rn(a, b);
    }
    *reinterpret_cast<uint4*>(dst + sw128_off(n, c)) = *reinterpret_cast<uint4*>(h);
  }
}

// kGrad (B1 of the pooling branch's backward, only <true, 128, 1, 0>): the same main loop recomputes the tile's
// pre-activations, and the epilogue turns them into dpre instead of the pooled output (see gs_pool_mlp_backward_dp)
template <bool kRowsA, int NT, int DEPTH, int PROD, bool kGrad = false>
__global__ void __launch_bounds__(MP_THREADS, NT == 128 ? 2 : 1) maxpool_mlp_kernel(const __grid_constant__ MpParams prm) {
  constexpr int ROWS_IMG = NT * 128;                      // gathered rows of one K-block
  constexpr int STAGE = ROWS_IMG + MP_IMG;                // rows image, then the weight image
  constexpr int CPT = NT / 32;                            // 16-byte row pieces per thread per K-block
  constexpr int LOOK = MP_STAGES - DEPTH;                 // K-blocks prefetched ahead of the one being multiplied
  constexpr int MI = kRowsA ? NT / 128 : 1;               // m64 blocks per warpgroup
  constexpr int NI = kRowsA ? 1 : NT / 128;               // n128 blocks
  constexpr int LD = NT + 1;                              // staging: [128 hidden][NT + 1]
  static_assert(128 * LD * 4 <= MP_STAGES * STAGE, "epilogue staging must fit in the operand ring");
  static_assert(LOOK >= 1, "at least one K-block of prefetch");
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full_b[MP_STAGES];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31, wq = (tid >> 5) & 3;
  const int slice = blockIdx.x % prm.n_slices;
  const int64_t t = blockIdx.x / prm.n_slices;
  const int kblocks = prm.kblocks;

  if (tid == 0) {
    for (int s = 0; s < MP_STAGES; ++s) mbar_init(&full_b[s], 1);
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
    const int64_t flat = t * rows_valid + r;        // index into the (group, j) row list
    rowp[i] = nullptr;
    if (r < rows_valid && flat < prm.n_groups * prm.k) {
      int64_t id = prm.row_ids ? (int64_t)prm.row_ids[flat] : prm.row0 + flat;
      if (id < 0 || id >= prm.n_rows) id = prm.n_rows - 1;
      rowp[i] = prm.table + id * prm.pitch;
    }
  }
  const unsigned char* wsrc = prm.wimg + (int64_t)slice * kblocks * MP_IMG;
  auto stage_of = [&](int kb) { return smem + (size_t)(kb % MP_STAGES) * STAGE; };
  // weight image by bulk copy (+ the row pieces by cp.async in the PROD 0 form) of K-block kb into its stage
  auto issue = [&](int kb) {
    if (kb < kblocks) {
      unsigned char* st = stage_of(kb);
      if (tid == 0) {
        mbar_expect_tx(&full_b[kb % MP_STAGES], MP_IMG);
        bulk_g2s(st + ROWS_IMG, wsrc + (int64_t)kb * MP_IMG, MP_IMG, &full_b[kb % MP_STAGES]);
      }
      if constexpr (PROD == 0) {
        const int col = kb * MP_KCOLS + c * 8;      // first bf16 column of this 16-byte piece
#pragma unroll
        for (int i = 0; i < CPT; ++i) {
          int nbytes = 0;
          if (rowp[i] != nullptr && col < prm.K) nbytes = min(8, prm.K - col) * 2;
          const void* src = nbytes ? (const void*)(rowp[i] + col) : (const void*)prm.table;
          cp_async16(st + sw128_off(r0 + 32 * i, c), src, nbytes);
        }
      }
    }
    if constexpr (PROD == 0) cp_async_commit();    // empty groups keep the group count uniform
  };
  uint4 regs[PROD == 1 ? CPT : 1];
  auto load_regs = [&](int kb) {                    // PROD 1: K-block kb's pieces into registers
    const int col = kb * MP_KCOLS + c * 8;
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
      regs[i] = make_uint4(0, 0, 0, 0);
      if (rowp[i] == nullptr || col >= prm.K) continue;
      if (col + 8 <= prm.K) {
        regs[i] = __ldg(reinterpret_cast<const uint4*>(rowp[i] + col));
      } else {
        unsigned short h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const unsigned short* src = reinterpret_cast<const unsigned short*>(rowp[i] + col);
        for (int e = 0; e < prm.K - col; ++e) h[e] = __ldg(src + e);
        regs[i] = *reinterpret_cast<const uint4*>(h);
      }
    }
  };

  for (int j = 0; j < LOOK; ++j) issue(j);
  if constexpr (PROD == 1) load_regs(0);
  float acc[MI * NI][64];
#pragma unroll
  for (int a = 0; a < MI * NI; ++a)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[a][i] = 0.f;
  for (int kb = 0; kb < kblocks; ++kb) {
    unsigned char* st = stage_of(kb);
    if constexpr (PROD == 0) {
      cp_async_wait<LOOK - 1>();                    // this thread's pieces of K-block kb have landed
    } else {
#pragma unroll
      for (int i = 0; i < CPT; ++i) *reinterpret_cast<uint4*>(st + sw128_off(r0 + 32 * i, c)) = regs[i];
    }
    fence_proxy_async();                            // generic-proxy writes -> visible to wgmma (async proxy)
    __syncthreads();                                // everyone's pieces are in; K-block kb - DEPTH's stage is free
    issue(kb + LOOK);
    if constexpr (PROD == 1) {
      if (kb + 1 < kblocks) load_regs(kb + 1);
    }
    mbar_wait(&full_b[kb % MP_STAGES], (uint32_t)(kb / MP_STAGES) & 1u);
    const uint32_t rows_s = smem_u32(st), w_s = smem_u32(st + ROWS_IMG);
#pragma unroll
    for (int a = 0; a < MI * NI; ++a) acc_fence(acc[a]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)                     // four K = 16 steps, 32 B apart inside the swizzle atom
#pragma unroll
      for (int mi = 0; mi < MI; ++mi)
#pragma unroll
        for (int ni = 0; ni < NI; ++ni) {
          const uint64_t adesc = kRowsA ? make_smem_desc(rows_s + (uint32_t)((wg * (NT / 2) + mi * 64) * 128))
                                        : make_smem_desc(w_s + (uint32_t)(wg * 64 * 128));
          const uint64_t bdesc = kRowsA ? make_smem_desc(w_s) : make_smem_desc(rows_s + (uint32_t)(ni * 128 * 128));
          wgmma_m64n128<true>(acc[mi * NI + ni], adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2),
                              (kb > 0 || k > 0) ? 1u : 0u);
        }
    wgmma_commit();
    wgmma_wait<DEPTH - 1>();
#pragma unroll
    for (int a = 0; a < MI * NI; ++a) acc_fence(acc[a]);
  }
  wgmma_wait<0>();
#pragma unroll
  for (int a = 0; a < MI * NI; ++a) acc_fence(acc[a]);
  if constexpr (PROD == 0) cp_async_wait<0>();
  __syncthreads();                                  // the operand ring becomes the staging tile

  // =============================== epilogue ===============================
  // raw accumulators go to the staging tile [hidden][row]; bias and ReLU are applied AFTER the max
  // (max_j relu(x_j + b) == relu(max_j x_j + b): b is per column, relu is monotone)
  float* stage = reinterpret_cast<float*>(smem);
#pragma unroll
  for (int mi = 0; mi < MI; ++mi)
#pragma unroll
    for (int ni = 0; ni < NI; ++ni)
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int m = wq * 16 + (lane >> 2) + 8 * (e >> 1);       // accumulator row within the m64 block
          const int n = 8 * j + 2 * (lane & 3) + (e & 1);           // accumulator column within the n128 block
          const int row = kRowsA ? wg * (NT / 2) + mi * 64 + m : ni * 128 + n;
          const int col = kRowsA ? n : wg * 64 + m;
          stage[col * LD + row] = acc[mi * NI + ni][4 * j + e];
        }
  __syncthreads();
  const int k = prm.k, G = prm.G;
  if constexpr (kGrad) {
    static_assert(kRowsA && NT == 128, "B1 reads the <rows as A, 128-row tile> staging layout");
    // thread = (column cc, group parity): dpre of each of its groups overwrites that group's staging entries;
    // the per-group sums (j order) are summed in g order per parity, then the two parities are added
    const int cc = tid & (TC_BN - 1), hcol = slice * 128 + cc;
    const float b = prm.bias ? prm.bias[hcol] : 0.f;
    float part = 0.f;
    for (int g = tid >> 7; g < G; g += 2) {
      const int64_t gg = t * G + g;
      if (gg >= prm.n_groups) break;
      float* p = stage + cc * LD + g * k;
      const float d = prm.dhp[gg * prm.lddhp + hcol];
      float s = 0.f;
      if (prm.pool_mean) {                          // dpre_j = (dhp / k) * [fl(pre_j + b) > 0]
        const float q = d / (float)k;
        for (int j = 0; j < k; ++j) {
          const float v = (p[j] + b > 0.f) ? q : 0.f;
          p[j] = v;
          s += v;
        }
      } else {                                      // ties at hp > 0 share dhp evenly; hp == 0: ReLU blocks everything
        float m = -3.0e38f;
        for (int j = 0; j < k; ++j) m = fmaxf(m, p[j]);
        const float hp = fmaxf(m + b, 0.f);
        int cnt = 0;
        if (hp > 0.f)
          for (int j = 0; j < k; ++j) cnt += (p[j] + b == hp) ? 1 : 0;
        const float q = cnt ? d / (float)cnt : 0.f;
        for (int j = 0; j < k; ++j) {
          const float v = (cnt && p[j] + b == hp) ? q : 0.f;
          p[j] = v;
          s += v;
        }
      }
      part += s;
    }
    float* red = stage + TC_BN * LD;                // [2][128] behind the staging tile, inside the operand ring
    red[(tid >> 7) * TC_BN + cc] = part;
    __syncthreads();
    if (tid < TC_BN) prm.dbm_part[t * (int64_t)prm.n_slices * 128 + hcol] = red[cc] + red[TC_BN + cc];
    // dP^T images of this (tile, slice): half h holds rows 64h .. 64h + 63; 16-byte piece = 8 rows of one hidden unit.
    // Padding rows and rows past the last group are zero.
    const int nvalid = (int)min((int64_t)G * k, prm.n_groups * k - t * (int64_t)G * k);
    unsigned char* img = prm.dp + (t * prm.n_slices + slice) * (int64_t)(2 * MP_IMG);
#pragma unroll
    for (int i = 0; i < (2 * 128 * 8) / MP_THREADS; ++i) {
      const int q = tid + MP_THREADS * i;
      const int h = q >> 10, n = (q >> 3) & 127, c = q & 7;
      const int r0 = h * 64 + c * 8;
      __nv_bfloat162 v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float a0 = (r0 + 2 * e < nvalid) ? stage[n * LD + r0 + 2 * e] : 0.f;
        const float a1 = (r0 + 2 * e + 1 < nvalid) ? stage[n * LD + r0 + 2 * e + 1] : 0.f;
        v[e] = __floats2bfloat162_rn(a0, a1);
      }
      *reinterpret_cast<uint4*>(img + h * MP_IMG + sw128_off(n, c)) = *reinterpret_cast<uint4*>(v);
    }
  } else {
    // thread = (column cc, group): consecutive threads take consecutive columns (conflict-free staging reads,
    // coalesced stores)
    for (int u = tid; u < TC_BN * G; u += MP_THREADS) {
      const int cc = u & (TC_BN - 1), g = u / TC_BN;
      const int64_t gg = t * G + g;
      if (gg >= prm.n_groups) break;
      const float* p = stage + cc * LD + g * k;
      const int hcol = slice * 128 + cc;
      const float b = prm.bias ? prm.bias[hcol] : 0.f;
      float res;
      if (prm.pool_mean) {
        // mean-pool (reference aggregators.py:246-273): ReLU does not commute with the mean, so bias + ReLU
        // are applied per element, summed in j order, divided by k
        float sacc = 0.f;
        for (int j = 0; j < k; ++j) sacc += fmaxf(p[j] + b, 0.f);
        res = sacc / (float)k;
      } else {
        float m = -3.0e38f;
        int j = 0;
        for (; j + 8 <= k; j += 8) {
          float v[8];
#pragma unroll
          for (int w = 0; w < 8; ++w) v[w] = p[j + w];
          m = fmaxf(m, fmaxf(fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3])), fmaxf(fmaxf(v[4], v[5]), fmaxf(v[6], v[7]))));
        }
        for (; j < k; ++j) m = fmaxf(m, p[j]);
        res = fmaxf(m + b, 0.f);                      // Dense bias + ReLU (commute with the max)
      }
      prm.out[gg * prm.ldo + hcol] = res;
    }
  }
}

template <bool kRowsA, int NT, int DEPTH, int PROD>
static int32_t launch_k4(const MpParams& prm, int64_t n_tiles, int cluster, cudaStream_t st) {
  const void* fn = (const void*)maxpool_mlp_kernel<kRowsA, NT, DEPTH, PROD>;
  const int smem = MP_STAGES * (NT * 128 + MP_IMG) + 1024;
  const int32_t rc_attr = ensure_dyn_smem(fn, smem);
  if (rc_attr != GS_OK) return rc_attr;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(n_tiles * prm.n_slices));
  cfg.blockDim = dim3((unsigned)MP_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr;
  if (cluster > 1) {                               // the grid is a multiple of n_slices, which cluster divides
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)cluster;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
  }
  MpParams p = prm;
  void* args[1] = {(void*)&p};
  GS_CUDA(cudaLaunchKernelExC(&cfg, fn, args));
  return launch_check("maxpool_mlp_kernel");
}

template <bool kRowsA, int NT>
static int32_t launch_k4_by(const MpParams& prm, int64_t n_tiles, int cluster, int depth, int producer, cudaStream_t st) {
  if (depth == 2)
    return producer == 1 ? launch_k4<kRowsA, NT, 2, 1>(prm, n_tiles, cluster, st) : launch_k4<kRowsA, NT, 2, 0>(prm, n_tiles, cluster, st);
  return producer == 1 ? launch_k4<kRowsA, NT, 1, 1>(prm, n_tiles, cluster, st) : launch_k4<kRowsA, NT, 1, 0>(prm, n_tiles, cluster, st);
}

}  // namespace gs

extern "C" {

// packed weights: [slices][ceil(K/64)] images of 128 x 128 B (SW128), re-packed per weight update, not per step
int64_t gs_maxpool_mlp_workspace_bytes(int32_t K, int32_t hidden) {
  if (K < 1 || hidden < 1) return -1;
  const int kblocks = (K + gs::MP_KCOLS - 1) / gs::MP_KCOLS, slices = (hidden + 127) / 128;
  return (int64_t)kblocks * slices * gs::MP_IMG;
}

int32_t gs_maxpool_mlp_pack(const float* Wm, int64_t ldw, int32_t K, int32_t hidden, void* workspace, void* stream) {
  GS_REQUIRE(Wm && workspace && K >= 1 && hidden >= 1 && ldw >= hidden, "gs_maxpool_mlp_pack: bad arguments");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 127u) == 0, "gs_maxpool_mlp_pack: workspace must be 128-byte aligned");
  const int kblocks = (K + gs::MP_KCOLS - 1) / gs::MP_KCOLS, slices = (hidden + 127) / 128;
  gs::maxpool_pack_kernel<<<kblocks * slices, 256, 0, (cudaStream_t)stream>>>(Wm, ldw, K, hidden, kblocks,
                                                                             (unsigned char*)workspace);
  return gs::launch_check("maxpool_pack_kernel");
}

static int32_t pool_mlp_fused(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch, const int32_t* row_ids,
                              int64_t row0, int64_t n_groups, int32_t k, const void* packed_weights, const float* bias,
                              int32_t hidden, float* out, int64_t ldo, int32_t pool_mean, void* stream) {
  GS_REQUIRE(n_groups >= 0 && k >= 1, "gs_maxpool_mlp_fused: bad n_groups / k");
  if (n_groups == 0) return GS_OK;
  GS_REQUIRE(table_bf16 && packed_weights && out, "gs_maxpool_mlp_fused: NULL pointer");
  GS_REQUIRE(n_rows > 0 && n_rows < 0x7fffffffLL && K >= 1 && pitch >= K, "gs_maxpool_mlp_fused: bad table shape");
  GS_REQUIRE((pitch * 2) % 16 == 0 && (reinterpret_cast<uintptr_t>(table_bf16) & 15u) == 0,
             "gs_maxpool_mlp_fused: table rows must be 16-byte multiples and 16-byte aligned (pitch %% 8 == 0)");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(packed_weights) & 127u) == 0, "gs_maxpool_mlp_fused: packed weights misaligned");
  const int nt = gs::tuning("k4_tile", 128) == 256 ? 256 : 128;
  if (k > nt || (K + gs::MP_KCOLS - 1) / gs::MP_KCOLS > gs::MP_MAX_KB || hidden % 128 != 0) {
    gs::set_error("gs_maxpool_mlp_fused: needs k <= %d, K <= %d, hidden %% 128 == 0 (k=%d K=%d hidden=%d)", nt,
                  gs::MP_MAX_KB * gs::MP_KCOLS, k, K, hidden);
    return GS_ERR_UNSUPPORTED;
  }
  GS_REQUIRE(ldo >= hidden, "gs_maxpool_mlp_fused: ldo < hidden");
  gs::MpParams prm;
  memset(&prm, 0, sizeof(prm));
  prm.table = (const __nv_bfloat16*)table_bf16;
  prm.n_rows = n_rows; prm.pitch = pitch; prm.K = K; prm.kblocks = (K + gs::MP_KCOLS - 1) / gs::MP_KCOLS;
  prm.row_ids = row_ids; prm.row0 = row0; prm.n_groups = n_groups; prm.k = k; prm.G = nt / k;
  prm.n_slices = hidden / 128;
  prm.wimg = (const unsigned char*)packed_weights; prm.bias = bias; prm.out = out; prm.ldo = ldo;
  prm.pool_mean = pool_mean;
  const int64_t n_tiles = (n_groups + prm.G - 1) / prm.G;
  GS_REQUIRE(n_tiles * prm.n_slices < 0x7fffffffLL, "gs_maxpool_mlp_fused: too many groups (%lld)", (long long)n_groups);
  int cluster = gs::tuning("k4_cluster", 0);       // -1 = all slices of a tile; clamped to a divisor of n_slices <= 8
  if (cluster < 0 || cluster > prm.n_slices) cluster = prm.n_slices;
  while (cluster > 1 && (cluster > 8 || prm.n_slices % cluster != 0)) --cluster;
  const int depth = gs::tuning("k4_mma_depth", 1) == 2 ? 2 : 1;
  const int producer = gs::tuning("k4_producer", 0) == 1 ? 1 : 0;
  const bool rows_a = gs::tuning("k4_operands", 1) != 0;
  const cudaStream_t st = (cudaStream_t)stream;
  if (rows_a)
    return nt == 256 ? gs::launch_k4_by<true, 256>(prm, n_tiles, cluster, depth, producer, st)
                     : gs::launch_k4_by<true, 128>(prm, n_tiles, cluster, depth, producer, st);
  return nt == 256 ? gs::launch_k4_by<false, 256>(prm, n_tiles, cluster, depth, producer, st)
                   : gs::launch_k4_by<false, 128>(prm, n_tiles, cluster, depth, producer, st);
}

int32_t gs_maxpool_mlp_fused(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch, const int32_t* row_ids,
                             int64_t row0, int64_t n_groups, int32_t k, const void* packed_weights, const float* bias,
                             int32_t hidden, float* out, int64_t ldo, void* stream) {
  return pool_mlp_fused(table_bf16, n_rows, K, pitch, row_ids, row0, n_groups, k, packed_weights, bias, hidden, out, ldo, 0,
                        stream);
}

int32_t gs_meanpool_mlp_fused(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch, const int32_t* row_ids,
                              int64_t row0, int64_t n_groups, int32_t k, const void* packed_weights, const float* bias,
                              int32_t hidden, float* out, int64_t ldo, void* stream) {
  return pool_mlp_fused(table_bf16, n_rows, K, pitch, row_ids, row0, n_groups, k, packed_weights, bias, hidden, out, ldo, 1,
                        stream);
}

// B1's output buffer: the dP^T tile images (n_tiles * hidden * 256 bytes), then the fp32 dbm partials [n_tiles][hidden]
int64_t gs_pool_mlp_dp_bytes(int64_t n_groups, int32_t k, int32_t hidden) {
  if (n_groups < 0 || k < 1 || k > 128 || hidden < 128 || hidden % 128 != 0) return -1;
  const int64_t G = 128 / k, n_tiles = (n_groups + G - 1) / G;
  return n_tiles * hidden * (256 + 4);
}

int32_t gs_pool_mlp_backward_dp(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch, const int32_t* row_ids,
                                int64_t row0, int64_t n_groups, int32_t k, const void* packed_weights, const float* bias,
                                int32_t hidden, const float* dhp, int64_t lddhp, int32_t pool_mean, void* dp, void* stream) {
  GS_REQUIRE(n_groups >= 0 && k >= 1, "gs_pool_mlp_backward_dp: bad n_groups / k");
  if (n_groups == 0) return GS_OK;
  GS_REQUIRE(table_bf16 && packed_weights && dhp && dp, "gs_pool_mlp_backward_dp: NULL pointer");
  GS_REQUIRE(n_rows > 0 && n_rows < 0x7fffffffLL && K >= 1 && pitch >= K, "gs_pool_mlp_backward_dp: bad table shape");
  GS_REQUIRE((pitch * 2) % 16 == 0 && (reinterpret_cast<uintptr_t>(table_bf16) & 15u) == 0,
             "gs_pool_mlp_backward_dp: table rows must be 16-byte multiples and 16-byte aligned (pitch %% 8 == 0)");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(packed_weights) & 127u) == 0 && (reinterpret_cast<uintptr_t>(dp) & 15u) == 0,
             "gs_pool_mlp_backward_dp: packed weights / dp misaligned");
  if (k > 128 || (K + gs::MP_KCOLS - 1) / gs::MP_KCOLS > gs::MP_MAX_KB || hidden % 128 != 0 || hidden < 128) {
    gs::set_error("gs_pool_mlp_backward_dp: needs k <= 128, K <= %d, hidden %% 128 == 0 (k=%d K=%d hidden=%d)",
                  gs::MP_MAX_KB * gs::MP_KCOLS, k, K, hidden);
    return GS_ERR_UNSUPPORTED;
  }
  GS_REQUIRE(lddhp >= hidden, "gs_pool_mlp_backward_dp: lddhp < hidden");
  gs::MpParams prm;
  memset(&prm, 0, sizeof(prm));
  prm.table = (const __nv_bfloat16*)table_bf16;
  prm.n_rows = n_rows; prm.pitch = pitch; prm.K = K; prm.kblocks = (K + gs::MP_KCOLS - 1) / gs::MP_KCOLS;
  prm.row_ids = row_ids; prm.row0 = row0; prm.n_groups = n_groups; prm.k = k; prm.G = 128 / k;
  prm.n_slices = hidden / 128;
  prm.wimg = (const unsigned char*)packed_weights; prm.bias = bias; prm.pool_mean = pool_mean;
  prm.dhp = dhp; prm.lddhp = lddhp;
  const int64_t n_tiles = (n_groups + prm.G - 1) / prm.G;
  prm.dp = (unsigned char*)dp;
  prm.dbm_part = reinterpret_cast<float*>((unsigned char*)dp + n_tiles * hidden * 256);
  GS_REQUIRE(n_tiles * prm.n_slices < 0x7fffffffLL, "gs_pool_mlp_backward_dp: too many groups (%lld)", (long long)n_groups);
  const void* fn = (const void*)gs::maxpool_mlp_kernel<true, 128, 1, 0, true>;
  const int smem = gs::MP_STAGES * (128 * 128 + gs::MP_IMG) + 1024;
  const int32_t rc_attr = gs::ensure_dyn_smem(fn, smem);
  if (rc_attr != GS_OK) return rc_attr;
  gs::maxpool_mlp_kernel<true, 128, 1, 0, true>
      <<<(unsigned)(n_tiles * prm.n_slices), gs::MP_THREADS, smem, (cudaStream_t)stream>>>(prm);
  return gs::launch_check("maxpool_mlp_kernel<grad>");
}

}  // extern "C"

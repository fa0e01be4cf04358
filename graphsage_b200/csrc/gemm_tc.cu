// Tensor-core path of gs_sage_gemm: the neigh_weights / self_weights contraction of the aggregators
// (reference graphsage/aggregators.py:51-64, 110-116, 184-195; Dense graphsage/layers.py:104-116)
// on the Hopper tensor cores (wgmma), fp32 in / fp32 out.
//
//   GS_MATH_TF32X3 : A = A_hi + A_lo, B = B_hi + B_lo (each exactly representable in tf32);
//                    D += A_hi*B_hi + A_hi*B_lo + A_lo*B_hi, fp32 accumulate in registers  -> fp32-grade result
//   GS_MATH_TF32   : one tf32 pass (operands masked to tf32)
//   GS_MATH_BF16   : one bf16 pass, operands rounded to bf16
//
// Structure (one CTA = one 128 x 128 output tile, two warpgroups of 128 threads, each owning 64 output rows):
//   B (weights): pre-swizzled tile images of W^T (built per weight update by pack_b_kernel into the caller's
//                workspace), one cp.async.bulk per K-block into a ring of stages, completion on an mbarrier.
//   A          : every thread loads its 16-byte chunks of the next K-block from global memory while the current
//                K-block's wgmmas run, then splits / converts them and stores the SW128 tile image; a part may name its
//                rows by id into a table (gs_sage_gemm_rows: the mean layer-0 self rows straight from the feature
//                table), resolved once per tile, so only the address of the load changes.
// A goes through registers on purpose: the hi/lo split (and the bf16 rounding) is arithmetic on the operand.
#include "tc_common.cuh"

namespace gs {

constexpr int TC_THREADS = 256;

struct TcPart {
  const float* A;
  int64_t lda;
  int32_t K;
  int32_t N;
  int32_t kblocks;     // ceil(K / BK)
  int32_t ntiles;      // ceil(N / 128)
  int64_t img_off;     // byte offset of this part's packed B images in the workspace
  const float* B;
  int64_t ldb;
};

struct TcParams {
  TcPart p[2];
  int32_t n_parts;
  int32_t combine;
  int64_t M;
  const float* bias;
  int32_t act;
  float* out;
  int64_t ldo;
  int32_t tiles_n0;    // number of N tiles of part 0 (CONCAT tile -> part mapping)
  gs_gemm_row_ids rid[2];       // part p's A rows by id (gs_sage_gemm_rows); n_ranges == 0: dense A
};

// ---------------------------------------------------------------------------------------------
// B packing: weights [K, N] row-major fp32 -> per (n tile, k block) tile images of W^T
// (N rows x BK k-elements, K-major, SW128), hi (+ lo) or bf16.  Tiny (<= a few MB), runs per weight update.
// MODE: 0 = tf32x3 (hi, lo images), 1 = tf32 (hi only), 2 = bf16
// ---------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(256) pack_b_kernel(TcParams prm, unsigned char* __restrict__ ws) {
  constexpr int BK = MODE == 2 ? 64 : 32;
  constexpr int EPC = MODE == 2 ? 8 : 4;        // elements per 16-byte chunk
  constexpr int NIMG = MODE == 0 ? 2 : 1;
  int unit = blockIdx.x;                        // (part, ntile, kblock) flattened
  int pi = 0;
  if (prm.n_parts == 2 && unit >= prm.p[0].ntiles * prm.p[0].kblocks) {
    unit -= prm.p[0].ntiles * prm.p[0].kblocks;
    pi = 1;
  }
  const TcPart& P = prm.p[pi];
  const int nt = unit / P.kblocks, kb = unit % P.kblocks;
  unsigned char* img = ws + P.img_off + ((int64_t)(nt * P.kblocks + kb) * NIMG) * TC_TILE_BYTES;
  for (int q = threadIdx.x; q < 128 * 8; q += blockDim.x) {
    const int c = q >> 7, n = q & 127;           // n fastest: coalesced reads along N
    const int gn = nt * TC_BN + n;
    const int k0 = kb * BK + c * EPC;
    float w[EPC];
#pragma unroll
    for (int e = 0; e < EPC; ++e) w[e] = (gn < P.N && k0 + e < P.K) ? P.B[(int64_t)(k0 + e) * P.ldb + gn] : 0.f;
    const uint32_t off = sw128_off(n, c);
    if constexpr (MODE == 2) {
      __nv_bfloat162 h[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(w[2 * e], w[2 * e + 1]);
      *reinterpret_cast<uint4*>(img + off) = *reinterpret_cast<uint4*>(h);
    } else {
      uint4 hi;
      hi.x = tf32_mask(w[0]); hi.y = tf32_mask(w[1]); hi.z = tf32_mask(w[2]); hi.w = tf32_mask(w[3]);
      *reinterpret_cast<uint4*>(img + off) = hi;
      if constexpr (MODE == 0) {
        uint4 lo;
        lo.x = tf32_mask(w[0] - __uint_as_float(hi.x)); lo.y = tf32_mask(w[1] - __uint_as_float(hi.y));
        lo.z = tf32_mask(w[2] - __uint_as_float(hi.z)); lo.w = tf32_mask(w[3] - __uint_as_float(hi.w));
        *reinterpret_cast<uint4*>(img + TC_TILE_BYTES + off) = lo;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// main kernel
// ---------------------------------------------------------------------------------------------
template <int MODE>
struct TcCfg {
  static constexpr int BK = MODE == 2 ? 64 : 32;             // K elements per block (128 B of operand row)
  static constexpr int NIMG = MODE == 0 ? 2 : 1;             // hi (+ lo)
  static constexpr int IMG_BYTES = NIMG * TC_TILE_BYTES;     // one operand's images for one K-block
  static constexpr int STAGES = MODE == 0 ? 3 : 4;           // A + B per stage: 64 KB (tf32x3) / 32 KB
  static constexpr int STAGE_BYTES = 2 * IMG_BYTES;          // A images, then B images
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;   // + slack for 1024-B alignment
  static constexpr int CPT = 4;                              // A chunks per thread per K-block (1024 / 256)
};

template <int MODE>
__device__ __forceinline__ void load_a_chunk(const TcPart& P, int64_t arow, int gcol, bool vec, float (&v)[8]) {
  constexpr int EPC = MODE == 2 ? 8 : 4;
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (arow < 0) return;                          // zero row (gemm_a_row)
  const float* src = P.A + arow * P.lda + gcol;
  if (vec && gcol + EPC <= P.K) {
    float4 a = ldg_nc_f4(reinterpret_cast<const float4*>(src));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    if constexpr (EPC == 8) {
      float4 b = ldg_nc_f4(reinterpret_cast<const float4*>(src) + 1);
      v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
  } else {
#pragma unroll
    for (int e = 0; e < EPC; ++e)
      if (gcol + e < P.K) v[e] = __ldg(src + e);
  }
}

template <int MODE>
__device__ __forceinline__ void store_a_chunk(unsigned char* tile, int row, int c, const float (&v)[8]) {
  const uint32_t off = sw128_off(row, c);
  if constexpr (MODE == 2) {
    __nv_bfloat162 h[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]);
    *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<uint4*>(h);
  } else {
    uint4 hi;
    hi.x = tf32_mask(v[0]); hi.y = tf32_mask(v[1]); hi.z = tf32_mask(v[2]); hi.w = tf32_mask(v[3]);
    *reinterpret_cast<uint4*>(tile + off) = hi;
    if constexpr (MODE == 0) {
      uint4 lo;
      lo.x = tf32_mask(v[0] - __uint_as_float(hi.x)); lo.y = tf32_mask(v[1] - __uint_as_float(hi.y));
      lo.z = tf32_mask(v[2] - __uint_as_float(hi.z)); lo.w = tf32_mask(v[3] - __uint_as_float(hi.w));
      *reinterpret_cast<uint4*>(tile + TC_TILE_BYTES + off) = lo;
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(TC_THREADS, 1) sage_gemm_tc_kernel(const __grid_constant__ TcParams prm,
                                                                     const unsigned char* __restrict__ ws) {
  using C = TcCfg<MODE>;
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full[C::STAGES];

  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31, wq = (tid >> 5) & 3;

  // ---- which output tile, which parts feed it
  const int64_t m0 = (int64_t)blockIdx.x * TC_BM;
  int part_lo = 0, part_hi = prm.n_parts, ntile = blockIdx.y, col_off = 0;
  if (prm.combine == GS_COMBINE_CONCAT && prm.n_parts == 2) {
    if ((int)blockIdx.y < prm.tiles_n0) part_hi = 1;
    else { part_lo = 1; ntile = blockIdx.y - prm.tiles_n0; col_off = prm.p[0].N; }
  }
  const int N = prm.p[part_lo].N;
  int total_it = 0;
  for (int pi = part_lo; pi < part_hi; ++pi) total_it += prm.p[pi].kblocks;
  auto locate = [&](int it, int& pi, int& kb) {
    pi = part_lo; kb = it;
    while (kb >= prm.p[pi].kblocks) { kb -= prm.p[pi].kblocks; ++pi; }
  };

  if (tid == 0) {
    for (int s = 0; s < C::STAGES; ++s) mbar_init(&full[s], 1);
    fence_mbar_init();
  }
  __syncthreads();

  // one thread posts the bulk copy of K-block `it`'s B images into its stage
  auto post = [&](int it) {
    if (tid != 0 || it >= total_it) return;
    int pi, kb;
    locate(it, pi, kb);
    const TcPart& P = prm.p[pi];
    const int s = it % C::STAGES;
    unsigned char* st = smem + (size_t)s * C::STAGE_BYTES;
    mbar_expect_tx(&full[s], C::IMG_BYTES);
    bulk_g2s(st + C::IMG_BYTES, ws + P.img_off + ((int64_t)ntile * P.kblocks + kb) * C::IMG_BYTES, C::IMG_BYTES, &full[s]);
  };
  // the A row behind each of this thread's chunks, for the tile's first and second part: fixed over the K loop, so a part
  // whose rows come by id looks each id up once per tile, not once per K-block
  int64_t arow_lo[C::CPT], arow_hi[C::CPT];
#pragma unroll
  for (int i = 0; i < C::CPT; ++i) {
    const int64_t r = m0 + ((tid + TC_THREADS * i) >> 3);
    arow_lo[i] = gemm_a_row(prm.rid[part_lo], prm.M, r);
    arow_hi[i] = part_hi - part_lo == 2 ? gemm_a_row(prm.rid[part_lo + 1], prm.M, r) : -1;
  }
  float cur[C::CPT][8];
  auto fetch = [&](int it) {
    int pi, kb;
    locate(it, pi, kb);
    const TcPart& P = prm.p[pi];
    const bool vec = ((P.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.A) & 15u) == 0);
#pragma unroll
    for (int i = 0; i < C::CPT; ++i) {
      const int q = tid + TC_THREADS * i;
      load_a_chunk<MODE>(P, pi == part_lo ? arow_lo[i] : arow_hi[i], kb * C::BK + (q & 7) * (MODE == 2 ? 8 : 4), vec, cur[i]);
    }
  };

  for (int j = 0; j < C::STAGES - 1; ++j) post(j);
  fetch(0);

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int it = 0; it < total_it; ++it) {
    const int s = it % C::STAGES;
    unsigned char* st = smem + (size_t)s * C::STAGE_BYTES;
#pragma unroll
    for (int i = 0; i < C::CPT; ++i) {
      const int q = tid + TC_THREADS * i;
      store_a_chunk<MODE>(st, q >> 3, q & 7, cur[i]);
    }
    fence_proxy_async();                         // generic-proxy stores -> visible to wgmma (async proxy)
    __syncthreads();                             // A stored; every warpgroup is done with K-block it - 1's stage
    post(it + C::STAGES - 1);                    // ... which is the stage this refills
    if (it + 1 < total_it) fetch(it + 1);        // next K-block's loads fly under this one's MMAs
    mbar_wait(&full[s], (uint32_t)(it / C::STAGES) & 1u);
    const uint32_t a_base = smem_u32(st) + (uint32_t)(wg * 64 * 128), b_base = smem_u32(st + C::IMG_BYTES);
    const uint64_t a_hi = make_smem_desc(a_base), b_hi = make_smem_desc(b_base);
    const uint64_t a_lo = make_smem_desc(a_base + TC_TILE_BYTES), b_lo = make_smem_desc(b_base + TC_TILE_BYTES);
    acc_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {                // four K steps of 32 B inside the 128-B swizzle atom
      const uint64_t koff = (uint64_t)((k * 32) >> 4);
      wgmma_m64n128<MODE == 2>(acc, a_hi + koff, b_hi + koff, (it > 0 || k > 0) ? 1u : 0u);
      if constexpr (MODE == 0) {
        wgmma_m64n128<false>(acc, a_hi + koff, b_lo + koff, 1u);
        wgmma_m64n128<false>(acc, a_lo + koff, b_hi + koff, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);
  }

  // =============================== epilogue: registers -> bias / ReLU -> global ===============================
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t grow = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
    if (grow >= prm.M) continue;
    float* dst_row = prm.out + grow * prm.ldo + col_off;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int gn = ntile * TC_BN + 8 * j + 2 * (lane & 3);
      float v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        v[e] = acc[4 * j + 2 * h + e];
        if (prm.bias && gn + e < N) v[e] += prm.bias[col_off + gn + e];
        if (prm.act == GS_ACT_RELU) v[e] = fmaxf(v[e], 0.f);
      }
      float* dst = dst_row + gn;
      if (gn + 2 <= N && (reinterpret_cast<uintptr_t>(dst) & 7u) == 0) {
        *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
      } else {
        if (gn < N) dst[0] = v[0];
        if (gn + 1 < N) dst[1] = v[1];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int mode_of(int32_t math) { return math == GS_MATH_TF32X3 ? 0 : math == GS_MATH_TF32 ? 1 : 2; }

static void fill_parts(TcParams& prm, int64_t M, const gs_gemm_part* parts, int32_t n_parts, int mode) {
  const int BK = mode == 2 ? 64 : 32;
  const int nimg = mode == 0 ? 2 : 1;
  memset(&prm, 0, sizeof(prm));
  prm.n_parts = n_parts;
  prm.M = M;
  int64_t off = 0;
  for (int i = 0; i < n_parts; ++i) {
    TcPart& P = prm.p[i];
    P.A = parts[i].A; P.lda = parts[i].lda; P.K = parts[i].K; P.N = parts[i].N;
    P.B = parts[i].B; P.ldb = parts[i].ldb;
    P.kblocks = (P.K + BK - 1) / BK;
    P.ntiles = (P.N + TC_BN - 1) / TC_BN;
    P.img_off = off;
    off += (int64_t)P.kblocks * P.ntiles * nimg * TC_TILE_BYTES;
  }
  prm.tiles_n0 = prm.p[0].ntiles;
}

int64_t sage_gemm_tc_workspace(int64_t M, const gs_gemm_part* parts, int32_t n_parts, int32_t math) {
  TcParams prm;
  fill_parts(prm, M, parts, n_parts, mode_of(math));
  const TcPart& L = prm.p[n_parts - 1];
  const int nimg = mode_of(math) == 0 ? 2 : 1;
  return L.img_off + (int64_t)L.kblocks * L.ntiles * nimg * TC_TILE_BYTES;
}

template <int MODE>
static int32_t launch_pack(const TcParams& prm, unsigned char* ws, cudaStream_t st) {
  int units = prm.p[0].ntiles * prm.p[0].kblocks + (prm.n_parts == 2 ? prm.p[1].ntiles * prm.p[1].kblocks : 0);
  pack_b_kernel<MODE><<<units, 256, 0, st>>>(prm, ws);
  return launch_check("pack_b_kernel");
}

template <int MODE>
static int32_t launch_tc(const TcParams& prm, const unsigned char* ws, cudaStream_t st) {
  using C = TcCfg<MODE>;
  const int32_t rc_attr = ensure_dyn_smem((const void*)sage_gemm_tc_kernel<MODE>, C::SMEM_BYTES);
  if (rc_attr != GS_OK) return rc_attr;
  int tiles_n = prm.p[0].ntiles;
  if (prm.combine == GS_COMBINE_CONCAT && prm.n_parts == 2) tiles_n += prm.p[1].ntiles;
  dim3 grid((unsigned)((prm.M + TC_BM - 1) / TC_BM), (unsigned)tiles_n);
  sage_gemm_tc_kernel<MODE><<<grid, TC_THREADS, C::SMEM_BYTES, st>>>(prm, ws);
  return launch_check("sage_gemm_tc_kernel");
}

int32_t sage_gemm_tc_pack(const gs_gemm_part* parts, int32_t n_parts, int32_t math, void* workspace, cudaStream_t st) {
  GS_REQUIRE(workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 127u) == 0,
             "gs_sage_gemm_pack: workspace must be non-NULL and 128-byte aligned");
  const int mode = mode_of(math);
  TcParams prm;
  fill_parts(prm, 0, parts, n_parts, mode);
  unsigned char* ws = (unsigned char*)workspace;
  if (mode == 0) return launch_pack<0>(prm, ws, st);
  if (mode == 1) return launch_pack<1>(prm, ws, st);
  return launch_pack<2>(prm, ws, st);
}

int32_t sage_gemm_tc(int64_t M, const gs_gemm_part* parts, const gs_gemm_row_ids* row_ids, int32_t n_parts, int32_t combine,
                     const float* bias, int32_t act, int32_t math, float* out, int64_t ldo, const void* workspace,
                     cudaStream_t st) {
  GS_REQUIRE(workspace != nullptr, "gs_sage_gemm: tensor-core math modes need the workspace (gs_sage_gemm_workspace_bytes)");
  GS_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 127u) == 0, "gs_sage_gemm: workspace must be 128-byte aligned");
  const int mode = mode_of(math);
  TcParams prm;
  fill_parts(prm, M, parts, n_parts, mode);
  for (int i = 0; row_ids && i < n_parts; ++i) prm.rid[i] = row_ids[i];
  prm.combine = combine;
  prm.bias = bias;
  prm.act = act;
  prm.out = out;
  prm.ldo = ldo;
  const unsigned char* ws = (const unsigned char*)workspace;
  if (mode == 0) return launch_tc<0>(prm, ws, st);
  if (mode == 1) return launch_tc<1>(prm, ws, st);
  return launch_tc<2>(prm, ws, st);
}

}  // namespace gs

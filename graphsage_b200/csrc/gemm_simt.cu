// fp32 CUDA-core GEMM for the aggregator contraction (GS_MATH_FP32_SIMT): the bring-up and
// cross-check path for the wgmma kernels in gemm_tc.cu.  Same math as
//   tf.matmul(neigh_means, neigh_weights), tf.matmul(self_vecs, self_weights),
//   tf.add_n / tf.concat, (+bias), act             reference graphsage/aggregators.py:51-64
//   Dense: matmul + bias + relu                      reference graphsage/layers.py:104-116
#include "common.cuh"

namespace gs {

struct GemmParts {
  gs_gemm_part p[2];
  int32_t n_parts;
  int32_t combine;
  gs_gemm_row_ids rid[2];   // part p's A rows by id (gs_sage_gemm_rows); n_ranges == 0: dense A
};

constexpr int BM = 64, BN = 64, BK = 16;

// grid.x = M tiles, grid.y = N tiles over the OUTPUT columns.  For CONCAT an N tile belongs to
// exactly one part (tiles never straddle: each part's columns are tiled separately).
__global__ void __launch_bounds__(256) sage_gemm_simt_kernel(int64_t M, const __grid_constant__ GemmParts gp,
                                                             const float* __restrict__ bias, int act,
                                                             float* __restrict__ out, int64_t ldo, int tiles_n0) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  int part_lo = 0, part_hi = gp.n_parts;  // parts summed into this tile
  int n0, col_off = 0;
  if (gp.combine == GS_COMBINE_CONCAT && gp.n_parts == 2) {
    if ((int)blockIdx.y < tiles_n0) { part_hi = 1; n0 = blockIdx.y * BN; }
    else { part_lo = 1; n0 = ((int)blockIdx.y - tiles_n0) * BN; col_off = gp.p[0].N; }
  } else {
    n0 = blockIdx.y * BN;
  }
  const int N = gp.p[part_lo].N;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int pi = part_lo; pi < part_hi; ++pi) {
    const gs_gemm_part& P = gp.p[pi];
    int64_t arow[4];                     // A row behind this thread's four A-tile rows (-1: zero row)
#pragma unroll
    for (int e = 0; e < 4; ++e) arow[e] = gemm_a_row(gp.rid[pi], M, m0 + ((threadIdx.x + e * 256) >> 4));
    for (int k0 = 0; k0 < P.K; k0 += BK) {
      // A tile: 64 rows x 16 k  (256 threads x 4 elements)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int idx = threadIdx.x + e * 256;
        int r = idx >> 4, kk = idx & 15;
        int gk = k0 + kk;
        As[kk][r] = (arow[e] >= 0 && gk < P.K) ? P.A[arow[e] * P.lda + gk] : 0.f;
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int idx = threadIdx.x + e * 256;
        int kk = idx >> 6, c = idx & 63;
        int gk = k0 + kk, gn = n0 + c;
        Bs[kk][c] = (gk < P.K && gn < N) ? P.B[(int64_t)gk * P.ldb + gn] : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int64_t gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[col_off + gn];
      if (act == GS_ACT_RELU) v = fmaxf(v, 0.f);
      out[gm * ldo + col_off + gn] = v;
    }
  }
}

int32_t sage_gemm_simt(int64_t M, const gs_gemm_part* parts, const gs_gemm_row_ids* row_ids, int32_t n_parts,
                       int32_t combine, const float* bias, int32_t act, float* out, int64_t ldo, cudaStream_t st) {
  GemmParts gp;
  memset(&gp, 0, sizeof(gp));
  gp.n_parts = n_parts;
  gp.combine = combine;
  for (int i = 0; i < n_parts; ++i) gp.p[i] = parts[i];
  for (int i = 0; row_ids && i < n_parts; ++i) gp.rid[i] = row_ids[i];
  int tiles_n0 = (parts[0].N + BN - 1) / BN;
  int tiles_n = tiles_n0;
  if (combine == GS_COMBINE_CONCAT && n_parts == 2) tiles_n += (parts[1].N + BN - 1) / BN;
  dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)tiles_n);
  sage_gemm_simt_kernel<<<grid, 256, 0, st>>>(M, gp, bias, act, out, ldo, tiles_n0);
  return launch_check("sage_gemm_simt_kernel");
}

}  // namespace gs

// Node2VecModel's skip-gram step (reference graphsage/models.py:459-501): lookups of the target / context tables, the
// biased logits, the sigmoid cross-entropy loss / B, the bias-free MRR affinities and the gradient of every lookup.
//
// The work of a step is small (B = 512 pairs, S = 20 shared negatives, d = 256: ~1 MB of rows and a [512 x 256] x [256 x 20]
// product, 5 MFLOP), so it is bound by latency, not by bandwidth or math: SIMT warps with shuffle reductions are the right
// tool and wgmma would not shorten it.  One warp per pair, 8 pairs per CTA:
//   skipgram_rows_kernel    - per pair: aff, neg_aff, the pair's loss term, gt and gc_pos rows; per CTA: the partial sums
//                             over its pairs of h_ij t_i (gc_neg) in ascending i (CTA k handles pair groups k, k + grid, ...)
//   skipgram_combine_kernel - gc_neg = the CTA partials added in CTA order; loss = the pair terms in a fixed order / B
// No atomics: the outputs are bit-identical on every call.  Contract: include/graphsage_b200.h.
#include "common.cuh"

namespace gs {
namespace {

constexpr int kRowsPerCta = 8;                 // one warp per pair
constexpr int kMaxCtas = 256;                  // fixed grid cap: the partial-sum layout does not depend on the GPU

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);   // every lane ends with the same bits
  return v;
}

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

struct Args {
  const float* target; int64_t ldt;
  const float* context; int64_t ldc;
  int64_t n_rows; int32_t d;
  const int32_t* batch1; const int32_t* batch2; int64_t B;
  const int32_t* neg; int32_t S;
  float* aff; float* neg_aff;
  float* gt; int64_t ldgt;
  float* gc_pos;
  int64_t ldgc;
  float* row_loss;           // workspace [B]
  float* partial;            // workspace [grid, S, d + 1]
};

__device__ __forceinline__ const float* row_of(const float* base, int64_t ld, int64_t n_rows, int32_t id) {
  return ((uint32_t)id < (uint64_t)n_rows) ? base + (int64_t)id * ld : nullptr;
}

__device__ __forceinline__ float col(const float* row, int c) { return row ? __ldg(row + c) : 0.f; }

__global__ void __launch_bounds__(kRowsPerCta * 32) skipgram_rows_kernel(const __grid_constant__ Args a) {
  __shared__ float h[kRowsPerCta][GS_MAX_UNIQUE_SAMPLED];
  __shared__ const float* trow[kRowsPerCta];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int d = a.d, S = a.S, width = d + 1;
  const float fB = (float)a.B;
  const int64_t n_groups = (a.B + kRowsPerCta - 1) / kRowsPerCta;
  float* part = a.partial + (int64_t)blockIdx.x * S * width;
  bool first = true;
  for (int64_t grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    const int64_t i = grp * kRowsPerCta + w;
    if (i < a.B) {
      const float* t = row_of(a.target, a.ldt, a.n_rows, a.batch1[i]);
      const float* c = row_of(a.context, a.ldc, a.n_rows, a.batch2[i]);
      // s = fmaf(t_q, c_q, s) per lane from +0 (and z below): nvcc contracts these two loops into FFMA chains.  They
      // are left as written because __fmaf_rn here allocates registers differently; the GPU test pins the bits.
      float s = 0.f;
      for (int q = lane; q < d; q += 32) s += col(t, q) * col(c, q);
      s = warp_sum(s);
      const float g = (sigmoid(s + (c ? c[d] : 0.f)) - 1.f) / fB;
      float loss = softplus(-(s + (c ? c[d] : 0.f)));
      for (int j = 0; j < S; ++j) {
        const float* n = row_of(a.context, a.ldc, a.n_rows, a.neg[j]);
        float z = 0.f;
        for (int q = lane; q < d; q += 32) z += col(t, q) * col(n, q);
        z = warp_sum(z);
        const float zb = z + (n ? n[d] : 0.f);
        loss += softplus(zb);
        if (lane == 0) {
          a.neg_aff[i * S + j] = z;
          h[w][j] = sigmoid(zb) / fB;
        }
      }
      if (lane == 0) {
        a.aff[i] = s;
        a.row_loss[i] = loss;
        trow[w] = t;
        a.gc_pos[i * a.ldgc + d] = g;
      }
      __syncwarp();
      for (int q = lane; q < d; q += 32) {
        float v = __fmul_rn(g, col(c, q));
        for (int j = 0; j < S; ++j) v = __fmaf_rn(h[w][j], col(row_of(a.context, a.ldc, a.n_rows, a.neg[j]), q), v);
        a.gt[i * a.ldgt + q] = v;
        a.gc_pos[i * a.ldgc + q] = __fmul_rn(g, col(t, q));
      }
    }
    __syncthreads();
    // this group's share of gc_neg[j, :] = sum_i h_ij [t_i, 1], pairs in ascending i, added to the CTA's running partial
    const int rows = (int)min((int64_t)kRowsPerCta, a.B - grp * kRowsPerCta);
    for (int e = threadIdx.x; e < S * width; e += blockDim.x) {
      const int j = e / width, q = e - j * width;
      float acc = first ? 0.f : part[e];
      for (int r = 0; r < rows; ++r) acc = __fmaf_rn(h[r][j], q < d ? col(trow[r], q) : 1.f, acc);
      part[e] = acc;
    }
    first = false;
    __syncthreads();
  }
}

// blocks 0 .. gridDim.x - 2: gc_neg elements; the last block: the loss
__global__ void __launch_bounds__(256) skipgram_combine_kernel(const float* __restrict__ partial, int32_t n_parts,
                                                               int32_t S, int32_t d, const float* __restrict__ row_loss,
                                                               int64_t B, float* __restrict__ gc_neg, int64_t ldgc,
                                                               float* __restrict__ loss) {
  const int width = d + 1;
  if (blockIdx.x == gridDim.x - 1) {
    if (threadIdx.x < 32) {
      // lane l adds pairs l, l + 32, ... in ascending order; the lanes are combined by the fixed butterfly
      float s = 0.f;
      for (int64_t i = threadIdx.x; i < B; i += 32) s += row_loss[i];
      s = warp_sum(s);
      if (threadIdx.x == 0) *loss = s / (float)B;
    }
    return;
  }
  const int64_t total = (int64_t)S * width;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)(gridDim.x - 1) * blockDim.x) {
    float acc = partial[e];
    for (int k = 1; k < n_parts; ++k) acc += partial[(int64_t)k * total + e];
    const int64_t j = e / width, q = e - j * width;
    gc_neg[j * ldgc + q] = acc;
  }
}

int64_t n_ctas(int64_t B) {
  const int64_t groups = (B + kRowsPerCta - 1) / kRowsPerCta;
  return groups < kMaxCtas ? groups : kMaxCtas;
}

}  // namespace
}  // namespace gs

extern "C" {

int64_t gs_skipgram_workspace_bytes(int64_t B, int32_t S, int32_t d) {
  if (B < 1 || S < 1 || d < 1) return -1;
  return (int64_t)(gs::align256((size_t)B * 4) + (size_t)gs::n_ctas(B) * S * (d + 1) * 4);
}

int32_t gs_skipgram_grad(const float* target, int64_t ldt, const float* context, int64_t ldc, int64_t n_rows, int32_t d,
                         const int32_t* batch1, const int32_t* batch2, int64_t B, const int32_t* neg, int32_t S, float* loss,
                         float* aff, float* neg_aff, float* gt, int64_t ldgt, float* gc_pos, float* gc_neg, int64_t ldgc,
                         void* workspace, int64_t workspace_bytes, void* stream) {
  GS_REQUIRE(B >= 1 && B < 0x7fffffffLL, "gs_skipgram_grad: need 1 <= B < 2^31 (got %lld)", (long long)B);
  GS_REQUIRE(S >= 1 && S <= GS_MAX_UNIQUE_SAMPLED, "gs_skipgram_grad: need 1 <= S <= %d (got %d)", GS_MAX_UNIQUE_SAMPLED, S);
  GS_REQUIRE(d >= 1, "gs_skipgram_grad: d must be >= 1");
  GS_REQUIRE(n_rows >= 0 && n_rows < 0x7fffffffLL, "gs_skipgram_grad: n_rows must be in [0, 2^31 - 1)");
  GS_REQUIRE(ldt >= d && ldc >= d + 1 && ldgt >= d && ldgc >= d + 1,
             "gs_skipgram_grad: need ldt >= d, ldc >= d + 1, ldgt >= d, ldgc >= d + 1");
  GS_REQUIRE(target && context && batch1 && batch2 && neg && loss && aff && neg_aff && gt && gc_pos && gc_neg,
             "gs_skipgram_grad: NULL pointer");
  const int64_t need = gs_skipgram_workspace_bytes(B, S, d);
  GS_REQUIRE(workspace != nullptr && workspace_bytes >= need, "gs_skipgram_grad: workspace of %lld bytes, %lld needed",
             (long long)workspace_bytes, (long long)need);
  cudaStream_t st = (cudaStream_t)stream;
  gs::Args a;
  a.target = target; a.ldt = ldt; a.context = context; a.ldc = ldc; a.n_rows = n_rows; a.d = d;
  a.batch1 = batch1; a.batch2 = batch2; a.B = B; a.neg = neg; a.S = S;
  a.aff = aff; a.neg_aff = neg_aff; a.gt = gt; a.ldgt = ldgt; a.gc_pos = gc_pos; a.ldgc = ldgc;
  a.row_loss = (float*)workspace;
  a.partial = (float*)((char*)workspace + gs::align256((size_t)B * 4));
  const int64_t grid = gs::n_ctas(B);
  gs::skipgram_rows_kernel<<<(unsigned)grid, gs::kRowsPerCta * 32, 0, st>>>(a);
  int32_t rc = gs::launch_check("skipgram_rows_kernel");
  if (rc != GS_OK) return rc;
  int64_t blocks = ((int64_t)S * (d + 1) + 255) / 256;
  const int64_t cap = (int64_t)gs::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  gs::skipgram_combine_kernel<<<(unsigned)(blocks + 1), 256, 0, st>>>(a.partial, (int32_t)grid, S, d, a.row_loss, B, gc_neg,
                                                                      ldgc, loss);
  return gs::launch_check("skipgram_combine_kernel");
}

}  // extern "C"

// One whole aggregator layer for a small number of output rows in a single launch (exact fp32 FFMA):
//   mean over the fanout -> self/neigh matmuls -> add | concat -> bias -> act -> row l2_normalize
//   reference graphsage/aggregators.py:43-64 (mean), :101-116 (gcn), graphsage/models.py:368.
// The last layers of the recursion have only B rows (512): a tensor-core tile pipeline is all
// latency there, and three or four launches cost more than the math.  Each CTA owns kRows output
// rows end to end, so the row norm is CTA-local.  Weights stream from L2 (they are shared by all CTAs).
#include "common.cuh"

namespace gs {

constexpr int LS_ROWS = 4;
constexpr int LS_THREADS = 512;

struct LsParams {
  const float* src;
  int64_t n_src_rows, pitch;
  int32_t F;
  gs_segment seg;
  int32_t include_self;
  gs_gemm_part p[2];
  int32_t n_parts, combine;
  const float* bias;
  int32_t act, l2norm;
  float* out;
  int64_t ldo;
  uint64_t* counter_dev;
  uint64_t counter_inc;
  int32_t vec;          // everything 16-byte friendly: 128-bit loads in both phases
  const uint8_t* src_i8;  // GS_I8ROW table (gs_sage_layer_small_i8; pitch in bytes), else NULL
};

__device__ __forceinline__ int64_t ls_clamp(int64_t id, int64_t n) { return (id < 0 || id >= n) ? n - 1 : id; }

// element c of source row `row`: the fp32 value, or (kI8) the dequantised fl(float(q_c) * s) of an int8 row
template <bool kI8>
__device__ __forceinline__ float ls_load(const LsParams& prm, int64_t row, int c) {
  if constexpr (kI8) {
    const uint8_t* r = prm.src_i8 + row * prm.pitch;
    return __fmul_rn((float)(int8_t)r[c], *reinterpret_cast<const float*>(r + ((prm.F + 3) & ~3)));
  } else {
    return prm.src[row * prm.pitch + c];
  }
}

// Latency is the enemy here (one CTA per SM, a few rows each): every load batch is made of
// independent loads (LS_ROWS rows x 5 neighbours in phase 1, 8 weight rows x K-slices in phase 2).
// kI8: the source is a GS_I8ROW table, read by the scalar phase 1 (its per-column sums are those of the vector one);
// phase 2 follows prm.vec as for the fp32 table
template <bool kI8>
__global__ void __launch_bounds__(LS_THREADS) sage_layer_small_kernel(const __grid_constant__ LsParams prm) {
  extern __shared__ float sm[];     // xs[LS_ROWS][F] | xm[LS_ROWS][F] | part[nslices][LS_ROWS][ncolp] | red[LS_ROWS][16]
  const int F = prm.F;
  float* xs = sm;
  float* xm = sm + LS_ROWS * F;
  const gs_segment& sg = prm.seg;
  const int k = sg.k;
  const int64_t row0 = (int64_t)blockIdx.x * LS_ROWS;
  // ---- phase 1: self rows and fanout means into shared memory
  if (!kI8 && prm.vec) {
    // thread = (row, float4 column); neighbours in independent batches of 5 x 128-bit loads
    const int f4 = F >> 2;
    for (int p = threadIdx.x; p < f4 * LS_ROWS; p += LS_THREADS) {
      const int r = p / f4, c4 = p - r * f4;
      const int64_t i = row0 + r;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f), sv = acc;
      if (i < sg.n) {
        const int64_t srow = ls_clamp(sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i, prm.n_src_rows);
        sv = ldg_nc_f4(reinterpret_cast<const float4*>(prm.src + srow * prm.pitch) + c4);
        for (int j0 = 0; j0 < k; j0 += 5) {
          float4 v[5];
#pragma unroll
          for (int u = 0; u < 5; ++u) {
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j0 + u < k) {
              const int64_t nr = ls_clamp(sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j0 + u] : sg.neigh_row0 + i * k + j0 + u,
                                          prm.n_src_rows);
              v[u] = ldg_nc_f4(reinterpret_cast<const float4*>(prm.src + nr * prm.pitch) + c4);
            }
          }
#pragma unroll
          for (int u = 0; u < 5; ++u) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
        }
        const float div = (float)(k + (prm.include_self ? 1 : 0));
        if (prm.include_self) { acc.x += sv.x; acc.y += sv.y; acc.z += sv.z; acc.w += sv.w; }
        acc.x /= div; acc.y /= div; acc.z /= div; acc.w /= div;
      }
      reinterpret_cast<float4*>(xs + r * F)[c4] = sv;
      reinterpret_cast<float4*>(xm + r * F)[c4] = acc;
    }
  } else
  for (int c = threadIdx.x; c < F; c += LS_THREADS) {
    float acc[LS_ROWS], sv[LS_ROWS];
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) {
      acc[r] = 0.f;
      const int64_t i = row0 + r;
      sv[r] = 0.f;
      if (i < sg.n) {
        const int64_t srow = ls_clamp(sg.self_ids ? (int64_t)sg.self_ids[i] : sg.self_row0 + i, prm.n_src_rows);
        sv[r] = ls_load<kI8>(prm, srow, c);
      }
    }
    for (int j0 = 0; j0 < k; j0 += 5) {
      float v[LS_ROWS][5];
#pragma unroll
      for (int r = 0; r < LS_ROWS; ++r) {
        const int64_t i = row0 + r;
#pragma unroll
        for (int u = 0; u < 5; ++u) {
          v[r][u] = 0.f;
          if (i < sg.n && j0 + u < k) {
            const int64_t nr = ls_clamp(sg.neigh_ids ? (int64_t)sg.neigh_ids[i * k + j0 + u] : sg.neigh_row0 + i * k + j0 + u,
                                        prm.n_src_rows);
            v[r][u] = ls_load<kI8>(prm, nr, c);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < LS_ROWS; ++r)
#pragma unroll
        for (int u = 0; u < 5; ++u) acc[r] += v[r][u];
    }
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) {
      float a = acc[r];
      if (prm.include_self) a += sv[r];
      a /= (float)(k + (prm.include_self ? 1 : 0));
      xs[r * F + c] = sv[r];
      xm[r * F + c] = (row0 + r < sg.n) ? a : 0.f;
    }
  }
  __syncthreads();
  // ---- phase 2: output columns, K split over `nslices` thread groups.
  //      CONCAT: columns [0, N0) use (xs, B0), [N0, N0+N1) use (xm, B1); ADD: every column sums both parts;
  //      single part: (xm, B0).
  const int N0 = prm.p[0].N;
  const int ntot = (prm.n_parts == 2 && prm.combine == GS_COMBINE_CONCAT) ? N0 + prm.p[1].N : N0;
  const int ncolp = (ntot + 31) & ~31;
  const int ncgp = prm.vec ? ((((ntot + 3) >> 2) + 31) & ~31) : 0;       // padded number of 4-column groups
  const int nslices = prm.vec ? (ncgp <= LS_THREADS ? LS_THREADS / ncgp : 1) : (ncolp <= LS_THREADS ? LS_THREADS / ncolp : 1);
  float* part = xm + LS_ROWS * F;                       // [nslices][LS_ROWS][ncolp]
  float* red = part + nslices * LS_ROWS * ncolp;        // [LS_ROWS][16]
  if (prm.vec) {
    // thread = (4-column group, K slice): per 4 k-steps 4 x LDG.128 of W rows, 8 x LDS.128 of x, 128 FMA
    const int ncg = ntot >> 2;
    const int sl = threadIdx.x / ncgp;
    const int cg0 = threadIdx.x - sl * ncgp;
    for (int cg = cg0; cg < ncg && sl < nslices; cg += (nslices == 1 ? LS_THREADS : ncgp)) {
      const int col = cg * 4;
      float4 acc[LS_ROWS];
#pragma unroll
      for (int r = 0; r < LS_ROWS; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int pi = 0; pi < prm.n_parts; ++pi) {
        int c = col;
        if (prm.n_parts == 2 && prm.combine == GS_COMBINE_CONCAT) {
          if ((pi == 0) != (col < N0)) continue;
          if (pi == 1) c = col - N0;
        }
        const gs_gemm_part& P = prm.p[pi];
        const float* x = (prm.n_parts == 1 || pi == 1) ? xm : xs;
        const float* w = P.B + c;
        const int kchunk = (((P.K + nslices - 1) / nslices) + 3) & ~3;
        const int kbeg = sl * kchunk, kend = min(P.K, kbeg + kchunk);   // K % 4 == 0 in the vector path
        float4 wn[4];                                    // software pipeline: next k-step's weights are in flight
        if (kbeg < kend) {
#pragma unroll
          for (int u = 0; u < 4; ++u) wn[u] = __ldg(reinterpret_cast<const float4*>(w + (int64_t)(kbeg + u) * P.ldb));
        }
        for (int kk = kbeg; kk < kend; kk += 4) {
          float4 wv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) wv[u] = wn[u];
          if (kk + 4 < kend) {
#pragma unroll
            for (int u = 0; u < 4; ++u) wn[u] = __ldg(reinterpret_cast<const float4*>(w + (int64_t)(kk + 4 + u) * P.ldb));
          }
#pragma unroll
          for (int r = 0; r < LS_ROWS; ++r) {
            const float4 xv = *reinterpret_cast<const float4*>(x + r * F + kk);
            acc[r].x = fmaf(xv.x, wv[0].x, acc[r].x); acc[r].y = fmaf(xv.x, wv[0].y, acc[r].y);
            acc[r].z = fmaf(xv.x, wv[0].z, acc[r].z); acc[r].w = fmaf(xv.x, wv[0].w, acc[r].w);
            acc[r].x = fmaf(xv.y, wv[1].x, acc[r].x); acc[r].y = fmaf(xv.y, wv[1].y, acc[r].y);
            acc[r].z = fmaf(xv.y, wv[1].z, acc[r].z); acc[r].w = fmaf(xv.y, wv[1].w, acc[r].w);
            acc[r].x = fmaf(xv.z, wv[2].x, acc[r].x); acc[r].y = fmaf(xv.z, wv[2].y, acc[r].y);
            acc[r].z = fmaf(xv.z, wv[2].z, acc[r].z); acc[r].w = fmaf(xv.z, wv[2].w, acc[r].w);
            acc[r].x = fmaf(xv.w, wv[3].x, acc[r].x); acc[r].y = fmaf(xv.w, wv[3].y, acc[r].y);
            acc[r].z = fmaf(xv.w, wv[3].z, acc[r].z); acc[r].w = fmaf(xv.w, wv[3].w, acc[r].w);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < LS_ROWS; ++r) *reinterpret_cast<float4*>(part + (sl * LS_ROWS + r) * ncolp + col) = acc[r];
      if (nslices > 1) break;
    }
  }
  const int slice = prm.vec ? nslices : (nslices == 1 ? 0 : threadIdx.x / ncolp);   // vec: scalar loop below is skipped
  const int col_step = nslices == 1 ? LS_THREADS : ncolp;
  for (int col = (nslices == 1 ? threadIdx.x : threadIdx.x % ncolp); col < ntot && slice < nslices; col += col_step) {
    float acc[LS_ROWS];
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) acc[r] = 0.f;
    for (int pi = 0; pi < prm.n_parts; ++pi) {
      int c = col;
      if (prm.n_parts == 2 && prm.combine == GS_COMBINE_CONCAT) {
        if ((pi == 0) != (col < N0)) continue;
        if (pi == 1) c = col - N0;
      }
      const gs_gemm_part& P = prm.p[pi];
      const float* x = (prm.n_parts == 1 || pi == 1) ? xm : xs;
      const float* w = P.B + c;
      const int kchunk = (((P.K + nslices - 1) / nslices) + 7) & ~7;
      const int kbeg = slice * kchunk, kend = min(P.K, kbeg + kchunk);
      int kk = kbeg;
      for (; kk + 8 <= kend; kk += 8) {
        float wv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) wv[u] = __ldg(w + (int64_t)(kk + u) * P.ldb);
#pragma unroll
        for (int u = 0; u < 8; ++u)
#pragma unroll
          for (int r = 0; r < LS_ROWS; ++r) acc[r] = fmaf(x[r * F + kk + u], wv[u], acc[r]);
      }
      for (; kk < kend; ++kk) {
        const float wv = __ldg(w + (int64_t)kk * P.ldb);
#pragma unroll
        for (int r = 0; r < LS_ROWS; ++r) acc[r] = fmaf(x[r * F + kk], wv, acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) part[(slice * LS_ROWS + r) * ncolp + col] = acc[r];
    if (nslices > 1) break;                              // one (column, slice) per thread when K is sliced
  }
  __syncthreads();
  // ---- phase 3: reduce the K slices, bias, activation, row sum of squares, store
  float ss[LS_ROWS];
#pragma unroll
  for (int r = 0; r < LS_ROWS; ++r) ss[r] = 0.f;
  for (int col = threadIdx.x; col < ntot; col += LS_THREADS) {
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) {
      float v = 0.f;
      for (int s2 = 0; s2 < nslices; ++s2) v += part[(s2 * LS_ROWS + r) * ncolp + col];
      if (prm.bias) v += prm.bias[col];
      if (prm.act == GS_ACT_RELU) v = fmaxf(v, 0.f);
      ss[r] += v * v;
      part[r * ncolp + col] = v;                         // slice-0 slot now holds the finished value (same thread re-reads it)
    }
  }
  float inv[LS_ROWS];
#pragma unroll
  for (int r = 0; r < LS_ROWS; ++r) inv[r] = 1.f;
  if (prm.l2norm) {
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) {
      float t = ss[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if ((threadIdx.x & 31) == 0) red[r * 16 + (threadIdx.x >> 5)] = t;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < LS_THREADS / 32; ++w) tot += red[r * 16 + w];
      inv[r] = 1.0f / sqrtf(fmaxf(tot, 1e-12f));
    }
  }
  for (int col = threadIdx.x; col < ntot; col += LS_THREADS) {
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r)
      if (row0 + r < sg.n) prm.out[(sg.out_row0 + row0 + r) * prm.ldo + col] = part[r * ncolp + col] * inv[r];
  }
  if (prm.counter_dev != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *prm.counter_dev += prm.counter_inc;
}

}  // namespace gs

static int32_t sage_layer_small(const void* src, bool i8, int64_t n_src_rows, int32_t F, int64_t pitch,
                                const gs_segment* segment_host, int32_t include_self, const gs_gemm_part* parts_host,
                                int32_t n_parts, int32_t combine, const float* bias, int32_t act, int32_t l2_normalize, float* out,
                                int64_t ldo, uint64_t* counter_dev, uint64_t counter_inc, void* stream) {
  GS_REQUIRE(src && segment_host && parts_host && out, "gs_sage_layer_small: NULL pointer");
  GS_REQUIRE(n_parts == 1 || n_parts == 2, "gs_sage_layer_small: n_parts=%d", n_parts);
  GS_REQUIRE(F >= 1 && F <= 2048 && pitch >= F && n_src_rows > 0, "gs_sage_layer_small: F=%d (max 2048) / pitch", F);
  if (i8)
    GS_REQUIRE(pitch % 16 == 0 && pitch >= gs_i8row_pitch(F) && (reinterpret_cast<uintptr_t>(src) & 15u) == 0,
               "gs_sage_layer_small_i8: needs 16-byte aligned rows of pitch %% 16 == 0 and >= gs_i8row_pitch(F)");
  GS_REQUIRE(segment_host->k >= 1 && segment_host->n >= 0, "gs_sage_layer_small: bad segment");
  GS_REQUIRE(combine == GS_COMBINE_ADD || combine == GS_COMBINE_CONCAT, "gs_sage_layer_small: combine=%d", combine);
  GS_REQUIRE(act == GS_ACT_NONE || act == GS_ACT_RELU, "gs_sage_layer_small: act=%d", act);
  gs::LsParams prm;
  memset(&prm, 0, sizeof(prm));
  int ntot = 0;
  for (int i = 0; i < n_parts; ++i) {
    GS_REQUIRE(parts_host[i].B && parts_host[i].K == F && parts_host[i].N >= 1 && parts_host[i].ldb >= parts_host[i].N,
               "gs_sage_layer_small: part %d must have K == F (%d) and a valid B", i, F);
    prm.p[i] = parts_host[i];
  }
  if (n_parts == 2 && combine == GS_COMBINE_ADD)
    GS_REQUIRE(parts_host[0].N == parts_host[1].N, "gs_sage_layer_small: ADD needs equal N");
  ntot = parts_host[0].N + ((n_parts == 2 && combine == GS_COMBINE_CONCAT) ? parts_host[1].N : 0);
  GS_REQUIRE(ntot <= 1024 && ldo >= ntot, "gs_sage_layer_small: output width %d (max 1024) / ldo", ntot);
  if (segment_host->n == 0) return GS_OK;
  prm.src = i8 ? nullptr : (const float*)src; prm.src_i8 = i8 ? (const uint8_t*)src : nullptr;
  prm.n_src_rows = n_src_rows; prm.pitch = pitch; prm.F = F;
  prm.seg = *segment_host; prm.include_self = include_self;
  prm.n_parts = n_parts; prm.combine = combine; prm.bias = bias; prm.act = act; prm.l2norm = l2_normalize;
  prm.out = out; prm.ldo = ldo; prm.counter_dev = counter_dev; prm.counter_inc = counter_inc;
  // an int8 table stands for its dequantised fp32 twin with an aligned pitch that is a multiple of 4 floats, so only the
  // conditions that do not depend on the source layout decide here
  bool vec = (F % 4 == 0) && (i8 || ((pitch % 4 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0))) && (ntot % 4 == 0) &&
             (parts_host[0].N % 4 == 0);
  for (int i = 0; i < n_parts; ++i)
    vec = vec && (parts_host[i].ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(parts_host[i].B) & 15u) == 0);
  prm.vec = vec ? 1 : 0;
  const int ncolp = (ntot + 31) & ~31;
  const int ncgp = (((ntot + 3) / 4) + 31) & ~31;
  const int nslices = vec ? (ncgp <= gs::LS_THREADS ? gs::LS_THREADS / ncgp : 1)
                          : (ncolp <= gs::LS_THREADS ? gs::LS_THREADS / ncolp : 1);
  const size_t smem = (size_t)(2 * gs::LS_ROWS * F + nslices * gs::LS_ROWS * ncolp + gs::LS_ROWS * 16) * sizeof(float);
  GS_REQUIRE(smem <= 200 * 1024, "gs_sage_layer_small: needs %zu bytes of shared memory", smem);
  const void* kernel = i8 ? (const void*)gs::sage_layer_small_kernel<true> : (const void*)gs::sage_layer_small_kernel<false>;
  {
    const int32_t rc_attr = gs::ensure_dyn_smem(kernel, 200 * 1024);
    if (rc_attr != GS_OK) return rc_attr;
  }
  unsigned blocks = (unsigned)((segment_host->n + gs::LS_ROWS - 1) / gs::LS_ROWS);
  if (i8)
    gs::sage_layer_small_kernel<true><<<blocks, gs::LS_THREADS, smem, (cudaStream_t)stream>>>(prm);
  else
    gs::sage_layer_small_kernel<false><<<blocks, gs::LS_THREADS, smem, (cudaStream_t)stream>>>(prm);
  return gs::launch_check("sage_layer_small_kernel");
}

extern "C" int32_t gs_sage_layer_small(const float* src, int64_t n_src_rows, int32_t F, int64_t pitch,
                                       const gs_segment* segment_host, int32_t include_self,
                                       const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine, const float* bias,
                                       int32_t act, int32_t l2_normalize, float* out, int64_t ldo, uint64_t* counter_dev,
                                       uint64_t counter_inc, void* stream) {
  return sage_layer_small(src, false, n_src_rows, F, pitch, segment_host, include_self, parts_host, n_parts, combine, bias, act,
                          l2_normalize, out, ldo, counter_dev, counter_inc, stream);
}

extern "C" int32_t gs_sage_layer_small_i8(const void* src, int64_t n_src_rows, int32_t F, int64_t pitch,
                                          const gs_segment* segment_host, int32_t include_self,
                                          const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine, const float* bias,
                                          int32_t act, int32_t l2_normalize, float* out, int64_t ldo, uint64_t* counter_dev,
                                          uint64_t counter_inc, void* stream) {
  return sage_layer_small(src, true, n_src_rows, F, pitch, segment_host, include_self, parts_host, n_parts, combine, bias, act,
                          l2_normalize, out, ldo, counter_dev, counter_inc, stream);
}

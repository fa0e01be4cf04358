// SeqAggregator's recurrence (reference graphsage/aggregators.py:363-449): TF 1.8's BasicLSTMCell run by dynamic_rnn over
// the sampled neighbours of every node, with the reference's length rule.  The input projection P = X·W_x + b is a plain
// GEMM (gs_sage_gemm) and the weight gradients are library matmuls; what is here is the part that is sequential in the
// fanout:
//   seq_lengths_kernel   - len[i] = max(1, number of rows of sequence i with a non-zero element)
//   lstm_forward_kernel  - z_t = P_t + h_{t-1}·W_h, the cell update, h after len_i steps (+ what the backward needs)
//   lstm_backward_kernel - backpropagation through time to dZ, with dh_{t-1} = dz_t·W_hᵀ carried inside the kernel
//
// fp32 FFMA on the CUDA cores.  A CTA owns a tile of S sequences and runs 512 threads: thread (g, u) owns hidden unit u of
// the kSeqPerThread sequences of group g, so the four gate columns of unit u and the cell state c[s][u] stay in the thread
// and the cell update needs no exchange.  h goes through shared memory (double-buffered, unit-major so one float4 load
// gives four sequences), W_h is read from L2 (256 KB at H = 128, 1 MB at H = 256) and is shared by the CTA's groups
// through L1.  S = 32 at H = 128 and 16 at H = 256: 160 / 320 CTAs at n = 5,120.  Each CTA reads all of W_h once per step,
// so the L2 traffic per FLOP falls as S grows; the forward's 113 registers leave room for one CTA per SM.
// Every sequence of a tile steps in lock-step over t < (longest length in the tile) with per-sequence masking, so the
// barriers are uniform; the loop bounds are read on the device (graph-capturable).  No atomics, no allocation, no
// synchronisation: two runs are bit-identical.  Contract: include/graphsage_b200.h.
#include "common.cuh"

namespace gs {
namespace {

constexpr int kThreads = 512;
constexpr int kSeqPerThread = 8;

template <int H>
struct SeqTile {
  static constexpr int kGroups = kThreads / H;               // 4 at H = 128, 2 at H = 256
  static constexpr int kSeqs = kGroups * kSeqPerThread;      // sequences per CTA
  static constexpr int kPitch = kSeqs + 4;                   // padded: the float4 stores of a quarter-warp hit 32 banks
};

__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// One warp per sequence.  -0.0f != 0.0f is false, so negative zeros count as zero (tf.sign(reduce_max(abs(.)))).
__global__ void __launch_bounds__(256) seq_lengths_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int32_t k,
                                                          int32_t K, int32_t* __restrict__ len) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); i < n; i += (int64_t)gridDim.x * 8) {
    int used = 0;
    for (int j = 0; j < k; ++j) {
      const float* row = x + (i * k + j) * ldx;
      bool nz = false;
      for (int c = lane; c < K; c += 32) nz |= row[c] != 0.f;
      used += __any_sync(0xffffffffu, nz) ? 1 : 0;
    }
    if (lane == 0) len[i] = used > 1 ? used : 1;
  }
}

// Sets lens[] (len clamped to [0, k]; 0 for rows past n) and returns the tile's longest length.  Ends with a barrier.
// The clamp below 0 keeps `L - 1` (the backward's dh_last step) free of overflow for any int32 length.
template <int S>
__device__ __forceinline__ int load_tile_lengths(const int32_t* __restrict__ len, int64_t s0, int64_t n, int32_t k,
                                                 int* lens, int* tile_len) {
  if (threadIdx.x < S) {
    const int64_t i = s0 + threadIdx.x;
    const int L = i < n ? len[i] : 0;
    lens[threadIdx.x] = L < 0 ? 0 : L < k ? L : k;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int m = 0;
    for (int s = 0; s < S; ++s) m = lens[s] > m ? lens[s] : m;
    *tile_len = m;
  }
  __syncthreads();
  return *tile_len;
}

struct FwdArgs {
  const float* P; int64_t ldp;
  const float* Wh; int64_t ldw;
  const int32_t* len;
  int64_t n; int32_t k;
  float* h_last; int64_t ldh;
  float* gates; int64_t ldg;       // optional (training)
  float* c; int64_t ldc;           // optional
  float* h_prev; int64_t ldhp;     // optional
};

template <int H>
__global__ void __launch_bounds__(kThreads) lstm_forward_kernel(const __grid_constant__ FwdArgs a) {
  constexpr int S = SeqTile<H>::kSeqs, SP = SeqTile<H>::kPitch, SPT = kSeqPerThread;
  __shared__ __align__(16) float hs[2][H][SP];   // h_{t-1} of the tile, unit-major
  __shared__ int lens[S];
  __shared__ int tile_len_s;
  const int u = threadIdx.x % H, my0 = (threadIdx.x / H) * SPT;
  const int64_t s0 = (int64_t)blockIdx.x * S;
  for (int e = threadIdx.x; e < H * SP; e += kThreads) (&hs[0][0][0])[e] = 0.f;
  const int tl = load_tile_lengths<S>(a.len, s0, a.n, a.k, lens, &tile_len_s);
  const bool save = a.gates != nullptr;
  int L[SPT];
  float c[SPT], h[SPT];
#pragma unroll
  for (int q = 0; q < SPT; ++q) {
    L[q] = lens[my0 + q];
    c[q] = 0.f;
    h[q] = 0.f;
  }
  int b = 0;
  for (int t = 0; t < a.k; ++t) {
    if (t >= tl) {                                     // CTA-uniform: every sequence of the tile has ended
      if (!save) break;
#pragma unroll
      for (int q = 0; q < SPT; ++q) {
        const int64_t i = s0 + my0 + q;
        if (i >= a.n) continue;
        const int64_t row = i * a.k + t;
#pragma unroll
        for (int g = 0; g < 4; ++g) a.gates[row * a.ldg + g * H + u] = 0.f;
        a.c[row * a.ldc + u] = 0.f;
        a.h_prev[row * a.ldhp + u] = 0.f;
      }
      continue;
    }
    float acc[SPT][4];
#pragma unroll
    for (int q = 0; q < SPT; ++q) {
      const float* p = a.P + ((s0 + my0 + q) * a.k + t) * a.ldp + u;
      const bool on = t < L[q];
#pragma unroll
      for (int g = 0; g < 4; ++g) acc[q][g] = on ? __ldg(p + g * H) : 0.f;
    }
#pragma unroll 4
    for (int m = 0; m < H; ++m) {
      const float* w = a.Wh + (int64_t)m * a.ldw + u;
      const float w0 = __ldg(w), w1 = __ldg(w + H), w2 = __ldg(w + 2 * H), w3 = __ldg(w + 3 * H);
      const float4 ha = *reinterpret_cast<const float4*>(&hs[b][m][my0]);
      const float4 hb = *reinterpret_cast<const float4*>(&hs[b][m][my0 + 4]);
      const float hv[SPT] = {ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w};
#pragma unroll
      for (int q = 0; q < SPT; ++q) {
        acc[q][0] = fmaf(hv[q], w0, acc[q][0]);
        acc[q][1] = fmaf(hv[q], w1, acc[q][1]);
        acc[q][2] = fmaf(hv[q], w2, acc[q][2]);
        acc[q][3] = fmaf(hv[q], w3, acc[q][3]);
      }
    }
#pragma unroll
    for (int q = 0; q < SPT; ++q) {
      const bool on = t < L[q];
      const float ig = sigmoid(acc[q][0]), jg = tanhf(acc[q][1]), fg = sigmoid(acc[q][2] + 1.f), og = sigmoid(acc[q][3]);
      const float cn = c[q] * fg + ig * jg;
      const float hn = tanhf(cn) * og;
      const int64_t i = s0 + my0 + q;
      if (save && i < a.n) {
        const int64_t row = i * a.k + t;
        float* gr = a.gates + row * a.ldg + u;
        gr[0] = on ? ig : 0.f;
        gr[H] = on ? jg : 0.f;
        gr[2 * H] = on ? fg : 0.f;
        gr[3 * H] = on ? og : 0.f;
        a.c[row * a.ldc + u] = on ? cn : 0.f;
        a.h_prev[row * a.ldhp + u] = on ? h[q] : 0.f;
      }
      if (on) {                                        // past its length a sequence's state is frozen
        c[q] = cn;
        h[q] = hn;
      }
    }
    *reinterpret_cast<float4*>(&hs[b ^ 1][u][my0]) = make_float4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<float4*>(&hs[b ^ 1][u][my0 + 4]) = make_float4(h[4], h[5], h[6], h[7]);
    __syncthreads();
    b ^= 1;
  }
#pragma unroll
  for (int q = 0; q < SPT; ++q) {
    const int64_t i = s0 + my0 + q;
    if (i < a.n) a.h_last[i * a.ldh + u] = h[q];
  }
}

struct BwdArgs {
  const float* dh_last; int64_t lddh;
  const float* gates; int64_t ldg;
  const float* c; int64_t ldc;
  const int32_t* len;
  const float* Wh; int64_t ldw;
  int64_t n; int32_t k;
  float* dZ; int64_t ldz;
};

template <int H>
__global__ void __launch_bounds__(kThreads) lstm_backward_kernel(const __grid_constant__ BwdArgs a) {
  constexpr int S = SeqTile<H>::kSeqs, SP = SeqTile<H>::kPitch, SPT = kSeqPerThread;
  extern __shared__ __align__(16) float dzs[];   // [4H][SP]: dz of the tile at step t, column-major in the sequences
  __shared__ int lens[S];
  __shared__ int tile_len_s;
  const int u = threadIdx.x % H, my0 = (threadIdx.x / H) * SPT;
  const int64_t s0 = (int64_t)blockIdx.x * S;
  const int tl = load_tile_lengths<S>(a.len, s0, a.n, a.k, lens, &tile_len_s);
  int L[SPT];
  float dh[SPT], dc[SPT];                          // dh_t carried from step t + 1 (through W_h), dc_t carried likewise
#pragma unroll
  for (int q = 0; q < SPT; ++q) {
    L[q] = lens[my0 + q];
    dh[q] = 0.f;
    dc[q] = 0.f;
  }
  const float* wrow = a.Wh + (int64_t)u * a.ldw;
  for (int t = a.k - 1; t >= 0; --t) {
    if (t >= tl) {                                   // CTA-uniform: past every length of the tile
#pragma unroll
      for (int q = 0; q < SPT; ++q) {
        const int64_t i = s0 + my0 + q;
        if (i >= a.n) continue;
        float* zr = a.dZ + (i * a.k + t) * a.ldz + u;
#pragma unroll
        for (int g = 0; g < 4; ++g) zr[g * H] = 0.f;
      }
      continue;
    }
    float z[4][SPT];
#pragma unroll
    for (int q = 0; q < SPT; ++q) {
      const int64_t i = s0 + my0 + q;
      const bool on = t < L[q];
      float zi = 0.f, zj = 0.f, zf = 0.f, zo = 0.f;
      if (on) {
        const int64_t row = i * a.k + t;
        const float* gr = a.gates + row * a.ldg + u;
        const float ig = gr[0], jg = gr[H], fg = gr[2 * H], og = gr[3 * H];
        const float ct = a.c[row * a.ldc + u];
        const float cp = t > 0 ? a.c[(row - 1) * a.ldc + u] : 0.f;
        const float d = dh[q] + (t == L[q] - 1 ? a.dh_last[i * a.lddh + u] : 0.f);
        const float tc = tanhf(ct);
        zo = d * tc * og * (1.f - og);
        const float dct = dc[q] + d * og * (1.f - tc * tc);
        zi = dct * jg * ig * (1.f - ig);
        zj = dct * ig * (1.f - jg * jg);
        zf = dct * cp * fg * (1.f - fg);
        dc[q] = dct * fg;
      }
      z[0][q] = zi;
      z[1][q] = zj;
      z[2][q] = zf;
      z[3][q] = zo;
      if (i < a.n) {
        float* zr = a.dZ + (i * a.k + t) * a.ldz + u;
#pragma unroll
        for (int g = 0; g < 4; ++g) zr[g * H] = z[g][q];
      }
    }
    if (t == 0) break;                               // dh_{-1} is not needed
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      float* dst = dzs + (g * H + u) * SP + my0;
      *reinterpret_cast<float4*>(dst) = make_float4(z[g][0], z[g][1], z[g][2], z[g][3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(z[g][4], z[g][5], z[g][6], z[g][7]);
    }
    __syncthreads();
    // dh_{t-1}[s][u] = sum over the 4H columns of dz_t[s][col] * W_h[u][col], columns ascending
    float acc[SPT];
#pragma unroll
    for (int q = 0; q < SPT; ++q) acc[q] = 0.f;
#pragma unroll 2
    for (int col = 0; col < 4 * H; col += 4) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(wrow + col));
      const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const float* zc = dzs + (col + cc) * SP + my0;
        const float4 za = *reinterpret_cast<const float4*>(zc);
        const float4 zb = *reinterpret_cast<const float4*>(zc + 4);
        const float zv[SPT] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
#pragma unroll
        for (int q = 0; q < SPT; ++q) acc[q] = fmaf(zv[q], wv[cc], acc[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < SPT; ++q) dh[q] = acc[q];
    __syncthreads();                                 // dzs is rewritten by the next step
  }
}

template <int H>
int64_t n_tiles(int64_t n) {
  return (n + SeqTile<H>::kSeqs - 1) / SeqTile<H>::kSeqs;
}

template <int H>
int32_t launch_forward(const FwdArgs& a, cudaStream_t st) {
  lstm_forward_kernel<H><<<(unsigned)n_tiles<H>(a.n), kThreads, 0, st>>>(a);
  return launch_check("lstm_forward_kernel");
}

template <int H>
int32_t launch_backward(const BwdArgs& a, cudaStream_t st) {
  const int smem = 4 * H * SeqTile<H>::kPitch * (int)sizeof(float);
  int32_t rc = ensure_dyn_smem((const void*)lstm_backward_kernel<H>, smem);
  if (rc != GS_OK) return rc;
  lstm_backward_kernel<H><<<(unsigned)n_tiles<H>(a.n), kThreads, smem, st>>>(a);
  return launch_check("lstm_backward_kernel");
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace
}  // namespace gs

extern "C" {

int32_t gs_seq_lengths(const float* x, int64_t ldx, int64_t n, int32_t k, int32_t K, int32_t* len, void* stream) {
  GS_REQUIRE(n >= 0 && n < 0x7fffffffLL && k >= 1 && K >= 0 && ldx >= K, "gs_seq_lengths: bad sizes");
  if (n == 0) return GS_OK;
  GS_REQUIRE(x && len, "gs_seq_lengths: NULL pointer");
  int64_t blocks = (n + 7) / 8;
  const int64_t cap = (int64_t)gs::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  gs::seq_lengths_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, ldx, n, k, K, len);
  return gs::launch_check("seq_lengths_kernel");
}

int32_t gs_lstm_forward(const float* P, int64_t ldp, const float* Wh, int64_t ldw, const int32_t* len, int64_t n, int32_t k,
                        int32_t H, float* h_last, int64_t ldh, float* gates, int64_t ldg, float* c, int64_t ldc,
                        float* h_prev, int64_t ldhp, void* stream) {
  GS_REQUIRE(H == 128 || H == 256, "gs_lstm_forward: H must be 128 or 256 (got %d)", H);
  GS_REQUIRE(n >= 0 && n < 0x7fffffffLL && k >= 1, "gs_lstm_forward: bad sizes");
  GS_REQUIRE(ldp >= 4 * H && ldw >= 4 * H && ldh >= H, "gs_lstm_forward: need ldp, ldw >= 4H and ldh >= H");
  const bool save = gates != nullptr;
  GS_REQUIRE(save == (c != nullptr) && save == (h_prev != nullptr),
             "gs_lstm_forward: gates, c and h_prev are given together or not at all");
  GS_REQUIRE(!save || (ldg >= 4 * H && ldc >= H && ldhp >= H), "gs_lstm_forward: need ldg >= 4H, ldc and ldhp >= H");
  if (n == 0) return GS_OK;
  GS_REQUIRE(P && Wh && len && h_last, "gs_lstm_forward: NULL pointer");
  gs::FwdArgs a{P, ldp, Wh, ldw, len, n, k, h_last, ldh, gates, ldg, c, ldc, h_prev, ldhp};
  cudaStream_t st = (cudaStream_t)stream;
  return H == 128 ? gs::launch_forward<128>(a, st) : gs::launch_forward<256>(a, st);
}

int32_t gs_lstm_backward(const float* dh_last, int64_t lddh, const float* gates, int64_t ldg, const float* c, int64_t ldc,
                         const int32_t* len, const float* Wh, int64_t ldw, int64_t n, int32_t k, int32_t H, float* dZ,
                         int64_t ldz, void* stream) {
  GS_REQUIRE(H == 128 || H == 256, "gs_lstm_backward: H must be 128 or 256 (got %d)", H);
  GS_REQUIRE(n >= 0 && n < 0x7fffffffLL && k >= 1, "gs_lstm_backward: bad sizes");
  GS_REQUIRE(lddh >= H && ldg >= 4 * H && ldc >= H && ldw >= 4 * H && ldz >= 4 * H, "gs_lstm_backward: bad leading dimensions");
  if (n == 0) return GS_OK;
  GS_REQUIRE(dh_last && gates && c && len && Wh && dZ, "gs_lstm_backward: NULL pointer");
  GS_REQUIRE(ldw % 4 == 0 && gs::aligned16(Wh), "gs_lstm_backward: W_h rows must be 16-byte aligned (ldw %% 4 == 0)");
  gs::BwdArgs a{dh_last, lddh, gates, ldg, c, ldc, len, Wh, ldw, n, k, dZ, ldz};
  cudaStream_t st = (cudaStream_t)stream;
  return H == 128 ? gs::launch_backward<128>(a, st) : gs::launch_backward<256>(a, st);
}

}  // extern "C"

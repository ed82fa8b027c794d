// Skinny-M FP8 weight-only GEMM for decoding:  y[M, N] = x[M, K] * (q[N, K] * inv[N])^T,  M <= 64.
//
// x and y are bf16, q holds e4m3 weights with one power-of-two dequantisation factor per output row (inv, fp32; see
// ops/fp8w.py for the quantisation rule).  At decode shapes the GEMM is a stream over the weights, so the kernel is laid out
// to keep every SM reading them:
//
//   * A and B are swapped: the weight rows (output channels) are the m16n8k16 M dimension and the tokens the N dimension,
//     padded to NT x 8.  A CTA owns 64 weight rows; its four warps split the CTA's K range (NT <= 4) or two warps own 32 rows
//     each and pairs split the K range (NT > 4, where the accumulators of 64 rows would not fit).
//   * Each lane reads 16 consecutive e4m3 bytes of a weight row per 64-wide k chunk (one 16-byte non-allocating load per row,
//     the next chunk's loads in flight under this chunk's MMAs) and converts them exactly to bf16 register A fragments
//     (e4m3 -> f16 -> f32 -> bf16 is exact).  The k index of the fragments is permuted so that those 16 bytes are exactly
//     the lane's A elements of four k16 steps, and its x operand is 32 consecutive bytes of one token row: no shuffles, no
//     shared memory on the main loop.  The permutation is the same for A and B, so the dot products are unchanged.
//   * Split-K across CTAs (grid.y) covers the GPU when N / 64 tiles are too few.  Partial sums are fp32; the warps of a CTA
//     are summed through shared memory in warp order, the CTAs of a tile through a workspace in split order by the CTA that
//     arrives last (an integer arrival counter, reset by that CTA).  No float atomics: results are bit-identical from run
//     to run, in a CUDA graph or not.
//   * Epilogue: inv[n] is applied in fp32 before the one bf16 rounding.  With the SwiGLU epilogue a tile holds 32 gate rows
//     and the matching 32 up rows (N = 2I, I % 32 == 0) and also writes act = silu(g) * u from the bf16-rounded g, u, as the
//     bf16 SwiGLU GEMM does (gemm_sm90.cu, kSwiGLU).
#include "common.cuh"
#include "fp8_rows.cuh"

using namespace odb;

namespace {

constexpr int kRows = 64;         // weight rows per CTA
constexpr int kChunk = 64;        // k per warp iteration
constexpr int kThreads = 128;
constexpr int kRS = kRows + 4;    // shared-memory stride (floats) of one token's 64 row sums: conflict-free fragment stores
constexpr int kMaxM = 64;

struct Args {
  const __nv_bfloat16* x;
  long long ldx;
  const uint8_t* q;
  const float* inv;
  __nv_bfloat16* y;
  long long ldy;
  __nv_bfloat16* act;             // SwiGLU: act [M, I] (row stride I)
  float* ws;                      // split-K partials [splits][tiles][NT * 8][64]
  int* counters;                  // split-K arrival counters [tiles], zero between launches
  int M, N, K, I, splits;
};

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t word(const uint4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// weight row of tile row r: plain tiles are 64 consecutive rows; SwiGLU tiles are 32 gate rows then the matching up rows
template <bool SWIGLU>
__device__ __forceinline__ int weight_row(const Args& p, int tile, int r) {
  if constexpr (!SWIGLU) return tile * kRows + r;
  return r < kRows / 2 ? tile * (kRows / 2) + r : p.I + tile * (kRows / 2) + (r - kRows / 2);
}

template <int NT, bool SWIGLU>
__global__ void __launch_bounds__(kThreads) fp8w_gemm_kernel(const Args p) {
  constexpr int WR = NT > 4 ? 2 : 1;     // warps along the rows
  constexpr int WK = 4 / WR;             // warps along K
  constexpr int MT = 4 / WR;             // m16 tiles per warp
  constexpr int MP = NT * 8;             // padded token count
  extern __shared__ float red[];         // [WK][MP][kRS]
  __shared__ int is_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tig = lane & 3;
  const int wr = warp / WK, wk = warp % WK;
  const int tile = blockIdx.x, split = blockIdx.y, tiles = gridDim.x;
  const int KC = p.K / kChunk;
  const int c_lo = (int)((long long)KC * split / p.splits), c_hi = (int)((long long)KC * (split + 1) / p.splits);

  const uint8_t* wp[MT][2];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      wp[mt][h] = p.q + (size_t)weight_row<SWIGLU>(p, tile, wr * 16 * MT + mt * 16 + g + 8 * h) * p.K + tig * 16;
  const __nv_bfloat16* xp[NT];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) xp[nt] = p.x + (size_t)min(nt * 8 + g, p.M - 1) * p.ldx + tig * 16;

  float acc[MT][NT][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;

  uint4 wcur[MT][2], wnext[MT][2];
  int c = c_lo + wk;
  if (c < c_hi) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) wcur[mt][h] = ld_nc_v4(wp[mt][h] + (size_t)c * kChunk);
  }
  for (; c < c_hi; c += WK) {
    if (c + WK < c_hi) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) wnext[mt][h] = ld_nc_v4(wp[mt][h] + (size_t)(c + WK) * kChunk);
    }
    // A fragments of the four k16 steps: word s of a row's 16 bytes holds the lane's elements of step s
    uint32_t a[MT][4][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const uint32_t lo = word(wcur[mt][0], s), hi = word(wcur[mt][1], s);
        a[mt][s][0] = e4m3x2_to_bf16x2(lo);
        a[mt][s][1] = e4m3x2_to_bf16x2(hi);
        a[mt][s][2] = e4m3x2_to_bf16x2(lo >> 16);
        a[mt][s][3] = e4m3x2_to_bf16x2(hi >> 16);
      }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      uint4 x0 = make_uint4(0, 0, 0, 0), x1 = x0;
      if (nt * 8 + g < p.M) {
        x0 = ld_v4(xp[nt] + (size_t)c * kChunk);
        x1 = ld_v4(xp[nt] + (size_t)c * kChunk + 8);
      }
      const uint32_t xw[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
      for (int s = 0; s < 4; ++s)
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) mma_bf16_16816(acc[mt][nt], a[mt][s], xw[2 * s], xw[2 * s + 1]);
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) wcur[mt][h] = wnext[mt][h];
  }

  // ---- the CTA's sum: the WK warps' partials through shared memory, in warp order
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = wr * 16 * MT + mt * 16 + g + 8 * (i >> 1), tok = nt * 8 + 2 * tig + (i & 1);
        red[(wk * MP + tok) * kRS + row] = acc[mt][nt][i];
      }
  __syncthreads();
  float* part = p.ws + ((size_t)split * tiles + tile) * MP * kRows;
  for (int idx = threadIdx.x; idx < MP * kRows; idx += kThreads) {
    const int tok = idx / kRows, r = idx % kRows;
    float v = red[tok * kRS + r];
#pragma unroll
    for (int w = 1; w < WK; ++w) v += red[(w * MP + tok) * kRS + r];
    if (p.splits == 1) red[tok * kRS + r] = v;
    else part[idx] = v;
  }
  if (p.splits > 1) {
    // ---- the tile's sum: the last CTA to arrive adds the splits' partials in split order
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(p.counters + tile, 1) == p.splits - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (int idx = threadIdx.x; idx < MP * kRows; idx += kThreads) {
      float v = 0.f;
      for (int s = 0; s < p.splits; ++s) v += __ldcg(p.ws + ((size_t)s * tiles + tile) * MP * kRows + idx);
      red[(idx / kRows) * kRS + idx % kRows] = v;
    }
    if (threadIdx.x == 0) p.counters[tile] = 0;
  }
  __syncthreads();

  // ---- epilogue: y = bf16(sum * inv[n])  (SwiGLU: also act = silu(g) * u of the rounded g, u)
  if constexpr (!SWIGLU) {
    for (int idx = threadIdx.x; idx < p.M * kRows; idx += kThreads) {
      const int tok = idx / kRows, r = idx % kRows, n = tile * kRows + r;
      p.y[(size_t)tok * p.ldy + n] = __float2bfloat16_rn(red[tok * kRS + r] * __ldg(p.inv + n));
    }
  } else {
    constexpr int H = kRows / 2;
    for (int idx = threadIdx.x; idx < p.M * H; idx += kThreads) {
      const int tok = idx / H, j = idx % H, ng = tile * H + j, nu = p.I + ng;
      const float gf = bf16_round(red[tok * kRS + j] * __ldg(p.inv + ng));
      const float uf = bf16_round(red[tok * kRS + H + j] * __ldg(p.inv + nu));
      p.y[(size_t)tok * p.ldy + ng] = __float2bfloat16_rn(gf);
      p.y[(size_t)tok * p.ldy + nu] = __float2bfloat16_rn(uf);
      p.act[(size_t)tok * p.I + ng] = __float2bfloat16_rn(gf * fast_sigmoid(gf) * uf);
    }
  }
}

template <bool SWIGLU>
int launch(const Args& p, cudaStream_t st) {
  const int NT = (p.M + 7) / 8;
  const int WK = NT > 4 ? 2 : 4;
  const int tiles = p.N / kRows;
  const size_t smem = (size_t)WK * NT * 8 * kRS * sizeof(float);
  const dim3 grid(tiles, p.splits);
  switch (NT) {
#define ODB_FP8W_CASE(n) \
  case n: fp8w_gemm_kernel<n, SWIGLU><<<grid, kThreads, smem, st>>>(p); break;
    ODB_FP8W_CASE(1) ODB_FP8W_CASE(2) ODB_FP8W_CASE(3) ODB_FP8W_CASE(4)
    ODB_FP8W_CASE(5) ODB_FP8W_CASE(6) ODB_FP8W_CASE(7) ODB_FP8W_CASE(8)
#undef ODB_FP8W_CASE
    default: return -1;
  }
  ODB_CHECK_LAST();
  return 0;
}

}  // namespace

// y[M, N] (bf16, row stride ldy) = x[M, K] (bf16, row stride ldx) * (q[N, K] (e4m3, contiguous) * inv[N])^T.
// act non-null selects the SwiGLU epilogue: N = 2I rows are gate | up, y = gu [M, 2I] and act [M, I] = silu(gate) * up.
// 1 <= M <= 64, K % 128 == 0, N % 64 == 0 (SwiGLU: I % 32 == 0), 1 <= splits <= K / 256.  splits > 1 needs ws (fp32,
// splits * N * 64 floats) and counters (int32, N / 64 entries, zero; they are zero again when the kernel ends).
ODB_EXPORT int odb_fp8w_gemm(const void* x, long long ldx, const void* q, const void* inv, void* y, long long ldy, void* act,
                             int M, int N, int K, int splits, void* ws, void* counters, cudaStream_t st) {
  if (M < 1 || M > kMaxM || K <= 0 || N <= 0 || K % 128 || N % kRows || splits < 1 || splits > K / 256) return -1;
  if (((uintptr_t)x & 15) || ldx % 8 || ((uintptr_t)q & 15) || (splits > 1 && (!ws || !counters))) return -1;
  Args p{(const __nv_bfloat16*)x, ldx, (const uint8_t*)q, (const float*)inv, (__nv_bfloat16*)y, ldy, (__nv_bfloat16*)act,
         (float*)ws, (int*)counters, M, N, K, N / 2, splits};
  if (act) {
    if ((N / 2) % (kRows / 2)) return -1;
    return launch<true>(p, st);
  }
  return launch<false>(p, st);
}

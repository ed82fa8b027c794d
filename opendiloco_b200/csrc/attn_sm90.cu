// Causal flash-attention forward for sm_90a (SURVEY.md §2.5 K5), head_dim 64, bf16, MHA + GQA.
//
// Reads q/k/v straight out of the packed projection buffer qkv[T, (Hq + 2*Hkv) * 64] (token-major rows: no transposes)
// through ONE tensor map, writes out[T, Hq*64] token-major (the o-proj GEMM's A operand) and lse[B, Hq, S] (natural log).
//
// One CTA per (batch, q-head, 64-query block), 160 threads:
//   warp 4        TMA: Q once, then the K_j / V_j 64-key tiles through a STAGES-deep full / empty mbarrier ring
//   warps 0-3     one warpgroup: S = Q K_j^T with wgmma m64n64k16 (both operands in shared memory, K-major), online
//                 softmax in the exp2 domain on the accumulator registers (causal mask on the diagonal tile), then
//                 O += P V_j with P as the register A operand and V_j as an MN-major shared-memory operand
// 40 KB of shared memory per CTA, so several CTAs share an SM and one's softmax overlaps another's MMAs.  The heaviest
// query blocks are scheduled first.
#include "common.cuh"
#include "sm90_ptx.cuh"

using namespace odb;
using namespace sm90;

namespace attn {

constexpr int BQ = 64, BKV = 64, D = 64;
constexpr int STAGES = 2;
constexpr int THREADS = 160;
constexpr int TILE = 64 * 128;                   // a [64 x 64] bf16 tile, 128-byte swizzled rows
constexpr int SMEM_BYTES = TILE + STAGES * 2 * TILE + 1024 /*align*/ + 128 /*barriers*/;

__global__ void __launch_bounds__(THREADS)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, __nv_bfloat16* __restrict__ out, float* __restrict__ lse, int S, int Hq,
                int Hkv, long long ld_out, float scale_log2) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + TILE;                    // [stage][K | V]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sKV + STAGES * 2 * TILE);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + STAGES;

  pdl_launch_dependents();
  const int nqb = S / BQ;
  const int qb = nqb - 1 - (int)blockIdx.x;
  const int h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (Hq / Hkv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = b * S;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_qkv);
    mbar_init(q_full, 1);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, TILE);
      tma_load_2d(sQ, &tmap_qkv, q_full, h * D, t0 + qb * BQ);
      for (int j = 0; j <= qb; ++j) {
        const int s = j % STAGES;
        mbar_wait(&empty[s], ((j / STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], 2 * TILE);
        tma_load_2d(sKV + s * 2 * TILE, &tmap_qkv, &full[s], (Hq + hk) * D, t0 + j * BKV);
        tma_load_2d(sKV + s * 2 * TILE + TILE, &tmap_qkv, &full[s], (Hq + Hkv + hk) * D, t0 + j * BKV);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- MMA + softmax warpgroup
  // accumulator fragment of m64n64: acc[4*i + 2*h + e] is row (16*warp + lane/4 + 8*h), column (8*i + 2*(lane%4) + e)
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const int qrow0 = qb * BQ + warp * 16 + (lane >> 2);
  const uint64_t qdesc = make_smem_desc_sw128(smem_u32(sQ), 16, 1024);
  mbar_wait(q_full, 0);

  for (int j = 0; j <= qb; ++j) {
    const int s = j % STAGES;
    mbar_wait(&full[s], (j / STAGES) & 1);
    const uint32_t k_addr = smem_u32(sKV + s * 2 * TILE);
    const uint64_t kdesc = make_smem_desc_sw128(k_addr, 16, 1024);
    const uint64_t vdesc = make_smem_desc_sw128(k_addr + TILE, TILE, 1024);   // V: [keys x 64] read MN-major

    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64k16_ss<0, 0>(sc, qdesc + 2 * k, kdesc + 2 * k, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();

    // online softmax (log2 domain); a row is spread over the 4 lanes of a quad
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v = sc[4 * i + 2 * hh + e] * scale_log2;
          if (j == qb && j * BKV + 8 * i + 2 * (lane & 3) + e > qrow0 + 8 * hh) v = -INFINITY;
          sc[4 * i + 2 * hh + e] = v;
          mx[hh] = fmaxf(mx[hh], v);
        }
      }
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m[r], mx[r]);
      alpha[r] = exp2f(m[r] - mn);
      m[r] = mn;
      l[r] *= alpha[r];
    }
    uint32_t pf[4][4];                           // P as the register A operand of P V (k = keys)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float pv[4];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          pv[2 * hh + e] = exp2f(sc[4 * i + 2 * hh + e] - m[hh]);
          l[hh] += pv[2 * hh + e];
        }
      }
      pf[i >> 1][(i & 1) * 2 + 0] = f2_to_bf2(pv[0], pv[1]);
      pf[i >> 1][(i & 1) * 2 + 1] = f2_to_bf2(pv[2], pv[3]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i + 0] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs<1>(o, pf[kk], vdesc + 128 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    if (threadIdx.x == 0) mbar_arrive(&empty[s]);   // this warpgroup's MMAs on the stage have retired
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = qrow0 + 8 * r;
    const float inv = 1.f / l[r];
    __nv_bfloat16* orow = out + (long long)(t0 + q) * ld_out + h * D + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(orow + 8 * i) = f2_to_bf2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
    if ((lane & 3) == 0) lse[((long long)b * Hq + h) * S + q] = (m[r] + __log2f(l[r])) * 0.6931471805599453f;
  }
}

}  // namespace attn

// qkv: [B*S, (Hq+2*Hkv)*64] bf16 (row stride ld_qkv elements); out: [B*S, Hq*64] bf16; lse: [B, Hq, S] fp32
ODB_EXPORT int odb_attn_fwd(const void* qkv, void* out, void* lse, int B, int S, int Hq, int Hkv, long long ld_qkv,
                            long long ld_out, float softmax_scale, cudaStream_t st) {
  using namespace attn;
  if (S % 128 || Hq % Hkv || ld_qkv % 8 || ld_out % 8) return -1;
  CUtensorMap tq;
  int rc;
  if ((rc = make_tmap_2d(&tq, qkv, (long long)B * S, (Hq + 2 * Hkv) * D, ld_qkv * 2, 64, 64, 2))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  launch_pdl(attn_fwd_kernel, dim3(S / BQ, Hq, B), dim3(THREADS), SMEM_BYTES, st, tq, (__nv_bfloat16*)out, (float*)lse, S, Hq, Hkv,
             ld_out, softmax_scale * 1.4426950408889634f);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

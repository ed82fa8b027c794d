// Causal flash-attention BACKWARD for sm_90a (SURVEY.md §2.5 K5), head_dim 64, bf16, MHA + GQA.
//
//   P  = exp(S*scale - lse)          S  = Q K^T
//   dV = P^T dO                      dP = dO V^T
//   dS = P * (dP - D) * scale        D  = rowsum(dO * O)        (pre-pass kernel)
//   dK = dS^T Q                      dQ = dS K                  (dQ: fp32 reduce-add across key tiles, post-pass -> bf16)
//
// One CTA per (128-key tile, kv-head, batch), 288 threads: warp 8 streams Q / dO tiles and the per-query statistics of
// the CTA's work items (query heads of its GQA group x causal range of 64-query tiles) through a STAGES-deep TMA +
// mbarrier ring; warps 0-3 and 4-7 are two wgmma warpgroups, each owning 64 of the keys with its dK / dV accumulators in
// registers.  Both consume the same stage (empty barrier count 2), so Q and dO are loaded once per 128 keys.  The MMAs
// of one warpgroup run in program order, and the other warpgroup's MMAs fill the tensor cores while one does its exp / dS
// work.  Issuing the next item's S^T / dP^T before this item's dV / dK / dQ keeps 64 more accumulators live: that
// variant needs 222 registers per thread (0 spills under __maxnreg__(224)), which a 288-thread CTA cannot launch with.
// Built as a 384-thread CTA with a producer warpgroup (setmaxnreg.dec 24 / 40, consumers .inc 240 / 232), ptxas 12.9
// still allocated it within 168 registers and spilled 300 bytes, so this layout keeps the in-order form.  The score tiles are computed TRANSPOSED (keys on the rows) so
// that P^T and dS^T are directly the register A operands of the dV / dK products:
//     S^T  = K  Q^T     A = K (smem, K-major)      B = Q  (smem, K-major)
//     dP^T = V  dO^T    A = V (smem, K-major)      B = dO (smem, K-major)
//     dV  += P^T dO     A = P^T (registers)        B = dO (smem, MN-major)
//     dK  += dS^T Q     A = dS^T (registers)       B = Q  (smem, MN-major)
//     dQ   = dS K       A = the [128 keys x 64 queries] dS^T tile both warpgroups write to smem, read MN-major;
//                       B = K (smem, MN-major); warpgroup w computes dQ columns 32w..32w+31 over all 128 keys
// The same swizzled [64 x 64] TMA tiles serve as K-major and as MN-major operands - only the descriptor changes.
// dQ leaves through shared memory: each warpgroup stages its fp32 [64 x 32] half with the 128-byte swizzle of the dQ
// accumulator's tensor map and one thread reduce-adds it into global memory with one bulk tensor reduction.
#include "common.cuh"
#include "sm90_ptx.cuh"

using namespace odb;
using namespace sm90;

namespace attn_bwd {

constexpr int BQ = 64, BKV = 128, D = 64;        // BKV keys per CTA, 64 per consumer warpgroup
constexpr int STAGES = 3;
constexpr int THREADS = 288;
constexpr int TILE = 64 * 128;                   // a [64 x 64] bf16 tile (or [64 x 32] fp32), 128-byte swizzled rows
constexpr int STAT_BYTES = 2 * 64 * 4;           // per work item: -lse * log2(e) [64], then -D * scale [64]
// K, V (2 tiles each), 2 x dS^T [128 x 64], 2 x dQ staging [64 x 32] fp32, STAGES x (Q, dO, stats)
constexpr int SMEM_BYTES = 4 * TILE + 4 * TILE + 2 * TILE + STAGES * (2 * TILE + STAT_BYTES) + 1024 /*align*/ + 128 /*barriers*/;

// stats: per query (b, h, s) the pre-pass layout [B, Hq, S/128, 2, 128]: -lse * log2(e), then -D * scale
__global__ void __launch_bounds__(THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_do,
                const __grid_constant__ CUtensorMap tmap_dq, const float* __restrict__ stats, __nv_bfloat16* __restrict__ dk,
                __nv_bfloat16* __restrict__ dv, const float* __restrict__ cos_t, const float* __restrict__ sin_t, int S, int Hq,
                int Hkv, long long ld_dkv, float scale, float scale_log2) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;                            // [128 keys][64], two TMA tiles
  uint8_t* sV = sK + 2 * TILE;
  uint8_t* sdS = sV + 2 * TILE;                  // [2 buffers] dS^T [128 keys][64 queries], 128-byte swizzle
  uint8_t* sdQ = sdS + 4 * TILE;                 // [warpgroup] fp32 dQ [64 queries][32], 128-byte swizzle
  uint8_t* sQ = sdQ + 2 * TILE;                  // [stage][Q | dO]
  float* sStat = reinterpret_cast<float*>(sQ + STAGES * 2 * TILE);   // [stage][2][64]
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sStat) + STAGES * STAT_BYTES);
  uint64_t* full = kv_full + 1;
  uint64_t* empty = full + STAGES;

  pdl_launch_dependents();
  const int kb = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int nqb = S / BQ;
  const int group = Hq / Hkv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = b * S;
  const int qb0 = kb * (BKV / BQ);               // causal: query tiles qb0 .. nqb-1
  const int per_head = nqb - qb0;
  const int n_items = group * per_head;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    tma_prefetch_desc(&tmap_dq);
    mbar_init(kv_full, 1);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(kv_full, 4 * TILE);
      for (int j = 0; j < 2; ++j) {
        tma_load_2d(sK + j * TILE, &tmap_qkv, kv_full, (Hq + hk) * D, t0 + kb * BKV + 64 * j);
        tma_load_2d(sV + j * TILE, &tmap_qkv, kv_full, (Hq + Hkv + hk) * D, t0 + kb * BKV + 64 * j);
      }
      for (int it = 0; it < n_items; ++it) {
        const int s = it % STAGES;
        const int h = hk * group + it / per_head, qb = qb0 + it % per_head;
        mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], 2 * TILE + STAT_BYTES);
        tma_load_2d(sQ + s * 2 * TILE, &tmap_qkv, &full[s], h * D, t0 + qb * BQ);
        tma_load_2d(sQ + s * 2 * TILE + TILE, &tmap_do, &full[s], h * D, t0 + qb * BQ);
        const int s0 = qb * BQ;
        const float* g = stats + (((long long)(b * Hq + h) * (S / 128) + s0 / 128) * 2) * 128 + (s0 % 128);
        bulk_load_1d(sStat + s * 128, g, 64 * 4, &full[s]);
        bulk_load_1d(sStat + s * 128 + 64, g + 128, 64 * 4, &full[s]);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- wgmma warpgroups
  // accumulator fragment of m64nN: acc[4*i + 2*h + e] is row (16*warp + lane/4 + 8*h), column (8*i + 2*(lane%4) + e)
  const int wg = warp >> 2;                      // this warpgroup's keys: kb*BKV + 64*wg ...
  const int tid = threadIdx.x & 127;
  const int diag = qb0 + wg;                     // the query tile on this warpgroup's diagonal
  float dvacc[32], dkacc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dvacc[i] = dkacc[i] = 0.f;
  const int krow = (warp & 3) * 16 + (lane >> 2);   // key row (inside the warpgroup's 64) of acc[.. h = 0 ..]
  const uint32_t k_addr = smem_u32(sK + wg * TILE), v_addr = smem_u32(sV + wg * TILE);
  const uint64_t kdesc = make_smem_desc_sw128(k_addr, 16, 1024);
  const uint64_t vdesc = make_smem_desc_sw128(v_addr, 16, 1024);
  const uint64_t k_mn = make_smem_desc_sw128(smem_u32(sK) + 64 * wg, TILE, 1024);   // K columns 32*wg .. 32*wg+31
  uint8_t* const my_dq = sdQ + wg * TILE;
  mbar_wait(kv_full, 0);

  float st[32], dpt[32], dq[16];
  uint32_t pf[4][4], dsf[4][4];

  // S^T and dP^T of item `it` into st / dpt (one wgmma group)
  auto issue_scores = [&](int it) {
    const int s = it % STAGES;
    mbar_wait(&full[s], (it / STAGES) & 1);
    const uint32_t q_addr = smem_u32(sQ + s * 2 * TILE);
    const uint64_t qdesc = make_smem_desc_sw128(q_addr, 16, 1024), dodesc = make_smem_desc_sw128(q_addr + TILE, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64k16_ss<0, 0>(st, kdesc + 2 * k, qdesc + 2 * k, k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64k16_ss<0, 0>(dpt, vdesc + 2 * k, dodesc + 2 * k, k > 0 ? 1u : 0u);
    wgmma_commit();
  };
  // dQ rows of item `it` (retired in dq): stage this warpgroup's half in smem, one thread reduce-adds it
  auto store_dq = [&](int it) {
    const int h = hk * group + it / per_head, qb = qb0 + it % per_head;
    if (tid == 0) bulk_wait_read<0>();           // the previous reduction has finished reading the staging tile
    named_bar_sync(2 + wg, 128);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = krow + 8 * hh;
#pragma unroll
      for (int i = 0; i < 4; ++i)
        *reinterpret_cast<float2*>(my_dq + r * 128 + (((2 * i + ((lane & 3) >> 1)) ^ (r & 7)) << 4) + 8 * (lane & 1)) =
            make_float2(dq[4 * i + 2 * hh], dq[4 * i + 2 * hh + 1]);
    }
    fence_proxy_async_smem();
    named_bar_sync(2 + wg, 128);
    if (tid == 0) {
      tma_reduce_add_2d(my_dq, &tmap_dq, h * D + 32 * wg, t0 + qb * BQ);
      bulk_commit();
    }
  };

  for (int it = 0; it < n_items; ++it) {
    const int s = it % STAGES;
    const int qb = qb0 + it % per_head;
    const float* lse2 = sStat + s * 128;
    const float* dsc = lse2 + 64;
    issue_scores(it);
    wgmma_wait<0>();
    // Causal mask on and before the diagonal tile.  The one query tile before it (the CTA's first tile, for the second
    // warpgroup) sees none of the keys: it runs the same MMAs with P = dS = 0, which keeps every wgmma out of divergent
    // code, and the idle warpgroup would otherwise only wait at the barrier below.
    const bool masked = qb <= diag;
    const int kq = 64 * (diag - qb) + krow;       // key row relative to the item's first query, for acc[.. h = 0 ..]
    // P^T, dS^T as register A operands (k = queries), dS^T also into this warpgroup's rows of the swizzled smem tile
    uint8_t* ds_buf = sdS + (it & 1) * 2 * TILE;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float pv[4], dsv[4];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * i + 2 * hh + e;
          const int qc = 8 * i + 2 * (lane & 3) + e;     // query column inside the tile
          float pe = exp2f(fmaf(st[x], scale_log2, lse2[qc]));
          if (masked && kq + 8 * hh > qc) pe = 0.f;
          pv[2 * hh + e] = pe;
          dsv[2 * hh + e] = pe * fmaf(dpt[x], scale, dsc[qc]);
        }
      }
      pf[i >> 1][(i & 1) * 2 + 0] = f2_to_bf2(pv[0], pv[1]);
      pf[i >> 1][(i & 1) * 2 + 1] = f2_to_bf2(pv[2], pv[3]);
      const uint32_t d0 = f2_to_bf2(dsv[0], dsv[1]), d1 = f2_to_bf2(dsv[2], dsv[3]);
      dsf[i >> 1][(i & 1) * 2 + 0] = d0;
      dsf[i >> 1][(i & 1) * 2 + 1] = d1;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = 64 * wg + krow + 8 * hh;
        *reinterpret_cast<uint32_t*>(ds_buf + r * 128 + ((i ^ (r & 7)) << 4) + 4 * (lane & 3)) = hh ? d1 : d0;
      }
    }
    fence_proxy_async_smem();                    // generic-proxy stores -> visible to wgmma
    // Both halves of the dS^T tile written.  The other buffer is free as well: each warpgroup retired the dQ MMAs that
    // read it (item it-1) before arriving here, so only one barrier per item joins the two warpgroups.
    named_bar_sync(1, 256);
    {
      const uint32_t q_addr = smem_u32(sQ + s * 2 * TILE);
      const uint64_t q_mn = make_smem_desc_sw128(q_addr, TILE, 1024), do_mn = make_smem_desc_sw128(q_addr + TILE, TILE, 1024);
      const uint64_t ds_mn = make_smem_desc_sw128(smem_u32(ds_buf), TILE, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs<1>(dvacc, pf[kk], do_mn + 128 * kk, 1u);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs<1>(dkacc, dsf[kk], q_mn + 128 * kk, 1u);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_m64n32k16_ss<1, 1>(dq, ds_mn + 128 * kk, k_mn + 128 * kk, kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
    }
    if (tid == 0) mbar_arrive(&empty[s]);
    store_dq(it);
  }
  if (tid == 0) bulk_wait<0>();                  // the staging tile stays valid until the last reduction completes

  // dK / dV of this warp's 16 keys; with cos/sin dK leaves with the RoPE rotation undone (rotation by -theta of the
  // pairs (j, j+32), which sit in accumulator groups i and i+4 of the same thread)
  const int key0 = kb * BKV + 64 * wg;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int pos = key0 + krow + 8 * hh;
    if (cos_t != nullptr) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * i + 2 * (lane & 3) + e;
          const float cs = cos_t[(size_t)pos * 32 + c], sn = sin_t[(size_t)pos * 32 + c];
          const float x = dkacc[4 * i + 2 * hh + e], y = dkacc[4 * (i + 4) + 2 * hh + e];
          dkacc[4 * i + 2 * hh + e] = x * cs + y * sn;
          dkacc[4 * (i + 4) + 2 * hh + e] = y * cs - x * sn;
        }
      }
    }
    const long long t = (long long)t0 + pos;
    __nv_bfloat16* krow_p = dk + t * ld_dkv + hk * D + 2 * (lane & 3);
    __nv_bfloat16* vrow_p = dv + t * ld_dkv + hk * D + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      *reinterpret_cast<uint32_t*>(krow_p + 8 * i) = f2_to_bf2(dkacc[4 * i + 2 * hh], dkacc[4 * i + 2 * hh + 1]);
      *reinterpret_cast<uint32_t*>(vrow_p + 8 * i) = f2_to_bf2(dvacc[4 * i + 2 * hh], dvacc[4 * i + 2 * hh + 1]);
    }
  }
}

// Pre-pass: per (token, head) D = sum_d dO * O, stored together with the forward's log-sum-exp in the layout the main
// kernel bulk-copies per query tile: stats[b, h, s/128, 0, s%128] = -lse * log2(e), stats[..., 1, ...] = -D * scale.
// Eight lanes per (token, head) (16 bytes of dO and O each); the same threads zero the fp32 dQ accumulator row.
__global__ void __launch_bounds__(256) attn_dsum_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ out,
                                                        const float* __restrict__ lse, float* __restrict__ stats,
                                                        float* __restrict__ dq_acc, int B, int S, int Hq, long long ld, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * S * Hq * 8;
  if (i >= total) return;                                // total is a multiple of 8: whole lane groups leave together
  const int sub = (int)(i & 7);
  const long long w = i >> 3;
  const long long t = w / Hq;
  const int h = (int)(w % Hq);
  float a[8], o[8];
  unpack8(ld_v4(dout + t * ld + h * 64 + sub * 8), a);
  unpack8(ld_v4(out + t * ld + h * 64 + sub * 8), o);
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) s = fmaf(a[j], o[j], s);
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  float4* z = reinterpret_cast<float4*>(dq_acc + (t * Hq + h) * 64 + sub * 8);
  z[0] = make_float4(0.f, 0.f, 0.f, 0.f);
  z[1] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (sub == 0) {
    const long long bb = t / S, ss = t % S;
    float* dst = stats + (((bb * Hq + h) * (S / 128) + ss / 128) * 2) * 128 + (ss % 128);
    dst[0] = -lse[(bb * Hq + h) * S + ss] * 1.4426950408889634f;
    dst[128] = -s * scale;
  }
}

// Post-pass: fp32 dQ accumulator -> bf16 into dq_out (row stride ld_out), and - when cos/sin tables are given - the
// transpose RoPE rotation of dQ on the way (the main kernel already rotated dK), so the packed dq|dk|dv buffer leaves
// ready for the projection's dgrad / wgrad GEMMs.  One thread per 8 rotation pairs: x[j..j+8) and x[j+32..j+40) of one
// (token, head).
__global__ void __launch_bounds__(256) attn_bwd_finish_kernel(const float* __restrict__ dq_acc, __nv_bfloat16* __restrict__ dq_out,
                                                              const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                              long long T, int S, int Hq, long long ld_out) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = T * Hq * 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int jv = (int)(i & 3);
  const long long th = i >> 2;
  const int head = (int)(th % Hq);
  const long long t = th / Hq;
  float a[8], b[8];
  const float* src = dq_acc + (t * Hq + head) * 64 + jv * 8;
  const float4 a0 = ld_f4(src), a1 = ld_f4(src + 4), b0 = ld_f4(src + 32), b1 = ld_f4(src + 36);
  a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
  b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
  __nv_bfloat16* dst = dq_out + t * ld_out + head * 64 + jv * 8;
  if (cos_t != nullptr) {
    const int pos = (int)(t % S);
    const float4 c0 = ld_f4(cos_t + (size_t)pos * 32 + jv * 8), c1 = ld_f4(cos_t + (size_t)pos * 32 + jv * 8 + 4);
    const float4 s0 = ld_f4(sin_t + (size_t)pos * 32 + jv * 8), s1 = ld_f4(sin_t + (size_t)pos * 32 + jv * 8 + 4);
    const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float x = a[j], y = b[j];
      a[j] = x * cs[j] + y * sn[j];                      // rotation by -theta
      b[j] = y * cs[j] - x * sn[j];
    }
  }
  st_v4(dst, pack8(a));
  st_v4(dst + 32, pack8(b));
}

}  // namespace attn_bwd

// stats: fp32 scratch of 2 * B * Hq * S elements (per-query statistics, written by the pre-pass);
// dq_acc: fp32 [T, Hq*64] scratch (zeroed by the pre-pass, reduce-added by the main kernel);
// dq, dk, dv: bf16 outputs with row strides ld_dq / ld_dkv elements - e.g. the three column blocks of one packed
// [T, (Hq+2*Hkv)*64] buffer.  With cos/sin (fp32 [S, 32] tables) dq and dk leave with the RoPE rotation undone.
ODB_EXPORT int odb_attn_bwd(const void* qkv, const void* out, const void* dout, const void* lse, void* stats, void* dq_acc,
                            void* dq, void* dk, void* dv, const void* cos_t, const void* sin_t, int B, int S, int Hq, int Hkv,
                            long long ld_qkv, long long ld_out, long long ld_dq, long long ld_dkv, float softmax_scale,
                            cudaStream_t st) {
  using namespace attn_bwd;
  if (S % 128 || Hq % Hkv || ld_qkv % 8 || ld_out % 8 || ld_dq % 8 || ld_dkv % 8) return -1;
  const long long T = (long long)B * S;
  {
    const long long threads = T * Hq * 8;
    launch_pdl(attn_dsum_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, (const __nv_bfloat16*)dout,
               (const __nv_bfloat16*)out, (const float*)lse, (float*)stats, (float*)dq_acc, B, S, Hq, ld_out, softmax_scale);
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  CUtensorMap tq, tdo, tdq;
  int rc;
  if ((rc = make_tmap_2d(&tq, qkv, T, (Hq + 2 * Hkv) * D, ld_qkv * 2, 64, 64, 2))) return rc;
  if ((rc = make_tmap_2d(&tdo, dout, T, Hq * D, ld_out * 2, 64, 64, 2))) return rc;
  if ((rc = make_tmap_2d(&tdq, dq_acc, T, Hq * D, (long long)Hq * D * 4, 64, 32, 4))) return rc;
  launch_pdl(attn_bwd_kernel, dim3(S / BKV, Hkv, B), dim3(THREADS), SMEM_BYTES, st, tq, tdo, tdq, (const float*)stats,
             (__nv_bfloat16*)dk, (__nv_bfloat16*)dv, (const float*)cos_t, (const float*)sin_t, S, Hq, Hkv, ld_dkv, softmax_scale,
             softmax_scale * 1.4426950408889634f);
  {
    const long long threads = T * Hq * 4;
    launch_pdl(attn_bwd_finish_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, (const float*)dq_acc,
               (__nv_bfloat16*)dq, (const float*)cos_t, (const float*)sin_t, T, S, Hq, ld_dq);
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

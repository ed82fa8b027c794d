// Autoregressive decode kernels for sm_90a (bf16, head_dim 64, MHA + GQA): the pieces of a KV-cached generation step that
// the training kernels do not cover.
//
//   odb_dec_rope_append   n new tokens per row (n = 1: the decode step; n > 1: an assisted round's verify pass): rotate q|k
//                         of token j at the row's own position pos[b] + j (read from device memory, so a captured graph stays
//                         valid at every step), write k and v into the layer's cache at (b, pos[b] + j)
//   odb_dec_kv_fill       prefill: copy the (already rotated) k|v columns of the packed qkv rows into the cache
//   odb_dec_attn          split-KV decode attention (flash-decoding) + the combine kernel that every split-KV attention
//                         here (decode, grouped, verify) ends with
//   odb_dec_sample        greedy / temperature + top-k + top-p + min-p sampler, one CTA per row, with HF's sequence bias,
//                         repetition penalty, n-gram ban, bad words, min-length and min-new-tokens over the row's device-side
//                         token history when the control blocks ask
//   odb_dec_accept        assisted generation / prompt lookup: speculative acceptance of one round's proposals
//   odb_dec_lookup_propose  prompt lookup: each row's proposals from an earlier occurrence of its last n-gram
//   odb_dec_beam_topk     beam search: per vocabulary split of a row, the (max, sum-exp) partial and the local top-K logits
//   odb_dec_beam_step     beam search: one CTA per prompt merges the candidates and does HF's selection and bookkeeping
//   odb_dec_beam_reorder  beam search: chunk-table update and partial-chunk K/V copy for beams that changed parent
//   odb_dec_attn_group    multi-sample generation: split-KV decode attention that loads a chunk shared by sibling rows once
//   odb_dec_fork          multi-sample generation: make the sibling rows of a prefilled prompt its children (chunk table)
//
// KV cache layout, per layer: K and V each [B, Hkv, Smax, 64] bf16, so the keys of one (row, kv head) are contiguous and a
// chunk of them is ONE bulk copy.
//
// FP8 KV cache (generate(fp8_kv_cache=True)): K and V each [B, Hkv, Smax, 64] e4m3 plus fp32 inv [B, Hkv, Smax], one
// power-of-two scale per (position, kv head) row by the rule of fp8_rows.cuh.  The writers quantise the bf16 row the bf16
// writer would store; the attention kernels dequantise each element as q * inv, which is exactly the bf16 value of the
// dequantised cache C^ = q * inv, so they compute bit for bit what the bf16 kernels compute on C^.  The kernels are
// templates on the cache element type T (bf16, or uint8_t for e4m3 bytes); the inv pointers are null for bf16.
#include <curand_kernel.h>

#include <algorithm>
#include <climits>
#include <type_traits>

#include "common.cuh"
#include "fp8_rows.cuh"
#include "sm90_ptx.cuh"

using namespace odb;
using namespace sm90;

namespace dec {

constexpr int D = 64;
constexpr int CH = 128;             // keys per attention CTA
constexpr int ATT_THREADS = 128;    // one thread per key in the score phase, four warps in P V

// ------------------------------------------------------------------------------------------------ FP8 cache rows
// One warp quantises one 64-value cache row, two values per lane: returns the lane's two e4m3 bytes (x0 low, x1 high); lane
// 0 writes the row's inv.  The amax is an integer max of the |x| bit patterns, so a NaN or inf reaches it (NaN bytes, inv NaN).
__device__ __forceinline__ uint32_t quantize_pair(float x0, float x1, float* __restrict__ inv) {
  const uint32_t m = __reduce_max_sync(0xffffffffu, max(__float_as_uint(fabsf(x0)), __float_as_uint(fabsf(x1))));
  float scale;
  const bool ok = fp8_scale(__uint_as_float(m), kE4M3Max, scale);
  if ((threadIdx.x & 31) == 0) *inv = ok ? 1.f / scale : __int_as_float(0x7fffffff);
  return ok ? (uint32_t)cvt2<false>(x0 * scale, x1 * scale) : 0x7f7fu;
}

// 8 e4m3 bytes -> q * inv in fp32 (exactly the bf16 value of C^ for rows above the bf16-normal limit)
__device__ __forceinline__ void dequant8(const uint2& w, float inv, float (&f)[8]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 v = e4m3x2_to_f2((k < 2 ? w.x : w.y) >> (16 * (k & 1)));
    f[2 * k] = v.x * inv;
    f[2 * k + 1] = v.y * inv;
  }
}

// ------------------------------------------------------------------------------------------------ RoPE + append
// One block per token.  row: the token's qkv row (q heads, k heads, v heads; unrotated GEMM output); p its position; b its
// sequence.  q is rotated in place; rotated k and v go to the cache at (b, p).  Rounding: fp32 rotation of the bf16 inputs,
// one rounding to bf16 (as ops.kernels.rope_).  FP8 cache: with blockDim a multiple of 32, one warp covers exactly one
// head per iteration (lane e holds elements e and e + 32 of a rotated head, 2e and 2e + 1 of a v head), so the row amax of
// the bf16-rounded values is one warp reduction.
template <typename T>
__device__ __forceinline__ void rope_append_token(__nv_bfloat16* __restrict__ row, int p, int b, const float* __restrict__ cos_t,
                                                  const float* __restrict__ sin_t, T* __restrict__ kc, T* __restrict__ vc, int Hq,
                                                  int Hkv, int Smax, float* __restrict__ kinv, float* __restrict__ vinv) {
  const float* cr = cos_t + (long long)p * (D / 2);
  const float* sr = sin_t + (long long)p * (D / 2);
  const int n_rot = (Hq + Hkv) * (D / 2);
  for (int i = threadIdx.x; i < n_rot + Hkv * (D / 2); i += blockDim.x) {
    if (i < n_rot) {
      const int h = i / (D / 2), e = i % (D / 2);
      __nv_bfloat16* x = row + h * D;
      const float a = __bfloat162float(x[e]), c = __bfloat162float(x[e + D / 2]);
      const float cs = cr[e], sn = sr[e];
      const __nv_bfloat16 lo = __float2bfloat16_rn(a * cs - c * sn), hi = __float2bfloat16_rn(c * cs + a * sn);
      if (h < Hq) {
        x[e] = lo;
        x[e + D / 2] = hi;
      } else if constexpr (sizeof(T) == 1) {
        const long long r = ((long long)b * Hkv + (h - Hq)) * Smax + p;
        const uint32_t qb = quantize_pair(__bfloat162float(lo), __bfloat162float(hi), kinv + r);
        kc[r * D + e] = (uint8_t)qb;
        kc[r * D + e + D / 2] = (uint8_t)(qb >> 8);
      } else {
        __nv_bfloat16* dst = kc + (((long long)b * Hkv + (h - Hq)) * Smax + p) * D;
        dst[e] = lo;
        dst[e + D / 2] = hi;
      }
    } else {
      const int j = i - n_rot, hk = j / (D / 2), e = j % (D / 2);
      const uint32_t v = reinterpret_cast<const uint32_t*>(row + (Hq + Hkv + hk) * D)[e];
      if constexpr (sizeof(T) == 1) {
        const long long r = ((long long)b * Hkv + hk) * Smax + p;
        const float2 f = bf2_to_f2(v);
        reinterpret_cast<uint16_t*>(vc + r * D)[e] = (uint16_t)quantize_pair(f.x, f.y, vinv + r);
      } else {
        reinterpret_cast<uint32_t*>(vc + (((long long)b * Hkv + hk) * Smax + p) * D)[e] = v;
      }
    }
  }
}

// grid (B, n), block 256: n tokens per row, slot-major rows (row j*B + b is token j of sequence b, at position pos[b] + j);
// n = 1 is the decode step.  pos is read from device memory, so a captured graph stays valid at every step.
template <typename T>
__global__ void __launch_bounds__(256)
rope_append_kernel(__nv_bfloat16* __restrict__ qkv, long long ld, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                   const int* __restrict__ pos, T* __restrict__ kc, T* __restrict__ vc, int Hq, int Hkv, int Smax,
                   float* __restrict__ kinv, float* __restrict__ vinv) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, j = blockIdx.y, B = gridDim.x;
  rope_append_token(qkv + ((long long)j * B + b) * ld, pos[b] + j, b, cos_t, sin_t, kc, vc, Hq, Hkv, Smax, kinv, vinv);
}

// ------------------------------------------------------------------------------------------------ prefill cache fill
// grid (Sp, B), block 128: row s < len[b] of batch row b -> cache row b * row_stride: 16-byte copies of the k and v heads
// (FP8 cache: one warp quantises one head, two values per lane).
template <typename T>
__global__ void __launch_bounds__(128)
kv_fill_kernel(const __nv_bfloat16* __restrict__ qkv, long long ld, const int* __restrict__ len, T* __restrict__ kc,
               T* __restrict__ vc, int Sp, int Hq, int Hkv, int Smax, int row_stride, float* __restrict__ kinv,
               float* __restrict__ vinv) {
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x, b = blockIdx.y;
  if (s >= len[b] || s >= Smax) return;
  const __nv_bfloat16* row = qkv + ((long long)b * Sp + s) * ld + Hq * D;
  if constexpr (sizeof(T) == 1) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int hh = warp; hh < 2 * Hkv; hh += blockDim.x >> 5) {
      const int kv = hh / Hkv, hk = hh % Hkv;
      const float2 f = bf2_to_f2(reinterpret_cast<const uint32_t*>(row + hh * D)[lane]);
      const long long r = ((long long)b * row_stride * Hkv + hk) * Smax + s;
      reinterpret_cast<uint16_t*>((kv ? vc : kc) + r * D)[lane] = (uint16_t)quantize_pair(f.x, f.y, (kv ? vinv : kinv) + r);
    }
  } else {
    for (int i = threadIdx.x; i < 2 * Hkv * (D / 8); i += blockDim.x) {
      const int kv = i / (Hkv * (D / 8)), r = i % (Hkv * (D / 8)), hk = r / (D / 8), c = r % (D / 8);
      const uint4 v = ld_nc_v4(row + (kv * Hkv + hk) * D + c * 8);
      __nv_bfloat16* dst = (kv ? vc : kc) + (((long long)b * row_stride * Hkv + hk) * Smax + s) * D + c * 8;
      st_v4(dst, v);
    }
  }
}

// ------------------------------------------------------------------------------------------------ split-KV attention
// grid (ceil(Smax / CH), Hkv, B), block 128.  CTA (c, hk, b) serves the G = Hq / Hkv query heads of kv head hk against keys
// [c*CH, min((c+1)*CH, pos[b]+1)) of row b: K and V of the chunk arrive by two bulk copies, scores are one thread per key,
// P V is one warp per 32 keys (lanes over dimension pairs) summed across the four warps.  Writes the unnormalised partial
// output and its (max, sum) in the log2 domain; chunks past the row's length exit at once.  With a chunk table (beam
// search), the keys of chunk c of row b are read from physical row table[b * nchunks + c]; without one, from row b.
// FP8 cache (T = uint8_t): the chunk's e4m3 K and V and its two inv runs (rounded up to 16 bytes, in bounds since Smax is a
// multiple of CH) arrive by four bulk copies, and every element is read as q * inv; the arithmetic is the bf16 kernel's.
template <int G, typename T = __nv_bfloat16>
struct AttSmem {
  static constexpr int E = (int)sizeof(T);
  static constexpr int K_OFF = 0;
  static constexpr int V_OFF = CH * D * E;
  static constexpr int KI_OFF = 2 * CH * D * E;                  // FP8 cache: fp32 [CH] inv of the keys, then of the values
  static constexpr int VI_OFF = KI_OFF + (E == 1 ? CH * 4 : 0);
  static constexpr int Q_OFF = VI_OFF + (E == 1 ? CH * 4 : 0);   // fp32 [G][64], pre-scaled by softmax_scale * log2(e)
  static constexpr int S_OFF = Q_OFF + G * D * 4;                 // fp32 [G][CH] scores, then probabilities
  static constexpr int R_OFF = S_OFF + G * CH * 4;                // fp32 [4][G][64] per-warp P V
  static constexpr int M_OFF = R_OFF + 4 * G * D * 4;             // fp32 [G][2] (max, sum)
  static constexpr int BAR_OFF = M_OFF + 2 * G * 4;
  static constexpr int BYTES = BAR_OFF + 16;
};

// The arithmetic of one partial: the G query heads of sQ (pre-scaled) against the n keys of sK / sV (and sKI / sVI) of
// chunk c, written to part_o / part_ml of row b.  decode_attn_kernel and decode_attn_group_kernel both compute every
// partial through this function, so their results are the same bits.  Ends with shared memory still being read (the
// caller synchronises before overwriting it).
template <int G, typename T>
__device__ __forceinline__ void attn_chunk_partial(uint8_t* smem, int n, int b, int hk, int c, int Hkv, int nchunks,
                                                   float* __restrict__ part_o, float* __restrict__ part_ml) {
  using L = AttSmem<G, T>;
  constexpr bool KV8 = sizeof(T) == 1;
  const T* sK = reinterpret_cast<const T*>(smem + L::K_OFF);
  const T* sV = reinterpret_cast<const T*>(smem + L::V_OFF);
  const float* sKI = reinterpret_cast<const float*>(smem + L::KI_OFF);
  const float* sVI = reinterpret_cast<const float*>(smem + L::VI_OFF);
  const float* sQ = reinterpret_cast<const float*>(smem + L::Q_OFF);
  float* sS = reinterpret_cast<float*>(smem + L::S_OFF);
  float* sR = reinterpret_cast<float*>(smem + L::R_OFF);
  float* sM = reinterpret_cast<float*>(smem + L::M_OFF);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // ---- scores: thread = key; the 16-byte chunks of a key row are visited in a rotated order (no bank conflicts)
  {
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
    if (tid < n) {
#pragma unroll
      for (int cc = 0; cc < D / 8; ++cc) {
        const int ch = (cc + tid) & (D / 8 - 1);
        float kf[8];
        if constexpr (KV8) dequant8(reinterpret_cast<const uint2*>(sK + tid * D)[ch], sKI[tid], kf);
        else unpack8(reinterpret_cast<const uint4*>(sK + tid * D)[ch], kf);
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float* qg = sQ + g * D + ch * 8;
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[g] = fmaf(qg[e], kf[e], acc[g]);
        }
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) sS[g * CH + tid] = tid < n ? acc[g] : -INFINITY;
  }
  __syncthreads();

  // ---- per-head max / exp2 / sum over the chunk: warp w takes heads w, w+4, ...
  for (int g = warp; g < G; g += 4) {
    float v[CH / 32], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < CH / 32; ++k) {
      v[k] = sS[g * CH + lane + 32 * k];
      mx = fmaxf(mx, v[k]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < CH / 32; ++k) {
      const float p = exp2f(v[k] - mx);          // masked keys: exp2(-inf) = 0
      sS[g * CH + lane + 32 * k] = p;
      sum += p;
    }
    sum = warp_sum(sum);
    if (lane == 0) {
      sM[2 * g] = mx;
      sM[2 * g + 1] = sum;
    }
  }
  __syncthreads();

  // ---- P V: warp w over keys [32w, 32w+32), lane over dimensions (2*lane, 2*lane+1)
  {
    float o[G][2];
#pragma unroll
    for (int g = 0; g < G; ++g) o[g][0] = o[g][1] = 0.f;
    const int jb = warp * 32, je = min(n, jb + 32);
    for (int j = jb; j < je; ++j) {
      float2 vv;
      if constexpr (KV8) {
        const float2 f = e4m3x2_to_f2(reinterpret_cast<const uint16_t*>(sV + j * D)[lane]);
        vv = make_float2(f.x * sVI[j], f.y * sVI[j]);
      } else {
        vv = bf2_to_f2(reinterpret_cast<const uint32_t*>(sV + j * D)[lane]);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float p = sS[g * CH + j];
        o[g][0] = fmaf(p, vv.x, o[g][0]);
        o[g][1] = fmaf(p, vv.y, o[g][1]);
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g)
      *reinterpret_cast<float2*>(sR + (warp * G + g) * D + 2 * lane) = make_float2(o[g][0], o[g][1]);
  }
  __syncthreads();
  const int Hq = Hkv * G;
  for (int i = tid; i < G * D; i += ATT_THREADS) {
    const int g = i / D, d = i % D;
    const float s = sR[i] + sR[G * D + i] + sR[2 * G * D + i] + sR[3 * G * D + i];
    part_o[(((long long)b * Hq + hk * G + g) * nchunks + c) * D + d] = s;
  }
  if (tid < G) {
    float* ml = part_ml + (((long long)b * Hq + hk * G + tid) * nchunks + c) * 2;
    ml[0] = sM[2 * tid];
    ml[1] = sM[2 * tid + 1];
  }
}

// Thread 0 of the CTA: bulk-copy keys [j0, j0 + n) of (physical row phys, kv head hk) into sK / sV (FP8 cache: also their two
// inv runs, rounded up to 16 bytes, in bounds since Smax is a multiple of CH), completing on bar.
template <int G, typename T>
__device__ __forceinline__ void attn_chunk_load(uint8_t* smem, const T* __restrict__ kc, const T* __restrict__ vc,
                                                const float* __restrict__ kinv, const float* __restrict__ vinv, int phys, int hk,
                                                int Hkv, int Smax, int j0, int n, uint64_t* bar) {
  using L = AttSmem<G, T>;
  const long long kv_off = (((long long)phys * Hkv + hk) * Smax + j0) * D;
  if constexpr (sizeof(T) == 1) {
    const long long i_off = ((long long)phys * Hkv + hk) * Smax + j0;
    const uint32_t ib = (n * 4 + 15) & ~15;
    mbar_arrive_expect_tx(bar, 2u * n * D + 2u * ib);
    bulk_load_1d(smem + L::K_OFF, kc + kv_off, n * D, bar);
    bulk_load_1d(smem + L::V_OFF, vc + kv_off, n * D, bar);
    bulk_load_1d(smem + L::KI_OFF, kinv + i_off, ib, bar);
    bulk_load_1d(smem + L::VI_OFF, vinv + i_off, ib, bar);
  } else {
    mbar_arrive_expect_tx(bar, 2u * n * D * 2);
    bulk_load_1d(smem + L::K_OFF, kc + kv_off, n * D * 2, bar);
    bulk_load_1d(smem + L::V_OFF, vc + kv_off, n * D * 2, bar);
  }
}

// The G query heads of kv head hk of row b -> sQ, pre-scaled by softmax_scale * log2(e).
template <int G, typename T>
__device__ __forceinline__ void attn_load_q(uint8_t* smem, const __nv_bfloat16* __restrict__ q, long long ldq, int b, int hk,
                                            float scale_log2) {
  float* sQ = reinterpret_cast<float*>(smem + AttSmem<G, T>::Q_OFF);
  const __nv_bfloat16* qrow = q + (long long)b * ldq + (long long)hk * G * D;
  for (int i = threadIdx.x; i < G * D; i += ATT_THREADS) sQ[i] = __bfloat162float(qrow[i]) * scale_log2;
}

template <int G, typename T>
__global__ void __launch_bounds__(ATT_THREADS)
decode_attn_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const T* __restrict__ kc, const T* __restrict__ vc,
                   const int* __restrict__ pos, float* __restrict__ part_o, float* __restrict__ part_ml, const int* __restrict__ table,
                   int Hkv, int Smax, int nchunks, float scale_log2, const float* __restrict__ kinv, const float* __restrict__ vinv) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + AttSmem<G, T>::BAR_OFF);
  pdl_launch_dependents();
  const int c = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  const int len = pos[b] + 1;
  const int j0 = c * CH;
  if (j0 >= len) return;                         // uniform over the CTA
  const int n = min(CH, len - j0);
  const int phys = table != nullptr ? table[b * nchunks + c] : b;
  if (threadIdx.x == 0) attn_chunk_load<G, T>(smem, kc, vc, kinv, vinv, phys, hk, Hkv, Smax, j0, n, bar);
  attn_load_q<G, T>(smem, q, ldq, b, hk, scale_log2);
  __syncthreads();
  mbar_wait(bar, 0);
  attn_chunk_partial<G, T>(smem, n, b, hk, c, Hkv, nchunks, part_o, part_ml);
}

// Sibling-grouped split-KV attention (multi-sample generation): rows p * ngrp .. p * ngrp + ngrp - 1 are the siblings of
// prompt p and read their keys through the chunk table, as decode_attn_kernel does.  grid (ceil(Smax / CH), Hkv, P * splits),
// block 128: CTA (c, hk, p * splits + s) serves siblings [s * per, min(ngrp, (s + 1) * per)) of prompt p, per =
// ceil(ngrp / splits), one after the other.  A sibling whose table entry for chunk c names the physical row already in
// shared memory, with at least its key count loaded, reuses that copy; otherwise the chunk is loaded again (after the
// fork: the chunk holding the prompt's tail and every later one, which each row owns).  Each sibling's partial is
// attn_chunk_partial on its own q, its own key count and the same bytes, so it is bit-identical to decode_attn_kernel's.
// At least four resident CTAs (128 registers a thread): without a minimum, ptxas holds G = 8 to 64 registers and spills.
template <int G, typename T>
__global__ void __launch_bounds__(ATT_THREADS, 4)
decode_attn_group_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const T* __restrict__ kc, const T* __restrict__ vc,
                         const int* __restrict__ pos, float* __restrict__ part_o, float* __restrict__ part_ml,
                         const int* __restrict__ table, int Hkv, int Smax, int nchunks, float scale_log2, const float* __restrict__ kinv,
                         const float* __restrict__ vinv, int ngrp, int splits) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + AttSmem<G, T>::BAR_OFF);
  pdl_launch_dependents();
  const int c = blockIdx.x, hk = blockIdx.y, p = blockIdx.z / splits, s = blockIdx.z % splits;
  const int per = ceil_div(ngrp, splits);
  const int r0 = p * ngrp + s * per, r1 = p * ngrp + min(ngrp, (s + 1) * per);
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  // The next sibling's q, position and table entry are loaded into registers while this sibling computes, so only the
  // first sibling waits for them.  q is scaled exactly as attn_load_q does.
  constexpr int QPT = (G * D + ATT_THREADS - 1) / ATT_THREADS;
  float qn[QPT];
  int pos_n = 0, phys_n = 0;
  const int tid = threadIdx.x, j0 = c * CH;
  auto fetch = [&](int r) {
    pos_n = pos[r];
    phys_n = table[r * nchunks + c];
    const __nv_bfloat16* qrow = q + (long long)r * ldq + (long long)hk * G * D;
#pragma unroll
    for (int k = 0; k < QPT; ++k)
      if (tid + k * ATT_THREADS < G * D) qn[k] = __bfloat162float(qrow[tid + k * ATT_THREADS]) * scale_log2;
  };
  float* sQ = reinterpret_cast<float*>(smem + AttSmem<G, T>::Q_OFF);
  int cur = -1, cur_n = 0;
  uint32_t phase = 0;
  if (r0 < r1) fetch(r0);
  for (int r = r0; r < r1; ++r) {
    const int len = pos_n + 1, phys = phys_n;
#pragma unroll
    for (int k = 0; k < QPT; ++k)
      if (tid + k * ATT_THREADS < G * D) sQ[tid + k * ATT_THREADS] = qn[k];
    if (r + 1 < r1) fetch(r + 1);
    if (j0 >= len) continue;                     // uniform over the CTA
    const int n = min(CH, len - j0);
    const bool load = phys != cur || n > cur_n;
    if (load && tid == 0) {
      fence_proxy_async_smem();                  // the previous sibling's reads of sK / sV come before the new copy
      attn_chunk_load<G, T>(smem, kc, vc, kinv, vinv, phys, hk, Hkv, Smax, j0, n, bar);
    }
    __syncthreads();
    if (load) {
      mbar_wait(bar, phase);
      phase ^= 1;
      cur = phys;
      cur_n = n;
    }
    attn_chunk_partial<G, T>(smem, n, r, hk, c, Hkv, nchunks, part_o, part_ml);
    __syncthreads();                             // every read of this sibling's shared memory is done
  }
}

// The combine of every split-KV attention here.  grid (Hq, n*B), block 64: merge the splits of query row r = j*B + b
// (slot-major, at position pos[b] + j; n = 1 for the decode kernels), head h, and write out[r, h*64 + d] (token-major: the
// o-proj GEMM's A operand).  Split s covers keys [s*span, (s+1)*span) and has cap slots per (row, head); the splits holding
// keys <= pos[b] + j each hold key s*span, so their max is finite.
__global__ void __launch_bounds__(64)
combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml, const int* __restrict__ pos,
               __nv_bfloat16* __restrict__ out, long long ldo, int cap, int span, int B) {
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, r = blockIdx.y, Hq = gridDim.x, d = threadIdx.x;
  const int b = r % B, j = r / B;
  const int used = ceil_div(pos[b] + j + 1, span);
  const long long base = ((long long)r * Hq + h) * cap;
  float M = -INFINITY;
  for (int c = 0; c < used; ++c) M = fmaxf(M, part_ml[(base + c) * 2]);
  float L = 0.f, acc = 0.f;
  for (int c = 0; c < used; ++c) {
    const float w = exp2f(part_ml[(base + c) * 2] - M);
    L = fmaf(part_ml[(base + c) * 2 + 1], w, L);
    acc = fmaf(part_o[(base + c) * D + d], w, acc);
  }
  out[(long long)r * ldo + h * D + d] = __float2bfloat16_rn(acc / L);
}

// ------------------------------------------------------------------------------------------------ sampler
// ictl (int64, device): [0] do_sample, [1] top_k, [2] seed, [3] pad_token_id, [4] number of EOS ids (<= 8), [5..12] EOS ids,
//                       [13] no_repeat_ngram_size, [14] min_new_tokens, [15] min_length, [16] entries of the sequence table
// fctl (fp32, device):  [0] temperature, [1] top_p, [2] repetition_penalty, [3] min_p
constexpr int SAMPLE_THREADS = 1024;
constexpr int MAX_EOS = 8;
constexpr int CTL_NGRAM = 13, CTL_MIN_NEW = 14, CTL_MIN_LEN = 15, CTL_N_SEQ = 16;
constexpr int MAX_SEQS = 1024;                   // entries of a sequence table (sequence_bias + bad_words_ids)

// ------------------------------------------------------------------------------------------------ logits processors
// HF's sequence bias, repetition penalty, n-gram ban, bad words, min-length and min-new-tokens, applied to the fp32 value of
// each logit (sampler) or log-prob (beam search).  The settings live in the control blocks and the sequence table, so a
// captured graph serves every value, "off" included.
__device__ __forceinline__ bool processors_on(const long long* __restrict__ ictl, const float* __restrict__ fctl) {
  return fctl[2] != 1.f || ictl[CTL_NGRAM] > 0 || ((ictl[CTL_MIN_NEW] > 0 || ictl[CTL_MIN_LEN] > 0) && ictl[4] > 0) ||
         ictl[CTL_N_SEQ] > 0;
}

// The sequence table of sequence_bias and bad_words_ids (ops/decode.py SeqTable): entry e is ids[off[e], off[e + 1]),
// kind[e] 0 (a bias of bias[e] on its last token) or 1 (a ban of its last token); n = ictl[CTL_N_SEQ] entries.  The
// bias entries come in HF's summation order: the length-1 sequences first, then the longer ones in dict order.
struct SeqTable {
  const int* off;                                // [MAX_SEQS + 1], then kind [MAX_SEQS], then the ids
  const float* bias;
  int n;
  __device__ __forceinline__ const int* kind() const { return off + MAX_SEQS + 1; }
  __device__ __forceinline__ const int* ids() const { return off + 2 * MAX_SEQS + 1; }
  __device__ __forceinline__ int last(int e) const { return ids()[off[e + 1] - 1]; }
};

// Entry e matches the history h (HF's SequenceBiasLogitsProcessor rule): a length-1 sequence always; a longer one of length
// n when L >= n and the history ends with its first n - 1 tokens.
template <class H>
__device__ __forceinline__ bool seq_match(const SeqTable& tab, int e, const H& h) {
  const int o = tab.off[e], n = tab.off[e + 1] - o;
  if (n == 1) return true;
  if (h.L < n) return false;
  const int* q = tab.ids() + o;
  const int s = h.L - n + 1;
  for (int k = 0; k < n - 1; ++k)
    if (h[s + k] != q[k]) return false;
  return true;
}

// Marks the table's matches whose last token lies in [lo, hi): a matched ban sets its bit of ban; a matched bias sets bit
// e of matched (shared, MAX_SEQS / 32 words, zero on entry) and the token's bit of biased (when not null).  The caller
// synchronises.
template <class H>
__device__ void mark_sequences(const SeqTable& tab, const H& h, int lo, int hi, unsigned* ban, unsigned* biased, unsigned* matched) {
  for (int e = threadIdx.x; e < tab.n; e += blockDim.x) {
    const int v = tab.last(e);
    if (v < lo || v >= hi || !seq_match(tab, e, h)) continue;
    if (tab.kind()[e] != 0) {
      atomicOr(ban + ((v - lo) >> 5), 1u << ((v - lo) & 31));
    } else {
      atomicOr(matched + (e >> 5), 1u << (e & 31));
      if (biased != nullptr) atomicOr(biased + ((v - lo) >> 5), 1u << ((v - lo) & 31));
    }
  }
}

// After mark_sequences: for the matched bias entry e, whether it is the first matched one of its token, and then the sum
// of the matched biases of that token in table order, starting from 0 (HF's fp32 order, so the result is its bit pattern).
// last (optional): the entries' last tokens staged in shared memory, so the scans read no global memory per entry.
__device__ __forceinline__ bool seq_bias_sum(const SeqTable& tab, const unsigned* matched, const int* last, int e, int v, float& sum) {
  for (int f = 0; f < e; ++f)
    if (((matched[f >> 5] >> (f & 31)) & 1u) && (last != nullptr ? last[f] : tab.last(f)) == v) return false;
  float s = 0.f;
  for (int f = e; f < tab.n; ++f)
    if (((matched[f >> 5] >> (f & 31)) & 1u) && (last != nullptr ? last[f] : tab.last(f)) == v) s = __fadd_rn(s, tab.bias[f]);
  sum = s;
  return true;
}

// HF's RepetitionPenaltyLogitsProcessor on one value.
__device__ __forceinline__ float penalise(float x, float p) { return x < 0.f ? __fmul_rn(x, p) : __fdiv_rn(x, p); }

// A row's token history h[0, L): h[0, n0) from a, then h[n0, L) from b (beam search: the prompt, then the beam's running
// sequence; plain decode: one buffer).
struct History {
  const int* a;
  const int* b;
  int n0, L;
  __device__ __forceinline__ int operator[](int i) const { return i < n0 ? a[i] : b[i - n0]; }
};

// Marks, for the tokens in [lo, hi), bit (token - lo) of pen (the token occurs in the history; only with penalise) and of
// ban (the token follows an earlier occurrence of the last n-1 tokens, n = ngram; or it is an EOS id and min_new_active).
// The n-gram scan looks at the follower h[s + n - 1] of every start s <= L - n first, so only starts whose follower is in
// range compare their n - 1 tokens.  The bitmaps must be zero on entry; the caller synchronises afterwards.
__device__ void mark_history(const History& h, int lo, int hi, bool penalise_on, int ngram, bool min_new_active,
                             const long long* __restrict__ ictl, unsigned* pen, unsigned* ban) {
  const int tid = threadIdx.x;
  if (penalise_on) {
    for (int i = tid; i < h.L; i += blockDim.x) {
      const int t = h[i];
      if (t >= lo && t < hi) atomicOr(pen + ((t - lo) >> 5), 1u << ((t - lo) & 31));
    }
  }
  if (ngram > 0 && h.L + 1 >= ngram) {
    const int q = h.L - ngram + 1;               // the last n - 1 tokens: h[q, L)
    for (int s = tid; s <= h.L - ngram; s += blockDim.x) {
      const int f = h[s + ngram - 1];
      if (f < lo || f >= hi) continue;
      bool eq = true;
      for (int k = 0; k < ngram - 1 && eq; ++k) eq = h[s + k] == h[q + k];
      if (eq) atomicOr(ban + ((f - lo) >> 5), 1u << ((f - lo) & 31));
    }
  }
  if (min_new_active && tid == 0) {
    const int n_eos = (int)min(ictl[4], (long long)MAX_EOS);
    for (int k = 0; k < n_eos; ++k) {
      const long long t = ictl[5 + k];
      if (t >= lo && t < hi) atomicOr(ban + ((t - lo) >> 5), 1u << ((t - lo) & 31));
    }
  }
}

// The value the sampler works on: the bf16 logit, or its processed fp32 value (bitmaps in global scratch, read past L1).
struct RawLogit {
  const __nv_bfloat16* row;
  __device__ __forceinline__ float operator()(int i) const { return __bfloat162float(row[i]); }
};
// With a sequence table, bias (not null) is the row's summed bias per token (0 where none, as HF's); the bias comes first.
struct ProcessedLogit {
  const __nv_bfloat16* row;
  const unsigned* pen;
  const unsigned* ban;
  float p;
  const float* bias;
  __device__ __forceinline__ float operator()(int i) const {
    float x = __bfloat162float(row[i]);
    const unsigned bit = 1u << (i & 31);
    if (bias != nullptr) x = __fadd_rn(x, __ldcg(bias + i));
    if (__ldcg(pen + (i >> 5)) & bit) x = penalise(x, p);
    if (__ldcg(ban + (i >> 5)) & bit) x = -INFINITY;
    return x;
  }
};

struct ArgMax {
  float v;
  int i;
};
__device__ __forceinline__ ArgMax argmax_merge(ArgMax a, ArgMax b) {
  // larger value wins; on equal values the lower index (torch.argmax); NaN never wins
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}

// Largest threshold t (on the bit pattern of a non-negative float) with  f(t) = sum over {e_i : bits(e_i) >= t} of w(e_i)
// >= target, where w = 1 (counts, top-k) or w = e (mass, top-p).  e_i <= 1, so t lies in [0, bits(1.0f)]: 30 bisection steps.
template <bool MASS>
__device__ uint32_t bisect_threshold(const float* e, int V, float target, float* red) {
  uint32_t lo = 0, hi = 0x3f800001u;             // f(lo) >= target ; f(hi) < target (nothing exceeds 1.0f)
  while (hi - lo > 1) {
    const uint32_t mid = lo + (hi - lo) / 2;
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      const float x = e[i];
      if (__float_as_uint(x) >= mid) s += MASS ? x : 1.f;
    }
    s = block_sum(s, red);
    if (s >= target) lo = mid; else hi = mid;
  }
  return lo;
}

// Block-wide argmax_merge of one (value, index) per thread; am: 32 shared slots.  Every thread gets the result.
__device__ ArgMax block_reduce_argmax(ArgMax best, ArgMax* am) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
    best = argmax_merge(best, other);
  }
  __syncthreads();                               // am may still be read by a previous call
  if (lane == 0) am[warp] = best;
  __syncthreads();
  if (warp == 0) {
    best = lane < (int)(blockDim.x >> 5) ? am[lane] : ArgMax{-INFINITY, INT_MAX};
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ArgMax other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
      best = argmax_merge(best, other);
    }
    if (lane == 0) am[0] = best;
  }
  __syncthreads();
  return am[0];
}

// Block-wide argmax of a row's values x(i) (ties to the lowest index); am: 32 shared slots.  Every thread gets the result.
template <class Load>
__device__ ArgMax block_argmax(Load x, int V, ArgMax* am) {
  ArgMax best = {-INFINITY, V};
  for (int i = threadIdx.x; i < V; i += blockDim.x) best = argmax_merge(best, ArgMax{x(i), i});
  best = block_reduce_argmax(best, am);
  if (best.i >= V) best.i = 0;                   // all-NaN row: token 0 rather than an out-of-range id
  return best;
}
__device__ ArgMax block_argmax(const __nv_bfloat16* __restrict__ row, int V, ArgMax* am) { return block_argmax(RawLogit{row}, V, am); }

// The unnormalised warped probability of logit x: exp(x / temp - mx).  Every user goes through this one expression, so
// a weight recomputed from the logits is bit-identical to the one the thresholds were found on.
__device__ __forceinline__ float warped_weight(float x, float temp, float mx) {
  return exp2f((x / temp - mx) * 1.4426950408889634f);
}

// HF warper order: temperature, then top-k, then top-p, then min-p.  Fills e[i] with the kept weights (0 elsewhere) and
// returns the threshold T on the weight's bit pattern: token i is kept iff bits(warped_weight(x_i)) >= T.  mx = max logit
// / temp, so the top weight is 1 and min-p (keep p_i >= min_p * p_max) keeps e_i >= min_p: one more bit-pattern threshold.
template <class Load>
__device__ uint32_t warp_weights(Load x, int V, float temp, int top_k, float top_p, float min_p, float mx, float* e, float* red) {
  const int tid = threadIdx.x;
  uint32_t T = 0;
  for (int i = tid; i < V; i += blockDim.x) e[i] = warped_weight(x(i), temp, mx);
  __syncthreads();
  if (top_k > 0 && top_k < V) {
    T = bisect_threshold<false>(e, V, (float)top_k, red);
    for (int i = tid; i < V; i += blockDim.x)
      if (__float_as_uint(e[i]) < T) e[i] = 0.f;
    __syncthreads();
  }
  if (top_p < 1.f) {
    float z = 0.f;
    for (int i = tid; i < V; i += blockDim.x) z += e[i];
    z = block_sum(z, red);
    const uint32_t t = bisect_threshold<true>(e, V, top_p * z, red);
    for (int i = tid; i < V; i += blockDim.x)
      if (__float_as_uint(e[i]) < t) e[i] = 0.f;
    __syncthreads();
    T = max(T, t);
  }
  if (min_p > 0.f) {
    const uint32_t t = __float_as_uint(min_p);
    for (int i = tid; i < V; i += blockDim.x)
      if (__float_as_uint(e[i]) < t) e[i] = 0.f;
    __syncthreads();
    T = max(T, t);
  }
  return T;
}
__device__ uint32_t warp_weights(const __nv_bfloat16* __restrict__ row, int V, float temp, int top_k, float top_p, float min_p, float mx,
                                 float* e, float* red) {
  return warp_weights(RawLogit{row}, V, temp, top_k, top_p, min_p, mx, e, red);
}

// Inverse CDF in index order over the weights e[0, V): u in (0, 1] picks the token; `fallback` when rounding leaves r
// outside every segment.  Thread t owns a contiguous segment; exclusive scan of the segment sums.  red: 33 floats.
__device__ int draw_index(const float* e, int V, float u, int fallback, float* red, int* tok_sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = ceil_div(V, (int)blockDim.x);
  const int s0 = min(V, tid * per), s1 = min(V, s0 + per);
  float local = 0.f;
  for (int i = s0; i < s1; ++i) local += e[i];
  float incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  __syncthreads();
  if (lane == 31) red[warp] = incl;
  if (tid == 0) *tok_sm = fallback;
  __syncthreads();
  if (warp == 0) {
    float w = red[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float y = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += y;
    }
    red[lane] = wi - w;                          // exclusive prefix of the warp totals
    if (lane == 31) red[32] = wi;                // total kept mass
  }
  __syncthreads();
  const float pre = red[warp] + incl - local, total = red[32];
  const float r = u * total;
  if (local > 0.f && pre <= r && r < pre + local) {
    float acc = pre;
    int pick = -1;
    for (int i = s0; i < s1; ++i) {
      if (e[i] > 0.f) {
        pick = i;
        acc += e[i];
        if (r < acc) break;
      }
    }
    *tok_sm = pick;                              // at most one thread's segment brackets r
  }
  __syncthreads();
  return *tok_sm;
}

// generate(output_scores / output_logits): where one emitted token's score row (fp32) and raw logits (bf16) go; either
// may be null.
struct ScoreOut {
  float* score;
  __nv_bfloat16* logit;
};
constexpr int SCORE_RAW = 0, SCORE_WARPED = 1, SCORE_ARGMAX = 2;

// One score row, HF's: SCORE_RAW the values x(i) (greedy: the processed logits); SCORE_WARPED x(i) / temp where
// bits(warped_weight(x(i))) >= T (warp_weights' kept set, which is exactly the set a draw picks from) and -inf elsewhere;
// SCORE_ARGMAX x(top) / temp at the argmax alone (top_k = 1, or a row with no finite value).  The raw logits are copied.
// Out of line, so the pass adds no registers to its callers.
template <class Load>
__device__ __noinline__ void store_scores(Load x, const __nv_bfloat16* __restrict__ row, int V, int mode, float temp, float mx,
                                          uint32_t T, int top, ScoreOut so) {
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    if (so.logit != nullptr) so.logit[i] = row[i];
    if (so.score == nullptr) continue;
    const float v = x(i);
    float s = v;
    if (mode == SCORE_WARPED) s = __float_as_uint(warped_weight(v, temp, mx)) >= T ? __fdiv_rn(v, temp) : -INFINITY;
    else if (mode == SCORE_ARGMAX) s = i == top ? __fdiv_rn(v, temp) : -INFINITY;
    so.score[i] = s;
  }
}

// One row's token from its values x(i): the argmax (greedy, and the reference point of the exponentials), or a draw from
// the warped weights.  finite_only: a row with no finite value keeps its argmax instead of drawing.  so (either pointer
// may be null): the row's score row and raw logits (row), from the same values and threshold the pick uses.
template <class Load>
__device__ int pick_token(Load x, const __nv_bfloat16* __restrict__ row, int V, const long long* __restrict__ ictl,
                          const float* __restrict__ fctl, int b, int g, bool finite_only, float* e, float* red, ArgMax* am, int* tok_sm,
                          ScoreOut so) {
  const ArgMax best = block_argmax(x, V, am);
  const bool do_sample = ictl[0] != 0;
  const int top_k = (int)ictl[1];
  const float temp = fctl[0];
  int tok = best.i;
  if (do_sample && top_k != 1 && (!finite_only || best.v > -INFINITY)) {
    const float mx = best.v / temp;
    const uint32_t T = warp_weights(x, V, temp, top_k, fctl[1], fctl[3], mx, e, red);
    curandStatePhilox4_32_10_t rng;
    curand_init((unsigned long long)ictl[2], (unsigned long long)b, (unsigned long long)g, &rng);
    tok = draw_index(e, V, curand_uniform(&rng), best.i, red, tok_sm);   // u in (0, 1]
    if (so.score != nullptr || so.logit != nullptr) store_scores(x, row, V, SCORE_WARPED, temp, mx, T, tok, so);
  } else if (so.score != nullptr || so.logit != nullptr) {
    store_scores(x, row, V, do_sample ? SCORE_ARGMAX : SCORE_RAW, temp, 0.f, 0u, best.i, so);
  }
  return tok;
}

// The sampler's sequence-table pass over a whole row: stage the entries' last tokens in last_sm, mark the matches (bans
// into ban), and store each biased token's summed bias in the row's zeroed bias.  Out of line, so its registers do not
// add to sample_kernel's.  Ends with a barrier.
__device__ __noinline__ void sample_sequences(const SeqTable tab, const History hh, int V, unsigned* ban, unsigned* matched, int* last_sm,
                                              float* bias) {
  for (int i = threadIdx.x; i < tab.n; i += blockDim.x) last_sm[i] = tab.last(i);
  mark_sequences(tab, hh, 0, V, ban, nullptr, matched);
  __syncthreads();
  for (int i = threadIdx.x; i < tab.n; i += blockDim.x) {
    float sum;
    if (((matched[i >> 5] >> (i & 31)) & 1u) && seq_bias_sum(tab, matched, last_sm, i, last_sm[i], sum)) bias[last_sm[i]] = sum;
  }
  __syncthreads();
}

// With a history (hist int32 [B, ldh]: row b's tokens at positions 0 .. pos[b]), the logits processors run when the control
// blocks turn them on: the row's bitmaps (scratch [B][2][nw] words, nw = ceil(V / 32): penalised, banned) are cleared and
// marked, and the token is picked from the processed values.  The emitted token is appended at hist[b, pos[b] + 1].
// With a sequence table (tab_off not null, ictl[CTL_N_SEQ] > 0), seq_scratch fp32 [B][V] (zero when the kernel starts, and
// again when it ends) takes the row's summed bias at the matched tokens, which are set back to 0 once the token is
// picked: the clearing costs one store per matched table entry, not a pass over V.
// score_out / logit_out (generate(output_scores / output_logits), each may be null): [score_cols, B, V]; a row that is not
// finished writes its score row (store_scores: the values and threshold of its pick) and raw logits at column gen[b].
__global__ void __launch_bounds__(SAMPLE_THREADS)
sample_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V, const long long* __restrict__ ictl,
              const float* __restrict__ fctl, int* __restrict__ pos, int* __restrict__ gen, int* __restrict__ finished,
              long long* __restrict__ out, int max_new, long long* __restrict__ ids_next, int* __restrict__ hist, int ldh,
              unsigned* __restrict__ scratch, const int* __restrict__ tab_off, const float* __restrict__ tab_bias,
              float* __restrict__ seq_scratch, float* __restrict__ score_out, __nv_bfloat16* __restrict__ logit_out, int score_cols) {
  extern __shared__ __align__(16) float e[];     // [V] exp(x - max) of the kept tokens, 0 elsewhere
  __shared__ float red[33];
  __shared__ ArgMax am[32];
  __shared__ int tok_sm;
  __shared__ unsigned matched[MAX_SEQS / 32];
  __shared__ int last_sm[MAX_SEQS];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, tid = threadIdx.x;
  const __nv_bfloat16* row = logits + (long long)b * ld;
  ScoreOut so{nullptr, nullptr};
  if (!finished[b] && gen[b] < score_cols) {     // a live row's column gen[b] of the [score_cols, B, V] score / logit buffers
    const long long at = ((long long)gen[b] * gridDim.x + b) * V;
    if (score_out != nullptr) so.score = score_out + at;
    if (logit_out != nullptr) so.logit = logit_out + at;
  }
  int tok;
  if (hist != nullptr && processors_on(ictl, fctl)) {
    const int nw = ceil_div(V, 32), L = pos[b] + 1, g = gen[b];
    unsigned* pen = scratch + (long long)b * 2 * nw;
    unsigned* ban = pen + nw;
    const SeqTable tab{tab_off, tab_bias, tab_off != nullptr ? (int)min(ictl[CTL_N_SEQ], (long long)MAX_SEQS) : 0};
    float* bias = tab.n > 0 ? seq_scratch + (long long)b * V : nullptr;
    for (int i = tid; i < 2 * nw; i += blockDim.x) pen[i] = 0u;
    for (int i = tid; i < MAX_SEQS / 32; i += blockDim.x) matched[i] = 0u;
    __syncthreads();
    const float p = fctl[2];
    const int* h = hist + (long long)b * ldh;
    const History hh{h, h, L, L};
    mark_history(hh, 0, V, p != 1.f, (int)ictl[CTL_NGRAM], g < ictl[CTL_MIN_NEW] || L < ictl[CTL_MIN_LEN], ictl, pen, ban);
    if (bias != nullptr) sample_sequences(tab, hh, V, ban, matched, last_sm, bias);
    __syncthreads();
    tok = pick_token(ProcessedLogit{row, pen, ban, p, bias}, row, V, ictl, fctl, b, g, true, e, red, am, &tok_sm, so);
    if (bias != nullptr) {
      __syncthreads();                           // every read of bias is done
      for (int i = tid; i < tab.n; i += blockDim.x)
        if ((matched[i >> 5] >> (i & 31)) & 1u) bias[last_sm[i]] = 0.f;
    }
  } else {
    tok = pick_token(RawLogit{row}, row, V, ictl, fctl, b, gen[b], false, e, red, am, &tok_sm, so);
  }
  if (tid == 0) {
    const int g = gen[b];
    const bool fin = finished[b] != 0;
    const long long t = fin ? ictl[3] : (long long)tok;
    if (g < max_new) out[(long long)b * max_new + g] = t;
    ids_next[b] = t;
    gen[b] = g + 1;
    if (hist != nullptr && pos[b] + 1 < ldh) hist[(long long)b * ldh + pos[b] + 1] = (int)t;
    pos[b] = pos[b] + 1;
    if (!fin) {
      const int n_eos = (int)min(ictl[4], (long long)MAX_EOS);
      for (int k = 0; k < n_eos; ++k)
        if (t == ictl[5 + k]) finished[b] = 1;
    }
  }
}

// ------------------------------------------------------------------------------------------------ verify attention
// Assisted generation scores n <= 8 tokens per row in one pass.  Rows are slot-major: row j*B + b is token j of sequence b,
// at position pos[b] + j, and it attends keys 0 .. pos[b] + j (causal inside the block).
//
// grid (splits, Hkv, B), 160 threads.  CTA (s, hk, b) takes the G*n <= 64 queries of kv head hk as ONE m64 tile (query
// qi = j*G + g is tile row qi; rows >= G*n are zero and masked) against the 64-key tiles [s*tps, (s+1)*tps) of the row's
// keys, stopping at the tile holding pos[b] + n - 1:
//   warp 4      TMA: the K and V tiles [64 keys x 64] of the [B*Hkv*Smax, 64] caches, 128-byte swizzle, through a
//               VSTAGES-deep full / empty mbarrier ring
//   warps 0-3   one warpgroup: Q gathered into shared memory in the same swizzled layout, S = Q K^T on wgmma m64n64k16,
//               causal mask + online softmax (exp2 domain) on the accumulators, O += P V with P as the register operand
// Writes the unnormalised partial output and its (max, sum) per query row; combine_kernel merges the splits.
//
// FP8 cache (KV8): warp 4 bulk-copies each tile's e4m3 K and V [64 keys x 64 bytes] and their two inv runs into an FP8
// stage of the ring; the warpgroup converts them (q * inv, exact in bf16) into ONE pair of bf16 K | V tiles in the same
// 128-byte swizzled layout the bf16 kernel's TMA writes, fences them for the async proxy and runs the same wgmmas, whose
// inputs are then exactly the bf16 kernel's on the dequantised cache.
constexpr int VB = 64;                           // keys per tile
constexpr int VSTAGES = 2;
constexpr int VTHREADS = 160;
constexpr int VTILE = 64 * 128;                  // a [64 x 64] bf16 tile, 128-byte swizzled rows
constexpr int VSMEM = VTILE + VSTAGES * 2 * VTILE + 1024 /*align*/ + 128 /*barriers*/;
constexpr int VFSTAGE = 2 * VB * D + 2 * VB * 4; // FP8 stage: e4m3 K, e4m3 V, inv of K, inv of V
constexpr int VSMEM8 = VTILE + 2 * VTILE + VSTAGES * VFSTAGE + 1024 /*align*/ + 128 /*barriers*/;

template <bool KV8>
__global__ void __launch_bounds__(VTHREADS)
verify_attn_kernel(const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                   const __nv_bfloat16* __restrict__ q, long long ldq, const int* __restrict__ pos, float* __restrict__ part_o,
                   float* __restrict__ part_ml, int Hkv, int Smax, int cap, int tps, float scale_log2, int lg, int n,
                   const uint8_t* __restrict__ kc8, const uint8_t* __restrict__ vc8, const float* __restrict__ kinv,
                   const float* __restrict__ vinv) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + VTILE;                   // [stage][K | V]; FP8: the converted K | V, then the FP8 stages
  uint8_t* s8 = sKV + 2 * VTILE;
  uint64_t* full = reinterpret_cast<uint64_t*>(KV8 ? s8 + VSTAGES * VFSTAGE : sKV + VSTAGES * 2 * VTILE);
  uint64_t* empty = full + VSTAGES;

  pdl_launch_dependents();
  const int s = blockIdx.x, hk = blockIdx.y, b = blockIdx.z, B = gridDim.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = 1 << lg, nq = G * n, Hq = Hkv * G;
  if (threadIdx.x == 0) {
    if constexpr (!KV8) {
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
    }
    for (int i = 0; i < VSTAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  const int p0 = pos[b];
  const int t_begin = s * tps, t_end = min((s + 1) * tps, ceil_div(p0 + n, VB));
  if (t_begin >= t_end) return;                  // uniform over the CTA
  const int row0 = (b * Hkv + hk) * Smax;

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      for (int t = t_begin; t < t_end; ++t) {
        const int i = t - t_begin, st = i % VSTAGES;
        mbar_wait(&empty[st], ((i / VSTAGES) & 1) ^ 1);
        if constexpr (KV8) {
          uint8_t* f8 = s8 + st * VFSTAGE;
          const long long r = (long long)row0 + t * VB;
          mbar_arrive_expect_tx(&full[st], VFSTAGE);
          bulk_load_1d(f8, kc8 + r * D, VB * D, &full[st]);
          bulk_load_1d(f8 + VB * D, vc8 + r * D, VB * D, &full[st]);
          bulk_load_1d(f8 + 2 * VB * D, kinv + r, VB * 4, &full[st]);
          bulk_load_1d(f8 + 2 * VB * D + VB * 4, vinv + r, VB * 4, &full[st]);
        } else {
          mbar_arrive_expect_tx(&full[st], 2 * VTILE);
          tma_load_2d(sKV + st * 2 * VTILE, &tmap_k, &full[st], 0, row0 + t * VB);
          tma_load_2d(sKV + st * 2 * VTILE + VTILE, &tmap_v, &full[st], 0, row0 + t * VB);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- Q tile: row qi, 16-byte chunk c at c ^ (qi & 7)
  for (int i = threadIdx.x; i < 64 * 8; i += 128) {
    const int qi = i >> 3, c = i & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (qi < nq)
      v = ld_nc_v4(q + ((long long)(qi >> lg) * B + b) * ldq + (long long)(hk * G + (qi & (G - 1))) * D + c * 8);
    *reinterpret_cast<uint4*>(sQ + qi * 128 + ((c ^ (qi & 7)) << 4)) = v;
  }
  fence_proxy_async_smem();                      // generic-proxy writes -> visible to wgmma
  named_bar_sync(1, 128);

  // accumulator fragment of m64n64: acc[4*i + 2*h + e] is row (16*warp + lane/4 + 8*h), column (8*i + 2*(lane%4) + e)
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  int last[2];                                   // the last key each of the thread's two rows may see (-1: padding row)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = 16 * warp + (lane >> 2) + 8 * hh;
    last[hh] = qi < nq ? p0 + (qi >> lg) : -1;
  }
  const uint64_t qdesc = make_smem_desc_sw128(smem_u32(sQ), 16, 1024);

  for (int t = t_begin; t < t_end; ++t) {
    const int i = t - t_begin, st = i % VSTAGES;
    mbar_wait(&full[st], (i / VSTAGES) & 1);
    if constexpr (KV8) {
      named_bar_sync(1, 128);                    // every warp's MMAs on the previous tile have retired: the bf16 tiles are free
      const uint8_t* f8 = s8 + st * VFSTAGE;
      const float* fi = reinterpret_cast<const float*>(f8 + 2 * VB * D);
      for (int x = threadIdx.x; x < 2 * VB * 8; x += 128) {     // (K | V, key r, 16-byte bf16 chunk c)
        const int kv = x >> 9, r = (x >> 3) & (VB - 1), c = x & 7;
        float f[8];
        dequant8(*reinterpret_cast<const uint2*>(f8 + kv * VB * D + r * D + c * 8), fi[kv * VB + r], f);
        *reinterpret_cast<uint4*>(sKV + kv * VTILE + r * 128 + ((c ^ (r & 7)) << 4)) = pack8(f);
      }
      fence_proxy_async_smem();                  // generic-proxy writes -> visible to wgmma
      named_bar_sync(1, 128);
      if (threadIdx.x == 0) mbar_arrive(&empty[st]);   // the FP8 stage has been read
    }
    const uint32_t k_addr = smem_u32(KV8 ? sKV : sKV + st * 2 * VTILE);
    const uint64_t kdesc = make_smem_desc_sw128(k_addr, 16, 1024);
    const uint64_t vdesc = make_smem_desc_sw128(k_addr + VTILE, VTILE, 1024);   // V: [keys x 64] read MN-major

    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64k16_ss<0, 0>(sc, qdesc + 2 * k, kdesc + 2 * k, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();

    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v = sc[4 * ii + 2 * hh + e] * scale_log2;
          if (t * VB + 8 * ii + 2 * (lane & 3) + e > last[hh]) v = -INFINITY;
          sc[4 * ii + 2 * hh + e] = v;
          mx[hh] = fmaxf(mx[hh], v);
        }
      }
    }
    float alpha[2], mref[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m[r], mx[r]);
      // a row that has seen no key yet keeps (max, sum, O) = (-inf, 0, 0): no -inf - -inf
      alpha[r] = mn == -INFINITY ? 1.f : exp2f(m[r] - mn);
      mref[r] = mn == -INFINITY ? 0.f : mn;
      m[r] = mn;
      l[r] *= alpha[r];
    }
    uint32_t pf[4][4];                           // P as the register A operand of P V (k = keys)
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      float pv[4];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          pv[2 * hh + e] = exp2f(sc[4 * ii + 2 * hh + e] - mref[hh]);
          l[hh] += pv[2 * hh + e];
        }
      }
      pf[ii >> 1][(ii & 1) * 2 + 0] = f2_to_bf2(pv[0], pv[1]);
      pf[ii >> 1][(ii & 1) * 2 + 1] = f2_to_bf2(pv[2], pv[3]);
    }
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      o[4 * ii + 0] *= alpha[0]; o[4 * ii + 1] *= alpha[0];
      o[4 * ii + 2] *= alpha[1]; o[4 * ii + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs<1>(o, pf[kk], vdesc + 128 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    if (!KV8 && threadIdx.x == 0) mbar_arrive(&empty[st]);   // this warpgroup's MMAs on the stage have retired
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = 16 * warp + (lane >> 2) + 8 * r;
    if (qi >= nq) continue;
    const long long orow = (long long)(qi >> lg) * B + b;
    const long long base = (orow * Hq + hk * G + (qi & (G - 1))) * cap + s;
    float* po = part_o + base * D + 2 * (lane & 3);
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) *reinterpret_cast<float2*>(po + 8 * ii) = make_float2(o[4 * ii + 2 * r], o[4 * ii + 2 * r + 1]);
    if ((lane & 3) == 0) {
      part_ml[base * 2] = m[r];
      part_ml[base * 2 + 1] = l[r];
    }
  }
}

// ------------------------------------------------------------------------------------------------ acceptance
// One CTA per row: the speculative-sampling decision of one assisted round (Leviathan et al. 2023, Chen et al. 2023).
//   plog [(K+1)*B, ldp] target logits, slot-major: slot i predicts the token at pos[b] + i + 1
//   qlog [K*B, ldq] draft logits of the proposals; tok [(K+1)*B]: slot 0 the row's last token, slots 1..K the proposals
// Greedy (do_sample = 0 or top_k = 1): accept while the proposal equals the target argmax, then emit the argmax.
// Sampling: p, q = the warped distributions (warp_weights: the sampler's rules); accept d_i with probability
// min(1, p(d_i) / q(d_i)); at the first rejection draw from normalise(max(0, p - q)); after K acceptances draw the bonus
// token from p_{K+1}.  Uniforms: Philox keyed by (seed, row, gen[b]*16 + 2*slot + {0, 1}).
// Then the emitted tokens go to out[b, gen..] (stopping after an EOS id or at max_new), pos / gen / finished advance, the
// new last token goes to tok slot 0 and the draft's position is set to the target's.  A row that finishes keeps its pos
// (every later round rewrites the same in-range cache positions); finished rows are left alone.
// stats [B, 2] int64: rounds the row took part in, proposals accepted.
//
// Point-mass mode (qlog == nullptr; prompt lookup): row b has cnt[b] <= K candidates in slots 1..cnt[b] (later slots hold
// a filler that is never accepted), and the draft is a point mass, q(d_i) = 1.  Greedy: as above, stopping at cnt[b].
// Sampling: accept d_i with probability p_i(d_i); at the first rejection draw from p_i with d_i removed (renormalised);
// with no candidate left (slot cnt[b], the bonus slot when cnt[b] = K) draw from p_{cnt[b]}.  The same Philox keys.
// hist (int32 [B, ldh], nullptr in assisted mode): every emitted token is appended at hist[b, pos[b] + 1 ...], so
// hist[b, :pos[b] + 1] stays the row's history.  draft_pos may be nullptr.
// score_out / logit_out (generate(output_scores / output_logits), each may be null): [max_new, B, V]; every slot that emits
// a token writes, at the token's column, its p row's score row (store_scores, with warp_weights' threshold) and raw logits.
// One CTA per SM (the fp32 vocabulary fills shared memory): asking for it lets ptxas go past 32 registers without spilling.
__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
accept_kernel(const __nv_bfloat16* __restrict__ plog, long long ldp, const __nv_bfloat16* __restrict__ qlog, long long ldq, int V,
              int K, const long long* __restrict__ ictl, const float* __restrict__ fctl, long long* __restrict__ tok,
              int* __restrict__ pos, int* __restrict__ gen, int* __restrict__ finished, long long* __restrict__ out, int ld_out,
              int max_new, int* __restrict__ draft_pos, long long* __restrict__ stats, const int* __restrict__ cnt,
              int* __restrict__ hist, int ldh, float* __restrict__ score_out, __nv_bfloat16* __restrict__ logit_out) {
  extern __shared__ __align__(16) float e[];
  __shared__ float red[33];
  __shared__ ArgMax am[32];
  __shared__ int tok_sm;
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, B = gridDim.x, tid = threadIdx.x;
  if (finished[b]) {
    if (tid == 0 && draft_pos != nullptr) draft_pos[b] = pos[b];
    return;
  }
  const bool greedy = !(ictl[0] != 0 && ictl[1] != 1);
  const int top_k = (int)ictl[1];
  const float temp = fctl[0], top_p = fctl[1], min_p = fctl[3];
  const int g0 = gen[b];
  const int c = cnt != nullptr ? min(max(cnt[b], 0), K) : K;   // candidates of this row
  int n_acc = 0, t_new = 0;
  bool stopped = false;                          // an accepted proposal before slot i is an EOS id
  for (int i = 0; i <= c; ++i) {
    const __nv_bfloat16* prow = plog + ((long long)i * B + b) * ldp;
    const ArgMax pm = block_argmax(prow, V, am);
    const long long d = i < c ? tok[(long long)(i + 1) * B + b] : -1;
    // every slot the loop reaches emits one token; it lands in column g0 + i unless an EOS id came first
    if (i > 0)
      for (int k = 0; k < (int)min(ictl[4], (long long)MAX_EOS); ++k) stopped |= tok[(long long)i * B + b] == ictl[5 + k];
    ScoreOut so{nullptr, nullptr};
    if (!stopped && g0 + i < max_new) {
      const long long at = ((long long)(g0 + i) * B + b) * V;
      if (score_out != nullptr) so.score = score_out + at;
      if (logit_out != nullptr) so.logit = logit_out + at;
    }
    if (greedy) {
      if (so.score != nullptr || so.logit != nullptr)
        store_scores(RawLogit{prow}, prow, V, ictl[0] != 0 ? SCORE_ARGMAX : SCORE_RAW, temp, 0.f, 0u, pm.i, so);
      if (d == pm.i) {
        ++n_acc;
        continue;
      }
      t_new = pm.i;
      break;
    }
    const float mxp = pm.v / temp;
    const uint32_t Tp = warp_weights(prow, V, temp, top_k, top_p, min_p, mxp, e, red);
    if (so.score != nullptr || so.logit != nullptr) store_scores(RawLogit{prow}, prow, V, SCORE_WARPED, temp, mxp, Tp, 0, so);
    curandStatePhilox4_32_10_t rng;
    curand_init((unsigned long long)ictl[2], (unsigned long long)b, (unsigned long long)g0 * 16ull + 2ull * i, &rng);
    const float u_acc = curand_uniform(&rng), u_draw = curand_uniform(&rng);    // (0, 1]
    if (i == c) {                                // no proposal left (assisted: all K accepted): draw from p_c
      t_new = draw_index(e, V, u_acc, pm.i, red, &tok_sm);
      break;
    }
    float zp = 0.f;
    for (int v = tid; v < V; v += blockDim.x) zp += e[v];
    zp = block_sum(zp, red);
    const float pd = e[d] / zp;
    if (qlog == nullptr) {                       // point mass: accept with probability p(d), else draw from p without d
      if (pd > 0.f && u_acc <= pd) {
        ++n_acc;
        continue;
      }
      __syncthreads();                           // every thread has read e[d]
      if (tid == 0) e[d] = 0.f;
      __syncthreads();
      // fallback of draw_index (r outside every segment by rounding): the residual's largest weight, never d itself
      ArgMax fb = {-INFINITY, V};
      for (int v = tid; v < V; v += blockDim.x) fb = argmax_merge(fb, ArgMax{e[v], v});
      fb = block_reduce_argmax(fb, am);
      t_new = draw_index(e, V, u_draw, fb.i, red, &tok_sm);
      break;
    }
    const __nv_bfloat16* qrow = qlog + ((long long)i * B + b) * ldq;
    const ArgMax qm = block_argmax(qrow, V, am);   // starts with a barrier: every thread has read e[d]
    warp_weights(qrow, V, temp, top_k, top_p, min_p, qm.v / temp, e, red);
    float zq = 0.f;
    for (int v = tid; v < V; v += blockDim.x) zq += e[v];
    zq = block_sum(zq, red);
    const float qd = e[d] / zq;
    if (pd > 0.f && u_acc * qd <= pd) {
      ++n_acc;
      continue;
    }
    // rejected: residual max(0, p - q), p recomputed from the logits with the same expression and threshold
    for (int v = tid; v < V; v += blockDim.x) {
      const float w = warped_weight(__bfloat162float(prow[v]), temp, mxp);
      const float pv = __float_as_uint(w) >= Tp ? w / zp : 0.f;
      e[v] = fmaxf(pv - e[v] / zq, 0.f);
    }
    __syncthreads();
    t_new = draw_index(e, V, u_draw, pm.i, red, &tok_sm);
    break;
  }
  if (tid == 0) {
    const int n_eos = (int)min(ictl[4], (long long)MAX_EOS);
    int g = g0;
    bool fin = false;
    for (int t = 0; t <= n_acc && !fin && g < max_new; ++t) {
      const long long x = t < n_acc ? tok[(long long)(t + 1) * B + b] : (long long)t_new;
      out[(long long)b * ld_out + g] = x;
      if (hist != nullptr && pos[b] + 1 + t < ldh) hist[(long long)b * ldh + pos[b] + 1 + t] = (int)x;
      ++g;
      for (int k = 0; k < n_eos; ++k)
        if (x == ictl[5 + k]) fin = true;
    }
    fin = fin || g >= max_new;
    stats[2 * b] += 1;
    stats[2 * b + 1] += n_acc;
    if (fin) finished[b] = 1;
    else pos[b] += n_acc + 1;
    gen[b] = g;
    tok[b] = t_new;
    if (draft_pos != nullptr) draft_pos[b] = pos[b];
  }
}

// ------------------------------------------------------------------------------------------------ prompt lookup
// One CTA per row: the proposals of one prompt-lookup round (transformers' PromptLookupCandidateGenerator).  Row b's history
// is h = hist[b, :L], L = pos[b] + 1.  For n from min(ngram, L - 1) down to 1, the earliest start s with h[s, s+n) equal to
// the last n tokens h[L-n, L) and s + n < L (a block-wide minimum over the starts, one pass per n); the first n with such an
// s wins.  Its candidates are h[s+n, min(s+n+K, L)), cut before the first EOS id of ictl.  They go to tok slots 1..c
// (slot j of row b: tok[j*B + b]); slots c+1..K get the filler id 0.  cnt[b] = c, proposed[b] += c.  Finished rows are left
// alone.  Every setting is a kernel argument or lives in device memory, so a captured round graph serves every round.
constexpr int LOOKUP_THREADS = 256;

__global__ void __launch_bounds__(LOOKUP_THREADS)
lookup_propose_kernel(const int* __restrict__ hist, int ldh, const int* __restrict__ pos, const int* __restrict__ finished,
                      const long long* __restrict__ ictl, long long* __restrict__ tok, int* __restrict__ cnt,
                      long long* __restrict__ proposed, int K, int ngram) {
  __shared__ int suffix[64];                     // the last n tokens (n <= MAX_NGRAM = 64)
  __shared__ int best;
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, B = gridDim.x, tid = threadIdx.x;
  if (finished[b]) return;
  const int* h = hist + (long long)b * ldh;
  const int L = min(pos[b] + 1, ldh);
  int s_win = -1, n_win = 0;
  for (int n = min(min(ngram, L - 1), 64); n >= 1; --n) {
    if (tid < n) suffix[tid] = h[L - n + tid];
    if (tid == 0) best = INT_MAX;
    __syncthreads();
    for (int s = tid; s + n < L; s += blockDim.x) {            // the first match of each thread is its smallest
      bool eq = true;
      for (int k = 0; k < n && eq; ++k) eq = h[s + k] == suffix[k];
      if (eq) {
        atomicMin(&best, s);
        break;
      }
    }
    __syncthreads();
    const int s = best;
    __syncthreads();                             // every thread has read best and suffix before the next pass
    if (s != INT_MAX) {
      s_win = s;
      n_win = n;
      break;
    }
  }
  if (tid == 0) {
    int c = 0;
    if (s_win >= 0) {
      const int start = s_win + n_win, n_eos = (int)min(ictl[4], (long long)MAX_EOS);
      const int end = min(start + K, L);
      for (int i = start; i < end; ++i) {
        bool is_eos = false;
        for (int k = 0; k < n_eos; ++k) is_eos |= (long long)h[i] == ictl[5 + k];
        if (is_eos) break;
        ++c;
      }
    }
    for (int j = 0; j < K; ++j) tok[(long long)(j + 1) * B + b] = j < c ? (long long)h[s_win + n_win + j] : 0ll;
    cnt[b] = c;
    proposed[b] += c;
  }
}

// ------------------------------------------------------------------------------------------------ beam search
// Deterministic beam search as transformers' GenerationMixin._beam_search (do_sample=False), one step per generated token:
// beam_topk + beam_step select, beam_reorder shares the history of the selected parents through a per-row chunk table.
constexpr int MAX_BEAMS = 8;
constexpr int MAX_KEEP = (1 + MAX_EOS) * MAX_BEAMS;  // beams_to_keep = max(2, 1 + n_eos) * num_beams
constexpr int MAX_TABLE = 256;                       // chunks of 128 positions per row: Smax <= 32768
constexpr int TOPK_THREADS = 128;
constexpr int TOPK_PER = 8;
constexpr int TOPK_SPLIT = TOPK_THREADS * TOPK_PER;  // vocabulary entries per beam_topk CTA
constexpr int STEP_THREADS = 512;                    // beam_step: one thread per (beam, split) candidate list
constexpr float NEG = -1.0e9f;                       // HF's score offset of a continuation that must not be chosen

// The K best of the entries in `avail` (bit e: key[e] of this thread, entry base + 128*e + tid), by value descending and
// then index ascending, to cv / ci[0..K) (index -1, value -inf once none is left).
__device__ __forceinline__ void split_topk(const float* key, unsigned avail, int base, int K, ArgMax* am, float* __restrict__ cv, int* __restrict__ ci) {
  const int tid = threadIdx.x;
  for (int k = 0; k < K; ++k) {
    ArgMax best{-INFINITY, INT_MAX};
#pragma unroll
    for (int e = 0; e < TOPK_PER; ++e)
      if ((avail >> e) & 1u) best = argmax_merge(best, ArgMax{key[e], base + e * TOPK_THREADS + tid});
    best = block_reduce_argmax(best, am);
    const bool none = best.i == INT_MAX;
    if (!none && (best.i - base) % TOPK_THREADS == tid) avail &= ~(1u << ((best.i - base) / TOPK_THREADS));
    if (tid == 0) {
      cv[k] = none ? -INFINITY : best.v;
      ci[k] = none ? -1 : best.i;
    }
  }
}

// grid (splits, rows), block 128.  Split s of row r is logits[r, s*1024 .. s*1024 + 1024); thread t holds entries
// s*1024 + 128*e + t in registers.  Writes part_ml[r][s] = (max, sum exp(x - max)) in fp32 and cand[r][s][0..K) = the
// split's K largest logits, by value descending and then index ascending (index -1, value -inf past the split's end).
// Within one row this is also the order of the log-probabilities.  cand rows hold ck >= K entries.
//
// With the logits processors on (fctl not null and the control blocks turn them on), the row's history is its prompt
// (prompt[g, 0 .. plens[g]), g = r / nb) followed by run_seq[tstep[g] & 1][r, 0 .. tstep[g]), and ck >= 2K.  A penalised
// token's log-prob (z - lse) * p is monotone in z within the penalised tokens, but not against the others, so the split
// gives two lists: cand[..][0..K) the best of the unpenalised tokens, with the banned ones (any class) as -inf, and
// cand[..][K..2K) the best of the penalised tokens that are not banned, by their raw logits.  beam_step maps and merges them.
//
// With a sequence table (tab_off not null, ictl[CTL_N_SEQ] > 0), a biased token (z - lse + bias, then maybe penalised) is
// monotone with neither list, so the biased tokens that are not banned leave both lists.  The split owns the table entries
// whose last token it holds, and writes slot [r][e] of each: for the first matched bias entry of a token, the token (with
// SLOT_PEN when it is penalised), its raw logit and its summed bias (seq_bias_sum); -1 for every other entry.  Every slot
// below ictl[CTL_N_SEQ] is written every step, so nothing needs clearing; beam_step scores the slots exactly.
constexpr int SLOT_PEN = 1 << 30;
__global__ void __launch_bounds__(TOPK_THREADS)
beam_topk_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V, int K, int ck, float* __restrict__ part_ml,
                 float* __restrict__ cand_v, int* __restrict__ cand_i, const long long* __restrict__ ictl, const float* __restrict__ fctl,
                 const int* __restrict__ prompt, int ldp, const int* __restrict__ plens, const int* __restrict__ run_seq,
                 const int* __restrict__ tstep, int nb, int max_new, const int* __restrict__ tab_off, const float* __restrict__ tab_bias,
                 int* __restrict__ slot_i, float2* __restrict__ slot_v) {
  __shared__ float red[33];
  __shared__ ArgMax am[32];
  __shared__ unsigned pen_sm[TOPK_SPLIT / 32], ban_sm[TOPK_SPLIT / 32], bsd_sm[TOPK_SPLIT / 32], matched[MAX_SEQS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x, r = blockIdx.y, ns = gridDim.x, tid = threadIdx.x;
  const int base = s * TOPK_SPLIT;
  const __nv_bfloat16* row = logits + (long long)r * ld;
  float x[TOPK_PER];
  float mx = -INFINITY;
#pragma unroll
  for (int e = 0; e < TOPK_PER; ++e) {
    const int i = base + e * TOPK_THREADS + tid;
    const float v = i < V ? __bfloat162float(row[i]) : -INFINITY;
    x[e] = v == v ? v : -INFINITY;               // NaN is never preferred
    mx = fmaxf(mx, x[e]);
  }
  mx = block_max(mx, red);
  float se = 0.f;
  if (mx > -INFINITY) {
#pragma unroll
    for (int e = 0; e < TOPK_PER; ++e) se += expf(x[e] - mx);
  }
  se = block_sum(se, red);
  const long long rs = (long long)r * ns + s;
  if (tid == 0) {
    part_ml[2 * rs] = mx;
    part_ml[2 * rs + 1] = se;
  }
  unsigned valid = 0u;                           // bit e: entry e of this thread is inside the vocabulary
#pragma unroll
  for (int e = 0; e < TOPK_PER; ++e)
    if (base + e * TOPK_THREADS + tid < V) valid |= 1u << e;
  if (fctl == nullptr || !processors_on(ictl, fctl)) {
    split_topk(x, valid, base, K, am, cand_v + rs * ck, cand_i + rs * ck);
    return;
  }
  // ---- processors: this split's bits of the row's penalised and banned tokens
  const int g = r / nb, t = tstep[g], rows = gridDim.y;
  const SeqTable tab{tab_off, tab_bias, tab_off != nullptr ? (int)min(ictl[CTL_N_SEQ], (long long)MAX_SEQS) : 0};
  for (int i = tid; i < TOPK_SPLIT / 32; i += TOPK_THREADS) pen_sm[i] = ban_sm[i] = bsd_sm[i] = 0u;
  for (int i = tid; i < MAX_SEQS / 32; i += TOPK_THREADS) matched[i] = 0u;
  __syncthreads();
  const float p = fctl[2];
  const History h{prompt + (long long)g * ldp, run_seq + ((long long)(t & 1) * rows + r) * max_new, plens[g], plens[g] + t};
  mark_history(h, base, base + TOPK_SPLIT, p != 1.f, (int)ictl[CTL_NGRAM], t < ictl[CTL_MIN_NEW] || h.L < ictl[CTL_MIN_LEN], ictl,
               pen_sm, ban_sm);
  if (tab.n > 0) mark_sequences(tab, h, base, base + TOPK_SPLIT, ban_sm, bsd_sm, matched);
  __syncthreads();
  for (int e = tid; e < tab.n; e += TOPK_THREADS) {
    const int v = tab.last(e);
    if (v < base || v >= base + TOPK_SPLIT) continue;
    const int j = v - base;
    float sum;
    int si = -1;
    if (((matched[e >> 5] >> (e & 31)) & 1u) && !((ban_sm[j >> 5] >> (j & 31)) & 1u) && seq_bias_sum(tab, matched, nullptr, e, v, sum)) {
      const float z = __bfloat162float(row[v]);
      si = v | (((pen_sm[j >> 5] >> (j & 31)) & 1u) ? SLOT_PEN : 0);
      slot_v[(long long)r * MAX_SEQS + e] = make_float2(z == z ? z : -INFINITY, sum);
    }
    slot_i[(long long)r * MAX_SEQS + e] = si;
  }
  unsigned in_pen = 0u;
#pragma unroll
  for (int e = 0; e < TOPK_PER; ++e) {
    const int j = e * TOPK_THREADS + tid;
    const unsigned bit = 1u << (j & 31);
    if (ban_sm[j >> 5] & bit) x[e] = -INFINITY;
    else if (bsd_sm[j >> 5] & bit) valid &= ~(1u << e);       // scored by beam_step from its slot
    else if (pen_sm[j >> 5] & bit) in_pen |= 1u << e;
  }
  in_pen &= valid;
  split_topk(x, valid & ~in_pen, base, K, am, cand_v + rs * ck, cand_i + rs * ck);
  split_topk(x, in_pen, base, K, am, cand_v + rs * ck + K, cand_i + rs * ck + K);
}

// generate(output_scores=True): the beam indices [2][rows][max_new] (int32, -1 past a hypothesis' end), double-buffered
// and gathered through the same sources as run_seq / fin_seq; a candidate's entry at t is its parent's global row.  Out of
// line, so beam_step keeps its registers.
__device__ __noinline__ void beam_indices_step(int* __restrict__ run_bi, int* __restrict__ fin_bi, int row0, int nb, int t, long long M,
                                               long long rows, int V, const int* sel_f, const int* run_src, const int* fin_src) {
  const int* rsrc = run_bi + (t & 1) * rows * M;
  int* rdst = run_bi + ((t & 1) ^ 1) * rows * M;
  const int* fsrc = fin_bi + (t & 1) * rows * M;
  int* fdst = fin_bi + ((t & 1) ^ 1) * rows * M;
  const int n = t + 1;
  for (int i = threadIdx.x; i < nb * n; i += blockDim.x) {
    const int j = i / n, c = i % n;
    const int f = sel_f[run_src[j]];
    rdst[(row0 + j) * M + c] = c < t ? rsrc[(row0 + f / V) * M + c] : row0 + f / V;
    const int m = fin_src[j];
    int v;
    if (m < nb) {
      v = fsrc[(row0 + m) * M + c];
    } else {
      const int fk = sel_f[m - nb];
      v = c < t ? rsrc[(row0 + fk / V) * M + c] : row0 + fk / V;
    }
    fdst[(row0 + j) * M + c] = v;
  }
}

// The log-sum-exp of one beam row from its beam_topk partials ml [ns][2], computed by one whole warp (every lane gets it).
// beam_step and beam_scores both call it, so the scores equal the selection's values bit for bit.
__device__ __forceinline__ float beam_row_lse(const float* __restrict__ ml, int ns) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int s = lane; s < ns; s += 32) m = fmaxf(m, ml[2 * s]);
  m = warp_max(m);
  float z = 0.f;
  for (int s = lane; s < ns; s += 32)
    if (ml[2 * s] > -INFINITY) z += ml[2 * s + 1] * expf(ml[2 * s] - m);
  z = warp_sum(z);
  return m + logf(z);
}

// One CTA per prompt g, whose beams are rows g*nb .. g*nb + nb-1.  One step of HF's beam search (t = tokens generated so
// far, tstep[g]):
//   c. score = logit - lse(row) + run_score(row); the K best over all beams (ties: lower beam * V + token), by a K-way
//      merge of the nb * splits sorted lists of beam_topk
//   d. a candidate hits the stopping criteria if its token is an EOS id (ictl, as the sampler) or t + 1 == max_new
//   e. the next running beams: the nb best of score + hit * -1e9
//   f. the finished hypotheses: the nb best of the old ones and score / (t+1)^length_penalty, plus -1e9 when the prompt's
//      finished set is full (early_stopping True), when the early-stop heuristic is satisfied, and for every candidate that
//      is not among the first nb or did not hit the stopping criteria
//   g. the early-stop heuristic (early_stopping: 0 False, 1 True, 2 "never") and done[g]
// Histories are int32 [2][rows][max_new], double-buffered by the parity of t: step t reads buffer t & 1 and writes the
// other one, so beams may swap parents.  Writes ids_next / parent (global row) / run_score of the new running beams, pos
// += 1, and the finished scores, flags and histories.  A prompt that is done is left untouched (parents = itself).
// Candidate rows hold ck entries.  With the logits processors on (fctl not null; see beam_topk_kernel) each thread also
// owns the split's penalised list, scored penalise(logit - lse, p) + run_score, and offers the better of its two heads.
// With a sequence table (slot_i not null, ictl[CTL_N_SEQ] = n > 0) thread l also owns the slots l, l + 512, ... of the
// prompt's nb * n (beam, entry) slots: each valid one is a candidate scored (logit - lse) + bias, penalised when marked,
// + run_score; the thread offers the best of its untaken ones too.
__global__ void __launch_bounds__(STEP_THREADS)
beam_step_kernel(const float* __restrict__ part_ml, const float* __restrict__ cand_v, const int* __restrict__ cand_i, int ns, int V,
                 int nb, int K, int ck, const long long* __restrict__ ictl, const float* __restrict__ fctl, float length_penalty,
                 int early_stopping, int max_new, float* __restrict__ run_score, float* __restrict__ fin_score, int* __restrict__ fin_flag,
                 int* __restrict__ run_seq, int* __restrict__ fin_seq, int* __restrict__ unsat, int* __restrict__ done,
                 int* __restrict__ tstep, int* __restrict__ pos, long long* __restrict__ ids_next, int* __restrict__ parent,
                 const int* __restrict__ slot_i, const float2* __restrict__ slot_v, int* __restrict__ run_bi, int* __restrict__ fin_bi) {
  __shared__ ArgMax am[32];
  __shared__ float lse[MAX_BEAMS];
  __shared__ float sel_v[MAX_KEEP], fcand[MAX_KEEP];
  __shared__ int sel_f[MAX_KEEP], hit[MAX_KEEP], taken[MAX_BEAMS + MAX_KEEP];
  __shared__ int run_src[MAX_BEAMS], fin_src[MAX_BEAMS], new_ff[MAX_BEAMS];
  __shared__ float new_rs[MAX_BEAMS], new_fs[MAX_BEAMS];
  pdl_launch_dependents();
  pdl_wait();
  const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row0 = g * nb;
  if (done[g]) {
    if (tid < nb) parent[row0 + tid] = row0 + tid;
    return;
  }
  const int t = tstep[g];

  // ---- log-sum-exp of each beam row from the split partials: warp j takes row j
  if (warp < nb) {
    const float l = beam_row_lse(part_ml + (long long)(row0 + warp) * ns * 2, ns);
    if (lane == 0) lse[warp] = l;
  }
  __syncthreads();

  // ---- c. K-way merge: thread l owns the sorted list of beam l / ns, split l % ns; its head advances when it wins
  const int nl = nb * ns, jb = tid / ns, sp = tid % ns;
  const bool two = fctl != nullptr && processors_on(ictl, fctl);
  const float pen = two ? fctl[2] : 1.f;
  const int nseq = two && slot_i != nullptr ? (int)min(ictl[CTL_N_SEQ], (long long)MAX_SEQS) : 0;
  int head = 0, head2 = 0;
  unsigned taken3 = 0u;                          // bit m: slot tid + m * STEP_THREADS was selected (nb * nseq <= 16 * 512)
  for (int k = 0; k < K; ++k) {
    ArgMax c{-INFINITY, INT_MAX};
    int src = 0;                                 // 0: first list, 1: penalised list, 2 + m: slot m of this thread
    if (tid < nl) {
      const long long at = ((long long)(row0 + jb) * ns + sp) * ck;
      if (head < K) {
        const int ci = cand_i[at + head];
        if (ci >= 0) c = ArgMax{(cand_v[at + head] - lse[jb]) + run_score[row0 + jb], jb * V + ci};
      }
      if (two && head2 < K) {
        const int ci = cand_i[at + K + head2];
        if (ci >= 0) {
          const ArgMax c2{penalise(cand_v[at + K + head2] - lse[jb], pen) + run_score[row0 + jb], jb * V + ci};
          if (argmax_merge(c, c2).i == c2.i) {
            c = c2;
            src = 1;
          }
        }
      }
    }
    for (int m = 0, q = tid; q < nb * nseq; ++m, q += STEP_THREADS) {
      if ((taken3 >> m) & 1u) continue;
      const int jq = q / nseq;
      const long long at = (long long)(row0 + jq) * MAX_SEQS + q % nseq;
      const int si = slot_i[at];
      if (si < 0) continue;
      const float2 zb = slot_v[at];
      float v = __fadd_rn(zb.x - lse[jq], zb.y);
      if (si & SLOT_PEN) v = penalise(v, pen);
      const ArgMax c3{v + run_score[row0 + jq], jq * V + (si & (SLOT_PEN - 1))};
      if (argmax_merge(c, c3).i == c3.i) {
        c = c3;
        src = 2 + m;
      }
    }
    const ArgMax w = block_reduce_argmax(c, am);
    if (c.i != INT_MAX && w.i == c.i) {          // beam * V + token is unique to one list or slot
      if (src >= 2) taken3 |= 1u << (src - 2);
      else if (src == 1) ++head2;
      else ++head;
    }
    if (tid == 0) {
      sel_v[k] = w.v;
      sel_f[k] = w.i;
    }
  }
  __syncthreads();

  // ---- d-g: K <= 72 candidates and nb <= 8 beams, one thread
  if (tid == 0) {
    const int n_eos = (int)min(ictl[4], (long long)MAX_EOS);
    const bool last = t + 1 >= max_new;
    for (int k = 0; k < K; ++k) {
      const long long tok = sel_f[k] % V;
      bool h = last;
      for (int e = 0; e < n_eos; ++e) h = h || tok == ictl[5 + e];
      hit[k] = h;
      taken[k] = 0;
    }
    // e. running beams: the nb best of score + hit * -1e9, ties to the lower candidate
    for (int j = 0; j < nb; ++j) {
      int bk = -1;
      float bv = -INFINITY;
      for (int k = 0; k < K; ++k) {
        if (taken[k]) continue;
        const float v = hit[k] ? sel_v[k] + NEG : sel_v[k];
        if (bk < 0 || v > bv) { bk = k; bv = v; }
      }
      taken[bk] = 1;
      run_src[j] = bk;
      new_rs[j] = bv;
    }
    // f. finished hypotheses: merge the old nb with the K candidates, keep the nb best (ties to the lower merged index)
    const float denom = (float)pow((double)(t + 1), (double)length_penalty);
    bool full = early_stopping == 1;
    for (int j = 0; j < nb; ++j) full = full && fin_flag[row0 + j] != 0;
    const bool uns = unsat[g] != 0;
    for (int k = 0; k < K; ++k) {
      float f = __fdiv_rn(sel_v[k], denom);
      if (full) f += NEG;
      if (!uns) f += NEG;
      if (!(hit[k] && k < nb)) f += NEG;
      fcand[k] = f;
    }
    for (int m = 0; m < nb + K; ++m) taken[m] = 0;
    for (int j = 0; j < nb; ++j) {
      int bm = -1;
      float bv = -INFINITY;
      for (int m = 0; m < nb + K; ++m) {
        if (taken[m]) continue;
        const float v = m < nb ? fin_score[row0 + m] : fcand[m - nb];
        if (bm < 0 || v > bv) { bm = m; bv = v; }
      }
      taken[bm] = 1;
      fin_src[j] = bm;
      new_fs[j] = bv;
      new_ff[j] = bm < nb ? fin_flag[row0 + bm] != 0 : (hit[bm - nb] && bm - nb < nb);
    }
    // g. early-stop heuristic on the new running and finished beams, at length t + 1
    const int best_len = (early_stopping == 2 && length_penalty > 0.f) ? max_new : t + 1;
    const float best_possible = __fdiv_rn(new_rs[0], (float)pow((double)best_len, (double)length_penalty));
    float worst = new_fs[0];
    bool all_fin = true;
    for (int j = 0; j < nb; ++j) {
      worst = fminf(worst, new_fs[j]);
      all_fin = all_fin && new_ff[j];
    }
    bool improvable = false;
    for (int j = 0; j < nb; ++j) improvable = improvable || best_possible > (new_ff[j] ? worst : NEG);
    const bool u = uns && improvable;
    unsat[g] = u;
    done[g] = !u || (early_stopping == 1 && all_fin) || last;
  }
  __syncthreads();

  // ---- histories [0, t] of the new running and finished beams, gathered through their sources
  const long long M = max_new, rows = (long long)gridDim.x * nb;
  const int* rsrc = run_seq + (t & 1) * rows * M;
  int* rdst = run_seq + ((t & 1) ^ 1) * rows * M;
  const int* fsrc = fin_seq + (t & 1) * rows * M;
  int* fdst = fin_seq + ((t & 1) ^ 1) * rows * M;
  const int n = t + 1;
  for (int i = tid; i < nb * n; i += blockDim.x) {
    const int j = i / n, c = i % n;
    const int f = sel_f[run_src[j]];
    rdst[(row0 + j) * M + c] = c < t ? rsrc[(row0 + f / V) * M + c] : f % V;
    const int m = fin_src[j];
    int v;
    if (m < nb) {
      v = fsrc[(row0 + m) * M + c];
    } else {
      const int fk = sel_f[m - nb];
      v = c < t ? rsrc[(row0 + fk / V) * M + c] : fk % V;
    }
    fdst[(row0 + j) * M + c] = v;
  }
  if (run_bi != nullptr) beam_indices_step(run_bi, fin_bi, row0, nb, t, M, rows, V, sel_f, run_src, fin_src);
  if (tid < nb) {
    const int f = sel_f[run_src[tid]];
    run_score[row0 + tid] = new_rs[tid];
    parent[row0 + tid] = row0 + f / V;
    ids_next[row0 + tid] = f % V;
    pos[row0 + tid] += 1;
    fin_score[row0 + tid] = new_fs[tid];
    fin_flag[row0 + tid] = new_ff[tid];
  }
  if (tid == 0) tstep[g] = t + 1;
}

// generate(num_beams > 1, output_scores / output_logits): HF's per-step log_probs of every beam row, launched between
// beam_topk and beam_step.  grid (splits, rows), block 128, split s of row r as in beam_topk.  For a prompt g that is not
// done, column t = tstep[g] of score_out fp32 [max_new, rows, V] gets, per token, the value beam_step ranks before it adds
// the running score: z - lse (lse from the partials, as beam_step computes it), + the token's summed sequence bias, then
// penalise() when the token is in the history, -inf when banned (the same device helpers and bitmaps as beam_topk; z NaN
// counts as -inf).  logit_out bf16 [max_new, rows, V] gets the raw logits.  Either may be nullptr.
__global__ void __launch_bounds__(TOPK_THREADS)
beam_scores_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V, const float* __restrict__ part_ml,
                   const long long* __restrict__ ictl, const float* __restrict__ fctl, const int* __restrict__ prompt, int ldp,
                   const int* __restrict__ plens, const int* __restrict__ run_seq, const int* __restrict__ tstep,
                   const int* __restrict__ done, int nb, int max_new, const int* __restrict__ tab_off,
                   const float* __restrict__ tab_bias, float* __restrict__ score_out, __nv_bfloat16* __restrict__ logit_out) {
  __shared__ unsigned pen_sm[TOPK_SPLIT / 32], ban_sm[TOPK_SPLIT / 32], bsd_sm[TOPK_SPLIT / 32], matched[MAX_SEQS / 32];
  __shared__ float bias_sm[TOPK_SPLIT];
  __shared__ float lse;
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x, r = blockIdx.y, ns = gridDim.x, rows = gridDim.y, tid = threadIdx.x;
  const int g = r / nb, t = tstep[g], base = s * TOPK_SPLIT;
  if (done[g] || t >= max_new) return;
  const __nv_bfloat16* row = logits + (long long)r * ld;
  const long long at = ((long long)t * rows + r) * V;
  const bool proc = fctl != nullptr && processors_on(ictl, fctl);
  for (int i = tid; i < TOPK_SPLIT / 32; i += TOPK_THREADS) pen_sm[i] = ban_sm[i] = bsd_sm[i] = 0u;
  for (int i = tid; i < MAX_SEQS / 32; i += TOPK_THREADS) matched[i] = 0u;
  if (tid < 32) {
    const float l = beam_row_lse(part_ml + (long long)r * ns * 2, ns);
    if (tid == 0) lse = l;
  }
  __syncthreads();
  const float p = proc ? fctl[2] : 1.f;
  if (proc) {
    const SeqTable tab{tab_off, tab_bias, tab_off != nullptr ? (int)min(ictl[CTL_N_SEQ], (long long)MAX_SEQS) : 0};
    const History h{prompt + (long long)g * ldp, run_seq + ((long long)(t & 1) * rows + r) * max_new, plens[g], plens[g] + t};
    mark_history(h, base, base + TOPK_SPLIT, p != 1.f, (int)ictl[CTL_NGRAM], t < ictl[CTL_MIN_NEW] || h.L < ictl[CTL_MIN_LEN], ictl,
                 pen_sm, ban_sm);
    if (tab.n > 0) mark_sequences(tab, h, base, base + TOPK_SPLIT, ban_sm, bsd_sm, matched);
    __syncthreads();
    for (int e = tid; e < tab.n; e += TOPK_THREADS) {
      const int v = tab.last(e);
      float sum;
      if (v >= base && v < base + TOPK_SPLIT && ((matched[e >> 5] >> (e & 31)) & 1u) && seq_bias_sum(tab, matched, nullptr, e, v, sum))
        bias_sm[v - base] = sum;
    }
    __syncthreads();
  }
  for (int j = tid; j < TOPK_SPLIT; j += TOPK_THREADS) {
    const int i = base + j;
    if (i >= V) break;
    const __nv_bfloat16 raw = row[i];
    if (logit_out != nullptr) logit_out[at + i] = raw;
    if (score_out == nullptr) continue;
    const float z = __bfloat162float(raw);
    float v = (z == z ? z : -INFINITY) - lse;
    const unsigned bit = 1u << (j & 31);
    if (bsd_sm[j >> 5] & bit) v = __fadd_rn(v, bias_sm[j]);
    if (pen_sm[j >> 5] & bit) v = penalise(v, p);
    if (ban_sm[j >> 5] & bit) v = -INFINITY;
    score_out[at + i] = v;
  }
}

// grid (L * 2 * Hkv, B), block 256, dynamic shared memory nb * CH * 64 * 2 bytes.  kv [L][2][rows][Hkv][Smax][64]: CTA
// (x, g) serves slab x / Hkv (a layer's K or V) and kv head x % Hkv of prompt g, whose beams all sit at position p =
// pos[g*nb].  Chunks c < p / CH are complete and never written again, so a child whose parent is another row takes the
// parent's table entries for them; only the partial chunk [CH * (p / CH), p) is copied, from the parent's row (which owns
// its current chunk) to the child's own row, and the child's entry for that chunk becomes itself.  Every source is staged
// in shared memory before any destination is written (beams may swap parents); the table is updated by the CTAs x = 0.
// generate() ends with p = P + max_new_tokens - 1 < Smax; a position of Smax (a full cache) copies nothing and writes
// only entries below Smax / CH.  T is the cache element type, so a position is D * sizeof(T) bytes (128 bf16, 64 e4m3);
// an FP8 cache also moves the positions' inv [L][2][rows][Hkv][Smax] (staged after the bytes), read through the same table.
template <typename T>
__global__ void __launch_bounds__(256)
beam_reorder_kernel(T* __restrict__ kv, int* __restrict__ table, const int* __restrict__ parent,
                    const int* __restrict__ pos, int nb, int Hkv, int Smax, int nchunks, float* __restrict__ inv) {
  extern __shared__ __align__(16) uint4 stage[];  // [nb][CH * RV] (FP8: then fp32 [nb][CH] inv)
  __shared__ int tstage[MAX_BEAMS * MAX_TABLE];
  constexpr int RV = D * (int)sizeof(T) / 16;    // 16-byte pieces per position
  constexpr bool KV8 = sizeof(T) == 1;
  pdl_launch_dependents();
  pdl_wait();
  const int slab = blockIdx.x / Hkv, hk = blockIdx.x % Hkv, g = blockIdx.y, tid = threadIdx.x;
  const long long rows = (long long)gridDim.y * nb;
  const int row0 = g * nb;
  const int p = pos[row0], c = p / CH, n = p - c * CH;
  T* base = kv + (long long)slab * rows * Hkv * Smax * D;
  for (int j = 0; j < nb; ++j) {
    const int par = parent[row0 + j];
    if (par == row0 + j) continue;
    const uint4* src = reinterpret_cast<const uint4*>(base + (((long long)par * Hkv + hk) * Smax + c * CH) * D);
    for (int i = tid; i < n * RV; i += blockDim.x) stage[j * CH * RV + i] = src[i];
    if constexpr (KV8) {
      const float* isrc = inv + ((long long)slab * rows * Hkv + (long long)par * Hkv + hk) * Smax + c * CH;
      float* istage = reinterpret_cast<float*>(stage + nb * CH * RV) + j * CH;
      for (int i = tid; i < n; i += blockDim.x) istage[i] = isrc[i];
    }
  }
  if (blockIdx.x == 0)
    for (int i = tid; i < nb * c; i += blockDim.x) tstage[i] = table[parent[row0 + i / c] * nchunks + i % c];
  __syncthreads();
  for (int j = 0; j < nb; ++j) {
    if (parent[row0 + j] == row0 + j) continue;
    uint4* dst = reinterpret_cast<uint4*>(base + (((long long)(row0 + j) * Hkv + hk) * Smax + c * CH) * D);
    for (int i = tid; i < n * RV; i += blockDim.x) dst[i] = stage[j * CH * RV + i];
    if constexpr (KV8) {
      float* idst = inv + ((long long)slab * rows * Hkv + (long long)(row0 + j) * Hkv + hk) * Smax + c * CH;
      const float* istage = reinterpret_cast<const float*>(stage + nb * CH * RV) + j * CH;
      for (int i = tid; i < n; i += blockDim.x) idst[i] = istage[i];
    }
  }
  if (blockIdx.x == 0) {
    for (int i = tid; i < nb * (c + 1); i += blockDim.x) {
      const int j = i / (c + 1), cc = i % (c + 1);
      if (parent[row0 + j] == row0 + j || cc >= nchunks) continue;   // p == Smax: no current chunk to point at
      table[(row0 + j) * nchunks + cc] = cc < c ? tstage[j * c + cc] : row0 + j;
    }
  }
}

// ------------------------------------------------------------------------------------------------ multi-sample fork
// grid (L * 2 * Hkv, B), block 256.  Prompt g's n rows g*n .. g*n + n - 1 after its prefill into row g*n, which holds
// positions [0, p), p = len[g]: the children g*n + 1 .. take row g*n's table entries for the complete chunks c < p / CH
// and get a copy of the partial chunk [CH * (p / CH), p) (FP8 cache: with its inv) in their own row; every other entry
// of the n rows names the row itself.  (x, g) copies slab x / Hkv (a layer's K or V), kv head x % Hkv; the table is written
// by the CTAs x = 0.  The source row is never a destination, so nothing is staged and n is unbounded.
template <typename T>
__global__ void __launch_bounds__(256)
fork_kernel(T* __restrict__ kv, int* __restrict__ table, const int* __restrict__ len, int n, int Hkv, int Smax, int nchunks,
            float* __restrict__ inv) {
  constexpr int RV = D * (int)sizeof(T) / 16;    // 16-byte pieces per position
  pdl_launch_dependents();
  pdl_wait();
  const int slab = blockIdx.x / Hkv, hk = blockIdx.x % Hkv, g = blockIdx.y, tid = threadIdx.x;
  const long long rows = (long long)gridDim.y * n;
  const int src = g * n, p = min(len[g], Smax), c = p / CH, m = (p - c * CH) * RV;
  T* base = kv + (long long)slab * rows * Hkv * Smax * D;
  const uint4* s4 = reinterpret_cast<const uint4*>(base + (((long long)src * Hkv + hk) * Smax + c * CH) * D);
  for (int i = tid; i < (n - 1) * m; i += blockDim.x) {
    const int j = 1 + i / m, e = i % m;
    reinterpret_cast<uint4*>(base + (((long long)(src + j) * Hkv + hk) * Smax + c * CH) * D)[e] = s4[e];
  }
  if constexpr (sizeof(T) == 1) {
    const int mi = p - c * CH;
    float* ibase = inv + (long long)slab * rows * Hkv * Smax;
    const float* isrc = ibase + ((long long)src * Hkv + hk) * Smax + c * CH;
    for (int i = tid; i < (n - 1) * mi; i += blockDim.x) {
      const int j = 1 + i / mi, e = i % mi;
      ibase[((long long)(src + j) * Hkv + hk) * Smax + c * CH + e] = isrc[e];
    }
  }
  if (blockIdx.x == 0)
    for (int i = tid; i < n * nchunks; i += blockDim.x) {
      const int j = i / nchunks, cc = i % nchunks;
      table[(src + j) * nchunks + cc] = j > 0 && cc < c ? src : src + j;
    }
}

// The GQA-group dispatch of the attention launchers: f(std::integral_constant<int, G>{}) for G = Hq / Hkv.
template <class F>
int with_group(int G, F&& f) {
  switch (G) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
    default: return -2;                          // GQA groups of 1, 2, 4 or 8 query heads
  }
}

// The cache-type dispatch: f(T{}) with T = uint8_t for an FP8 cache (e4m3 bytes), __nv_bfloat16 for a bf16 one.
template <class F>
int with_cache(bool kv8, F&& f) {
  return kv8 ? f(uint8_t{}) : f(__nv_bfloat16{});
}

template <int G, typename T>
int launch_attn(const void* q, long long ldq, const void* kc, const void* vc, const void* pos, void* part_o, void* part_ml, void* out,
                long long ldo, const void* table, int B, int Hkv, int Smax, float scale, const void* kinv, const void* vinv,
                cudaStream_t st) {
  static bool attr_set = false;
  const int smem = AttSmem<G, T>::BYTES;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(decode_attn_kernel<G, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int nchunks = ceil_div(Smax, CH);
  launch_pdl(decode_attn_kernel<G, T>, dim3(nchunks, Hkv, B), dim3(ATT_THREADS), smem, st, (const __nv_bfloat16*)q, ldq,
             (const T*)kc, (const T*)vc, (const int*)pos, (float*)part_o, (float*)part_ml, (const int*)table, Hkv, Smax, nchunks,
             scale * 1.4426950408889634f, (const float*)kinv, (const float*)vinv);
  ODB_CHECK_LAST();
  launch_pdl(combine_kernel, dim3(Hkv * G, B), dim3(D), 0, st, (const float*)part_o, (const float*)part_ml, (const int*)pos,
             (__nv_bfloat16*)out, ldo, nchunks, CH, B);
  ODB_CHECK_LAST();
  return 0;
}

// Siblings per CTA of decode_attn_group_kernel.  A CTA runs its siblings one after the other, so fewer siblings per CTA
// buy parallelism with repeated loads of the shared chunks: at most max(1, 4 / G) siblings per CTA (the best of the splits
// measured at G 1 and G 8, profiles/README.md), and more CTAs while the (chunk, kv head, prompt, split) grid would not
// fill one wave of resident CTAs on the device.  splits > 0 forces the split (tests).
template <int G, typename T>
int attn_group_splits(int P, int ngrp, int Hkv, int nchunks) {
  static int wave = 0;
  if (wave == 0) {
    int dev, sms, per_sm;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess)
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decode_attn_group_kernel<G, T>, ATT_THREADS, AttSmem<G, T>::BYTES);
    if (e != cudaSuccess) return -(int)e;
    wave = sms * std::max(per_sm, 1);
  }
  const long long base = (long long)nchunks * Hkv * P;
  const int per = std::max(1, 4 / G);
  return (int)std::min<long long>(ngrp, std::max<long long>(ceil_div(ngrp, per), (wave + base - 1) / base));
}

template <int G, typename T>
int launch_attn_group(const void* q, long long ldq, const void* kc, const void* vc, const void* pos, void* part_o, void* part_ml,
                      void* out, long long ldo, const void* table, int rows, int ngrp, int Hkv, int Smax, float scale,
                      const void* kinv, const void* vinv, int splits, cudaStream_t st) {
  static bool attr_set = false;
  const int smem = AttSmem<G, T>::BYTES;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(decode_attn_group_kernel<G, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int nchunks = ceil_div(Smax, CH), P = rows / ngrp;
  if (splits <= 0) splits = attn_group_splits<G, T>(P, ngrp, Hkv, nchunks);
  if (splits <= 0) return -splits;
  splits = ceil_div(ngrp, ceil_div(ngrp, std::min(splits, ngrp)));   // no CTA without a sibling
  launch_pdl(decode_attn_group_kernel<G, T>, dim3(nchunks, Hkv, P * splits), dim3(ATT_THREADS), smem, st, (const __nv_bfloat16*)q,
             ldq, (const T*)kc, (const T*)vc, (const int*)pos, (float*)part_o, (float*)part_ml, (const int*)table, Hkv, Smax, nchunks,
             scale * 1.4426950408889634f, (const float*)kinv, (const float*)vinv, ngrp, splits);
  ODB_CHECK_LAST();
  launch_pdl(combine_kernel, dim3(Hkv * G, rows), dim3(D), 0, st, (const float*)part_o, (const float*)part_ml, (const int*)pos,
             (__nv_bfloat16*)out, ldo, nchunks, CH, rows);
  ODB_CHECK_LAST();
  return 0;
}

template <typename T>
int launch_beam_reorder(void* kv, void* inv, void* table, const void* parent, const void* pos, int B, int nb, int L, int Hkv, int Smax,
                        cudaStream_t st) {
  constexpr int extra = sizeof(T) == 1 ? CH * 4 : 0;                  // FP8: the staged inv of a position chunk
  const int smem = nb * (CH * D * (int)sizeof(T) + extra);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(beam_reorder_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         MAX_BEAMS * (CH * D * (int)sizeof(T) + extra));
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  launch_pdl(beam_reorder_kernel<T>, dim3(L * 2 * Hkv, B), dim3(256), smem, st, (T*)kv, (int*)table, (const int*)parent,
             (const int*)pos, nb, Hkv, Smax, Smax / CH, (float*)inv);
  ODB_CHECK_LAST();
  return 0;
}

}  // namespace dec

// Every cache argument below is either bf16 (kinv = vinv = nullptr) or an FP8 cache: e4m3 bytes of the same shape plus fp32
// kinv / vinv [B, Hkv, Smax] (16-byte aligned, Smax a multiple of 128), written and read as described at the top of the file.

// qkv [n*B, ld] bf16, slot-major (row j*B + b: token j of sequence b, at position pos[b] + j; n = 1: one token per row);
// cos/sin fp32 [max_pos, 32]; pos int32 [B]; kc/vc [B, Hkv, Smax, 64]
ODB_EXPORT int odb_dec_rope_append(void* qkv, long long ld, const void* cos_t, const void* sin_t, const void* pos, void* kc, void* vc,
                                   int B, int n, int Hq, int Hkv, int Smax, void* kinv, void* vinv, cudaStream_t st) {
  if (ld % 2 || n < 1) return -1;
  return dec::with_cache(kinv != nullptr, [&](auto t) {
    using T = decltype(t);
    launch_pdl(dec::rope_append_kernel<T>, dim3(B, n), dim3(256), 0, st, (__nv_bfloat16*)qkv, ld, (const float*)cos_t,
               (const float*)sin_t, (const int*)pos, (T*)kc, (T*)vc, Hq, Hkv, Smax, (float*)kinv, (float*)vinv);
    ODB_CHECK_LAST();
    return 0;
  });
}

// qkv [B*Sp, ld] bf16 (rotated prefill projections); len int32 [B]: rows s < len[b] are copied into cache row b * row_stride
ODB_EXPORT int odb_dec_kv_fill(const void* qkv, long long ld, const void* len, void* kc, void* vc, int B, int Sp, int Hq, int Hkv,
                               int Smax, int row_stride, void* kinv, void* vinv, cudaStream_t st) {
  if (ld % 8 || row_stride < 1) return -1;
  return dec::with_cache(kinv != nullptr, [&](auto t) {
    using T = decltype(t);
    launch_pdl(dec::kv_fill_kernel<T>, dim3(Sp, B), dim3(128), 0, st, (const __nv_bfloat16*)qkv, ld, (const int*)len, (T*)kc, (T*)vc,
               Sp, Hq, Hkv, Smax, row_stride, (float*)kinv, (float*)vinv);
    ODB_CHECK_LAST();
    return 0;
  });
}

// Number of key chunks of the split-KV attention for a cache of Smax positions (sizes the partial buffers).
ODB_EXPORT int odb_dec_attn_chunks(int Smax) { return odb::ceil_div(Smax, dec::CH); }

// q [B, ldq] bf16 (the q heads first); kc/vc [B, Hkv, Smax, 64]; pos int32 [B] (keys 0..pos[b] are attended);
// part_o fp32 [B, Hq, chunks, 64]; part_ml fp32 [B, Hq, chunks, 2]; out [B, ldo] bf16; table: nullptr, or int32 [B, chunks]
// (chunk c of row b is read from physical cache row table[b][c])
ODB_EXPORT int odb_dec_attn(const void* q, long long ldq, const void* kc, const void* vc, const void* pos, void* part_o, void* part_ml,
                            void* out, long long ldo, const void* table, int B, int Hq, int Hkv, int Smax, float softmax_scale,
                            const void* kinv, const void* vinv, cudaStream_t st) {
  if (Hq % Hkv || ldq % 8 || (kinv != nullptr && Smax % dec::CH)) return -1;
  return dec::with_group(Hq / Hkv, [&](auto g) {
    return dec::with_cache(kinv != nullptr, [&](auto t) {
      return dec::launch_attn<decltype(g)::value, decltype(t)>(q, ldq, kc, vc, pos, part_o, part_ml, out, ldo, table, B, Hkv, Smax,
                                                               softmax_scale, kinv, vinv, st);
    });
  });
}

// Multi-sample decode attention: as odb_dec_attn with a chunk table (required), over rows = P * ngrp rows where rows
// p * ngrp .. p * ngrp + ngrp - 1 are the siblings of prompt p; a chunk that siblings share through the table is loaded once
// per CTA.  The partials and out are bit-identical to odb_dec_attn's with the same table.  splits: 0 lets the launcher
// choose how many CTAs share a prompt's siblings (odb_dec_attn_group_splits; an FP8 cache at G = 1 runs odb_dec_attn through
// the table, which measured faster there), > 0 forces the grouped kernel with that split.  See dec::decode_attn_group_kernel.
ODB_EXPORT int odb_dec_attn_group(const void* q, long long ldq, const void* kc, const void* vc, const void* pos, void* part_o,
                                  void* part_ml, void* out, long long ldo, const void* table, int rows, int ngrp, int Hq, int Hkv,
                                  int Smax, float softmax_scale, const void* kinv, const void* vinv, int splits, cudaStream_t st) {
  if (Hq % Hkv || ldq % 8 || ngrp < 1 || rows % ngrp || table == nullptr || (kinv != nullptr && Smax % dec::CH)) return -1;
  if (splits <= 0 && kinv != nullptr && Hq == Hkv)   // measured: an FP8 cache at G = 1 reads faster through the table path
    return odb_dec_attn(q, ldq, kc, vc, pos, part_o, part_ml, out, ldo, table, rows, Hq, Hkv, Smax, softmax_scale, kinv, vinv, st);
  return dec::with_group(Hq / Hkv, [&](auto g) {
    return dec::with_cache(kinv != nullptr, [&](auto t) {
      return dec::launch_attn_group<decltype(g)::value, decltype(t)>(q, ldq, kc, vc, pos, part_o, part_ml, out, ldo, table, rows, ngrp,
                                                                     Hkv, Smax, softmax_scale, kinv, vinv, splits, st);
    });
  });
}

// The sibling split odb_dec_attn_group chooses for these shapes (CTAs per prompt and chunk; needs a device); 0: it runs
// odb_dec_attn through the table instead; < 0: an error.
ODB_EXPORT int odb_dec_attn_group_splits(int rows, int ngrp, int Hq, int Hkv, int Smax, int kv8) {
  if (ngrp < 1 || rows % ngrp || Hq % Hkv) return -1;
  if (kv8 && Hq == Hkv) return 0;
  const int P = rows / ngrp, nch = odb::ceil_div(Smax, dec::CH);
  int s = 0;
  const int rc = dec::with_group(Hq / Hkv, [&](auto g) {
    s = dec::with_cache(kv8 != 0, [&](auto t) { return dec::attn_group_splits<decltype(g)::value, decltype(t)>(P, ngrp, Hkv, nch); });
    return 0;
  });
  if (rc) return rc;
  return s <= 0 ? s - 1 : odb::ceil_div(ngrp, odb::ceil_div(ngrp, s));
}

// logits [B, ld] bf16; ictl / fctl: see dec::sample_kernel; pos / gen / finished int32 [B]; out int64 [B, max_new];
// ids_next int64 [B]; hist: nullptr (no logits processors), or int32 [B, ldh] with scratch int32 [B, 2 * ceil(V / 32)].
// score_out fp32 / logit_out bf16 [score_cols, B, V] (each may be nullptr): a live row's score row and raw logits at column
// gen[b] < score_cols (see dec::store_scores).  The vocabulary lives in shared memory as fp32: V <= 56000.
ODB_EXPORT int odb_dec_sample(const void* logits, long long ld, int V, const void* ictl, const void* fctl, void* pos, void* gen,
                              void* finished, void* out, int max_new, void* ids_next, void* hist, int ldh, void* scratch,
                              const void* tab_off, const void* tab_bias, void* seq_scratch, void* score_out, void* logit_out,
                              int score_cols, int B, cudaStream_t st) {
  if (tab_off != nullptr && (hist == nullptr || tab_bias == nullptr || seq_scratch == nullptr)) return -1;
  const int smem = V * 4;
  if (smem > 224000) return -1;
  static int attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(dec::sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    attr = smem;
  }
  launch_pdl(dec::sample_kernel, dim3(B), dim3(dec::SAMPLE_THREADS), smem, st, (const __nv_bfloat16*)logits, ld, V,
             (const long long*)ictl, (const float*)fctl, (int*)pos, (int*)gen, (int*)finished, (long long*)out, max_new,
             (long long*)ids_next, (int*)hist, ldh, (unsigned*)scratch, (const int*)tab_off, (const float*)tab_bias,
             (float*)seq_scratch, (float*)score_out, (__nv_bfloat16*)logit_out, score_cols);
  ODB_CHECK_LAST();
  return 0;
}

// q [n*B, ldq] bf16 slot-major (the q heads first); query row j*B + b attends keys 0..pos[b]+j; kc/vc [B, Hkv, Smax, 64]
// (Smax a multiple of 64); part_o fp32 [n*B, Hq, cap, 64]; part_ml fp32 [n*B, Hq, cap, 2] with cap = Smax / 64;
// out [n*B, ldo] bf16.  G = Hq / Hkv in {1, 2, 4, 8}, n <= 8 (G*n <= 64 queries: one m64 tile), pos[b] + n <= Smax.
// The keys are split so that about two CTAs per SM run: splits = min(tiles, ceil(264 / (Hkv*B))).
ODB_EXPORT int odb_dec_verify_attn(const void* q, long long ldq, const void* kc, const void* vc, const void* pos, void* part_o,
                                   void* part_ml, void* out, long long ldo, int B, int n, int Hq, int Hkv, int Smax, float softmax_scale,
                                   const void* kinv, const void* vinv, cudaStream_t st) {
  if (Hq % Hkv || ldq % 8 || n < 1 || n > 8 || Smax % dec::VB) return -1;
  const int G = Hq / Hkv;
  const int lg = G == 1 ? 0 : G == 2 ? 1 : G == 4 ? 2 : G == 8 ? 3 : -1;
  if (lg < 0) return -2;                         // GQA groups of 1, 2, 4 or 8 query heads
  const int cap = Smax / dec::VB;
  int splits = std::min(cap, std::max(1, odb::ceil_div(264, Hkv * B)));
  const int tps = odb::ceil_div(cap, splits);
  splits = odb::ceil_div(cap, tps);
  if (kinv != nullptr) {
    static bool attr8 = false;
    if (!attr8) {
      cudaError_t e = cudaFuncSetAttribute(dec::verify_attn_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dec::VSMEM8);
      if (e != cudaSuccess) return (int)e;
      attr8 = true;
    }
    CUtensorMap unused{};
    launch_pdl(dec::verify_attn_kernel<true>, dim3(splits, Hkv, B), dim3(dec::VTHREADS), dec::VSMEM8, st, unused, unused,
               (const __nv_bfloat16*)q, ldq, (const int*)pos, (float*)part_o, (float*)part_ml, Hkv, Smax, cap, tps,
               softmax_scale * 1.4426950408889634f, lg, n, (const uint8_t*)kc, (const uint8_t*)vc, (const float*)kinv,
               (const float*)vinv);
  } else {
    CUtensorMap tk, tv;
    int rc;
    const long long rows = (long long)B * Hkv * Smax;
    if ((rc = make_tmap_2d(&tk, kc, rows, dec::D, dec::D * 2, dec::VB, dec::D, 2))) return rc;
    if ((rc = make_tmap_2d(&tv, vc, rows, dec::D, dec::D * 2, dec::VB, dec::D, 2))) return rc;
    static bool attr_set = false;
    if (!attr_set) {
      cudaError_t e = cudaFuncSetAttribute(dec::verify_attn_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dec::VSMEM);
      if (e != cudaSuccess) return (int)e;
      attr_set = true;
    }
    launch_pdl(dec::verify_attn_kernel<false>, dim3(splits, Hkv, B), dim3(dec::VTHREADS), dec::VSMEM, st, tk, tv,
               (const __nv_bfloat16*)q, ldq, (const int*)pos, (float*)part_o, (float*)part_ml, Hkv, Smax, cap, tps,
               softmax_scale * 1.4426950408889634f, lg, n, (const uint8_t*)nullptr, (const uint8_t*)nullptr, (const float*)nullptr,
               (const float*)nullptr);
  }
  ODB_CHECK_LAST();
  launch_pdl(dec::combine_kernel, dim3(Hq, n * B), dim3(dec::D), 0, st, (const float*)part_o, (const float*)part_ml,
             (const int*)pos, (__nv_bfloat16*)out, ldo, cap, tps * dec::VB, B);
  ODB_CHECK_LAST();
  return 0;
}

// plog [(K+1)*B, ldp] / qlog [K*B, ldq] bf16 slot-major; tok int64 [(K+1)*B]; ictl / fctl: see dec::sample_kernel; pos / gen /
// finished / draft_pos int32 [B]; out int64 [B, ld_out]; stats int64 [B, 2].  V <= 56000 (fp32 vocabulary in shared memory).
// Point-mass mode (prompt lookup): qlog nullptr, cnt int32 [B] candidate counts, hist int32 [B, ldh] (or nullptr), draft_pos
// may be nullptr.  score_out fp32 / logit_out bf16 [max_new, B, V] (each may be nullptr): the score row and raw logits of
// the slot that emitted each token, at its column.  See dec::accept_kernel.
ODB_EXPORT int odb_dec_accept(const void* plog, long long ldp, const void* qlog, long long ldq, int V, int K, const void* ictl,
                              const void* fctl, void* tok, void* pos, void* gen, void* finished, void* out, int ld_out, int max_new,
                              void* draft_pos, void* stats, const void* cnt, void* hist, int ldh, void* score_out, void* logit_out,
                              int B, cudaStream_t st) {
  const int smem = V * 4;
  if (smem > 224000 || K < 1 || K > 7 || (qlog == nullptr && cnt == nullptr)) return -1;
  static int attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(dec::accept_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    attr = smem;
  }
  launch_pdl(dec::accept_kernel, dim3(B), dim3(dec::SAMPLE_THREADS), smem, st, (const __nv_bfloat16*)plog, ldp,
             (const __nv_bfloat16*)qlog, ldq, V, K, (const long long*)ictl, (const float*)fctl, (long long*)tok, (int*)pos, (int*)gen,
             (int*)finished, (long long*)out, ld_out, max_new, (int*)draft_pos, (long long*)stats, (const int*)cnt, (int*)hist, ldh,
             (float*)score_out, (__nv_bfloat16*)logit_out);
  ODB_CHECK_LAST();
  return 0;
}

// hist int32 [B, ldh]; pos / finished / cnt int32 [B]; ictl: see dec::sample_kernel (EOS ids); tok int64 [(K+1)*B] slot-major
// (slots 1..K written); proposed int64 [B].  1 <= K <= 7, 1 <= ngram <= 64.  See dec::lookup_propose_kernel.
ODB_EXPORT int odb_dec_lookup_propose(const void* hist, int ldh, const void* pos, const void* finished, const void* ictl, void* tok,
                                      void* cnt, void* proposed, int K, int ngram, int B, cudaStream_t st) {
  if (K < 1 || K > 7 || ngram < 1 || ngram > 64 || ldh < 1) return -1;
  launch_pdl(dec::lookup_propose_kernel, dim3(B), dim3(dec::LOOKUP_THREADS), 0, st, (const int*)hist, ldh, (const int*)pos,
             (const int*)finished, (const long long*)ictl, (long long*)tok, (int*)cnt, (long long*)proposed, K, ngram);
  ODB_CHECK_LAST();
  return 0;
}

// Vocabulary splits of beam_topk for a vocabulary of V (sizes its partials).
ODB_EXPORT int odb_dec_beam_splits(int V) { return odb::ceil_div(V, dec::TOPK_SPLIT); }

// logits [rows, ld] bf16; part_ml fp32 [rows, splits, 2]; cand_v fp32 / cand_i int32 [rows, splits, ck]; K <= 72.
// fctl: nullptr (no logits processors), or the sampler's fp32 control block with ck >= 2K, prompt int32 [rows / nb, ldp],
// plens / tstep int32 [rows / nb] and run_seq int32 [2, rows, max_new] (see dec::beam_topk_kernel).
ODB_EXPORT int odb_dec_beam_topk(const void* logits, long long ld, int V, int K, int ck, void* part_ml, void* cand_v, void* cand_i,
                                 const void* ictl, const void* fctl, const void* prompt, int ldp, const void* plens, const void* run_seq,
                                 const void* tstep, int nb, int max_new, int rows, const void* tab_off, const void* tab_bias, void* slot_i,
                                 void* slot_v, cudaStream_t st) {
  if (K < 1 || K > dec::MAX_KEEP || V < K || ck < K || (fctl != nullptr && (ck < 2 * K || nb < 1 || rows % nb))) return -1;
  if (tab_off != nullptr && (fctl == nullptr || tab_bias == nullptr || slot_i == nullptr || slot_v == nullptr)) return -1;
  launch_pdl(dec::beam_topk_kernel, dim3(odb::ceil_div(V, dec::TOPK_SPLIT), rows), dim3(dec::TOPK_THREADS), 0, st,
             (const __nv_bfloat16*)logits, ld, V, K, ck, (float*)part_ml, (float*)cand_v, (int*)cand_i, (const long long*)ictl,
             (const float*)fctl, (const int*)prompt, ldp, (const int*)plens, (const int*)run_seq, (const int*)tstep, nb, max_new,
             (const int*)tab_off, (const float*)tab_bias, (int*)slot_i, (float2*)slot_v);
  ODB_CHECK_LAST();
  return 0;
}

// B prompts of nb <= 8 beams (rows = B * nb); the beam_topk partials of V; ictl: the sampler's control block (EOS ids);
// early_stopping 0 False, 1 True, 2 "never"; run_score / fin_score fp32 [rows]; fin_flag / pos / parent int32 [rows];
// run_seq / fin_seq int32 [2, rows, max_new]; unsat / done / tstep int32 [B]; ids_next int64 [rows]; candidate rows of ck
// entries; fctl: nullptr, or the processors' control block as for beam_topk.  See dec::beam_step_kernel.
ODB_EXPORT int odb_dec_beam_step(const void* part_ml, const void* cand_v, const void* cand_i, int V, int nb, int K, int ck,
                                 const void* ictl, const void* fctl, float length_penalty, int early_stopping, int max_new, void* run_score,
                                 void* fin_score, void* fin_flag, void* run_seq, void* fin_seq, void* unsat, void* done, void* tstep,
                                 void* pos, void* ids_next, void* parent, const void* slot_i, const void* slot_v, void* run_bi, void* fin_bi,
                                 int B, cudaStream_t st) {
  const int ns = odb::ceil_div(V, dec::TOPK_SPLIT);
  if (nb < 1 || nb > dec::MAX_BEAMS || K < 1 || K > dec::MAX_KEEP || nb * ns > dec::STEP_THREADS || early_stopping < 0 ||
      early_stopping > 2 || max_new < 1 || ck < K || (fctl != nullptr && ck < 2 * K))
    return -1;
  launch_pdl(dec::beam_step_kernel, dim3(B), dim3(dec::STEP_THREADS), 0, st, (const float*)part_ml, (const float*)cand_v,
             (const int*)cand_i, ns, V, nb, K, ck, (const long long*)ictl, (const float*)fctl, length_penalty, early_stopping, max_new,
             (float*)run_score,
             (float*)fin_score, (int*)fin_flag, (int*)run_seq, (int*)fin_seq, (int*)unsat, (int*)done, (int*)tstep, (int*)pos,
             (long long*)ids_next, (int*)parent, (const int*)slot_i, (const float2*)slot_v, (int*)run_bi, (int*)fin_bi);
  ODB_CHECK_LAST();
  return 0;
}

// Between beam_topk and beam_step, with its arguments: score_out fp32 / logit_out bf16 [max_new, rows, V] (either may be
// nullptr).  See dec::beam_scores_kernel.
ODB_EXPORT int odb_dec_beam_scores(const void* logits, long long ld, int V, const void* part_ml, const void* ictl, const void* fctl,
                                   const void* prompt, int ldp, const void* plens, const void* run_seq, const void* tstep, const void* done,
                                   int nb, int max_new, int rows, const void* tab_off, const void* tab_bias, void* score_out,
                                   void* logit_out, cudaStream_t st) {
  if (nb < 1 || rows % nb || max_new < 1 || (fctl != nullptr && (prompt == nullptr || plens == nullptr))) return -1;
  if (tab_off != nullptr && (fctl == nullptr || tab_bias == nullptr)) return -1;
  launch_pdl(dec::beam_scores_kernel, dim3(odb::ceil_div(V, dec::TOPK_SPLIT), rows), dim3(dec::TOPK_THREADS), 0, st,
             (const __nv_bfloat16*)logits, ld, V, (const float*)part_ml, (const long long*)ictl, (const float*)fctl, (const int*)prompt,
             ldp, (const int*)plens, (const int*)run_seq, (const int*)tstep, (const int*)done, nb, max_new, (const int*)tab_off,
             (const float*)tab_bias, (float*)score_out, (__nv_bfloat16*)logit_out);
  ODB_CHECK_LAST();
  return 0;
}

// kv [L, 2, B*nb, Hkv, Smax, 64] (every layer's K and V of the beam rows, one allocation; bf16, or e4m3 bytes with inv fp32
// [L, 2, B*nb, Hkv, Smax], also one allocation); table int32 [B*nb, Smax/128]; parent / pos int32 [B*nb] (pos: the next
// position to be written, equal over a prompt's beams).  See dec::beam_reorder_kernel.
ODB_EXPORT int odb_dec_beam_reorder(void* kv, void* table, const void* parent, const void* pos, int B, int nb, int L, int Hkv, int Smax,
                                    void* inv, cudaStream_t st) {
  if (nb < 1 || nb > dec::MAX_BEAMS || Smax % dec::CH || Smax / dec::CH > dec::MAX_TABLE) return -1;
  return dec::with_cache(inv != nullptr, [&](auto t) {
    return dec::launch_beam_reorder<decltype(t)>(kv, inv, table, parent, pos, B, nb, L, Hkv, Smax, st);
  });
}

// kv [L, 2, B*n, Hkv, Smax, 64] (every layer's K and V, one allocation; bf16, or e4m3 bytes with inv fp32
// [L, 2, B*n, Hkv, Smax], also one allocation); table int32 [B*n, Smax/128]; len int32 [B]: prompt g was prefilled into
// row g*n, positions [0, len[g]).  Makes rows g*n + 1 .. g*n + n - 1 its children.  See dec::fork_kernel.
ODB_EXPORT int odb_dec_fork(void* kv, void* table, const void* len, int B, int n, int L, int Hkv, int Smax, void* inv, cudaStream_t st) {
  if (n < 1 || Smax % dec::CH) return -1;
  return dec::with_cache(inv != nullptr, [&](auto t) {
    using T = decltype(t);
    launch_pdl(dec::fork_kernel<T>, dim3(L * 2 * Hkv, B), dim3(256), 0, st, (T*)kv, (int*)table, (const int*)len, n, Hkv, Smax,
               Smax / dec::CH, (float*)inv);
    ODB_CHECK_LAST();
    return 0;
  });
}

// Autoregressive decode kernels for sm_90a (bf16, head_dim 64, MHA + GQA): the pieces of a KV-cached generation step that
// the training kernels do not cover.
//
//   odb_dec_rope_append   one new token per row: rotate q|k at the row's own position pos[b] (read from device memory, so a
//                         captured graph stays valid at every step), write k and v into the layer's cache at (b, pos[b])
//   odb_dec_kv_fill       prefill: copy the (already rotated) k|v columns of the packed qkv rows into the cache
//   odb_dec_attn          split-KV decode attention (flash-decoding) + a combine kernel
//   odb_dec_sample        greedy / temperature + top-k + top-p sampler, one CTA per row
//
// KV cache layout, per layer: K and V each [B, Hkv, Smax, 64] bf16, so the keys of one (row, kv head) are contiguous and a
// chunk of them is ONE bulk copy.
#include <curand_kernel.h>

#include "common.cuh"
#include "sm90_ptx.cuh"

using namespace odb;
using namespace sm90;

namespace dec {

constexpr int D = 64;
constexpr int CH = 128;             // keys per attention CTA
constexpr int ATT_THREADS = 128;    // one thread per key in the score phase, four warps in P V

// ------------------------------------------------------------------------------------------------ RoPE + append
// grid B, block 256.  qkv [B, ld] (q heads, k heads, v heads; unrotated GEMM output).  q is rotated in place; rotated k and
// v go to the cache.  Rounding: fp32 rotation of the bf16 inputs, one rounding to bf16 (as ops.kernels.rope_).
__global__ void __launch_bounds__(256)
rope_append_kernel(__nv_bfloat16* __restrict__ qkv, long long ld, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                   const int* __restrict__ pos, __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc, int Hq, int Hkv,
                   int Smax) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const int p = pos[b];
  __nv_bfloat16* row = qkv + (long long)b * ld;
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
      } else {
        __nv_bfloat16* dst = kc + (((long long)b * Hkv + (h - Hq)) * Smax + p) * D;
        dst[e] = lo;
        dst[e + D / 2] = hi;
      }
    } else {
      const int j = i - n_rot, hk = j / (D / 2), e = j % (D / 2);
      const uint32_t v = reinterpret_cast<const uint32_t*>(row + (Hq + Hkv + hk) * D)[e];
      reinterpret_cast<uint32_t*>(vc + (((long long)b * Hkv + hk) * Smax + p) * D)[e] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------ prefill cache fill
// grid (Sp, B), block 128: row s < len[b] of batch row b: 16-byte copies of the k and v heads.
__global__ void __launch_bounds__(128)
kv_fill_kernel(const __nv_bfloat16* __restrict__ qkv, long long ld, const int* __restrict__ len, __nv_bfloat16* __restrict__ kc,
               __nv_bfloat16* __restrict__ vc, int Sp, int Hq, int Hkv, int Smax) {
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x, b = blockIdx.y;
  if (s >= len[b] || s >= Smax) return;
  const __nv_bfloat16* row = qkv + ((long long)b * Sp + s) * ld + Hq * D;
  for (int i = threadIdx.x; i < 2 * Hkv * (D / 8); i += blockDim.x) {
    const int kv = i / (Hkv * (D / 8)), r = i % (Hkv * (D / 8)), hk = r / (D / 8), c = r % (D / 8);
    const uint4 v = ld_nc_v4(row + (kv * Hkv + hk) * D + c * 8);
    __nv_bfloat16* dst = (kv ? vc : kc) + (((long long)b * Hkv + hk) * Smax + s) * D + c * 8;
    st_v4(dst, v);
  }
}

// ------------------------------------------------------------------------------------------------ split-KV attention
// grid (ceil(Smax / CH), Hkv, B), block 128.  CTA (c, hk, b) serves the G = Hq / Hkv query heads of kv head hk against keys
// [c*CH, min((c+1)*CH, pos[b]+1)) of row b: K and V of the chunk arrive by two bulk copies, scores are one thread per key,
// P V is one warp per 32 keys (lanes over dimension pairs) summed across the four warps.  Writes the unnormalised partial
// output and its (max, sum) in the log2 domain; chunks past the row's length exit at once.
template <int G>
struct AttSmem {
  static constexpr int K_OFF = 0;
  static constexpr int V_OFF = CH * D * 2;
  static constexpr int Q_OFF = 2 * CH * D * 2;                   // fp32 [G][64], pre-scaled by softmax_scale * log2(e)
  static constexpr int S_OFF = Q_OFF + G * D * 4;                 // fp32 [G][CH] scores, then probabilities
  static constexpr int R_OFF = S_OFF + G * CH * 4;                // fp32 [4][G][64] per-warp P V
  static constexpr int M_OFF = R_OFF + 4 * G * D * 4;             // fp32 [G][2] (max, sum)
  static constexpr int BAR_OFF = M_OFF + 2 * G * 4;
  static constexpr int BYTES = BAR_OFF + 16;
};

template <int G>
__global__ void __launch_bounds__(ATT_THREADS)
decode_attn_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const __nv_bfloat16* __restrict__ kc,
                   const __nv_bfloat16* __restrict__ vc, const int* __restrict__ pos, float* __restrict__ part_o,
                   float* __restrict__ part_ml, int Hkv, int Smax, int nchunks, float scale_log2) {
  using L = AttSmem<G>;
  extern __shared__ __align__(128) uint8_t smem[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(smem + L::K_OFF);
  __nv_bfloat16* sV = reinterpret_cast<__nv_bfloat16*>(smem + L::V_OFF);
  float* sQ = reinterpret_cast<float*>(smem + L::Q_OFF);
  float* sS = reinterpret_cast<float*>(smem + L::S_OFF);
  float* sR = reinterpret_cast<float*>(smem + L::R_OFF);
  float* sM = reinterpret_cast<float*>(smem + L::M_OFF);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);

  pdl_launch_dependents();
  const int c = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  const int len = pos[b] + 1;
  const int j0 = c * CH;
  if (j0 >= len) return;                         // uniform over the CTA
  const int n = min(CH, len - j0);
  const long long kv_off = (((long long)b * Hkv + hk) * Smax + j0) * D;
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 2u * n * D * 2);
    bulk_load_1d(sK, kc + kv_off, n * D * 2, bar);
    bulk_load_1d(sV, vc + kv_off, n * D * 2, bar);
  }
  const __nv_bfloat16* qrow = q + (long long)b * ldq + (long long)hk * G * D;
  for (int i = tid; i < G * D; i += ATT_THREADS) sQ[i] = __bfloat162float(qrow[i]) * scale_log2;
  __syncthreads();
  mbar_wait(bar, 0);

  // ---- scores: thread = key; the 16-byte chunks of a key row are visited in a rotated order (no bank conflicts)
  {
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
    if (tid < n) {
      const uint4* krow = reinterpret_cast<const uint4*>(sK + tid * D);
#pragma unroll
      for (int cc = 0; cc < D / 8; ++cc) {
        const int ch = (cc + tid) & (D / 8 - 1);
        float kf[8];
        unpack8(krow[ch], kf);
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
      const float2 vv = bf2_to_f2(reinterpret_cast<const uint32_t*>(sV + j * D)[lane]);
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

// grid (Hq, B), block 64: merge the chunks of (b, h) and write out[b, h*64 + d] (token-major: the o-proj GEMM's A operand).
__global__ void __launch_bounds__(64)
decode_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml, const int* __restrict__ pos,
                      __nv_bfloat16* __restrict__ out, long long ldo, int nchunks) {
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, b = blockIdx.y, Hq = gridDim.x, d = threadIdx.x;
  const int used = ceil_div(pos[b] + 1, CH);
  const long long base = ((long long)b * Hq + h) * nchunks;
  float M = -INFINITY;
  for (int c = 0; c < used; ++c) M = fmaxf(M, part_ml[(base + c) * 2]);
  float L = 0.f, acc = 0.f;
  for (int c = 0; c < used; ++c) {
    const float w = exp2f(part_ml[(base + c) * 2] - M);
    L = fmaf(part_ml[(base + c) * 2 + 1], w, L);
    acc = fmaf(part_o[(base + c) * D + d], w, acc);
  }
  out[(long long)b * ldo + h * D + d] = __float2bfloat16_rn(acc / L);
}

// ------------------------------------------------------------------------------------------------ sampler
// ictl (int64, device): [0] do_sample, [1] top_k, [2] seed, [3] pad_token_id, [4] number of EOS ids (<= 8), [5..12] EOS ids
// fctl (fp32, device):  [0] temperature, [1] top_p
constexpr int SAMPLE_THREADS = 1024;
constexpr int MAX_EOS = 8;

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

__global__ void __launch_bounds__(SAMPLE_THREADS)
sample_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V, const long long* __restrict__ ictl,
              const float* __restrict__ fctl, int* __restrict__ pos, int* __restrict__ gen, int* __restrict__ finished,
              long long* __restrict__ out, int max_new, long long* __restrict__ ids_next) {
  extern __shared__ __align__(16) float e[];     // [V] exp(x - max) of the kept tokens, 0 elsewhere
  __shared__ float red[33];
  __shared__ ArgMax am[32];
  __shared__ int tok_sm;
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __nv_bfloat16* row = logits + (long long)b * ld;

  // ---- argmax (greedy, and the reference point of the exponentials)
  ArgMax best = {-INFINITY, V};
  for (int i = tid; i < V; i += SAMPLE_THREADS) best = argmax_merge(best, ArgMax{__bfloat162float(row[i]), i});
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
    best = argmax_merge(best, other);
  }
  if (lane == 0) am[warp] = best;
  __syncthreads();
  if (warp == 0) {
    best = am[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ArgMax other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
      best = argmax_merge(best, other);
    }
    if (lane == 0) am[0] = best;
  }
  __syncthreads();
  best = am[0];
  if (best.i >= V) best.i = 0;                   // all-NaN row: emit token 0 rather than an out-of-range id

  const bool do_sample = ictl[0] != 0;
  const int top_k = (int)ictl[1];
  if (tid == 0) tok_sm = best.i;
  if (do_sample && top_k != 1) {
    const float temp = fctl[0], top_p = fctl[1];
    const float mx = best.v / temp;
    // HF warper order: temperature, then top-k, then top-p; probabilities are exp(x - max) up to the normaliser
    for (int i = tid; i < V; i += SAMPLE_THREADS) e[i] = exp2f((__bfloat162float(row[i]) / temp - mx) * 1.4426950408889634f);
    __syncthreads();
    if (top_k > 0 && top_k < V) {
      const uint32_t t = bisect_threshold<false>(e, V, (float)top_k, red);
      for (int i = tid; i < V; i += SAMPLE_THREADS)
        if (__float_as_uint(e[i]) < t) e[i] = 0.f;
      __syncthreads();
    }
    if (top_p < 1.f) {
      float z = 0.f;
      for (int i = tid; i < V; i += SAMPLE_THREADS) z += e[i];
      z = block_sum(z, red);
      const uint32_t t = bisect_threshold<true>(e, V, top_p * z, red);
      for (int i = tid; i < V; i += SAMPLE_THREADS)
        if (__float_as_uint(e[i]) < t) e[i] = 0.f;
      __syncthreads();
    }
    // inverse CDF in index order: thread t owns a contiguous segment; exclusive scan of the segment sums
    const int per = ceil_div(V, SAMPLE_THREADS);
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
    __syncthreads();
    if (warp == 0) {
      float w = red[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float y = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += y;
      }
      red[lane] = wi - w;                        // exclusive prefix of the warp totals
      if (lane == 31) red[32] = wi;              // total kept mass
    }
    __syncthreads();
    const float pre = red[warp] + incl - local, total = red[32];
    curandStatePhilox4_32_10_t rng;
    curand_init((unsigned long long)ictl[2], (unsigned long long)b, (unsigned long long)gen[b], &rng);
    const float r = curand_uniform(&rng) * total;   // u in (0, 1]
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
      tok_sm = pick;                             // at most one thread's segment brackets r
    }
  }
  __syncthreads();
  if (tid == 0) {
    const int g = gen[b];
    const bool fin = finished[b] != 0;
    const long long tok = fin ? ictl[3] : (long long)tok_sm;
    if (g < max_new) out[(long long)b * max_new + g] = tok;
    ids_next[b] = tok;
    gen[b] = g + 1;
    pos[b] = pos[b] + 1;
    if (!fin) {
      const int n_eos = (int)min(ictl[4], (long long)MAX_EOS);
      for (int k = 0; k < n_eos; ++k)
        if (tok == ictl[5 + k]) finished[b] = 1;
    }
  }
}

template <int G>
int launch_attn(const void* q, long long ldq, const void* kc, const void* vc, const void* pos, void* part_o, void* part_ml, void* out,
                long long ldo, int B, int Hkv, int Smax, float scale, cudaStream_t st) {
  static bool attr_set = false;
  const int smem = AttSmem<G>::BYTES;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(decode_attn_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int nchunks = ceil_div(Smax, CH);
  launch_pdl(decode_attn_kernel<G>, dim3(nchunks, Hkv, B), dim3(ATT_THREADS), smem, st, (const __nv_bfloat16*)q, ldq,
             (const __nv_bfloat16*)kc, (const __nv_bfloat16*)vc, (const int*)pos, (float*)part_o, (float*)part_ml, Hkv, Smax,
             nchunks, scale * 1.4426950408889634f);
  ODB_CHECK_LAST();
  launch_pdl(decode_combine_kernel, dim3(Hkv * G, B), dim3(D), 0, st, (const float*)part_o, (const float*)part_ml, (const int*)pos,
             (__nv_bfloat16*)out, ldo, nchunks);
  ODB_CHECK_LAST();
  return 0;
}

}  // namespace dec

// qkv [B, ld] bf16 (one token per row); cos/sin fp32 [max_pos, 32]; pos int32 [B]; kc/vc [B, Hkv, Smax, 64] bf16
ODB_EXPORT int odb_dec_rope_append(void* qkv, long long ld, const void* cos_t, const void* sin_t, const void* pos, void* kc, void* vc,
                                   int B, int Hq, int Hkv, int Smax, cudaStream_t st) {
  if (ld % 2) return -1;
  launch_pdl(dec::rope_append_kernel, dim3(B), dim3(256), 0, st, (__nv_bfloat16*)qkv, ld, (const float*)cos_t, (const float*)sin_t,
             (const int*)pos, (__nv_bfloat16*)kc, (__nv_bfloat16*)vc, Hq, Hkv, Smax);
  ODB_CHECK_LAST();
  return 0;
}

// qkv [B*Sp, ld] bf16 (rotated prefill projections); len int32 [B]: rows s < len[b] are copied into the cache
ODB_EXPORT int odb_dec_kv_fill(const void* qkv, long long ld, const void* len, void* kc, void* vc, int B, int Sp, int Hq, int Hkv,
                               int Smax, cudaStream_t st) {
  if (ld % 8) return -1;
  launch_pdl(dec::kv_fill_kernel, dim3(Sp, B), dim3(128), 0, st, (const __nv_bfloat16*)qkv, ld, (const int*)len, (__nv_bfloat16*)kc,
             (__nv_bfloat16*)vc, Sp, Hq, Hkv, Smax);
  ODB_CHECK_LAST();
  return 0;
}

// Number of key chunks of the split-KV attention for a cache of Smax positions (sizes the partial buffers).
ODB_EXPORT int odb_dec_attn_chunks(int Smax) { return odb::ceil_div(Smax, dec::CH); }

// q [B, ldq] bf16 (the q heads first); kc/vc [B, Hkv, Smax, 64]; pos int32 [B] (keys 0..pos[b] are attended);
// part_o fp32 [B, Hq, chunks, 64]; part_ml fp32 [B, Hq, chunks, 2]; out [B, ldo] bf16
ODB_EXPORT int odb_dec_attn(const void* q, long long ldq, const void* kc, const void* vc, const void* pos, void* part_o, void* part_ml,
                            void* out, long long ldo, int B, int Hq, int Hkv, int Smax, float softmax_scale, cudaStream_t st) {
  if (Hq % Hkv || ldq % 8) return -1;
  switch (Hq / Hkv) {
    case 1: return dec::launch_attn<1>(q, ldq, kc, vc, pos, part_o, part_ml, out, ldo, B, Hkv, Smax, softmax_scale, st);
    case 2: return dec::launch_attn<2>(q, ldq, kc, vc, pos, part_o, part_ml, out, ldo, B, Hkv, Smax, softmax_scale, st);
    case 4: return dec::launch_attn<4>(q, ldq, kc, vc, pos, part_o, part_ml, out, ldo, B, Hkv, Smax, softmax_scale, st);
    case 8: return dec::launch_attn<8>(q, ldq, kc, vc, pos, part_o, part_ml, out, ldo, B, Hkv, Smax, softmax_scale, st);
    default: return -2;                          // GQA groups of 1, 2, 4 or 8 query heads
  }
}

// logits [B, ld] bf16; ictl / fctl: see dec::sample_kernel; pos / gen / finished int32 [B]; out int64 [B, max_new];
// ids_next int64 [B].  The vocabulary lives in shared memory as fp32: V <= 56000.
ODB_EXPORT int odb_dec_sample(const void* logits, long long ld, int V, const void* ictl, const void* fctl, void* pos, void* gen,
                              void* finished, void* out, int max_new, void* ids_next, int B, cudaStream_t st) {
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
             (long long*)ids_next);
  ODB_CHECK_LAST();
  return 0;
}

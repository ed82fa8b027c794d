// Flat-arena optimizer kernels for sm_90a (SURVEY.md §2.5 K9-K12, K14).
//
//  * grad_sqnorm:   one pass over the fp32 gradient arena -> per-CTA partial sums of squares + non-finite flag
//  * adamw_step:    one launch: (clip coefficient from the partials) -> AdamW on fp32 master weights ->
//                   bf16 shadow weights -> zero the gradient.  Replaces clip_grad_norm_ + foreach AdamW + zero_grad
//                   (reference: train_diloco_torch.py:321-334, train_fsdp.py:390-408).
//  * outer kernels: pseudo-gradient (theta_outer - theta_local), optional bf16 cast, and the SGD-Nesterov update with
//                   write-back of theta_local + bf16 shadow (reference: train_diloco_torch.py:340-353).
//
// Hyper-parameters that change every step (lr, bias corrections) are read from a small device-side fp32 block so
// the launches can sit inside a CUDA graph without re-capture.
#include "common.cuh"

using namespace odb;

constexpr int kNormThreads = 512;
constexpr int kMaxPartials = 2048;

// partials[b] = sum of squares seen by CTA b ; flag[0] |= any non-finite
__global__ void __launch_bounds__(kNormThreads) grad_sqnorm_kernel(const float* __restrict__ g, long long n4,
                                                                   float* __restrict__ partials, int* __restrict__ flag) {
  __shared__ float sm[33];
  float s = 0.f;
  bool bad = false;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = ld_f4(reinterpret_cast<const float*>(g4 + i));
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  bad = !isfinite(s);
  s = block_sum(s, sm);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
  if (bad) atomicOr(flag, 1);
}

// hp layout (fp32): [0]=lr [1]=beta1 [2]=beta2 [3]=eps [4]=weight_decay [5]=bias_corr1 [6]=bias_corr2
//                   [7]=max_norm (<=0: no clipping) [8]=grad_scale_inv (1/loss-scale, fp16 path; 1 otherwise)
// out_stats (fp32): [0]=total grad norm (after unscale), [1]=clip coefficient actually applied
template <bool kWriteShadow, bool kZeroGrad>
__global__ void __launch_bounds__(256) adamw_step_kernel(float* __restrict__ p, float* __restrict__ g,
                                                         float* __restrict__ m, float* __restrict__ v,
                                                         __nv_bfloat16* __restrict__ shadow, long long n4,
                                                         const float* __restrict__ hp, const float* __restrict__ partials,
                                                         int n_partials, const int* __restrict__ found_inf,
                                                         int* __restrict__ skipped, float* __restrict__ out_stats) {
  __shared__ float sm[33];
  // every CTA re-reduces the (<= 2048) partials: deterministic, no atomics, no extra launch
  float s = 0.f;
  for (int i = threadIdx.x; i < n_partials; i += blockDim.x) s += partials[i];
  s = block_sum(s, sm);
  const float lr = hp[0], b1 = hp[1], b2 = hp[2], eps = hp[3], wd = hp[4];
  const float max_norm = hp[7], inv_scale = hp[8];
  float bc1, bc2;
  adamw_bias_corrections(hp, skipped, bc1, bc2);
  const float gnorm = sqrtf(s) * inv_scale;
  float coef = inv_scale;
  float clip = 1.f;
  if (max_norm > 0.f) {
    clip = fminf(1.f, max_norm / (gnorm + 1e-6f));
    coef *= clip;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && out_stats) { out_stats[0] = gnorm; out_stats[1] = clip; }
  // GradScaler semantics: skip the update (but still zero the grads) when a non-finite gradient was found
  const bool skip = (found_inf != nullptr) && (*found_inf != 0);
  adamw_count_skip(hp, skipped, skip);
  const float step_size = lr / bc1;
  const float sqrt_bc2 = sqrtf(bc2);
  const float decay = 1.f - lr * wd;

  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 gg = ld_nc_f4(g + i * 4);
    if (!skip) {
      float4 pp = ld_f4(p + i * 4), mm = ld_f4(m + i * 4), vv = ld_f4(v + i * 4);
      float* P = &pp.x; float* M = &mm.x; float* V = &vv.x; float* G = &gg.x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gr = G[j] * coef;
        const float pj = P[j] * decay;
        M[j] = M[j] + (1.f - b1) * (gr - M[j]);          // torch lerp form
        V[j] = b2 * V[j] + (1.f - b2) * gr * gr;
        const float denom = sqrtf(V[j]) / sqrt_bc2 + eps;
        P[j] = pj - step_size * (M[j] / denom);
      }
      st_f4(p + i * 4, pp);
      st_f4(m + i * 4, mm);
      st_f4(v + i * 4, vv);
      if (kWriteShadow) {
        uint2 o = make_uint2(f2_to_bf2(pp.x, pp.y), f2_to_bf2(pp.z, pp.w));
        *reinterpret_cast<uint2*>(shadow + i * 4) = o;
      }
    }
    if (kZeroGrad) st_f4(g + i * 4, make_float4(0.f, 0.f, 0.f, 0.f));
  }
}

// ------------------------------------------------------------------------------------------------ outer step
// delta = theta_outer - theta_local, written as fp32 or bf16 (the "fp32->bf16 cast" of BASELINE.json)
template <typename OutT>
__global__ void __launch_bounds__(256) pseudo_grad_kernel(const float* __restrict__ theta_outer,
                                                          const float* __restrict__ theta_local, OutT* __restrict__ delta,
                                                          long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = ld_nc_f4(theta_outer + i * 4), b = ld_nc_f4(theta_local + i * 4);
    const float4 d = make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
    if constexpr (sizeof(OutT) == 4) {
      st_f4(reinterpret_cast<float*>(delta) + i * 4, d);
    } else {
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(delta) + i * 4) =
          make_uint2(f2_to_bf2(d.x, d.y), f2_to_bf2(d.z, d.w));
    }
  }
}

// SGD with (Nesterov) momentum on the outer copy, torch.optim.SGD semantics (dampening 0, wd 0):
//   buf = mu*buf + d ; step = nesterov ? d + mu*buf : buf ; theta_outer -= lr*step
// then theta_local <- theta_outer and shadow <- bf16(theta_outer).
// kFusedDelta: compute d = (theta_outer - theta_local) * dscale in-kernel (single-worker outer step: no collective).
// otherwise d = delta[i] * dscale (delta already summed across workers; dscale = 1/world for SUM collectives).
template <typename InT, bool kFusedDelta>
__global__ void __launch_bounds__(256) nesterov_outer_kernel(float* __restrict__ theta_outer, float* __restrict__ buf,
                                                             const InT* __restrict__ delta, float* __restrict__ theta_local,
                                                             __nv_bfloat16* __restrict__ shadow, long long n4, float lr,
                                                             float mu, int nesterov, float dscale) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 to = ld_f4(theta_outer + i * 4);
    float4 bb = ld_f4(buf + i * 4);
    float4 d;
    if constexpr (kFusedDelta) {
      const float4 tl = ld_f4(theta_local + i * 4);
      d = make_float4(to.x - tl.x, to.y - tl.y, to.z - tl.z, to.w - tl.w);
    } else if constexpr (sizeof(InT) == 4) {
      d = ld_nc_f4(reinterpret_cast<const float*>(delta) + i * 4);
    } else {
      const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(delta) + i * 4);
      const float2 lo = bf2_to_f2(u.x), hi = bf2_to_f2(u.y);
      d = make_float4(lo.x, lo.y, hi.x, hi.y);
    }
    float* T = &to.x; float* B = &bb.x; float* D = &d.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float dj = D[j] * dscale;
      B[j] = mu * B[j] + dj;
      const float stp = nesterov ? (dj + mu * B[j]) : B[j];
      T[j] = T[j] - lr * stp;
    }
    st_f4(theta_outer + i * 4, to);
    st_f4(buf + i * 4, bb);
    st_f4(theta_local + i * 4, to);
    if (shadow) *reinterpret_cast<uint2*>(shadow + i * 4) = make_uint2(f2_to_bf2(to.x, to.y), f2_to_bf2(to.z, to.w));
  }
}

// ------------------------------------------------------------------------------------------------ launchers
static inline int flat_grid(long long n4, int threads, int waves) {
  long long g = ceil_div_ll(n4, threads);
  long long cap = (long long)sm_count() * waves;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// returns the number of partials written (>0) or a negative error
ODB_EXPORT int odb_grad_sqnorm(const void* g, long long n, void* partials, void* flag, cudaStream_t st) {
  if (n % 4) return -1;
  int grid = flat_grid(n / 4, kNormThreads, 4);
  if (grid > kMaxPartials) grid = kMaxPartials;
  grad_sqnorm_kernel<<<grid, kNormThreads, 0, st>>>((const float*)g, n / 4, (float*)partials, (int*)flag);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return -(int)e;
  return grid;
}

ODB_EXPORT int odb_adamw_step(void* p, void* g, void* m, void* v, void* shadow, long long n, const void* hp,
                              const void* partials, int n_partials, const void* found_inf, void* skipped,
                              void* out_stats, int zero_grad, cudaStream_t st) {
  if (n % 4) return -1;
  const int grid = flat_grid(n / 4, 256, 8);
#define ODB_ADAMW(WS, ZG)                                                                                         \
  adamw_step_kernel<WS, ZG><<<grid, 256, 0, st>>>((float*)p, (float*)g, (float*)m, (float*)v, (__nv_bfloat16*)shadow, \
                                                  n / 4, (const float*)hp, (const float*)partials, n_partials,      \
                                                  (const int*)found_inf, (int*)skipped, (float*)out_stats)
  if (shadow && zero_grad) ODB_ADAMW(true, true);
  else if (shadow) ODB_ADAMW(true, false);
  else if (zero_grad) ODB_ADAMW(false, true);
  else ODB_ADAMW(false, false);
#undef ODB_ADAMW
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_pseudo_grad(const void* theta_outer, const void* theta_local, void* delta, long long n, int out_bf16,
                               cudaStream_t st) {
  if (n % 4) return -1;
  const int grid = flat_grid(n / 4, 256, 8);
  if (out_bf16)
    pseudo_grad_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const float*)theta_outer, (const float*)theta_local,
                                                            (__nv_bfloat16*)delta, n / 4);
  else
    pseudo_grad_kernel<float><<<grid, 256, 0, st>>>((const float*)theta_outer, (const float*)theta_local, (float*)delta,
                                                    n / 4);
  ODB_CHECK_LAST();
  return 0;
}

// delta == nullptr -> fused single-worker form (delta computed in-kernel)
ODB_EXPORT int odb_nesterov_outer(void* theta_outer, void* buf, const void* delta, int delta_bf16, void* theta_local,
                                  void* shadow, long long n, float lr, float mu, int nesterov, float dscale,
                                  cudaStream_t st) {
  if (n % 4) return -1;
  const int grid = flat_grid(n / 4, 256, 8);
  if (delta == nullptr)
    nesterov_outer_kernel<float, true><<<grid, 256, 0, st>>>((float*)theta_outer, (float*)buf, nullptr,
                                                             (float*)theta_local, (__nv_bfloat16*)shadow, n / 4, lr, mu,
                                                             nesterov, dscale);
  else if (delta_bf16)
    nesterov_outer_kernel<__nv_bfloat16, false><<<grid, 256, 0, st>>>(
        (float*)theta_outer, (float*)buf, (const __nv_bfloat16*)delta, (float*)theta_local, (__nv_bfloat16*)shadow, n / 4,
        lr, mu, nesterov, dscale);
  else
    nesterov_outer_kernel<float, false><<<grid, 256, 0, st>>>((float*)theta_outer, (float*)buf, (const float*)delta,
                                                              (float*)theta_local, (__nv_bfloat16*)shadow, n / 4, lr, mu,
                                                              nesterov, dscale);
  ODB_CHECK_LAST();
  return 0;
}

// ------------------------------------------------------------------------------------------------ state fingerprint
// Wrap-around integer checksum of a buffer's 32-bit words (order independent, exact): the drift detector DiLoCo workers
// exchange after a full outer round (two workers hold bit-identical theta_outer iff their checksums agree, up to 2^-64).
// One pass at HBM speed; `out` (int64) is ACCUMULATED (zero it first).
__global__ void __launch_bounds__(512) checksum_i32_kernel(const int4* __restrict__ buf, long long n4, unsigned long long* __restrict__ out) {
  __shared__ long long sm[16];
  long long s = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = ld_nc_v4(buf + i);
    s += (long long)(int)v.x + (long long)(int)v.y + (long long)(int)v.z + (long long)(int)v.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sm[w];
    atomicAdd(out, (unsigned long long)t);
  }
}

ODB_EXPORT int odb_checksum_i32(const void* buf, long long n_words, void* out, cudaStream_t st) {
  if (n_words % 4) return -1;
  const long long n4 = n_words / 4;
  long long blocks = ceil_div_ll(n4, 512 * 8);
  const long long cap = (long long)sm_count() * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  checksum_i32_kernel<<<(int)blocks, 512, 0, st>>>((const int4*)buf, n4, (unsigned long long*)out);
  ODB_CHECK_LAST();
  return 0;
}

// Muon inner optimizer kernels for sm_90a (the step of optim/muon.py::FusedMuon; torch.optim.Muon semantics).
//
//  * muon_prepare:    per 64K-element chunk of the Muon matrices: clip coefficient (from the gradient-norm partials, as in
//                     adamw_step) -> g' = coef * g -> momentum buf = lerp(buf, g', 1 - mu) -> u = nesterov ? lerp(g', buf, mu)
//                     : buf -> one partial sum of u^2 per chunk.  Fixed chunking and a fixed reduction order: no float
//                     atomics, so replicas that see the same gradients stay bit-identical.
//  * muon_scale:      one CTA per matrix: (clip coefficient, 1 / max(||u||_F, eps)) from the fixed-order sum of its chunk
//                     partials, so the normalise pass reads two floats per tile instead of re-reducing the partials.
//  * muon_normalize:  X = bf16(u / max(||u||_F, eps)) into the stacked Newton-Schulz scratch, oriented so that X is wide
//                     (tall matrices are transposed through shared memory).  u is recomputed from g and the new momentum
//                     with the same arithmetic as in muon_prepare instead of being stored.
//  * (Newton-Schulz: odb_gemm_batched_axpby_tn / _nn in gemm_sm90.cu)
//  * muon_apply:      theta = theta * (1 - lr * wd) - lr * adjust * O (O transposed back where needed) into the fp32 master
//                     and the bf16 shadow, and optionally zeroes the gradient.
//  * adamw_segments:  adamw_step's math on a list of chunks of the flat arena (embedding, LM head, norm weights) in one
//                     launch (float4 accesses on 16-byte aligned chunks).
//
// Every hyper-parameter that a schedule may change is read from the device block `hp` (layout: optim/muon.py), so the
// launches can be graph-captured.  A non-finite gradient (GradScaler) leaves momentum, moments and weights untouched.
#include "common.cuh"

using namespace odb;

namespace {

// hp slots shared with adamw_step (optim.cu) + the Muon group's own
// (slots 5, 6 and 13-15 are read by adamw_bias_corrections, common.cuh)
constexpr int HP_LR = 0, HP_B1 = 1, HP_B2 = 2, HP_EPS = 3, HP_WD = 4, HP_MAXNORM = 7, HP_INVSCALE = 8;
constexpr int HP_MLR = 9, HP_MOM = 10, HP_MWD = 11, HP_NESTEROV = 12;
constexpr int kTile = 32;
constexpr int kTableCols = 8;   // matrix table row: flat offset, rows, cols, transposed, chunk0, chunk1, scratch offset, adjust (f32 bits)

// clip coefficient of adamw_step (inv_scale * min(1, max_norm / (norm + 1e-6))); every CTA re-reduces the partials
__device__ __forceinline__ float clip_coef(const float* hp, const float* partials, int n_partials, float* sm, float* gnorm_out,
                                           float* clip_out) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n_partials; i += blockDim.x) s += partials[i];
  s = block_sum(s, sm);
  const float max_norm = hp[HP_MAXNORM], inv_scale = hp[HP_INVSCALE];
  const float gnorm = sqrtf(s) * inv_scale;
  float clip = 1.f;
  if (max_norm > 0.f) clip = fminf(1.f, max_norm / (gnorm + 1e-6f));
  if (gnorm_out) { *gnorm_out = gnorm; *clip_out = clip; }
  return inv_scale * clip;
}

__device__ __forceinline__ float momentum_update(float gr, float& b, float mu, bool nesterov) {
  b = b + (1.f - mu) * (gr - b);                 // buf.lerp_(g, 1 - mu)
  return nesterov ? gr + mu * (b - gr) : b;      // g.lerp(buf, mu) or buf
}

__global__ void __launch_bounds__(256) muon_prepare_kernel(const float* __restrict__ g, float* __restrict__ buf,
                                                           const long long* __restrict__ chunks, const float* __restrict__ hp,
                                                           const float* __restrict__ gpart, int n_gpart,
                                                           const int* __restrict__ found_inf, float* __restrict__ upart,
                                                           float* __restrict__ out_stats) {
  __shared__ float sm[33];
  float gnorm, clip;
  const float coef = clip_coef(hp, gpart, n_gpart, sm, &gnorm, &clip);
  if (blockIdx.x == 0 && threadIdx.x == 0 && out_stats) { out_stats[0] = gnorm; out_stats[1] = clip; }
  const bool skip = found_inf != nullptr && *found_inf != 0;
  const float mu = hp[HP_MOM];
  const bool nesterov = hp[HP_NESTEROV] != 0.f;
  const long long start = chunks[2 * blockIdx.x], len = chunks[2 * blockIdx.x + 1];
  float s = 0.f;
  for (long long i = threadIdx.x; i < len; i += blockDim.x) {
    float b = buf[start + i];
    const float u = momentum_update(g[start + i] * coef, b, mu, nesterov);
    if (!skip) buf[start + i] = b;
    s += u * u;
  }
  s = block_sum(s, sm);
  if (threadIdx.x == 0) upart[blockIdx.x] = s;
}

// blockIdx.x: matrix j with chunk range mats[j] = (c0, c1) -> scale[2 c0] = clip coefficient, scale[2 c0 + 1] = 1 / max(||u||, eps)
__global__ void __launch_bounds__(256) muon_scale_kernel(const long long* __restrict__ mats, const float* __restrict__ hp,
                                                         const float* __restrict__ gpart, int n_gpart,
                                                         const float* __restrict__ upart, float* __restrict__ scale, float eps) {
  __shared__ float sm[33];
  const long long c0 = mats[2 * blockIdx.x], c1 = mats[2 * blockIdx.x + 1];
  const float coef = clip_coef(hp, gpart, n_gpart, sm, nullptr, nullptr);
  float s = 0.f;
  for (long long c = c0 + threadIdx.x; c < c1; c += blockDim.x) s += upart[c];
  s = block_sum(s, sm);
  if (threadIdx.x == 0) {
    scale[2 * c0] = coef;
    scale[2 * c0 + 1] = 1.f / fmaxf(sqrtf(s), eps);
  }
}

// blockIdx.y: matrix of the table; blockIdx.x: 32 x 32 tile of its oriented [m, n] scratch image
__global__ void __launch_bounds__(256) muon_normalize_kernel(const float* __restrict__ g, const float* __restrict__ buf,
                                                             const long long* __restrict__ table, int m, int n,
                                                             const float* __restrict__ hp, const float* __restrict__ scale,
                                                             __nv_bfloat16* __restrict__ x) {
  __shared__ float tile[kTile][kTile + 1];
  const long long* t = table + (size_t)blockIdx.y * kTableCols;
  const long long off = t[0], cols = t[2], c0 = t[4], xoff = t[6];
  const bool tr = t[3] != 0;
  const float coef = scale[2 * c0], inv = scale[2 * c0 + 1];
  const float mu = hp[HP_MOM];
  const bool nesterov = hp[HP_NESTEROV] != 0.f;
  const int tiles_n = n / kTile;
  const int i0 = (blockIdx.x / tiles_n) * kTile, j0 = (blockIdx.x % tiles_n) * kTile;
  const int tx = threadIdx.x % kTile, ty = threadIdx.x / kTile;
  for (int y = ty; y < kTile; y += blockDim.x / kTile) {
    const long long pr = tr ? j0 + y : i0 + y, pc = tr ? i0 + tx : j0 + tx;   // element of the parameter's [rows, cols]
    const long long e = off + pr * cols + pc;
    // buf holds the updated momentum b' (on a skipped step the old one; muon_apply then discards the result):
    // the same arithmetic as momentum_update's return value
    const float gr = g[e] * coef, b = buf[e];
    const float u = nesterov ? gr + mu * (b - gr) : b;
    tile[y][tx] = u * inv;
  }
  __syncthreads();
  for (int y = ty; y < kTile; y += blockDim.x / kTile) {
    const float v = tr ? tile[tx][y] : tile[y][tx];
    x[xoff + (long long)(i0 + y) * n + j0 + tx] = __float2bfloat16_rn(v);
  }
}

__global__ void __launch_bounds__(256) muon_apply_kernel(float* __restrict__ p, float* __restrict__ g,
                                                         __nv_bfloat16* __restrict__ shadow, const long long* __restrict__ table,
                                                         int m, int n, const float* __restrict__ hp,
                                                         const __nv_bfloat16* __restrict__ x, const int* __restrict__ found_inf,
                                                         int zero_grad) {
  __shared__ float tile[kTile][kTile + 1];
  const long long* t = table + (size_t)blockIdx.y * kTableCols;
  const long long off = t[0], cols = t[2], xoff = t[6];
  const bool tr = t[3] != 0;
  const float adjust = __int_as_float((int)(t[7] & 0xffffffffll));
  const float lr = hp[HP_MLR], wd = hp[HP_MWD];
  const float decay = 1.f - lr * wd, step = lr * adjust;
  const bool skip = found_inf != nullptr && *found_inf != 0;
  const int tiles_n = n / kTile;
  const int i0 = (blockIdx.x / tiles_n) * kTile, j0 = (blockIdx.x % tiles_n) * kTile;
  const int tx = threadIdx.x % kTile, ty = threadIdx.x / kTile;
  for (int y = ty; y < kTile; y += blockDim.x / kTile)
    tile[y][tx] = __bfloat162float(x[xoff + (long long)(i0 + y) * n + j0 + tx]);
  __syncthreads();
  for (int y = ty; y < kTile; y += blockDim.x / kTile) {
    const long long pr = tr ? j0 + y : i0 + y, pc = tr ? i0 + tx : j0 + tx;
    const long long e = off + pr * cols + pc;
    if (!skip) {
      const float o = tr ? tile[tx][y] : tile[y][tx];
      const float v = p[e] * decay - step * o;
      p[e] = v;
      if (shadow) shadow[e] = __float2bfloat16_rn(v);
    }
    if (zero_grad) g[e] = 0.f;
  }
}

__global__ void __launch_bounds__(256) adamw_segments_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                                             float* __restrict__ v, __nv_bfloat16* __restrict__ shadow,
                                                             const long long* __restrict__ chunks, const float* __restrict__ hp,
                                                             const float* __restrict__ gpart, int n_gpart,
                                                             const int* __restrict__ found_inf, int* __restrict__ skipped,
                                                             int zero_grad) {
  __shared__ float sm[33];
  const float coef = clip_coef(hp, gpart, n_gpart, sm, nullptr, nullptr);
  const bool skip = found_inf != nullptr && *found_inf != 0;
  adamw_count_skip(hp, skipped, skip);
  const float lr = hp[HP_LR], b1 = hp[HP_B1], b2 = hp[HP_B2], eps = hp[HP_EPS], wd = hp[HP_WD];
  float bc1, bc2;
  adamw_bias_corrections(hp, skipped, bc1, bc2);
  const float step_size = lr / bc1, sqrt_bc2 = sqrtf(bc2), decay = 1.f - lr * wd;
  const long long start = chunks[2 * blockIdx.x], len = chunks[2 * blockIdx.x + 1];
  if (start % 4 == 0 && len % 4 == 0) {               // 16-byte aligned chunk: the float4 body of adamw_step
    for (long long i = start + 4 * threadIdx.x; i < start + len; i += 4 * blockDim.x) {
      float4 gg = ld_nc_f4(g + i);
      if (!skip) {
        float4 pp = ld_f4(p + i), mm = ld_f4(m + i), vv = ld_f4(v + i);
        float* P = &pp.x; float* Mv = &mm.x; float* V = &vv.x; float* G = &gg.x;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float gr = G[j] * coef;
          const float pj = P[j] * decay;
          Mv[j] = Mv[j] + (1.f - b1) * (gr - Mv[j]);
          V[j] = b2 * V[j] + (1.f - b2) * gr * gr;
          P[j] = pj - step_size * (Mv[j] / (sqrtf(V[j]) / sqrt_bc2 + eps));
        }
        st_f4(p + i, pp);
        st_f4(m + i, mm);
        st_f4(v + i, vv);
        if (shadow) *reinterpret_cast<uint2*>(shadow + i) = make_uint2(f2_to_bf2(pp.x, pp.y), f2_to_bf2(pp.z, pp.w));
      }
      if (zero_grad) st_f4(g + i, make_float4(0.f, 0.f, 0.f, 0.f));
    }
    return;
  }
  for (long long i = start + threadIdx.x; i < start + len; i += blockDim.x) {
    if (!skip) {
      const float gr = g[i] * coef;
      const float pj = p[i] * decay;
      const float mj = m[i] + (1.f - b1) * (gr - m[i]);
      const float vj = b2 * v[i] + (1.f - b2) * gr * gr;
      const float pn = pj - step_size * (mj / (sqrtf(vj) / sqrt_bc2 + eps));
      m[i] = mj;
      v[i] = vj;
      p[i] = pn;
      if (shadow) shadow[i] = __float2bfloat16_rn(pn);
    }
    if (zero_grad) g[i] = 0.f;
  }
}

}  // namespace

// chunks: int64 [n_chunks, 2] = (flat offset, length); upart: fp32 [n_chunks]
ODB_EXPORT int odb_muon_prepare(const void* g, void* buf, const void* chunks, int n_chunks, const void* hp, const void* gpart,
                                int n_gpart, const void* found_inf, void* upart, void* out_stats, cudaStream_t st) {
  if (n_chunks <= 0) return -1;
  muon_prepare_kernel<<<n_chunks, 256, 0, st>>>((const float*)g, (float*)buf, (const long long*)chunks, (const float*)hp,
                                                (const float*)gpart, n_gpart, (const int*)found_inf, (float*)upart,
                                                (float*)out_stats);
  ODB_CHECK_LAST();
  return 0;
}

// mats: int64 [n_mat, 2] = chunk range (c0, c1) of each matrix; scale: fp32 [2 * n_chunks], written at 2 c0 and 2 c0 + 1
ODB_EXPORT int odb_muon_scale(const void* mats, int n_mat, const void* hp, const void* gpart, int n_gpart, const void* upart,
                              void* scale, float eps, cudaStream_t st) {
  if (n_mat <= 0) return -1;
  muon_scale_kernel<<<n_mat, 256, 0, st>>>((const long long*)mats, (const float*)hp, (const float*)gpart, n_gpart,
                                           (const float*)upart, (float*)scale, eps);
  ODB_CHECK_LAST();
  return 0;
}

// table: int64 [n_mat, 8] for matrices whose oriented image is [m, n] (m <= n, both % 32 == 0); x: bf16 scratch
ODB_EXPORT int odb_muon_normalize(const void* g, const void* buf, const void* table, int n_mat, int m, int n, const void* hp,
                                  const void* scale, void* x, cudaStream_t st) {
  if (n_mat <= 0 || m % kTile || n % kTile) return -1;
  muon_normalize_kernel<<<dim3((m / kTile) * (n / kTile), n_mat), 256, 0, st>>>(
      (const float*)g, (const float*)buf, (const long long*)table, m, n, (const float*)hp, (const float*)scale,
      (__nv_bfloat16*)x);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_muon_apply(void* p, void* g, void* shadow, const void* table, int n_mat, int m, int n, const void* hp,
                              const void* x, const void* found_inf, int zero_grad, cudaStream_t st) {
  if (n_mat <= 0 || m % kTile || n % kTile) return -1;
  muon_apply_kernel<<<dim3((m / kTile) * (n / kTile), n_mat), 256, 0, st>>>(
      (float*)p, (float*)g, (__nv_bfloat16*)shadow, (const long long*)table, m, n, (const float*)hp, (const __nv_bfloat16*)x,
      (const int*)found_inf, zero_grad);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_adamw_segments(void* p, void* g, void* m, void* v, void* shadow, const void* chunks, int n_chunks,
                                  const void* hp, const void* gpart, int n_gpart, const void* found_inf, void* skipped,
                                  int zero_grad, cudaStream_t st) {
  if (n_chunks <= 0) return -1;
  adamw_segments_kernel<<<n_chunks, 256, 0, st>>>((float*)p, (float*)g, (float*)m, (float*)v, (__nv_bfloat16*)shadow,
                                                  (const long long*)chunks, (const float*)hp, (const float*)gpart, n_gpart,
                                                  (const int*)found_inf, (int*)skipped, zero_grad);
  ODB_CHECK_LAST();
  return 0;
}

// Cross-entropy over a logits tile for the chunked linear-cross-entropy path (SURVEY.md §2.5 K7).
// The LM-head GEMM writes a [Tc, V] bf16 tile; this kernel turns it IN PLACE into d(loss)/d(logits) and
// accumulates the un-normalised loss sum, so the fp32 [T, V] logits tensor of the reference
// (modeling_llama.py:487-491 -> loss_utils.py:45-67) never exists.
//   row r (label y, -100 = ignore):  lse = log sum_j exp(x_j) ;  loss_r = lse - x_y
//   dlogits_j = (softmax_j - [j == y]) * gscale        gscale = loss_scale / n_valid  (read from device memory)
// One CTA per row; the whole row is cached in registers (V <= 256*8*NV) so HBM sees one read and one write.
#include <limits.h>

#include "common.cuh"
#include "packed_math.cuh"

using namespace odb;

// max of the two bf16 halves of each word, packed (HMNMX2.BF16): the row maximum needs no unpacking
__device__ __forceinline__ uint32_t max_bf16x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("max.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
// One CTA per row; the row stays packed (bf16) in registers across the three passes and the arithmetic is packed fp32x2
// (FFMA2 / FADD2 / FMUL2) with branch-free loops (out-of-range vectors are padded with -inf, the label element is read
// and patched by one thread): ~7 instructions per logit instead of ~19, which is what bounded this kernel (32000 logits
// per row, 55 rows per SM per 8192-row chunk), leaving the 16-lane MUFU (one ex2 per logit) and HBM as the limits.
template <int NV, bool kSumSq>
__global__ void __launch_bounds__(256) ce_fwd_bwd_kernel(__nv_bfloat16* __restrict__ logits,
                                                         const long long* __restrict__ labels, int V, long long row_stride,
                                                         const float* __restrict__ gscale_ptr, float* __restrict__ loss_sum,
                                                         float* __restrict__ lse_out, float* __restrict__ sumsq) {
  using namespace packed_math;
  __shared__ float sm[33];
  const int row = blockIdx.x;
  const long long y = labels[row];
  __nv_bfloat16* lrow = logits + (size_t)row * row_stride;
  uint4* xr = reinterpret_cast<uint4*>(lrow);
  const int nvec = V / 8;
  const bool ignore = (y < 0);
  if (ignore && !kSumSq) {
    // masked token: gradient is zero, no loss contribution
    for (int c = threadIdx.x; c < nvec; c += 256) st_na_v4(xr + c, make_uint4(0, 0, 0, 0));
    if (lse_out && threadIdx.x == 0) lse_out[row] = 0.f;
    return;
  }
  const float x_label = (!ignore && threadIdx.x == 0) ? __bfloat162float(lrow[y]) : 0.f;   // read before the row is overwritten
  uint32_t raw[NV][4];
#pragma unroll
  for (int k = 0; k < NV; ++k) {                         // all loads of the row in flight at once
    const int c = threadIdx.x + k * 256;
    uint4 v = make_uint4(0xff80ff80u, 0xff80ff80u, 0xff80ff80u, 0xff80ff80u);      // -inf padding: exp -> 0
    if (c < nvec) v = ld_nc_v4(xr + c);
    raw[k][0] = v.x; raw[k][1] = v.y; raw[k][2] = v.z; raw[k][3] = v.w;
  }
  uint32_t m2 = 0xff80ff80u;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    m2 = max_bf16x2(max_bf16x2(m2, raw[k][0]), max_bf16x2(raw[k][1], max_bf16x2(raw[k][2], raw[k][3])));
    if constexpr (kSumSq) {
      if (threadIdx.x + k * 256 < nvec) {
        float f[8];
        unpack8(make_uint4(raw[k][0], raw[k][1], raw[k][2], raw[k][3]), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) sq += f[j] * f[j];
      }
    }
  }
  float mx = fmaxf(__uint_as_float(m2 << 16), __uint_as_float(m2 & 0xffff0000u));
  mx = block_max(mx, sm);
  // exp() once per element: the fp32 values feed the row sum, their bf16 roundings replace the logits in registers and
  // become the softmax numerators of the last pass (the output is bf16 anyway).
  const float L2E = 1.4426950408889634f;
  const uint64_t l2 = pack2(L2E, L2E), nm2 = pack2(-mx * L2E, -mx * L2E);
  uint64_t s2 = pack2(0.f, 0.f);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t w = raw[k][i];
      float e0, e1;
      unpack2(ffma2(pack2u(w << 16, w & 0xffff0000u), l2, nm2), e0, e1);
      const uint64_t e = pack2(fast_exp2(e0), fast_exp2(e1));
      s2 = fadd2(s2, e);
      raw[k][i] = cvt_bf16x2(e);
    }
  }
  float s;
  {
    float sa, sb;
    unpack2(s2, sa, sb);
    s = block_sum(sa + sb, sm);
  }
  if constexpr (kSumSq) {
    sq = block_sum(sq, sm);
    if (threadIdx.x == 0) atomicAdd(sumsq, sq);
  }
  const float lse = mx + __logf(s);
  const float gscale = ignore ? 0.f : *gscale_ptr;
  const float inv_s = gscale / s;
  const uint64_t is2 = pack2(inv_s, inv_s);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = threadIdx.x + k * 256;
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t w = raw[k][i];
      o[i] = cvt_bf16x2(fmul2(pack2u(w << 16, w & 0xffff0000u), is2));
    }
    if (c < nvec) st_na_v4(xr + c, make_uint4(o[0], o[1], o[2], o[3]));
  }
  if (!ignore) {
    __syncthreads();                                     // the vector store that covers the label element is ordered first
    if (threadIdx.x == 0) {
      // softmax - onehot at the label, from the same bf16-rounded numerator the vector pass used
      const float e_lab = bf16_round(fast_exp2(fmaf(x_label, L2E, -mx * L2E)));
      lrow[y] = __float2bfloat16(e_lab * inv_s - gscale);
      atomicAdd(loss_sum, lse - x_label);
    }
  }
  if (lse_out && threadIdx.x == 0) lse_out[row] = ignore ? 0.f : lse;
}

// forward only (evaluation): loss sum, no gradient written
template <int NV>
__global__ void __launch_bounds__(256) ce_fwd_kernel(const __nv_bfloat16* __restrict__ logits,
                                                     const long long* __restrict__ labels, int V, long long row_stride,
                                                     float* __restrict__ loss_sum) {
  __shared__ float sm[33];
  const int row = blockIdx.x;
  const long long y = labels[row];
  if (y < 0) return;
  const uint4* xr = reinterpret_cast<const uint4*>(logits + (size_t)row * row_stride);
  const int nvec = V / 8;
  uint4 raw[NV];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = threadIdx.x + k * 256;
    if (c < nvec) {
      raw[k] = ld_nc_v4(xr + c);
      float f[8];
      unpack8(raw[k], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, f[j]);
    }
  }
  mx = block_max(mx, sm);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = threadIdx.x + k * 256;
    if (c < nvec) {
      float f[8];
      unpack8(raw[k], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += __expf(f[j] - mx);
    }
  }
  s = block_sum(s, sm);
  if (threadIdx.x == 0) {
    const float xy = __bfloat162float(logits[(size_t)row * row_stride + y]);
    atomicAdd(loss_sum, mx + __logf(s) - xy);
  }
}

#define ODB_DISPATCH_NV(V, ...)                                 \
  do {                                                          \
    const int _n = ceil_div((V), 2048);                         \
    if (_n <= 1) { constexpr int NV = 1; __VA_ARGS__; }         \
    else if (_n <= 2) { constexpr int NV = 2; __VA_ARGS__; }    \
    else if (_n <= 4) { constexpr int NV = 4; __VA_ARGS__; }    \
    else if (_n <= 8) { constexpr int NV = 8; __VA_ARGS__; }    \
    else if (_n <= 16) { constexpr int NV = 16; __VA_ARGS__; }  \
    else if (_n <= 32) { constexpr int NV = 32; __VA_ARGS__; }  \
    else return -2;                                             \
  } while (0)

ODB_EXPORT int odb_ce_fwd_bwd(void* logits, const void* labels, int rows, int V, long long row_stride,
                              const void* gscale_ptr, void* loss_sum, void* lse_out, void* sumsq, cudaStream_t st) {
  if (V % 8 || row_stride % 8) return -1;
  if (rows <= 0) return 0;
  if (sumsq) {
    ODB_DISPATCH_NV(V, (ce_fwd_bwd_kernel<NV, true><<<rows, 256, 0, st>>>((__nv_bfloat16*)logits, (const long long*)labels, V,
                                                                          row_stride, (const float*)gscale_ptr,
                                                                          (float*)loss_sum, (float*)lse_out, (float*)sumsq)));
  } else {
    ODB_DISPATCH_NV(V, (ce_fwd_bwd_kernel<NV, false><<<rows, 256, 0, st>>>((__nv_bfloat16*)logits, (const long long*)labels, V,
                                                                           row_stride, (const float*)gscale_ptr,
                                                                           (float*)loss_sum, (float*)lse_out, (float*)sumsq)));
  }
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_ce_fwd(const void* logits, const void* labels, int rows, int V, long long row_stride, void* loss_sum,
                          cudaStream_t st) {
  if (V % 8 || row_stride % 8) return -1;
  if (rows <= 0) return 0;
  ODB_DISPATCH_NV(V, (ce_fwd_kernel<NV><<<rows, 256, 0, st>>>((const __nv_bfloat16*)logits, (const long long*)labels, V,
                                                              row_stride, (float*)loss_sum)));
  ODB_CHECK_LAST();
  return 0;
}

// =============================================================================================== fused linear-cross-entropy
// Host-free bookkeeping + the two thin passes around the LCE GEMMs of gemm_sm90.cu (kLCEFwd / kLCEdX):
//
//   lce_prep       labels -> HF-shifted labels (position s predicts token s+1, last position ignored), n_valid,
//                  gscale = loss_scale / max(n_valid, 1), loss_sum = 0             (replaces eight ATen launches)
//   lce_label_dot  c[t] = x[t] . W[label[t]] + 58 ln 2  (fp32)  - the shift of the exponentials, known BEFORE the GEMM,
//                  which is what lets the GEMM epilogue emit exp(z - c) directly instead of logits: the label term of
//                  sum_v exp(z_v - c) is 2^-58, so the row sum can never underflow, and loss_t = log(sum) + 58 ln 2
//   lce_finalize   per row: S = sum of the partial planes ; loss += log S ; rowscale = gscale / S ;
//                  xs[t] = bf16(rowscale * x[t])   (B operand of the dW GEMM: dW = E^T xs - scatter)
//                  dW[label[t]] += -gscale * x[t] + 2^-58 (rowscale * x[t] - xs[t])   (the one-hot term, a vector red.add
//                  per row, and the bf16 rounding of xs on the label's own product E_y xs[t], see below)
// The shift is placed kLceShiftOffset = 58 ln 2 nats ABOVE the label logit: the fp32 row sum then has head-room for best
// logits up to (100 + 58) ln 2 = 109.5 nats above the label (the GEMM epilogue clamps the exponent at 2^100), while the
// label term keeps the sum far from underflow.  loss_t = log(sum_v exp(z_v - c_t)) + kLceShiftOffset.
// The offset is a whole number of octaves so that the label's exponential is an exact power of two: the GEMM's z_y differs
// from the label dot by ~1e-5 nats, far below half a bf16 ulp, so the stored E_y is exactly 2^-58 and the gradient GEMMs see
// rowscale * E_y - gscale = gscale (p_y - 1) without a rounding bias.  (With an offset of 40, bf16(exp(-40)) is 0.17% above
// exp(-40) on every row: the label's gradient changed sign once p_y > 0.9983, pushing confident predictions down.)
constexpr float kLceShiftOffset = 40.2025365f;          // 58 ln 2
constexpr float kLceLabelExp = 3.4694470e-18f;          // 2^-58: the label's exponential, exact in bf16

__global__ void __launch_bounds__(1024) lce_prep_kernel(const long long* __restrict__ src, long long* __restrict__ dst, int B, int S,
                                                        float loss_scale, float* __restrict__ n_valid,
                                                        float* __restrict__ gscale, float* __restrict__ loss_sum) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sm[33];
  const int T = B * S;
  float cnt = 0.f;
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const int s = t % S;
    const long long y = (s == S - 1) ? -100 : src[t + 1];
    dst[t] = y;
    cnt += (y >= 0) ? 1.f : 0.f;
  }
  cnt = block_sum(cnt, sm);
  if (threadIdx.x == 0) {
    const float nv = fmaxf(cnt, 1.f);
    *n_valid = nv;
    *gscale = loss_scale / nv;
    *loss_sum = 0.f;
  }
}

__global__ void __launch_bounds__(256) lce_label_dot_kernel(const __nv_bfloat16* __restrict__ x, long long ldx,
                                                            const __nv_bfloat16* __restrict__ W, long long ldw,
                                                            const long long* __restrict__ labels, float* __restrict__ c,
                                                            int T, int h) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < T; t += gridDim.x * wpb) {
    const long long y = labels[t];
    float acc = 0.f;
    if (y >= 0) {
      const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)t * ldx);
      const uint4* wr = reinterpret_cast<const uint4*>(W + (size_t)y * ldw);
      for (int k = lane; k < h / 8; k += 32) {
        float a[8], b[8];
        unpack8(ld_nc_v4(xr + k), a);
        unpack8(ld_nc_v4(wr + k), b);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc = fmaf(a[j], b[j], acc);
      }
      acc = warp_sum(acc);
    }
    if (lane == 0) c[t] = (y >= 0) ? acc + kLceShiftOffset : 0.f;
  }
}

constexpr int LCE_FIN_ROWS = 64;       // rows per CTA of lce_finalize (256 threads: 4 plane-slices x 64 rows, then 8 warps x 8 rows)

__global__ void __launch_bounds__(256) lce_finalize_kernel(const float* __restrict__ partials, int planes, int T,
                                                           const long long* __restrict__ labels,
                                                           const float* __restrict__ gscale_ptr, float* __restrict__ loss_sum,
                                                           float* __restrict__ sumsq_out, float* __restrict__ rowscale,
                                                           const __nv_bfloat16* __restrict__ x, long long ldx,
                                                           __nv_bfloat16* __restrict__ xs, long long ldxs,
                                                           float* __restrict__ dW, long long lddw, int h) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_part[4][LCE_FIN_ROWS];
  __shared__ float s_sq[4][LCE_FIN_ROWS];
  __shared__ float s_scale[LCE_FIN_ROWS];
  __shared__ float sm[33];
  const int r = threadIdx.x & (LCE_FIN_ROWS - 1), q = threadIdx.x >> 6;
  const int t0 = blockIdx.x * LCE_FIN_ROWS;
  const int t = t0 + r;
  float s = 0.f, sq = 0.f;
  if (t < T) {
#pragma unroll 4
    for (int pl = q; pl < planes; pl += 4) s += partials[(size_t)pl * T + t];       // coalesced over the 64 rows
    if (sumsq_out) {
#pragma unroll 4
      for (int pl = q; pl < planes; pl += 4) sq += partials[(size_t)(planes + pl) * T + t];
    }
  }
  s_part[q][r] = s;
  s_sq[q][r] = sq;
  __syncthreads();
  const float gscale = *gscale_ptr;
  float loss = 0.f, sqsum = 0.f;
  if (q == 0) {
    const float S = s_part[0][r] + s_part[1][r] + s_part[2][r] + s_part[3][r];
    const bool valid = (t < T) && labels[t] >= 0;
    loss = valid ? __logf(S) + kLceShiftOffset : 0.f;
    const float rs = valid ? gscale / S : 0.f;
    s_scale[r] = rs;
    if (t < T && rowscale) rowscale[t] = rs;
    sqsum = s_sq[0][r] + s_sq[1][r] + s_sq[2][r] + s_sq[3][r];
  }
  loss = block_sum(loss, sm);                            // also orders s_scale for the second phase
  if (threadIdx.x == 0) atomicAdd(loss_sum, loss);
  if (sumsq_out) {
    sqsum = block_sum(sqsum, sm);
    if (threadIdx.x == 0) atomicAdd(sumsq_out, sqsum);
  }
  if (!xs) return;                                       // evaluation: loss only
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int rr = warp; rr < LCE_FIN_ROWS; rr += 8) {
    const int tt = t0 + rr;
    if (tt >= T) break;
    const float rs = s_scale[rr];
    const long long y = labels[tt];
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)tt * ldx);
    uint4* xo = reinterpret_cast<uint4*>(xs + (size_t)tt * ldxs);
    float* dwr = (y >= 0 && dW) ? dW + (size_t)y * lddw : nullptr;
    for (int k = lane; k < h / 8; k += 32) {
      float f[8], o[8];
      unpack8(ld_nc_v4(xr + k), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = f[j] * rs;
      const uint4 ob = pack8(o);
      st_na_v4(xo + k, ob);
      if (dwr) {
        // The dW GEMM adds E_y * xs[t] = 2^-58 bf16(rowscale x) to this row; -gscale x cancels most of it when p_y -> 1,
        // which would leave the bf16 rounding of xs (2^-9 of p_y gscale x) as the result.  Adding 2^-58 (rowscale x - xs)
        // here makes the label's own term exact to fp32: gscale (p_y - 1) x.
        float r[8];
        unpack8(ob, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = fmaf(kLceLabelExp, o[j] - r[j], -gscale * f[j]);
        red_add_f4(dwr + k * 8, make_float4(r[0], r[1], r[2], r[3]));
        red_add_f4(dwr + k * 8 + 4, make_float4(r[4], r[5], r[6], r[7]));
      }
    }
  }
}

ODB_EXPORT int odb_lce_prep(const void* labels_in, void* labels_out, int B, int S, float loss_scale, void* n_valid, void* gscale,
                            void* loss_sum, cudaStream_t st) {
  if (B <= 0 || S <= 0) return -1;
  launch_pdl(lce_prep_kernel, dim3(1), dim3(1024), 0, st, (const long long*)labels_in, (long long*)labels_out, B, S, loss_scale,
             (float*)n_valid, (float*)gscale, (float*)loss_sum);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_lce_label_dot(const void* x, long long ldx, const void* W, long long ldw, const void* labels, void* c, int T,
                                 int h, cudaStream_t st) {
  if (h % 8 || ldx % 8 || ldw % 8) return -1;
  const int blocks = ceil_div(T, 8) < sm_count() * 8 ? ceil_div(T, 8) : sm_count() * 8;
  launch_pdl(lce_label_dot_kernel, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)W, ldw,
             (const long long*)labels, (float*)c, T, h);
  ODB_CHECK_LAST();
  return 0;
}

// xs / dW / rowscale / sumsq may be null (evaluation: only the loss is produced)
ODB_EXPORT int odb_lce_finalize(const void* partials, int planes, int T, const void* labels, const void* gscale, void* loss_sum,
                                void* sumsq, void* rowscale, const void* x, long long ldx, void* xs, long long ldxs, void* dW,
                                long long lddw, int h, cudaStream_t st) {
  if (h % 8 || ldx % 8 || ldxs % 8 || lddw % 4) return -1;
  launch_pdl(lce_finalize_kernel, dim3(ceil_div(T, LCE_FIN_ROWS)), dim3(256), 0, st, (const float*)partials, planes, T,
             (const long long*)labels, (const float*)gscale, (float*)loss_sum, (float*)sumsq, (float*)rowscale,
             (const __nv_bfloat16*)x, ldx, (__nv_bfloat16*)xs, ldxs, (float*)dW, lddw, h);
  ODB_CHECK_LAST();
  return 0;
}

// =============================================================================================== scoring (per-token log-likelihood)
// Merge of the per-plane statistics of the kLCEScore GEMM epilogue (gemm_sm90.cu), per row t:
//   M* = max_p m_p ; argmax = lowest idx_p among the planes with m_p == M* ; lse = M* + log sum_p s_p exp(m_p - M*)
//   logprob[t] = z_label - lse ; greedy[t] = (argmax == label) ; rows with label < 0 give 0 / false
// Every exponent is <= 0, so the result holds for any logit range.  Same layout as lce_finalize: 256 threads = 4 plane-slices
// x 64 rows, coalesced over the rows of a plane.
__device__ __forceinline__ void score_merge(float& m, float& s, int& i, float m2, float s2, int i2) {
  if (m2 > m) {
    s = s * expf(m - m2) + s2;
    m = m2;
    i = i2;
  } else if (m2 != -INFINITY) {
    s += s2 * expf(m2 - m);
    if (m2 == m && i2 < i) i = i2;
  }
}

__global__ void __launch_bounds__(256) lce_score_finalize_kernel(const float* __restrict__ pmax, const float* __restrict__ psum,
                                                                 const int* __restrict__ pidx, const float* __restrict__ zlab,
                                                                 int planes, int T, const long long* __restrict__ labels,
                                                                 float* __restrict__ logprob, bool* __restrict__ greedy,
                                                                 float* __restrict__ lse_out, int* __restrict__ argmax_out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_m[4][LCE_FIN_ROWS], s_s[4][LCE_FIN_ROWS];
  __shared__ int s_i[4][LCE_FIN_ROWS];
  const int r = threadIdx.x & (LCE_FIN_ROWS - 1), q = threadIdx.x >> 6;
  const int t = blockIdx.x * LCE_FIN_ROWS + r;
  float m = -INFINITY, s = 0.f;
  int i = INT_MAX;
  if (t < T) {
    for (int pl = q; pl < planes; pl += 4) {
      const size_t o = (size_t)pl * T + t;
      score_merge(m, s, i, pmax[o], psum[o], pidx[o]);
    }
  }
  s_m[q][r] = m;
  s_s[q][r] = s;
  s_i[q][r] = i;
  __syncthreads();
  if (q != 0 || t >= T) return;
#pragma unroll
  for (int k = 1; k < 4; ++k) score_merge(m, s, i, s_m[k][r], s_s[k][r], s_i[k][r]);
  const float lse = m + logf(s);
  const long long y = labels[t];
  logprob[t] = y >= 0 ? zlab[t] - lse : 0.f;
  greedy[t] = y >= 0 && (long long)i == y;
  if (lse_out) lse_out[t] = lse;
  if (argmax_out) argmax_out[t] = i;
}

ODB_EXPORT int odb_lce_score_finalize(const void* pmax, const void* psum, const void* pidx, const void* zlab, int planes, int T,
                                      const void* labels, void* logprob, void* greedy, void* lse, void* argmax, cudaStream_t st) {
  if (planes <= 0 || T < 0) return -1;
  if (T == 0) return 0;
  launch_pdl(lce_score_finalize_kernel, dim3(ceil_div(T, LCE_FIN_ROWS)), dim3(256), 0, st, (const float*)pmax, (const float*)psum,
             (const int*)pidx, (const float*)zlab, planes, T, (const long long*)labels, (float*)logprob, (bool*)greedy, (float*)lse,
             (int*)argmax);
  ODB_CHECK_LAST();
  return 0;
}

// Bandwidth-bound Llama kernels for sm_90a: embedding, (residual+)RMSNorm fwd/bwd, RoPE, SwiGLU.
// All activations are bf16, all statistics / reductions fp32. 16-byte vector accesses everywhere;
// one warp owns one token row so there is no block-level synchronisation on the forward path.
//
// Reference semantics (the reference delegates to HF transformers; see SURVEY.md §2.5 K1,K2,K4,K6):
//   RMSNorm  modeling_llama.py:62-67    RoPE  modeling_llama.py:117-168    SwiGLU  modeling_llama.py:182-184
#include "common.cuh"

using namespace odb;

// =============================================================== embedding
// out[t, :] = W[ids[t], :]   (bf16 table, int64 ids)
__global__ void __launch_bounds__(256) embedding_fwd_kernel(const long long* __restrict__ ids,
                                                            const __nv_bfloat16* __restrict__ W,
                                                            __nv_bfloat16* __restrict__ out, int T, int h) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int t = blockIdx.x * warps_per_block + (threadIdx.x >> 5); t < T; t += gridDim.x * warps_per_block) {
    const long long id = ids[t];
    const uint4* src = reinterpret_cast<const uint4*>(W + (size_t)id * h);
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)t * h);
    for (int c = lane; c < h / 8; c += 32) st_na_v4(dst + c, ld_v4(src + c));
  }
}

// dW[ids[t], :] += dout[t, :]   (fp32 gradient table, vector red.add)
__global__ void __launch_bounds__(256) embedding_bwd_kernel(const long long* __restrict__ ids,
                                                            const __nv_bfloat16* __restrict__ dout,
                                                            float* __restrict__ dW, int T, int h, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int t = blockIdx.x * warps_per_block + (threadIdx.x >> 5); t < T; t += gridDim.x * warps_per_block) {
    const long long id = ids[t];
    const uint4* src = reinterpret_cast<const uint4*>(dout + (size_t)t * h);
    float* dst = dW + (size_t)id * h;
    for (int c = lane; c < h / 8; c += 32) {
      float f[8];
      unpack8(ld_nc_v4(src + c), f);
      red_add_f4(dst + c * 8, make_float4(f[0] * scale, f[1] * scale, f[2] * scale, f[3] * scale));
      red_add_f4(dst + c * 8 + 4, make_float4(f[4] * scale, f[5] * scale, f[6] * scale, f[7] * scale));
    }
  }
}

// =============================================================== RMSNorm forward (+ fused residual add)
// if delta != nullptr:  x_out <- bf16(x_in + delta)  (the new residual stream value; x_out may alias x_in)
// y = bf16( w * bf16(x * rstd) ),  rstd = rsqrt(mean(x^2) + eps) in fp32.   NCH = ceil(h / 256) register chunks.
template <int NCH>
__global__ void __launch_bounds__(256) rmsnorm_fwd_kernel(const __nv_bfloat16* x_in, __nv_bfloat16* x_out,
                                                          const __nv_bfloat16* __restrict__ delta,
                                                          const __nv_bfloat16* __restrict__ w,
                                                          __nv_bfloat16* __restrict__ y, float* __restrict__ rstd_out,
                                                          int T, int h, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int nvec = h / 8;
  // rows are software-pipelined: the next token's x / delta rows are requested before the current one is reduced
  const int stride = gridDim.x * warps_per_block;
  int t = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  constexpr bool kPipe = NCH <= 4;
  uint4 nxv[NCH], ndv[NCH];
  auto fetch = [&](int tt) {
    const uint4* xr = reinterpret_cast<const uint4*>(x_in + (size_t)tt * h);
    const uint4* dr = delta ? reinterpret_cast<const uint4*>(delta + (size_t)tt * h) : nullptr;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = lane + k * 32;
      if (c < nvec) {
        nxv[k] = ld_v4(xr + c);
        if (dr) ndv[k] = ld_nc_v4(dr + c);
      }
    }
  };
  if (kPipe && t < T) fetch(t);
  for (; t < T; t += stride) {
    if constexpr (!kPipe) fetch(t);
    uint4* xo = reinterpret_cast<uint4*>(x_out + (size_t)t * h);
    float v[NCH][8];
    uint4 cdv[NCH];
#pragma unroll
    for (int k = 0; k < NCH; ++k) { unpack8(nxv[k], v[k]); cdv[k] = ndv[k]; }
    if (kPipe && t + stride < T) fetch(t + stride);      // (x_out may alias x_in: rows of different tokens never overlap)
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = lane + k * 32;
      if (c < nvec) {
        if (delta) {
          float d[8];
          unpack8(cdv[k], d);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[k][j] = bf16_round(v[k][j] + d[j]);
          st_v4(xo + c, pack8(v[k]));
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += v[k][j] * v[k][j];
      }
    }
    ss = warp_sum(ss);
    const float r = rsqrtf(ss / (float)h + eps);
    if (lane == 0) rstd_out[t] = r;
    uint4* yr = reinterpret_cast<uint4*>(y + (size_t)t * h);
    const uint4* wr = reinterpret_cast<const uint4*>(w);
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = lane + k * 32;
      if (c < nvec) {
        float wv[8], o[8];
        unpack8(ld_v4(wr + c), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = wv[j] * bf16_round(v[k][j] * r);
        st_na_v4(yr + c, pack8(o));
      }
    }
  }
}

// =============================================================== RMSNorm backward
// xhat = x*rstd ; g = w*dy ; dx = rstd * (g - xhat * mean(g*xhat)) ; dw += sum_t dy*xhat
// dres (the gradient flowing down the residual stream) is updated in place: dres <- bf16(dres + dx).
// If dres_in == nullptr the kernel writes dres = dx (used for the final norm, where no skip path exists).
// Each warp keeps per-lane dw partial sums in registers across its rows; one smem reduction + atomics per CTA.
// 190 registers, one CTA per SM at h = 1024.
template <int NCH, bool kRegAcc>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                          const __nv_bfloat16* __restrict__ x,
                                                          const __nv_bfloat16* __restrict__ w,
                                                          const float* __restrict__ rstd,
                                                          const __nv_bfloat16* __restrict__ dres_in,
                                                          __nv_bfloat16* __restrict__ dres_out,
                                                          float* __restrict__ dw, int T, int h) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sm_dw[];  // [h] CTA accumulators
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int nvec = h / 8;
  for (int i = threadIdx.x; i < h; i += blockDim.x) sm_dw[i] = 0.f;
  __syncthreads();

  constexpr int NACC = kRegAcc ? NCH : 1;
  float acc[NACC][8];
#pragma unroll
  for (int k = 0; k < NACC; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  const uint4* wr = reinterpret_cast<const uint4*>(w);

  // The rows of a warp are software-pipelined: the three input rows of the NEXT token are requested before the current
  // one is processed, so loads stay in flight during the arithmetic (a warp owns ~14 rows; without this every row pays
  // a full memory latency).  Rows stay packed (bf16) in registers between the two passes.
  const int stride = gridDim.x * warps_per_block;
  int t = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  uint4 ndy[NCH], nx[NCH], nres[NCH];
  float nr = 0.f;
  auto fetch = [&](int tt) {
    const uint4* dyr = reinterpret_cast<const uint4*>(dy + (size_t)tt * h);
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)tt * h);
    const uint4* dir = dres_in ? reinterpret_cast<const uint4*>(dres_in + (size_t)tt * h) : nullptr;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = lane + k * 32;
      if (c < nvec) {
        ndy[k] = ld_nc_v4(dyr + c);
        nx[k] = ld_nc_v4(xr + c);
        if (dir) nres[k] = ld_v4(dir + c);
      }
    }
    nr = rstd[tt];
  };
  constexpr bool kPipe = NCH <= 4;            // wider rows do not have the registers for a second row in flight
  if (kPipe && t < T) fetch(t);
  for (; t < T; t += stride) {
    if constexpr (!kPipe) fetch(t);
    uint4 rdy[NCH], rx[NCH], rres[NCH];
#pragma unroll
    for (int k = 0; k < NCH; ++k) { rdy[k] = ndy[k]; rx[k] = nx[k]; rres[k] = nres[k]; }
    const float r = nr;
    if (kPipe && t + stride < T) fetch(t + stride);
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = lane + k * 32;
      if (c < nvec) {
        float d[8], xv[8], wv[8];
        unpack8(rdy[k], d);
        unpack8(rx[k], xv);
        unpack8(ld_v4(wr + c), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = xv[j] * r;
          dot += d[j] * wv[j] * xh;
          const float contrib = d[j] * bf16_round(xh);
          if constexpr (kRegAcc) acc[k][j] += contrib;
          else atomicAdd(&sm_dw[c * 8 + j], contrib);
        }
      }
    }
    dot = warp_sum(dot) / (float)h;
    uint4* dor = reinterpret_cast<uint4*>(dres_out + (size_t)t * h);
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = lane + k * 32;
      if (c < nvec) {
        float d[8], xv[8], wv[8], o[8];
        unpack8(rdy[k], d);
        unpack8(rx[k], xv);
        unpack8(ld_v4(wr + c), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = r * (d[j] * wv[j] - xv[j] * r * dot);
        if (dres_in) {
          float p[8];
          unpack8(rres[k], p);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += p[j];
        }
        st_v4(dor + c, pack8(o));
      }
    }
  }
  if constexpr (kRegAcc) {
    // CTA reduction of the per-warp dw partials, then one global atomic per column per CTA
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = lane + k * 32;
      if (c < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(&sm_dw[c * 8 + j], acc[k][j]);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < h; i += blockDim.x) atomicAdd(&dw[i], sm_dw[i]);
}

// =============================================================== RoPE (in place on the q and k slices of the fused qkv buffer)
// qkv row layout: [ q: n_q heads x D | k: n_kv heads x D | v: n_kv heads x D ].  HF "rotate_half" convention:
//   out[j]       = x[j]*cos[j] - x[j+D/2]*sin[j]
//   out[j+D/2]   = x[j+D/2]*cos[j] + x[j]*sin[j]            j in [0, D/2)
// position of token t is (t % S). sign = +1 forward, -1 backward (the transpose rotation).
__global__ void __launch_bounds__(256) rope_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ cos_t,
                                                   const float* __restrict__ sin_t, int T, int S, int n_rot_heads,
                                                   int D, int row_stride, float sign) {
  // one thread handles 8 consecutive j of one (token, head): loads x[j..j+8) and x[j+D/2 .. j+D/2+8)
  const int half = D / 2;
  const int vec_per_head = half / 8;
  const long long total = (long long)T * n_rot_heads * vec_per_head;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int jv = (int)(i % vec_per_head);
    const long long th = i / vec_per_head;
    const int head = (int)(th % n_rot_heads);
    const long long t = th / n_rot_heads;
    const int pos = (int)(t % S);
    __nv_bfloat16* base = qkv + (size_t)t * row_stride + (size_t)head * D + jv * 8;
    float a[8], b[8];
    unpack8(ld_v4(base), a);
    unpack8(ld_v4(base + half), b);
    const float4 c0 = ld_f4(cos_t + (size_t)pos * half + jv * 8), c1 = ld_f4(cos_t + (size_t)pos * half + jv * 8 + 4);
    const float4 s0 = ld_f4(sin_t + (size_t)pos * half + jv * 8), s1 = ld_f4(sin_t + (size_t)pos * half + jv * 8 + 4);
    const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    float oa[8], ob[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float s = sn[j] * sign;
      oa[j] = a[j] * cs[j] - b[j] * s;
      ob[j] = b[j] * cs[j] + a[j] * s;
    }
    st_v4(base, pack8(oa));
    st_v4(base + half, pack8(ob));
  }
}

// =============================================================== SwiGLU
// gu row layout: [ gate: I | up: I ] ; a = silu(gate) * up
__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ gu,
                                                         __nv_bfloat16* __restrict__ a, long long T, int I) {
  const int vec_per_row = I / 8;
  const long long total = T * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / vec_per_row;
    const int c = (int)(i % vec_per_row);
    const __nv_bfloat16* row = gu + (size_t)t * 2 * I;
    float g[8], u[8], o[8];
    unpack8(ld_nc_v4(row + c * 8), g);
    unpack8(ld_nc_v4(row + I + c * 8), u);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-g[j]));
      o[j] = g[j] * sg * u[j];
    }
    st_na_v4(a + (size_t)t * I + c * 8, pack8(o));
  }
}

// dgate = da * up * sig(g) * (1 + g*(1-sig(g))) ; dup = da * silu(g).   dgu may alias gu (in place).
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ da,
                                                         const __nv_bfloat16* gu, __nv_bfloat16* dgu, long long T,
                                                         int I) {
  const int vec_per_row = I / 8;
  const long long total = T * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / vec_per_row;
    const int c = (int)(i % vec_per_row);
    const __nv_bfloat16* row = gu + (size_t)t * 2 * I;
    __nv_bfloat16* drow = dgu + (size_t)t * 2 * I;
    float g[8], u[8], d[8], og[8], ou[8];
    unpack8(ld_v4(row + c * 8), g);
    unpack8(ld_v4(row + I + c * 8), u);
    unpack8(ld_nc_v4(da + (size_t)t * I + c * 8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-g[j]));
      og[j] = d[j] * u[j] * sg * (1.f + g[j] * (1.f - sg));
      ou[j] = d[j] * g[j] * sg;
    }
    st_v4(drow + c * 8, pack8(og));
    st_v4(drow + I + c * 8, pack8(ou));
  }
}

// =============================================================== casts / misc
__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                            long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = ld_nc_f4(src + i * 8), b = ld_nc_f4(src + i * 8 + 4);
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    st_na_v4(dst + i * 8, pack8(f));
  }
}

// out = bf16(a + b)  (plain residual add, used where no norm follows)
__global__ void __launch_bounds__(256) add_bf16_kernel(const __nv_bfloat16* a, const __nv_bfloat16* b, __nv_bfloat16* out,
                                                       long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float x[8], y[8];
    unpack8(ld_v4(a + i * 8), x);
    unpack8(ld_v4(b + i * 8), y);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] += y[j];
    st_v4(out + i * 8, pack8(x));
  }
}

// =============================================================== host launchers (C ABI)
static inline int grid_for(long long work_items, int per_block, int max_waves = 8) {
  long long g = ceil_div_ll(work_items, per_block);
  long long cap = (long long)sm_count() * max_waves;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

ODB_EXPORT int odb_embedding_fwd(const void* ids, const void* W, void* out, int T, int h, cudaStream_t st) {
  if (h % 8) return -1;
  launch_pdl(embedding_fwd_kernel, dim3(grid_for(T, 8)), dim3(256), 0, st, (const long long*)ids, (const __nv_bfloat16*)W,
             (__nv_bfloat16*)out, T, h);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_embedding_bwd(const void* ids, const void* dout, void* dW, int T, int h, float scale, cudaStream_t st) {
  if (h % 8) return -1;
  launch_pdl(embedding_bwd_kernel, dim3(grid_for(T, 8)), dim3(256), 0, st, (const long long*)ids, (const __nv_bfloat16*)dout,
             (float*)dW, T, h, scale);
  ODB_CHECK_LAST();
  return 0;
}

#define ODB_DISPATCH_NCH(h, ...)                                   \
  do {                                                             \
    const int _n = ceil_div((h), 256);                             \
    if (_n <= 1) { constexpr int NCH = 1; __VA_ARGS__; }           \
    else if (_n <= 2) { constexpr int NCH = 2; __VA_ARGS__; }      \
    else if (_n <= 3) { constexpr int NCH = 3; __VA_ARGS__; }      \
    else if (_n <= 4) { constexpr int NCH = 4; __VA_ARGS__; }      \
    else if (_n <= 8) { constexpr int NCH = 8; __VA_ARGS__; }      \
    else if (_n <= 16) { constexpr int NCH = 16; __VA_ARGS__; }    \
    else return -2;                                                \
  } while (0)

ODB_EXPORT int odb_rmsnorm_fwd(const void* x_in, void* x_out, const void* delta, const void* w, void* y, void* rstd, int T,
                               int h, float eps, cudaStream_t st) {
  if (h % 8) return -1;
  const int grid = grid_for(T, 8, 4);
  ODB_DISPATCH_NCH(h, (launch_pdl(rmsnorm_fwd_kernel<NCH>, dim3(grid), dim3(256), 0, st, (const __nv_bfloat16*)x_in,
                                  (__nv_bfloat16*)x_out, (const __nv_bfloat16*)delta, (const __nv_bfloat16*)w, (__nv_bfloat16*)y,
                                  (float*)rstd, T, h, eps)));
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_rmsnorm_bwd(const void* dy, const void* x, const void* w, const void* rstd, const void* dres_in,
                               void* dres_out, void* dw, int T, int h, cudaStream_t st) {
  if (h % 8) return -1;
  const size_t smem = (size_t)h * sizeof(float);
  const int grid = grid_for(T, 8, 2);
  ODB_DISPATCH_NCH(h, (launch_pdl(rmsnorm_bwd_kernel<NCH, (NCH <= 8)>, dim3(grid), dim3(256), smem, st,
                                  (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const float*)rstd,
                                  (const __nv_bfloat16*)dres_in, (__nv_bfloat16*)dres_out, (float*)dw, T, h)));
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_rope(void* qkv, const void* cos_t, const void* sin_t, int T, int S, int n_rot_heads, int D,
                        int row_stride, float sign, cudaStream_t st) {
  if (D % 16 || row_stride % 8) return -1;
  const long long total = (long long)T * n_rot_heads * (D / 16);
  rope_kernel<<<grid_for(total, 256), 256, 0, st>>>((__nv_bfloat16*)qkv, (const float*)cos_t, (const float*)sin_t, T, S,
                                                    n_rot_heads, D, row_stride, sign);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_swiglu_fwd(const void* gu, void* a, long long T, int I, cudaStream_t st) {
  if (I % 8) return -1;
  swiglu_fwd_kernel<<<grid_for(T * (I / 8), 256), 256, 0, st>>>((const __nv_bfloat16*)gu, (__nv_bfloat16*)a, T, I);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_swiglu_bwd(const void* da, const void* gu, void* dgu, long long T, int I, cudaStream_t st) {
  if (I % 8) return -1;
  swiglu_bwd_kernel<<<grid_for(T * (I / 8), 256), 256, 0, st>>>((const __nv_bfloat16*)da, (const __nv_bfloat16*)gu,
                                                                (__nv_bfloat16*)dgu, T, I);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_cast_f32_bf16(const void* src, void* dst, long long n, cudaStream_t st) {
  if (n % 8) return -1;
  cast_f32_bf16_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>((const float*)src, (__nv_bfloat16*)dst, n / 8);
  ODB_CHECK_LAST();
  return 0;
}

ODB_EXPORT int odb_add_bf16(const void* a, const void* b, void* out, long long n, cudaStream_t st) {
  if (n % 8) return -1;
  add_bf16_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>((const __nv_bfloat16*)a, (const __nv_bfloat16*)b,
                                                        (__nv_bfloat16*)out, n / 8);
  ODB_CHECK_LAST();
  return 0;
}

// Shared device helpers for the sm_90a kernels of opendiloco_b200.
// Everything here is header-only; each .cu is compiled on its own into libodb200.so.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdlib.h>

#define ODB_EXPORT extern "C" __attribute__((visibility("default")))

#define ODB_CHECK_LAST()                                                        \
  do {                                                                          \
    cudaError_t _e = cudaGetLastError();                                        \
    if (_e != cudaSuccess) return (int)_e;                                      \
  } while (0)

namespace odb {

constexpr int kWarp = 32;

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------- vector memory ops
// 16-byte streaming load/store: bypass L1 allocation for data touched once.
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ld_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_na_v4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_v4(void* p, const uint4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_nc_f4(const float* p) {
  uint4 r = ld_nc_v4(p);
  return make_float4(__uint_as_float(r.x), __uint_as_float(r.y), __uint_as_float(r.z), __uint_as_float(r.w));
}
__device__ __forceinline__ float4 ld_f4(const float* p) {
  uint4 r = ld_v4(p);
  return make_float4(__uint_as_float(r.x), __uint_as_float(r.y), __uint_as_float(r.z), __uint_as_float(r.w));
}
__device__ __forceinline__ void st_f4(float* p, const float4& v) {
  uint4 r = make_uint4(__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w));
  st_v4(p, r);
}
__device__ __forceinline__ void st_na_f4(float* p, const float4& v) {
  uint4 r = make_uint4(__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w));
  st_na_v4(p, r);
}
// vector fp32 reduction into global memory (sm_90+): one transaction for 4 floats
__device__ __forceinline__ void red_add_f4(float* p, const float4& v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---------------------------------------------------------------- bf16 pack / unpack
__device__ __forceinline__ float2 bf2_to_f2(uint32_t u) {
  // bf16 -> fp32 is a 16-bit shift
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
// sigmoid(x) = 0.5 * tanh(0.5 x) + 0.5 with the hardware tanh (ONE MUFU op instead of ex2 + rcp; rel. error ~2^-11, below
// the bf16 rounding of everything it feeds) - the SwiGLU GEMM epilogues are MUFU-bound otherwise
__device__ __forceinline__ float fast_sigmoid(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
  return fmaf(t, 0.5f, 0.5f);
}

__device__ __forceinline__ uint32_t f2_to_bf2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  float2 a = bf2_to_f2(u.x), b = bf2_to_f2(u.y), c = bf2_to_f2(u.z), d = bf2_to_f2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(f2_to_bf2(f[0], f[1]), f2_to_bf2(f[2], f[3]), f2_to_bf2(f[4], f[5]), f2_to_bf2(f[6], f[7]));
}
__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// ---------------------------------------------------------------- reductions
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum, result valid in every thread. `sm` must hold >= 33 floats.
__device__ __forceinline__ float block_sum(float v, float* sm) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? sm[threadIdx.x] : 0.f;
  if (wid == 0) { r = warp_sum(r); if (lane == 0) sm[32] = r; }
  __syncthreads();
  return sm[32];
}
__device__ __forceinline__ float block_max(float v, float* sm) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? sm[threadIdx.x] : -INFINITY;
  if (wid == 0) { r = warp_max(r); if (lane == 0) sm[32] = r; }
  __syncthreads();
  return sm[32];
}

// ---------------------------------------------------------------- AdamW bias corrections (adamw_step, adamw_segments, ZeRO step)
// hp[5], hp[6] hold 1 - beta^t for the host's step count t = hp[13], computed by the host in double.  A step that a
// non-finite gradient skipped (GradScaler) is not an update, so the corrections must use t minus the steps skipped so far.
// That count lives on the device, in two int slots `skipped` (nullable: no skip accounting): a launch reads slot t & 1 and
// writes slot (t + 1) & 1, which only the next step reads, so readers and the writer never share a slot and the host
// never has to read the verdict.  After a skip the corrections are recomputed in double from beta = hp[1] + hp[14]
// (resp. hp[2] + hp[15]): the fp32 slot plus the residual of the host's double.
constexpr int kHpStep = 13, kHpB1Lo = 14, kHpB2Lo = 15;
__device__ __forceinline__ void adamw_bias_corrections(const float* hp, const int* skipped, float& bc1, float& bc2) {
  bc1 = hp[5];
  bc2 = hp[6];
  if (skipped == nullptr) return;
  const int t = (int)hp[kHpStep];
  const int s = skipped[t & 1];
  if (s == 0) return;
  const double b1 = (double)hp[1] + (double)hp[kHpB1Lo], b2 = (double)hp[2] + (double)hp[kHpB2Lo];
  bc1 = (float)(1.0 - pow(b1, (double)(t - s)));
  bc2 = (float)(1.0 - pow(b2, (double)(t - s)));
}
// one thread of the launch carries the count forward: skipped[(t + 1) & 1] = skipped[t & 1] + (this step skipped)
__device__ __forceinline__ void adamw_count_skip(const float* hp, int* skipped, bool skip) {
  if (skipped == nullptr || blockIdx.x != 0 || threadIdx.x != 0) return;
  const int t = (int)hp[kHpStep];
  skipped[(t + 1) & 1] = skipped[t & 1] + (skip ? 1 : 0);
}

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// Every kernel of the micro-step raises `launch_dependents` on entry and executes `griddepcontrol.wait` before its first
// global-memory access; launched with the programmatic-serialization attribute, the NEXT kernel's CTAs are scheduled as soon
// as SM resources free up and run their prologue (barrier init, tensor-map prefetch, index math) while the
// previous kernel drains its last wave.  The wait returns only when the previous grid has completed and flushed, so the
// data dependence is exactly the stream order (also inside a captured CUDA graph, where the edge becomes programmatic).
// The attribute is OFF by default (ODB_PDL=1 turns it on); without it both instructions are no-ops and the launch is an
// ordinary one.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

inline int pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("ODB_PDL");
    v = (e && e[0] == '1') ? 1 : 0;
  }
  return v;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

}  // namespace odb

// fp32 pairs carried in one 64-bit register (two scalar FFMA / FADD / FMUL on sm_90) and exp2 helpers of the
// cross-entropy kernels.
#pragma once
#include "common.cuh"

namespace packed_math {
using namespace odb;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ---- fp32 pair helpers: two lanes of a 64-bit register pair
__device__ __forceinline__ uint64_t pack2(float a, float b) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ uint64_t pack2u(uint32_t a, uint32_t b) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(a), "r"(b));
  return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ uint64_t ffma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
__device__ __forceinline__ uint64_t fadd2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(a0 + b0, a1 + b1);
}
__device__ __forceinline__ uint32_t cvt_bf16x2(uint64_t v) {
  float a, b;
  unpack2(v, a, b);
  return f2_to_bf2(a, b);
}
__device__ __forceinline__ uint64_t fmul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(a0 * b0, a1 * b1);
}

}  // namespace packed_math

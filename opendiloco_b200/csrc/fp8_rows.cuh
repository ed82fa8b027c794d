// The FP8 rule shared by the quantisers (fp8.cu), the FP8 weight-only GEMM (fp8w_gemm_sm90.cu) and the FP8 KV cache of the
// decode kernels (decode_sm90.cu): one power-of-two scale per tensor or row, scale = 2^floor(log2(FP8_MAX / amax)),
// q = cvt.rn.satfinite(x * scale), inv = 1 / scale.  Power-of-two scales make x * scale and the dequantisation q * inv
// exact, so q * inv is a bf16 number (for inv >= 2^-126 / 2^-7 of the smallest normal: amax >= 448 * 2^-125).
#pragma once

#include <cuda_fp8.h>
#include <float.h>

#include "common.cuh"

namespace odb {

constexpr float kE4M3Max = 448.f, kE5M2Max = 57344.f;

// scale = 2^e, e = floor(log2(fmax / amax)) clamped to [-126, 126]; returns false for a non-finite amax
__device__ __forceinline__ bool fp8_scale(float amax, float fmax, float& scale) {
  if (!(amax <= FLT_MAX)) { scale = 1.f; return false; }
  if (amax == 0.f) { scale = 1.f; return true; }
  const float r = fmax / amax;                                   // IEEE division (no fast-math in this build)
  int e = isinf(r) ? 126 : (int)((__float_as_uint(r) >> 23) & 0xffu) - 127;
  e = min(126, max(-126, e));
  scale = __uint_as_float((uint32_t)(e + 127) << 23);
  return true;
}

template <bool E5M2>
__device__ __forceinline__ uint16_t cvt2(float a, float b) {
  return __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, E5M2 ? __NV_E5M2 : __NV_E4M3);
}

// two e4m3 bytes (the low 16 bits of v) -> fp32, exactly (e4m3 -> f16 is exact)
__device__ __forceinline__ float2 e4m3x2_to_f2(uint32_t v) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(v & 0xffffu), __NV_E4M3);
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}

// two e4m3 bytes -> a bf16x2 word, exactly (every e4m3 value is a bf16 number)
__device__ __forceinline__ uint32_t e4m3x2_to_bf16x2(uint32_t v) {
  const float2 f = e4m3x2_to_f2(v);
  return f2_to_bf2(f.x, f.y);
}

}  // namespace odb

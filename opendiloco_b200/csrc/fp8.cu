// Per-tensor current scaling to FP8 (e4m3 for activations and weights, e5m2 for gradients) for the FP8 GEMMs of
// gemm_sm90.cu.
//
//   amax : slot = max |x| over a bf16 tensor.  The slot is reset in-stream (memset) and reduced with an integer atomicMax
//          on the fp32 bit pattern of |x|: for non-negative floats the bit order is the value order, and inf / NaN order
//          above every finite value, so a non-finite input always reaches the slot (fmaxf would drop a NaN).
//   cast : scale = 2^floor(log2(FP8_MAX / amax)) (1 when amax = 0), q = cvt.rn.satfinite(x * scale) into the row-major copy,
//          the transposed copy or both; inv = 1 / scale for the GEMM epilogue.  A non-finite amax writes the FP8 NaN byte
//          everywhere (and inv = NaN): a diverging tensor stays visible instead of saturating to finite values.
// Power-of-two scales make x * scale and the dequantisation exact, so an FP8 GEMM equals the bf16 GEMM of the
// quantised-dequantised operands up to accumulation order.
//
//   quantize_rows : the same rule per ROW of a weight matrix (FP8 weight-only generation, ops/fp8w.py): one warp per row
//          takes the row's amax, then writes q (e4m3), inv = 1 / scale and the dequantised bf16 row q * inv.  One launch
//          covers a table of matrices (every projection of every layer).
#include "common.cuh"
#include "fp8_rows.cuh"

using namespace odb;

namespace {

constexpr int kTile = 64;          // cast tile: 64 rows x 64 columns

__device__ __forceinline__ uint32_t bf16_abs_bits_max(uint32_t acc, uint32_t w) {
  // two bf16 in one word: |x| bit patterns, widened to fp32 bit patterns
  const uint32_t lo = (w & 0x7fffu) << 16, hi = (w >> 16 & 0x7fffu) << 16;
  return max(acc, max(lo, hi));
}

__global__ void __launch_bounds__(256) amax_kernel(const uint4* __restrict__ x, long long n8, unsigned int* __restrict__ slot) {
  pdl_launch_dependents();
  pdl_wait();
  uint32_t m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = ld_nc_v4(x + i);
    m = bf16_abs_bits_max(m, v.x);
    m = bf16_abs_bits_max(m, v.y);
    m = bf16_abs_bits_max(m, v.z);
    m = bf16_abs_bits_max(m, v.w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ uint32_t sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = max(m, sm[w]);
    atomicMax(slot, m);
  }
}

// One 64 x 64 tile per CTA.  Row-major: each thread converts 2 x 8 consecutive elements (16-byte load, 8-byte store).
// Transposed: the FP8 tile goes through shared memory and each thread writes 16 consecutive bytes of one output row.
template <bool E5M2>
__global__ void __launch_bounds__(256) cast_kernel(const __nv_bfloat16* __restrict__ x, int rows, int cols,
                                                   const float* __restrict__ amax, uint8_t* __restrict__ out,
                                                   uint8_t* __restrict__ out_t, float* __restrict__ inv) {
  __shared__ uint8_t tile[kTile][kTile + 4];
  pdl_launch_dependents();
  pdl_wait();
  float scale;
  const bool ok = fp8_scale(*amax, E5M2 ? kE5M2Max : kE4M3Max, scale);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *inv = ok ? 1.f / scale : __int_as_float(0x7fffffff);
  const int r0 = blockIdx.y * kTile, c0 = blockIdx.x * kTile;
  const int c8 = (threadIdx.x & 7) * 8;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int r = (threadIdx.x >> 3) + 32 * j;
    const uint4 u = ld_nc_v4(x + (size_t)(r0 + r) * cols + c0 + c8);
    float f[8];
    unpack8(u, f);
    uint32_t w[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const uint32_t lo = cvt2<E5M2>(f[4 * k] * scale, f[4 * k + 1] * scale);
      const uint32_t hi = cvt2<E5M2>(f[4 * k + 2] * scale, f[4 * k + 3] * scale);
      w[k] = ok ? (lo | hi << 16) : 0x7f7f7f7fu;
    }
    if (out) *reinterpret_cast<uint2*>(out + (size_t)(r0 + r) * cols + c0 + c8) = make_uint2(w[0], w[1]);
    if (out_t) {
#pragma unroll
      for (int k = 0; k < 8; ++k) tile[r][c8 + k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
    }
  }
  if (out_t) {
    __syncthreads();
    const int c = threadIdx.x >> 2, rr = (threadIdx.x & 3) * 16;
    uint32_t v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      v[k] = (uint32_t)tile[rr + 4 * k][c] | (uint32_t)tile[rr + 4 * k + 1][c] << 8 | (uint32_t)tile[rr + 4 * k + 2][c] << 16 |
             (uint32_t)tile[rr + 4 * k + 3][c] << 24;
    *reinterpret_cast<uint4*>(out_t + (size_t)(c0 + c) * rows + r0 + rr) = make_uint4(v[0], v[1], v[2], v[3]);
  }
}

// One warp per row; blockIdx.y selects the matrix of the segment table: {src bf16*, q e4m3*, inv fp32*, deq bf16*, rows, cols}.
__global__ void __launch_bounds__(256) quantize_rows_kernel(const long long* __restrict__ segs) {
  const long long* sg = segs + 6 * blockIdx.y;
  const int rows = (int)sg[4], cols = (int)sg[5];
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(sg[0]) + (size_t)r * cols;
  uint8_t* q = reinterpret_cast<uint8_t*>(sg[1]) + (size_t)r * cols;
  float* inv = reinterpret_cast<float*>(sg[2]);
  __nv_bfloat16* deq = reinterpret_cast<__nv_bfloat16*>(sg[3]) + (size_t)r * cols;
  uint32_t m = 0;
  for (int c = lane * 8; c < cols; c += 256) {
    const uint4 v = ld_v4(x + c);
    m = bf16_abs_bits_max(m, v.x);
    m = bf16_abs_bits_max(m, v.y);
    m = bf16_abs_bits_max(m, v.z);
    m = bf16_abs_bits_max(m, v.w);
  }
  m = __reduce_max_sync(0xffffffffu, m);
  float scale;
  const bool ok = fp8_scale(__uint_as_float(m), kE4M3Max, scale);
  const float iv = ok ? 1.f / scale : __int_as_float(0x7fffffff);
  if (lane == 0) inv[r] = iv;
  for (int c = lane * 8; c < cols; c += 256) {
    float f[8];
    unpack8(ld_nc_v4(x + c), f);
    uint32_t w[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const uint32_t lo = cvt2<false>(f[4 * k] * scale, f[4 * k + 1] * scale);
      const uint32_t hi = cvt2<false>(f[4 * k + 2] * scale, f[4 * k + 3] * scale);
      w[k] = ok ? (lo | hi << 16) : 0x7f7f7f7fu;
    }
    *reinterpret_cast<uint2*>(q + c) = make_uint2(w[0], w[1]);
    float d[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 v = e4m3x2_to_f2(w[k >> 1] >> (16 * (k & 1)));
      d[2 * k] = v.x * iv;
      d[2 * k + 1] = v.y * iv;
    }
    st_v4(deq + c, pack8(d));
  }
}

}  // namespace

// Per-row e4m3 quantisation of n_seg bf16 matrices described by segs (device memory, 6 int64 per matrix: src, q, inv, deq
// pointers, rows, cols; cols % 8 == 0 and every row 16-byte aligned): inv[r] = 1 / scale of row r's amax, q = e4m3 copy,
// deq = bf16 q * inv.  max_rows: the largest rows of the table.
ODB_EXPORT int odb_fp8_quantize_rows(const void* segs, int n_seg, int max_rows, cudaStream_t st) {
  if (n_seg <= 0 || max_rows <= 0) return -1;
  quantize_rows_kernel<<<dim3((unsigned)ceil_div(max_rows, 8), (unsigned)n_seg), 256, 0, st>>>((const long long*)segs);
  ODB_CHECK_LAST();
  return 0;
}

// slot (fp32 device scalar) = max |x| over x[n] (bf16, n % 8 == 0, 16-byte aligned); inf / NaN propagate.
ODB_EXPORT int odb_fp8_amax(const void* x, long long n, void* slot, cudaStream_t st) {
  if (n % 8 || ((uintptr_t)x & 15)) return -1;
  cudaError_t e = cudaMemsetAsync(slot, 0, sizeof(float), st);
  if (e != cudaSuccess) return (int)e;
  if (n == 0) return 0;
  long long blocks = ceil_div_ll(n / 8, 256 * 4);
  const long long cap = (long long)sm_count() * 4;
  if (blocks > cap) blocks = cap;
  launch_pdl(amax_kernel, dim3((unsigned)blocks), dim3(256), 0, st, (const uint4*)x, n / 8, (unsigned int*)slot);
  ODB_CHECK_LAST();
  return 0;
}

// x[rows, cols] (bf16, contiguous; rows, cols % 64 == 0) -> out[rows, cols] and / or out_t[cols, rows] (FP8 bytes; either may
// be null), with the scale derived from *amax (see the file comment) and *inv = 1 / scale.  e5m2 = 0: e4m3, 1: e5m2.
ODB_EXPORT int odb_fp8_cast(const void* x, int rows, int cols, const void* amax, int e5m2, void* out, void* out_t, void* inv,
                            cudaStream_t st) {
  if (rows % kTile || cols % kTile || rows <= 0 || cols <= 0 || ((uintptr_t)x & 15) || ((uintptr_t)out & 7) ||
      ((uintptr_t)out_t & 15))
    return -1;
  const dim3 grid(cols / kTile, rows / kTile);
  if (e5m2)
    launch_pdl(cast_kernel<true>, grid, dim3(256), 0, st, (const __nv_bfloat16*)x, rows, cols, (const float*)amax, (uint8_t*)out,
               (uint8_t*)out_t, (float*)inv);
  else
    launch_pdl(cast_kernel<false>, grid, dim3(256), 0, st, (const __nv_bfloat16*)x, rows, cols, (const float*)amax, (uint8_t*)out,
               (uint8_t*)out_t, (float*)inv);
  ODB_CHECK_LAST();
  return 0;
}

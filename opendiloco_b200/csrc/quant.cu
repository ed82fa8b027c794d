// 8-bit codecs for the compressed pseudo-gradient round (SURVEY.md §2.5 K16; reference: hivemind.compression via
// open_diloco/utils.py:83-121 - CPU numpy there, bitsandbytes CUDA for the blockwise one).
//
//   blockwise8 : per-block (4096) absmax scaling to int8           q = rint(x / absmax * 127)
//   affine8    : uniform buckets  q = clamp(rint((x - mean) / scale) + 128, 0, 255)     (Uniform8BitQuantization)
//   bucket8    : arbitrary sorted borders (quantile codec), binary search in shared memory
//   lookup dequant (+ optional accumulate) : out (+)= alpha * table[q]   - the reduce stage of the butterfly averages
//                                            N dequantised parts in fp32 without materialising them
//   bucket stats: per-code fp32 sum and int32 count (shared-memory histogram) -> code book of bucket means
#include "common.cuh"

using namespace odb;

constexpr int kQBlock = 4096;

// ---------------------------------------------------------------------------------------- blockwise absmax int8
__global__ void __launch_bounds__(256) quant_blockwise8_kernel(const float* __restrict__ x, int8_t* __restrict__ q,
                                                               float* __restrict__ absmax, long long n) {
  __shared__ float sm[33];
  const long long base = (long long)blockIdx.x * kQBlock;
  float v[kQBlock / 256];
  float mx = 0.f;
#pragma unroll
  for (int k = 0; k < kQBlock / 256; ++k) {
    const long long i = base + threadIdx.x + k * 256;
    v[k] = (i < n) ? x[i] : 0.f;
    mx = fmaxf(mx, fabsf(v[k]));
  }
  mx = block_max(mx, sm);
  if (threadIdx.x == 0) absmax[blockIdx.x] = mx;
  const float inv = mx > 0.f ? 127.f / mx : 0.f;
#pragma unroll
  for (int k = 0; k < kQBlock / 256; ++k) {
    const long long i = base + threadIdx.x + k * 256;
    if (i < n) q[i] = (int8_t)__float2int_rn(v[k] * inv);
  }
}

// out (+)= alpha * q * absmax / 127
__global__ void __launch_bounds__(256) dequant_blockwise8_kernel(const int8_t* __restrict__ q, const float* __restrict__ absmax,
                                                                 float* __restrict__ out, long long n, float alpha,
                                                                 int accumulate) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float s = absmax[i / kQBlock] * (alpha / 127.f);
    const float val = (float)q[i] * s;
    out[i] = accumulate ? out[i] + val : val;
  }
}

// ---------------------------------------------------------------------------------------- affine uint8
__global__ void __launch_bounds__(256) quant_affine8_kernel(const float* __restrict__ x, uint8_t* __restrict__ q, long long n,
                                                            const float* __restrict__ mean_scale /* [mean, scale] */) {
  const float mean = mean_scale[0];
  const float inv = mean_scale[1] > 0.f ? 1.f / mean_scale[1] : 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int c = __float2int_rn((x[i] - mean) * inv) + 128;
    c = c < 0 ? 0 : (c > 255 ? 255 : c);
    q[i] = (uint8_t)c;
  }
}

// ---------------------------------------------------------------------------------------- sorted-border bucketize
// code = number of borders <= x   (255 borders -> codes 0..255)
__global__ void __launch_bounds__(256) quant_bucket8_kernel(const float* __restrict__ x, uint8_t* __restrict__ q, long long n,
                                                            const float* __restrict__ borders) {
  __shared__ float b[256];
  if (threadIdx.x < 255) b[threadIdx.x] = borders[threadIdx.x];
  if (threadIdx.x == 255) b[255] = INFINITY;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    int lo = 0, hi = 255;   // first index with b[idx] > v
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int mid = (lo + hi) >> 1;
      if (b[mid] <= v) lo = mid + 1; else hi = mid;
    }
    q[i] = (uint8_t)lo;
  }
}

// ---------------------------------------------------------------------------------------- code-book statistics
__global__ void __launch_bounds__(256) bucket_stats_kernel(const float* __restrict__ x, const uint8_t* __restrict__ q,
                                                           long long n, float* __restrict__ sums, int* __restrict__ counts) {
  // counts are integers: an fp32 count stops being exact past 2^24 members, which one bucket of a large part can hold
  __shared__ float s_sum[256];
  __shared__ int s_cnt[256];
  s_sum[threadIdx.x] = 0.f;
  s_cnt[threadIdx.x] = 0;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = q[i];
    atomicAdd(&s_sum[c], x[i]);
    atomicAdd(&s_cnt[c], 1);
  }
  __syncthreads();
  if (s_cnt[threadIdx.x] > 0) {
    atomicAdd(&sums[threadIdx.x], s_sum[threadIdx.x]);
    atomicAdd(&counts[threadIdx.x], s_cnt[threadIdx.x]);
  }
}

// out (+)= alpha * table[q]
__global__ void __launch_bounds__(256) dequant_lookup8_kernel(const uint8_t* __restrict__ q, const float* __restrict__ table,
                                                              float* __restrict__ out, long long n, float alpha, int accumulate) {
  __shared__ float t[256];
  t[threadIdx.x] = table[threadIdx.x] * alpha;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float val = t[q[i]];
    out[i] = accumulate ? out[i] + val : val;
  }
}

// ---------------------------------------------------------------------------------------- launchers
static inline int qgrid(long long n) {
  long long g = ceil_div_ll(n, 256 * 8);
  const long long cap = (long long)sm_count() * 8;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

ODB_EXPORT int odb_quant_blockwise8(const void* x, void* q, void* absmax, long long n, cudaStream_t st) {
  const int blocks = (int)ceil_div_ll(n, kQBlock);
  if (blocks == 0) return 0;
  quant_blockwise8_kernel<<<blocks, 256, 0, st>>>((const float*)x, (int8_t*)q, (float*)absmax, n);
  ODB_CHECK_LAST();
  return 0;
}
ODB_EXPORT int odb_dequant_blockwise8(const void* q, const void* absmax, void* out, long long n, float alpha, int accumulate,
                                      cudaStream_t st) {
  if (n == 0) return 0;
  dequant_blockwise8_kernel<<<qgrid(n), 256, 0, st>>>((const int8_t*)q, (const float*)absmax, (float*)out, n, alpha, accumulate);
  ODB_CHECK_LAST();
  return 0;
}
ODB_EXPORT int odb_quant_affine8(const void* x, void* q, long long n, const void* mean_scale, cudaStream_t st) {
  if (n == 0) return 0;
  quant_affine8_kernel<<<qgrid(n), 256, 0, st>>>((const float*)x, (uint8_t*)q, n, (const float*)mean_scale);
  ODB_CHECK_LAST();
  return 0;
}
ODB_EXPORT int odb_quant_bucket8(const void* x, void* q, long long n, const void* borders, cudaStream_t st) {
  if (n == 0) return 0;
  quant_bucket8_kernel<<<qgrid(n), 256, 0, st>>>((const float*)x, (uint8_t*)q, n, (const float*)borders);
  ODB_CHECK_LAST();
  return 0;
}
ODB_EXPORT int odb_bucket_stats(const void* x, const void* q, long long n, void* sums, void* counts, cudaStream_t st) {
  if (n == 0) return 0;
  bucket_stats_kernel<<<qgrid(n), 256, 0, st>>>((const float*)x, (const uint8_t*)q, n, (float*)sums, (int*)counts);
  ODB_CHECK_LAST();
  return 0;
}
ODB_EXPORT int odb_dequant_lookup8(const void* q, const void* table, void* out, long long n, float alpha, int accumulate,
                                   cudaStream_t st) {
  if (n == 0) return 0;
  dequant_lookup8_kernel<<<qgrid(n), 256, 0, st>>>((const uint8_t*)q, (const float*)table, (float*)out, n, alpha, accumulate);
  ODB_CHECK_LAST();
  return 0;
}

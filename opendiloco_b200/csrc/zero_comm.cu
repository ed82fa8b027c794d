// The optimizer step of a ZeRO-sharded DiLoCo worker as ONE kernel over NVLink/NVSwitch peer memory (SURVEY.md §2.5 N4,
// §2.3 "ZeRO-2-within-worker"; reference: FSDP SHARD_GRAD_OP / _HYBRID_SHARD_ZERO2, train_fsdp.py:239-245,395,403).
//
// Replaces   ncclReduceScatter(fp32 grads) -> norm pass -> all-reduce of the norm -> AdamW kernel -> ncclAllGather(bf16)
// by a single cooperative launch per GPU.  The fp32 gradient arena and the bf16 compute-weight arena of every GPU of the
// worker live in symmetric windows (peer-mapped + multicast-bound):
//
//   entry    every rank raises ready (stream order: its backward is complete) and waits for the G ranks of the worker
//   phase 1  rank r owns slab r:  g = (1/G) multimem.ld_reduce(grad[i])  (in-switch reduce-scatter, fp32)
//            -> written back to the own slab of the local gradient arena ; per-CTA sum of squares + non-finite flag
//   norm     grid barrier ; CTA 0 sums the partials and publishes (sumsq, flag) to every rank's exchange slots ; all ranks
//            add the G values in rank order (bit-identical norm everywhere) ; grid barrier
//   phase 2  clip + AdamW on the slab (master, m, v read / written by their owner only) ;
//            bf16(theta) multicast into EVERY rank's compute-weight arena (multimem.st = the all-gather) ;
//            the whole local gradient arena is zeroed (the other slabs were consumed by their owners in phase 1)
//   exit     done flags: nobody leaves before every owner's weights have landed everywhere
//
// Hyper-parameters are read from the same device block as adamw_step_kernel (optim.cu).
#include <cooperative_groups.h>

#include "common.cuh"

using namespace odb;
namespace cg = cooperative_groups;

namespace zero {

constexpr int kMaxPeers = 16;
constexpr int kMaxPartials = 2048;

struct PeerPtrs {
  void* p[kMaxPeers];
};

__device__ unsigned long long g_timeout_ns = 20000000000ull;

__device__ __forceinline__ float4 mm_ld_reduce_f32x4(const void* mc) {
  float4 r;
  asm volatile("multimem.ld_reduce.weak.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ void mm_st_bf16x8(void* mc, const uint4& v) {
  asm volatile("multimem.st.weak.global.v4.bf16x2 [%0], {%1,%2,%3,%4};"
               :: "l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_volatile_f32(const float* p) {
  float v;
  asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ bool spin_until_ge(const unsigned* p, unsigned seq, int* timeout_flag) {
  if (ld_acquire_sys(p) >= seq) return true;
  const unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  while (ld_acquire_sys(p) < seq) {
    if ((++spins & 1023u) == 0 && globaltimer_ns() - t0 > g_timeout_ns) {
      atomicExch(timeout_flag, 1);
      return false;
    }
  }
  return true;
}

// flag window layout per rank (uint32 words):  [0, P) ready | [P, 2P) norm published | [2P, 3P) done
// exchange window per rank (floats):           [2 * r], [2 * r + 1] = (sumsq, non-finite flag) written by rank r
// Cross-GPU barrier for the whole grid: grid.sync, CTA 0 signals every peer and waits for every peer, grid.sync.
__device__ __forceinline__ bool world_barrier(cg::grid_group& grid, const PeerPtrs& flags, int slot, int rank, int world,
                                              unsigned seq, int* timeout_flag) {
  __threadfence_system();
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x < world) {
    st_release_sys(reinterpret_cast<unsigned*>(flags.p[threadIdx.x]) + slot * kMaxPeers + rank, seq);
    spin_until_ge(reinterpret_cast<const unsigned*>(flags.p[rank]) + slot * kMaxPeers + threadIdx.x, seq, timeout_flag);
  }
  grid.sync();
  __threadfence_system();
  return *reinterpret_cast<volatile int*>(timeout_flag) == 0;
}

// kShadow: 0 = no low-precision copy (fp32 compute), 1 = multicast into every rank's arena (ZeRO-2: replicated compute
// weights), 2 = store into this rank's persistent shard only (FULL_SHARD: the engine all-gathers at forward / backward)
template <int kShadow>
__global__ void __launch_bounds__(512) zero_step_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                                        float* grad_local, const float* grad_mc, __nv_bfloat16* shadow_mc,
                                                        PeerPtrs flags, PeerPtrs xchg, int rank, int world, long long n,
                                                        const float* __restrict__ hp, float* __restrict__ partials,
                                                        float* __restrict__ bcast, int check_inf, int* __restrict__ found_inf,
                                                        int* __restrict__ skipped, float* __restrict__ out_stats, unsigned seq,
                                                        int* timeout_flag) {
  cg::grid_group grid = cg::this_grid();
  __shared__ float sm[33];
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const long long n4 = n / 4, slab4 = n4 / world;
  const long long lo = (long long)rank * slab4, hi = lo + slab4;
  const float inv_world = 1.f / (float)world;

  // ---------------- entry: the gradients of every rank of the worker are final
  if (!world_barrier(grid, flags, 0, rank, world, seq, timeout_flag)) return;

  // ---------------- phase 1: in-switch reduce-scatter of my slab + sum of squares
  float s = 0.f;
  constexpr int U = 4;
  for (long long i0 = lo + tid; i0 < hi; i0 += nthreads * U) {
    float4 g[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * nthreads;
      if (i < hi) g[u] = mm_ld_reduce_f32x4(grad_mc + i * 4);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * nthreads;
      if (i < hi) {
        g[u].x *= inv_world; g[u].y *= inv_world; g[u].z *= inv_world; g[u].w *= inv_world;
        s += g[u].x * g[u].x + g[u].y * g[u].y + g[u].z * g[u].z + g[u].w * g[u].w;
        st_f4(grad_local + i * 4, g[u]);
      }
    }
  }
  const bool bad = !isfinite(s);
  s = block_sum(s, sm);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
  if (bad) atomicOr(found_inf, 1);

  // ---------------- norm: one value per rank, summed in rank order on every rank
  __threadfence();
  grid.sync();
  if (blockIdx.x == 0) {
    float t = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) t += partials[i];
    t = block_sum(t, sm);
    if (threadIdx.x < world) {
      float* peer = reinterpret_cast<float*>(xchg.p[threadIdx.x]) + 2 * rank;
      peer[0] = t;
      peer[1] = (float)(*reinterpret_cast<volatile int*>(found_inf));
      __threadfence_system();
      st_release_sys(reinterpret_cast<unsigned*>(flags.p[threadIdx.x]) + 1 * kMaxPeers + rank, seq);
      spin_until_ge(reinterpret_cast<const unsigned*>(flags.p[rank]) + 1 * kMaxPeers + threadIdx.x, seq, timeout_flag);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const float* mine = reinterpret_cast<const float*>(xchg.p[rank]);
      float tot = 0.f, inf = 0.f;
      for (int r = 0; r < world; ++r) { tot += ld_volatile_f32(mine + 2 * r); inf += ld_volatile_f32(mine + 2 * r + 1); }
      bcast[0] = tot;
      bcast[1] = inf;
      if (inf != 0.f) *found_inf = 1;
    }
  }
  __threadfence();
  grid.sync();
  if (*reinterpret_cast<volatile int*>(timeout_flag)) return;

  // ---------------- phase 2: clip + AdamW on my slab, multicast the bf16 weights, zero the gradient arena
  const float lr = hp[0], b1 = hp[1], b2 = hp[2], eps = hp[3], wd = hp[4];
  const float max_norm = hp[7], inv_scale = hp[8];
  float bc1, bc2;
  adamw_bias_corrections(hp, skipped, bc1, bc2);
  const float gnorm = sqrtf(ld_volatile_f32(bcast)) * inv_scale;
  float coef = inv_scale, clip = 1.f;
  if (max_norm > 0.f) {
    clip = fminf(1.f, max_norm / (gnorm + 1e-6f));
    coef *= clip;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && out_stats) { out_stats[0] = gnorm; out_stats[1] = clip; }
  const bool skip = check_inf && (ld_volatile_f32(bcast + 1) != 0.f);
  adamw_count_skip(hp, skipped, skip);
  const float step_size = lr / bc1, sqrt_bc2 = sqrtf(bc2), decay = 1.f - lr * wd;
  // two float4 (= 8 weights = one 16-byte bf16 vector) per thread iteration; the slab is a multiple of 8 elements
  const long long slab8 = slab4 / 2, lo8 = (long long)rank * slab8;
  for (long long k = tid; k < slab8; k += nthreads) {
    const long long i = (lo8 + k) * 2;             // float4 index of the first half
    const long long j = k * 2;                     // same, inside the slab-local m / v / master buffers
    float w8[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float4 pp = ld_f4(p + (j + h) * 4);
      const float4 gg = ld_f4(grad_local + (i + h) * 4);
      st_f4(grad_local + (i + h) * 4, make_float4(0.f, 0.f, 0.f, 0.f));      // own slab: zeroed by the thread that consumed it
      if (!skip) {
        float4 mm = ld_f4(m + (j + h) * 4), vv = ld_f4(v + (j + h) * 4);
        float* P = &pp.x; float* M = &mm.x; float* V = &vv.x; const float* G = &gg.x;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float gr = G[e] * coef;
          const float pj = P[e] * decay;
          M[e] = M[e] + (1.f - b1) * (gr - M[e]);
          V[e] = b2 * V[e] + (1.f - b2) * gr * gr;
          P[e] = pj - step_size * (M[e] / (sqrtf(V[e]) / sqrt_bc2 + eps));
        }
        st_f4(p + (j + h) * 4, pp);
        st_f4(m + (j + h) * 4, mm);
        st_f4(v + (j + h) * 4, vv);
      }
      w8[h * 4 + 0] = pp.x; w8[h * 4 + 1] = pp.y; w8[h * 4 + 2] = pp.z; w8[h * 4 + 3] = pp.w;
    }
    if (kShadow == 1 && !skip) mm_st_bf16x8(shadow_mc + (lo8 + k) * 8, pack8(w8));
    if (kShadow == 2 && !skip) st_v4(shadow_mc + k * 8, pack8(w8));          // shadow_mc = the local shard here
  }
  // the other slabs were consumed by their owners in phase 1 (the norm exchange was the barrier): zero them here.  The own
  // slab is NOT touched by this loop - other threads of this grid may still be reading it in the AdamW loop above.
  for (long long i = tid; i < n4; i += nthreads) {
    if (i < lo || i >= hi) st_f4(grad_local + i * 4, make_float4(0.f, 0.f, 0.f, 0.f));
  }

  // ---------------- exit: every owner's weights are on every rank
  world_barrier(grid, flags, 2, rank, world, seq, timeout_flag);
}

}  // namespace zero

// p / m / v: this rank's slab (n / world elements).  grad_local / grad_mc: the full fp32 gradient arena in its symmetric
// window and the multicast alias.  shadow: multicast alias of the bf16 compute-weight arena (shadow_mode 1), this rank's
// bf16 shard (shadow_mode 2, FULL_SHARD) or null (shadow_mode 0: fp32 compute - the caller gathers).  flags / xchg: per-rank symmetric windows (3 * 16 uint32 / 2 * 16 floats), zero-initialised once.
// partials: >= 2048 floats, bcast: 2 floats (device scratch).  skipped: the optimizer's int32 [2] skipped-step counter
// (adamw_bias_corrections, common.cuh).  n % (8 * world) == 0.
ODB_EXPORT int odb_zero_fused_step(void* p, void* m, void* v, void* grad_local, void* grad_mc, void* shadow_mc, int shadow_mode,
                                   const void* const* flag_ptrs, const void* const* xchg_ptrs, int rank, int world, long long n,
                                   const void* hp, void* partials, void* bcast, int check_inf, void* found_inf, void* skipped,
                                   void* out_stats, unsigned seq, void* timeout_flag, cudaStream_t st) {
  using namespace zero;
  if (world > kMaxPeers || world < 1 || n % (8ll * world) || grad_mc == nullptr) return -1;
  PeerPtrs fp{}, xp{};
  for (int i = 0; i < world; ++i) { fp.p[i] = const_cast<void*>(flag_ptrs[i]); xp.p[i] = const_cast<void*>(xchg_ptrs[i]); }
  if ((shadow_mode != 0) != (shadow_mc != nullptr) || shadow_mode < 0 || shadow_mode > 2) return -1;
  void* fn = shadow_mode == 1 ? (void*)zero_step_kernel<1> : (shadow_mode == 2 ? (void*)zero_step_kernel<2> : (void*)zero_step_kernel<0>);
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 512, 0);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) return -3;
  int grid = sm_count() * (per_sm > 2 ? 2 : per_sm);
  if (grid > kMaxPartials) grid = kMaxPartials;
  float* a0 = (float*)p; float* a1 = (float*)m; float* a2 = (float*)v; float* a3 = (float*)grad_local;
  const float* a4 = (const float*)grad_mc; __nv_bfloat16* a5 = (__nv_bfloat16*)shadow_mc;
  const float* a6 = (const float*)hp; float* a7 = (float*)partials; float* a8 = (float*)bcast; int* a9 = (int*)found_inf;
  float* a10 = (float*)out_stats; int* a11 = (int*)timeout_flag; int* a12 = (int*)skipped;
  void* args[] = {&a0, &a1, &a2, &a3, &a4, &a5, &fp, &xp, &rank, &world, &n, &a6, &a7, &a8, &check_inf, &a9, &a12, &a10, &seq, &a11};
  e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(512), args, 0, st);
  return (int)e;
}

ODB_EXPORT int odb_zero_set_timeout_ms(int ms) {
  const unsigned long long ns = (unsigned long long)(ms > 0 ? ms : 1) * 1000000ull;
  return (int)cudaMemcpyToSymbol(zero::g_timeout_ns, &ns, sizeof(ns));
}

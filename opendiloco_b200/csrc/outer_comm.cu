// K14' - the DiLoCo outer step as ONE kernel over NVLink/NVSwitch peer memory (SURVEY.md §2.5 K14', §5.8).
//
// Replaces, per outer step, the reference's 111 x {H2D copy, subtract, NCCL all_reduce} + foreach SGD + 111 D2H copies
// (train_diloco_torch.py:340-353) and, on the hivemind path, GPU->CPU copies + libp2p butterfly all-reduce + CPU SGD
// (hivemind_diloco.py:158-167,617-665).
//
// Every rank launches the same persistent cooperative grid.  `sym` is this rank's window of a symmetric allocation
// (same size on every rank, peer-mapped and - when the fabric supports it - bound to a multicast object):
//
//   phase 0  delta = theta_outer - theta_local  -> sym (own HBM), fp32 or bf16                    [all CTAs, full vector]
//   barrier  grid + cross-GPU (flags in a second symmetric window, release/acquire at .sys scope)
//   phase 1  rank r owns slice r:  mean = (1/N) * sum_p sym_p[slice]     multimem.ld_reduce (in-switch NVLS reduction)
//            or N peer loads;      sym_p[slice] <- mean for every p       multimem.st (switch multicast) or N peer stores
//   barrier  grid + cross-GPU
//   phase 2  buf = mu*buf + mean ; theta_outer -= lr*(mean + mu*buf) ; theta_local = theta_outer ; shadow = bf16(...)
//
// i.e. compute -> reduce-scatter -> all-gather -> update, tile by tile over peer memory, in one launch.
#include <cooperative_groups.h>

#include "common.cuh"

using namespace odb;
namespace cg = cooperative_groups;

constexpr int kMaxPeers = 16;

struct PeerPtrs {
  void* p[kMaxPeers];
};

// ---------------------------------------------------------------------------------------------- multimem PTX
__device__ __forceinline__ float4 multimem_ld_reduce_f32x4(const void* mc) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st_f32x4(void* mc, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// weak (non-.sys) forms: ordering is provided by the explicit barriers around the phase, as in NCCL's NVLS kernels
__device__ __forceinline__ float4 multimem_ld_reduce_f32x4_weak(const void* mc) {
  float4 r;
  asm volatile("multimem.ld_reduce.weak.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st_f32x4_weak(void* mc, const float4& v) {
  asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// 8 bf16 values, reduced with fp32 accumulation inside the switch
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st_bf16x8(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};"
               :: "l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// loads of data written by other GPUs during this kernel: never served from a stale L1 line
__device__ __forceinline__ uint4 ld_vol_v4(const void* p) {
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ float4 ld_vol_f4(const float* p) {
  const uint4 r = ld_vol_v4(p);
  return make_float4(__uint_as_float(r.x), __uint_as_float(r.y), __uint_as_float(r.z), __uint_as_float(r.w));
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Cross-GPU waits are bounded by WALL CLOCK (globaltimer): a peer that never arrives raises the timeout flag after
// g_outer_timeout_ns (default 20 s, odb_outer_set_timeout_ms) and the kernel returns without touching any state that the
// missing data would have fed - the host polls the flag (FusedOuterStep.poll_timeout) and raises.
__device__ unsigned long long g_outer_timeout_ns = 20000000000ull;

__device__ __forceinline__ bool spin_until_ge(const unsigned* p, unsigned seq, int* timeout_flag) {
  if (ld_acquire_sys(p) >= seq) return true;
  const unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  while (ld_acquire_sys(p) < seq) {
    if ((++spins & 1023u) == 0 && globaltimer_ns() - t0 > g_outer_timeout_ns) {
      atomicExch(timeout_flag, 1);
      return false;
    }
  }
  return true;
}

// grid barrier (cooperative) + all-ranks barrier through the flag window.  flags[p][slot*kMaxPeers + r] on rank p is
// written by rank r.  `seq` increases monotonically across launches so flags never need resetting.
__device__ __forceinline__ void world_barrier(cg::grid_group& grid, const PeerPtrs& flag_ptrs, int rank, int world,
                                              unsigned seq, int slot, int* timeout_flag) {
  __threadfence_system();
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x < world) {
    const int peer = threadIdx.x;
    unsigned* remote = reinterpret_cast<unsigned*>(flag_ptrs.p[peer]) + slot * kMaxPeers + rank;
    st_release_sys(remote, seq);
    const unsigned* mine = reinterpret_cast<const unsigned*>(flag_ptrs.p[rank]) + slot * kMaxPeers + peer;
    spin_until_ge(mine, seq, timeout_flag);      // a peer is gone: flag it instead of hanging the GPU
  }
  grid.sync();
  __threadfence_system();
}

template <bool kBf16Delta, bool kMultimem>
__global__ void __launch_bounds__(512) fused_outer_kernel(float* __restrict__ theta_outer, float* __restrict__ buf,
                                                          float* __restrict__ theta_local, __nv_bfloat16* __restrict__ shadow,
                                                          void* sym_local, void* sym_mc, PeerPtrs sym_peers, PeerPtrs flag_ptrs,
                                                          int rank, int world, long long n, float lr, float mu, int nesterov,
                                                          unsigned seq, int* timeout_flag, int p1_ctas, int mm_weak, unsigned long long* stamps) {
  cg::grid_group grid = cg::this_grid();
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  constexpr int VEC = kBf16Delta ? 8 : 4;         // elements per 16-byte vector of the delta window
  const long long nvec = n / VEC;

  const bool stamp = stamps != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  if (stamp) stamps[0] = globaltimer_ns();
  // ---------------- phase 0: pseudo-gradient into the local symmetric window
  for (long long i = tid; i < nvec; i += nthreads) {
    if constexpr (kBf16Delta) {
      const float4 a0 = ld_f4(theta_outer + i * 8), a1 = ld_f4(theta_outer + i * 8 + 4);
      const float4 b0 = ld_f4(theta_local + i * 8), b1 = ld_f4(theta_local + i * 8 + 4);
      const float d[8] = {a0.x - b0.x, a0.y - b0.y, a0.z - b0.z, a0.w - b0.w, a1.x - b1.x, a1.y - b1.y, a1.z - b1.z, a1.w - b1.w};
      st_v4(reinterpret_cast<__nv_bfloat16*>(sym_local) + i * 8, pack8(d));
    } else {
      const float4 a = ld_f4(theta_outer + i * 4), b = ld_f4(theta_local + i * 4);
      st_f4(reinterpret_cast<float*>(sym_local) + i * 4, make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w));
    }
  }
  if (stamp) stamps[1] = globaltimer_ns();
  world_barrier(grid, flag_ptrs, rank, world, seq, 0, timeout_flag);
  if (*reinterpret_cast<volatile int*>(timeout_flag)) return;      // a peer never arrived: leave theta / momentum untouched
  if (stamp) stamps[2] = globaltimer_ns();

  // ---------------- phase 1: reduce my slice across ranks, publish the mean to every rank
  const float inv_world = 1.f / (float)world;
  const long long per = (nvec + world - 1) / world;
  const long long lo = per * rank, hi = (lo + per < nvec) ? lo + per : nvec;
  if constexpr (kMultimem) {
    // U independent in-switch reductions in flight per thread before the dependent multicast stores; only the first
    // p1_ctas CTAs take part (the NVLink fabric, not the SMs, is the limit of this phase)
    constexpr int U = 8;
    const long long nthreads1 = (long long)p1_ctas * blockDim.x;
    const long long nthreads = nthreads1;
    if (blockIdx.x < p1_ctas)
    for (long long i0 = lo + tid; i0 < hi; i0 += nthreads * U) {
      if constexpr (kBf16Delta) {
        uint4 s[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * nthreads;
          if (i < hi) s[u] = multimem_ld_reduce_bf16x8(reinterpret_cast<const __nv_bfloat16*>(sym_mc) + i * 8);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * nthreads;
          if (i < hi) {
            float f[8];
            unpack8(s[u], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] *= inv_world;
            multimem_st_bf16x8(reinterpret_cast<__nv_bfloat16*>(sym_mc) + i * 8, pack8(f));
          }
        }
      } else {
        float4 s[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * nthreads;
          if (i < hi) s[u] = mm_weak ? multimem_ld_reduce_f32x4_weak(reinterpret_cast<const float*>(sym_mc) + i * 4)
                                     : multimem_ld_reduce_f32x4(reinterpret_cast<const float*>(sym_mc) + i * 4);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * nthreads;
          if (i < hi) {
            s[u].x *= inv_world; s[u].y *= inv_world; s[u].z *= inv_world; s[u].w *= inv_world;
            if (mm_weak) multimem_st_f32x4_weak(reinterpret_cast<float*>(sym_mc) + i * 4, s[u]);
            else multimem_st_f32x4(reinterpret_cast<float*>(sym_mc) + i * 4, s[u]);
          }
        }
      }
    }
  } else {
    for (long long i = lo + tid; i < hi; i += nthreads) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int p = 0; p < world; ++p) {
        const int src = (rank + p) % world;          // stagger peers so the links are used evenly
        if constexpr (kBf16Delta) {
          float f[8];
          unpack8(ld_vol_v4(reinterpret_cast<const __nv_bfloat16*>(sym_peers.p[src]) + i * 8), f);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += f[j];
        } else {
          const float4 v = ld_vol_f4(reinterpret_cast<const float*>(sym_peers.p[src]) + i * 4);
          acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] *= inv_world;
      for (int p = 0; p < world; ++p) {
        const int dst = (rank + p) % world;
        if constexpr (kBf16Delta) st_v4(reinterpret_cast<__nv_bfloat16*>(sym_peers.p[dst]) + i * 8, pack8(acc));
        else st_f4(reinterpret_cast<float*>(sym_peers.p[dst]) + i * 4, make_float4(acc[0], acc[1], acc[2], acc[3]));
      }
    }
  }
  if (stamp) stamps[3] = globaltimer_ns();
  world_barrier(grid, flag_ptrs, rank, world, seq + 1, 1, timeout_flag);
  if (*reinterpret_cast<volatile int*>(timeout_flag)) return;      // window only partially averaged: do not apply it
  if (stamp) stamps[4] = globaltimer_ns();

  // ---------------- phase 2: SGD-Nesterov on the whole vector from the (now averaged) local window
  for (long long i = tid; i < n / 4; i += nthreads) {
    float4 d;
    if constexpr (kBf16Delta) {
      uint2 u;
      asm volatile("ld.volatile.global.v2.u32 {%0,%1}, [%2];" : "=r"(u.x), "=r"(u.y)
                   : "l"(reinterpret_cast<const __nv_bfloat16*>(sym_local) + i * 4) : "memory");
      const float2 a = bf2_to_f2(u.x), b = bf2_to_f2(u.y);
      d = make_float4(a.x, a.y, b.x, b.y);
    } else {
      d = ld_vol_f4(reinterpret_cast<const float*>(sym_local) + i * 4);
    }
    float4 to = ld_f4(theta_outer + i * 4), bb = ld_f4(buf + i * 4);
    float* T = &to.x; float* B = &bb.x; const float* D = &d.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      B[j] = mu * B[j] + D[j];
      const float stp = nesterov ? (D[j] + mu * B[j]) : B[j];
      T[j] -= lr * stp;
    }
    st_f4(theta_outer + i * 4, to);
    st_f4(buf + i * 4, bb);
    st_f4(theta_local + i * 4, to);
    if (shadow) *reinterpret_cast<uint2*>(shadow + i * 4) = make_uint2(f2_to_bf2(to.x, to.y), f2_to_bf2(to.z, to.w));
  }
  if (stamp) stamps[5] = globaltimer_ns();   // block 0's own end (other CTAs may still be in phase 2)
}

// =====================================================================================================================
// Pipelined version: the vector is cut into `nchunk` chunks and the three stages run as a software pipeline over chunks,
// on disjoint sets of CTAs, so the NVLink/NVSwitch reduction of chunk c overlaps the HBM-bound delta / Nesterov work on
// the other chunks (run back-to-back by the kernel above, overlapped here).
//
//   local CTAs :  for c: delta(chunk c) -> window ; last CTA to finish chunk c raises ready[c] on every rank
//                 for c: wait done[c] from every rank ; Nesterov(chunk c)
//   comm  CTAs :  for c: wait ready[c] from every rank ; multimem.ld_reduce my slice of chunk c, scale, multimem.st ;
//                        last comm CTA raises done[c] on every rank
//
// Cross-GPU flags live in the symmetric flag window (word [c*kMaxPeers + r] is written by rank r), carry a sequence
// number that grows with every launch (no resets), and are exchanged with st.release.sys / ld.acquire.sys.  Intra-GPU
// completion is counted with global atomics whose target grows with the launch index.  Every wait is bounded.
constexpr int kMaxChunks = 64;

struct PipeCounters {            // device memory, zero-initialised once, monotonic
  unsigned ready[kMaxChunks];
  unsigned done[kMaxChunks];
};

__device__ __forceinline__ bool wait_flags(const unsigned* base, int world, unsigned seq, int* timeout_flag) {
  // one thread per peer polls; returns false on timeout
  bool ok = true;
  if (threadIdx.x < world) ok = spin_until_ge(base + threadIdx.x, seq, timeout_flag);
  return __syncthreads_and(ok);
}

template <bool kBf16Delta>
__global__ void __launch_bounds__(512) fused_outer_pipelined_kernel(
    float* __restrict__ theta_outer, float* __restrict__ buf, float* __restrict__ theta_local, __nv_bfloat16* __restrict__ shadow,
    void* sym_local, void* sym_mc, PeerPtrs flag_ptrs, int rank, int world, long long n, float lr, float mu, int nesterov,
    unsigned seq, unsigned launch_idx, int nchunk, int n_comm, PipeCounters* cnt, int* timeout_flag) {
  constexpr int VEC = kBf16Delta ? 8 : 4;
  const long long nvec = n / VEC;                   // 16-byte vectors of the window
  const long long cvec = nvec / nchunk;             // per chunk (host guarantees divisibility by nchunk * world)
  const float inv_world = 1.f / (float)world;
  unsigned* my_flags = reinterpret_cast<unsigned*>(flag_ptrs.p[rank]);
  // flag layout: [0, kMaxChunks*kMaxPeers) ready, then done
  const int DONE_OFF = kMaxChunks * kMaxPeers;
  __shared__ int s_last;

  if ((int)blockIdx.x < n_comm) {
    // ------------------------------------------------------------------------------- communication CTAs
    const long long svec = cvec / world;            // my slice of every chunk
    const long long ctid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long cthreads = (long long)n_comm * blockDim.x;
    for (int c = 0; c < nchunk; ++c) {
      if (!wait_flags(my_flags + c * kMaxPeers, world, seq, timeout_flag)) return;
      const long long lo = (long long)c * cvec + (long long)rank * svec, hi = lo + svec;
      constexpr int U = 4;
      for (long long i0 = lo + ctid; i0 < hi; i0 += cthreads * U) {
        if constexpr (kBf16Delta) {
          uint4 sv[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const long long i = i0 + u * cthreads;
            if (i < hi) sv[u] = multimem_ld_reduce_bf16x8(reinterpret_cast<const __nv_bfloat16*>(sym_mc) + i * 8);
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const long long i = i0 + u * cthreads;
            if (i < hi) {
              float f[8];
              unpack8(sv[u], f);
#pragma unroll
              for (int j = 0; j < 8; ++j) f[j] *= inv_world;
              multimem_st_bf16x8(reinterpret_cast<__nv_bfloat16*>(sym_mc) + i * 8, pack8(f));
            }
          }
        } else {
          float4 sv[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const long long i = i0 + u * cthreads;
            if (i < hi) sv[u] = multimem_ld_reduce_f32x4_weak(reinterpret_cast<const float*>(sym_mc) + i * 4);
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const long long i = i0 + u * cthreads;
            if (i < hi) {
              sv[u].x *= inv_world; sv[u].y *= inv_world; sv[u].z *= inv_world; sv[u].w *= inv_world;
              multimem_st_f32x4_weak(reinterpret_cast<float*>(sym_mc) + i * 4, sv[u]);
            }
          }
        }
      }
      __threadfence_system();
      __syncthreads();
      if (threadIdx.x == 0) s_last = (atomicAdd(&cnt->done[c], 1u) + 1u == (unsigned)n_comm * launch_idx);
      __syncthreads();
      if (s_last && threadIdx.x < world) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<unsigned*>(flag_ptrs.p[threadIdx.x]) + DONE_OFF + c * kMaxPeers + rank, seq);
      }
    }
  } else {
    // ------------------------------------------------------------------------------- local (HBM-bound) CTAs
    const int n_local = gridDim.x - n_comm;
    const long long ltid = (long long)(blockIdx.x - n_comm) * blockDim.x + threadIdx.x;
    const long long lthreads = (long long)n_local * blockDim.x;
    // stage A: pseudo-gradient of every chunk into the window
    for (int c = 0; c < nchunk; ++c) {
      const long long lo = (long long)c * cvec, hi = lo + cvec;
      for (long long i = lo + ltid; i < hi; i += lthreads) {
        if constexpr (kBf16Delta) {
          const float4 a0 = ld_f4(theta_outer + i * 8), a1 = ld_f4(theta_outer + i * 8 + 4);
          const float4 b0 = ld_f4(theta_local + i * 8), b1 = ld_f4(theta_local + i * 8 + 4);
          const float d[8] = {a0.x - b0.x, a0.y - b0.y, a0.z - b0.z, a0.w - b0.w, a1.x - b1.x, a1.y - b1.y, a1.z - b1.z, a1.w - b1.w};
          st_v4(reinterpret_cast<__nv_bfloat16*>(sym_local) + i * 8, pack8(d));
        } else {
          const float4 a = ld_f4(theta_outer + i * 4), b = ld_f4(theta_local + i * 4);
          st_f4(reinterpret_cast<float*>(sym_local) + i * 4, make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w));
        }
      }
      __threadfence_system();
      __syncthreads();
      if (threadIdx.x == 0) s_last = (atomicAdd(&cnt->ready[c], 1u) + 1u == (unsigned)n_local * launch_idx);
      __syncthreads();
      if (s_last && threadIdx.x < world) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<unsigned*>(flag_ptrs.p[threadIdx.x]) + c * kMaxPeers + rank, seq);
      }
    }
    // stage C: Nesterov on every chunk as soon as all ranks published its mean
    for (int c = 0; c < nchunk; ++c) {
      if (!wait_flags(my_flags + DONE_OFF + c * kMaxPeers, world, seq, timeout_flag)) return;
      __threadfence_system();
      const long long lo4 = (long long)c * cvec * VEC / 4, hi4 = lo4 + cvec * VEC / 4;     // in float4 units of theta
      for (long long i = lo4 + ltid; i < hi4; i += lthreads) {
        float4 d;
        if constexpr (kBf16Delta) {
          uint2 u;
          asm volatile("ld.volatile.global.v2.u32 {%0,%1}, [%2];" : "=r"(u.x), "=r"(u.y)
                       : "l"(reinterpret_cast<const __nv_bfloat16*>(sym_local) + i * 4) : "memory");
          const float2 a = bf2_to_f2(u.x), b = bf2_to_f2(u.y);
          d = make_float4(a.x, a.y, b.x, b.y);
        } else {
          d = ld_vol_f4(reinterpret_cast<const float*>(sym_local) + i * 4);
        }
        float4 to = ld_f4(theta_outer + i * 4), bb = ld_f4(buf + i * 4);
        float* T = &to.x; float* B = &bb.x; const float* D = &d.x;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          B[j] = mu * B[j] + D[j];
          const float stp = nesterov ? (D[j] + mu * B[j]) : B[j];
          T[j] -= lr * stp;
        }
        st_f4(theta_outer + i * 4, to);
        st_f4(buf + i * 4, bb);
        st_f4(theta_local + i * 4, to);
        if (shadow) *reinterpret_cast<uint2*>(shadow + i * 4) = make_uint2(f2_to_bf2(to.x, to.y), f2_to_bf2(to.z, to.w));
      }
    }
  }
}

// =====================================================================================================================
// Sharded in-place version (fp32, multimem): the outer optimizer is ZeRO-1 over the swarm and the all-reduce runs on the
// MASTER WEIGHTS themselves, which live in the symmetric window:
//
//     mean_local = (1/N) multimem.ld_reduce(theta_local[i])        i in MY slab           (in-switch reduction)
//     d = theta_outer[i] - mean_local ; buf[i] = mu buf[i] + d ; theta_outer[i] -= lr (d + mu buf[i])      (my slab only)
//     multimem.st(theta_local[i] <- theta_outer[i])                                  (switch multicast, every rank)
//     every rank: shadow[j] = bf16(theta_local[j]) ; theta_outer[j] = theta_local[j]  for the slabs it does not own
//
// mean_p(theta_outer - theta_local_p) = theta_outer - mean_p(theta_local_p), so no pseudo-gradient is ever materialised:
// there is no pre-pass, the NVLink phase starts with the kernel, the momentum is read and written by its owner only
// (4 B/param/N instead of 8 B/param on every rank) and the only full-vector pass left is the bf16 shadow refresh.  HBM
// traffic per rank ~18 B/param (was 46 with the replicated update), NVLink traffic unchanged (4 B/param each way).
// The owner's momentum slab is re-replicated to the peers in the background by the host (one NCCL all-gather on a side
// stream that overlaps the next inner steps), so checkpoints / elastic rounds still see the full outer-optimizer state.
//
// Rank r owns the contiguous slab r (n/N elements); a slab is cut into nchunk chunks and the comm CTAs publish
// done[c] when chunk c of THEIR slab is on every rank; the post CTAs process chunk c of all N slabs once every rank has
// published done[c].  Entry barrier: every rank raises ready[0] when its kernel starts (stream order: its last AdamW step
// is complete), and nobody reduces before all N have.
template <int kDummy>
__global__ void __launch_bounds__(512, 2) fused_outer_sharded_kernel(
    float* __restrict__ theta_outer, float* __restrict__ buf, float* theta_local, __nv_bfloat16* __restrict__ shadow,
    float* theta_mc, PeerPtrs flag_ptrs, int rank, int world, long long n, float lr, float mu, int nesterov, unsigned seq,
    unsigned launch_idx, int nchunk, int n_comm, PipeCounters* cnt, int* timeout_flag, long long* fingerprint,
    unsigned long long* stamps) {
  const long long n4 = n / 4;                       // float4 vectors
  // optional phase profile (globaltimer, ns): [0] start, [1] entry barrier passed, [2] comm CTA 0 done, [3] a post CTA done
  if (stamps && blockIdx.x == 0 && threadIdx.x == 0) stamps[0] = globaltimer_ns();
  const long long slab4 = n4 / world;               // per owner
  const long long sub4 = slab4 / nchunk;            // per (owner, chunk)
  const float inv_world = 1.f / (float)world;
  unsigned* my_flags = reinterpret_cast<unsigned*>(flag_ptrs.p[rank]);
  const int DONE_OFF = kMaxChunks * kMaxPeers;
  __shared__ int s_last;
  __shared__ long long s_fp[16];

  if ((int)blockIdx.x < n_comm) {
    // ------------------------------------------------------------------------------- owner CTAs: reduce, update, multicast
    if (threadIdx.x < world)
      st_release_sys(reinterpret_cast<unsigned*>(flag_ptrs.p[threadIdx.x]) + rank, seq);       // ready[0][rank] on every peer
    if (!wait_flags(my_flags, world, seq, timeout_flag)) return;
    if (stamps && blockIdx.x == 0 && threadIdx.x == 0) stamps[1] = globaltimer_ns();
    const long long ctid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long cthreads = (long long)n_comm * blockDim.x;
    for (int c = 0; c < nchunk; ++c) {
      const long long lo = (long long)rank * slab4 + (long long)c * sub4, hi = lo + sub4;
      // U in-switch reductions in flight per thread (the NVLS round trip is microseconds: bytes in flight / latency is
      // what bounds this phase); theta_outer / momentum are local and fetched only when the reduced value has arrived
      constexpr int U = 6;
      for (long long i0 = lo + ctid; i0 < hi; i0 += cthreads * U) {
        float4 sv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * cthreads;
          if (i < hi) sv[u] = multimem_ld_reduce_f32x4_weak(theta_mc + i * 4);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * cthreads;
          if (i < hi) {
            float4 to = ld_f4(theta_outer + i * 4), bb = ld_f4(buf + i * 4);
            float* T = &to.x; float* B = &bb.x; const float* S = &sv[u].x;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float d = T[j] - S[j] * inv_world;
              B[j] = mu * B[j] + d;
              const float stp = nesterov ? (d + mu * B[j]) : B[j];
              T[j] -= lr * stp;
            }
            st_f4(theta_outer + i * 4, to);
            st_f4(buf + i * 4, bb);
            multimem_st_f32x4_weak(theta_mc + i * 4, to);
          }
        }
      }
      __threadfence_system();
      __syncthreads();
      if (threadIdx.x == 0) s_last = (atomicAdd(&cnt->done[c], 1u) + 1u == (unsigned)n_comm * launch_idx);
      __syncthreads();
      if (s_last && threadIdx.x < world) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<unsigned*>(flag_ptrs.p[threadIdx.x]) + DONE_OFF + c * kMaxPeers + rank, seq);
      }
    }
    if (stamps && blockIdx.x == 0 && threadIdx.x == 0) stamps[2] = globaltimer_ns();
  } else {
    // ------------------------------------------------------------------------------- post CTAs: shadow + theta_outer refresh
    const int n_local = gridDim.x - n_comm;
    const long long ltid = (long long)(blockIdx.x - n_comm) * blockDim.x + threadIdx.x;
    const long long lthreads = (long long)n_local * blockDim.x;
    long long fp = 0;
    for (int c = 0; c < nchunk; ++c) {
      if (!wait_flags(my_flags + DONE_OFF + c * kMaxPeers, world, seq, timeout_flag)) return;
      __threadfence_system();
      for (int owner = 0; owner < world; ++owner) {
        const long long lo = (long long)owner * slab4 + (long long)c * sub4, hi = lo + sub4;
        for (long long i = lo + ltid; i < hi; i += lthreads) {
          const float4 t = ld_vol_f4(theta_local + i * 4);           // written by the owner's multicast store
          if (owner != rank) st_f4(theta_outer + i * 4, t);
          if (shadow) *reinterpret_cast<uint2*>(shadow + i * 4) = make_uint2(f2_to_bf2(t.x, t.y), f2_to_bf2(t.z, t.w));
          fp += (long long)__float_as_int(t.x) + (long long)__float_as_int(t.y) + (long long)__float_as_int(t.z) +
                (long long)__float_as_int(t.w);
        }
      }
    }
    if (stamps && (int)blockIdx.x == n_comm && threadIdx.x == 0) stamps[3] = globaltimer_ns();
    if (fingerprint) {      // wrap-around integer checksum of the new theta (order independent): the drift detector
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) fp += __shfl_xor_sync(0xffffffffu, fp, o);
      if ((threadIdx.x & 31) == 0) s_fp[threadIdx.x >> 5] = fp;
      __syncthreads();
      if (threadIdx.x == 0) {
        long long tot = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += s_fp[w];
        atomicAdd(reinterpret_cast<unsigned long long*>(fingerprint), (unsigned long long)tot);
      }
    }
  }
}

// theta_local / theta_mc: this rank's window of the symmetric master-weight allocation and its multicast alias, both
// already offset to the slice the outer group averages.  n % (4 * world * nchunk) must be 0.  `fingerprint` (int64, may be
// null) must be zeroed by the caller.
ODB_EXPORT int odb_fused_outer_sharded(void* theta_outer, void* buf, void* theta_local, void* shadow, void* theta_mc,
                                       const void* const* flag_ptrs, int rank, int world, long long n, float lr, float mu,
                                       int nesterov, unsigned seq, unsigned launch_idx, int nchunk, int n_comm, void* cnt,
                                       void* timeout_flag, void* fingerprint, void* stamps, cudaStream_t st) {
  if (world > kMaxPeers || nchunk > kMaxChunks || nchunk < 1 || theta_mc == nullptr) return -1;
  if (n % (4ll * world * nchunk)) return -2;
  PeerPtrs fp{};
  for (int i = 0; i < world; ++i) fp.p[i] = const_cast<void*>(flag_ptrs[i]);
  void* fn = (void*)fused_outer_sharded_kernel<0>;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 512, 0);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) return -3;
  const int grid = sm_count() * (per_sm > 2 ? 2 : per_sm);
  // owner CTAs: the NVLS round trips saturate with well under 100 CTAs, so 64 own the slabs and the rest of the grid runs
  // the HBM-bound post pass (a choice not yet measured on H100 / NVLink 4)
  if (n_comm <= 0 || n_comm >= grid) n_comm = grid / 3 < 64 ? grid / 3 : 64;
  float* a0 = (float*)theta_outer; float* a1 = (float*)buf; float* a2 = (float*)theta_local;
  __nv_bfloat16* a3 = (__nv_bfloat16*)shadow; float* a4 = (float*)theta_mc; int* tf = (int*)timeout_flag;
  PipeCounters* pc = (PipeCounters*)cnt; long long* fpr = (long long*)fingerprint;
  unsigned long long* stp = (unsigned long long*)stamps;
  void* args[] = {&a0, &a1, &a2, &a3, &a4, &fp, &rank, &world, &n, &lr, &mu, &nesterov, &seq, &launch_idx, &nchunk, &n_comm,
                  &pc, &tf, &fpr, &stp};
  e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(512), args, 0, st);   // cooperative = all CTAs co-resident (they spin)
  return (int)e;
}

ODB_EXPORT int odb_outer_set_timeout_ms(int ms) {
  const unsigned long long ns = (unsigned long long)(ms > 0 ? ms : 1) * 1000000ull;
  return (int)cudaMemcpyToSymbol(g_outer_timeout_ns, &ns, sizeof(ns));
}

// =====================================================================================================================
// Partial (elastic) round over the symmetric window: only the ranks listed in `members` take part - the workers that
// missed the matchmaking window are neither waited for nor read.  Same three phases as fused_outer_kernel with peer
// loads / stores (a multicast group spans all ranks, a subset cannot use it): member k of the round owns slice k of the
// vector, sums the members' windows for it and writes the mean back into every member's window; every member then
// applies Nesterov to its own full copy of theta_outer / momentum (the replicated outer state of an elastic swarm).
struct Members {
  int rank[kMaxPeers];
};

__device__ __forceinline__ void members_barrier(cg::grid_group& grid, const PeerPtrs& flag_ptrs, const Members& mem, int nm,
                                                int rank, unsigned seq, int slot, int* timeout_flag) {
  __threadfence_system();
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x < nm) {
    const int peer = mem.rank[threadIdx.x];
    st_release_sys(reinterpret_cast<unsigned*>(flag_ptrs.p[peer]) + slot * kMaxPeers + rank, seq);
    spin_until_ge(reinterpret_cast<const unsigned*>(flag_ptrs.p[rank]) + slot * kMaxPeers + peer, seq, timeout_flag);
  }
  grid.sync();
  __threadfence_system();
}

template <bool kBf16Delta>
__global__ void __launch_bounds__(512) fused_outer_subset_kernel(float* __restrict__ theta_outer, float* __restrict__ buf,
                                                                 float* __restrict__ theta_local, __nv_bfloat16* __restrict__ shadow,
                                                                 void* sym_local, PeerPtrs sym_peers, PeerPtrs flag_ptrs, Members mem,
                                                                 int nm, int my_idx, int rank, long long n, float lr, float mu,
                                                                 int nesterov, unsigned seq, int* timeout_flag) {
  cg::grid_group grid = cg::this_grid();
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  constexpr int VEC = kBf16Delta ? 8 : 4;
  const long long nvec = n / VEC;
  for (long long i = tid; i < nvec; i += nthreads) {
    if constexpr (kBf16Delta) {
      const float4 a0 = ld_f4(theta_outer + i * 8), a1 = ld_f4(theta_outer + i * 8 + 4);
      const float4 b0 = ld_f4(theta_local + i * 8), b1 = ld_f4(theta_local + i * 8 + 4);
      const float d[8] = {a0.x - b0.x, a0.y - b0.y, a0.z - b0.z, a0.w - b0.w, a1.x - b1.x, a1.y - b1.y, a1.z - b1.z, a1.w - b1.w};
      st_v4(reinterpret_cast<__nv_bfloat16*>(sym_local) + i * 8, pack8(d));
    } else {
      const float4 a = ld_f4(theta_outer + i * 4), b = ld_f4(theta_local + i * 4);
      st_f4(reinterpret_cast<float*>(sym_local) + i * 4, make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w));
    }
  }
  members_barrier(grid, flag_ptrs, mem, nm, rank, seq, 0, timeout_flag);
  if (*reinterpret_cast<volatile int*>(timeout_flag)) return;
  const float inv = 1.f / (float)nm;
  const long long per = (nvec + nm - 1) / nm;
  const long long lo = per * my_idx, hi = (lo + per < nvec) ? lo + per : nvec;
  for (long long i = lo + tid; i < hi; i += nthreads) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < nm; ++k) {
      const int src = mem.rank[(my_idx + k) % nm];         // stagger the peers so the links are used evenly
      if constexpr (kBf16Delta) {
        float f[8];
        unpack8(ld_vol_v4(reinterpret_cast<const __nv_bfloat16*>(sym_peers.p[src]) + i * 8), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      } else {
        const float4 v = ld_vol_f4(reinterpret_cast<const float*>(sym_peers.p[src]) + i * 4);
        acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    for (int k = 0; k < nm; ++k) {
      const int dst = mem.rank[(my_idx + k) % nm];
      if constexpr (kBf16Delta) st_v4(reinterpret_cast<__nv_bfloat16*>(sym_peers.p[dst]) + i * 8, pack8(acc));
      else st_f4(reinterpret_cast<float*>(sym_peers.p[dst]) + i * 4, make_float4(acc[0], acc[1], acc[2], acc[3]));
    }
  }
  members_barrier(grid, flag_ptrs, mem, nm, rank, seq + 1, 1, timeout_flag);
  if (*reinterpret_cast<volatile int*>(timeout_flag)) return;
  for (long long i = tid; i < n / 4; i += nthreads) {
    float4 d;
    if constexpr (kBf16Delta) {
      uint2 u;
      asm volatile("ld.volatile.global.v2.u32 {%0,%1}, [%2];" : "=r"(u.x), "=r"(u.y)
                   : "l"(reinterpret_cast<const __nv_bfloat16*>(sym_local) + i * 4) : "memory");
      const float2 a = bf2_to_f2(u.x), b = bf2_to_f2(u.y);
      d = make_float4(a.x, a.y, b.x, b.y);
    } else {
      d = ld_vol_f4(reinterpret_cast<const float*>(sym_local) + i * 4);
    }
    float4 to = ld_f4(theta_outer + i * 4), bb = ld_f4(buf + i * 4);
    float* T = &to.x; float* B = &bb.x; const float* D = &d.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      B[j] = mu * B[j] + D[j];
      const float stp = nesterov ? (D[j] + mu * B[j]) : B[j];
      T[j] -= lr * stp;
    }
    st_f4(theta_outer + i * 4, to);
    st_f4(buf + i * 4, bb);
    st_f4(theta_local + i * 4, to);
    if (shadow) *reinterpret_cast<uint2*>(shadow + i * 4) = make_uint2(f2_to_bf2(to.x, to.y), f2_to_bf2(to.z, to.w));
  }
}

// members: sorted ranks (inside the outer group) of this round, nm of them, this rank included.  n % 8 == 0.
ODB_EXPORT int odb_fused_outer_subset(void* theta_outer, void* buf, void* theta_local, void* shadow, void* sym_local,
                                      const void* const* sym_peers, const void* const* flag_ptrs, const int* members, int nm,
                                      int rank, int world, long long n, float lr, float mu, int nesterov, unsigned seq,
                                      int delta_bf16, void* timeout_flag, cudaStream_t st) {
  if (world > kMaxPeers || nm < 2 || nm > world || n % 8) return -1;
  PeerPtrs sp{}, fp{};
  for (int i = 0; i < world; ++i) {
    sp.p[i] = const_cast<void*>(sym_peers[i]);
    fp.p[i] = const_cast<void*>(flag_ptrs[i]);
  }
  Members mem{};
  int my_idx = -1;
  for (int k = 0; k < nm; ++k) {
    mem.rank[k] = members[k];
    if (members[k] == rank) my_idx = k;
  }
  if (my_idx < 0) return -2;
  void* fn = delta_bf16 ? (void*)fused_outer_subset_kernel<true> : (void*)fused_outer_subset_kernel<false>;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 512, 0);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) return -3;
  const int grid = sm_count() * (per_sm > 2 ? 2 : per_sm);
  float* a0 = (float*)theta_outer; float* a1 = (float*)buf; float* a2 = (float*)theta_local;
  __nv_bfloat16* a3 = (__nv_bfloat16*)shadow; int* tf = (int*)timeout_flag;
  void* args[] = {&a0, &a1, &a2, &a3, &sym_local, &sp, &fp, &mem, &nm, &my_idx, &rank, &n, &lr, &mu, &nesterov, &seq, &tf};
  e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(512), args, 0, st);
  return (int)e;
}

// Pipelined launch (multimem only).  `cnt` = zero-initialised PipeCounters in device memory owned by the caller;
// `launch_idx` = 1, 2, 3, ... ; `seq` as for the kernel above.  n % (8 * world * nchunk) must be 0.
ODB_EXPORT int odb_fused_outer_pipelined(void* theta_outer, void* buf, void* theta_local, void* shadow, void* sym_local,
                                         void* sym_mc, const void* const* flag_ptrs, int rank, int world, long long n, float lr,
                                         float mu, int nesterov, unsigned seq, unsigned launch_idx, int nchunk, int n_comm,
                                         int delta_bf16, void* cnt, void* timeout_flag, cudaStream_t st) {
  if (world > kMaxPeers || nchunk > kMaxChunks || nchunk < 1 || sym_mc == nullptr) return -1;
  if (n % (8ll * world * nchunk)) return -2;
  PeerPtrs fp{};
  for (int i = 0; i < world; ++i) fp.p[i] = const_cast<void*>(flag_ptrs[i]);
  void* fn = delta_bf16 ? (void*)fused_outer_pipelined_kernel<true> : (void*)fused_outer_pipelined_kernel<false>;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 512, 0);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) return -3;
  const int grid = sm_count() * (per_sm > 2 ? 2 : per_sm);
  if (n_comm <= 0 || n_comm >= grid) n_comm = grid / 6;
  float* a0 = (float*)theta_outer; float* a1 = (float*)buf; float* a2 = (float*)theta_local;
  __nv_bfloat16* a3 = (__nv_bfloat16*)shadow; int* tf = (int*)timeout_flag; PipeCounters* pc = (PipeCounters*)cnt;
  void* args[] = {&a0, &a1, &a2, &a3, &sym_local, &sym_mc, &fp, &rank, &world, &n, &lr, &mu, &nesterov, &seq, &launch_idx,
                  &nchunk, &n_comm, &pc, &tf};
  e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(512), args, 0, st);   // cooperative = all CTAs co-resident (they spin)
  return (int)e;
}

// n must be a multiple of 8*world (flat arenas are padded to 16384).  Returns 0, a cudaError, or -3 if co-residency fails.
ODB_EXPORT int odb_fused_outer_step(void* theta_outer, void* buf, void* theta_local, void* shadow, void* sym_local,
                                    void* sym_mc, const void* const* sym_peers, const void* const* flag_ptrs, int rank,
                                    int world, long long n, float lr, float mu, int nesterov, unsigned seq, int delta_bf16,
                                    void* timeout_flag, int p1_ctas, int mm_weak, void* stamps, cudaStream_t st) {
  if (world > kMaxPeers || n % (8ll * world)) return -1;
  PeerPtrs sp{}, fp{};
  for (int i = 0; i < world; ++i) {
    sp.p[i] = const_cast<void*>(sym_peers[i]);
    fp.p[i] = const_cast<void*>(flag_ptrs[i]);
  }
  const bool mm = sym_mc != nullptr;
  void* fn;
  if (delta_bf16) fn = mm ? (void*)fused_outer_kernel<true, true> : (void*)fused_outer_kernel<true, false>;
  else fn = mm ? (void*)fused_outer_kernel<false, true> : (void*)fused_outer_kernel<false, false>;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 512, 0);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) return -3;
  const int grid = sm_count() * (per_sm > 2 ? 2 : per_sm);
  float* a0 = (float*)theta_outer; float* a1 = (float*)buf; float* a2 = (float*)theta_local;
  __nv_bfloat16* a3 = (__nv_bfloat16*)shadow; int* tf = (int*)timeout_flag;
  if (p1_ctas <= 0 || p1_ctas > grid) p1_ctas = grid;
  void* args[] = {&a0, &a1, &a2, &a3, &sym_local, &sym_mc, &sp, &fp, &rank, &world, &n, &lr, &mu, &nesterov, &seq, &tf, &p1_ctas, &mm_weak, &stamps};
  e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(512), args, 0, st);
  return (int)e;
}

// wgmma / TMA / mbarrier GEMM family for sm_90a with fused Llama epilogues (SURVEY.md §2.5 K3, K4, K6, K7).
//
//   C[M,N] = A[M,K] * B[N,K]^T      bf16 operands, fp32 accumulation in registers
//
// 128 x 256 output tiles, 384 threads in three warpgroups, persistent: the grid has min(work items, SMs) CTAs and CTA c
// computes work items c, c + gridDim.x, c + 2 gridDim.x, ...  (the items running at any moment are consecutive, so the
// rasterisation of tile_coords holds).
//   warpgroup 0    TMA producer (one thread): A tile 128x64, B tile 256x64 per stage (128-byte swizzle), mbarrier
//                  full/empty ring of STAGES stages that runs on across all of the CTA's tiles (stage and phase carry
//                  over), so the next tile's first stages load while the MMA warpgroups run an epilogue; gives its
//                  registers to the MMA warpgroups (setmaxnreg)
//   warpgroups 1-2 MMA + epilogue: each issues wgmma m64n256k16 for its 64 rows of the tile (4 per 64-deep k-block),
//                  keeps one wgmma group in flight, releases the tile's last stage as soon as its MMAs retire, then runs
//                  the fused epilogue from the accumulator registers.  Stored outputs go through a 16 KB staging buffer per
//                  warpgroup (two 64-row x 128-byte boxes, 128-byte swizzle, the layout TMA writes for a load) and leave by
//                  TMA (cp.async.bulk.tensor stores, fp32 reduce-add for the weight gradient); the tensor map of the
//                  output clips partial tiles.  A box is rewritten only after the store that read it has (bulk_wait_read).
//
// Operand layouts (template flags, the shared-memory descriptor expresses both - no transposed copies are made):
//   A_MN = false : A is [M, K] row-major (K-major)          A_MN = true : A is [K, M] row-major (MN-major, wgrad)
//   B_MN = false : B is [N, K] row-major (K-major)          B_MN = true : B is [K, N] row-major (MN-major, dgrad)
//
// Epilogues:
//   kStore   : plain bf16 store
//   kSwiGLU  : B rows are [gate rows n0..n0+127 | up rows I+n0..I+n0+127]; writes gate|up (needed by backward) AND
//              act = silu(gate) * up, so the SwiGLU kernel and its re-read of the 2I-wide tensor disappear
//   kSwiGLUBwd: the GEMM result is d(act) of the down projection; the epilogue reads the matching gate / up values of
//              C = gu [M, 2I] and turns them IN PLACE into d(gate) / d(up) - d(act) never reaches memory.  The producer
//              carries the gate / up values through the operand ring behind the tile's last k-block (one ring entry per
//              64-column round), so they arrive while the last MMAs run; d(gate) / d(up) leave by TMA like the other outputs
//   kRoPE    : C is the packed qkv buffer; 64-column chunks are heads; chunks below `rope_cols` are rotated with the
//              HF rotate-half convention using fp32 cos/sin tables (position = row % S)
//   kLCEFwd  : fused linear-cross-entropy forward.  The accumulator holds a tile of LM-head logits z; the epilogue turns
//              it into shifted exponentials e = exp(z - c_row) (c_row = the row's label logit + 58 ln 2, so the label's
//              e is exactly 2^-58 in bf16 and loss_row = log sum_v e + 58 ln 2; csrc/lce.cu), writes the tile's row sums
//              into one partial plane per 256-column tile and
//              (training only) stores bf16(e).  Logits are never written.
//   kLCEdX   : dgrad of the LM head on the shifted exponentials: out = rowscale * acc - g * W[label]
//   kLCEScore: scoring (evaluation) statistics of the LM head, per row and 256-column plane: the plane maximum m, its lowest
//              column, s = sum exp(z - m) (every exponent <= 0: exact for any logit range, no clamp) and the label logit z_y
//              taken from the same accumulator.  Nothing of size [M, N] is written.
//   kWgradAcc: fp32 reduce-add of the tile into dW (gradient accumulation across micro-batches + split-K over tokens)
//   kAxpby   : C[b] = alpha * acc + beta * D[b] (D bf16 in C's layout, may be null), for a batch of equal-shaped problems
//              stacked along rows: work item w is tile w % tiles of problem b = w / tiles, which reads A rows from b * a_rows and B rows from
//              b * b_rows of the stacked tensors (Newton-Schulz of the Muon optimizer, csrc/muon.cu).  The stacking is
//              exact when K % 64 == 0: a tile then never reads another problem's rows into a valid output element.
//
// Element type (ELEM): 0 = bf16 operands (everything above).  1 / 2 = FP8 operands, A e4m3 / e5m2, B e4m3, both K-major
// (odb_gemm_fp8_*, odb_wgrad_fp8).  An FP8 k-block is 128 elements deep: the same 128-byte swizzle rows as bf16.  The
// tensor core's FP8 accumulation is narrower than fp32, so each consumer warpgroup issues every k-block as 4 x m64n128k32
// into a fresh 64-register scratch accumulator, waits, and adds it into its fp32 accumulator: partial sums are promoted to
// fp32 once per 128 products.  Scratch plus accumulator are kept within the 168 registers a thread of a 384-thread CTA
// is launched with (a tile relying on the setmaxnreg budget was not tried), so the FP8 tile is 128 x 128 (64 + 64 registers)
// instead of 128 x 256; the epilogues take the tile width as a constant.  They first multiply the accumulator by the two
// dequantisation factors (device scalars inv_a * inv_b, powers of two), then run as for bf16.
#include <limits.h>
#include <stdlib.h>

#include "common.cuh"
#include "sm90_ptx.cuh"

using namespace odb;
using namespace sm90;

namespace gemm {

constexpr int BM = 128, BN = 256, BK = 64;
constexpr int BK8 = 128;                   // k-block depth of the FP8 kernels (128 one-byte elements = one swizzle row)
constexpr int A_BYTES = BM * BK * 2;       // 16 KB
constexpr int B_BYTES = BN * BK * 2;       // 32 KB
constexpr int BOX_BYTES = 64 * 64 * 2;     // one 64 x 64 box of an MN-major operand
constexpr int STAGES = 4;
constexpr int THREADS = 384;
constexpr int OUT_BOX = 64 * 128;          // one output box: 64 rows x 128 bytes (64 bf16 or 32 fp32 columns)
constexpr int STG_BYTES = 2 * OUT_BOX;     // output staging of one MMA warpgroup
constexpr int SMEM_BYTES = STAGES * (A_BYTES + B_BYTES) + 2 * STG_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static_assert(SMEM_BYTES <= 232448, "sm_90 opt-in shared memory per block");
constexpr int GROUP_M = 8;                 // rasterisation: 8 m-blocks x all n-blocks per super-block (L2 reuse of A and B)

enum Epi { kStore = 0, kSwiGLU = 1, kRoPE = 2, kSwiGLUBwd = 3, kLCEFwd = 4, kLCEdX = 5, kWgradAcc = 6, kLCEScore = 7, kAxpby = 8 };

// group_m > 0: groups of group_m m-blocks x all n-blocks, m fastest inside a group (A and B tiles of a group stay in L2).
// group_m == 0: n fastest over the whole problem - for a few n-blocks and a very deep K (the LM-head dX: 4 n-blocks,
// K = vocabulary) the CTAs that share an A row-block then run side by side and A is fetched from HBM once.
__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int group_m, int& m_blk, int& n_blk) {
  if (group_m == 0) {
    m_blk = tile / num_n;
    n_blk = tile - m_blk * num_n;
    return;
  }
  const int group_size = group_m * num_n;
  const int group_id = tile / group_size;
  const int first_m = group_id * group_m;
  const int gsz = (num_m - first_m) < group_m ? (num_m - first_m) : group_m;
  const int r = tile - group_id * group_size;
  m_blk = first_m + r % gsz;
  n_blk = r / gsz;
}

struct Params {
  int M, N, K;
  int num_m, num_n;          // tile counts
  int group_m;               // rasterisation (see tile_coords)
  int splits, kb_per_split;  // split-K (kWgradAcc): work item = tile * splits + split
  void* C; long long ldc;
  void* aux; long long ldaux;
  int I;                     // kSwiGLU / kSwiGLUBwd: intermediate size
  int S, rope_cols;          // kRoPE: sequence length, number of leading columns that get rotated
  const float* cos_t;        // [S, 32] fp32 (head_dim 64)
  const float* sin_t;
  int ks1, ks2;              // A split along K (A_MN = false) or along M (A_MN = true) into up to three tensors:
                             // blocks [0,ks1) from A, [ks1,ks2) from A1, [ks2,..) from A2 (0/0 = single tensor)
  const float* row_shift;    // kLCEFwd: c_row [M] (label logit + 58 ln 2; 0 for ignored rows)
  float* partials;           // kLCEFwd: [num_n (+ num_n when want_sumsq)][M] partial row sums of exp(z - c)
  int want_sumsq;            // kLCEFwd: also accumulate sum z^2 into the second half of partials
  int store;                 // kLCEFwd: 1 = write bf16(e) to C (training) ; 0 = statistics only (evaluation)
  const float* rowscale;     // kLCEdX: s_row [M] = gscale / sum_v e  (0 for ignored rows)
  const long long* labels;   // kLCEdX: [M], < 0 = ignored
  const float* gscale;       // kLCEdX: device scalar loss_scale / n_valid
  const __nv_bfloat16* wlab; // kLCEdX: the LM-head weight [V, N] (row stride ldwlab) for the one-hot gather
  long long ldwlab;
  float* sc_max;             // kLCEScore: [num_n][M] plane maxima (labels: [M], < 0 = no label logit written)
  float* sc_sum;             // kLCEScore: [num_n][M] sum over the plane of exp(z - plane maximum)
  int* sc_idx;               // kLCEScore: [num_n][M] lowest column holding the plane maximum
  float* sc_zlab;            // kLCEScore: [M] the label logit
  const float* inv_a;        // FP8: device scalars 1 / scale of A and of B (dequantisation in the epilogue)
  const float* inv_b;
  int a_rows, b_rows;        // kAxpby: row offset of problem b in the stacked A / B tensors is b * a_rows / b * b_rows
  long long c_bstride;       // kAxpby: elements between consecutive problems of C and D (D = aux, row stride ldc)
  float alpha, beta;         // kAxpby
  int batch;                 // kAxpby: number of problems (1 otherwise)
};

__device__ __forceinline__ void st_bf2(void* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = f2_to_bf2(a, b); }
__device__ __forceinline__ float2 ld_bf2(const void* p) { return bf2_to_f2(*reinterpret_cast<const uint32_t*>(p)); }
__device__ __forceinline__ void sts_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_f2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// One work item: a tile of the output (a K-slice of it for split-K) of problem b (kAxpby)
struct Tile {
  int m_blk, n_blk, m0, n0, kb0, kb1, b;
};

template <int ELEM>
__device__ __forceinline__ Tile tile_of(const Params& p, int work) {
  constexpr int KB = ELEM ? BK8 : BK;            // elements per k-block
  constexpr int BNE = ELEM ? BN / 2 : BN;        // tile columns
  const int per_batch = p.num_m * p.num_n * p.splits;
  Tile t;
  t.b = work / per_batch;
  work -= t.b * per_batch;
  const int tile = work / p.splits, split = work - tile * p.splits;
  tile_coords(tile, p.num_m, p.num_n, p.group_m, t.m_blk, t.n_blk);
  t.m0 = t.m_blk * BM;
  t.n0 = t.n_blk * BNE;
  t.kb0 = split * p.kb_per_split;
  t.kb1 = min((p.K + KB - 1) / KB, t.kb0 + p.kb_per_split);
  return t;
}

// kSwiGLUBwd: ring entries that carry a tile's gate / up values, one per 64-column round of the tile's d(act) columns
// n0.. below I (I % 64 == 0: a round is wholly inside I or wholly beyond it).  The producer and the consumers both count
// with this function: a disagreement would desynchronise the ring's phases.
template <int BNE>
__device__ __forceinline__ int swiglu_bwd_rounds(const Params& p, int n0) {
  return min(BNE / 64, (p.I - n0) / 64);
}

template <int EPI, bool A_MN, bool B_MN, int ELEM>
__device__ __forceinline__ void mma_and_epilogue(const Params& p, const CUtensorMap* tmap_c, const CUtensorMap* tmap_c2,
                                                 uint8_t* smem_a, uint8_t* smem_b, uint8_t* smem_c, uint64_t* full_bar,
                                                 uint64_t* empty_bar, int cw, const Tile& tl, int& stage, uint32_t& phase);

// Output maps (tmap_c, tmap_c2): C (gu for kSwiGLU and kSwiGLUBwd, which also loads from it; fp32 dW for kWgradAcc) and
// act (kSwiGLU); see launch().
template <int EPI, bool A_MN, bool B_MN, int ELEM = 0>
__global__ void __launch_bounds__(THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a1,
            const __grid_constant__ CUtensorMap tmap_a2, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_c2, Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_BYTES;
  uint8_t* smem_c = smem_b + STAGES * B_BYTES;   // output staging, STG_BYTES per MMA warpgroup
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_c + 2 * STG_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  pdl_launch_dependents();
  static_assert(ELEM == 0 || (!A_MN && !B_MN), "FP8 wgmma takes K-major operands only");
  constexpr int KB = ELEM ? BK8 : BK;            // elements per k-block
  constexpr int BNE = ELEM ? BN / 2 : BN;        // tile columns
  constexpr bool TMA_OUT =
      EPI == kStore || EPI == kRoPE || EPI == kSwiGLU || EPI == kSwiGLUBwd || EPI == kLCEFwd || EPI == kWgradAcc;
  const int wg = threadIdx.x >> 7;
  const int work_total = p.num_m * p.num_n * p.splits * p.batch;
  const int work_first = blockIdx.x, work_step = gridDim.x;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if constexpr (TMA_OUT) tma_prefetch_desc(&tmap_c);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int work = work_first; work < work_total; work += work_step) {
        const Tile t = tile_of<ELEM>(p, work);
        // which A tensor this tile reads (A_MN: the split is along M, so it is fixed per tile)
        const CUtensorMap* ta_m = &tmap_a;
        int am0 = t.m0;
        int bk0 = 0, bn0 = t.n0;                // kAxpby: this problem's first B row (MN-major: along K; K-major: along N)
        if constexpr (EPI == kAxpby) {
          am0 += t.b * p.a_rows;
          if constexpr (B_MN) bk0 = t.b * p.b_rows;
          else bn0 += t.b * p.b_rows;
        }
        if constexpr (A_MN) {
          if (p.ks1 && t.m_blk >= p.ks2) { ta_m = &tmap_a2; am0 = t.m0 - p.ks2 * BM; }
          else if (p.ks1 && t.m_blk >= p.ks1) { ta_m = &tmap_a1; am0 = t.m0 - p.ks1 * BM; }
        }
        for (int kb = t.kb0; kb < t.kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], A_BYTES + BNE * 128);
          uint8_t* sa = smem_a + stage * A_BYTES;
          uint8_t* sb = smem_b + stage * B_BYTES;
          if constexpr (A_MN) {     // [K rows, M cols]: two 64(m) x 64(k) boxes
            tma_load_2d(sa, ta_m, &full_bar[stage], am0, kb * BK);
            tma_load_2d(sa + BOX_BYTES, ta_m, &full_bar[stage], am0 + 64, kb * BK);
          } else {
            if (p.ks1 == 0 || kb < p.ks1) tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * KB, am0);
            else if (kb < p.ks2) tma_load_2d(sa, &tmap_a1, &full_bar[stage], (kb - p.ks1) * BK, t.m0);
            else tma_load_2d(sa, &tmap_a2, &full_bar[stage], (kb - p.ks2) * BK, t.m0);
          }
          if constexpr (B_MN) {     // [K rows, N cols]: four 64(n) x 64(k) boxes
#pragma unroll
            for (int j = 0; j < 4; ++j) tma_load_2d(sb + j * BOX_BYTES, &tmap_b, &full_bar[stage], t.n0 + 64 * j, bk0 + kb * BK);
          } else if constexpr (EPI == kSwiGLU) {
            const int g0 = t.n_blk * (BNE / 2);
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * KB, g0);
            tma_load_2d(sb + BNE / 2 * 128, &tmap_b, &full_bar[stage], kb * KB, p.I + g0);
          } else {
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * KB, bn0);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if constexpr (EPI == kSwiGLUBwd) {
          // the epilogue's gate / up values, 64 columns per entry: the gate boxes of rows m0 and m0 + 64 in the A slot, the
          // up boxes in the B slot (rows beyond M arrive as zeros and count towards the transaction bytes)
          const int rounds = swiglu_bwd_rounds<BNE>(p, t.n0);
          for (int c = 0; c < rounds; ++c) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], 4 * OUT_BOX);
            uint8_t* sa = smem_a + stage * A_BYTES;
            uint8_t* sb = smem_b + stage * B_BYTES;
            const int col = t.n0 + 64 * c;
            tma_load_2d(sa, &tmap_c, &full_bar[stage], col, t.m0);
            tma_load_2d(sa + OUT_BOX, &tmap_c, &full_bar[stage], col, t.m0 + 64);
            tma_load_2d(sb, &tmap_c, &full_bar[stage], p.I + col, t.m0);
            tma_load_2d(sb + OUT_BOX, &tmap_c, &full_bar[stage], p.I + col, t.m0 + 64);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    reg_alloc<232>();
    const int cw = wg - 1;                       // this warpgroup's 64 rows of each tile
    int stage = 0;
    uint32_t phase = 0;
    for (int work = work_first; work < work_total; work += work_step) {
      const Tile t = tile_of<ELEM>(p, work);
      mma_and_epilogue<EPI, A_MN, B_MN, ELEM>(p, &tmap_c, &tmap_c2, smem_a, smem_b, smem_c, full_bar, empty_bar, cw, t, stage,
                                              phase);
    }
    if constexpr (TMA_OUT) {
      if ((threadIdx.x & 127) == 0) bulk_wait<0>();   // the last stores have read the staging and reached memory
    }
  }
}

// ---------------------------------------------------------------------------------------- output staging (TMA epilogues)
// A box is 64 rows x 128 bytes, 1024-byte aligned, in the 128-byte swizzle: the 16-byte chunk j of row r is stored at
// chunk j ^ (r % 8).  In the accumulator fragment a warp's lanes hold rows lane / 4 (+ 8) and 4-byte column pairs
// lane % 4 of each 8-column group, so the eight rows of one bf16 store land in eight different chunks: no bank conflicts.
// `at` is the address of this thread's first element in chunk 0 of its row r0 (box + r0 * 128 + byte offset in the chunk,
// XOR (r0 % 8) << 4): chunk j of rows r0 and r0 + 8 is then at (at ^ j << 4) and 1024 bytes further.
__device__ __forceinline__ uint32_t stage_addr(uint32_t box, int r0, int byte_in_chunk) {
  return (box + r0 * 128 + byte_in_chunk) ^ ((r0 & 7) << 4);
}
// bf16: the 8-column groups i0 .. i0+7 of v (fragment layout) become one 64 x 64 box; `at` = stage_addr(box, r0, 2 * cq)
template <int N>
__device__ __forceinline__ void stage_bf16(uint32_t at, const float (&v)[N], int i0) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      sts_b32((at ^ (j << 4)) + 1024 * h, f2_to_bf2(v[4 * (i0 + j) + 2 * h], v[4 * (i0 + j) + 2 * h + 1]));
}
// fp32: the 8-column groups i0 .. i0+3 of v become one 64 x 32 box: columns 8j + cq, 8j + cq + 1 are 8 bytes of chunk
// 2j + cq / 4; `at` = stage_addr(box, r0, 4 * (cq & 2))
__device__ __forceinline__ void stage_f32(uint32_t at, const float (&v)[128], int i0, int cq) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      sts_f2((at ^ ((2 * j + cq / 4) << 4)) + 1024 * h, v[4 * (i0 + j) + 2 * h], v[4 * (i0 + j) + 2 * h + 1]);
}
// Round of the staging protocol of one MMA warpgroup (named barrier 1 + cw): the leader's earlier stores have finished
// reading the staging before anyone writes it; the writes are visible to the async proxy before the leader stores them.
__device__ __forceinline__ void staging_acquire(int cw, bool leader) {
  if (leader) bulk_wait_read<0>();
  named_bar_sync(1 + cw, 128);
}
__device__ __forceinline__ void staging_publish(int cw) {
  fence_proxy_async_smem();
  named_bar_sync(1 + cw, 128);
}

template <int EPI, bool A_MN, bool B_MN, int ELEM>
__device__ __forceinline__ void mma_and_epilogue(const Params& p, const CUtensorMap* tmap_c, const CUtensorMap* tmap_c2,
                                                 uint8_t* smem_a, uint8_t* smem_b, uint8_t* smem_c, uint64_t* full_bar,
                                                 uint64_t* empty_bar, int cw, const Tile& tl, int& stage, uint32_t& phase) {
  constexpr int NI = ELEM ? 16 : 32;             // 8-column groups of the tile: acc[4*i + 2*h + e], i < NI
  constexpr int BNE = 8 * NI;
  const int m0 = tl.m0, n0 = tl.n0, n_blk = tl.n_blk, kb0 = tl.kb0, kb1 = tl.kb1;
  float acc[128];
  if constexpr (ELEM != 0) {
    // FP8: per k-block 4 x k32 into `part` (same fragment layout as acc[0..63]), then acc += part in fp32 (promotion)
    float part[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.f;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint64_t adesc = make_smem_desc_sw128(smem_u32(smem_a + stage * A_BYTES) + cw * 64 * 128, 16, 1024);
      const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smem_b + stage * B_BYTES), 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK8 / 32; ++k)         // 32 fp8 = 32 bytes further along the swizzle row (+2 descriptor units)
        wgmma_m64n128k32_f8<ELEM>(part, adesc + 2 * k, bdesc + 2 * k, k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);     // the k-block has retired: release the stage
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] += part[j];
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    const float dq = *p.inv_a * *p.inv_b;
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] *= dq;
  } else {
    auto release = [&](int s) {                  // hand a stage back to the producer
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[s]);
    };
    // scale_d = 0 on the tile's first k-block discards acc, but the wgmma operands read it: zeroing it here ends the
    // previous tile's values (which would otherwise stay live through its epilogue and spill)
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0.f;
    int prev_stage = stage;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_base = smem_u32(smem_a + stage * A_BYTES) + (A_MN ? cw * BOX_BYTES : cw * 64 * 128);
      const uint32_t b_base = smem_u32(smem_b + stage * B_BYTES);
      const uint64_t adesc = A_MN ? make_smem_desc_sw128(a_base, BOX_BYTES, 1024) : make_smem_desc_sw128(a_base, 16, 1024);
      const uint64_t bdesc = B_MN ? make_smem_desc_sw128(b_base, BOX_BYTES, 1024) : make_smem_desc_sw128(b_base, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        // K-major: 16 bf16 = 32 bytes further along the 128-byte swizzle row (+2 descriptor units);
        // MN-major: 16 rows of 128 B further (+128 units)
        wgmma_m64n256k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc + (A_MN ? 128 : 2) * k, bdesc + (B_MN ? 128 : 2) * k,
                                                     (kb > kb0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();                           // the previous k-block's MMAs have retired: release its stage
      if (kb > kb0) release(prev_stage);
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (kb1 > kb0) release(prev_stage);          // before the epilogue: the producer refills it for the next tile meanwhile
  }

  // -------------------------------------------------------------------- epilogue from the accumulator registers
  // Fragment of m64n256: acc[4*i + 2*h + e] is row (16*warp + lane/4 + 8*h), column (8*i + 2*(lane%4) + e).
  const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  const int r0 = warp * 16 + (lane >> 2);        // rows r0 and r0 + 8 of this warpgroup's 64
  const int rbase = m0 + cw * 64 + r0;
  const int cq = 2 * (lane & 3);
  // TMA epilogues: this warpgroup's boxes start at row `row0`; two staging boxes s0, s1; thread 0 of the warpgroup stores
  const int row0 = m0 + cw * 64;
  const bool leader = t == 0, rows_ok = row0 < p.M;
  uint8_t* stg0 = smem_c + cw * STG_BYTES;
  uint8_t* stg1 = stg0 + OUT_BOX;
  const uint32_t s0 = stage_addr(smem_u32(stg0), r0, 2 * cq), s1 = s0 + OUT_BOX;   // bf16 boxes
  // the bf16 tile in acc to C columns n0.. (boxes wholly right of N are skipped, the others clipped by the map)
  auto store_tile = [&]() {
#pragma unroll
    for (int c = 0; c < NI / 8; c += 2) {
      staging_acquire(cw, leader);
      stage_bf16(s0, acc, 8 * c);
      stage_bf16(s1, acc, 8 * c + 8);
      staging_publish(cw);
      if (leader && rows_ok) {
        if (n0 + 64 * c < p.N) tma_store_2d(stg0, tmap_c, n0 + 64 * c, row0);
        if (n0 + 64 * c + 64 < p.N) tma_store_2d(stg1, tmap_c, n0 + 64 * c + 64, row0);
        bulk_commit();
      }
    }
  };

  if constexpr (EPI == kStore || EPI == kRoPE) {
    if (EPI == kRoPE && n0 < p.rope_cols) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pos = (rbase + 8 * h) % p.S;   // rows beyond M are computed too (in-range table rows) and clipped
#pragma unroll
        for (int c = 0; c < NI / 8; ++c) {
          if (n0 + c * 64 >= p.rope_cols) continue;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int j = 8 * i + cq + e;
              float& va = acc[4 * (8 * c + i) + 2 * h + e];
              float& vb = acc[4 * (8 * c + i + 4) + 2 * h + e];
              const float a = bf16_round(va), b = bf16_round(vb);   // match the unfused path: rotate the bf16 projection
              const float cs = p.cos_t[(size_t)pos * 32 + j], sn = p.sin_t[(size_t)pos * 32 + j];
              va = a * cs - b * sn;
              vb = b * cs + a * sn;
            }
          }
        }
      }
    }
    store_tile();
  } else if constexpr (EPI == kSwiGLU) {
    // tile columns [0,BNE/2) are gate columns g0.., [BNE/2,BNE) the matching up columns; C = gu [M, 2I] (tmap_c),
    // aux = act [M, I] (tmap_c2).  I % 64 == 0: a 64-column box is either all gate (up) columns or wholly beyond I.
    constexpr int NB = NI / 16;                  // 64-column boxes of gate (of up, of act) per tile
    const int g0 = n_blk * (BNE / 2);
#pragma unroll
    for (int c = 0; c < NB; ++c) {
      staging_acquire(cw, leader);
      stage_bf16(s0, acc, 8 * c);
      stage_bf16(s1, acc, NI / 2 + 8 * c);
      staging_publish(cw);
      if (leader && rows_ok && g0 + 64 * c < p.I) {
        tma_store_2d(stg0, tmap_c, g0 + 64 * c, row0);
        tma_store_2d(stg1, tmap_c, p.I + g0 + 64 * c, row0);
        bulk_commit();
      }
    }
    // the activation, from the bf16 values the backward will see, replaces the gate half of acc
#pragma unroll
    for (int j = 0; j < 2 * NI; ++j) {
      const float g = bf16_round(acc[j]), u = bf16_round(acc[j + 2 * NI]);
      acc[j] = g * fast_sigmoid(g) * u;
    }
#pragma unroll
    for (int c = 0; c < NB; c += 2) {
      staging_acquire(cw, leader);
      stage_bf16(s0, acc, 8 * c);
      if (c + 1 < NB) stage_bf16(s1, acc, 8 * c + 8);
      staging_publish(cw);
      if (leader && rows_ok) {
        if (g0 + 64 * c < p.I) tma_store_2d(stg0, tmap_c2, g0 + 64 * c, row0);
        if (c + 1 < NB && g0 + 64 * c + 64 < p.I) tma_store_2d(stg1, tmap_c2, g0 + 64 * c + 64, row0);
        bulk_commit();
      }
    }
  } else if constexpr (EPI == kSwiGLUBwd) {
    // Round c takes the ring entry the producer filled with the gate / up boxes of gate columns n0 + 64c.. (this
    // warpgroup's box at cw * OUT_BOX of the A / B slot, the staging layout) and the accumulator's 8-column groups
    // 8c .. 8c+7; d(gate) / d(up) go to the staging and are stored in place into gu (tmap_c).  The ring entry is released
    // once every thread has passed the staging barrier, so the producer refills it without waiting for the stores.
    const int rounds = swiglu_bwd_rounds<BNE>(p, n0);
#pragma unroll
    for (int c = 0; c < NI / 8; ++c) {
      if (c >= rounds) break;
      mbar_wait(&full_bar[stage], phase);
      staging_acquire(cw, leader);
      const uint32_t g_at = stage_addr(smem_u32(smem_a + stage * A_BYTES) + cw * OUT_BOX, r0, 2 * cq);
      const uint32_t u_at = stage_addr(smem_u32(smem_b + stage * B_BYTES) + cw * OUT_BOX, r0, 2 * cq);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t gv[8], uv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          gv[j] = lds_b32((g_at ^ (j << 4)) + 1024 * h);
          uv[j] = lds_b32((u_at ^ (j << 4)) + 1024 * h);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 g = bf2_to_f2(gv[j]), u = bf2_to_f2(uv[j]);
          float og[2], ou[2];
          const float gg[2] = {g.x, g.y}, uu[2] = {u.x, u.y};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float dj = bf16_round(acc[4 * (8 * c + j) + 2 * h + e]);   // the un-fused path rounds d(act) to bf16 first
            const float sg = fast_sigmoid(gg[e]);
            og[e] = dj * uu[e] * sg * (1.f + gg[e] * (1.f - sg));
            ou[e] = dj * gg[e] * sg;
          }
          sts_b32((s0 ^ (j << 4)) + 1024 * h, f2_to_bf2(og[0], og[1]));
          sts_b32((s1 ^ (j << 4)) + 1024 * h, f2_to_bf2(ou[0], ou[1]));
        }
      }
      staging_publish(cw);
      if (leader) {
        mbar_arrive(&empty_bar[stage]);
        if (rows_ok) {
          tma_store_2d(stg0, tmap_c, n0 + 64 * c, row0);
          tma_store_2d(stg1, tmap_c, p.I + n0 + 64 * c, row0);
          bulk_commit();
        }
      }
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
  } else if constexpr (EPI == kLCEFwd) {
    static_assert(ELEM == 0, "bf16 only");
    constexpr float L2E = 1.4426950408889634f;
    float shift[2], psum[2] = {0.f, 0.f}, psq[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) shift[h] = rbase + 8 * h < p.M ? p.row_shift[rbase + 8 * h] * L2E : 0.f;
    // 128 columns (two boxes) at a time: e replaces the logits in acc and is stored right away (training)
#pragma unroll
    for (int c = 0; c < 4; c += 2) {
#pragma unroll
      for (int i = 8 * c; i < 8 * c + 16; ++i) {
        const int col = n0 + 8 * i + cq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& v = acc[4 * i + 2 * h + e];
            const bool ok = col + e < p.N;
            // clamp at 2^100: a row whose label is > (100 + 58) ln 2 = 109.5 nats below its best logit saturates here
            // instead of overflowing the fp32 row sum
            float x;
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(x) : "f"(fminf(fmaf(v, L2E, -shift[h]), 100.f)));
            psq[h] += ok ? v * v : 0.f;
            v = ok ? x : 0.f;
            psum[h] += v;
          }
        }
      }
      if (p.store) {
        staging_acquire(cw, leader);
        stage_bf16(s0, acc, 8 * c);
        stage_bf16(s1, acc, 8 * c + 8);
        staging_publish(cw);
        if (leader && rows_ok) {
          if (n0 + 64 * c < p.N) tma_store_2d(stg0, tmap_c, n0 + 64 * c, row0);
          if (n0 + 64 * c + 64 < p.N) tma_store_2d(stg1, tmap_c, n0 + 64 * c + 64, row0);
          bulk_commit();
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rbase + 8 * h;
      float ps = psum[h], pq = psq[h];
      ps += __shfl_xor_sync(0xffffffffu, ps, 1);
      ps += __shfl_xor_sync(0xffffffffu, ps, 2);
      pq += __shfl_xor_sync(0xffffffffu, pq, 1);
      pq += __shfl_xor_sync(0xffffffffu, pq, 2);
      if (row < p.M && (lane & 3) == 0) {
        p.partials[(size_t)n_blk * p.M + row] = ps;
        if (p.want_sumsq) p.partials[((size_t)p.num_n + n_blk) * p.M + row] = pq;
      }
    }
  } else if constexpr (EPI == kLCEdX) {
    __nv_bfloat16* C = reinterpret_cast<__nv_bfloat16*>(p.C);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rbase + 8 * h;
      if (row >= p.M) continue;
      const float rs = p.rowscale[row];
      const long long y = p.labels[row];
      const float g = y >= 0 ? *p.gscale : 0.f;
      const __nv_bfloat16* wl = p.wlab + (size_t)(y >= 0 ? y : 0) * p.ldwlab;
      __nv_bfloat16* crow = C + (size_t)row * p.ldc;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = n0 + 8 * i + cq;
        if (col >= p.N) continue;                // N % 64 == 0
        const float2 w = y >= 0 ? ld_bf2(wl + col) : make_float2(0.f, 0.f);
        st_bf2(crow + col, fmaf(rs, acc[4 * i + 2 * h], -g * w.x), fmaf(rs, acc[4 * i + 2 * h + 1], -g * w.y));
      }
    }
  } else if constexpr (EPI == kLCEScore) {
    constexpr float L2E = 1.4426950408889634f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rbase + 8 * h;
      const bool row_ok = row < p.M;
      const long long y = row_ok ? p.labels[row] : -1;
      // columns relative to this thread's first one (n0 + cq): the compares below are against constants
      const int lim = p.N - n0 - cq;
      const long long yr = y - n0 - cq;
      const int lab = (y >= 0 && yr >= 0 && yr < BN) ? (int)yr : -1;
      // this thread's 64 columns of the row, in increasing order: the maximum (strict > keeps the lowest column) ...
      float m = -INFINITY, zl = 0.f;
      int idx = INT_MAX;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = acc[4 * i + 2 * h + e];
          if (8 * i + e < lim && v > m) { m = v; idx = 8 * i + e; }
          if (8 * i + e == lab) zl = v;
        }
      }
      if (idx != INT_MAX) idx += n0 + cq;
      // ... then the sum of exp(z - m) with every exponent <= 0
      const float mb = m * L2E;
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float x;
          asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(x) : "f"(fmaf(acc[4 * i + 2 * h + e], L2E, -mb)));
          s += 8 * i + e < lim ? x : 0.f;
        }
      }
      // merge (max, column, sum) over the quad that shares the row
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, m, off), so = __shfl_xor_sync(0xffffffffu, s, off);
        const int io = __shfl_xor_sync(0xffffffffu, idx, off);
        const float mn = fmaxf(m, mo);
        if (mn != -INFINITY) {
          float a, b;
          asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(a) : "f"((m - mn) * L2E));
          asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(b) : "f"((mo - mn) * L2E));
          s = s * a + so * b;
        }
        idx = (mo > m || (mo == m && io < idx)) ? io : idx;
        m = mn;
      }
      if (row_ok && (lane & 3) == 0) {
        const size_t o = (size_t)n_blk * p.M + row;
        p.sc_max[o] = m;
        p.sc_sum[o] = s;
        p.sc_idx[o] = idx;
      }
      if (row_ok && lab >= 0 && (lab & 6) == 0) p.sc_zlab[row] = zl;     // this thread owns the label column
    }
  } else if constexpr (EPI == kAxpby) {
    const size_t boff = (size_t)tl.b * p.c_bstride;
    __nv_bfloat16* C = reinterpret_cast<__nv_bfloat16*>(p.C) + boff;
    const __nv_bfloat16* D = p.aux ? reinterpret_cast<const __nv_bfloat16*>(p.aux) + boff : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rbase + 8 * h;
      if (row >= p.M) continue;
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        const int col = n0 + 8 * i + cq;
        if (col >= p.N) continue;                // N % 64 == 0
        float v0 = p.alpha * acc[4 * i + 2 * h], v1 = p.alpha * acc[4 * i + 2 * h + 1];
        if (D) {
          const float2 d = ld_bf2(D + (size_t)row * p.ldc + col);
          v0 = fmaf(p.beta, d.x, v0);
          v1 = fmaf(p.beta, d.y, v1);
        }
        st_bf2(C + (size_t)row * p.ldc + col, v0, v1);
      }
    }
  } else if constexpr (EPI == kWgradAcc) {
    // fp32 reduce-add into dW (tmap_c) in 64 x 32 boxes: the split-K items of a tile and later micro-batches add into it
    const uint32_t f0 = stage_addr(smem_u32(stg0), r0, 4 * (cq & 2));
#pragma unroll
    for (int c = 0; c < NI / 4; c += 2) {
      staging_acquire(cw, leader);
      stage_f32(f0, acc, 4 * c, cq);
      stage_f32(f0 + OUT_BOX, acc, 4 * c + 4, cq);
      staging_publish(cw);
      if (leader && rows_ok) {
        if (n0 + 32 * c < p.N) tma_reduce_add_2d(stg0, tmap_c, n0 + 32 * c, row0);
        if (n0 + 32 * c + 32 < p.N) tma_reduce_add_2d(stg1, tmap_c, n0 + 32 * c + 32, row0);
        bulk_commit();
      }
    }
  }
}

// What launch() needs besides Params: the operands its tensor maps are built from (the kernel sees only the maps).  A
// three-piece A operand [A | A1 | A2] is read in place, split along K (A_MN = false) or along M (A_MN = true); K0, K1, K2
// are the extents of the pieces along that dimension, K0 == 0: A is one tensor.
struct Operands {
  const void* A = nullptr; long long lda = 0;
  const void* B = nullptr; long long ldb = 0;
  const void* A1 = nullptr; long long lda1 = 0;
  const void* A2 = nullptr; long long lda2 = 0;
  int K0 = 0, K1 = 0, K2 = 0;
};

// The caller sets the fields of p that its epilogue reads (at least M, N, K; strides in elements); launch() fills in the
// schedule (num_m, num_n, group_m, splits, kb_per_split, ks1, ks2) and S = 1, batch = 1 when they are left at 0.
template <int EPI, bool A_MN, bool B_MN, int ELEM = 0>
static int launch(const Operands& o, Params p, cudaStream_t st) {
  const int M = p.M, N = p.N, K = p.K, I = p.I;
  if (p.S <= 0) p.S = 1;
  if (p.batch <= 0) p.batch = 1;
  // kAxpby: the tensor maps span the whole stacked batch; problem b starts p.a_rows * b / p.b_rows * b rows in
  const int a_rows_all = EPI == kAxpby ? p.batch * p.a_rows : (A_MN ? K : M);
  const int b_rows_all = EPI == kAxpby ? p.batch * p.b_rows : (B_MN ? K : N);
  constexpr int EB = ELEM ? 1 : 2;               // operand bytes per element
  constexpr int KB = ELEM ? BK8 : BK;
  constexpr int BNE = ELEM ? BN / 2 : BN;        // tile columns
  CUtensorMap ta, ta1, ta2, tb;
  int rc;
  if (ELEM) {          // FP8: K-major A and B, no split
    if ((rc = make_tmap_2d(&ta, o.A, M, K, o.lda, BM, KB, EB))) return rc;
  } else if (A_MN) {          // A given as [K rows, M cols] (possibly three tensors side by side along M)
    if ((rc = make_tmap_2d(&ta, o.A, K, o.K0 ? o.K0 : M, o.lda * 2, 64, 64, 2))) return rc;
  } else {
    if ((rc = make_tmap_2d(&ta, o.A, a_rows_all, o.K0 ? o.K0 : K, o.lda * 2, BM, BK, 2))) return rc;
  }
  ta1 = ta; ta2 = ta;
  if (o.K0) {
    if (A_MN) {
      if (o.K1 && (rc = make_tmap_2d(&ta1, o.A1, K, o.K1, o.lda1 * 2, 64, 64, 2))) return rc;
      if (o.K2 && (rc = make_tmap_2d(&ta2, o.A2, K, o.K2, o.lda2 * 2, 64, 64, 2))) return rc;
    } else {
      if ((rc = make_tmap_2d(&ta1, o.A1, M, o.K1, o.lda1 * 2, BM, BK, 2))) return rc;
      if ((rc = make_tmap_2d(&ta2, o.A2, M, o.K2, o.lda2 * 2, BM, BK, 2))) return rc;
    }
  }
  if (B_MN) {
    if ((rc = make_tmap_2d(&tb, o.B, b_rows_all, N, o.ldb * 2, 64, 64, 2))) return rc;   // [K rows, N cols], 64 x 64 boxes
  } else if (EPI == kSwiGLU) {
    if ((rc = make_tmap_2d(&tb, o.B, 2 * I, K, o.ldb * EB, BNE / 2, KB, EB))) return rc;
  } else {
    if ((rc = make_tmap_2d(&tb, o.B, b_rows_all, K, o.ldb * EB, BNE, KB, EB))) return rc;
  }
  // outputs stored by TMA: 64-row boxes of 128 bytes on the caller's view (base, [rows, cols], row stride), so partial
  // tiles are clipped to it.  TMA needs a 16-byte aligned base: a misaligned output is refused (-1).
  CUtensorMap tc = tb, tc2 = tb;                 // unused maps stay valid copies
  auto out_map = [](CUtensorMap* m, void* base, int rows, int cols, long long ld, int eb) {
    if (reinterpret_cast<uintptr_t>(base) % 16) return -1;
    return make_tmap_2d(m, base, rows, cols, ld * eb, 64, 128 / eb, eb);
  };
  if (EPI == kStore || EPI == kRoPE || (EPI == kLCEFwd && p.store)) {
    if ((rc = out_map(&tc, p.C, M, N, p.ldc, 2))) return rc;
  } else if (EPI == kSwiGLU) {
    if ((rc = out_map(&tc, p.C, M, 2 * I, p.ldc, 2)) || (rc = out_map(&tc2, p.aux, M, I, p.ldaux, 2))) return rc;
  } else if (EPI == kSwiGLUBwd) {
    if ((rc = out_map(&tc, p.C, M, 2 * I, p.ldc, 2))) return rc;      // gu: the epilogue's gate / up loads and its stores
  } else if (EPI == kWgradAcc) {
    if ((rc = out_map(&tc, p.C, M, N, p.ldc, 4))) return rc;
  }
  p.num_m = ceil_div(M, BM);
  p.num_n = (EPI == kSwiGLU) ? ceil_div(I, BNE / 2) : ceil_div(N, BNE);
  p.group_m = EPI == kLCEdX ? 0 : GROUP_M;
  const int split_blk = A_MN ? BM : BK;
  p.ks1 = o.K0 ? o.K0 / split_blk : 0;
  p.ks2 = o.K0 ? (o.K0 + o.K1) / split_blk : 0;
  const int tiles = p.num_m * p.num_n;
  const int kb_total = ceil_div(K, KB);
  p.splits = 1;
  p.kb_per_split = kb_total;
  if (EPI == kWgradAcc) {
    // split-K over the tokens (>= 16 k-blocks per work item), chosen by the time of the busiest persistent CTA: its work
    // items x (k-blocks per item + the item's fixed cost).  The fixed cost is mostly the epilogue, the fp32 reduce-add of
    // a whole tile into dW, and measures as about WGRAD_ITEM_KB k-blocks (split-count sweeps on an H100 SXM at 700 W,
    // Llama-150M and 1B weight-gradient shapes): more, shorter items only pay off when they fill the grid much better.
    constexpr int WGRAD_ITEM_KB = 32;
    int best = 1;
    long long best_cost = LLONG_MAX;
    for (int s = 1; s <= 64 && kb_total / s >= 16; ++s) {
      const int kps = ceil_div(kb_total, s);
      const long long cost = (long long)ceil_div(tiles * ceil_div(kb_total, kps), sm_count()) * (kps + WGRAD_ITEM_KB);
      if (cost < best_cost) { best_cost = cost; best = s; }
    }
    p.kb_per_split = ceil_div(kb_total, best);
    p.splits = ceil_div(kb_total, p.kb_per_split);   // no empty slices
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_kernel<EPI, A_MN, B_MN, ELEM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  // persistent grid: one CTA per SM, or fewer when there are fewer work items
  const int work = p.num_m * p.num_n * p.splits * p.batch;
  const int ctas = work < sm_count() ? work : sm_count();
  launch_pdl(gemm_kernel<EPI, A_MN, B_MN, ELEM>, dim3(ctas), dim3(THREADS), SMEM_BYTES, st, ta, ta1, ta2, tb, tc, tc2, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

}  // namespace gemm

// C[M,N] (bf16, row stride ldc) = A[M,K] (row stride lda) * B[N,K]^T (row stride ldb); strides in elements.
ODB_EXPORT int odb_gemm_bf16_tn(const void* A, const void* B, void* C, int M, int N, int K, long long lda, long long ldb,
                                long long ldc, cudaStream_t st) {
  if (K % 8 || lda % 8 || ldb % 8 || ldc % 8) return -1;
  gemm::Operands o;
  o.A = A; o.lda = lda; o.B = B; o.ldb = ldb;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc;
  return gemm::launch<gemm::kStore, false, false>(o, p, st);
}

// gu[M,2I] = x[M,K] * Wgu[2I,K]^T and act[M,I] = silu(gu[:, :I]) * gu[:, I:]   (I % 64 == 0)
ODB_EXPORT int odb_gemm_swiglu(const void* X, const void* Wgu, void* gu, void* act, int M, int I, int K, cudaStream_t st) {
  if (K % 8 || I % 64) return -1;
  gemm::Operands o;
  o.A = X; o.lda = K; o.B = Wgu; o.ldb = K;
  gemm::Params p{};
  p.M = M; p.N = 2 * I; p.K = K; p.C = gu; p.ldc = 2 * I; p.aux = act; p.ldaux = I; p.I = I;
  return gemm::launch<gemm::kSwiGLU, false, false>(o, p, st);
}

// Backward of the SwiGLU MLP's middle: gu[M,2I] (gate|up, bf16) is replaced IN PLACE by d(gate)|d(up), where
// d(act)[M,I] = dY[M,K] * WdT[I,K]^T is formed in registers only (I % 64 == 0; gu is read and written by TMA, so a base
// that is not 16-byte aligned is refused with -1).
ODB_EXPORT int odb_gemm_swiglu_bwd(const void* dY, const void* WdT, void* gu, int M, int I, int K, long long lda, long long ldb,
                                   cudaStream_t st) {
  if (K % 8 || I % 64 || lda % 8 || ldb % 8) return -1;
  gemm::Operands o;
  o.A = dY; o.lda = lda; o.B = WdT; o.ldb = ldb;
  gemm::Params p{};
  p.M = M; p.N = I; p.K = K; p.C = gu; p.ldc = 2 * I; p.I = I;
  return gemm::launch<gemm::kSwiGLUBwd, false, false>(o, p, st);
}

// qkv[M,N] = x[M,K] * Wqkv[N,K]^T with RoPE applied to the first rope_cols columns (head_dim 64, position = row % S)
ODB_EXPORT int odb_gemm_qkv_rope(const void* X, const void* W, void* qkv, int M, int N, int K, int S, int rope_cols,
                                 const void* cos_t, const void* sin_t, cudaStream_t st) {
  if (K % 8 || N % 64 || rope_cols % 64) return -1;
  gemm::Operands o;
  o.A = X; o.lda = K; o.B = W; o.ldb = K;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K; p.C = qkv; p.ldc = N;
  p.S = S; p.rope_cols = rope_cols; p.cos_t = (const float*)cos_t; p.sin_t = (const float*)sin_t;
  return gemm::launch<gemm::kRoPE, false, false>(o, p, st);
}

// C[M,N] = A[M,K] * B[K,N] with B row-major (the dgrad dX = dY W on the forward [out, in] weight layout)
ODB_EXPORT int odb_gemm_bf16_nn(const void* A, const void* B, void* C, int M, int N, int K, long long lda, long long ldb,
                                long long ldc, cudaStream_t st) {
  if (K % 8 || N % 8 || lda % 8 || ldb % 8 || ldc % 8) return -1;
  gemm::Operands o;
  o.A = A; o.lda = lda; o.B = B; o.ldb = ldb;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc;
  return gemm::launch<gemm::kStore, false, true>(o, p, st);
}

// C[M,N] = [A0 | A1 | A2][M, K0+K1+K2] * W[K0+K1+K2, N] with the three A pieces read in place and W in its forward layout
// (K0, K1, K2 % 64 == 0; dgrad of the fused QKV projection)
ODB_EXPORT int odb_gemm_bf16_nn_a3(const void* A0, const void* A1, const void* A2, long long lda0, long long lda1, long long lda2,
                                   int K0, int K1, int K2, const void* B, void* C, int M, int N, long long ldb, long long ldc,
                                   cudaStream_t st) {
  if (K0 % 64 || K1 % 64 || K2 % 64 || K0 <= 0 || K1 <= 0 || K2 <= 0 || N % 8 || ldb % 8) return -1;
  gemm::Operands o;
  o.A = A0; o.lda = lda0; o.B = B; o.ldb = ldb;
  o.A1 = A1; o.lda1 = lda1; o.A2 = A2; o.lda2 = lda2; o.K0 = K0; o.K1 = K1; o.K2 = K2;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K0 + K1 + K2; p.C = C; p.ldc = ldc;
  return gemm::launch<gemm::kStore, false, true>(o, p, st);
}

// as odb_gemm_swiglu_bwd with the down-projection weight Wd[K, I] in its forward layout (MN-major B operand)
ODB_EXPORT int odb_gemm_swiglu_bwd_nn(const void* dY, const void* Wd, void* gu, int M, int I, int K, long long lda, long long ldb,
                                      cudaStream_t st) {
  if (K % 8 || I % 64 || lda % 8 || ldb % 8) return -1;
  gemm::Operands o;
  o.A = dY; o.lda = lda; o.B = Wd; o.ldb = ldb;
  gemm::Params p{};
  p.M = M; p.N = I; p.K = K; p.C = gu; p.ldc = 2 * I; p.I = I;
  return gemm::launch<gemm::kSwiGLUBwd, false, true>(o, p, st);
}

// ---------------------------------------------------------------------------------------------------- fused linear-cross-entropy
// E[M,V] = exp(X W^T - row_shift) (bf16, only when store) and the partial row sums of E (one plane per 256 vocabulary columns)
ODB_EXPORT int odb_lce_fwd(const void* X, const void* W, void* E, int M, int V, int K, long long ldx, long long ldw, long long lde,
                           const void* row_shift, void* partials, int want_sumsq, int store, cudaStream_t st) {
  if (K % 8 || ldx % 8 || ldw % 8 || (store && (lde % 8 || !E))) return -1;
  gemm::Operands o;
  o.A = X; o.lda = ldx; o.B = W; o.ldb = ldw;
  gemm::Params p{};
  p.M = M; p.N = V; p.K = K; p.C = E; p.ldc = lde;
  p.row_shift = (const float*)row_shift; p.partials = (float*)partials; p.want_sumsq = want_sumsq; p.store = store;
  return gemm::launch<gemm::kLCEFwd, false, false>(o, p, st);
}

ODB_EXPORT int odb_lce_planes(int V) { return (V + gemm::BN - 1) / gemm::BN; }

// dX[M,N] (bf16) = rowscale[M] * (E[M,V] * W[V,N]) - gscale * [label >= 0] * W[label]     (N % 64 == 0)
ODB_EXPORT int odb_lce_dx(const void* E, const void* W, void* dX, int M, int N, int V, long long lde, long long ldw, long long ldd,
                          const void* rowscale, const void* labels, const void* gscale, cudaStream_t st) {
  if (V % 8 || N % 64 || lde % 8 || ldw % 8 || ldd % 8) return -1;
  gemm::Operands o;
  o.A = E; o.lda = lde; o.B = W; o.ldb = ldw;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = V; p.C = dX; p.ldc = ldd;
  p.rowscale = (const float*)rowscale; p.labels = (const long long*)labels; p.gscale = (const float*)gscale;
  p.wlab = (const __nv_bfloat16*)W; p.ldwlab = ldw;
  return gemm::launch<gemm::kLCEdX, false, true>(o, p, st);
}

// Scoring statistics of logits Z = X W^T without writing Z: per row and 256-column plane pl (planes = odb_lce_planes(V))
// pmax[pl][M] = max of the plane, pidx[pl][M] = its lowest column, psum[pl][M] = sum exp(z - pmax), and zlab[M] = z[label]
// (rows with label < 0 leave zlab untouched).  Merged into log-probabilities by odb_lce_score_finalize (lce.cu).
ODB_EXPORT int odb_lce_score(const void* X, const void* W, int M, int V, int K, long long ldx, long long ldw, const void* labels,
                             void* pmax, void* psum, void* pidx, void* zlab, cudaStream_t st) {
  if (K % 8 || ldx % 8 || ldw % 8) return -1;
  gemm::Operands o;
  o.A = X; o.lda = ldx; o.B = W; o.ldb = ldw;
  gemm::Params p{};
  p.M = M; p.N = V; p.K = K; p.labels = (const long long*)labels;
  p.sc_max = (float*)pmax; p.sc_sum = (float*)psum; p.sc_idx = (int*)pidx; p.sc_zlab = (float*)zlab;
  return gemm::launch<gemm::kLCEScore, false, false>(o, p, st);
}

// ---------------------------------------------------------------------------------------------------- weight gradient
// dW[N_out, K_out] (fp32, row stride ldw) += [dY0 | dY1 | dY2][T, N_out]^T * X[T, K_out]
// Both operands are MN-major for the tensor core (the reduction index t is the slow memory dimension).  n1, n2: column
// counts of the 2nd / 3rd dY tensors (0 = unused; then dY0 has all N_out columns); when used, every piece must be a
// multiple of 256 columns.  T, N_out, K_out need no alignment beyond 8 elements (TMA clips).
ODB_EXPORT int odb_wgrad_bf16(const void* dY0, const void* dY1, const void* dY2, long long ld0, long long ld1, long long ld2,
                              int n0, int n1, int n2, const void* X, long long ldx, void* dW, long long ldw, int T, int K_out,
                              cudaStream_t st) {
  const int N_out = n0 + n1 + n2;
  if ((n1 || n2) && (n0 % 256 || n1 % 256 || n2 % 256)) return -1;
  if (ld0 % 8 || ldx % 8 || ldw % 4 || T <= 0) return -1;
  gemm::Operands o;
  o.A = dY0; o.lda = ld0; o.B = X; o.ldb = ldx;
  if (n1 || n2) { o.A1 = dY1; o.A2 = dY2; o.lda1 = ld1; o.lda2 = ld2; o.K0 = n0; o.K1 = n1; o.K2 = n2; }
  gemm::Params p{};
  p.M = N_out; p.N = K_out; p.K = T; p.C = dW; p.ldc = ldw;
  return gemm::launch<gemm::kWgradAcc, true, true>(o, p, st);
}

// ---------------------------------------------------------------------------------------------------- FP8 (e4m3 / e5m2)
// Operands are FP8 bytes, K-major (row strides in elements = bytes, multiples of 16); inv_a / inv_b are device fp32 scalars
// (1 / scale of each operand, written by odb_fp8_cast) that the epilogue multiplies into the fp32 accumulator.
// a_e5m2 = 0: A is e4m3 (forward), 1: A is e5m2 (gradients).  B is always e4m3.  Outputs are as for the bf16 exports.
static bool fp8_ok(int K, long long lda, long long ldb) { return K % 16 == 0 && lda % 16 == 0 && ldb % 16 == 0; }

// C[M,N] (bf16) = A[M,K] * B[N,K]^T
ODB_EXPORT int odb_gemm_fp8_tn(const void* A, const void* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
                               int a_e5m2, const void* inv_a, const void* inv_b, cudaStream_t st) {
  if (!fp8_ok(K, lda, ldb) || ldc % 8) return -1;
  gemm::Operands o;
  o.A = A; o.lda = lda; o.B = B; o.ldb = ldb;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc; p.inv_a = (const float*)inv_a; p.inv_b = (const float*)inv_b;
  return a_e5m2 ? gemm::launch<gemm::kStore, false, false, 2>(o, p, st) : gemm::launch<gemm::kStore, false, false, 1>(o, p, st);
}

// as odb_gemm_qkv_rope with e4m3 x[M,K] and Wqkv[N,K]
ODB_EXPORT int odb_gemm_fp8_qkv_rope(const void* X, const void* W, void* qkv, int M, int N, int K, int S, int rope_cols,
                                     const void* cos_t, const void* sin_t, const void* inv_a, const void* inv_b, cudaStream_t st) {
  if (!fp8_ok(K, K, K) || N % 64 || rope_cols % 64) return -1;
  gemm::Operands o;
  o.A = X; o.lda = K; o.B = W; o.ldb = K;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K; p.C = qkv; p.ldc = N;
  p.S = S; p.rope_cols = rope_cols; p.cos_t = (const float*)cos_t; p.sin_t = (const float*)sin_t;
  p.inv_a = (const float*)inv_a; p.inv_b = (const float*)inv_b;
  return gemm::launch<gemm::kRoPE, false, false, 1>(o, p, st);
}

// as odb_gemm_swiglu with e4m3 x[M,K] and Wgu[2I,K]
ODB_EXPORT int odb_gemm_fp8_swiglu(const void* X, const void* Wgu, void* gu, void* act, int M, int I, int K, const void* inv_a,
                                   const void* inv_b, cudaStream_t st) {
  if (!fp8_ok(K, K, K) || I % 64) return -1;
  gemm::Operands o;
  o.A = X; o.lda = K; o.B = Wgu; o.ldb = K;
  gemm::Params p{};
  p.M = M; p.N = 2 * I; p.K = K; p.C = gu; p.ldc = 2 * I; p.aux = act; p.ldaux = I; p.I = I;
  p.inv_a = (const float*)inv_a; p.inv_b = (const float*)inv_b;
  return gemm::launch<gemm::kSwiGLU, false, false, 1>(o, p, st);
}

// as odb_gemm_swiglu_bwd with e5m2 dY[M,K] and e4m3 WdT[I,K] (the transposed down-projection weight)
ODB_EXPORT int odb_gemm_fp8_swiglu_bwd(const void* dY, const void* WdT, void* gu, int M, int I, int K, long long lda, long long ldb,
                                       const void* inv_a, const void* inv_b, cudaStream_t st) {
  if (!fp8_ok(K, lda, ldb) || I % 64) return -1;
  gemm::Operands o;
  o.A = dY; o.lda = lda; o.B = WdT; o.ldb = ldb;
  gemm::Params p{};
  p.M = M; p.N = I; p.K = K; p.C = gu; p.ldc = 2 * I; p.I = I;
  p.inv_a = (const float*)inv_a; p.inv_b = (const float*)inv_b;
  return gemm::launch<gemm::kSwiGLUBwd, false, false, 2>(o, p, st);
}

// dW[N_out, K_out] (fp32, row stride ldw) += dYt[N_out, T] * Xt[K_out, T]^T with e5m2 dYt and e4m3 Xt: the transposed
// copies written by odb_fp8_cast, so that the reduction over tokens is the K-major dimension.  Split-K over T as for bf16.
ODB_EXPORT int odb_wgrad_fp8(const void* dYt, const void* Xt, void* dW, int N_out, int K_out, int T, long long ld_dyt, long long ld_xt,
                             long long ldw, const void* inv_a, const void* inv_b, cudaStream_t st) {
  if (!fp8_ok(T, ld_dyt, ld_xt) || ldw % 4 || T <= 0) return -1;
  gemm::Operands o;
  o.A = dYt; o.lda = ld_dyt; o.B = Xt; o.ldb = ld_xt;
  gemm::Params p{};
  p.M = N_out; p.N = K_out; p.K = T; p.C = dW; p.ldc = ldw; p.inv_a = (const float*)inv_a; p.inv_b = (const float*)inv_b;
  return gemm::launch<gemm::kWgradAcc, false, false, 2>(o, p, st);
}

// Batched C[b] = alpha * A[b] * B[b]^T + beta * D[b] over `batch` problems stacked along rows: A[b] is [M, K] at row b * M
// of A, B[b] is [N, K] at row b * N of B, C[b] and D[b] are [M, N] with row stride ldc, consecutive problems M * ldc
// elements apart.  D may be null (beta unused); it may be A or B, never C.  M, N, K % 64 == 0.
ODB_EXPORT int odb_gemm_batched_axpby_tn(const void* A, const void* B, void* C, const void* D, int batch, int M, int N, int K,
                                         long long ldc, float alpha, float beta, cudaStream_t st) {
  if (batch <= 0 || M % 64 || N % 64 || K % 64 || ldc % 8 || ldc < N) return -1;
  gemm::Operands o;
  o.A = A; o.lda = K; o.B = B; o.ldb = K;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc; p.aux = const_cast<void*>(D); p.ldaux = ldc;
  p.batch = batch; p.a_rows = M; p.b_rows = N; p.c_bstride = (long long)M * ldc; p.alpha = alpha; p.beta = beta;
  return gemm::launch<gemm::kAxpby, false, false>(o, p, st);
}

// as odb_gemm_batched_axpby_tn with B[b] = [K, N] row-major at row b * K of B (MN-major operand): C[b] = alpha A[b] B[b] + beta D[b]
ODB_EXPORT int odb_gemm_batched_axpby_nn(const void* A, const void* B, void* C, const void* D, int batch, int M, int N, int K,
                                         long long ldc, float alpha, float beta, cudaStream_t st) {
  if (batch <= 0 || M % 64 || N % 64 || K % 64 || ldc % 8 || ldc < N) return -1;
  gemm::Operands o;
  o.A = A; o.lda = K; o.B = B; o.ldb = N;
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc; p.aux = const_cast<void*>(D); p.ldaux = ldc;
  p.batch = batch; p.a_rows = M; p.b_rows = K; p.c_bstride = (long long)M * ldc; p.alpha = alpha; p.beta = beta;
  return gemm::launch<gemm::kAxpby, false, true>(o, p, st);
}

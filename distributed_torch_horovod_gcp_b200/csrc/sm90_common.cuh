// Shared sm_90a device helpers: mbarrier / TMA / wgmma PTX wrappers, GMMA shared-memory descriptors, the
// fused register->smem->TMA-store epilogue and the persistent kernel body of the GEMM (gemm_sm90.cu) and
// the implicit-GEMM convolution (conv_sm90.cu), and their host side (tensor maps, launches, split-K
// workspaces), partly shared with the attention kernels (attn_sm90.cu).
//
// wgmma keeps its accumulator in the registers of the issuing warpgroup, in a fragment layout (each warp
// holds 16 rows, each thread two rows x pairs of columns).  The epilogue works on that fragment: each
// thread applies it to its own elements and writes bf16 pairs into a 128B-swizzled staging copy of the
// whole tile (or, in the add / store modes, pairs straight to global memory).  After a barrier, each warp
// bulk-stores one 32-row x 64-column box of it and walks its columns for the BatchNorm statistics.  No fp32 copy of the tile goes
// through shared memory, so the space goes to the operand ring instead.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "philox.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 bf16 = 128 bytes = one 128B swizzle atom
constexpr int WGMMA_K = 16;        // K of one wgmma (bf16)
constexpr int NUM_THREADS = 384;     // warpgroup 0: TMA producer; warpgroups 1-2: wgmma + epilogue (8 warps)
constexpr int SMEM_LIMIT = 232448;   // 227 KB of dynamic shared memory per block on sm_90

struct GemmParams {
  int M, N;
  int ldc;                 // elements
  int num_m_blocks, num_n_blocks, num_k_blocks;
  int splits;              // split-K factor (>=1)
  int act;                 // 0 none, 1 relu, 2 gelu(erf), 3 *gelu'(aux), 4 *(aux>0)  [aux = residual ptr]
  int out_mode;            // 0: bf16 via swizzled smem + TMA bulk store, 1: add into C, 2: store into C (1/2
                           // with split-K: see splitk_finish_tile)
  int c_bf16;              // out_mode 1/2: C is bf16 (else fp32)
  void* C;
  const void* bias;        // bf16 [N] or nullptr
  const void* bias_f32;    // fp32 [N] or nullptr
  const void* residual;    // bf16 [M, ldc] or nullptr (added after act; or `aux` for act 3/4)
  void* preact;            // optional bf16 [M, ldc]: pre-activation values (saved for backward)
  int n_fastest;           // tile order: consecutive CTAs walk the N blocks of one M block first (A tile is
                           // fetched from HBM once and re-used from L2 while the whole B matrix stays in L2)
  float alpha;
  float res_scale;         // multiplies the residual of the fused epilogue (act 0..2): alpha acc + res_scale residual
  const unsigned char* res_mask;   // optional, with a plain residual (act 0..2): bit j of byte [row][col/8] keeps
                           // residual element (row, 8*(col/8)+j) — the ReLU sign bits of the block output whose
                           // skip-branch gradient the residual is (N % 64 == 0 required)
  float* stats;            // optional fp32 [2][N]: per-column sum | sum of squares of the bf16 OUTPUT (the batch
                           // statistics of the BatchNorm that follows), accumulated by the epilogue
  // split-K (splits > 1, out_mode 1/2): per-launch workspace — one fp32 slice of splitk_slice elements per split,
  // laid out like C, and one arrival counter per output tile (zero on entry); see splitk_finish_tile
  float* splitk_ws;
  int* splitk_count;
  long long splitk_slice;
};

// Shared-memory accumulators for GemmParams::stats, after the barriers: one PRIVATE region per epilogue warp
// (sum[128] | sumsq[128] floats for the <= 128 tile columns the warp drains).  Every address is only ever
// touched by one lane, so accumulation is plain ld/add/st — fp32 atomicAdd on shared memory compiles to a
// CAS loop (ATOMS.CAST.SPIN) and the four lane-quarter warps of a tile hit the same columns.
constexpr int STATS_MAX_N = 2048;
constexpr int STATS_WARP_FLOATS = 256;
constexpr int STATS_SMEM_BYTES = 8 * STATS_WARP_FLOATS * 4;

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // try_wait suspends for a bounded time per attempt; a %globaltimer watchdog (4 s) turns a protocol
  // bug (lost arrive / wrong phase) into a trap ("unspecified launch failure") instead of a GPU hang.
  uint32_t done = 0;
  unsigned long long t0 = 0;
  for (uint32_t tries = 0; !done; ++tries) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (!done && (tries & 1023u) == 1023u) {
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ull) __trap();
    }
  }
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
// 4D tiled loads/stores (NHWC activations as {C, W, H, N} tensors): out-of-bounds box elements — negative
// or past-the-end coordinates, i.e. the convolution's zero padding — are zero-filled on load and skipped
// on store by the TMA unit itself.
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], "
      "[%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2,
                                             int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving reads of the accumulator above the wgmma.wait_group that completes it
template <int R>
__device__ __forceinline__ void wg_fence_operands(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void named_bar(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---- generated: one wrapper per accumulator width (the operand list of wgmma is fixed-size)
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n64(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n128(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}

__device__ __forceinline__ void wgmma_tf32_n32(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(acc));
}


// 64-bit GMMA shared-memory descriptor, 128B swizzle.
//   K-major  : rows of 128 B (64 bf16 of K), 8-row groups 1024 B apart (SBO); LBO unused (=1).
//   MN-major : [k rows][64 mn elements] atoms of 128 B rows; 8-row k-groups SBO=1024 B apart,
//              64-element mn chunks LBO bytes apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                              uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;   // layout type: SWIZZLE_128B
  return d;
}

// One elected lane of a converged warp (PTX elect.sync).  Code guarded by it is known to the compiler
// to run in a single thread, so TMA operands stay in uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// Descriptor without the start address (bits 0..13): OR / add `(smem_addr >> 4)` to place it; advancing
// along K or by whole rows is then a 64-bit add of `(bytes >> 4)` — no rebuild in the MMA issue loop.
__device__ __forceinline__ uint64_t make_desc_base(uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return make_desc(0, lbo_bytes, sbo_bytes);
}
__device__ __forceinline__ uint64_t desc_addr(uint32_t smem_addr) { return (uint64_t)((smem_addr & 0x3FFFF) >> 4); }

template <int BN, bool TA, bool TB>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  static_assert(BN == 64 || BN == 128, "wgmma width");
  if constexpr (BN == 64) wgmma_bf16_n64<TA ? 1 : 0, TB ? 1 : 0>(d, a, b, acc);
  else wgmma_bf16_n128<TA ? 1 : 0, TB ? 1 : 0>(d, a, b, acc);
}

// Consumer side of the TMA operand ring: this warpgroup's 64 rows (wg 0/1) of a 128 x BN tile, summed over
// nkb 64-deep K blocks into the register fragment d.  A stage is released (one arrival per warpgroup on
// its empty barrier, which counts 2) as soon as the wgmmas of the NEXT stage are issued and the ones
// reading it have retired, so one stage of MMAs is always in flight.
// Operand tiles: A K-major [128 rows][64 k] or MN-major 2 x [64 k][64 m] (either way rows 64..127 start
// 8 KB in), B K-major [BN rows][64 k] or MN-major BN/64 x [64 k][64 n]; all 128B-swizzled.
template <int BN, bool A_MN, bool B_MN, int STAGES, int A_BYTES, int B_BYTES>
__device__ __forceinline__ void wg_mainloop(float* d, uint32_t sa, uint32_t sb, uint64_t* full_bar, uint64_t* empty_bar,
                                            int& stage, uint32_t& phase, int nkb, int wg) {
  constexpr uint32_t KSTEP_A = A_MN ? ((WGMMA_K * 128) >> 4) : ((WGMMA_K * 2) >> 4);
  constexpr uint32_t KSTEP_B = B_MN ? ((WGMMA_K * 128) >> 4) : ((WGMMA_K * 2) >> 4);
  const uint64_t a0 = (A_MN ? make_desc_base(BLOCK_K * 128, 1024) : make_desc_base(16, 1024)) +
                      desc_addr(sa + (uint32_t)wg * 8192u);
  const uint64_t b0 = (B_MN ? make_desc_base(BLOCK_K * 128, 1024) : make_desc_base(16, 1024)) + desc_addr(sb);
  const bool leader = (threadIdx.x & 127) == 0;
  int prev = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint64_t da = a0 + (uint64_t)(stage * (A_BYTES >> 4));
    const uint64_t db = b0 + (uint64_t)(stage * (B_BYTES >> 4));
    wg_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
      wgmma_bf16<BN, A_MN, B_MN>(d, da + k * KSTEP_A, db + k * KSTEP_B, (kb | k) ? 1u : 0u);
    wg_commit();
    wg_wait<1>();
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wg_wait<0>();
  wg_fence_operands<BN / 2>(d);
  if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
}

// erf via Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7, far below bf16 resolution): 1 rcp + 1 ex2 + 6 fma
// instead of the ~40-instruction erff — the epilogue, not the MMA, bounds the GELU GEMMs.
__device__ __forceinline__ float fast_erf(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float y = 1.0f - poly * t * __expf(-ax * ax);
  return copysignf(y, x);
}
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + fast_erf(x * 0.70710678118654752f));
}

__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.0f + fast_erf(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

__device__ __forceinline__ void unpack8(const uint4& x, float* f) {
  const uint32_t wv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    f[2 * t] = __uint_as_float(wv[t] << 16);
    f[2 * t + 1] = __uint_as_float(wv[t] & 0xffff0000u);
  }
}

template <int BN>
struct Cfg {
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BN * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // bf16 staging of one whole output tile: [4 slabs][BN / 64 chunks] boxes of 32 rows x 128 B (128B-swizzled),
  // one bulk store each
  static constexpr int NCH = BN / 64;
  static constexpr int STORE_BYTES = BLOCK_M * BN * 2;
  static constexpr int FIXED_BYTES = STORE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + STATS_SMEM_BYTES;
  // as many operand stages as fit next to the staging tile: BN 64: 8, BN 128: 5 (measured on an H100, a
  // 4-stage cap for BN 64 gained nothing)
  static constexpr int STAGES = (SMEM_LIMIT - FIXED_BYTES) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED_BYTES;
  static_assert(STAGES >= 4, "shared memory");
  static_assert(2 * STAGES * 8 <= 256, "barrier space");
};

// Where the rows of a tile go.  rank4 == 0: rows m_row0.. of the row-major [M, ldc] matrix (2D map).
// rank4 == 1 (convolution): a 32-row slab is the {64 c, sw, sh, sn} sub-box at pixel (w, h, n) of an NHWC
// tensor.
struct StoreAt {
  int rank4, w, h, n;
  // rank4 only (statistics of a convolution output): the slab is an {sw, sh, .} pixel box of which only
  // vw x vh x vn pixels lie inside the image / batch — rows outside are computed from partly valid taps
  // (NOT zero) and must not be counted; the TMA store clips them by itself.
  int sw, sh, vw, vh, vn;
};

// explicit shared-space accesses (a generic pointer into shared memory costs 64-bit address arithmetic
// and the generic LD/ST path: measured, the epilogue is issue-bound)
__device__ __forceinline__ void epi_sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void epi_sts32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t epi_lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
// prmt.b32 in its default mode: selector nibble bit 3 = replicate the selected byte's sign bit
__device__ __forceinline__ uint32_t prmt_sign(uint32_t a, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(0u), "r"(sel));
  return d;
}
__device__ __forceinline__ uint32_t cvt_bf16x2(float lo, float hi) {
  uint32_t o;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o) : "f"(hi), "f"(lo));
  return o;
}
// (+0) + v with subnormals flushed: what red.add.f32 (RED.ADD.F32.FTZ) leaves in a zeroed fp32 buffer, so a
// -0 becomes +0.  Written as PTX so that the add is neither folded nor done without FTZ.
__device__ __forceinline__ float zero_plus_ftz(float v) {
  float o;
  asm("add.ftz.f32 %0, %1, %2;" : "=f"(o) : "f"(0.0f), "f"(v));
  return o;
}

// Byte offset of (tile row r, 16-byte column unit u) in the staging tile: box (r / 32, u / 8), row r % 32, and
// unit u % 8 at its 128B-swizzle position (u ^ r) % 8 — the shared-memory image the bulk stores read.
template <int BN>
__device__ __forceinline__ uint32_t stage_off(int r, int u) {
  return (uint32_t)((((r >> 5) * (BN / 64) + (u >> 3)) << 12) + ((r & 31) << 7) + (((u ^ r) & 7) << 4));
}

// Residual of the 16 tile rows r0.. that this warp holds in its fragment (rows m0 + r0.. of the [M, ldc]
// matrix): COALESCED 16-byte loads, zero past M and past N, then staged at the output's place in the staging
// tile (res_stage) so that each thread reads its elements back in fragment layout.
template <int BN>
__device__ __forceinline__ void res_load(const GemmParams& p, uint4* rv, int m0, int r0, int n_idx, int lane) {
  const __nv_bfloat16* rbase = reinterpret_cast<const __nv_bfloat16*>(p.residual);
#pragma unroll
  for (int i = 0; i < BN / 16; ++i) {
    const int e = i * 32 + lane, row = m0 + r0 + e / (BN / 8), col = n_idx + (e % (BN / 8)) * 8;
    rv[i] = (row < p.M && col < p.N) ? *reinterpret_cast<const uint4*>(rbase + (size_t)row * p.ldc + col)
                                     : make_uint4(0, 0, 0, 0);
  }
  if (p.res_mask != nullptr) {
    // ReLU sign bits of the residual (1 byte per 8 channels): bit j -> 16-bit lane j.  Byte k of
    // ((bits * 0x01010101) & 0x08040201) + 0x7f7f7f7f has its MSB set iff bit k is, and PRMT's
    // sign-replicate mode turns that MSB into 0x00 / 0xff bytes.
    uint32_t mbits[BN / 16];
#pragma unroll
    for (int i = 0; i < BN / 16; ++i) {
      const int e = i * 32 + lane, row = m0 + r0 + e / (BN / 8), col = n_idx + (e % (BN / 8)) * 8;
      mbits[i] = (row < p.M && col < p.N) ? (uint32_t)p.res_mask[(size_t)row * (size_t)(p.N >> 3) + (size_t)(col >> 3)]
                                          : 0u;
    }
#pragma unroll
    for (int i = 0; i < BN / 16; ++i) {
      const uint32_t rep = mbits[i] * 0x01010101u;
      const uint32_t lo = (rep & 0x08040201u) + 0x7f7f7f7fu, hi = (rep & 0x80402010u) + 0x7f7f7f7fu;
      rv[i].x &= prmt_sign(lo, 0x9988u);
      rv[i].y &= prmt_sign(lo, 0xbbaau);
      rv[i].z &= prmt_sign(hi, 0x9988u);
      rv[i].w &= prmt_sign(hi, 0xbbaau);
    }
  }
}
template <int BN>
__device__ __forceinline__ void res_stage(const uint4* rv, uint32_t stg, int r0, int lane) {
#pragma unroll
  for (int i = 0; i < BN / 16; ++i) {
    const int e = i * 32 + lane;
    epi_sts128(stg + stage_off<BN>(r0 + e / (BN / 8), e % (BN / 8)), rv[i]);
  }
}

// Epilogue of this thread's part of a finished 128 x BN tile, straight from the wgmma fragment d of
// warpgroup wg — tile rows r and r + 8 (r = 64 wg + 16 warp + lane / 4), columns 8j + 2 (lane % 4) + {0, 1}:
// alpha, bias, pre-activation, activation, residual (times res_scale); then bf16 pairs into the staging tile
// (out_mode 0: the 8 rows of a warp store hit 8 different swizzle positions, so the 4-byte stores are conflict-free), or pairs
// added into C (out_mode 1) or stored (out_mode 2) at column offset c_off, in C's dtype; with split-K, fp32
// pairs stored into the workspace slice of the item's split.  m0: first row of the tile in the [M, ldc]
// matrix.  A residual (out_mode != 1) has been staged at the output's place; every element is read and then
// overwritten by the one thread that owns it.
template <int BN>
__device__ __forceinline__ void epilogue_frag(const GemmParams& p, const float* d, uint32_t stg, int wg, int m0,
                                              int n_idx, int split, long long c_off) {
  const int t = threadIdx.x & 127, lane = t & 31;
  const int r = wg * 64 + (t >> 5) * 16 + (lane >> 2);
  const uint32_t x = (uint32_t)(r & 7);
  const uint32_t sbase = stg + (uint32_t)(((r >> 5) * (BN / 64)) << 12) + (uint32_t)((r & 31) << 7) +
                         (uint32_t)(lane & 3) * 4u;
  // staging address of column pair j of row r + 8h
  auto sa = [&](int j, int h) -> uint32_t {
    return sbase + (uint32_t)(h * 1024 + ((j >> 3) << 12)) + ((((uint32_t)j & 7u) ^ x) << 4);
  };
  const bool plain = p.out_mode == 0 && p.alpha == 1.0f && p.bias == nullptr && p.bias_f32 == nullptr &&
                     p.preact == nullptr && p.act == 0 && p.residual == nullptr;
  const bool res_only = p.out_mode == 0 && p.residual != nullptr && p.preact == nullptr && p.alpha == 1.0f &&
                        p.res_scale == 1.0f && p.bias == nullptr && p.bias_f32 == nullptr && p.act == 0;
  if (plain) {
    // the common case (plain bf16 output, optionally with BN statistics)
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) epi_sts32(sa(j, h), cvt_bf16x2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]));
    return;
  }
  if (res_only) {
    // skip-gradient path of the dgrad GEMMs: bf16(acc + residual)
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t a = epi_lds32(sa(j, h));
        epi_sts32(sa(j, h), cvt_bf16x2(d[4 * j + 2 * h] + __uint_as_float(a << 16),
                                       d[4 * j + 2 * h + 1] + __uint_as_float(a & 0xffff0000u)));
      }
    return;
  }
  const int cq = n_idx + 2 * (lane & 3);
  // out_mode 1/2: C in its dtype, or with split-K the fp32 workspace slice of the item's split
  const size_t esz = (p.splits > 1 || !p.c_bf16) ? 4 : 2;
  char* const cbase = (p.splits > 1 ? reinterpret_cast<char*>(p.splitk_ws + split * p.splitk_slice)
                                    : reinterpret_cast<char*>(p.C)) + c_off * esz;
  // bias, pre-activation, activation, residual (out_mode 0 / 2; the add mode ignores them)
  const bool fused = p.out_mode != 1 && (p.bias != nullptr || p.bias_f32 != nullptr || p.preact != nullptr ||
                                         p.act != 0 || p.residual != nullptr);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = cq + 8 * j;
    const bool col_ok = col < p.N;                    // N % 8 == 0: col + 1 < N too
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + r + 8 * h;
      float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
      if (p.alpha != 1.0f) {
        v0 *= p.alpha;
        v1 *= p.alpha;
      }
      if (fused) {
        if (p.bias != nullptr) {
          if (col_ok) {
            const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(p.bias) + col;
            v0 += __bfloat162float(b[0]);
            v1 += __bfloat162float(b[1]);
          }
        } else if (p.bias_f32 != nullptr) {
          if (col_ok) {
            const float* b = reinterpret_cast<const float*>(p.bias_f32) + col;
            v0 += b[0];
            v1 += b[1];
          }
        }
        if (p.preact != nullptr && row < p.M && col_ok)
          *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.preact) + (size_t)row * p.ldc + col) =
              cvt_bf16x2(v0, v1);
        if (p.act == 1) {
          v0 = fmaxf(v0, 0.0f);
          v1 = fmaxf(v1, 0.0f);
        } else if (p.act == 2) {
          v0 = gelu_erf(v0);
          v1 = gelu_erf(v1);
        }
        if (p.residual != nullptr) {
          const uint32_t a = epi_lds32(sa(j, h));
          const float a0 = __uint_as_float(a << 16), a1 = __uint_as_float(a & 0xffff0000u);
          if (p.act == 3) {
            v0 *= gelu_erf_grad(a0);
            v1 *= gelu_erf_grad(a1);
          } else if (p.act == 4) {
            v0 = a0 > 0.0f ? v0 : 0.0f;
            v1 = a1 > 0.0f ? v1 : 0.0f;
          } else {  // one rounding: with res_scale == 1 these are the bits of v + a
            v0 = fmaf(p.res_scale, a0, v0);
            v1 = fmaf(p.res_scale, a1, v1);
          }
        }
      }
      if (p.out_mode == 0) {
        epi_sts32(sa(j, h), cvt_bf16x2(v0, v1));
      } else if (row < p.M && col_ok) {
        const size_t e = (size_t)row * p.ldc + col;
        if (p.splits > 1) {
          float* dst = reinterpret_cast<float*>(cbase) + e;
          asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(v0), "f"(v1) : "memory");
        } else {
          // one split: this thread is the only writer of the pair.  (+0) + v first, so that the result is
          // that of accumulating into a zeroed fp32 buffer and then adding it to C
          v0 = zero_plus_ftz(v0);
          v1 = zero_plus_ftz(v1);
          if (p.c_bf16) {
            __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(cbase) + e;
            if (p.out_mode == 1) {
              uint32_t o;
              asm volatile("ld.global.b32 %0, [%1];" : "=r"(o) : "l"(dst) : "memory");
              v0 += __uint_as_float(o << 16);
              v1 += __uint_as_float(o & 0xffff0000u);
            }
            asm volatile("st.global.b32 [%0], %1;" ::"l"(dst), "r"(cvt_bf16x2(v0, v1)) : "memory");
          } else {
            float* dst = reinterpret_cast<float*>(cbase) + e;
            if (p.out_mode == 2)
              asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(v0), "f"(v1) : "memory");
            else
              asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(v0), "f"(v1) : "memory");
          }
        }
      }
    }
  }
}

// Bulk store of slab q (tile rows 32q..32q+31, columns c_begin..c_end-1) of the staged tile, after the tile's
// epilogue barrier, and the batch statistics of the following BatchNorm: column sums of the staged bf16
// values.  Lane l owns columns 2l, 2l+1 of a 64-column chunk and walks the 32 rows of the slab in order
// (one conflict-free 4-byte shared load per row); partials go to the warp's private shared accumulators.
// Rows that are not part of the output are masked: rows of a convolution tile outside the image (they see
// partly valid taps) and GEMM rows past M (zero-filled operands, but the epilogue may still have added a bias
// or an activation of it).
template <int BN>
__device__ __forceinline__ void store_slab(const GemmParams& p, const CUtensorMap* map_c, const uint8_t* stg_ptr,
                                           int q, int lane, int m_row0, int n_idx, int c_begin, int c_end,
                                           const StoreAt at, float* s_stats) {
#pragma unroll 1
  for (int c0 = c_begin; c0 < c_end; c0 += 64) {
    const int col0 = n_idx + c0;
    if (col0 >= p.N) continue;                       // warp-uniform
    const uint8_t* buf = stg_ptr + ((q * (BN / 64) + (c0 >> 6)) << 12);
    if (s_stats != nullptr) {
      float sum_lo = 0.f, sum_hi = 0.f, sq_lo = 0.f, sq_hi = 0.f;
      const uint32_t base = smem_u32(buf) + (uint32_t)((lane & 3) << 2);
      const uint32_t u = (uint32_t)(lane >> 2);
      if (at.rank4 || m_row0 + 32 > p.M) {      // lane r decides for slab row r
        bool ok;
        if (at.rank4) {
          const int rw = lane % at.sw, rh = (lane / at.sw) % at.sh, rn = lane / (at.sw * at.sh);
          ok = rw < at.vw && rh < at.vh && rn < at.vn;
        } else {
          ok = m_row0 + lane < p.M;
        }
        const uint32_t rows_ok = __ballot_sync(0xffffffffu, ok);
#pragma unroll
        for (int rr = 0; rr < 32; ++rr) {
          uint32_t w = epi_lds32(base + rr * 128 + ((u ^ (rr & 7)) << 4));
          if (!((rows_ok >> rr) & 1u)) w = 0u;
          const float lo = __uint_as_float(w << 16), hi = __uint_as_float(w & 0xffff0000u);
          sum_lo += lo; sum_hi += hi;
          sq_lo = fmaf(lo, lo, sq_lo); sq_hi = fmaf(hi, hi, sq_hi);
        }
      } else {
#pragma unroll
        for (int rr = 0; rr < 32; ++rr) {
          const uint32_t w = epi_lds32(base + rr * 128 + ((u ^ (rr & 7)) << 4));
          const float lo = __uint_as_float(w << 16), hi = __uint_as_float(w & 0xffff0000u);
          sum_lo += lo; sum_hi += hi;
          sq_lo = fmaf(lo, lo, sq_lo); sq_hi = fmaf(hi, hi, sq_hi);
        }
      }
      // lane-private slots of the warp's region (columns past N hold zeros: zero-filled B rows)
      const uint32_t ps = smem_u32(s_stats) + (uint32_t)(((c0 - c_begin) + 2 * lane) << 2);
      float a0, a1, b0, b1;
      asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(a0), "=f"(a1) : "r"(ps));
      asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(b0), "=f"(b1) : "r"(ps + (STATS_WARP_FLOATS / 2) * 4));
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(ps), "f"(a0 + sum_lo), "f"(a1 + sum_hi) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(ps + (STATS_WARP_FLOATS / 2) * 4), "f"(b0 + sq_lo),
                   "f"(b1 + sq_hi)
                   : "memory");
    }
    if (lane == 0) {
      if (at.rank4) tma_store_4d(map_c, buf, col0, at.w, at.h, at.n);
      else tma_store_2d(map_c, buf, col0, m_row0);
      tma_store_commit();
    }
  }
}

// shared accumulators of GemmParams::stats: zero (all threads, before the kernel's first __syncthreads) and
// flush (all 8 epilogue warps together — named barrier 2 among the 256 of them — whenever the CTA moves to
// another column block and after its last tile): the four lane-quarter regions of a column are summed and
// added to this CTA's slot in global memory.  stats_finalize: the last CTA to finish adds the slots of all
// CTAs, in CTA order, to GemmParams::stats — the statistics (and everything computed from them) come out
// bit-identical from run to run, which fp32 atomics from the CTAs would not.
constexpr int STATS_MAX_CTAS = 256;
__device__ float g_stats_slots[STATS_MAX_CTAS * 2 * STATS_MAX_N];
__device__ unsigned int g_stats_done;
__device__ __forceinline__ float* stats_slot() { return g_stats_slots + (size_t)blockIdx.x * (2 * STATS_MAX_N); }
__device__ __forceinline__ void stats_zero(float* s_stats, int nthreads, int N) {
  for (int i = threadIdx.x; i < 8 * STATS_WARP_FLOATS; i += nthreads) s_stats[i] = 0.f;
  float* slot = stats_slot();
  for (int i = threadIdx.x; i < N; i += nthreads) {
    slot[i] = 0.f;
    slot[STATS_MAX_N + i] = 0.f;
  }
}
// all 256 epilogue threads, after their last stats_flush
__device__ __forceinline__ void stats_finalize(const GemmParams& p, int epi_tid) {
  __shared__ bool last;
  __threadfence();
  asm volatile("bar.sync 2, 256;" ::: "memory");
  if (epi_tid == 0) last = atomicAdd(&g_stats_done, 1u) == gridDim.x - 1;
  asm volatile("bar.sync 2, 256;" ::: "memory");
  if (!last) return;
  __threadfence();
  for (int c = epi_tid; c < p.N; c += 256) {
    float s = 0.f, q = 0.f;
    for (unsigned b = 0; b < gridDim.x; ++b) {
      s += __ldcg(g_stats_slots + (size_t)b * (2 * STATS_MAX_N) + c);
      q += __ldcg(g_stats_slots + (size_t)b * (2 * STATS_MAX_N) + STATS_MAX_N + c);
    }
    p.stats[c] += s;
    p.stats[p.N + c] += q;
  }
  if (epi_tid == 0) g_stats_done = 0u;
}

// Split-K in a fixed order without waiting: every split stores its partial tile into its own workspace
// slice, then counts itself in on the tile's counter; the split that arrives LAST sums the slices of all
// splits in split order and writes C + (0 + sum) (out_mode 1) or 0 + sum (out_mode 2), rounded once to C's
// dtype — the bits of adding the sum to a zeroed fp32 buffer and that buffer to C, signed zeros included.
// No CTA ever waits for another, so the kernel needs no co-residency, and the result is bit-identical from
// run to run (fp32 RED.ADDs from the splits would sum in arrival order).  All 256 epilogue threads, after
// the tile's epilogue; c_off = column offset of the tile's output inside C and inside each slice (the
// convolution's tap column).
__device__ __forceinline__ void splitk_finish_tile(const GemmParams& p, int tile, int m_idx, int n_idx, int bn,
                                                   long long c_off, int epi_tid, int* s_last) {
  __threadfence();
  asm volatile("bar.sync 3, 256;" ::: "memory");
  if (epi_tid == 0) *s_last = atomicAdd(p.splitk_count + tile, 1) == p.splits - 1;
  asm volatile("bar.sync 3, 256;" ::: "memory");
  if (!*s_last) return;
  __threadfence();
  const int rows = min(BLOCK_M, p.M - m_idx), c4n = min(bn, p.N - n_idx) >> 2;   // N % 8 == 0
  const bool add = p.out_mode == 1;
  for (int e = epi_tid; e < rows * c4n; e += 256) {
    const long long off = c_off + (long long)(m_idx + e / c4n) * p.ldc + n_idx + (e % c4n) * 4;
    float4 s = __ldcg(reinterpret_cast<const float4*>(p.splitk_ws + off));
    for (int k = 1; k < p.splits; ++k) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(p.splitk_ws + (long long)k * p.splitk_slice + off));
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    // not an identity for -0, so the compiler keeps these adds
    s.x = 0.0f + s.x; s.y = 0.0f + s.y; s.z = 0.0f + s.z; s.w = 0.0f + s.w;
    if (p.c_bf16) {
      uint2* c = reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.C) + off);
      if (add) {
        const uint2 o = *c;
        s.x += __uint_as_float(o.x << 16); s.y += __uint_as_float(o.x & 0xffff0000u);
        s.z += __uint_as_float(o.y << 16); s.w += __uint_as_float(o.y & 0xffff0000u);
      }
      *c = make_uint2(cvt_bf16x2(s.x, s.y), cvt_bf16x2(s.z, s.w));
    } else {
      float4* c = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.C) + off);
      if (add) {
        const float4 o = *c;
        s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
      }
      *c = s;
    }
  }
}

template <int BN>
__device__ __forceinline__ void stats_flush(const GemmParams& p, float* s_stats, int n_idx, int epi_tid) {
  constexpr int HALF = (BN >= 128) ? BN / 2 : BN;         // columns per epilogue warp
  asm volatile("bar.sync 2, 256;" ::: "memory");
  if (epi_tid < BN) {
    const int h = epi_tid / HALF, l = epi_tid % HALF;
    const float* r = s_stats + (h * 4) * STATS_WARP_FLOATS + l;
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      s += r[k * STATS_WARP_FLOATS];
      q += r[k * STATS_WARP_FLOATS + STATS_WARP_FLOATS / 2];
    }
    if (n_idx + epi_tid < p.N) {
      float* slot = stats_slot();
      slot[n_idx + epi_tid] += s;
      slot[STATS_MAX_N + n_idx + epi_tid] += q;
    }
  }
  asm volatile("bar.sync 2, 256;" ::: "memory");
#pragma unroll
  for (int i = 0; i < 8; ++i) s_stats[i * 256 + epi_tid] = 0.f;
  asm volatile("bar.sync 2, 256;" ::: "memory");
}

// ------------------------------------------------------------------ persistent GEMM / convolution body
// Persistent, warp-specialised, one CTA per SM, NUM_THREADS threads:
//   warpgroup 0    : TMA producer (one thread) filling the STAGES-deep operand ring
//   warpgroups 1-2 : 64 rows of the 128 x BN tile each (wg_mainloop), then the epilogue of those rows from
//                    the fragment (epilogue_frag) into the staging tile; after a barrier each of the 8 warps
//                    stores one 32-row slab, half of the columns (store_slab).  The producer keeps filling
//                    the ring during the epilogue.
// CTA b takes work items b, b + gridDim.x, ...; an item is one output tile, or one split of it.  What the
// items are is the kernel's Work description:
//   items             number of work items
//   kStats, kSplitK   whether the kernel can produce BN statistics / split-K partials at all
//   prefetch()        prefetches the tensor maps the kernel reads
//   num_kb(w)         64-deep K blocks of item w
//   load(w, next)     issues the TMA loads of item w: for each K block, `const Stage s = next()` waits for a
//                     free stage and arms its barrier for STAGE_BYTES; the A / B tiles go to s.a / s.b on s.bar
//   slab(w, q)        where rows 32q..32q+31 of item w's tile go
// Work holds POINTERS to the kernel's __grid_constant__ tensor maps: TMA reads a map from parameter,
// constant or global memory, never from a local copy.
struct Stage {
  uint8_t* a;
  uint8_t* b;
  uint64_t* bar;
};
struct Slab {
  const CUtensorMap* map_c;   // out_mode 0: output store map
  int m_row0, n_idx;          // first row of the slab in a row-major output (rank-2 StoreAt), first column
  StoreAt at;
  int tile;                   // split-K: arrival counter of the output tile
  int m_idx;                  // rank-2 outputs: first row of the output tile
  long long c_off;            // out_mode 1/2: column offset of the tile in C and in each workspace slice
  int split;                  // split-K: the item's split, whose workspace slice its partial tile goes to
};

template <int BN, bool A_MN, bool B_MN, class Work>
__device__ __forceinline__ void persistent_body(const Work& wk, const GemmParams& p) {
  using C = Cfg<BN>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + C::STAGES * C::A_BYTES;
  uint8_t* smem_store = smem + C::STAGES * C::STAGE_BYTES;   // 1024B-aligned staging tile of the bulk stores
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_store + C::STORE_BYTES);
  uint64_t* full_bar = bars;                     // [STAGES]
  uint64_t* empty_bar = bars + C::STAGES;        // [STAGES]
  float* s_stats = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);
  const bool want_stats = Work::kStats && p.stats != nullptr && p.out_mode == 0;
  if (want_stats) stats_zero(s_stats, NUM_THREADS, p.N);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    wk.prefetch();
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);               // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ============================ TMA producer ============================
    // one thread issues the loads: the warpgroup hands its registers to the consumers.  It is elected here
    // rather than tested with the lane == 0 of the set-up above, whose predicate would otherwise stay live
    // through the whole kernel (ptxas then spills the predicates of the 128-column GEMM to local memory)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      auto next = [&]() {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], C::STAGE_BYTES);
        const Stage s{smem_a + stage * C::A_BYTES, smem_b + stage * C::B_BYTES, &full_bar[stage]};
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        return s;
      };
      for (int w = blockIdx.x; w < wk.items; w += gridDim.x) wk.load(w, next);
    }
  } else {
    // ============================ wgmma + epilogue (warpgroups 1-2) ============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int cw = warp - 4;                      // consumer warp 0..7
    const int wg = cw >> 2;                       // rows 64*wg .. 64*wg+63 of the tile: its wgmma fragment
    const int r0 = wg * 64 + (cw & 3) * 16;       // the 16 fragment rows of this warp
    const int q = cw & 3;                         // 32-row slab this warp stores
    const int half = cw >> 2;                     // which half of the columns this warp stores
    const int c_begin = (BN >= 128) ? half * (BN / 2) : 0;
    const int c_end = (BN >= 128) ? c_begin + BN / 2 : (half == 0 ? BN : 0);
    const int epi_tid = cw * 32 + lane;
    float* my_stats = s_stats + cw * STATS_WARP_FLOATS;
    const uint32_t stg = smem_u32(smem_store);
    __shared__ int s_last;
    int stats_n = -1;                             // column block the shared statistics belong to
    int stage = 0;
    uint32_t phase = 0;
    float d[BN / 2];
    for (int w = blockIdx.x; w < wk.items; w += gridDim.x) {
      // where the tile goes is worked out while the first operand stage is still in flight, not after the MMAs
      const Slab s = wk.slab(w, q);
      wg_mainloop<BN, A_MN, B_MN, C::STAGES, C::A_BYTES, C::B_BYTES>(d, smem_u32(smem_a), smem_u32(smem_b), full_bar,
                                                                     empty_bar, stage, phase, wk.num_kb(w), wg);
      if (want_stats && s.n_idx != stats_n) {
        if (stats_n >= 0) stats_flush<BN>(p, s_stats, stats_n, epi_tid);
        stats_n = s.n_idx;
      }
      const bool res = p.residual != nullptr && p.out_mode != 1;
      uint4 rv[BN / 16];
      if (res) res_load<BN>(p, rv, s.m_idx, r0, s.n_idx, lane);
      if (p.out_mode == 0) {
        // the staging tile is rewritten once every bulk store and statistics walk of the previous tile has read it
        if (lane == 0) tma_store_wait_read<0>();
        named_bar(1, 256);
      }
      if (res) {
        __syncwarp();
        res_stage<BN>(rv, stg, r0, lane);
        __syncwarp();
      }
      epilogue_frag<BN>(p, d, stg, wg, s.m_idx, s.n_idx, s.split, s.c_off);
      if (p.out_mode == 0) {
        fence_async_smem();                       // the staged tile -> visible to the bulk stores
        named_bar(1, 256);
        store_slab<BN>(p, s.map_c, smem_store, q, lane, s.m_row0, s.n_idx, c_begin, c_end, s.at,
                       want_stats ? my_stats : nullptr);
      }
      if (Work::kSplitK && p.splits > 1) splitk_finish_tile(p, s.tile, s.m_idx, s.n_idx, BN, s.c_off, epi_tid, &s_last);
    }
    if (want_stats && stats_n >= 0) stats_flush<BN>(p, s_stats, stats_n, epi_tid);
    if (want_stats) stats_finalize(p, epi_tid);
    if (p.out_mode == 0 && lane == 0) tma_store_wait_all();   // smem must outlive the bulk reads
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
thread_local char g_err[512];    // one per source file: its b200dp_*_last_error
int g_num_sms = 0;

int fail(const char* msg, int code = 0) {
  snprintf(g_err, sizeof(g_err), "%s (%d)", msg, code);
  return -1;
}

// cuTensorMapEncode* is a driver-API call: it fails with CUDA_ERROR_INVALID_CONTEXT on a thread that
// has not yet bound the primary context (e.g. an autograd worker whose first GPU op is one of ours).
inline void bind_primary_context() {
  static thread_local bool bound = false;
  if (!bound) {
    cudaFree(nullptr);
    bound = true;
  }
}

int ensure_init() {
  bind_primary_context();
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult st;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &st);
  if (e != cudaSuccess || st != cudaDriverEntryPointSuccess || !fn)
    return fail("cuTensorMapEncodeTiled entry point unavailable", (int)e);
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  return 0;
}

// bf16 tensor map of `rank` dimensions, 128B swizzle: dims[0] is contiguous, byte_strides[i] is the pitch of
// dims[i + 1], out-of-bounds elements read as zero.
int encode_map(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* byte_strides,
               const cuuint32_t* box) {
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims, byte_strides, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed", (int)r);
  return 0;
}

// 2D bf16 map: `rows` x `cols` (cols contiguous), row pitch `ld` elements, box {64, box_rows}
// (the same encoding serves the operand loads and the 32-row bulk stores)
int make_map2(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {ld * 2};
  const cuuint32_t box[2] = {64, box_rows};
  return encode_map(m, ptr, 2, dims, strides, box);
}

// sets Kernel's dynamic shared memory limit on its first launch
template <auto Kernel>
int smem_attr_once(int bytes) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
    attr_set = true;
  }
  return 0;
}

// A persistent_body kernel over `work` items: one CTA per SM at most, fewer with max_ctas > 0, and never more
// than the BN statistics have slots for.
template <auto Kernel, int BN, class... Args>
int launch_persistent(int work, int max_ctas, cudaStream_t st, const Args&... args) {
  if (smem_attr_once<Kernel>(Cfg<BN>::SMEM_BYTES)) return -1;
  int grid = work < g_num_sms ? work : g_num_sms;
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  if (grid > STATS_MAX_CTAS) grid = STATS_MAX_CTAS;
  Kernel<<<grid, NUM_THREADS, Cfg<BN>::SMEM_BYTES, st>>>(args...);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  return 0;
}

// Runs launch() with a split-K workspace (p.splits > 1) for `tiles` output tiles of p.splitk_slice elements,
// stream-ordered on the launch stream so that concurrent launches never share one: the fp32 slices and the
// zeroed per-tile arrival counters of splitk_finish_tile, freed with cudaFreeAsync after the launch.
template <class Launch>
int run_splitk(GemmParams& p, int tiles, cudaStream_t st, Launch&& launch) {
  void* ws = nullptr;
  if (p.splits > 1) {
    const size_t slices = (size_t)p.splits * (size_t)p.splitk_slice * sizeof(float);
    cudaError_t e = cudaMallocAsync(&ws, slices + (size_t)tiles * sizeof(int), st);
    if (e == cudaSuccess) {
      p.splitk_ws = reinterpret_cast<float*>(ws);
      p.splitk_count = reinterpret_cast<int*>(reinterpret_cast<char*>(ws) + slices);
      e = cudaMemsetAsync(p.splitk_count, 0, (size_t)tiles * sizeof(int), st);
    }
    if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  }
  const int rc = launch();
  if (ws != nullptr) {
    cudaError_t e = cudaFreeAsync(ws, st);
    if (e != cudaSuccess && rc == 0) return fail(cudaGetErrorString(e), (int)e);
  }
  return rc;
}

// K splits over kblocks K blocks, clamped to 1..kblocks and reduced until no split is empty
int normalize_splits(int splits, int kblocks) {
  if (splits > kblocks) splits = kblocks;
  if (splits < 1) splits = 1;
  const int per = (kblocks + splits - 1) / splits;
  return (kblocks + per - 1) / per;
}

// tile width: 0 picks 64 or 128 from the output width n; 256 runs as 128, the widest tile whose accumulator
// image fits in shared memory next to the operand ring
int pick_bn(int n, int block_n) {
  if (block_n == 0) return n > 64 ? 128 : 64;
  if (block_n == 256) return 128;
  if (block_n != 64 && block_n != 128) return fail("block_n must be 64/128/256");
  return block_n;
}

}  // namespace

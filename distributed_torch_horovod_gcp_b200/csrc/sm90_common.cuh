// Shared sm_90a device helpers: mbarrier / TMA / wgmma PTX wrappers, GMMA shared-memory descriptors and the
// fused accumulator->register->smem->TMA-store epilogue used by the GEMM (gemm_sm90.cu), the implicit-GEMM
// convolution (conv_sm90.cu) and the attention kernels (attn_sm90.cu).
//
// wgmma keeps its accumulator in the registers of the issuing warpgroup, in a fragment layout (each warp
// holds 16 rows, each thread two rows x pairs of columns).  The epilogues work on one accumulator ROW per
// lane, so a finished tile is written once to a row-major fp32 image in shared memory ("accumulator
// image", row pitch = columns + 4 floats: conflict-free 16-byte reads of one row per lane) and the
// epilogue warps read 32-column runs of their rows from it.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 bf16 = 128 bytes = one 128B swizzle atom
constexpr int WGMMA_K = 16;        // K of one wgmma (bf16)
constexpr int NUM_THREADS = 384;     // warpgroup 0: TMA producer; warpgroups 1-2: wgmma + epilogue (8 warps)
constexpr int EPI_WARPS = 8;
constexpr int SMEM_LIMIT = 232448;   // 227 KB of dynamic shared memory per block on sm_90

struct GemmParams {
  int M, N, K;
  int ldc;                 // elements
  int num_m_blocks, num_n_blocks, num_k_blocks;
  int splits;              // split-K factor (>=1)
  int act;                 // 0 none, 1 relu, 2 gelu(erf), 3 *gelu'(aux), 4 *(aux>0)  [aux = residual ptr]
  int out_mode;            // 0: bf16 store, 1: fp32 atomic add (split-K / accumulate), 2: fp32 store
  void* C;
  const void* bias;        // bf16 [N] or nullptr
  const void* bias_f32;    // fp32 [N] or nullptr
  const void* residual;    // bf16 [M, ldc] or nullptr (added after act; or `aux` for act 3/4)
  void* preact;            // optional bf16 [M, ldc]: pre-activation values (saved for backward)
  int tma_store;           // out_mode 0: stage the tile in swizzled smem and write it with TMA bulk stores
  int n_fastest;           // tile order: consecutive CTAs walk the N blocks of one M block first (A tile is
                           // fetched from HBM once and re-used from L2 while the whole B matrix stays in L2)
  float alpha;
  const unsigned char* res_mask;   // optional, with a plain residual (act 0..2): bit j of byte [row][col/8] keeps
                           // residual element (row, 8*(col/8)+j) — the ReLU sign bits of the block output whose
                           // skip-branch gradient the residual is (N % 64 == 0 required)
  float* stats;            // optional fp32 [2][N]: per-column sum | sum of squares of the bf16 OUTPUT (the batch
                           // statistics of the BatchNorm that follows), accumulated by the epilogue
  // split-K (splits > 1, out_mode 1): per-launch workspace — one fp32 slice of splitk_slice elements per split,
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


// m64 x N accumulator fragment of this thread's warpgroup -> rows row0.. of a row-major fp32 image
template <int N>
__device__ __forceinline__ void acc_to_smem(const float* d, uint32_t img, int ld, int row0) {
  const int t = threadIdx.x & 127;
  const int r = row0 + (t >> 5) * 16 + ((t & 31) >> 2);
  const uint32_t p0 = img + (uint32_t)((r * ld + 2 * (t & 3)) * 4);
  const uint32_t p1 = p0 + (uint32_t)(8 * ld * 4);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p0 + j * 32), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p1 + j * 32), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
  }
}
// 32 consecutive fp32 of one image row (bit patterns)
__device__ __forceinline__ void acc_ld32(uint32_t addr, uint32_t* r) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[4 * i]), "=r"(r[4 * i + 1]), "=r"(r[4 * i + 2]), "=r"(r[4 * i + 3])
                 : "r"(addr + 16 * i)
                 : "memory");
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

__device__ __forceinline__ uint4 pack8(const float* v) {
  uint32_t wv[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * t], v[2 * t + 1]);
    wv[t] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(wv[0], wv[1], wv[2], wv[3]);
}

template <int BN>
struct Cfg {
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BN * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_LD = BN + 4;          // accumulator image row pitch (floats)
  static constexpr int ACC_BYTES = BLOCK_M * ACC_LD * 4;
  static constexpr int STORE_BYTES = EPI_WARPS * 2 * 4096;   // per epilogue warp: out + preact staging (32 rows x 128 B each)
  static constexpr int FIXED_BYTES = STORE_BYTES + ACC_BYTES + 1024 /*align*/ + 256 /*barriers*/ + STATS_SMEM_BYTES;
  // as many operand stages as fit next to the accumulator image (BN 64: 4, BN 128: 2)
  static constexpr int STAGES = (SMEM_LIMIT - FIXED_BYTES) / STAGE_BYTES > 4 ? 4 : (SMEM_LIMIT - FIXED_BYTES) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED_BYTES;
  static_assert(STAGES >= 2, "shared memory");
};

// Epilogue of one 32-row slab (rows 32q..32q+31) of a 128 x BN accumulator: accumulator image ->
// registers -> alpha/bias/activation/residual -> bf16 via swizzled smem + TMA bulk store, or fp32
// store / atomic add.
// Where a 32-row slab goes.  rank4 == 0: rows m_row0.. of the row-major [M, ldc] matrix (2D map).
// rank4 == 1 (convolution): the slab is the {64 c, sw, sh, sn} sub-box at pixel (w, h, n) of an NHWC
// tensor; c_ptr/ld override p.C/p.ldc for the fp32 modes (per-tap column offset of the wgrad output).
struct StoreAt {
  int rank4, w, h, n;
  void* c_ptr;
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
__device__ __forceinline__ uint4 epi_lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
// prmt.b32 in its default mode: selector nibble bit 3 = replicate the selected byte's sign bit
__device__ __forceinline__ uint32_t prmt_sign(uint32_t a, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(0u), "r"(sel));
  return d;
}
__device__ __forceinline__ uint4 pack8r(const uint32_t* r) {   // 8 fp32 bit patterns -> 8 bf16
  uint4 o;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.x) : "f"(__uint_as_float(r[1])), "f"(__uint_as_float(r[0])));
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.y) : "f"(__uint_as_float(r[3])), "f"(__uint_as_float(r[2])));
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.z) : "f"(__uint_as_float(r[5])), "f"(__uint_as_float(r[4])));
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.w) : "f"(__uint_as_float(r[7])), "f"(__uint_as_float(r[6])));
  return o;
}

template <int BN>
__device__ __forceinline__ void epilogue_rows(const GemmParams& p, const CUtensorMap* map_c,
                                              const CUtensorMap* map_z, uint32_t acc_img, int acc, int q,
                                              int lane, int m_row0, int n_idx, int c_begin, int c_end,
                                              uint8_t* my_store, const StoreAt at = StoreAt{0, 0, 0, 0, nullptr, 32, 1, 32, 1, 1},
                                              float* s_stats = nullptr) {
  // A 64-column chunk (one 128-byte bf16 row per lane, one TMA store box) is produced in two 32-column
  // halves: 32 accumulator values + 32 results live per thread instead of 64 + 64 — the previous
  // single-pass version spilled ~300 B per thread at the 168-register budget of a 320-thread CTA, and the
  // epilogue, not the MMA, bounds every K <= 512 GEMM / convolution here.
  const int row = m_row0 + lane;
  const bool row_ok = row < p.M;
  const bool to_tma = p.out_mode == 0 && p.tma_store;
  const bool z_tma = p.preact != nullptr && to_tma;
  const bool res_smem = p.residual != nullptr && p.preact == nullptr && p.out_mode != 1;
  // the common case (plain bf16 output, optionally with BN statistics): no per-element work at all
  const bool plain = to_tma && p.alpha == 1.0f && p.bias == nullptr && p.bias_f32 == nullptr &&
                     p.preact == nullptr && p.act == 0 && p.residual == nullptr;
  const bool res_only = to_tma && res_smem && p.alpha == 1.0f && p.bias == nullptr && p.bias_f32 == nullptr &&
                        p.act == 0;
  const uint32_t store_s = smem_u32(my_store);
  const uint32_t lane_row = (uint32_t)lane * 128u;
  const uint32_t lsw = (uint32_t)(lane & 7);
#pragma unroll 1
  for (int c0 = c_begin; c0 < c_end; c0 += 64) {
    const int col0 = n_idx + c0;
    if (col0 >= p.N) continue;                       // warp-uniform
    const int ncols = min(64, p.N - col0);           // N % 8 == 0 is enforced by the host
    // Residual / auxiliary operand of the slab: COALESCED 16-byte loads (a warp instruction covers 4 rows
    // x 128 B), issued before the accumulator loads so that their latency overlaps, then transposed to
    // row-per-lane through the second (pre-activation) staging buffer.
    uint4 resv[8];
    if (res_smem) {
      const __nv_bfloat16* rbase = reinterpret_cast<const __nv_bfloat16*>(p.residual);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + (lane >> 3), u = lane & 7;
        resv[i] = (m_row0 + rr < p.M && u * 8 < ncols)
                      ? *reinterpret_cast<const uint4*>(rbase + (size_t)(m_row0 + rr) * p.ldc + col0 + u * 8)
                      : make_uint4(0, 0, 0, 0);
      }
      if (p.res_mask != nullptr) {
        // ReLU sign bits of the residual (1 byte per 8 channels): bit j -> 16-bit lane j.  Byte k of
        // ((bits * 0x01010101) & 0x08040201) + 0x7f7f7f7f has its MSB set iff bit k is, and PRMT's
        // sign-replicate mode turns that MSB into 0x00 / 0xff bytes.
        uint32_t mbits[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int rr = i * 4 + (lane >> 3), u = lane & 7;
          mbits[i] = (m_row0 + rr < p.M && u * 8 < ncols)
                         ? (uint32_t)p.res_mask[(size_t)(m_row0 + rr) * (size_t)(p.N >> 3) + (size_t)((col0 >> 3) + u)]
                         : 0u;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const uint32_t rep = mbits[i] * 0x01010101u;
          const uint32_t lo = (rep & 0x08040201u) + 0x7f7f7f7fu, hi = (rep & 0x80402010u) + 0x7f7f7f7fu;
          resv[i].x &= prmt_sign(lo, 0x9988u);
          resv[i].y &= prmt_sign(lo, 0xbbaau);
          resv[i].z &= prmt_sign(hi, 0x9988u);
          resv[i].w &= prmt_sign(hi, 0xbbaau);
        }
      }
    }
    // Staging: two 4 KB buffers per warp.  When the second one is not needed for the pre-activation tile or
    // the residual transpose, consecutive chunks ALTERNATE between them and only wait for the store issued
    // two chunks ago (cp.async.bulk.wait_group.read 1) — otherwise every chunk stalls on its predecessor's
    // bulk store reading shared memory.
    const bool dbuf = to_tma && !z_tma && !res_smem;
    // buffer parity must alternate over the sequence of chunks THIS warp stages, across tiles: with an even
    // number of chunks per tile the chunk index does it, with one chunk per tile the (alternating) accumulator
    // index does
    const int par = (((c0 - c_begin) >> 6) + acc * (((c_end - c_begin) >> 6) & 1)) & 1;
    const uint32_t out_s = store_s + ((dbuf && par) ? 4096u : 0u);
    if (res_smem) {
      if (lane == 0) tma_store_wait_read<0>();       // (second buffer is about to be rewritten)
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + (lane >> 3), u = lane & 7;
        epi_sts128(store_s + 4096u + rr * 128 + ((u ^ (rr & 7)) << 4), resv[i]);
      }
      __syncwarp();
    }
    const uint32_t taddr = acc_img + (uint32_t)(((q * 32 + lane) * (BN + 4) + c0) * 4);
    if (plain) {
      // ---- fast path: accumulator -> bf16 -> swizzled staging rows, nothing else ----
      uint32_t r[32];
      acc_ld32(taddr, r);
      if (lane == 0) {       // the bulk store that last read this buffer must be done reading it
        if (dbuf) tma_store_wait_read<1>();
        else tma_store_wait_read<0>();
      }
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; ++j) epi_sts128(out_s + lane_row + ((j ^ lsw) << 4), pack8r(r + j * 8));
      if (ncols > 32) {
        acc_ld32(taddr + 128, r);
#pragma unroll
        for (int j = 0; j < 4; ++j) epi_sts128(out_s + lane_row + (((4 + j) ^ lsw) << 4), pack8r(r + j * 8));
      }
    } else if (res_only) {
      // ---- skip-gradient path of the dgrad GEMMs: bf16(acc + residual) ----
#pragma unroll 1
      for (int half = 0; half < 2; ++half) {
        if (half * 32 >= ncols) break;
        uint32_t r[32];
        acc_ld32(taddr + half * 128, r);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t off = lane_row + (((half * 4 + j) ^ lsw) << 4);
          const uint4 rv = epi_lds128(store_s + 4096u + off);
          const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
          uint4 o;
          uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            const float s0 = __uint_as_float(r[j * 8 + 2 * w]) + __uint_as_float(rw[w] << 16);
            const float s1 = __uint_as_float(r[j * 8 + 2 * w + 1]) + __uint_as_float(rw[w] & 0xffff0000u);
            asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(ow[w]) : "f"(s1), "f"(s0));
          }
          epi_sts128(out_s + off, o);      // the store that read this buffer was waited for above (res_smem)
        }
      }
    } else {
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
      const int hc = half * 32;                      // first column of this half inside the chunk
      if (hc >= ncols) break;                        // warp-uniform
      const int hcols = min(32, ncols - hc);
      uint32_t r[32];
      acc_ld32(taddr + hc * 4, r);
      float v[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
      if (p.alpha != 1.0f) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] *= p.alpha;
      }
      if (p.out_mode != 1) {
        if (p.bias != nullptr) {
          const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(p.bias) + col0 + hc;
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (i < hcols) v[i] += __bfloat162float(b[i]);
        } else if (p.bias_f32 != nullptr) {
          const float* b = reinterpret_cast<const float*>(p.bias_f32) + col0 + hc;
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (i < hcols) v[i] += b[i];
        }
        if (p.preact != nullptr) {
          if (z_tma) {            // pre-activation tile -> second staging buffer (stored by TMA with the output)
            if (half == 0) {
              if (lane == 0) tma_store_wait_read<0>();
              __syncwarp();
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
              epi_sts128(store_s + 4096u + lane_row + (((half * 4 + j) ^ lsw) << 4), pack8(v + j * 8));
          } else if (row_ok) {
            uint4* pp = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.preact) +
                                                 (size_t)row * p.ldc + col0 + hc);
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (j * 8 < hcols) pp[j] = pack8(v + j * 8);
          }
        }
        if (p.act == 1) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.0f);
        } else if (p.act == 2) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
        }
        if (p.residual != nullptr && (row_ok || res_smem)) {
          const uint4* rp = reinterpret_cast<const uint4*>(
              reinterpret_cast<const __nv_bfloat16*>(p.residual) + (size_t)row * p.ldc + col0 + hc);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (j * 8 < hcols) {
              float a[8];
              unpack8(res_smem ? epi_lds128(store_s + 4096u + lane_row + (((half * 4 + j) ^ lsw) << 4)) : rp[j], a);
#pragma unroll
              for (int t = 0; t < 8; ++t) {
                if (p.act == 3) v[j * 8 + t] *= gelu_erf_grad(a[t]);
                else if (p.act == 4) v[j * 8 + t] = a[t] > 0.0f ? v[j * 8 + t] : 0.0f;
                else v[j * 8 + t] += a[t];
              }
            }
          }
        }
      }
      if (to_tma) {
        if (half == 0) {       // the bulk store that last read this buffer must be done reading it
          if (lane == 0) {
            if (dbuf) tma_store_wait_read<1>();
            else tma_store_wait_read<0>();
          }
          __syncwarp();
        }
        // this half of the 32 x 128 B swizzled staging rows (conflict-free 16-byte stores)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          epi_sts128(out_s + lane_row + (((half * 4 + j) ^ lsw) << 4), pack8(v + j * 8));
      } else if (p.out_mode == 1) {
        // fp32 accumulation: transpose the 32 x 32 fp32 half through the staging buffer so that a
        // warp-level RED covers four 128-byte row segments with 16-byte vectors (red.global.add.v4.f32).
        // With split-K the partial tile is STORED into this split's workspace slice (at.c_ptr) instead.
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; ++j)
          epi_sts128(store_s + lane_row + ((j ^ lsw) << 4),
                 make_uint4(__float_as_uint(v[4 * j]), __float_as_uint(v[4 * j + 1]), __float_as_uint(v[4 * j + 2]),
                            __float_as_uint(v[4 * j + 3])));
        __syncwarp();
        float* cbase = reinterpret_cast<float*>(at.c_ptr ? at.c_ptr : p.C);
        const int ch = lane & 7;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int rr = it * 4 + (lane >> 3);
          const uint4 t = epi_lds128(store_s + rr * 128 + ((ch ^ (rr & 7)) << 4));
          if (m_row0 + rr < p.M && ch * 4 < hcols) {
            float* dst = cbase + (size_t)(m_row0 + rr) * p.ldc + col0 + hc + ch * 4;
            if (p.splits > 1)
              asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(t.x), "r"(t.y), "r"(t.z),
                           "r"(t.w)
                           : "memory");
            else
              asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(t.x), "r"(t.y), "r"(t.z),
                           "r"(t.w)
                           : "memory");
          }
        }
        __syncwarp();
      } else if (row_ok) {
        if (p.out_mode == 0) {
          uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.C) + (size_t)row * p.ldc + col0 + hc);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (j * 8 < hcols) dst[j] = pack8(v + j * 8);
        } else {   // out_mode 2: fp32 store
          float* dst = reinterpret_cast<float*>(at.c_ptr ? at.c_ptr : p.C) + (size_t)row * p.ldc + col0 + hc;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (j * 4 < hcols)
              reinterpret_cast<float4*>(dst)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        }
      }
    }
    }
    if (to_tma) {
      fence_async_smem();
      __syncwarp();
      if (s_stats != nullptr) {
        // batch statistics of the following BatchNorm: column sums of the bf16 values just staged.  Lane l
        // owns columns 2l, 2l+1 of this 64-column chunk and walks the 32 staged rows (one conflict-free
        // 4-byte shared load per row); partials go to the warp's private shared
        // accumulators.  GEMM rows past M come from zero-filled operands and add nothing; rows of a
        // convolution tile outside the image are masked (they see partly valid taps).
        float sum_lo = 0.f, sum_hi = 0.f, sq_lo = 0.f, sq_hi = 0.f;
        const uint32_t base = out_s + (uint32_t)((lane & 3) << 2);
        const uint32_t u = (uint32_t)(lane >> 2);
        if (at.rank4) {      // lane r decides for slab row r
          const int rw = lane % at.sw, rh = (lane / at.sw) % at.sh, rn = lane / (at.sw * at.sh);
          const uint32_t rows_ok = __ballot_sync(0xffffffffu, rw < at.vw && rh < at.vh && rn < at.vn);
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            uint32_t w;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(base + rr * 128 + ((u ^ (rr & 7)) << 4)));
            if (!((rows_ok >> rr) & 1u)) w = 0u;
            const float lo = __uint_as_float(w << 16), hi = __uint_as_float(w & 0xffff0000u);
            sum_lo += lo; sum_hi += hi;
            sq_lo = fmaf(lo, lo, sq_lo); sq_hi = fmaf(hi, hi, sq_hi);
          }
        } else {
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            uint32_t w;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(base + rr * 128 + ((u ^ (rr & 7)) << 4)));
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
        const uint8_t* buf = my_store + (out_s - store_s);
        if (at.rank4) {
          tma_store_4d(map_c, buf, col0, at.w, at.h, at.n);
        } else {
          tma_store_2d(map_c, buf, col0, m_row0);
          if (p.preact != nullptr) tma_store_2d(map_z, buf + 4096, col0, m_row0);
        }
        tma_store_commit();
      }
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
// splits in split order and adds the sum to C.  No CTA ever waits for another, so the kernel needs no
// co-residency, and the result is bit-identical from run to run (fp32 RED.ADDs from the splits would
// sum in arrival order).  All 256 epilogue threads, after the tile's epilogue; c_off = column offset of
// the tile's output inside C and inside each slice (the convolution's tap column).
__device__ __forceinline__ void splitk_finish_tile(const GemmParams& p, int tile, int m_idx, int n_idx, int bn,
                                                   long long c_off, int epi_tid, int* s_last) {
  __threadfence();
  asm volatile("bar.sync 3, 256;" ::: "memory");
  if (epi_tid == 0) *s_last = atomicAdd(p.splitk_count + tile, 1) == p.splits - 1;
  asm volatile("bar.sync 3, 256;" ::: "memory");
  if (!*s_last) return;
  __threadfence();
  const int rows = min(BLOCK_M, p.M - m_idx), c4n = min(bn, p.N - n_idx) >> 2;   // N % 8 == 0
  float* C = reinterpret_cast<float*>(p.C);
  for (int e = epi_tid; e < rows * c4n; e += 256) {
    const long long off = c_off + (long long)(m_idx + e / c4n) * p.ldc + n_idx + (e % c4n) * 4;
    float4 s = __ldcg(reinterpret_cast<const float4*>(p.splitk_ws + off));
    for (int k = 1; k < p.splits; ++k) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(p.splitk_ws + (long long)k * p.splitk_slice + off));
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    float4* c = reinterpret_cast<float4*>(C + off);
    float4 o = *c;
    o.x += s.x; o.y += s.y; o.z += s.z; o.w += s.w;
    *c = o;
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

// Split-K workspace for one launch, stream-ordered on the launch stream (so concurrent launches never share
// one; freed with cudaFreeAsync on the same stream after the launch): the fp32 slices and the zeroed per-tile
// arrival counters of splitk_finish_tile.
inline cudaError_t splitk_alloc(void** ws, GemmParams* p, int tiles, cudaStream_t st) {
  const size_t slices = (size_t)p->splits * (size_t)p->splitk_slice * sizeof(float);
  cudaError_t e = cudaMallocAsync(ws, slices + (size_t)tiles * sizeof(int), st);
  if (e != cudaSuccess) return e;
  p->splitk_ws = reinterpret_cast<float*>(*ws);
  p->splitk_count = reinterpret_cast<int*>(reinterpret_cast<char*>(*ws) + slices);
  return cudaMemsetAsync(p->splitk_count, 0, (size_t)tiles * sizeof(int), st);
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

}  // namespace

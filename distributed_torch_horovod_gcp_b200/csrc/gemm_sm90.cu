// bf16 GEMM for sm_90a: TMA -> shared (128B swizzle) -> wgmma -> registers -> fused epilogue.
//
//   C[M,N] (+)= act( A[M,K] * B[N,K]^T + bias[N] ) + residual[M,N]
//
// A and B can each be K-major (row-major [rows][K]) or MN-major (stored [K][rows]), so the
// same kernel serves linear / 1x1-conv forward (A=x, B=W), dgrad (A=dy, B=W as MN-major) and
// wgrad (A=dy^T, B=x^T, both MN-major, split-K with fp32 atomics) without any transpose pass:
// wgmma reads MN-major bf16 operands through its transpose flags.
//
// Structure (persistent, warp-specialised, one CTA per SM, 384 threads):
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor.2d, mbarrier complete_tx)
//   warpgroups 1-2 : 64 rows of the 128 x BN tile each (wgmma m64nBNk16, accumulator in registers);
//                    then all 8 warps run the epilogue (accumulator image -> bias/act/residual ->
//                    swizzled smem -> TMA bulk store), two warps per 32-row slab, each taking half of
//                    the columns.  The producer keeps filling the ring during the epilogue.
//
// This replaces the cuBLAS addmm / cuDNN 1x1-conv calls on the model zoo's hot path.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "sm90_common.cuh"

namespace {


template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_c, const __grid_constant__ CUtensorMap map_z,
                 const GemmParams p) {
  using C = Cfg<BN>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + C::STAGES * C::A_BYTES;
  uint8_t* smem_store = smem + C::STAGES * C::STAGE_BYTES;   // 1024B-aligned staging for TMA stores
  uint8_t* smem_acc = smem_store + C::STORE_BYTES;           // accumulator image [128][BN + 4] fp32
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_acc + C::ACC_BYTES);
  uint64_t* full_bar = bars;                     // [STAGES]
  uint64_t* empty_bar = bars + C::STAGES;        // [STAGES]
  float* s_stats = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);
  const bool want_stats = p.stats != nullptr && p.out_mode == 0 && p.tma_store;
  if (want_stats) stats_zero(s_stats, NUM_THREADS, p.N);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    if (p.tma_store) tma_prefetch_desc(&map_c);
    if (p.tma_store && p.preact != nullptr) tma_prefetch_desc(&map_z);
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);               // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int tiles = p.num_m_blocks * p.num_n_blocks;
  const int work_items = tiles * p.splits;
  const int kb_per_split = (p.num_k_blocks + p.splits - 1) / p.splits;

  if (warp < 4) {
    // ============================ TMA producer ============================
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < work_items; w += gridDim.x) {
        const int tile = w % tiles, split = w / tiles;
        const int m_idx = (p.n_fastest ? tile / p.num_n_blocks : tile % p.num_m_blocks) * BLOCK_M;
        const int n_idx = (p.n_fastest ? tile % p.num_n_blocks : tile / p.num_m_blocks) * BN;
        const int kb0 = split * kb_per_split;
        const int kb1 = min(kb0 + kb_per_split, p.num_k_blocks);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          uint8_t* sa = smem_a + stage * C::A_BYTES;
          uint8_t* sb = smem_b + stage * C::B_BYTES;
          const int k_idx = kb * BLOCK_K;
          if (!A_MN) {
            tma_load_2d(&map_a, &full_bar[stage], sa, k_idx, m_idx);           // box {64 k, 128 m}
          } else {
#pragma unroll
            for (int c = 0; c < BLOCK_M / 64; ++c)                                // box {64 m, 64 k}
              tma_load_2d(&map_a, &full_bar[stage], sa + c * (BLOCK_K * 128), m_idx + 64 * c, k_idx);
          }
          if (!B_MN) {
            tma_load_2d(&map_b, &full_bar[stage], sb, k_idx, n_idx);           // box {64 k, BN n}
          } else {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)
              tma_load_2d(&map_b, &full_bar[stage], sb + c * (BLOCK_K * 128), n_idx + 64 * c, k_idx);
          }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ============================ wgmma + epilogue (warpgroups 1-2) ============================
    const int cw = warp - 4;                      // consumer warp 0..7
    const int wg = cw >> 2;                       // rows 64*wg .. 64*wg+63 of the tile
    const int q = cw & 3;                         // 32-row slab this warp drains
    const int half = cw >> 2;                     // which half of the columns this warp drains
    const int c_begin = (BN >= 128) ? half * (BN / 2) : 0;
    const int c_end = (BN >= 128) ? c_begin + BN / 2 : (half == 0 ? BN : 0);
    uint8_t* my_store = smem_store + cw * (2 * 4096);
    float* my_stats = s_stats + cw * STATS_WARP_FLOATS;
    const uint32_t img = smem_u32(smem_acc);
    __shared__ int s_last;
    int stats_n = -1;                             // column block the shared statistics belong to
    int stage = 0, acc = 0;
    uint32_t phase = 0;
    float d[BN / 2];
    for (int w = blockIdx.x; w < work_items; w += gridDim.x) {
      const int tile = w % tiles, split = w / tiles;
      const int m_idx = (p.n_fastest ? tile / p.num_n_blocks : tile % p.num_m_blocks) * BLOCK_M;
      const int n_idx = (p.n_fastest ? tile % p.num_n_blocks : tile / p.num_m_blocks) * BN;
      const int kb0 = split * kb_per_split;
      const int nkb = min(kb0 + kb_per_split, p.num_k_blocks) - kb0;
      wg_mainloop<BN, A_MN, B_MN, C::STAGES, C::A_BYTES, C::B_BYTES>(d, smem_u32(smem_a), smem_u32(smem_b), full_bar,
                                                                     empty_bar, stage, phase, nkb, wg);
      if (want_stats && n_idx != stats_n) {
        if (stats_n >= 0) stats_flush<BN>(p, s_stats, stats_n, cw * 32 + lane);
        stats_n = n_idx;
      }
      named_bar(1, 256);                          // the previous tile's image has been read
      acc_to_smem<BN>(d, img, BN + 4, wg * 64);
      named_bar(1, 256);
      epilogue_rows<BN>(p, &map_c, &map_z, img, acc, q, lane, m_idx + q * 32, n_idx, c_begin, c_end,
                        my_store,
                        StoreAt{0, 0, 0, 0, p.splits > 1 ? p.splitk_ws + (long long)split * p.splitk_slice : nullptr},
                        want_stats ? my_stats : nullptr);
      if (p.splits > 1) splitk_finish_tile(p, tile, m_idx, n_idx, BN, 0, cw * 32 + lane, &s_last);
      acc ^= 1;
    }
    if (want_stats && stats_n >= 0) stats_flush<BN>(p, s_stats, stats_n, cw * 32 + lane);
    if (want_stats) stats_finalize(p, cw * 32 + lane);
    if (p.tma_store && lane == 0) tma_store_wait_all();   // smem must outlive the bulk reads
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
thread_local char g_err[512];
int g_num_sms = 0;

int fail(const char* msg, int code = 0) {
  snprintf(g_err, sizeof(g_err), "%s (%d)", msg, code);
  return -1;
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

// 2D bf16 tensor map: `rows` x `cols` (cols contiguous), row pitch `ld` elements, box {64, box_rows}.
// (the same encoding serves the loads of A/B and the 32-row bulk stores of C)
int make_map(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed", (int)r);
  return 0;
}

template <int BN, bool A_MN, bool B_MN>
int launch(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mc, const CUtensorMap& mz,
           const GemmParams& p, int max_ctas, cudaStream_t st) {
  using C = Cfg<BN>;
  auto kern = gemm_bf16_kernel<BN, A_MN, B_MN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
    attr_set = true;
  }
  const int work = p.num_m_blocks * p.num_n_blocks * p.splits;
  int grid = work < g_num_sms ? work : g_num_sms;
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  if (grid > STATS_MAX_CTAS) grid = STATS_MAX_CTAS;
  kern<<<grid, NUM_THREADS, C::SMEM_BYTES, st>>>(ma, mb, mc, mz, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  return 0;
}

int launch_bn(int BN, int a_mn, int b_mn, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mc,
              const CUtensorMap& mz, const GemmParams& p, int max_ctas, cudaStream_t st) {
#define DISPATCH(BNV)                                                                         \
  if (BN == BNV) {                                                                            \
    if (!a_mn && !b_mn) return launch<BNV, false, false>(ma, mb, mc, mz, p, max_ctas, st);            \
    if (!a_mn && b_mn) return launch<BNV, false, true>(ma, mb, mc, mz, p, max_ctas, st);              \
    if (a_mn && !b_mn) return launch<BNV, true, false>(ma, mb, mc, mz, p, max_ctas, st);              \
    return launch<BNV, true, true>(ma, mb, mc, mz, p, max_ctas, st);                                  \
  }
  DISPATCH(64)
  DISPATCH(128)
#undef DISPATCH
  return fail("unreachable");
}

}  // namespace

extern "C" {

const char* b200dp_gemm_last_error() { return g_err; }

// A: K-major -> [M][lda>=K]; MN-major -> [K][lda>=M].   B: K-major -> [N][ldb>=K]; MN-major -> [K][ldb>=N].
// C: [M][ldc>=N].  out_mode 0: bf16 = act(alpha*AB + bias) + residual; 1: fp32 atomic +=; 2: fp32 store.
// Requirements: K % 8 == 0 for K-major operands, M % 8 (A) / N % 8 (B) == 0 for MN-major, N % 8 == 0,
// 16-byte aligned base pointers and leading dimensions.
int b200dp_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                     int a_mn, int b_mn, const void* bias_bf16, const void* bias_f32, const void* residual,
                     void* preact, int act, int out_mode, float alpha, int splits, int block_n, int max_ctas,
                     float* stats, const void* res_mask, unsigned long long stream) {
  if (ensure_init()) return -1;
  if (M <= 0 || N <= 0 || K <= 0) return fail("bad shape");
  if ((N % 8) || (lda % 8) || (ldb % 8) || (ldc % 4) || ((out_mode == 0) && (ldc % 8)))
    return fail("alignment: N, lda, ldb, ldc must be multiples of 8");
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)C) & 15) return fail("pointers must be 16-byte aligned");
  int BN = block_n;
  if (BN == 0) BN = (N > 64) ? 128 : 64;
  if (BN != 64 && BN != 128 && BN != 256) return fail("block_n must be 64/128/256");
  // 128 is the widest tile whose accumulator image fits in shared memory next to the operand ring
  if (BN == 256) BN = 128;
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.num_m_blocks = (M + BLOCK_M - 1) / BLOCK_M;
  p.num_n_blocks = (N + BN - 1) / BN;
  p.num_k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  p.splits = splits < 1 ? 1 : splits;
  if (p.splits > p.num_k_blocks) p.splits = p.num_k_blocks;
  if (p.splits > 1 && out_mode != 1) return fail("split-K requires out_mode=1 (fp32 atomic add)");
  {  // no empty splits
    const int per = (p.num_k_blocks + p.splits - 1) / p.splits;
    p.splits = (p.num_k_blocks + per - 1) / per;
  }
  p.act = act; p.out_mode = out_mode; p.C = C; p.bias = bias_bf16; p.bias_f32 = bias_f32;
  p.residual = residual; p.preact = preact; p.alpha = alpha;
  p.stats = stats;
  p.res_mask = reinterpret_cast<const unsigned char*>(res_mask);
  if (res_mask != nullptr && (residual == nullptr || preact != nullptr || act > 2 || out_mode != 0 || (N % 64) ||
                              ldc != N))
    return fail("res_mask: plain bf16 residual, dense rows and N % 64 == 0 required");
  if (stats != nullptr && (N > STATS_MAX_N || out_mode != 0)) return fail("stats: N <= 2048 and bf16 output required");
  p.tma_store = (out_mode == 0) ? 1 : 0;
  // B (N x K bf16) small enough to live in the 50 MB L2 next to the in-flight A tiles -> walk N first
  p.n_fastest = ((size_t)N * (size_t)K * 2 <= ((size_t)20 << 20)) ? 1 : 0;
  CUtensorMap ma, mb, mc, mz;
  if (a_mn ? make_map(&ma, A, K, M, lda, BLOCK_K) : make_map(&ma, A, M, K, lda, BLOCK_M)) return -1;
  if (b_mn ? make_map(&mb, B, K, N, ldb, BLOCK_K) : make_map(&mb, B, N, K, ldb, BN)) return -1;
  if (p.tma_store) {
    if (make_map(&mc, C, M, N, ldc, 32)) return -1;
  } else {
    mc = ma;   // unused
  }
  if (p.tma_store && preact != nullptr) {
    if (make_map(&mz, preact, M, N, ldc, 32)) return -1;
  } else {
    mz = mc;   // unused
  }
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  p.splitk_ws = nullptr; p.splitk_count = nullptr; p.splitk_slice = 0;
  void* ws = nullptr;
  if (p.splits > 1) {
    p.splitk_slice = (long long)M * ldc;
    cudaError_t e = splitk_alloc(&ws, &p, p.num_m_blocks * p.num_n_blocks, st);
    if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  }
  const int rc = launch_bn(BN, a_mn, b_mn, ma, mb, mc, mz, p, max_ctas, st);
  if (ws != nullptr) {
    cudaError_t e = cudaFreeAsync(ws, st);
    if (e != cudaSuccess && rc == 0) return fail(cudaGetErrorString(e), (int)e);
  }
  return rc;
}

}  // extern "C"

// bf16 GEMM for sm_90a: TMA -> shared (128B swizzle) -> wgmma -> registers -> fused epilogue.
//
//   C[M,N] (+)= act( A[M,K] * B[N,K]^T + bias[N] ) + residual[M,N]
//
// A and B can each be K-major (row-major [rows][K]) or MN-major (stored [K][rows]), so the
// same kernel serves linear / 1x1-conv forward (A=x, B=W), dgrad (A=dy, B=W as MN-major) and
// wgrad (A=dy^T, B=x^T, both MN-major, split-K summed in split order) without any transpose pass:
// wgmma reads MN-major bf16 operands through its transpose flags.
//
// The kernel is persistent_body (sm90_common.cuh) over the output tiles (and K splits) of C, with
// cp.async.bulk.tensor.2d operand loads.
//
// This replaces the cuBLAS addmm / cuDNN 1x1-conv calls on the model zoo's hot path.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "sm90_common.cuh"

namespace {

// Work item w = split * tiles + tile (see persistent_body); GemmParams::n_fastest picks the tile order.
template <int BN, bool A_MN, bool B_MN>
struct GemmWork {
  static constexpr bool kStats = true, kSplitK = true;
  const CUtensorMap *a, *b, *c;
  const GemmParams& p;
  int tiles, items, kb_per_split;

  __device__ GemmWork(const CUtensorMap* a_, const CUtensorMap* b_, const CUtensorMap* c_, const GemmParams& p_)
      : a(a_), b(b_), c(c_), p(p_), tiles(p_.num_m_blocks * p_.num_n_blocks), items(tiles * p_.splits),
        kb_per_split((p_.num_k_blocks + p_.splits - 1) / p_.splits) {}
  __device__ void prefetch() const {
    tma_prefetch_desc(a);
    tma_prefetch_desc(b);
    if (p.out_mode == 0) tma_prefetch_desc(c);
  }
  __device__ int m_idx(int tile) const {
    return (p.n_fastest ? tile / p.num_n_blocks : tile % p.num_m_blocks) * BLOCK_M;
  }
  __device__ int n_idx(int tile) const { return (p.n_fastest ? tile % p.num_n_blocks : tile / p.num_m_blocks) * BN; }
  __device__ int num_kb(int w) const {
    const int kb0 = (w / tiles) * kb_per_split;
    return min(kb0 + kb_per_split, p.num_k_blocks) - kb0;
  }
  template <class Next>
  __device__ void load(int w, Next& next) const {
    const int tile = w % tiles;
    const int m0 = m_idx(tile), n0 = n_idx(tile);
    const int kb0 = (w / tiles) * kb_per_split;
    const int kb1 = min(kb0 + kb_per_split, p.num_k_blocks);
    for (int kb = kb0; kb < kb1; ++kb) {
      const Stage s = next();
      const int k_idx = kb * BLOCK_K;
      if (!A_MN) {
        tma_load_2d(a, s.bar, s.a, k_idx, m0);                                 // box {64 k, 128 m}
      } else {
#pragma unroll
        for (int c = 0; c < BLOCK_M / 64; ++c)                                  // box {64 m, 64 k}
          tma_load_2d(a, s.bar, s.a + c * (BLOCK_K * 128), m0 + 64 * c, k_idx);
      }
      if (!B_MN) {
        tma_load_2d(b, s.bar, s.b, k_idx, n0);                                 // box {64 k, BN n}
      } else {
#pragma unroll
        for (int c = 0; c < BN / 64; ++c)
          tma_load_2d(b, s.bar, s.b + c * (BLOCK_K * 128), n0 + 64 * c, k_idx);
      }
    }
  }
  __device__ Slab slab(int w, int q) const {
    const int tile = w % tiles, split = w / tiles;
    const int m0 = m_idx(tile);
    return Slab{c, m0 + q * 32, n_idx(tile), StoreAt{}, tile, m0, 0, split};
  }
};

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_c, const __grid_constant__ GemmParams p) {
  persistent_body<BN, A_MN, B_MN>(GemmWork<BN, A_MN, B_MN>(&map_a, &map_b, &map_c, p), p);
}

int launch_bn(int BN, int a_mn, int b_mn, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mc,
              const GemmParams& p, int max_ctas, cudaStream_t st) {
  const int work = p.num_m_blocks * p.num_n_blocks * p.splits;
#define LAUNCH(BNV, AMN, BMN) \
  launch_persistent<gemm_bf16_kernel<BNV, AMN, BMN>, BNV>(work, max_ctas, st, ma, mb, mc, p)
#define DISPATCH(BNV)                                          \
  if (BN == BNV) {                                             \
    if (!a_mn && !b_mn) return LAUNCH(BNV, false, false);      \
    if (!a_mn && b_mn) return LAUNCH(BNV, false, true);        \
    if (a_mn && !b_mn) return LAUNCH(BNV, true, false);        \
    return LAUNCH(BNV, true, true);                            \
  }
  DISPATCH(64)
  DISPATCH(128)
#undef DISPATCH
#undef LAUNCH
  return fail("unreachable");
}

}  // namespace

extern "C" {

const char* b200dp_gemm_last_error() { return g_err; }

// A: K-major -> [M][lda>=K]; MN-major -> [K][lda>=M].   B: K-major -> [N][ldb>=K]; MN-major -> [K][ldb>=N].
// C: [M][ldc>=N].  out_mode 0: bf16 = act(alpha*AB + bias) + residual; 1: C += alpha*AB; 2: C = alpha*AB, in
// C's dtype (out_bf16: bf16, else fp32), rounded once from fp32.  With splits > 1 (out_mode 1/2 only) the last
// split to finish a tile sums the partials of all splits in split order.
// Requirements: K % 8 == 0 for K-major operands, M % 8 (A) / N % 8 (B) == 0 for MN-major, N % 8 == 0,
// 16-byte aligned base pointers and leading dimensions.
int b200dp_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                     int a_mn, int b_mn, const void* bias_bf16, const void* bias_f32, const void* residual,
                     void* preact, int act, int out_mode, int out_bf16, float alpha, int splits, int block_n,
                     int max_ctas, float* stats, const void* res_mask, unsigned long long stream) {
  if (ensure_init()) return -1;
  if (M <= 0 || N <= 0 || K <= 0) return fail("bad shape");
  if ((N % 8) || (lda % 8) || (ldb % 8) || (ldc % 4) || ((out_mode == 0 || out_bf16) && (ldc % 8)))
    return fail("alignment: N, lda, ldb, ldc must be multiples of 8");
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)C) & 15) return fail("pointers must be 16-byte aligned");
  const int BN = pick_bn(N, block_n);
  if (BN < 0) return -1;
  GemmParams p{};
  p.M = M; p.N = N; p.ldc = ldc;
  p.num_m_blocks = (M + BLOCK_M - 1) / BLOCK_M;
  p.num_n_blocks = (N + BN - 1) / BN;
  p.num_k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  p.splits = normalize_splits(splits, p.num_k_blocks);
  if (p.splits > 1 && (out_mode == 0 || bias_bf16 || bias_f32 || residual || preact || act))
    return fail("split-K requires out_mode 1/2 without bias, residual or activation");
  p.act = act; p.out_mode = out_mode; p.c_bf16 = out_bf16 ? 1 : 0; p.C = C; p.bias = bias_bf16; p.bias_f32 = bias_f32;
  p.residual = residual; p.preact = preact; p.alpha = alpha;
  p.stats = stats;
  p.res_mask = reinterpret_cast<const unsigned char*>(res_mask);
  if (res_mask != nullptr && (residual == nullptr || preact != nullptr || act > 2 || out_mode != 0 || (N % 64) ||
                              ldc != N))
    return fail("res_mask: plain bf16 residual, dense rows and N % 64 == 0 required");
  if (stats != nullptr && (N > STATS_MAX_N || out_mode != 0)) return fail("stats: N <= 2048 and bf16 output required");
  // B (N x K bf16) small enough to live in the 50 MB L2 next to the in-flight A tiles -> walk N first
  p.n_fastest = ((size_t)N * (size_t)K * 2 <= ((size_t)20 << 20)) ? 1 : 0;
  CUtensorMap ma, mb, mc;
  if (a_mn ? make_map2(&ma, A, K, M, lda, BLOCK_K) : make_map2(&ma, A, M, K, lda, BLOCK_M)) return -1;
  if (b_mn ? make_map2(&mb, B, K, N, ldb, BLOCK_K) : make_map2(&mb, B, N, K, ldb, BN)) return -1;
  if (out_mode == 0) {
    if (make_map2(&mc, C, M, N, ldc, 32)) return -1;
  } else {
    mc = ma;   // unused
  }
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  if (p.splits > 1) p.splitk_slice = (long long)M * ldc;
  return run_splitk(p, p.num_m_blocks * p.num_n_blocks, st,
                    [&] { return launch_bn(BN, a_mn, b_mn, ma, mb, mc, p, max_ctas, st); });
}

}  // extern "C"

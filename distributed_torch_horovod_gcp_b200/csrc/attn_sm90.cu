// Flash attention for sm_90a (bf16, head dim 64, non-causal): forward and backward on wgmma.
//
//   O = softmax(Q K^T / sqrt(d)) V           per (batch, head); S x S scores never leave the SM.
//
// Forward, one CTA per (batch, head, 128-query tile), 288 threads:
//   warp 8          TMA producer: Q tile once, then K_0, V_0, K_1, V_1, ... through a 3-tile ring
//                   (4D tensor maps {64 d, S, H, B}: any [B,H,S,d] / [B,S,H,d] strided layout, rows >= S zero-filled)
//   warpgroups 0-1  64 query rows each (FlashAttention-2 on wgmma): S_j = Q K_j^T (m64n128k16, fp32 in
//                   registers), online softmax on the register fragment (row max / sum over the 4 lanes
//                   that share a row), P_j as bf16 into the K-major 128B-swizzled layout the next wgmma
//                   reads, O = alpha O + P_j V_j (m64n64k16, V as the MN-major operand straight from its
//                   [key][d] tile).  The running output never leaves the registers.
//
// Backward, one CTA per (batch, head, 128-key block) looping over the query tiles (FlashAttention-2
// order): S = Q_i K_j^T and dP = dO_i V_j^T per warpgroup (64 query rows each); P = exp2(S c - LSE),
// dS = P (dP - D) / sqrt(d) on the fragment -> bf16 smem; then each warpgroup owns 64 keys:
// dV_j += P^T dO_i, dK_j += dS^T Q_i (A operands = the SAME smem tiles read MN-major, no transposes,
// accumulators resident in registers across the query loop), and its 64 query rows of dQ_i = dS K_j go
// out as fp32 RED.ADDs into a workspace (the only cross-CTA reduction).
//
// Replaces F.scaled_dot_product_attention (cuDNN / flash library kernels) on the ViT-B/16 path.
// The reference application has no attention.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "sm90_common.cuh"

namespace {

constexpr int AT = 288;              // threads: warpgroups 0-1 wgmma + softmax, warp 8 TMA
constexpr int HD = 64;               // head dim
constexpr int TILE = 128;            // query rows / keys per block
constexpr int TILE_BYTES = TILE * HD * 2;   // 16 KB

struct AttnFwdParams {
  int B, H, S, q_tiles, kv_blocks;
  float scale_log2;                  // log2(e) / sqrt(d)
  __nv_bfloat16* o;
  long long o_sb, o_sh, o_ss;        // element strides of O (d contiguous)
  float* lse;                        // [B][H][S] natural-log sum-exp of the scaled scores (nullptr: not saved)
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void fence_async_cta() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One bf16 pair of a wgmma fragment (columns col, col + 1 of row `row`) into a K-major [rows][64] 128B-swizzled
// tile set: 64-column chunks `chunk_bytes` apart.
__device__ __forceinline__ void st_pair_sw(uint32_t base, int row, int col, int chunk_bytes, float lo, float hi) {
  uint32_t v;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(v) : "f"(hi), "f"(lo));
  const uint32_t a = base + (uint32_t)((col >> 6) * chunk_bytes + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) +
                                       ((col & 7) << 1));
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  uint32_t v;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(v) : "f"(hi), "f"(lo));
  return v;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ---------------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------------
constexpr int FW_RING = 3;
constexpr int FW_SMEM = TILE_BYTES * (1 + FW_RING) + 2 * TILE_BYTES /*P*/ + 1024 + 256;

// Fragment of an m64 x N wgmma accumulator held by thread t of a warpgroup: element 4j + e is row
// 16 (t / 32) + (t % 32) / 4 + 8 (e / 2), column 8 j + 2 (t % 4) + e % 2.
__global__ void __launch_bounds__(AT, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                const __grid_constant__ CUtensorMap map_v, const AttnFwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sT = smem + TILE_BYTES;                       // ring of K / V tiles
  uint8_t* sP = sT + FW_RING * TILE_BYTES;               // 2 chunks (64 keys each) x [128 rows x 128 B]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sP + 2 * TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                          // [3]
  uint64_t* kv_empty = bars + 4;                         // [3]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x % p.q_tiles;
  const int bh = blockIdx.x / p.q_tiles;
  const int h = bh % p.H, b = bh / p.H;
  const int nb = p.kv_blocks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < FW_RING; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);                        // one arrival per warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (elect_one()) {
      mbar_expect_tx(q_full, TILE_BYTES);
      tma_load_4d(&map_q, q_full, sQ, 0, qt * TILE, h, b);
      for (int t = 0; t < 2 * nb; ++t) {
        const int st = t % FW_RING;
        mbar_wait(&kv_empty[st], ((t / FW_RING) & 1) ^ 1);
        mbar_expect_tx(&kv_full[st], TILE_BYTES);
        tma_load_4d((t & 1) ? &map_v : &map_k, &kv_full[st], sT + st * TILE_BYTES, 0, (t >> 1) * TILE, h, b);
      }
    }
  } else {
    const int wg = warp >> 2;                            // query rows 64 wg .. 64 wg + 63 of the tile
    const int t128 = threadIdx.x & 127;
    const int r0 = 64 * wg + (t128 >> 5) * 16 + (lane >> 2);   // tile rows of fragment elements e = 0,1 | 2,3: r0, r0 + 8
    const int cq = 2 * (lane & 3);
    const bool leader = t128 == 0;
    const uint64_t kmaj = make_desc_base(16, 1024);
    const uint64_t mnmaj = make_desc_base(BLOCK_K * 128, 1024);
    const uint64_t dq = kmaj + desc_addr(smem_u32(sQ) + (uint32_t)wg * 8192u);
    const uint32_t sT_u = smem_u32(sT), sP_u = smem_u32(sP);
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    mbar_wait(q_full, 0);
    for (int j = 0; j < nb; ++j) {
      const int valid = min(TILE, p.S - j * TILE);
      // ---- S_j = Q K_j^T
      int t = 2 * j, st = t % FW_RING;
      mbar_wait(&kv_full[st], (t / FW_RING) & 1);
      float sc[TILE / 2];
      {
        const uint64_t dk = kmaj + desc_addr(sT_u + st * TILE_BYTES);
        wg_fence();
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) wgmma_bf16<128, false, false>(sc, dq + 2 * k, dk + 2 * k, k ? 1u : 0u);
        wg_commit();
        wg_wait<0>();
        wg_fence_operands<TILE / 2>(sc);
      }
      if (leader) mbar_arrive(&kv_empty[st]);
      // ---- online softmax on the fragment
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int jj = 0; jj < TILE / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (8 * jj + cq + (e & 1) < valid) mx[e >> 1] = fmaxf(mx[e >> 1], sc[4 * jj + e]);
      float mn[2], alpha[2];
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        mn[h2] = fmaxf(m[h2], quad_max(mx[h2]) * p.scale_log2);
        alpha[h2] = (m[h2] == -INFINITY) ? 0.f : ex2(m[h2] - mn[h2]);
        m[h2] = mn[h2];
        l[h2] *= alpha[h2];
      }
#pragma unroll
      for (int jj = 0; jj < TILE / 8; ++jj) {
        float pe[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          pe[e] = (8 * jj + cq + (e & 1) < valid) ? ex2(fmaf(sc[4 * jj + e], p.scale_log2, -mn[e >> 1])) : 0.f;
          l[e >> 1] += pe[e];
        }
        st_pair_sw(sP_u, r0, 8 * jj + cq, TILE_BYTES, pe[0], pe[1]);
        st_pair_sw(sP_u, r0 + 8, 8 * jj + cq, TILE_BYTES, pe[2], pe[3]);
      }
#pragma unroll
      for (int i = 0; i < HD / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      fence_async_cta();                                 // P (generic stores) -> wgmma operand reads
      named_bar(1 + wg, 128);
      // ---- O += P_j V_j
      t = 2 * j + 1; st = t % FW_RING;
      mbar_wait(&kv_full[st], (t / FW_RING) & 1);
      {
        const uint64_t dv = mnmaj + desc_addr(sT_u + st * TILE_BYTES);
        wg_fence();
#pragma unroll
        for (int k = 0; k < TILE / 16; ++k) {
          const uint64_t dp = kmaj + desc_addr(sP_u + (k >> 2) * TILE_BYTES + (uint32_t)wg * 8192u + (k & 3) * 32);
          wgmma_bf16<64, false, true>(o, dp, dv + (uint64_t)(k * 128), 1u);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_operands<HD / 2>(o);
      }
      if (leader) mbar_arrive(&kv_empty[st]);
    }
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      const float lt = quad_sum(l[h2]);
      const int qrow = qt * TILE + r0 + 8 * h2;
      if (qrow < p.S) {
        const float inv = __fdividef(1.0f, lt);
        uint32_t* dst = reinterpret_cast<uint32_t*>(p.o + (size_t)b * p.o_sb + (size_t)h * p.o_sh + (size_t)qrow * p.o_ss);
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
          dst[(8 * jj + cq) >> 1] = pack2(o[4 * jj + 2 * h2] * inv, o[4 * jj + 2 * h2 + 1] * inv);
        if (p.lse != nullptr && (lane & 3) == 0)
          p.lse[((size_t)b * p.H + h) * p.S + qrow] = (m[h2] + log2f(lt)) * 0.6931471805599453f;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------------
struct AttnBwdParams {
  int B, H, S, q_tiles, kv_blocks;
  float scale_log2, scale;
  const float* lse;                  // [B][H][S]
  const float* delta;                // [B][H][S]  rowsum(dO * O)
  float* dq_acc;                     // fp32, zero on entry; element strides dq_sb / dq_sh / dq_ss (64 contiguous)
  long long dq_sb, dq_sh, dq_ss;
  __nv_bfloat16* dk; __nv_bfloat16* dv;
  long long dk_sb, dk_sh, dk_ss, dv_sb, dv_sh, dv_ss;
};

// delta[b][h][s] = sum_d dO * O   (8 lanes per row: one 16-byte load of each tensor per lane)
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ o,
                                                         const __nv_bfloat16* __restrict__ dout,
                                                         float* __restrict__ delta, int B, int H, int S, long long o_sb,
                                                         long long o_sh, long long o_ss, long long d_sb, long long d_sh,
                                                         long long d_ss) {
  const unsigned total = (unsigned)B * (unsigned)H * (unsigned)S;
  const unsigned row = blockIdx.x * 32u + (threadIdx.x >> 3);
  const int sub = threadIdx.x & 7;
  float v = 0.f;
  if (row < total) {
    const unsigned s = row % (unsigned)S;
    const unsigned bh = row / (unsigned)S;
    const unsigned h = bh % (unsigned)H, b = bh / (unsigned)H;
    const uint4 ov = *reinterpret_cast<const uint4*>(o + b * o_sb + h * o_sh + s * o_ss + sub * 8);
    const uint4 dv = *reinterpret_cast<const uint4*>(dout + b * d_sb + h * d_sh + s * d_ss + sub * 8);
    float a[8], c[8];
    unpack8(ov, a);
    unpack8(dv, c);
#pragma unroll
    for (int i = 0; i < 8; ++i) v = fmaf(a[i], c[i], v);
  }
#pragma unroll
  for (int off = 4; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if (sub == 0 && row < total) delta[row] = v;
}

// smem: K_j, V_j (resident), ring of 2 x {Q_i, dO_i}, P (32 KB), dS (32 KB)
constexpr int BW_RING = 2;
constexpr int BW_SMEM = TILE_BYTES * (2 + 2 * BW_RING) + 4 * TILE_BYTES + 1024 + 256;

__global__ void __launch_bounds__(AT, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_do,
                const AttnBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sK = smem;
  uint8_t* sV = smem + TILE_BYTES;
  uint8_t* sR = sV + TILE_BYTES;                         // ring: [stage][Q | dO]
  uint8_t* sP = sR + 2 * BW_RING * TILE_BYTES;           // P  [128 q rows][128 keys] bf16, 2 chunks
  uint8_t* sS = sP + 2 * TILE_BYTES;                     // dS same layout
  uint64_t* bars = reinterpret_cast<uint64_t*>(sS + 2 * TILE_BYTES);
  uint64_t* kv_full = bars;
  uint64_t* r_full = bars + 1;                           // [2]
  uint64_t* r_empty = bars + 3;                          // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb = blockIdx.x % p.kv_blocks;
  const int bh = blockIdx.x / p.kv_blocks;
  const int h = bh % p.H, b = bh / p.H;
  const int nq = p.q_tiles;
  const int kvalid = min(TILE, p.S - kb * TILE);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    tma_prefetch_desc(&map_do);
    mbar_init(kv_full, 1);
    for (int i = 0; i < BW_RING; ++i) {
      mbar_init(&r_full[i], 1);
      mbar_init(&r_empty[i], 2);                         // one arrival per warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (elect_one()) {
      mbar_expect_tx(kv_full, 2 * TILE_BYTES);
      tma_load_4d(&map_k, kv_full, sK, 0, kb * TILE, h, b);
      tma_load_4d(&map_v, kv_full, sV, 0, kb * TILE, h, b);
      for (int i = 0; i < nq; ++i) {
        const int st = i % BW_RING;
        mbar_wait(&r_empty[st], ((i / BW_RING) & 1) ^ 1);
        mbar_expect_tx(&r_full[st], 2 * TILE_BYTES);
        tma_load_4d(&map_q, &r_full[st], sR + (2 * st) * TILE_BYTES, 0, i * TILE, h, b);
        tma_load_4d(&map_do, &r_full[st], sR + (2 * st + 1) * TILE_BYTES, 0, i * TILE, h, b);
      }
    }
  } else {
    // warpgroup wg: query rows 64 wg .. +63 of every Q tile (S, dP, dQ) and keys 64 wg .. +63 (dK, dV)
    const int wg = warp >> 2;
    const int t128 = threadIdx.x & 127;
    const int r0 = 64 * wg + (t128 >> 5) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const bool leader = t128 == 0;
    const uint64_t kmaj = make_desc_base(16, 1024);
    const uint64_t mnmaj = make_desc_base(BLOCK_K * 128, 1024);
    const uint32_t sP_u = smem_u32(sP), sS_u = smem_u32(sS);
    const uint64_t dK_k = kmaj + desc_addr(smem_u32(sK));      // K_j as K-major B (N = keys, K = d)
    const uint64_t dV_k = kmaj + desc_addr(smem_u32(sV));      // V_j as K-major B
    const uint64_t dK_mn = mnmaj + desc_addr(smem_u32(sK));    // K_j as MN-major B (N = d, K = keys)
    // P / dS as MN-major A (M = this warpgroup's 64 keys = chunk wg, K = q rows 128 B apart)
    const uint64_t aP = mnmaj + desc_addr(sP_u + (uint32_t)wg * TILE_BYTES);
    const uint64_t aS = mnmaj + desc_addr(sS_u + (uint32_t)wg * TILE_BYTES);
    const size_t bh_off = ((size_t)b * p.H + h) * p.S;
    float dv[HD / 2], dk[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
    mbar_wait(kv_full, 0);
    for (int i = 0; i < nq; ++i) {
      const int st = i % BW_RING;
      const uint32_t sQ_u = smem_u32(sR + (2 * st) * TILE_BYTES), sO_u = sQ_u + TILE_BYTES;
      mbar_wait(&r_full[st], (i / BW_RING) & 1);
      // ---- S = Q_i K_j^T, dP = dO_i V_j^T for this warpgroup's 64 query rows
      float sc[TILE / 2], dp[TILE / 2];
      {
        const uint64_t aq = kmaj + desc_addr(sQ_u + (uint32_t)wg * 8192u);
        const uint64_t ao = kmaj + desc_addr(sO_u + (uint32_t)wg * 8192u);
        wg_fence();
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) wgmma_bf16<128, false, false>(sc, aq + 2 * k, dK_k + 2 * k, k ? 1u : 0u);
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) wgmma_bf16<128, false, false>(dp, ao + 2 * k, dV_k + 2 * k, k ? 1u : 0u);
        wg_commit();
        wg_wait<0>();
        wg_fence_operands<TILE / 2>(sc);
        wg_fence_operands<TILE / 2>(dp);
      }
      // ---- P = exp2(S c - LSE), dS = P (dP - D) / sqrt(d) -> bf16 smem
      float lse2[2], dl[2];
      bool qok[2];
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int qrow = i * TILE + r0 + 8 * h2;
        qok[h2] = qrow < p.S;
        lse2[h2] = qok[h2] ? p.lse[bh_off + qrow] * 1.4426950408889634f : 0.f;
        dl[h2] = qok[h2] ? p.delta[bh_off + qrow] : 0.f;
      }
#pragma unroll
      for (int jj = 0; jj < TILE / 8; ++jj) {
        float pv[4], ds[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int h2 = e >> 1;
          const bool ok = qok[h2] && (8 * jj + cq + (e & 1) < kvalid);
          const float pe = ok ? ex2(fmaf(sc[4 * jj + e], p.scale_log2, -lse2[h2])) : 0.f;
          pv[e] = pe;
          ds[e] = pe * (dp[4 * jj + e] - dl[h2]) * p.scale;
        }
        st_pair_sw(sP_u, r0, 8 * jj + cq, TILE_BYTES, pv[0], pv[1]);
        st_pair_sw(sP_u, r0 + 8, 8 * jj + cq, TILE_BYTES, pv[2], pv[3]);
        st_pair_sw(sS_u, r0, 8 * jj + cq, TILE_BYTES, ds[0], ds[1]);
        st_pair_sw(sS_u, r0 + 8, 8 * jj + cq, TILE_BYTES, ds[2], ds[3]);
      }
      fence_async_cta();
      named_bar(1, 256);                                 // P / dS of all 128 query rows are in smem
      // ---- dV += P^T dO_i, dK += dS^T Q_i (this warpgroup's 64 keys); dQ_i = dS K_j (its 64 query rows)
      float dqv[HD / 2];
      {
        const uint64_t bO = mnmaj + desc_addr(sO_u), bQ = mnmaj + desc_addr(sQ_u);
        wg_fence();
#pragma unroll
        for (int k = 0; k < TILE / 16; ++k) wgmma_bf16<64, true, true>(dv, aP + k * 128, bO + k * 128, 1u);
#pragma unroll
        for (int k = 0; k < TILE / 16; ++k) wgmma_bf16<64, true, true>(dk, aS + k * 128, bQ + k * 128, 1u);
#pragma unroll
        for (int k = 0; k < TILE / 16; ++k) {
          const uint64_t da = kmaj + desc_addr(sS_u + (k >> 2) * TILE_BYTES + (uint32_t)wg * 8192u + (k & 3) * 32);
          wgmma_bf16<64, false, true>(dqv, da, dK_mn + (uint64_t)(k * 128), k ? 1u : 0u);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_operands<HD / 2>(dv);
        wg_fence_operands<HD / 2>(dk);
        wg_fence_operands<HD / 2>(dqv);
      }
      if (leader) mbar_arrive(&r_empty[st]);
      // ---- dQ_i -> fp32 RED.ADD into the workspace
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        if (qok[h2]) {
          float* dst = p.dq_acc + (size_t)b * p.dq_sb + (size_t)h * p.dq_sh + (size_t)(i * TILE + r0 + 8 * h2) * p.dq_ss;
#pragma unroll
          for (int jj = 0; jj < HD / 8; ++jj)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + 8 * jj + cq), "f"(dqv[4 * jj + 2 * h2]),
                         "f"(dqv[4 * jj + 2 * h2 + 1])
                         : "memory");
        }
      }
      named_bar(1, 256);                                 // both warpgroups are done reading P / dS
    }
    // ---- dK_j, dV_j: rows = keys 64 wg ..
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      const int krow = kb * TILE + r0 + 8 * h2;
      if (krow < p.S) {
        uint32_t* pk = reinterpret_cast<uint32_t*>(p.dk + (size_t)b * p.dk_sb + (size_t)h * p.dk_sh + (size_t)krow * p.dk_ss);
        uint32_t* pv = reinterpret_cast<uint32_t*>(p.dv + (size_t)b * p.dv_sb + (size_t)h * p.dv_sh + (size_t)krow * p.dv_ss);
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj) {
          pk[(8 * jj + cq) >> 1] = pack2(dk[4 * jj + 2 * h2], dk[4 * jj + 2 * h2 + 1]);
          pv[(8 * jj + cq) >> 1] = pack2(dv[4 * jj + 2 * h2], dv[4 * jj + 2 * h2 + 1]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
thread_local char g_err[512];

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
  return 0;
}
// {64 d, S, H, B} view with element strides (ss, sh, sb); box {64, 128, 1, 1}
int make_qkv_map(CUtensorMap* m, const void* ptr, int B, int H, int S, long long sb, long long sh, long long ss) {
  if ((ss % 8) || (sh % 8) || (sb % 8) || ((uintptr_t)ptr & 15)) return fail("attention operands must be 16-byte aligned");
  cuuint64_t dims[4] = {(cuuint64_t)HD, (cuuint64_t)S, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)ss * 2, (cuuint64_t)sh * 2, (cuuint64_t)sb * 2};
  cuuint32_t box[4] = {64, TILE, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(attention) failed", (int)r);
  return 0;
}

}  // namespace

extern "C" {

const char* b200dp_attn_last_error() { return g_err; }

// strides: element strides {batch, head, seq} of each tensor (head dim 64 contiguous)
int b200dp_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int S, int D,
                    const long long* qs, const long long* ks, const long long* vs, const long long* os, float scale,
                    unsigned long long stream) {
  if (ensure_init()) return -1;
  if (D != HD) return fail("head dim must be 64");
  CUtensorMap mq, mk, mv;
  if (make_qkv_map(&mq, q, B, H, S, qs[0], qs[1], qs[2]) || make_qkv_map(&mk, k, B, H, S, ks[0], ks[1], ks[2]) ||
      make_qkv_map(&mv, v, B, H, S, vs[0], vs[1], vs[2]))
    return -1;
  if ((os[0] % 8) || (os[1] % 8) || (os[2] % 8) || ((uintptr_t)o & 15)) return fail("output must be 16-byte aligned");
  AttnFwdParams p;
  p.B = B; p.H = H; p.S = S;
  p.q_tiles = (S + TILE - 1) / TILE;
  p.kv_blocks = (S + TILE - 1) / TILE;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_sb = os[0]; p.o_sh = os[1]; p.o_ss = os[2];
  p.lse = lse;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FW_SMEM);
    if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
    attr_set = true;
  }
  attn_fwd_kernel<<<B * H * p.q_tiles, AT, FW_SMEM, (cudaStream_t)(uintptr_t)stream>>>(mq, mk, mv, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  return 0;
}

// dq_acc: fp32 workspace (strides dqs, 64 contiguous) zeroed by the caller; delta: [B][H][S] fp32 workspace
int b200dp_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                    float* delta, float* dq_acc, void* dk, void* dv, int B, int H, int S, int D, const long long* qs,
                    const long long* ks, const long long* vs, const long long* os, const long long* dos,
                    const long long* dqs, const long long* dks, const long long* dvs, float scale,
                    unsigned long long stream) {
  if (ensure_init()) return -1;
  if (D != HD) return fail("head dim must be 64");
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  CUtensorMap mq, mk, mv, mdo;
  if (make_qkv_map(&mq, q, B, H, S, qs[0], qs[1], qs[2]) || make_qkv_map(&mk, k, B, H, S, ks[0], ks[1], ks[2]) ||
      make_qkv_map(&mv, v, B, H, S, vs[0], vs[1], vs[2]) || make_qkv_map(&mdo, dout, B, H, S, dos[0], dos[1], dos[2]))
    return -1;
  const long long rows = (long long)B * H * S;
  attn_delta_kernel<<<(unsigned)((rows + 31) / 32), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(o), reinterpret_cast<const __nv_bfloat16*>(dout), delta, B, H, S, os[0],
      os[1], os[2], dos[0], dos[1], dos[2]);
  AttnBwdParams p;
  p.B = B; p.H = H; p.S = S;
  p.q_tiles = (S + TILE - 1) / TILE;
  p.kv_blocks = (S + TILE - 1) / TILE;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.lse = lse; p.delta = delta; p.dq_acc = dq_acc;
  p.dq_sb = dqs[0]; p.dq_sh = dqs[1]; p.dq_ss = dqs[2];
  if ((dqs[0] % 4) || (dqs[1] % 4) || (dqs[2] % 4)) return fail("dq workspace strides must be multiples of 4");
  p.dk = reinterpret_cast<__nv_bfloat16*>(dk); p.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  p.dk_sb = dks[0]; p.dk_sh = dks[1]; p.dk_ss = dks[2];
  p.dv_sb = dvs[0]; p.dv_sh = dvs[1]; p.dv_ss = dvs[2];
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM);
    if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
    attr_set = true;
  }
  attn_bwd_kernel<<<B * H * p.kv_blocks, AT, BW_SMEM, st>>>(mq, mk, mv, mdo, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  return 0;
}

}  // extern "C"

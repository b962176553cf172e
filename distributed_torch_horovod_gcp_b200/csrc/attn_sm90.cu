// Flash attention for sm_90a (bf16, head dim 64, optionally causal): forward and backward on wgmma.
//
//   O = softmax(Q K^T / sqrt(d) [+ causal mask]) V     per (batch, head); S x S scores never leave the SM.
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
// Causal (CAUSAL = true, query i sees keys 0..i): query and key tiles are both 128 wide, so only the
// diagonal tile is partly masked.  Forward query tile qt visits KV tiles 0..qt; backward KV block kb visits
// query tiles kb..q_tiles-1; on the diagonal tile a key column past the query row is dropped wherever the
// sequence-tail mask drops columns (row max, P, dS), so masked products are exact zeros.  The causal grids
// launch the longest tiles first.
//
// Dropout (DROPOUT = true, probability p > 0; p = 0 launches the DROPOUT = false kernels):
//   O = (Z o P) V with P the softmax and Z = keep / q, keep in {0, 1}, q = t / 2^16 the keep probability,
//   t = round((1 - p) 2^16) (philox.cuh: p has a resolution of 2^-16; t = 0, i.e. p = 1, gives scale 0 and
//   exact zeros).  Forward: the row sum l and the saved LSE are the un-dropped ones, the P tile that feeds the
//   PV wgmma is keep ? P : 0, and 1/q = 2^16 / t is folded into the final 1 / l multiply.  Backward, with the
//   same bits recomputed: dV += (keep o P)^T dO, scaled by 1/q once at the end; dS = P o (Z o dP - D) / sqrt(d),
//   where D = rowsum(dO o O) of the dropped O (= rowsum(P o Z o dP)), so attn_delta_kernel is unchanged.
//
//   The mask.  Each (b, h, query row r, key column c) has one keep bit, a pure function of the 128-bit seed
//   (seed[0], seed[1] in device memory, drawn by torch's CUDA generator) and of (b, h, r, c) alone, so it
//   does not depend on tiles, grid, strides or CAUSAL:
//     u    = Philox4x32-10(key = (seed[0] mod 2^32, seed[0] / 2^32),
//                          counter = (4 (c / 16) + (c mod 8) / 2,  8 (r / 16) + r mod 8,  b H + h,  seed[1] mod 2^32))
//     word = u[2 ((r / 8) mod 2) + (c / 8) mod 2]           (u[0..3] = the four 32-bit outputs)
//     bits = (c mod 2) ? word >> 16 : word mod 2^16
//     keep = bits < t
//   One Philox call covers rows {r, r + 8} x columns {c, c + 1, c + 8, c + 9} (r mod 16 < 8, c mod 16 < 8,
//   c even): exactly the 8 elements one thread holds for fragment column pairs jj = 2m, 2m + 1 (see the
//   fragment layout above attn_fwd_kernel; S = Q K^T has the same layout in the backward), so each thread
//   draws each Philox output once: 8 calls per 128 x 128 tile.
//
// Sequence parallelism (SP = true; CAUSAL or not, never DROPOUT): "rank r of W" holds a zigzag shard of the
// sequence.  The global sequence is 2W chunks of c tiles (S_glob = 2 W c 128); rank r holds chunks r and
// 2W - 1 - r, in that order, as its local rows (S_loc = 2 c 128), so under the causal mask every rank has the
// same number of (query tile, key tile) pairs.  zz_global / zz_local map a local tile to its global tile and
// back.  The operands owned by other ranks arrive as gathered [W][B][S_loc][H][64] views (what an all-gather
// of each rank's tensor delivers), loaded through 5D tensor maps {64 d, S_loc, H, B, W}; the kernels reach other
// ranks' data only through those buffers (no peer pointers, no barriers), so one GPU can run any rank.
//   Forward: one CTA per (batch, head, local query tile) visits the key tiles in global order (0..its global
//   tile when causal) from the gathered K / V; the mask is on global positions.  Each CTA computes exactly
//   what the full-sequence kernel computes for that query tile, so O and LSE are bit-identical to it.
//   Backward: one CTA per (batch, head, local key block) loops over the query tiles of all ranks in global
//   order, reading the gathered Q, dO, LSE and delta, so dK / dV are bit-identical to the full-sequence
//   kernel's; dQ partials go by fp32 RED.ADD into a [W][B][S_loc][H][64] workspace (row block of each query's
//   owner), which the caller reduce-scatters.
//
// Replaces F.scaled_dot_product_attention (cuDNN / flash library kernels) on the ViT-B/16 and GPT paths.
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
  const unsigned long long* seed;    // DROPOUT: Philox key, offset (2 words in device memory)
  uint32_t drop_thr;                 // DROPOUT: keep when the element's 16 bits are below this (t)
  float drop_scale;                  // DROPOUT: 2^16 / t (0 when t = 0)
  int sp_rank, sp_world, sp_c;       // SP: this rank, the world, tiles per zigzag chunk
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
// SP zigzag map (see the header): global tile of local tile lt on rank r, and owner / local tile of global tile g.
__device__ __forceinline__ int zz_global(int lt, int r, int W, int c) {
  return lt < c ? r * c + lt : (2 * W - 1 - r) * c + (lt - c);
}
__device__ __forceinline__ void zz_local(int g, int W, int c, int& r, int& lt) {
  const int ch = g / c, w = g - ch * c;
  r = ch < W ? ch : 2 * W - 1 - ch;
  lt = ch < W ? w : c + w;
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], "
      "[%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Dropout bits (see the header): the Philox output for query rows {row, row + 8} (row = the global row of the
// thread's r0) and key columns col + cq + {0, 1, 8, 9} (col = the global column of fragment pair jj, jj even).
__device__ __forceinline__ uint4 drop_draw(const unsigned long long* seed, int bh, int row, int col, int cq) {
  const unsigned long long k = seed[0];
  const uint32_t off = (uint32_t)seed[1];
  return philox4x32_10(make_uint4((uint32_t)((col >> 4) * 4 + (cq >> 1)), (uint32_t)((row >> 4) * 8 + (row & 7)),
                                  (uint32_t)bh, off),
                       make_uint2((uint32_t)k, (uint32_t)(k >> 32)));
}
// Keep bit of fragment element 4 jj + e from the draw of pair 2 (jj / 2): row r0 + 8 (e / 2), column
// 8 jj + cq + e % 2 -> word 2 (e / 2) + jj % 2, low / high 16 bits for e % 2 = 0 / 1.
__device__ __forceinline__ bool drop_keep(const uint4& u, int jj, int e, uint32_t thr) {
  const int w = 2 * (e >> 1) + (jj & 1);
  const uint32_t word = w == 0 ? u.x : w == 1 ? u.y : w == 2 ? u.z : u.w;
  return ((e & 1) ? word >> 16 : word & 0xffffu) < thr;
}

// ---------------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------------
constexpr int FW_RING = 3;
constexpr int FW_SMEM = TILE_BYTES * (1 + FW_RING) + 2 * TILE_BYTES /*P*/ + 1024 + 256;

// Fragment of an m64 x N wgmma accumulator held by thread t of a warpgroup: element 4j + e is row
// 16 (t / 32) + (t % 32) / 4 + 8 (e / 2), column 8 j + 2 (t % 4) + e % 2.
template <bool CAUSAL, bool DROPOUT, bool SP = false>
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
  const int BH = p.B * p.H;
  const int qt = CAUSAL ? p.q_tiles - 1 - blockIdx.x / BH : blockIdx.x % p.q_tiles;
  const int bh = CAUSAL ? blockIdx.x % BH : blockIdx.x / p.q_tiles;
  const int h = bh % p.H, b = bh / p.H;
  static_assert(!(SP && DROPOUT), "no dropout under sequence parallelism");
  const int qg = SP ? zz_global(qt, p.sp_rank, p.sp_world, p.sp_c) : qt;   // global query tile (SP: local qt)
  const int nb = CAUSAL ? qg + 1 : p.kv_blocks;

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
        if constexpr (SP) {
          int r, lt;
          zz_local(t >> 1, p.sp_world, p.sp_c, r, lt);
          tma_load_5d((t & 1) ? &map_v : &map_k, &kv_full[st], sT + st * TILE_BYTES, 0, lt * TILE, h, b, r);
        } else {
          tma_load_4d((t & 1) ? &map_v : &map_k, &kv_full[st], sT + st * TILE_BYTES, 0, (t >> 1) * TILE, h, b);
        }
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
      const int valid = SP ? TILE : min(TILE, p.S - j * TILE);   // SP: S_loc is a multiple of 2 tiles
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
      const bool diag = CAUSAL && j == qg;                // causal diagonal tile: key column <= query row
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int jj = 0; jj < TILE / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (8 * jj + cq + (e & 1) < valid && (!diag || 8 * jj + cq + (e & 1) <= r0 + 8 * (e >> 1)))
            mx[e >> 1] = fmaxf(mx[e >> 1], sc[4 * jj + e]);
      float mn[2], alpha[2];
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        mn[h2] = fmaxf(m[h2], quad_max(mx[h2]) * p.scale_log2);
        alpha[h2] = (m[h2] == -INFINITY) ? 0.f : ex2(m[h2] - mn[h2]);
        m[h2] = mn[h2];
        l[h2] *= alpha[h2];
      }
      uint4 rnd;
#pragma unroll
      for (int jj = 0; jj < TILE / 8; ++jj) {
        if constexpr (DROPOUT) {
          if ((jj & 1) == 0) rnd = drop_draw(p.seed, bh, qt * TILE + r0, j * TILE + 8 * jj, cq);
        }
        float pe[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          pe[e] = (8 * jj + cq + (e & 1) < valid && (!diag || 8 * jj + cq + (e & 1) <= r0 + 8 * (e >> 1)))
                      ? ex2(fmaf(sc[4 * jj + e], p.scale_log2, -mn[e >> 1])) : 0.f;
          l[e >> 1] += pe[e];
          if constexpr (DROPOUT) {
            if (!drop_keep(rnd, jj, e, p.drop_thr)) pe[e] = 0.f;   // l keeps the un-dropped sum
          }
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
        const float inv = __fdividef(1.0f, lt) * (DROPOUT ? p.drop_scale : 1.0f);   // dropout: 1/q folded in
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
  const unsigned long long* seed;    // DROPOUT: as in AttnFwdParams
  uint32_t drop_thr;
  float drop_scale;
  int sp_rank, sp_world, sp_c;       // SP: as in AttnFwdParams
  long long lse_sw, dq_sw;           // SP: rank strides (elements) of the gathered lse / delta and of dq_acc
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

template <bool CAUSAL, bool DROPOUT, bool SP = false>
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
  const int BH = p.B * p.H;
  const int kb = CAUSAL ? blockIdx.x / BH : blockIdx.x % p.kv_blocks;
  const int bh = CAUSAL ? blockIdx.x % BH : blockIdx.x / p.kv_blocks;
  const int h = bh % p.H, b = bh / p.H;
  const int nq = p.q_tiles;
  static_assert(!(SP && DROPOUT), "no dropout under sequence parallelism");
  const int kg = SP ? zz_global(kb, p.sp_rank, p.sp_world, p.sp_c) : kb;   // global key block (SP: local kb)
  const int i0 = CAUSAL ? kg : 0;                        // first query tile that sees this key block
  const int kvalid = SP ? TILE : min(TILE, p.S - kb * TILE);

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
      for (int i = i0; i < nq; ++i) {
        const int st = (i - i0) % BW_RING;
        mbar_wait(&r_empty[st], (((i - i0) / BW_RING) & 1) ^ 1);
        mbar_expect_tx(&r_full[st], 2 * TILE_BYTES);
        if constexpr (SP) {
          int r, lt;
          zz_local(i, p.sp_world, p.sp_c, r, lt);
          tma_load_5d(&map_q, &r_full[st], sR + (2 * st) * TILE_BYTES, 0, lt * TILE, h, b, r);
          tma_load_5d(&map_do, &r_full[st], sR + (2 * st + 1) * TILE_BYTES, 0, lt * TILE, h, b, r);
        } else {
          tma_load_4d(&map_q, &r_full[st], sR + (2 * st) * TILE_BYTES, 0, i * TILE, h, b);
          tma_load_4d(&map_do, &r_full[st], sR + (2 * st + 1) * TILE_BYTES, 0, i * TILE, h, b);
        }
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
    for (int i = i0; i < nq; ++i) {
      const int st = (i - i0) % BW_RING;
      const uint32_t sQ_u = smem_u32(sR + (2 * st) * TILE_BYTES), sO_u = sQ_u + TILE_BYTES;
      mbar_wait(&r_full[st], ((i - i0) / BW_RING) & 1);
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
      const bool diag = CAUSAL && i == kg;                // causal diagonal tile: key column <= query row
      int qr = 0, ql = i;                                // SP: the owner of query tile i and its local tile there
      if constexpr (SP) zz_local(i, p.sp_world, p.sp_c, qr, ql);
      const size_t row_off = SP ? (size_t)qr * p.lse_sw + bh_off : bh_off;
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int qrow = ql * TILE + r0 + 8 * h2;
        qok[h2] = qrow < p.S;
        lse2[h2] = qok[h2] ? p.lse[row_off + qrow] * 1.4426950408889634f : 0.f;
        dl[h2] = qok[h2] ? p.delta[row_off + qrow] : 0.f;
      }
      uint4 rnd;
#pragma unroll
      for (int jj = 0; jj < TILE / 8; ++jj) {
        if constexpr (DROPOUT) {
          if ((jj & 1) == 0) rnd = drop_draw(p.seed, bh, i * TILE + r0, kb * TILE + 8 * jj, cq);
        }
        float pv[4], ds[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int h2 = e >> 1;
          const bool ok = qok[h2] && (8 * jj + cq + (e & 1) < kvalid) && (!diag || 8 * jj + cq + (e & 1) <= r0 + 8 * h2);
          const float pe = ok ? ex2(fmaf(sc[4 * jj + e], p.scale_log2, -lse2[h2])) : 0.f;
          if constexpr (DROPOUT) {
            // dV takes keep o P (1/q applied at the end); dS = P (Z dP - D) / sqrt(d)
            const bool kp = drop_keep(rnd, jj, e, p.drop_thr);
            pv[e] = kp ? pe : 0.f;
            ds[e] = pe * ((kp ? dp[4 * jj + e] * p.drop_scale : 0.f) - dl[h2]) * p.scale;
          } else {
            pv[e] = pe;
            ds[e] = pe * (dp[4 * jj + e] - dl[h2]) * p.scale;
          }
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
          float* dst = p.dq_acc + (SP ? (size_t)qr * p.dq_sw : 0) + (size_t)b * p.dq_sb + (size_t)h * p.dq_sh +
                       (size_t)(ql * TILE + r0 + 8 * h2) * p.dq_ss;
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
          if constexpr (DROPOUT)
            pv[(8 * jj + cq) >> 1] = pack2(dv[4 * jj + 2 * h2] * p.drop_scale, dv[4 * jj + 2 * h2 + 1] * p.drop_scale);
          else
            pv[(8 * jj + cq) >> 1] = pack2(dv[4 * jj + 2 * h2], dv[4 * jj + 2 * h2 + 1]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------ host side
// {64 d, S, H, B} view with element strides (ss, sh, sb); box {64, 128, 1, 1}
int make_qkv_map(CUtensorMap* m, const void* ptr, int B, int H, int S, long long sb, long long sh, long long ss) {
  if ((ss % 8) || (sh % 8) || (sb % 8) || ((uintptr_t)ptr & 15)) return fail("attention operands must be 16-byte aligned");
  const cuuint64_t dims[4] = {(cuuint64_t)HD, (cuuint64_t)S, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)ss * 2, (cuuint64_t)sh * 2, (cuuint64_t)sb * 2};
  const cuuint32_t box[4] = {64, TILE, 1, 1};
  return encode_map(m, ptr, 4, dims, strides, box);
}

// causal / dropout arguments shared by the forward and the backward; fills the dropout fields of the params
template <typename Params>
int check_mode(int causal, const unsigned long long* seed, float drop_p, Params& p) {
  if (causal != 0 && causal != 1) return fail("causal must be 0 or 1");
  if (!(drop_p >= 0.f && drop_p <= 1.f)) return fail("attention dropout p must be in [0, 1]");
  if (drop_p > 0.f && seed == nullptr) return fail("attention dropout needs a seed");
  p.seed = seed;
  p.drop_thr = dropout_thr16(drop_p);
  p.drop_scale = dropout_scale16(p.drop_thr);
  return 0;
}

template <bool CAUSAL, bool DROPOUT, bool SP = false, typename... Args>
int launch_fwd(dim3 grid, cudaStream_t st, Args... args) {
  if (smem_attr_once<attn_fwd_kernel<CAUSAL, DROPOUT, SP>>(FW_SMEM)) return -1;
  attn_fwd_kernel<CAUSAL, DROPOUT, SP><<<grid, AT, FW_SMEM, st>>>(args...);
  return 0;
}
template <bool CAUSAL, bool DROPOUT, bool SP = false, typename... Args>
int launch_bwd(dim3 grid, cudaStream_t st, Args... args) {
  if (smem_attr_once<attn_bwd_kernel<CAUSAL, DROPOUT, SP>>(BW_SMEM)) return -1;
  attn_bwd_kernel<CAUSAL, DROPOUT, SP><<<grid, AT, BW_SMEM, st>>>(args...);
  return 0;
}

// SP: a gathered [W][B][S][H][64] operand as a {64 d, S, H, B, W} map with element strides s = {w, b, h, s};
// box {64, 128, 1, 1, 1}
int make_gathered_map(CUtensorMap* m, const void* ptr, int W, int B, int H, int S, const long long* s) {
  if ((s[0] % 8) || (s[1] % 8) || (s[2] % 8) || (s[3] % 8) || ((uintptr_t)ptr & 15))
    return fail("gathered attention operands must be 16-byte aligned");
  const cuuint64_t dims[5] = {(cuuint64_t)HD, (cuuint64_t)S, (cuuint64_t)H, (cuuint64_t)B, (cuuint64_t)W};
  const cuuint64_t strides[4] = {(cuuint64_t)s[3] * 2, (cuuint64_t)s[2] * 2, (cuuint64_t)s[1] * 2, (cuuint64_t)s[0] * 2};
  const cuuint32_t box[5] = {64, TILE, 1, 1, 1};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed", (int)r);
  return 0;
}

// SP arguments shared by the forward and the backward; fills the zigzag fields of the params
template <typename Params>
int check_sp(int B, int H, int S, int D, int causal, int rank, int world, Params& p) {
  if (D != HD) return fail("head dim must be 64");
  if (causal != 0 && causal != 1) return fail("causal must be 0 or 1");
  if (B < 1 || H < 1) return fail("attention shapes must be positive");
  if (world < 1 || rank < 0 || rank >= world) return fail("sequence parallelism needs 0 <= rank < world");
  if (S < 2 * TILE || S % (2 * TILE)) return fail("sequence-parallel shards must be a positive multiple of 256 rows");
  if ((long long)S * world > (1 << 30)) return fail("sequence too long");
  p.B = B; p.H = H; p.S = S;
  p.sp_rank = rank; p.sp_world = world; p.sp_c = S / (2 * TILE);
  p.seed = nullptr; p.drop_thr = 0; p.drop_scale = 1.f;
  return 0;
}

int launched() {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  return 0;
}

}  // namespace

extern "C" {

const char* b200dp_attn_last_error() { return g_err; }

// strides: element strides {batch, head, seq} of each tensor (head dim 64 contiguous).  causal: 0 or 1 (query i
// sees keys 0..i; q, k and v share one sequence length S, so the mask always applies).  drop_p: attention
// dropout probability in [0, 1]; 0 runs the kernels without dropout, otherwise `seed` is 2 words in device
// memory (Philox key, offset: see the header for the mask).
int b200dp_attn_fwd_dropout(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int S,
                            int D, const long long* qs, const long long* ks, const long long* vs, const long long* os,
                            float scale, int causal, const unsigned long long* seed, float drop_p,
                            unsigned long long stream) {
  if (ensure_init()) return -1;
  if (D != HD) return fail("head dim must be 64");
  AttnFwdParams p;
  if (check_mode(causal, seed, drop_p, p)) return -1;
  if (B < 1 || H < 1 || S < 1) return fail("attention shapes must be positive");
  CUtensorMap mq, mk, mv;
  if (make_qkv_map(&mq, q, B, H, S, qs[0], qs[1], qs[2]) || make_qkv_map(&mk, k, B, H, S, ks[0], ks[1], ks[2]) ||
      make_qkv_map(&mv, v, B, H, S, vs[0], vs[1], vs[2]))
    return -1;
  if ((os[0] % 8) || (os[1] % 8) || (os[2] % 8) || ((uintptr_t)o & 15)) return fail("output must be 16-byte aligned");
  p.B = B; p.H = H; p.S = S;
  p.q_tiles = (S + TILE - 1) / TILE;
  p.kv_blocks = (S + TILE - 1) / TILE;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_sb = os[0]; p.o_sh = os[1]; p.o_ss = os[2];
  p.lse = lse;
  const dim3 grid(B * H * p.q_tiles);
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const bool drop = drop_p > 0.f;
  const int rc = causal ? (drop ? launch_fwd<true, true>(grid, st, mq, mk, mv, p) : launch_fwd<true, false>(grid, st, mq, mk, mv, p))
                        : (drop ? launch_fwd<false, true>(grid, st, mq, mk, mv, p) : launch_fwd<false, false>(grid, st, mq, mk, mv, p));
  return rc ? rc : launched();
}

// The forward without dropout under its earlier signatures, which Python callers bind with fixed ctypes argtypes.
int b200dp_attn_fwd_ex(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int S, int D,
                       const long long* qs, const long long* ks, const long long* vs, const long long* os, float scale,
                       int causal, unsigned long long stream) {
  return b200dp_attn_fwd_dropout(q, k, v, o, lse, B, H, S, D, qs, ks, vs, os, scale, causal, nullptr, 0.f, stream);
}
int b200dp_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int S, int D,
                    const long long* qs, const long long* ks, const long long* vs, const long long* os, float scale,
                    unsigned long long stream) {
  return b200dp_attn_fwd_dropout(q, k, v, o, lse, B, H, S, D, qs, ks, vs, os, scale, 0, nullptr, 0.f, stream);
}

// dq_acc: fp32 workspace (strides dqs, 64 contiguous) zeroed by the caller; delta: [B][H][S] fp32 workspace.
// o is the (dropped) forward output; causal, seed and drop_p as given to the forward.
int b200dp_attn_bwd_dropout(const void* q, const void* k, const void* v, const void* o, const void* dout,
                            const float* lse, float* delta, float* dq_acc, void* dk, void* dv, int B, int H, int S,
                            int D, const long long* qs, const long long* ks, const long long* vs, const long long* os,
                            const long long* dos, const long long* dqs, const long long* dks, const long long* dvs,
                            float scale, int causal, const unsigned long long* seed, float drop_p,
                            unsigned long long stream) {
  if (ensure_init()) return -1;
  if (D != HD) return fail("head dim must be 64");
  AttnBwdParams p;
  if (check_mode(causal, seed, drop_p, p)) return -1;
  if (B < 1 || H < 1 || S < 1) return fail("attention shapes must be positive");
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  CUtensorMap mq, mk, mv, mdo;
  if (make_qkv_map(&mq, q, B, H, S, qs[0], qs[1], qs[2]) || make_qkv_map(&mk, k, B, H, S, ks[0], ks[1], ks[2]) ||
      make_qkv_map(&mv, v, B, H, S, vs[0], vs[1], vs[2]) || make_qkv_map(&mdo, dout, B, H, S, dos[0], dos[1], dos[2]))
    return -1;
  const long long rows = (long long)B * H * S;
  attn_delta_kernel<<<(unsigned)((rows + 31) / 32), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(o), reinterpret_cast<const __nv_bfloat16*>(dout), delta, B, H, S, os[0],
      os[1], os[2], dos[0], dos[1], dos[2]);
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
  const dim3 grid(B * H * p.kv_blocks);
  const bool drop = drop_p > 0.f;
  const int rc = causal ? (drop ? launch_bwd<true, true>(grid, st, mq, mk, mv, mdo, p)
                                : launch_bwd<true, false>(grid, st, mq, mk, mv, mdo, p))
                        : (drop ? launch_bwd<false, true>(grid, st, mq, mk, mv, mdo, p)
                                : launch_bwd<false, false>(grid, st, mq, mk, mv, mdo, p));
  return rc ? rc : launched();
}

// delta[b][h][s] = sum_d dO * O (the backward's first pass on its own).  o, dout: [B, H, S, 64] with element
// strides os / dos {batch, head, seq}; delta: [B][H][S] fp32.
int b200dp_attn_delta(const void* o, const void* dout, float* delta, int B, int H, int S, int D, const long long* os,
                      const long long* dos, unsigned long long stream) {
  if (D != HD) return fail("head dim must be 64");
  if (B < 1 || H < 1 || S < 1) return fail("attention shapes must be positive");
  if ((os[0] % 8) || (os[1] % 8) || (os[2] % 8) || ((uintptr_t)o & 15) || (dos[0] % 8) || (dos[1] % 8) ||
      (dos[2] % 8) || ((uintptr_t)dout & 15))
    return fail("attention delta operands must be 16-byte aligned");
  const long long rows = (long long)B * H * S;
  attn_delta_kernel<<<(unsigned)((rows + 31) / 32), 256, 0, (cudaStream_t)(uintptr_t)stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(o), reinterpret_cast<const __nv_bfloat16*>(dout), delta, B, H, S, os[0],
      os[1], os[2], dos[0], dos[1], dos[2]);
  return launched();
}

// Sequence-parallel forward (see the header): rank `rank` of `world`, S = S_loc rows per rank (a multiple of 256).
// q, o: this rank's [B, H, S, 64] shard, strides {batch, head, seq}; k, v: the gathered [W, B, H, S, 64] views,
// strides {rank, batch, head, seq}; lse: [B][H][S] (nullptr: not saved).  No dropout.
int b200dp_attn_sp_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int S, int D,
                       const long long* qs, const long long* ks, const long long* vs, const long long* os, float scale,
                       int causal, int rank, int world, unsigned long long stream) {
  if (ensure_init()) return -1;
  AttnFwdParams p;
  if (check_sp(B, H, S, D, causal, rank, world, p)) return -1;
  CUtensorMap mq, mk, mv;
  if (make_qkv_map(&mq, q, B, H, S, qs[0], qs[1], qs[2]) || make_gathered_map(&mk, k, world, B, H, S, ks) ||
      make_gathered_map(&mv, v, world, B, H, S, vs))
    return -1;
  if ((os[0] % 8) || (os[1] % 8) || (os[2] % 8) || ((uintptr_t)o & 15)) return fail("output must be 16-byte aligned");
  p.q_tiles = S / TILE;                                  // local query tiles
  p.kv_blocks = world * (S / TILE);                      // global key tiles
  p.scale_log2 = scale * 1.4426950408889634f;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_sb = os[0]; p.o_sh = os[1]; p.o_ss = os[2];
  p.lse = lse;
  const dim3 grid(B * H * p.q_tiles);
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int rc = causal ? launch_fwd<true, false, true>(grid, st, mq, mk, mv, p)
                        : launch_fwd<false, false, true>(grid, st, mq, mk, mv, p);
  return rc ? rc : launched();
}

// Sequence-parallel backward: k, v, dk, dv: this rank's [B, H, S, 64] shard (strides {batch, head, seq}); q, dout:
// gathered [W, B, H, S, 64] views (strides {rank, batch, head, seq}); lse, delta: gathered [W][B][H][S] fp32 with
// rank stride ld_sw elements (delta from b200dp_attn_delta on each rank); dq_acc: fp32 [W, B, H, S, 64] workspace
// (strides dqs {rank, batch, head, seq}, 64 contiguous) zeroed by the caller, which gets this rank's partial dQ of
// every rank's queries.
int b200dp_attn_sp_bwd(const void* q, const void* k, const void* v, const void* dout, const float* lse,
                       const float* delta, float* dq_acc, void* dk, void* dv, int B, int H, int S, int D,
                       const long long* qs, const long long* ks, const long long* vs, const long long* dos,
                       const long long* dqs, const long long* dks, const long long* dvs, long long ld_sw, float scale,
                       int causal, int rank, int world, unsigned long long stream) {
  if (ensure_init()) return -1;
  AttnBwdParams p;
  if (check_sp(B, H, S, D, causal, rank, world, p)) return -1;
  CUtensorMap mq, mk, mv, mdo;
  if (make_gathered_map(&mq, q, world, B, H, S, qs) || make_qkv_map(&mk, k, B, H, S, ks[0], ks[1], ks[2]) ||
      make_qkv_map(&mv, v, B, H, S, vs[0], vs[1], vs[2]) || make_gathered_map(&mdo, dout, world, B, H, S, dos))
    return -1;
  if ((dqs[0] % 4) || (dqs[1] % 4) || (dqs[2] % 4) || (dqs[3] % 4)) return fail("dq workspace strides must be multiples of 4");
  if (ld_sw < (long long)B * H * S) return fail("lse / delta rank stride is shorter than one rank's rows");
  p.q_tiles = world * (S / TILE);                        // global query tiles
  p.kv_blocks = S / TILE;                                // local key blocks
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.lse = lse; p.delta = delta; p.dq_acc = dq_acc;
  p.lse_sw = ld_sw;
  p.dq_sw = dqs[0]; p.dq_sb = dqs[1]; p.dq_sh = dqs[2]; p.dq_ss = dqs[3];
  p.dk = reinterpret_cast<__nv_bfloat16*>(dk); p.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  p.dk_sb = dks[0]; p.dk_sh = dks[1]; p.dk_ss = dks[2];
  p.dv_sb = dvs[0]; p.dv_sh = dvs[1]; p.dv_ss = dvs[2];
  const dim3 grid(B * H * p.kv_blocks);
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int rc = causal ? launch_bwd<true, false, true>(grid, st, mq, mk, mv, mdo, p)
                        : launch_bwd<false, false, true>(grid, st, mq, mk, mv, mdo, p);
  return rc ? rc : launched();
}

// The backward without dropout under its earlier signature.
int b200dp_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                    float* delta, float* dq_acc, void* dk, void* dv, int B, int H, int S, int D, const long long* qs,
                    const long long* ks, const long long* vs, const long long* os, const long long* dos,
                    const long long* dqs, const long long* dks, const long long* dvs, float scale, int causal,
                    unsigned long long stream) {
  return b200dp_attn_bwd_dropout(q, k, v, o, dout, lse, delta, dq_acc, dk, dv, B, H, S, D, qs, ks, vs, os, dos, dqs,
                                 dks, dvs, scale, causal, nullptr, 0.f, stream);
}

}  // extern "C"

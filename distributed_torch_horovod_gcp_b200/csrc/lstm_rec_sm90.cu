// K5 — persistent LSTM recurrence for sm_90a (fp32 I/O, tf32 tensor cores, fp32 accumulation/state).
//
// The reference's only compute-heavy op is nn.LSTM(23 -> 256) over 10 timesteps at batch 32
// (app/torch_train.py of the reference application).  On an H100 that is a pure
// latency problem: 10 dependent [32 x 256] x [256 x 1024] products.  cuDNN re-reads W_hh (1 MB) from L2
// every step; here a CLUSTER OF 8 CTAs keeps it on chip for the whole sequence:
//
//   * CTA c owns hidden units [32c, 32c+32) and therefore gate rows {g*256 + 32c + j}: a 128 x 256 slice
//     of W_hh, resident in shared memory (128 KB) as the K-major, 128B-swizzled A operand of
//     wgmma tf32 (M = 128 gate rows as two m64 halves, N = 32 batch, K = 256 hidden);
//   * per step: the CTA's one warpgroup issues 64 wgmmas (m64n32k8) -> accumulator fragments -> a row-major
//     image in shared memory -> each warp reads its gate type (rows 32w..32w+31 == gate i/f/g/o), adds the
//     precomputed input projection, applies the
//     nonlinearity, swap gates through shared memory, update c (registers, never leaves the SM) and h;
//   * h_t (32 units x 32 batch) is written straight into the B-operand buffers of all 8 CTAs through
//     distributed shared memory (st.shared::cluster into the swizzled layout), one
//     barrier.cluster per step orders it — no global-memory round trip, no kernel boundary;
//   * large batches (the reference validates on the whole test set in one batch) are tiled by 32
//     across 16 clusters with the weights staying resident.
//
// Backward runs the same cluster in reverse: dgates for the own units (SIMT, fp32), partial
// dh_{t-1}[256 x 32] = W_slice^T (K-major copy of the transposed slice, 128 KB) x dgates^T on the tensor
// core, reduce-scatter of the 8 partials through DSMEM.  dgates_t is also streamed to global memory and
// the weight/bias/input gradients are ONE extra kernel over all SMs (they are sums over (t, b), not part
// of the serial chain).  The x-projection (x_t W_ih^T + b_ih + b_hh for all t) is likewise hoisted out of
// the recurrence into one small kernel.
//
// Replaces cuDNN's RNN kernels.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "sm90_common.cuh"

namespace {

constexpr int LH = 256;            // hidden size (8 CTAs x 32 units)
constexpr int LG = 4 * LH;         // gate rows
constexpr int CL = 8;              // cluster size
constexpr int LU = LH / CL;        // units per CTA (32)
constexpr int NB = 32;             // batch tile (wgmma N)
constexpr int LTHREADS = 128;      // one warpgroup: wgmma, then gate/cell math (warp == gate type)
constexpr int IMG_BYTES = 128 * NB * 4;   // accumulator image [128 rows][32] fp32
constexpr int EPI_T = 128;

thread_local char g_lerr[512];
int lfail(const char* msg, int code = 0) {
  snprintf(g_lerr, sizeof(g_lerr), "%s (%d)", msg, code);
  return -1;
}

__device__ __forceinline__ uint32_t my_cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void st_cluster_v4(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}
__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// generic-proxy writes to shared memory (local CTA / any CTA of the cluster) -> visible to the async proxy
// (wgmma operand reads).  The state-space qualified forms are far cheaper than the full
// `fence.proxy.async` (which ptxas expands to MEMBAR.ALL.CTA + ERRBAR + FENCE.VIEW.ASYNC).
__device__ __forceinline__ void fence_proxy_async_all() {
  asm volatile("fence.proxy.async.shared::cluster;" ::: "memory");
}
__device__ __forceinline__ void sts_v4(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void sts_f32(uint32_t addr, float a) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(a) : "memory");
}
__device__ __forceinline__ float4 lds_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void epi_barrier() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// m64 x 32 wgmma fragment -> rows row0.. of the [rows][32] fp32 accumulator image; 16-byte units are
// XOR-swizzled by row so that both these stores and the one-row-per-lane reads below are conflict-free
__device__ __forceinline__ void frag32_to_img(const float* d, uint32_t img, int row0) {
  const int t = threadIdx.x & 127;
  const int r = row0 + (t >> 5) * 16 + ((t & 31) >> 2);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int col = 8 * j + 2 * (t & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rr = r + 8 * h;
      const uint32_t a = img + (uint32_t)(rr * 128 + ((((col >> 2) ^ (rr & 7))) << 4) + ((col & 3) << 2));
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(d[4 * j + 2 * h]), "f"(d[4 * j + 2 * h + 1])
                   : "memory");
    }
  }
}
__device__ __forceinline__ void img_row32(uint32_t img, int row, uint32_t* r) {
#pragma unroll
  for (int u = 0; u < 8; ++u)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[4 * u]), "=r"(r[4 * u + 1]), "=r"(r[4 * u + 2]), "=r"(r[4 * u + 3])
                 : "r"(img + (uint32_t)(row * 128 + ((u ^ (row & 7)) << 4)))
                 : "memory");
}

__device__ __forceinline__ float sigmoidf_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float tanhf_fast(float x) { return 2.0f * sigmoidf_fast(2.0f * x) - 1.0f; }

// byte offset of fp32 element (row, k) inside a K-major 128B-swizzled operand made of 32-column chunks
// of `rows_per_chunk` rows (what a TMA box {32 fp32, rows} with SWIZZLE_128B would produce)
__device__ __forceinline__ uint32_t sw_off(int row, int k, int rows_per_chunk) {
  const int chunk = k >> 5, col = k & 31;
  return (uint32_t)(chunk * rows_per_chunk * 128 + row * 128 + ((((col >> 2) ^ (row & 7))) << 4) + ((col & 3) << 2));
}

// ---------------------------------------------------------------------------------------------------
// x-projection: xp[t][b][r] = b_ih[r] + b_hh[r] + sum_f x[b][t][f] * W_ih[r][f]        (all t at once)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) lstm_xproj_kernel(const float* __restrict__ x, const float* __restrict__ w_ih,
                                                         const float* __restrict__ b_ih, const float* __restrict__ b_hh,
                                                         float* __restrict__ xp, int B, int T, int F) {
  extern __shared__ float sx[];          // [8 rows][F]
  const int row0 = blockIdx.x * 8;       // rows of the [T*B] x F matrix, ordered (t, b)
  const int nrows = min(8, T * B - row0);
  for (int i = threadIdx.x; i < nrows * F; i += blockDim.x) {
    const int rr = row0 + i / F, f = i % F;
    const int t = rr / B, b = rr % B;
    sx[i] = x[((size_t)b * T + t) * F + f];
  }
  __syncthreads();
  for (int r = threadIdx.x; r < LG; r += blockDim.x) {
    float acc[8];
    const float bias = b_ih[r] + b_hh[r];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = bias;
    const float* w = w_ih + (size_t)r * F;
    for (int f = 0; f < F; ++f) {
      const float wv = __ldg(w + f);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(wv, sx[i * F + f], acc[i]);
    }
    for (int i = 0; i < nrows; ++i) xp[(size_t)(row0 + i) * LG + r] = acc[i];
  }
}

// ---------------------------------------------------------------------------------------------------
// forward recurrence
// ---------------------------------------------------------------------------------------------------
struct RecFwdParams {
  const float* w_hh;    // [1024][256]
  const float* xp;      // [T][B][1024]
  const float* h0;      // [B][256]
  const float* c0;      // [B][256]
  float* seq;           // [B][T][256]
  float* hT;            // [B][256]
  float* cT;            // [B][256]
  float* gates;         // [T][B][1024] post-activation i,f,g,o   (nullptr: inference, nothing saved)
  float* cs;            // [T][B][256]  c_t                       (nullptr: inference)
  int B, T;
};

constexpr int FW_A_BYTES = 128 * 1024;               // 8 chunks x [128 rows x 128 B]
constexpr int FW_B_BYTES = 32 * 1024;                // 8 chunks x [32 rows x 128 B], double buffered
constexpr int FW_G_BYTES = 16 * 1024;                // gate exchange [4][32][32] fp32
constexpr int FW_SMEM = FW_A_BYTES + 2 * FW_B_BYTES + FW_G_BYTES + IMG_BYTES + 1024;

__global__ void __launch_bounds__(LTHREADS, 1) lstm_rec_fwd_kernel(const RecFwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + FW_A_BYTES;
  uint8_t* sG = sB + 2 * FW_B_BYTES;
  const uint32_t img = smem_u32(sG + FW_G_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t c = my_cluster_rank();
  const int cluster_id = blockIdx.x / CL, num_clusters = gridDim.x / CL;

  // ---- resident A operand: W_hh rows {g*256 + 32c + j}, K-major tf32, 128B swizzle.  Loads are issued in
  // batches of 8 independent 128-bit requests per thread before any store (latency-bound otherwise).
  {
    const uint32_t sA_u = smem_u32(sA);
    constexpr int TOTAL = 128 * 64, BATCH = 8;
    for (int base = tid; base < TOTAL; base += LTHREADS * BATCH) {
      float4 v[BATCH];
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const int i = base + u * LTHREADS;
        if (i < TOTAL) {
          const int r = i >> 6, k4 = i & 63;
          const int grow = (r >> 5) * LH + (int)c * LU + (r & 31);
          v[u] = __ldg(reinterpret_cast<const float4*>(p.w_hh + (size_t)grow * LH + k4 * 4));
        }
      }
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const int i = base + u * LTHREADS;
        if (i < TOTAL) sts_v4(sA_u + sw_off(i >> 6, (i & 63) * 4, 128), v[u].x, v[u].y, v[u].z, v[u].w);
      }
    }
  }
  fence_proxy_async_all();
  __syncthreads();

  const int num_tiles = (p.B + NB - 1) / NB;
  for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
    const int b0 = tile * NB;
    // ---- h_{-1} = h0 into B buffer 0 (every CTA needs all 256 hidden units); c0 into registers
    for (int i = tid; i < NB * 64; i += LTHREADS) {
      const int b = i >> 6, k4 = i & 63;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b0 + b < p.B) v = *reinterpret_cast<const float4*>(p.h0 + (size_t)(b0 + b) * LH + k4 * 4);
      sts_v4(smem_u32(sB) + sw_off(b, k4 * 4, NB), v.x, v.y, v.z, v.w);
    }
    float cstate[8], hlast[8];
    const int ju = lane;                       // unit owned by this thread in the cell update
    const int bb = warp * 8;                   // its 8 batch rows
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + bb + i;
      cstate[i] = (b < p.B) ? p.c0[(size_t)b * LH + c * LU + ju] : 0.f;
      hlast[i] = 0.f;
    }
    fence_proxy_async_all();
    cluster_barrier();                         // nobody writes into a peer's buffers before it finished the last tile

    for (int t = 0; t < p.T; ++t) {
      const int cur = t & 1, nxt = cur ^ 1;
      {
        // gate pre-activations h_{t-1} W_slice^T: two m64 halves of the 128 gate rows
        float d0[16], d1[16];
        const uint64_t a0 = make_desc_base(16, 1024) + desc_addr(smem_u32(sA));
        const uint64_t bq = make_desc_base(16, 1024) + desc_addr(smem_u32(sB + cur * FW_B_BYTES));
        fence_proxy_async_all();
        wg_fence();
#pragma unroll
        for (int kc = 0; kc < 8; ++kc) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint64_t db = bq + (uint64_t)((kc * 4096 + ks * 32) >> 4);
            wgmma_tf32_n32(d0, a0 + (uint64_t)((kc * 16384 + ks * 32) >> 4), db, (kc | ks) ? 1u : 0u);
            wgmma_tf32_n32(d1, a0 + (uint64_t)((kc * 16384 + 8192 + ks * 32) >> 4), db, (kc | ks) ? 1u : 0u);
          }
        }
        wg_commit();
        // gate warp `warp` == gate type (i, f, g, o); lane == unit; 32 columns == batch
        const int grow = warp * LH + (int)c * LU + lane;
        float xv[NB];
#pragma unroll
        for (int b = 0; b < NB; ++b)                       // fetch the input projection while the MMAs run
          xv[b] = (b0 + b < p.B) ? __ldg(p.xp + ((size_t)t * p.B + b0 + b) * LG + grow) : 0.f;
        wg_wait<0>();
        wg_fence_operands<16>(d0);
        wg_fence_operands<16>(d1);
        frag32_to_img(d0, img, 0);
        frag32_to_img(d1, img, 64);
        epi_barrier();
        uint32_t r[NB];
        img_row32(img, warp * 32 + lane, r);
        float v[NB];
#pragma unroll
        for (int b = 0; b < NB; ++b) {
          const float pre = __uint_as_float(r[b]) + xv[b];
          v[b] = (warp == 2) ? tanhf_fast(pre) : sigmoidf_fast(pre);
        }
        if (p.gates != nullptr) {
#pragma unroll
          for (int b = 0; b < NB; ++b)
            if (b0 + b < p.B) p.gates[((size_t)t * p.B + b0 + b) * LG + grow] = v[b];
        }
        const uint32_t gx = smem_u32(sG);
#pragma unroll
        for (int cb = 0; cb < 8; ++cb)
          sts_v4(gx + (uint32_t)(((warp * 32 + lane) * 32 + ((cb ^ (lane & 7)) << 2)) * 4), v[4 * cb], v[4 * cb + 1],
                 v[4 * cb + 2], v[4 * cb + 3]);
        epi_barrier();
        // ---- cell update for (unit ju, batch bb .. bb+7)
        float gi[8], gf[8], gg[8], go[8];
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int cb = (bb >> 2) + h2;
          const int pos = ((cb ^ (ju & 7)) << 2);
          const float4 vi = lds_v4(gx + (uint32_t)(((0 * 32 + ju) * 32 + pos) * 4));
          const float4 vf = lds_v4(gx + (uint32_t)(((1 * 32 + ju) * 32 + pos) * 4));
          const float4 vg = lds_v4(gx + (uint32_t)(((2 * 32 + ju) * 32 + pos) * 4));
          const float4 vo = lds_v4(gx + (uint32_t)(((3 * 32 + ju) * 32 + pos) * 4));
          gi[4 * h2] = vi.x; gi[4 * h2 + 1] = vi.y; gi[4 * h2 + 2] = vi.z; gi[4 * h2 + 3] = vi.w;
          gf[4 * h2] = vf.x; gf[4 * h2 + 1] = vf.y; gf[4 * h2 + 2] = vf.z; gf[4 * h2 + 3] = vf.w;
          gg[4 * h2] = vg.x; gg[4 * h2 + 1] = vg.y; gg[4 * h2 + 2] = vg.z; gg[4 * h2 + 3] = vg.w;
          go[4 * h2] = vo.x; go[4 * h2 + 1] = vo.y; go[4 * h2 + 2] = vo.z; go[4 * h2 + 3] = vo.w;
        }
        const int kglob = (int)c * LU + ju;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          cstate[i] = gf[i] * cstate[i] + gi[i] * gg[i];
          hlast[i] = go[i] * tanhf_fast(cstate[i]);
          const int b = b0 + bb + i;
          if (b < p.B) {
            p.seq[((size_t)b * p.T + t) * LH + kglob] = hlast[i];
            if (p.cs != nullptr) p.cs[((size_t)t * p.B + b) * LH + kglob] = cstate[i];
          }
        }
        if (t + 1 < p.T) {
          // h_t -> chunk `c` of the next step's B operand in ALL 8 CTAs (swizzled K-major rows = batch)
          const uint32_t base = smem_u32(sB + nxt * FW_B_BYTES);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const uint32_t off = base + sw_off(bb + i, kglob, NB);
#pragma unroll
            for (int peer = 0; peer < CL; ++peer) st_cluster_f32(map_to_cta(off, (uint32_t)peer), hlast[i]);
          }
        }
        epi_barrier();                          // sG and the image are rewritten next step
      }
      fence_proxy_async_all();
      cluster_barrier();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + bb + i;
      if (b < p.B) {
        p.hT[(size_t)b * LH + c * LU + ju] = hlast[i];
        p.cT[(size_t)b * LH + c * LU + ju] = cstate[i];
      }
    }
  }
  cluster_barrier();                            // no CTA exits while a peer may still address its smem
}

// ---------------------------------------------------------------------------------------------------
// backward recurrence
// ---------------------------------------------------------------------------------------------------
struct RecBwdParams {
  const float* __restrict__ w_hh;    // [1024][256]
  const float* __restrict__ gates;   // [T][B][1024]
  const float* __restrict__ cs;      // [T][B][256]
  const float* __restrict__ c0;      // [B][256]
  const float* __restrict__ dseq;    // [B][T][256]   (may be nullptr)
  const float* __restrict__ dhT;     // [B][256]      (may be nullptr)
  const float* __restrict__ dcT;     // [B][256]      (may be nullptr)
  float* __restrict__ dgates;        // [T][B][1024]
  float* dh0;           // [B][256]
  float* dc0;           // [B][256]
  int B, T;
};
constexpr int BW_A_BYTES = 128 * 1024;               // W_slice^T: 4 chunks x [256 rows (k) x 128 B (32 gate rows)]
constexpr int BW_B_BYTES = 16 * 1024;                // dgates: 4 chunks x [32 rows (b) x 128 B]
constexpr int BW_R_BYTES = 32 * 1024;                // partial dh from 8 sources [8][32 j][32 b], double buffered
constexpr int BW_SMEM = BW_A_BYTES + BW_B_BYTES + 2 * BW_R_BYTES + IMG_BYTES + 1024;

__global__ void __launch_bounds__(LTHREADS, 1) lstm_rec_bwd_kernel(const RecBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + BW_A_BYTES;
  uint8_t* sR = sB + BW_B_BYTES;
  const uint32_t img = smem_u32(sR + 2 * BW_R_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t c = my_cluster_rank();
  const int cluster_id = blockIdx.x / CL, num_clusters = gridDim.x / CL;

  // ---- resident A operand: (W_slice)^T, rows = k (256), K = local gate row r (128), K-major, swizzled.
  // W rows are read coalesced (128-bit, 8 requests in flight per thread) and scattered transposed.
  {
    const uint32_t sA_u = smem_u32(sA);
    constexpr int TOTAL = 128 * 64, BATCH = 8;
    for (int base = tid; base < TOTAL; base += LTHREADS * BATCH) {
      float4 v[BATCH];
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const int i = base + u * LTHREADS;
        if (i < TOTAL) {
          const int r = i >> 6, k4 = i & 63;
          const int grow = (r >> 5) * LH + (int)c * LU + (r & 31);
          v[u] = __ldg(reinterpret_cast<const float4*>(p.w_hh + (size_t)grow * LH + k4 * 4));
        }
      }
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const int i = base + u * LTHREADS;
        if (i < TOTAL) {
          const int r = i >> 6, k = (i & 63) * 4;
          sts_f32(sA_u + sw_off(k + 0, r, LH), v[u].x);
          sts_f32(sA_u + sw_off(k + 1, r, LH), v[u].y);
          sts_f32(sA_u + sw_off(k + 2, r, LH), v[u].z);
          sts_f32(sA_u + sw_off(k + 3, r, LH), v[u].w);
        }
      }
    }
  }
  fence_proxy_async_all();
  __syncthreads();

  const int num_tiles = (p.B + NB - 1) / NB;
  for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
    const int b0 = tile * NB;
    const int ju = lane, bb = warp * 8;
    const int kglob = (int)c * LU + ju;
    float dc_next[8], dh_rec[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + bb + i;
      dc_next[i] = (p.dcT != nullptr && b < p.B) ? p.dcT[(size_t)b * LH + kglob] : 0.f;
      dh_rec[i] = (p.dhT != nullptr && b < p.B) ? p.dhT[(size_t)b * LH + kglob] : 0.f;
    }
    cluster_barrier();

    for (int t = p.T - 1; t >= 0; --t) {
      const int cur = (p.T - 1 - t) & 1;        // reduce buffer written during this step
      {
        // ---- dgates for (unit ju, batch bb..bb+7)
        const uint32_t sB_u = smem_u32(sB);
        // all global operands of the 8 batch rows first (one memory round trip instead of eight)
        float gi[8], gf[8], gg[8], go[8], ct[8], cprev[8], dsq[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int b = b0 + bb + i;
          const bool ok = b < p.B;
          const size_t gbase = ((size_t)t * p.B + (ok ? b : 0)) * LG + kglob;
          gi[i] = ok ? __ldg(p.gates + gbase) : 0.f;
          gf[i] = ok ? __ldg(p.gates + gbase + LH) : 0.f;
          gg[i] = ok ? __ldg(p.gates + gbase + 2 * LH) : 0.f;
          go[i] = ok ? __ldg(p.gates + gbase + 3 * LH) : 0.f;
          ct[i] = ok ? __ldg(p.cs + ((size_t)t * p.B + b) * LH + kglob) : 0.f;
          cprev[i] = !ok ? 0.f
                         : ((t > 0) ? __ldg(p.cs + ((size_t)(t - 1) * p.B + b) * LH + kglob)
                                    : __ldg(p.c0 + (size_t)b * LH + kglob));
          dsq[i] = (ok && p.dseq != nullptr) ? __ldg(p.dseq + ((size_t)b * p.T + t) * LH + kglob) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int b = b0 + bb + i;
          float di = 0.f, df = 0.f, dg = 0.f, dob = 0.f;
          if (b < p.B) {
            const size_t gbase = ((size_t)t * p.B + b) * LG + kglob;
            const float dh = dh_rec[i] + dsq[i];
            const float tc = tanhf_fast(ct[i]);
            const float dc = dc_next[i] + dh * go[i] * (1.0f - tc * tc);
            dob = dh * tc * go[i] * (1.0f - go[i]);
            di = dc * gg[i] * gi[i] * (1.0f - gi[i]);
            df = dc * cprev[i] * gf[i] * (1.0f - gf[i]);
            dg = dc * gi[i] * (1.0f - gg[i] * gg[i]);
            dc_next[i] = dc * gf[i];
            p.dgates[gbase] = di;
            p.dgates[gbase + LH] = df;
            p.dgates[gbase + 2 * LH] = dg;
            p.dgates[gbase + 3 * LH] = dob;
          } else {
            dc_next[i] = 0.f;
          }
          // B operand: rows = batch, K = local gate row (g*32 + ju)
          sts_f32(sB_u + sw_off(bb + i, 0 * 32 + ju, NB), di);
          sts_f32(sB_u + sw_off(bb + i, 1 * 32 + ju, NB), df);
          sts_f32(sB_u + sw_off(bb + i, 2 * 32 + ju, NB), dg);
          sts_f32(sB_u + sw_off(bb + i, 3 * 32 + ju, NB), dob);
        }
      }
      fence_proxy_async_all();
      __syncthreads();
      {
        // partial dh_{t-1} rows k = 0..255 as four m64 blocks: A = W_slice^T (chunk kc of 32 local gate rows
        // at +kc*LH*128, k rows 128 B apart), B = dgates (rows = batch)
        float d[4][16];
        const uint64_t a0 = make_desc_base(16, 1024) + desc_addr(smem_u32(sA));
        const uint64_t bq = make_desc_base(16, 1024) + desc_addr(smem_u32(sB));
        wg_fence();
#pragma unroll
        for (int mb = 0; mb < 4; ++mb) {
#pragma unroll
          for (int kc = 0; kc < 4; ++kc) {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks)
              wgmma_tf32_n32(d[mb], a0 + (uint64_t)((kc * (LH * 128) + mb * (64 * 128) + ks * 32) >> 4),
                             bq + (uint64_t)((kc * 4096 + ks * 32) >> 4), (kc | ks) ? 1u : 0u);
          }
        }
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int mb = 0; mb < 4; ++mb) wg_fence_operands<16>(d[mb]);
        // rows k = 128 m + 32 warp + lane of the partial dh_{t-1}; owner CTA of those units = 4 m + warp
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          frag32_to_img(d[2 * m], img, 0);
          frag32_to_img(d[2 * m + 1], img, 64);
          epi_barrier();
          uint32_t r[NB];
          img_row32(img, warp * 32 + lane, r);
          const uint32_t peer = (uint32_t)(4 * m + warp);
          const uint32_t dst = map_to_cta(smem_u32(sR + cur * BW_R_BYTES) + (uint32_t)(((int)c * 32 + lane) * 128), peer);
#pragma unroll
          for (int q = 0; q < 8; ++q)
            st_cluster_v4(dst + q * 16, __uint_as_float(r[4 * q]), __uint_as_float(r[4 * q + 1]),
                          __uint_as_float(r[4 * q + 2]), __uint_as_float(r[4 * q + 3]));
          epi_barrier();                        // the image is rewritten by the next half
        }
      }
      cluster_barrier();
      {
        // dh_{t-1}[unit ju][batch bb..bb+7] = sum over the 8 source CTAs
        const uint32_t red = smem_u32(sR + cur * BW_R_BYTES);
#pragma unroll
        for (int i = 0; i < 8; ++i) dh_rec[i] = 0.f;
#pragma unroll
        for (int s = 0; s < CL; ++s) {
          const float4 v0 = lds_v4(red + (uint32_t)(((s * 32 + ju) * 32 + bb) * 4));
          const float4 v1 = lds_v4(red + (uint32_t)(((s * 32 + ju) * 32 + bb + 4) * 4));
          dh_rec[0] += v0.x; dh_rec[1] += v0.y; dh_rec[2] += v0.z; dh_rec[3] += v0.w;
          dh_rec[4] += v1.x; dh_rec[5] += v1.y; dh_rec[6] += v1.z; dh_rec[7] += v1.w;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + bb + i;
      if (b < p.B) {
        if (p.dh0 != nullptr) p.dh0[(size_t)b * LH + kglob] = dh_rec[i];
        if (p.dc0 != nullptr) p.dc0[(size_t)b * LH + kglob] = dc_next[i];
      }
    }
  }
  cluster_barrier();
}

// ---------------------------------------------------------------------------------------------------
// weight / bias / input gradients: sums over (t, b), off the serial chain -> all SMs, fp32 SIMT
//   dW_hh[r][k] = sum dG[t][b][r] * hprev[t][b][k]     (hprev[0] = h0, hprev[t] = seq[:, t-1])
//   dW_ih[r][f] = sum dG[t][b][r] * x[b][t][f],   db[r] = sum dG[t][b][r]
//   dx[b][t][f] = sum_r dG[t][b][r] * W_ih[r][f]                                   (optional)
// ---------------------------------------------------------------------------------------------------
struct WgParams {
  const float* dG; const float* seq; const float* h0; const float* x; const float* w_ih;
  float* dW_hh; float* dW_ih; float* db_ih; float* db_hh; float* dx;
  int B, T, F, ksplit;
};
constexpr int WG_TR = 64, WG_TK = 64, WG_KC = 16;

__global__ void __launch_bounds__(256) lstm_wgrad_kernel(const WgParams p) {
  __shared__ float sD[WG_KC][WG_TR + 1];
  __shared__ float sH[WG_KC][WG_TK + 1];
  const int TB = p.T * p.B;
  const int hh_blocks = (LG / WG_TR) * (LH / WG_TK) * p.ksplit;
  const int tid = threadIdx.x;
  if ((int)blockIdx.x < hh_blocks) {
    const int ks = blockIdx.x % p.ksplit;
    const int tile = blockIdx.x / p.ksplit;
    const int r0 = (tile / (LH / WG_TK)) * WG_TR, k0 = (tile % (LH / WG_TK)) * WG_TK;
    const int per = (TB + p.ksplit - 1) / p.ksplit;
    const int q0 = ks * per, q1 = min(q0 + per, TB);
    const int tr = (tid >> 4) * 4, tk = (tid & 15) * 4;      // 4 x 4 outputs per thread
    float acc[4][4] = {};
    for (int q = q0; q < q1; q += WG_KC) {
      for (int i = tid; i < WG_KC * WG_TR; i += 256) {
        const int kk = i / WG_TR, rr = i % WG_TR;
        const int qq = q + kk;
        sD[kk][rr] = (qq < q1) ? p.dG[(size_t)qq * LG + r0 + rr] : 0.f;
        float hv = 0.f;
        if (qq < q1) {
          const int t = qq / p.B, b = qq % p.B;
          hv = (t == 0) ? p.h0[(size_t)b * LH + k0 + rr] : p.seq[((size_t)b * p.T + (t - 1)) * LH + k0 + rr];
        }
        sH[kk][rr] = hv;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < WG_KC; ++kk) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i] = sD[kk][tr + i]; b[i] = sH[kk][tk + i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) atomicAdd(p.dW_hh + (size_t)(r0 + tr + i) * LH + k0 + tk + j, acc[i][j]);
    return;
  }
  // ---- dW_ih / db: one block per 8 gate rows; warp w owns row r0 + w, lanes stride (t, b)
  const int blk = blockIdx.x - hh_blocks;
  const int ih_blocks = LG / 8;
  if (blk < ih_blocks) {
    const int r = blk * 8 + (tid >> 5), lane = tid & 31;
    float bsum = 0.f;
    float wacc[32];
#pragma unroll
    for (int f = 0; f < 32; ++f) wacc[f] = 0.f;
    for (int q = lane; q < TB; q += 32) {
      const float g = p.dG[(size_t)q * LG + r];
      bsum += g;
      const int t = q / p.B, b = q % p.B;
      const float* xr = p.x + ((size_t)b * p.T + t) * p.F;
#pragma unroll
      for (int f = 0; f < 32; ++f)
        if (f < p.F) wacc[f] = fmaf(g, xr[f], wacc[f]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bsum += __shfl_xor_sync(0xffffffffu, bsum, o);
#pragma unroll
    for (int f = 0; f < 32; ++f) {
      if (f < p.F) {
        float v = wacc[f];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) p.dW_ih[(size_t)r * p.F + f] = v;
      }
    }
    if (lane == 0) {
      p.db_ih[r] = bsum;
      p.db_hh[r] = bsum;
    }
    return;
  }
  // ---- dx (only when the input requires a gradient): one warp per (t, b) row
  if (p.dx == nullptr) return;
  const int row = (blk - ih_blocks) * 8 + (tid >> 5), lane = tid & 31;
  if (row >= TB) return;
  float acc[32];
#pragma unroll
  for (int f = 0; f < 32; ++f) acc[f] = 0.f;
  for (int r = lane; r < LG; r += 32) {
    const float g = p.dG[(size_t)row * LG + r];
    const float* w = p.w_ih + (size_t)r * p.F;
#pragma unroll
    for (int f = 0; f < 32; ++f)
      if (f < p.F) acc[f] = fmaf(g, __ldg(w + f), acc[f]);
  }
  const int t = row / p.B, b = row % p.B;
#pragma unroll
  for (int f = 0; f < 32; ++f) {
    if (f < p.F) {
      float v = acc[f];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) p.dx[((size_t)b * p.T + t) * p.F + f] = v;
    }
  }
}

int g_sms = 0;
int sms() {
  if (!g_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return g_sms;
}

template <typename K, typename P>
int launch_cluster(K kern, const P& p, int clusters, int smem_bytes, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  if (e != cudaSuccess) return lfail(cudaGetErrorString(e), (int)e);
  cudaLaunchConfig_t cfg;
  cfg = cudaLaunchConfig_t{};
  cfg.gridDim = dim3(CL * clusters);
  cfg.blockDim = dim3(LTHREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, kern, p);
  if (e != cudaSuccess) return lfail(cudaGetErrorString(e), (int)e);
  return 0;
}

}  // namespace

extern "C" {

const char* b200dp_lstm_rec_last_error() { return g_lerr; }

int b200dp_lstm_rec_supported(int H, int F) { return (H == LH && F >= 1 && F <= 32) ? 1 : 0; }

// Forward: x [B][T][F], h0/c0 [B][256], weights in PyTorch layout; outputs seq [B][T][256], hT/cT [B][256].
// xp_ws: [T][B][1024] workspace.  gates/cs: saved for backward ([T][B][1024] / [T][B][256]) or null.
int b200dp_lstm_rec_fwd(const float* x, const float* h0, const float* c0, const float* w_ih, const float* w_hh,
                        const float* b_ih, const float* b_hh, float* xp_ws, float* seq, float* hT, float* cT,
                        float* gates, float* cs, int B, int T, int F, unsigned long long stream) {
  if (!b200dp_lstm_rec_supported(LH, F)) return lfail("unsupported LSTM shape");
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int rows = T * B;
  lstm_xproj_kernel<<<(rows + 7) / 8, 256, 8 * F * sizeof(float), st>>>(x, w_ih, b_ih, b_hh, xp_ws, B, T, F);
  RecFwdParams p{w_hh, xp_ws, h0, c0, seq, hT, cT, gates, cs, B, T};
  const int tiles = (B + NB - 1) / NB;
  int clusters = sms() / CL;
  if (clusters > tiles) clusters = tiles;
  if (clusters < 1) clusters = 1;
  return launch_cluster(lstm_rec_fwd_kernel, p, clusters, FW_SMEM, st);
}

// Backward of the recurrence + all parameter gradients.  dW_hh [1024][256] must be ZERO on entry (split-K
// atomics); dW_ih / db_ih / db_hh are overwritten; dx may be null.
int b200dp_lstm_rec_bwd(const float* x, const float* h0, const float* c0, const float* w_ih, const float* w_hh,
                        const float* seq, const float* gates, const float* cs, const float* dseq, const float* dhT,
                        const float* dcT, float* dgates_ws, float* dh0, float* dc0, float* dW_ih, float* dW_hh,
                        float* db_ih, float* db_hh, float* dx, int B, int T, int F, unsigned long long stream) {
  if (!b200dp_lstm_rec_supported(LH, F)) return lfail("unsupported LSTM shape");
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  RecBwdParams p{w_hh, gates, cs, c0, dseq, dhT, dcT, dgates_ws, dh0, dc0, B, T};
  const int tiles = (B + NB - 1) / NB;
  int clusters = sms() / CL;
  if (clusters > tiles) clusters = tiles;
  if (clusters < 1) clusters = 1;
  if (launch_cluster(lstm_rec_bwd_kernel, p, clusters, BW_SMEM, st)) return -1;
  WgParams w{dgates_ws, seq, h0, x, w_ih, dW_hh, dW_ih, db_ih, db_hh, dx, B, T, F, 4};
  const int TB = T * B;
  if (TB < 256) w.ksplit = 2;
  const int blocks = (LG / WG_TR) * (LH / WG_TK) * w.ksplit + LG / 8 + (dx != nullptr ? (TB + 7) / 8 : 0);
  lstm_wgrad_kernel<<<blocks, 256, 0, st>>>(w);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return lfail(cudaGetErrorString(e), (int)e);
  return 0;
}

}  // extern "C"

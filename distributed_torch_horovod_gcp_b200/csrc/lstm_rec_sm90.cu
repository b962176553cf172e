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
// the recurrence into one small kernel.  Inter-layer dropout is a keep-bit mask per dropped layer output, drawn
// by a Philox kernel and applied by the next layer's input-side products (lstm_in_mma_kernel<MODE, true>).
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
struct RecFwdParams {   // one direction
  const float* w_hh;    // [1024][256]
  const float* xp;      // [T][B][1024]
  const float* h0;      // [B][256]
  const float* c0;      // [B][256]
  float* seq;           // [B][T][ld], this direction's 256 columns (pointer already at its column offset)
  float* hT;            // [B][256]
  float* cT;            // [B][256]
  float* gates;         // [T][B][1024] post-activation i,f,g,o   (nullptr: inference, nothing saved)
  float* cs;            // [T][B][256]  c_t                       (nullptr: inference)
  int reverse;          // walk t = T-1 .. 0
};
// The directions of a layer are independent chains: clusters [d * cpd, (d + 1) * cpd) run direction d
// (cpd = clusters per direction), so every cluster loads one W_hh once and no cluster waits on another.
struct RecFwdLaunch {
  RecFwdParams d[2];
  int ndir, B, T, ld;   // ld: row stride of seq (256 * ndir)
};

constexpr int FW_A_BYTES = 128 * 1024;               // 8 chunks x [128 rows x 128 B]
constexpr int FW_B_BYTES = 32 * 1024;                // 8 chunks x [32 rows x 128 B], double buffered
constexpr int FW_G_BYTES = 16 * 1024;                // gate exchange [4][32][32] fp32
constexpr int FW_SMEM = FW_A_BYTES + 2 * FW_B_BYTES + FW_G_BYTES + IMG_BYTES + 1024;

__global__ void __launch_bounds__(LTHREADS, 1) lstm_rec_fwd_kernel(const RecFwdLaunch L) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + FW_A_BYTES;
  uint8_t* sG = sB + 2 * FW_B_BYTES;
  const uint32_t img = smem_u32(sG + FW_G_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t c = my_cluster_rank();
  const int cpd = gridDim.x / CL / L.ndir;
  const int dir = (int)(blockIdx.x / CL) / cpd;
  const int cluster_id = (int)(blockIdx.x / CL) - dir * cpd, num_clusters = cpd;
  const RecFwdParams p = dir ? L.d[1] : L.d[0];
  const int B = L.B, T = L.T;

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

  const int num_tiles = (B + NB - 1) / NB;
  for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
    const int b0 = tile * NB;
    // ---- h_{-1} = h0 into B buffer 0 (every CTA needs all 256 hidden units); c0 into registers
    for (int i = tid; i < NB * 64; i += LTHREADS) {
      const int b = i >> 6, k4 = i & 63;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b0 + b < B) v = *reinterpret_cast<const float4*>(p.h0 + (size_t)(b0 + b) * LH + k4 * 4);
      sts_v4(smem_u32(sB) + sw_off(b, k4 * 4, NB), v.x, v.y, v.z, v.w);
    }
    float cstate[8], hlast[8];
    const int ju = lane;                       // unit owned by this thread in the cell update
    const int bb = warp * 8;                   // its 8 batch rows
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + bb + i;
      cstate[i] = (b < B) ? p.c0[(size_t)b * LH + c * LU + ju] : 0.f;
      hlast[i] = 0.f;
    }
    fence_proxy_async_all();
    cluster_barrier();                         // nobody writes into a peer's buffers before it finished the last tile

    for (int s = 0; s < T; ++s) {
      const int t = p.reverse ? T - 1 - s : s;
      const int cur = s & 1, nxt = cur ^ 1;
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
          xv[b] = (b0 + b < B) ? __ldg(p.xp + ((size_t)t * B + b0 + b) * LG + grow) : 0.f;
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
            if (b0 + b < B) p.gates[((size_t)t * B + b0 + b) * LG + grow] = v[b];
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
          if (b < B) {
            p.seq[((size_t)b * T + t) * L.ld + kglob] = hlast[i];
            if (p.cs != nullptr) p.cs[((size_t)t * B + b) * LH + kglob] = cstate[i];
          }
        }
        if (s + 1 < T) {
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
      if (b < B) {
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
struct RecBwdParams {   // one direction
  const float* __restrict__ w_hh;    // [1024][256]
  const float* __restrict__ gates;   // [T][B][1024]
  const float* __restrict__ cs;      // [T][B][256]
  const float* __restrict__ c0;      // [B][256]
  const float* __restrict__ dseq;    // [B][T][ld] at this direction's column offset (may be nullptr)
  const float* __restrict__ dhT;     // [B][256]      (may be nullptr)
  const float* __restrict__ dcT;     // [B][256]      (may be nullptr)
  float* __restrict__ dgates;        // [T][B][1024]
  float* dh0;           // [B][256]
  float* dc0;           // [B][256]
  int reverse;          // the forward walked t = T-1 .. 0, so this walks t = 0 .. T-1
};
struct RecBwdLaunch {   // clusters are split between the directions as in RecFwdLaunch
  RecBwdParams d[2];
  int ndir, B, T, ld;
};
constexpr int BW_A_BYTES = 128 * 1024;               // W_slice^T: 4 chunks x [256 rows (k) x 128 B (32 gate rows)]
constexpr int BW_B_BYTES = 16 * 1024;                // dgates: 4 chunks x [32 rows (b) x 128 B]
constexpr int BW_R_BYTES = 32 * 1024;                // partial dh from 8 sources [8][32 j][32 b], double buffered
constexpr int BW_SMEM = BW_A_BYTES + BW_B_BYTES + 2 * BW_R_BYTES + IMG_BYTES + 1024;

__global__ void __launch_bounds__(LTHREADS, 1) lstm_rec_bwd_kernel(const RecBwdLaunch L) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + BW_A_BYTES;
  uint8_t* sR = sB + BW_B_BYTES;
  const uint32_t img = smem_u32(sR + 2 * BW_R_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t c = my_cluster_rank();
  const int cpd = gridDim.x / CL / L.ndir;
  const int dir = (int)(blockIdx.x / CL) / cpd;
  const int cluster_id = (int)(blockIdx.x / CL) - dir * cpd, num_clusters = cpd;
  const RecBwdParams p = dir ? L.d[1] : L.d[0];
  const int B = L.B, T = L.T;

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

  const int num_tiles = (B + NB - 1) / NB;
  for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
    const int b0 = tile * NB;
    const int ju = lane, bb = warp * 8;
    const int kglob = (int)c * LU + ju;
    float dc_next[8], dh_rec[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + bb + i;
      dc_next[i] = (p.dcT != nullptr && b < B) ? p.dcT[(size_t)b * LH + kglob] : 0.f;
      dh_rec[i] = (p.dhT != nullptr && b < B) ? p.dhT[(size_t)b * LH + kglob] : 0.f;
    }
    cluster_barrier();

    for (int s = 0; s < T; ++s) {
      const int t = p.reverse ? s : T - 1 - s;
      const int tp = p.reverse ? t + 1 : t - 1;  // the step that produced c_{t-1} / h_{t-1}
      const int cur = s & 1;                     // reduce buffer written during this step
      {
        // ---- dgates for (unit ju, batch bb..bb+7)
        const uint32_t sB_u = smem_u32(sB);
        // all global operands of the 8 batch rows first (one memory round trip instead of eight)
        float gi[8], gf[8], gg[8], go[8], ct[8], cprev[8], dsq[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int b = b0 + bb + i;
          const bool ok = b < B;
          const size_t gbase = ((size_t)t * B + (ok ? b : 0)) * LG + kglob;
          gi[i] = ok ? __ldg(p.gates + gbase) : 0.f;
          gf[i] = ok ? __ldg(p.gates + gbase + LH) : 0.f;
          gg[i] = ok ? __ldg(p.gates + gbase + 2 * LH) : 0.f;
          go[i] = ok ? __ldg(p.gates + gbase + 3 * LH) : 0.f;
          ct[i] = ok ? __ldg(p.cs + ((size_t)t * B + b) * LH + kglob) : 0.f;
          cprev[i] = !ok ? 0.f
                         : ((s + 1 < T) ? __ldg(p.cs + ((size_t)tp * B + b) * LH + kglob)
                                    : __ldg(p.c0 + (size_t)b * LH + kglob));
          dsq[i] = (ok && p.dseq != nullptr) ? __ldg(p.dseq + ((size_t)b * T + t) * L.ld + kglob) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int b = b0 + bb + i;
          float di = 0.f, df = 0.f, dg = 0.f, dob = 0.f;
          if (b < B) {
            const size_t gbase = ((size_t)t * B + b) * LG + kglob;
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
        for (int src = 0; src < CL; ++src) {
          const float4 v0 = lds_v4(red + (uint32_t)(((src * 32 + ju) * 32 + bb) * 4));
          const float4 v1 = lds_v4(red + (uint32_t)(((src * 32 + ju) * 32 + bb + 4) * 4));
          dh_rec[0] += v0.x; dh_rec[1] += v0.y; dh_rec[2] += v0.z; dh_rec[3] += v0.w;
          dh_rec[4] += v1.x; dh_rec[5] += v1.y; dh_rec[6] += v1.z; dh_rec[7] += v1.w;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + bb + i;
      if (b < B) {
        if (p.dh0 != nullptr) p.dh0[(size_t)b * LH + kglob] = dh_rec[i];
        if (p.dc0 != nullptr) p.dc0[(size_t)b * LH + kglob] = dc_next[i];
      }
    }
  }
  cluster_barrier();
}

// ---------------------------------------------------------------------------------------------------
// weight / bias / input gradients: sums over (t, b), off the serial chain -> all SMs, fp32 SIMT
//   dW_hh[r][k] = sum dG[t][b][r] * hprev[t][b][k]     (hprev[0] = h0, hprev[t] = seq[:, t-1]; a reverse
//                                                       direction: hprev[T-1] = h0, hprev[t] = seq[:, t+1])
//   dW_ih[r][f] = sum dG[t][b][r] * x[b][t][f],   db[r] = sum dG[t][b][r]              (F <= 32)
//   dx[b][t][f] = sum_r dG[t][b][r] * W_ih[r][f]                          (optional, one direction)
// One launch per direction.  For F > 32 the dW_ih / db blocks are not launched and for two directions no dx
// blocks are: lstm_ih_wgrad_kernel / lstm_dx_kernel compute those.
// ---------------------------------------------------------------------------------------------------
struct WgParams {
  const float* dG; const float* seq; const float* h0; const float* x; const float* w_ih;
  float* dW_hh; float* dW_ih; float* db_ih; float* db_hh; float* dx;
  int B, T, F, ksplit;
  int ld, reverse;      // row stride of seq (at this direction's column offset); direction
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
          const int tp = p.reverse ? t + 1 : t - 1;
          hv = (tp < 0 || tp == p.T) ? p.h0[(size_t)b * LH + k0 + rr]
                                     : p.seq[((size_t)b * p.T + tp) * p.ld + k0 + rr];
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

// ---------------------------------------------------------------------------------------------------
// input-side products for inputs wider than the register-array paths above (F > 32: the layers above the
// first see 256 or 512 features), and dx of a layer with two directions.  Each is a [T*B] x F x 1024 product
// on tf32 wgmma with fp32 accumulation, the numerics of the recurrence:
//   xp[t][b][r]  = sum_f x[b][t][f] W_ih[r][f] + (b_ih[r] + b_hh[r])      MODE_XPROJ  M = (t,b), N = r, K = f
//   dW_ih[r][f]  = sum_(t,b) dG[t][b][r] x[b][t][f]                         MODE_WGRAD  M = r, N = f, K = (t,b)
//   db[r]        = sum_(t,b) dG[t][b][r]     (column N = F of the same product, against a column of ones)
//   dx[b][t][f]  = sum_r dG_fwd W_ih_fwd  (+ sum_r dG_rev W_ih_rev)        MODE_DX     M = (t,b), N = f, K = r
// One warpgroup per CTA, a 128 x 64 output tile (two m64 halves x two n32 halves), K staged 32 at a time into
// 128B-swizzled K-major shared memory.  tf32 wgmma has no transposed-operand mode, so operands that are
// MN-major in memory (dG and x for dW_ih, W_ih for dx) are read along MN (coalesced) and transposed by the
// shared-memory store; the next chunk's loads are in flight while the current chunk's MMAs run.
// Every sum has a fixed order and no atomics: a CTA owns the whole K of its tile, except that dW_ih / db split
// (t, b) into ranges whose partial tiles go to their own workspace slices, summed in split order by
// lstm_ih_wgrad_finish_kernel.  dx of two directions is (forward sum) + (reverse sum), in that order.
// ---------------------------------------------------------------------------------------------------
struct IhDir {          // one direction's input-side operands
  const float* w_ih; const float* b_ih; const float* b_hh; float* xp;   // forward
  const float* dG; float* dW_ih; float* db_ih; float* db_hh;            // backward
};
constexpr int XPROJ_SIMT_MAX_F = 32;   // F up to this uses lstm_xproj_kernel / the lstm_wgrad_kernel branches
constexpr int IM = 128, IN = 64, IK = 32;
constexpr int MODE_XPROJ = 0, MODE_WGRAD = 1, MODE_DX = 2;

struct InMmaArgs {
  IhDir d0, d1;
  const float* x;       // layer input [B][T][F]
  float* out;           // MODE_DX: dx [B][T][F];  MODE_WGRAD: workspace [ndir][splits][1024][F + 1]
  int B, T, F, ndir, splits, per;   // per: (t, b) rows of one dW_ih split (a multiple of IK)
  // inter-layer dropout of x (read only by the DROP instantiations): one keep bit per element of x, element
  // e = (b T + t) F + f at bit e % 32 of word e / 32; kept elements are multiplied by `scale` = 1 / (1 - p)
  const uint32_t* keep;
  float scale;
};

// ---------------------------------------------------------------------------------------------------
// inter-layer dropout mask: keep[w] bit i = (element 32 w + i of the layer's output is kept), drawn with
// Philox4x32-10 (Salmon et al., SC'11): key = seed[0], counter = (e / 4, seed[1]), output word e % 4,
// kept when it is below `thr` = (1 - p) 2^32.  The seed lives in device memory (drawn by torch's CUDA
// generator), so a replayed CUDA graph draws a fresh mask.  philox4x32_10 is in philox.cuh.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) lstm_dropout_mask_kernel(uint32_t* __restrict__ keep,
                                                                const unsigned long long* __restrict__ seed,
                                                                size_t words, uint32_t thr) {
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= words) return;
  const unsigned long long k = seed[0], off = seed[1];
  const uint2 key = make_uint2((uint32_t)k, (uint32_t)(k >> 32));
  uint32_t bits = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const unsigned long long q = w * 8 + j;             // index of the element quad 4 q .. 4 q + 3
    const uint4 u = philox4x32_10(make_uint4((uint32_t)q, (uint32_t)(q >> 32), (uint32_t)off, (uint32_t)(off >> 32)),
                                  key);
    bits |= ((uint32_t)(u.x < thr) | (uint32_t)(u.y < thr) << 1 | (uint32_t)(u.z < thr) << 2 |
             (uint32_t)(u.w < thr) << 3) << (4 * j);
  }
  keep[w] = bits;
}

__device__ __forceinline__ bool kept(const uint32_t* keep, size_t e) { return (__ldg(keep + (e >> 5)) >> (e & 31)) & 1u; }

// Stage ROWS x 32 fp32 of an operand into K-major swizzled shared memory: element (row, k) of the chunk.
// K_CONTIG: consecutive k are adjacent in memory (a warp reads one row); otherwise consecutive rows are (a warp
// reads 32 rows of one k and the store transposes them).
template <int ROWS, bool K_CONTIG, typename Get>
__device__ __forceinline__ void stage(uint32_t s, Get get) {
#pragma unroll 4
  for (int u = 0; u < ROWS * IK / 128; ++u) {
    const int i = threadIdx.x + 128 * u;
    const int row = K_CONTIG ? i / IK : i % ROWS, k = K_CONTIG ? i % IK : i / ROWS;
    sts_f32(s + sw_off(row, k, ROWS), get(row, k));
  }
}

constexpr int IBUF = (IM + IN) * IK * 4;   // one stage: A [128 x 32] + B [64 x 32] fp32

// acc[mh][nq] += A[128 x K] B[64 x K]^T over chunks [0, nk) of K.  Two stages: the loads and stores of chunk
// kc + 1 run while the MMAs of chunk kc do.
template <bool A_K, bool B_K, typename GetA, typename GetB>
__device__ __forceinline__ void in_mma_loop(float (&acc)[2][2][16], uint32_t smem, int nk, GetA ga, GetB gb) {
  for (int kc = 0; kc < nk; ++kc) {
    const uint32_t sA = smem + (kc & 1) * IBUF, sB = sA + IM * IK * 4;
    const int k0 = kc * IK;
    stage<IM, A_K>(sA, [&](int r, int k) { return ga(r, k0 + k); });
    stage<IN, B_K>(sB, [&](int r, int k) { return gb(r, k0 + k); });
    fence_proxy_async_all();
    __syncthreads();
    const uint64_t da = make_desc_base(16, 1024) + desc_addr(sA);
    const uint64_t db = make_desc_base(16, 1024) + desc_addr(sB);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < IK / 8; ++ks)
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int nq = 0; nq < 2; ++nq)
          wgmma_tf32_n32(acc[mh][nq], da + (uint64_t)((mh * 64 * 128 + ks * 32) >> 4),
                         db + (uint64_t)((nq * 32 * 128 + ks * 32) >> 4), 1u);
    wg_commit();
    wg_wait<1>();                                        // chunk kc - 1 is done: its stage is free again
  }
  wg_wait<0>();
#pragma unroll
  for (int mh = 0; mh < 2; ++mh)
#pragma unroll
    for (int nq = 0; nq < 2; ++nq) wg_fence_operands<16>(acc[mh][nq]);
  __syncthreads();                                       // the stages may be restaged by a following loop
}

// element (m, n) of the tile held by this thread: fragment value acc[mh][nq][4 j + 2 h + e]
template <typename Put>
__device__ __forceinline__ void in_mma_epilogue(const float (&acc)[2][2][16], Put put) {
  const int t = threadIdx.x;
#pragma unroll
  for (int mh = 0; mh < 2; ++mh)
#pragma unroll
    for (int nq = 0; nq < 2; ++nq)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            put(mh * 64 + (t >> 5) * 16 + ((t & 31) >> 2) + 8 * h, nq * 32 + 8 * j + 2 * (t & 3) + e,
                acc[mh][nq][4 * j + 2 * h + e]);
}

// DROP: x is the output of the layer below seen through inter-layer dropout (a.keep / a.scale): the x-projection
// and dW_ih read x * keep * scale, and dx is stored as keep ? dx * scale : 0 (the gradient of the layer below's
// output).
template <int MODE, bool DROP>
__global__ void __launch_bounds__(128, 1) lstm_in_mma_kernel(const InMmaArgs a) {
  __shared__ __align__(1024) uint8_t smem_raw[2 * IBUF];
  const uint32_t smem = smem_u32(smem_raw);
  const int B = a.B, T = a.T, F = a.F, TB = T * B;
  const int m0 = blockIdx.x * IM, n0 = blockIdx.y * IN;
  // x row of (t, b) index q (x is [B][T][F])
  auto xrow = [&](int q) { return a.x + ((size_t)(q % B) * T + q / B) * F; };
  // element f of that row, as the layer reads it
  auto xval = [&](int q, int f) {
    const float v = __ldg(xrow(q) + f);
    if constexpr (DROP) return kept(a.keep, ((size_t)(q % B) * T + q / B) * F + f) ? v * a.scale : 0.f;
    return v;
  };
  // dx element (q, f) as stored: masked for the layer below when DROP
  auto dxval = [&](int q, int f, float v) {
    if constexpr (DROP) return kept(a.keep, ((size_t)(q % B) * T + q / B) * F + f) ? v * a.scale : 0.f;
    return v;
  };
  float acc[2][2][16];
#pragma unroll
  for (int mh = 0; mh < 2; ++mh)
#pragma unroll
    for (int nq = 0; nq < 2; ++nq)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[mh][nq][i] = 0.f;

  if constexpr (MODE == MODE_XPROJ) {
    const IhDir d = blockIdx.z ? a.d1 : a.d0;
    in_mma_loop<true, true>(
        acc, smem, (F + IK - 1) / IK,
        [&](int r, int k) { const int q = m0 + r; return (q < TB && k < F) ? xval(q, k) : 0.f; },
        [&](int r, int k) { return k < F ? __ldg(d.w_ih + (size_t)(n0 + r) * F + k) : 0.f; });
    in_mma_epilogue(acc, [&](int m, int n, float v) {
      const int q = m0 + m, r = n0 + n;
      if (q < TB) d.xp[(size_t)q * LG + r] = v + (d.b_ih[r] + d.b_hh[r]);
    });
  } else if constexpr (MODE == MODE_WGRAD) {
    const int dir = blockIdx.z / a.splits, split = blockIdx.z % a.splits;
    const IhDir d = dir ? a.d1 : a.d0;
    const int q0 = split * a.per, q1 = min(q0 + a.per, TB);
    in_mma_loop<false, false>(
        acc, smem, (q1 - q0 + IK - 1) / IK,
        [&](int r, int k) { const int q = q0 + k; return q < q1 ? __ldg(d.dG + (size_t)q * LG + m0 + r) : 0.f; },
        [&](int r, int k) {
          const int q = q0 + k, f = n0 + r;
          if (q >= q1 || f > F) return 0.f;
          return f == F ? 1.f : xval(q, f);
        });
    float* ws = a.out + ((size_t)dir * a.splits + split) * LG * (F + 1);
    in_mma_epilogue(acc, [&](int m, int n, float v) {
      if (n0 + n <= F) ws[(size_t)(m0 + m) * (F + 1) + n0 + n] = v;
    });
  } else {
    in_mma_loop<true, false>(
        acc, smem, LG / IK,
        [&](int r, int k) { const int q = m0 + r; return q < TB ? __ldg(a.d0.dG + (size_t)q * LG + k) : 0.f; },
        [&](int r, int k) { const int f = n0 + r; return f < F ? __ldg(a.d0.w_ih + (size_t)k * F + f) : 0.f; });
    in_mma_epilogue(acc, [&](int m, int n, float v) {
      const int q = m0 + m, f = n0 + n;
      if (q < TB && f < F) a.out[((size_t)(q % B) * T + q / B) * F + f] = (DROP && a.ndir == 1) ? dxval(q, f, v) : v;
    });
    if (a.ndir == 2) {                                   // + the reverse direction's sum, read back by its writer
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int nq = 0; nq < 2; ++nq)
#pragma unroll
          for (int i = 0; i < 16; ++i) acc[mh][nq][i] = 0.f;
      in_mma_loop<true, false>(
          acc, smem, LG / IK,
          [&](int r, int k) { const int q = m0 + r; return q < TB ? __ldg(a.d1.dG + (size_t)q * LG + k) : 0.f; },
          [&](int r, int k) { const int f = n0 + r; return f < F ? __ldg(a.d1.w_ih + (size_t)k * F + f) : 0.f; });
      in_mma_epilogue(acc, [&](int m, int n, float v) {
        const int q = m0 + m, f = n0 + n;
        if (q < TB && f < F) {
          float* o = a.out + ((size_t)(q % B) * T + q / B) * F + f;
          *o = dxval(q, f, *o + v);
        }
      });
    }
  }
}

// dW_ih / db of every direction: the split slices of each element summed in split order
__global__ void __launch_bounds__(256) lstm_ih_wgrad_finish_kernel(const InMmaArgs a) {
  const int F1 = a.F + 1;
  const size_t per_dir = (size_t)LG * F1;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= per_dir * a.ndir) return;
  const int dir = (int)(i / per_dir);
  const size_t e = i % per_dir;
  const float* ws = a.out + (size_t)dir * a.splits * per_dir + e;
  float s = ws[0];
  for (int k = 1; k < a.splits; ++k) s += ws[(size_t)k * per_dir];
  const IhDir d = dir ? a.d1 : a.d0;
  const int r = (int)(e / F1), f = (int)(e % F1);
  if (f < a.F) {
    d.dW_ih[(size_t)r * a.F + f] = s;
  } else {
    d.db_ih[r] = s;
    d.db_hh[r] = s;
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

constexpr int MAX_F = 512;   // widest input: the 512 outputs of a bidirectional layer

int cluster_split(int B, int ndir) {   // clusters per direction
  const int tiles = (B + NB - 1) / NB;
  int cpd = sms() / CL / ndir;
  if (cpd > tiles) cpd = tiles;
  if (cpd < 1) cpd = 1;
  return cpd;
}

// drop_in / drop_out: the layer's input / output goes through inter-layer dropout with probability p.  A dropped
// input is the output of a layer below (256 or 512 features), which only the tf32 input products read.
int check_shape(int ndir, int B, int T, int F, double p, bool drop_in, bool drop_out) {
  if (F < 1 || F > MAX_F || ndir < 1 || ndir > 2 || B < 1 || T < 1)
    return lfail("unsupported LSTM shape: H=256 needs F in 1..512, 1 or 2 directions, B >= 1, T >= 1", F);
  if ((drop_in || drop_out) && !(p > 0.0 && p <= 1.0))
    return lfail("unsupported LSTM dropout: a dropout mask needs 0 < p <= 1", (int)(p * 100));
  if (drop_in && F <= XPROJ_SIMT_MAX_F)
    return lfail("unsupported LSTM dropout: only the input of a layer above the first (F > 32) is dropped", F);
  return 0;
}

template <int MODE>
void launch_in_mma(const InMmaArgs& a, dim3 grid, cudaStream_t st) {
  if (a.keep != nullptr)
    lstm_in_mma_kernel<MODE, true><<<grid, 128, 0, st>>>(a);
  else
    lstm_in_mma_kernel<MODE, false><<<grid, 128, 0, st>>>(a);
}

float dropout_scale(double p) { return p < 1.0 ? (float)(1.0 / (1.0 - p)) : 0.f; }

enum { FW_W_IH, FW_W_HH, FW_B_IH, FW_B_HH, FW_H0, FW_C0, FW_XP, FW_GATES, FW_CS, FW_HT, FW_CT, FW_NPTR };
enum { BW_W_IH, BW_W_HH, BW_H0, BW_C0, BW_GATES, BW_CS, BW_DHT, BW_DCT, BW_DGATES, BW_DH0, BW_DC0, BW_DW_IH,
       BW_DW_HH, BW_DB_IH, BW_DB_HH, BW_NPTR };

// dW_ih / db of one layer on tf32 wgmma: the (t, b) sum is split so that the tiles fill the GPU; each split's
// partial tile goes to its own workspace slice (allocated on the stream, so CUDA graphs capture it) and the
// finish kernel sums the slices in split order.
int launch_ih_wgrad(InMmaArgs a, cudaStream_t st) {
  const int TB = a.T * a.B;
  const int tiles = (LG / IM) * ((a.F + 1 + IN - 1) / IN) * a.ndir;
  int splits = (2 * sms() + tiles - 1) / tiles;
  const int max_splits = (TB + 4 * IK - 1) / (4 * IK);          // at least 128 (t, b) rows per split
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  a.per = ((TB + splits - 1) / splits + IK - 1) / IK * IK;
  a.splits = (TB + a.per - 1) / a.per;
  const size_t n = (size_t)a.ndir * a.splits * LG * (a.F + 1);
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&a.out), n * sizeof(float), st);
  if (e != cudaSuccess) return lfail(cudaGetErrorString(e), (int)e);
  launch_in_mma<MODE_WGRAD>(a, dim3(LG / IM, (a.F + 1 + IN - 1) / IN, a.ndir * a.splits), st);
  const size_t outs = (size_t)a.ndir * LG * (a.F + 1);
  lstm_ih_wgrad_finish_kernel<<<(unsigned)((outs + 255) / 256), 256, 0, st>>>(a);
  e = cudaFreeAsync(a.out, st);
  if (e != cudaSuccess) return lfail(cudaGetErrorString(e), (int)e);
  return 0;
}

}  // namespace

extern "C" {

const char* b200dp_lstm_rec_last_error() { return g_lerr; }

// Hidden size 256; input widths 1..512 (layer 0 of a model, or 256 / 512 above a one- / two-direction layer).
int b200dp_lstm_rec_supported(int H, int F) { return (H == LH && F >= 1 && F <= MAX_F) ? 1 : 0; }

// One layer, one or both directions (direction 1 is the reverse one).  x [B][T][F]; seq [B][T][256 * ndir],
// direction d writes columns [256 d, 256 d + 256).  `dir_ptrs` holds FW_NPTR pointers per direction, in the
// order of the FW_* enum: weights in PyTorch layout, h0/c0/hT/cT [B][256] (slices of the [layers * ndir][B][256]
// state), the xp workspace [T][B][1024], and gates/cs saved for backward ([T][B][1024] / [T][B][256]) or null.
// Inter-layer dropout with probability p (null pointers: none): `in_keep` is the keep-bit mask of x (the output
// of the layer below, as drawn by its forward), which the x-projection applies; `out_keep` [B * T * ndir * 8]
// words receives a fresh mask of seq drawn from `out_seed` (2 words in device memory: Philox key and offset).
int b200dp_lstm_rec_fwd(const float* x, float* seq, const void* const* dir_ptrs, int ndir, int B, int T, int F,
                        double p, const uint32_t* in_keep, const unsigned long long* out_seed, uint32_t* out_keep,
                        unsigned long long stream) {
  if (check_shape(ndir, B, T, F, p, in_keep != nullptr, out_keep != nullptr)) return -1;
  if (out_keep != nullptr && out_seed == nullptr) return lfail("LSTM dropout: an output mask needs a seed");
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int rows = T * B;
  if (out_keep != nullptr) {
    const size_t words = (size_t)rows * ndir * (LH / 32);
    const double k = (1.0 - p) * 4294967296.0;        // keep when a 32-bit draw is below (1 - p) 2^32
    const uint32_t thr = k >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)k;
    lstm_dropout_mask_kernel<<<(unsigned)((words + 255) / 256), 256, 0, st>>>(out_keep, out_seed, words, thr);
  }
  RecFwdLaunch L{};
  IhDir ih[2] = {};
  L.ndir = ndir; L.B = B; L.T = T; L.ld = LH * ndir;
  for (int d = 0; d < ndir; ++d) {
    const float* const* v = reinterpret_cast<const float* const*>(dir_ptrs) + d * FW_NPTR;
    float* xp = const_cast<float*>(v[FW_XP]);
    if (F <= XPROJ_SIMT_MAX_F)
      lstm_xproj_kernel<<<(rows + 7) / 8, 256, 8 * F * sizeof(float), st>>>(x, v[FW_W_IH], v[FW_B_IH], v[FW_B_HH],
                                                                            xp, B, T, F);
    ih[d].w_ih = v[FW_W_IH]; ih[d].b_ih = v[FW_B_IH]; ih[d].b_hh = v[FW_B_HH]; ih[d].xp = xp;
    L.d[d] = RecFwdParams{v[FW_W_HH], xp, v[FW_H0], v[FW_C0], seq + d * LH, const_cast<float*>(v[FW_HT]),
                          const_cast<float*>(v[FW_CT]), const_cast<float*>(v[FW_GATES]),
                          const_cast<float*>(v[FW_CS]), d};
  }
  if (F > XPROJ_SIMT_MAX_F) {
    const InMmaArgs a{ih[0], ih[ndir - 1], x, nullptr, B, T, F, ndir, 1, 0, in_keep, dropout_scale(p)};
    launch_in_mma<MODE_XPROJ>(a, dim3((rows + IM - 1) / IM, LG / IN, ndir), st);
  }
  return launch_cluster(lstm_rec_fwd_kernel, L, cluster_split(B, ndir) * ndir, FW_SMEM, st);
}

// Backward of one layer + all its parameter gradients.  seq / dseq [B][T][256 * ndir] as in the forward (dseq
// may be null); dx [B][T][F] or null; with two directions dx is the sum of both.  `dir_ptrs` holds BW_NPTR
// pointers per direction in the order of the BW_* enum (dhT/dcT/dh0/dc0 may be null).  dW_hh [1024][256] must be
// ZERO on entry (split-K atomics); dW_ih / db_ih / db_hh are overwritten.  `in_keep` (or null) is the forward's
// dropout mask of x with probability p: dW_ih reads the dropped x, and dx is the gradient of the undropped x
// (the layer below's output), i.e. zero where x was dropped.
int b200dp_lstm_rec_bwd(const float* x, const float* seq, const float* dseq, float* dx, const void* const* dir_ptrs,
                        int ndir, int B, int T, int F, double p, const uint32_t* in_keep, unsigned long long stream) {
  if (check_shape(ndir, B, T, F, p, in_keep != nullptr, false)) return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int TB = T * B;
  RecBwdLaunch L{};
  WgParams w[2] = {};
  IhDir ih[2] = {};
  L.ndir = ndir; L.B = B; L.T = T; L.ld = LH * ndir;
  const bool ih_simt = F <= XPROJ_SIMT_MAX_F;
  const bool dx_simt = ih_simt && ndir == 1 && dx != nullptr;
  for (int d = 0; d < ndir; ++d) {
    const float* const* v = reinterpret_cast<const float* const*>(dir_ptrs) + d * BW_NPTR;
    float* dG = const_cast<float*>(v[BW_DGATES]);
    L.d[d] = RecBwdParams{v[BW_W_HH], v[BW_GATES], v[BW_CS], v[BW_C0], dseq != nullptr ? dseq + d * LH : nullptr,
                          v[BW_DHT], v[BW_DCT], dG, const_cast<float*>(v[BW_DH0]), const_cast<float*>(v[BW_DC0]), d};
    w[d] = WgParams{dG, seq + d * LH, v[BW_H0], x, v[BW_W_IH], const_cast<float*>(v[BW_DW_HH]),
                    const_cast<float*>(v[BW_DW_IH]), const_cast<float*>(v[BW_DB_IH]), const_cast<float*>(v[BW_DB_HH]),
                    dx_simt ? dx : nullptr, B, T, F, TB < 256 ? 2 : 4, LH * ndir, d};
    ih[d] = IhDir{v[BW_W_IH], nullptr, nullptr, nullptr, dG, const_cast<float*>(v[BW_DW_IH]),
                  const_cast<float*>(v[BW_DB_IH]), const_cast<float*>(v[BW_DB_HH])};
  }
  if (launch_cluster(lstm_rec_bwd_kernel, L, cluster_split(B, ndir) * ndir, BW_SMEM, st)) return -1;
  const int blocks = (LG / WG_TR) * (LH / WG_TK) * w[0].ksplit + (ih_simt ? LG / 8 : 0) + (dx_simt ? (TB + 7) / 8 : 0);
  for (int d = 0; d < ndir; ++d) lstm_wgrad_kernel<<<blocks, 256, 0, st>>>(w[d]);
  const float scale = dropout_scale(p);
  if (!ih_simt &&
      launch_ih_wgrad(InMmaArgs{ih[0], ih[ndir - 1], x, nullptr, B, T, F, ndir, 1, 0, in_keep, scale}, st))
    return -1;
  if (dx != nullptr && !dx_simt) {
    const InMmaArgs a{ih[0], ih[ndir - 1], x, dx, B, T, F, ndir, 1, 0, in_keep, scale};
    launch_in_mma<MODE_DX>(a, dim3((TB + IM - 1) / IM, (F + IN - 1) / IN), st);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return lfail(cudaGetErrorString(e), (int)e);
  return 0;
}

}  // extern "C"

// Fused LM-head cross-entropy for sm_90a: the loss of the logits z = x W^T without ever storing them.
//
//   loss_i = lse_i - z_{i, t_i},  lse_i = log sum_j exp(z_ij)       x [N, D], W [V, D] bf16 (both K-major)
//
// Both kernels have the GEMM's structure (sm90_common.cuh): persistent, one CTA per SM, warpgroup 0 a TMA
// producer filling the Cfg<128> operand ring, warpgroups 1-2 wg_mainloop into a 128 x 128 fp32 register
// fragment (thread t of warpgroup wg: tile rows r = 64 wg + 16 (t / 32) + (t % 32) / 4 and r + 8, columns
// 8j + 2 (t % 4) + {0, 1}).  Only the epilogue differs from the GEMM's.
//
// Forward (xent_fwd_kernel): a work item is one 128-row block and a contiguous range of 128-wide vocab tiles.
// Items are numbered range-major, so the CTAs running at one time walk the same W tiles (W does not fit in L2
// at GPT-2's 50304 x 768; x does).  Per tile, each thread folds its fragment into a running (max, sum of ex2)
// per row, in log2 units; columns >= V are -inf.  The thread holding column t_i stores that fp32 logit to
// zt[i]: a column index is compared with the target, memory is never indexed by it.  At the end of a range the
// four lanes of a row combine their pairs in a fixed order and write one partial per (range, row).
// xent_finish_kernel folds each row's partials in range order into lse_i and loss_i (0 for an ignored row,
// NaN for a target outside [0, V)) and one (sum, count) per block; xent_total_kernel adds the blocks in order.
// Nothing waits on the host or on another CTA, and every sum has a fixed order.
//
// Backward (xent_grad_kernel), over the rows of one chunk: the same tiles again, one per item (row blocks
// fastest, so concurrent CTAs share a W tile), and dlogits = s_i (exp(z - lse_i) - [j == t_i]) in bf16 through
// the staging tile and bulk stores of the GEMM epilogue.  s_i (the incoming gradient, divided by the count for
// "mean"; 0 for an ignored row, NaN for an out-of-range target) is read from device memory.  dX and dW of the
// chunk are GEMMs on that buffer (ops/xent.py).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "sm90_common.cuh"

namespace {

constexpr int XBN = 128;                                   // vocab columns per tile
using XC = Cfg<XBN>;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr int FIN_THREADS = 256;

struct XentParams {
  int N, V;
  int num_m, num_v, num_kb;  // 128-row blocks (of the chunk, backward), 128-column vocab tiles, 64-deep K blocks
  int ranges;                // vocab ranges per row block (backward: num_v, one tile each)
  int row0, rows;            // rows row0 .. row0 + rows - 1 of x (forward: 0, N)
  const long long* targets;  // [N]
  long long ignore_index;
  float* zt;                 // forward: [N] target logits
  float2* part;              // forward: [ranges][N] (max in log2 units, sum of ex2)
  const float* lse;          // backward: [N]
  const float* grad;         // backward: [N] (grad_per_row) or [1]
  int grad_per_row;
  const float* count;        // backward, "mean": the number of rows not ignored; nullptr otherwise
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// (m, s) <- (m, s) combined with (m2, s2): the sum of 2^(x - m) over both parts, against the larger maximum
__device__ __forceinline__ void lse_combine(float& m, float& s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  if (mn == -INFINITY) return;                             // both parts empty
  s = s * ex2(m - mn) + s2 * ex2(m2 - mn);
  m = mn;
}

template <bool GRAD>
__device__ __forceinline__ void xent_body(const CUtensorMap* map_x, const CUtensorMap* map_w, const CUtensorMap* map_g,
                                          const XentParams& p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + XC::STAGES * XC::A_BYTES;
  uint8_t* smem_store = smem + XC::STAGES * XC::STAGE_BYTES;   // backward: bf16 staging tile of the bulk stores
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_store + XC::STORE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + XC::STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int items = p.num_m * p.ranges;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(map_x);
    tma_prefetch_desc(map_w);
    if (GRAD) tma_prefetch_desc(map_g);
    for (int i = 0; i < XC::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);                         // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // item w: rows m0 .. m0 + 127 (of the chunk), vocab tiles [t0, t1) of range w / num_m
  auto item = [&](int w, int& m0, int& range, int& t0, int& t1) {
    range = w / p.num_m;
    m0 = (w % p.num_m) * BLOCK_M;
    t0 = (int)((long long)range * p.num_v / p.ranges);
    t1 = (int)((long long)(range + 1) * p.num_v / p.ranges);
  };

  if (warp < 4) {
    // ============================ TMA producer ============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < items; w += gridDim.x) {
        int m0, range, t0, t1;
        item(w, m0, range, t0, t1);
        for (int t = t0; t < t1; ++t) {
          for (int kb = 0; kb < p.num_kb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_expect_tx(&full_bar[stage], XC::STAGE_BYTES);
            tma_load_2d(map_x, &full_bar[stage], smem_a + stage * XC::A_BYTES, kb * BLOCK_K, p.row0 + m0);
            tma_load_2d(map_w, &full_bar[stage], smem_b + stage * XC::B_BYTES, kb * BLOCK_K, t * XBN);
            if (++stage == XC::STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ============================ wgmma + epilogue (warpgroups 1-2) ============================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int cw = warp - 4;                                 // consumer warp 0..7
  const int wg = cw >> 2;
  const int r = wg * 64 + (cw & 3) * 16 + (lane >> 2);     // this thread's fragment rows: r, r + 8
  const int cq = 2 * (lane & 3);
  const int q = cw & 3;                                    // backward: the 32-row slab this warp stores
  const int c_begin = (cw >> 2) * (XBN / 2);               // and its half of the columns
  const uint32_t stg = smem_u32(smem_store);
  int stage = 0;
  uint32_t phase = 0;
  float d[XBN / 2];
  for (int w = blockIdx.x; w < items; w += gridDim.x) {
    int m0, range, t0, t1;
    item(w, m0, range, t0, t1);
    // the rows' targets (as column offsets: -1 for none), and in the backward their lse and gradient scale
    long long tg[2];
    bool row_ok[2];
    float lse2[2], sc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + r + 8 * h;
      row_ok[h] = row < p.rows;
      const long long t = row_ok[h] ? p.targets[p.row0 + row] : -1;
      tg[h] = (t == p.ignore_index) ? -1 : t;
      if (GRAD) {
        lse2[h] = row_ok[h] ? p.lse[p.row0 + row] * kLog2e : 0.f;
        float s = 0.f;
        if (row_ok[h] && t != p.ignore_index) {
          if (t < 0 || t >= p.V) {
            s = __int_as_float(0x7fc00000);                // NaN: the row's target is out of range
          } else {
            s = p.grad[p.grad_per_row ? p.row0 + row : 0];
            if (p.count != nullptr) s = __fdiv_rn(s, *p.count);
          }
        }
        sc[h] = s;
      }
    }
    float mrun[2] = {-INFINITY, -INFINITY}, srun[2] = {0.f, 0.f};
    for (int t = t0; t < t1; ++t) {
      wg_mainloop<XBN, false, false, XC::STAGES, XC::A_BYTES, XC::B_BYTES>(d, smem_u32(smem_a), smem_u32(smem_b),
                                                                          full_bar, empty_bar, stage, phase,
                                                                          p.num_kb, wg);
      const int n0 = t * XBN;
      int tl[2];                                           // the target's column in this tile, or -1
#pragma unroll
      for (int h = 0; h < 2; ++h) tl[h] = (tg[h] >= n0 && tg[h] < n0 + XBN) ? (int)(tg[h] - n0) : -1;
      if (!GRAD) {
        if (n0 + XBN > p.V) {                              // the last tile: columns >= V take no part
#pragma unroll
          for (int j = 0; j < XBN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (n0 + 8 * j + cq + (e & 1) >= p.V) d[4 * j + e] = -INFINITY;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (tl[h] >= 0 && (tl[h] & 6) == cq && row_ok[h]) {   // this thread holds the row's target column
            float z = 0.f;
#pragma unroll
            for (int j = 0; j < XBN / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (8 * j + cq + e == tl[h]) z = d[4 * j + 2 * h + e];
            p.zt[p.row0 + m0 + r + 8 * h] = z;
          }
          float mx = -INFINITY;
#pragma unroll
          for (int j = 0; j < XBN / 8; ++j) mx = fmaxf(mx, fmaxf(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]));
          const float mn = fmaxf(mrun[h], mx * kLog2e);
          if (mn == -INFINITY) continue;                   // every column so far is masked
          const float alpha = ex2(mrun[h] - mn);           // 0 while mrun is -inf
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int j = 0; j < XBN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) acc[j & 3] += ex2(fmaf(d[4 * j + 2 * h + e], kLog2e, -mn));
          srun[h] = srun[h] * alpha + ((acc[0] + acc[1]) + (acc[2] + acc[3]));
          mrun[h] = mn;
        }
      } else {
        // staging address of column pair j of row r + 8h (as in the GEMM epilogue)
        const uint32_t sbase = stg + (uint32_t)(((r >> 5) * (XBN / 64)) << 12) + (uint32_t)((r & 31) << 7) +
                               (uint32_t)(lane & 3) * 4u;
        const uint32_t x7 = (uint32_t)(r & 7);
        // the staging tile is rewritten once the bulk stores of the previous tile have read it
        if (lane == 0) tma_store_wait_read<0>();
        named_bar(1, 256);
#pragma unroll
        for (int j = 0; j < XBN / 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float pe = ex2(fmaf(d[4 * j + 2 * h + e], kLog2e, -lse2[h]));
              v[e] = sc[h] * (8 * j + cq + e == tl[h] ? pe - 1.0f : pe);
            }
            epi_sts32(sbase + (uint32_t)(h * 1024 + ((j >> 3) << 12)) + ((((uint32_t)j & 7u) ^ x7) << 4),
                      cvt_bf16x2(v[0], v[1]));
          }
        fence_async_smem();                                // the staged tile -> visible to the bulk stores
        named_bar(1, 256);
        GemmParams gp{};
        gp.M = p.rows;
        gp.N = p.V;
        store_slab<XBN>(gp, map_g, smem_store, q, lane, m0 + 32 * q, n0, c_begin, c_begin + XBN / 2, StoreAt{},
                        nullptr);
      }
    }
    if (!GRAD) {
      // the four lanes of a row: (0, 1) and (2, 3), then the two pairs; lane 4k writes the row's partial
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        lse_combine(mrun[h], srun[h], __shfl_xor_sync(0xffffffffu, mrun[h], 1),
                    __shfl_xor_sync(0xffffffffu, srun[h], 1));
        lse_combine(mrun[h], srun[h], __shfl_xor_sync(0xffffffffu, mrun[h], 2),
                    __shfl_xor_sync(0xffffffffu, srun[h], 2));
        if ((lane & 3) == 0 && row_ok[h])
          p.part[(size_t)range * p.N + (size_t)(m0 + r + 8 * h)] = make_float2(mrun[h], srun[h]);
      }
    }
  }
  if (GRAD && lane == 0) tma_store_wait_all();             // shared memory must outlive the bulk reads
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
xent_fwd_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                const __grid_constant__ XentParams p) {
  xent_body<false>(&map_x, &map_w, nullptr, p);
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
xent_grad_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                 const __grid_constant__ CUtensorMap map_g, const __grid_constant__ XentParams p) {
  xent_body<true>(&map_x, &map_w, &map_g, p);
}

// Fixed-order tree sum of the block's (sum, count) pairs; thread 0 returns the totals.
__device__ __forceinline__ float2 block_sum2(float a, float b) {
  __shared__ float sa[FIN_THREADS], sb[FIN_THREADS];
  sa[threadIdx.x] = a;
  sb[threadIdx.x] = b;
  __syncthreads();
#pragma unroll
  for (int s = FIN_THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      sa[threadIdx.x] += sa[threadIdx.x + s];
      sb[threadIdx.x] += sb[threadIdx.x + s];
    }
    __syncthreads();
  }
  return make_float2(sa[0], sb[0]);
}

// One row per thread: the ranges' partials folded in range order, lse and the row's loss; one (sum of losses,
// rows not ignored) per block.
__global__ void __launch_bounds__(FIN_THREADS)
xent_finish_kernel(const float2* __restrict__ part, const float* __restrict__ zt,
                   const long long* __restrict__ targets, float* __restrict__ lse, float* __restrict__ loss_rows,
                   float2* __restrict__ blk, int N, int V, int ranges, long long ignore_index) {
  const int row = blockIdx.x * FIN_THREADS + threadIdx.x;
  float loss = 0.f, cnt = 0.f;
  if (row < N) {
    float m = part[row].x, s = part[row].y;
    for (int k = 1; k < ranges; ++k) {
      const float2 pk = part[(size_t)k * N + row];
      lse_combine(m, s, pk.x, pk.y);
    }
    const float l = (m + log2f(s)) * kLn2;
    lse[row] = l;
    const long long t = targets[row];
    if (t != ignore_index) {
      cnt = 1.f;
      loss = (t < 0 || t >= V) ? __int_as_float(0x7fc00000) : l - zt[row];
    }
    if (loss_rows != nullptr) loss_rows[row] = loss;
  }
  const float2 tot = block_sum2(loss, cnt);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
}

// One block: the blocks' (sum, count) in block order -> stats = {sum, count}; out = sum ("sum") or sum / count
// ("mean", NaN when every row is ignored).
__global__ void __launch_bounds__(FIN_THREADS)
xent_total_kernel(const float2* __restrict__ blk, int nblk, float* __restrict__ stats, float* __restrict__ out,
                  int mean) {
  float a = 0.f, b = 0.f;
  for (int i = threadIdx.x; i < nblk; i += FIN_THREADS) {
    a += blk[i].x;
    b += blk[i].y;
  }
  const float2 tot = block_sum2(a, b);
  if (threadIdx.x == 0) {
    stats[0] = tot.x;
    stats[1] = tot.y;
    if (out != nullptr) *out = mean ? __fdiv_rn(tot.x, tot.y) : tot.x;
  }
}

// Vocab ranges per row block: the count that gives the busiest CTA the fewest tiles (the smallest on a tie).
int pick_ranges(int num_m, int num_v, int grid_cap) {
  int best = 1;
  long long best_cost = -1;
  for (int r = 1; r <= num_v && r <= 1024; ++r) {
    const long long items = (long long)num_m * r;
    const long long grid = items < grid_cap ? items : grid_cap;
    const long long cost = ((items + grid - 1) / grid) * ((num_v + r - 1) / r);
    if (best_cost < 0 || cost < best_cost) {
      best_cost = cost;
      best = r;
    }
  }
  return best;
}

int check_shapes(const void* x, const void* w, int N, int D, int V) {
  if (N <= 0 || D <= 0 || V <= 0) return fail("bad shape");
  if ((D % 8) || (V % 8)) return fail("D and V must be multiples of 8");
  if (N >= (1 << 24)) return fail("at most 2^24 - 1 rows");
  if (((uintptr_t)x | (uintptr_t)w) & 15) return fail("pointers must be 16-byte aligned");
  return 0;
}

int grid_cap(int max_ctas) {
  int g = g_num_sms < STATS_MAX_CTAS ? g_num_sms : STATS_MAX_CTAS;
  if (max_ctas > 0 && g > max_ctas) g = max_ctas;
  return g;
}

}  // namespace

extern "C" {

const char* b200dp_xent_last_error() { return g_err; }

// x [N, D], w [V, D] bf16 with dense rows; targets [N] int64.  Writes lse [N]; loss_rows [N] (or nullptr): the
// per-row losses; stats (or nullptr): {sum of the losses, rows not ignored}, and then out (or nullptr): the sum
// (mean = 0) or the mean (mean = 1).  All fp32, all on the device, in a fixed order.
int b200dp_xent_fwd(const void* x, const void* w, const long long* targets, float* lse, float* loss_rows, float* stats,
                    float* out, int N, int D, int V, long long ignore_index, int mean, int max_ctas,
                    unsigned long long stream) {
  if (ensure_init()) return -1;
  if (check_shapes(x, w, N, D, V)) return -1;
  XentParams p{};
  p.N = N; p.V = V;
  p.num_m = (N + BLOCK_M - 1) / BLOCK_M;
  p.num_v = (V + XBN - 1) / XBN;
  p.num_kb = (D + BLOCK_K - 1) / BLOCK_K;
  p.ranges = pick_ranges(p.num_m, p.num_v, grid_cap(max_ctas));
  p.row0 = 0; p.rows = N;
  p.targets = targets;
  p.ignore_index = ignore_index;
  CUtensorMap mx, mw;
  if (make_map2(&mx, x, N, D, D, BLOCK_M) || make_map2(&mw, w, V, D, D, XBN)) return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int nblk = (N + FIN_THREADS - 1) / FIN_THREADS;
  const size_t part_bytes = (size_t)p.ranges * N * sizeof(float2);
  const size_t zt_bytes = ((size_t)N * sizeof(float) + 15) & ~(size_t)15;
  void* ws = nullptr;
  cudaError_t e = cudaMallocAsync(&ws, part_bytes + zt_bytes + (size_t)nblk * sizeof(float2), st);
  if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
  p.part = reinterpret_cast<float2*>(ws);
  p.zt = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + part_bytes);
  float2* blk = reinterpret_cast<float2*>(reinterpret_cast<char*>(ws) + part_bytes + zt_bytes);
  int rc = launch_persistent<xent_fwd_kernel, XBN>(p.num_m * p.ranges, max_ctas, st, mx, mw, p);
  if (rc == 0) {
    xent_finish_kernel<<<nblk, FIN_THREADS, 0, st>>>(p.part, p.zt, targets, lse, loss_rows, blk, N, V, p.ranges,
                                                     ignore_index);
    if (stats != nullptr) xent_total_kernel<<<1, FIN_THREADS, 0, st>>>(blk, nblk, stats, out, mean);
    e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(cudaGetErrorString(e), (int)e);
  }
  e = cudaFreeAsync(ws, st);
  if (e != cudaSuccess && rc == 0) return fail(cudaGetErrorString(e), (int)e);
  return rc;
}

// dlogits [rows, V] bf16 (dense rows) for rows row0 .. row0 + rows - 1 of x: s_i (softmax(z_i) - onehot(t_i)),
// s_i = grad[i] (grad_per_row) or grad[0], divided by *count when count is given; 0 for ignored rows.
int b200dp_xent_grad(const void* x, const void* w, const long long* targets, const float* lse, const float* grad,
                     int grad_per_row, const float* count, void* dlogits, int row0, int rows, int N, int D, int V,
                     long long ignore_index, int max_ctas, unsigned long long stream) {
  if (ensure_init()) return -1;
  if (check_shapes(x, w, N, D, V)) return -1;
  if (row0 < 0 || rows <= 0 || row0 + rows > N) return fail("bad row range");
  if ((uintptr_t)dlogits & 15) return fail("pointers must be 16-byte aligned");
  XentParams p{};
  p.N = N; p.V = V;
  p.num_m = (rows + BLOCK_M - 1) / BLOCK_M;
  p.num_v = (V + XBN - 1) / XBN;
  p.num_kb = (D + BLOCK_K - 1) / BLOCK_K;
  p.ranges = p.num_v;
  p.row0 = row0; p.rows = rows;
  p.targets = targets;
  p.ignore_index = ignore_index;
  p.lse = lse; p.grad = grad; p.grad_per_row = grad_per_row ? 1 : 0; p.count = count;
  CUtensorMap mx, mw, mg;
  if (make_map2(&mx, x, N, D, D, BLOCK_M) || make_map2(&mw, w, V, D, D, XBN) || make_map2(&mg, dlogits, rows, V, V, 32))
    return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  return launch_persistent<xent_grad_kernel, XBN>(p.num_m * p.num_v, max_ctas, st, mx, mw, mg, p);
}

}  // extern "C"

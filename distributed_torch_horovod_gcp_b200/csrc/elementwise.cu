// Fused NHWC bf16 batch-norm kernels for sm_90a (memory-bound; 128-bit vector access).
//
// A channels-last activation is a row-major [M = N*H*W, C] matrix, so per-channel statistics are
// column reductions and normalisation is a per-column affine.  Fusions (vs the eager
// BN -> add -> ReLU chain, SURVEY.md §7.1 step 9 "fused BN+ReLU"):
//   forward : stats pass (1 read) + ONE apply pass  y = relu(x*a[c] + b[c] + residual)
//             (3 reads + 1 write instead of 5 reads + 3 writes)
//   backward: reduce pass with the ReLU mask recomputed from y, + ONE apply pass that writes dx and
//             the residual-branch gradient together.
// Statistics accumulate in fp32 (vector registers -> shared -> one slot per block, summed in block order
// by the last block: see block_reduce_to_global).
#include <initializer_list>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "philox.cuh"

namespace {

constexpr int THREADS = 256;

__device__ __forceinline__ void unpack8(const uint4& x, float* f) {
  const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    f[2 * t] = __uint_as_float(w[t] << 16);
    f[2 * t + 1] = __uint_as_float(w[t] & 0xffff0000u);
  }
}
__device__ __forceinline__ uint4 pack8(const float* v) {
  uint32_t w[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * t], v[2 * t + 1]);
    w[t] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

// Column reduction scaffold: the flattened vector index i (8 channels per vector) maps to channel
// group i % V.  The total thread count is a multiple of V, so a thread always owns ONE channel
// group and accumulates NACC x 8 partial sums in registers; threads of a block that share a group
// are combined through shared memory and the block writes its partial sums to its own slot.  The
// last block to finish adds the slots of all blocks in block order to `outs`: the result does not
// depend on which block finished when, so a training step computes the same bits every run
// (fp32 atomics would sum in arrival order).
constexpr int RED_MAX_BLOCKS = 256;
constexpr int RED_MAX_COLS = 2 * 2048;                  // NACC x channels
__device__ float g_red_slots[RED_MAX_BLOCKS * RED_MAX_COLS];
__device__ unsigned int g_red_done;

template <int NACC, int NT>
__device__ __forceinline__ void block_reduce_to_global(float (&acc)[NACC][8], int V, float* const* outs) {
  __shared__ float sm[NT][8 + 1];
  __shared__ bool last;
  const int tid = threadIdx.x;
  const int groups = NT / V;      // threads per channel group inside this block (>=1)
  const int C = V * 8;
  float* slot = g_red_slots + (size_t)blockIdx.x * (NACC * C);
#pragma unroll
  for (int q = 0; q < NACC; ++q) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) sm[tid][j] = acc[q][j];
    __syncthreads();
    // V*8 channel sums, each over `groups` partials: spread over all threads (8 per group)
    for (int item = tid; item < C; item += NT) {
      const int g0 = item >> 3, j = item & 7;
      float s = 0.f;
      for (int g = 0; g < groups; ++g) s += sm[g0 + g * V][j];
      slot[q * C + item] = s;
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) last = atomicAdd(&g_red_done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int item = tid; item < NACC * C; item += NT) {
    float s = 0.f;
    for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(g_red_slots + (size_t)b * (NACC * C) + item);
    outs[item / C][item % C] += s;
  }
  if (tid == 0) g_red_done = 0u;
}

// Reduction kernels run ONE 1024-thread block per SM: the last block sums one slot per block, so the
// number of blocks — not the data size — sets the tail of the reduction.
constexpr int RTHREADS = 1024;

// HBM3 needs >= ~32 KB in flight per SM to saturate (3.35 TB/s x ~1 us over 132 SMs): every kernel below
// issues UNROLL independent 128-bit loads per thread per input before consuming any of them.
__device__ __forceinline__ uint4 ld_or_zero(const uint4* p, long long i, long long n) {
  return i < n ? ldg_stream(p + i) : make_uint4(0, 0, 0, 0);
}

// ---- forward statistics: sum[c], sumsq[c] -------------------------------------------------------
__global__ void __launch_bounds__(RTHREADS, 1) bn_stats_kernel(const uint4* __restrict__ x, float* sum,
                                                               float* sumsq, long long nvec, int V) {
  constexpr int U = 8;
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  const long long stride = (long long)gridDim.x * RTHREADS;
  for (long long i = (long long)blockIdx.x * RTHREADS + threadIdx.x; i < nvec; i += U * stride) {
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) raw[u] = ld_or_zero(x, i + u * stride, nvec);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float f[8];
      unpack8(raw[u], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[0][j] += f[j];
        acc[1][j] = fmaf(f[j], f[j], acc[1][j]);
      }
    }
  }
  float* outs[2] = {sum, sumsq};
  block_reduce_to_global<2, RTHREADS>(acc, V, outs);
}

// ---- finalize: mean/invstd, affine (a, b), running statistics ------------------------------------
__device__ __forceinline__ float ld_param(const void* p, int c, int bf16) {
  return bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[c])
              : reinterpret_cast<const float*>(p)[c];
}
__device__ __forceinline__ void st_param(void* p, int c, int bf16, float v) {
  if (bf16) reinterpret_cast<__nv_bfloat16*>(p)[c] = __float2bfloat16_rn(v);
  else reinterpret_cast<float*>(p)[c] = v;
}

// gamma/beta/running_* are the module's tensors in their own dtype (fp32 or bf16: `pbf16`).
// DEV_COUNT (SyncBatchNorm): `count` is the row count summed over all ranks, read from `count_dev` on the device.
// A template argument, so that the plain instantiation compiles to the same instructions (and bits) as without it.
template <bool DEV_COUNT>
__global__ void bn_finalize_kernel(float* sum, float* sumsq, const void* gamma,
                                   const void* beta, float* mean, float* invstd, float* a, float* b,
                                   void* running_mean, void* running_var, float count, float eps,
                                   float momentum, int C, int pbf16, int rezero = 0,
                                   long long* num_batches_tracked = nullptr, const float* count_dev = nullptr) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0 && num_batches_tracked != nullptr) *num_batches_tracked += 1;   // nn.BatchNorm2d bookkeeping
  if (c >= C) return;
  if constexpr (DEV_COUNT) count = *count_dev;
  const float m = sum[c] / count;
  const float var = fmaxf(sumsq[c] / count - m * m, 0.f);
  if (rezero) {      // persistent accumulators filled by the producing GEMM / conv epilogue: ready for the next step
    sum[c] = 0.f;
    sumsq[c] = 0.f;
  }
  const float is = rsqrtf(var + eps);
  mean[c] = m;
  invstd[c] = is;
  const float g = gamma ? ld_param(gamma, c, pbf16) : 1.f;
  a[c] = g * is;
  b[c] = (beta ? ld_param(beta, c, pbf16) : 0.f) - m * g * is;
  if (running_mean) {
    const float unbiased = var * (count / fmaxf(count - 1.f, 1.f));
    st_param(running_mean, c, pbf16, (1.f - momentum) * ld_param(running_mean, c, pbf16) + momentum * m);
    st_param(running_var, c, pbf16,
             (1.f - momentum) * ld_param(running_var, c, pbf16) + momentum * unbiased);
  }
}

// ---- forward apply: y = relu(x*a + b + residual) ---------------------------------------------------
__global__ void __launch_bounds__(THREADS, 4) bn_apply_kernel(const uint4* __restrict__ x,
                                                              const uint4* __restrict__ res, uint4* y,
                                                              const float* __restrict__ a,
                                                              const float* __restrict__ b, long long nvec,
                                                              int V, int relu, uint8_t* __restrict__ mask) {
  constexpr int U = 4;
  const long long stride = (long long)gridDim.x * THREADS;
  const long long i0 = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (i0 >= nvec) return;
  const int cg = (int)(i0 % V);
  float av[8], bv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    av[j] = a[cg * 8 + j];
    bv[j] = b[cg * 8 + j];
  }
  for (long long i = i0; i < nvec; i += U * stride) {
    uint4 rx[U], rr[U];
#pragma unroll
    for (int u = 0; u < U; ++u) rx[u] = ld_or_zero(x, i + u * stride, nvec);
    if (res) {
#pragma unroll
      for (int u = 0; u < U; ++u) rr[u] = ld_or_zero(res, i + u * stride, nvec);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (i + u * stride >= nvec) break;
      float f[8];
      unpack8(rx[u], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaf(f[j], av[j], bv[j]);
      if (res) {
        float r[8];
        unpack8(rr[u], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += r[j];
      }
      if (relu) {
        if (mask) {       // 1 bit per element: the backward reads this instead of re-reading y
          uint32_t m = 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) m |= (f[j] > 0.f ? 1u : 0u) << j;
          mask[i + u * stride] = (uint8_t)m;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
      }
      y[i + u * stride] = pack8(f);
    }
  }
}

// ---- backward reduce: sum_dy[c], sum_dy_xhat[c] (dy masked by y > 0 when relu) ----------------------
// Accumulates sum(dz) and sum(dz * (x - mean)); the invstd factor is applied when the sums are used.
__global__ void __launch_bounds__(RTHREADS, 1) bn_bwd_reduce_kernel(
    const uint4* __restrict__ dy, const uint4* __restrict__ x, const uint8_t* __restrict__ mask,
    const float* __restrict__ mean, float* sum_dy, float* sum_dy_xc, long long nvec, int V, int relu) {
  constexpr int U = 2;
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  const long long stride = (long long)gridDim.x * RTHREADS;
  const long long i0 = (long long)blockIdx.x * RTHREADS + threadIdx.x;
  float mv[8];
  {
    const int cg = (int)(i0 % V);
#pragma unroll
    for (int j = 0; j < 8; ++j) mv[j] = mean[cg * 8 + j];
  }
  for (long long i = i0; i < nvec; i += U * stride) {
    uint4 rg[U], rx[U];
    uint32_t rm[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      rg[u] = ld_or_zero(dy, i + u * stride, nvec);
      rx[u] = ld_or_zero(x, i + u * stride, nvec);
      rm[u] = (relu && i + u * stride < nvec) ? (uint32_t)__ldg(mask + i + u * stride) : 0xffu;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float g[8], xv[8];
      unpack8(rg[u], g);
      unpack8(rx[u], xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = ((rm[u] >> j) & 1u) ? g[j] : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[0][j] += g[j];
        acc[1][j] = fmaf(g[j], xv[j] - mv[j], acc[1][j]);
      }
    }
  }
  float* outs[2] = {sum_dy, sum_dy_xc};
  block_reduce_to_global<2, RTHREADS>(acc, V, outs);
}

// ---- backward apply: dx = a*(dz - sum_dy/M - xhat*sum_dy_xhat/M), dres = dz ------------------------
// DEV_COUNT (SyncBatchNorm): 1/M from the global row count `count_dev` on the device instead of `inv_count`.  A
// template argument, so that the plain instantiation compiles to the same instructions (and bits) as without it.
template <bool DEV_COUNT>
__global__ void __launch_bounds__(THREADS, 4) bn_bwd_apply_kernel(
    const uint4* __restrict__ dy, const uint4* __restrict__ x, const uint8_t* __restrict__ mask, uint4* dx,
    uint4* dres, const float* __restrict__ mean, const float* __restrict__ invstd,
    const float* __restrict__ scale_a, const float* __restrict__ sum_dy,
    const float* __restrict__ sum_dy_xhat, float inv_count, long long nvec, int V, int relu,
    void* dgamma, void* dbeta, int pbf16, const float* __restrict__ count_dev = nullptr) {
  constexpr int U = 2;
  const long long stride = (long long)gridDim.x * THREADS;
  const long long i0 = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (blockIdx.x == 0 && dgamma != nullptr) {     // parameter gradients, written in the param dtype
    for (int c = threadIdx.x; c < V * 8; c += THREADS) {
      st_param(dbeta, c, pbf16, sum_dy[c]);
      st_param(dgamma, c, pbf16, sum_dy_xhat[c] * invstd[c]);
    }
  }
  if (i0 >= nvec) return;
  // 1 / (global row count) in double rounded to fp32, as the host computes inv_count
  if constexpr (DEV_COUNT) inv_count = (float)(1.0 / (double)*count_dev);
  const int cg = (int)(i0 % V);
  float mv[8], iv[8], k1[8], k2[8], sc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = cg * 8 + j;
    mv[j] = mean[c];
    iv[j] = invstd[c];
    sc[j] = scale_a[c];      // gamma * invstd, saved by the forward
    k1[j] = sum_dy[c] * inv_count;
    k2[j] = sum_dy_xhat[c] * iv[j] * inv_count;   // reduce pass stored sum(dz*(x-mean))
  }
  for (long long i = i0; i < nvec; i += U * stride) {
    uint4 rg[U], rx[U];
    uint32_t rm[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      rg[u] = ld_or_zero(dy, i + u * stride, nvec);
      rx[u] = ld_or_zero(x, i + u * stride, nvec);
      rm[u] = (relu && i + u * stride < nvec) ? (uint32_t)__ldg(mask + i + u * stride) : 0xffu;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (i + u * stride >= nvec) break;
      float g[8], xv[8], o[8];
      unpack8(rg[u], g);
      unpack8(rx[u], xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = ((rm[u] >> j) & 1u) ? g[j] : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xhat = (xv[j] - mv[j]) * iv[j];
        o[j] = sc[j] * (g[j] - k1[j] - xhat * k2[j]);
      }
      dx[i + u * stride] = pack8(o);
      if (dres) dres[i + u * stride] = pack8(g);
    }
  }
}

// ---- LayerNorm over the last dimension, bf16 in/out, fp32 statistics -------------------------------------
// One warp per row; a lane owns VPL 8-element vectors (C = 256 * VPL).  The backward fuses the input
// gradient with the gamma/beta column reductions: per-lane register partials over the rows a warp
// visits -> shared memory across the block's warps -> one atomicAdd per (column, quantity) per block.
// (torch's GammaBetaBackward kernel takes 233 us per ViT-B layer at 25k rows; this takes the time of
// one extra read of dy and x.)
constexpr int LN_WARPS = 16;

template <int VPL>
__global__ void __launch_bounds__(LN_WARPS * 32) ln_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y,
                                                               const void* gamma, const void* beta,
                                                               float* __restrict__ mean, float* __restrict__ rstd,
                                                               long long rows, float eps, int pbf16) {
  constexpr int C = 256 * VPL;
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * LN_WARPS;
  float g[VPL][8], b[VPL][8];
#pragma unroll
  for (int v = 0; v < VPL; ++v)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = (v * 32 + lane) * 8 + j;
      g[v][j] = ld_param(gamma, c, pbf16);
      b[v][j] = ld_param(beta, c, pbf16);
    }
  for (long long r = warp; r < rows; r += nwarps) {
    const uint4* xr = x + r * (C / 8);
    float f[VPL][8];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      unpack8(ldg_stream(xr + v * 32 + lane), f[v]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[v][j];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float m = s * (1.f / C);
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = f[v][j] - m;
        q = fmaf(d, d, q);
      }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rs = rsqrtf(q * (1.f / C) + eps);
    if (lane == 0) {
      mean[r] = m;
      rstd[r] = rs;
    }
    uint4* yr = y + r * (C / 8);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf((f[v][j] - m) * rs, g[v][j], b[v][j]);
      yr[v * 32 + lane] = pack8(o);
    }
  }
}

template <int VPL>
__global__ void __launch_bounds__(LN_WARPS * 32) ln_bwd_kernel(const uint4* __restrict__ dy,
                                                               const uint4* __restrict__ x, uint4* __restrict__ dx,
                                                               const void* gamma, const float* __restrict__ mean,
                                                               const float* __restrict__ rstd, float* sums,
                                                               long long rows, int pbf16) {
  constexpr int C = 256 * VPL;
  extern __shared__ float red[];                 // [LN_WARPS][C]
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long warp = (long long)blockIdx.x * LN_WARPS + wib;
  const long long nwarps = (long long)gridDim.x * LN_WARPS;
  float g[VPL][8], dg[VPL][8], db[VPL][8];
#pragma unroll
  for (int v = 0; v < VPL; ++v)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      g[v][j] = ld_param(gamma, (v * 32 + lane) * 8 + j, pbf16);
      dg[v][j] = db[v][j] = 0.f;
    }
  for (long long r = warp; r < rows; r += nwarps) {
    const float m = mean[r], rs = rstd[r];
    float d[VPL][8], xh[VPL][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      float xv[8];
      unpack8(ldg_stream(dy + r * (C / 8) + v * 32 + lane), d[v]);
      unpack8(ldg_stream(x + r * (C / 8) + v * 32 + lane), xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xh[v][j] = (xv[j] - m) * rs;
        db[v][j] += d[v][j];
        dg[v][j] = fmaf(d[v][j], xh[v][j], dg[v][j]);
        const float gd = d[v][j] * g[v][j];
        s1 += gd;
        s2 = fmaf(gd, xh[v][j], s2);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    s1 *= (1.f / C);
    s2 *= (1.f / C);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rs * (d[v][j] * g[v][j] - s1 - xh[v][j] * s2);
      dx[r * (C / 8) + v * 32 + lane] = pack8(o);
    }
  }
  // block reduction of the column partials, one quantity at a time
#pragma unroll
  for (int qn = 0; qn < 2; ++qn) {
    __syncthreads();
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int j = 0; j < 8; ++j) red[wib * C + (v * 32 + lane) * 8 + j] = qn == 0 ? dg[v][j] : db[v][j];
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += LN_WARPS * 32) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < LN_WARPS; ++w) s += red[w * C + c];
      atomicAdd(sums + qn * C + c, s);
    }
  }
}

__global__ void ln_param_grad_kernel(const float* sums, void* dgamma, void* dbeta, int C, int pbf16) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  st_param(dgamma, c, pbf16, sums[c]);
  st_param(dbeta, c, pbf16, sums[C + c]);
}

// ---- 3x3 stride-2 pad-1 max pooling, NHWC bf16 -------------------------------------------------------
// forward stores the arg-max tap (0..8) as one byte per output element; backward is a gather: every
// input pixel looks at the <= 4 windows that cover it and takes dy where it was the arg-max (no atomics).
__global__ void __launch_bounds__(THREADS) maxpool_fwd_kernel(const uint4* __restrict__ x, uint4* y,
                                                              uint2* __restrict__ idx, int N, int H, int W,
                                                              int OH, int OW, int V) {
  const long long total = (long long)N * OH * OW * V;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * THREADS) {
    const int cv = (int)(i % V);
    long long t = i / V;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH);
    const int n = (int)(t / OH);
    float best[8];
    uint32_t arg[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; arg[j] = 0; }
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = oh * 2 - 1 + kh;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int iw = ow * 2 - 1 + kw;
        if (iw < 0 || iw >= W) continue;
        float f[8];
        unpack8(x[(((long long)n * H + ih) * W + iw) * V + cv], f);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (f[j] > best[j]) { best[j] = f[j]; arg[j] = kh * 3 + kw; }
      }
    }
    y[i] = pack8(best);
    uint2 packed;
    packed.x = arg[0] | (arg[1] << 8) | (arg[2] << 16) | (arg[3] << 24);
    packed.y = arg[4] | (arg[5] << 8) | (arg[6] << 16) | (arg[7] << 24);
    idx[i] = packed;
  }
}

__global__ void __launch_bounds__(THREADS) maxpool_bwd_kernel(const uint4* __restrict__ dy,
                                                              const uint2* __restrict__ idx, uint4* dx,
                                                              int N, int H, int W, int OH, int OW, int V) {
  const long long total = (long long)N * H * W * V;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * THREADS) {
    const int cv = (int)(i % V);
    long long t = i / V;
    const int iw = (int)(t % W); t /= W;
    const int ih = (int)(t % H);
    const int n = (int)(t / H);
    float g[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = 0.f;
    // windows (oh, ow) with oh*2-1 <= ih <= oh*2+1
    const int oh0 = max((ih - 1 + 1) / 2, 0), oh1 = min((ih + 1) / 2, OH - 1);
    const int ow0 = max((iw - 1 + 1) / 2, 0), ow1 = min((iw + 1) / 2, OW - 1);
    for (int oh = oh0; oh <= oh1; ++oh) {
      const int kh = ih - (oh * 2 - 1);
      for (int ow = ow0; ow <= ow1; ++ow) {
        const int kw = iw - (ow * 2 - 1);
        const uint32_t tap = (uint32_t)(kh * 3 + kw);
        const long long o = (((long long)n * OH + oh) * OW + ow) * V + cv;
        const uint2 a = idx[o];
        float d[8];
        unpack8(dy[o], d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t aj = ((j < 4 ? a.x : a.y) >> (8 * (j & 3))) & 0xffu;
          if (aj == tap) g[j] += d[j];
        }
      }
    }
    dx[i] = pack8(g);
  }
}


// Backward, H and W even (the network case): one thread owns a 2x2 input patch x 8 channels.  The patch is
// covered by exactly the four windows (a..a+1, b..b+1), so dy / arg-max are loaded once per window (96 B in
// for 64 B out instead of 2.25 windows per pixel), the byte arg-max comparison is done 4 channels at a time
// (SWAR equality -> PRMT sign-replicate -> 16-bit lane masks) and contributions are summed with packed bf16
// adds (ATen's NHWC backward also accumulates in bf16).
__device__ __forceinline__ uint32_t prmt_msb(uint32_t a, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(0u), "r"(sel));
  return d;
}
template <int TAP>
__device__ __forceinline__ void pool_take(uint4& acc, const uint4& d, const uint2& ix) {
  constexpr uint32_t t4 = (uint32_t)TAP * 0x01010101u;
  // byte == TAP  <=>  MSB of ((byte ^ TAP) | 0x80) - 1 is clear   (arg-max bytes are 0..8)
  const uint32_t e0 = ~(((ix.x ^ t4) | 0x80808080u) - 0x01010101u);
  const uint32_t e1 = ~(((ix.y ^ t4) | 0x80808080u) - 0x01010101u);
  const uint32_t m0 = d.x & prmt_msb(e0, 0x9988u), m1 = d.y & prmt_msb(e0, 0xbbaau);
  const uint32_t m2 = d.z & prmt_msb(e1, 0x9988u), m3 = d.w & prmt_msb(e1, 0xbbaau);
  asm("add.rn.bf16x2 %0, %0, %1;" : "+r"(acc.x) : "r"(m0));
  asm("add.rn.bf16x2 %0, %0, %1;" : "+r"(acc.y) : "r"(m1));
  asm("add.rn.bf16x2 %0, %0, %1;" : "+r"(acc.z) : "r"(m2));
  asm("add.rn.bf16x2 %0, %0, %1;" : "+r"(acc.w) : "r"(m3));
}
__global__ void __launch_bounds__(THREADS) maxpool_bwd_patch_kernel(const uint4* __restrict__ dy,
                                                                    const uint2* __restrict__ idx, uint4* dx,
                                                                    int N, int H, int W, int OH, int OW, int V) {
  const int HP = H / 2, WP = W / 2;
  const long long total = (long long)N * HP * WP * V;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * THREADS) {
    const int cv = (int)(i % V);
    long long t = i / V;
    const int b = (int)(t % WP); t /= WP;
    const int a = (int)(t % HP);
    const int n = (int)(t / HP);
    uint4 p00 = make_uint4(0, 0, 0, 0), p01 = p00, p10 = p00, p11 = p00;   // (row 2a+i, col 2b+j)
    const long long o00 = (((long long)n * OH + a) * OW + b) * V + cv;
    const bool hb = b + 1 < OW, ha = a + 1 < OH;
    {   // window (a, b): rows 2a-1..2a+1, cols 2b-1..2b+1 -> taps (1,1) (1,2) (2,1) (2,2)
      const uint4 d = dy[o00];
      const uint2 ix = idx[o00];
      pool_take<4>(p00, d, ix); pool_take<5>(p01, d, ix); pool_take<7>(p10, d, ix); pool_take<8>(p11, d, ix);
    }
    if (hb) {   // window (a, b+1): cols 2b+1..2b+3 -> taps (1,0) (2,0)
      const uint4 d = dy[o00 + V];
      const uint2 ix = idx[o00 + V];
      pool_take<3>(p01, d, ix); pool_take<6>(p11, d, ix);
    }
    if (ha) {   // window (a+1, b): rows 2a+1..2a+3 -> taps (0,1) (0,2)
      const uint4 d = dy[o00 + (long long)OW * V];
      const uint2 ix = idx[o00 + (long long)OW * V];
      pool_take<1>(p10, d, ix); pool_take<2>(p11, d, ix);
      if (hb) {   // window (a+1, b+1) -> tap (0,0)
        const uint4 d2 = dy[o00 + (long long)OW * V + V];
        const uint2 ix2 = idx[o00 + (long long)OW * V + V];
        pool_take<0>(p11, d2, ix2);
      }
    }
    const long long x00 = (((long long)n * H + 2 * a) * W + 2 * b) * V + cv;
    dx[x00] = p00;
    dx[x00 + V] = p01;
    dx[x00 + (long long)W * V] = p10;
    dx[x00 + (long long)W * V + V] = p11;
  }
}

// ---- stem im2col: 7x7 / stride 2 / pad 3 over NHWC bf16 with C = 3 ------------------------------------
// Turns the ResNet stem into a plain GEMM for the wgmma kernel: A[m][k], m = (n, oh, ow),
// k = kh*24 + j, j = kw*3 + c for j < 21 and three more elements (the next pixel) for j = 21..23 that
// the packed weights multiply by zero — row pitch KP = 7*24 = 168.  With that K order every (pixel, kh)
// segment is a straight 48-byte copy of the (zero-padded) input row starting at byte 12*ow, i.e. 4-byte
// aligned on the source side and 16-byte aligned on the destination side: four LDS.32 + one 16-byte
// store per unit instead of eight predicated 2-byte gathers (the first version ran at 0.25 of HBM).
// One block per output row (n, oh): the 7 input rows it needs are staged in shared memory behind a
// 3-pixel zero border.
constexpr int STEM_KP = 168;
__global__ void __launch_bounds__(THREADS) stem_im2col_kernel(const __nv_bfloat16* __restrict__ x,
                                                              uint4* __restrict__ out, int H, int W,
                                                              int OH, int OW) {
  extern __shared__ __align__(16) __nv_bfloat16 rows[];     // [7][pitch], pitch = 9 + W*3 + 15 (mult. of 8)
  const int n = blockIdx.x / OH, oh = blockIdx.x % OH;
  const int row_elems = W * 3;
  const int pitch = (9 + row_elems + 15 + 7) & ~7;
  // zero borders: elements [0, 9) and [9 + row_elems, pitch) of every row
  for (int i = threadIdx.x; i < 7 * (pitch - row_elems); i += THREADS) {
    const int r = i / (pitch - row_elems), e = i % (pitch - row_elems);
    rows[r * pitch + (e < 9 ? e : row_elems + e)] = __float2bfloat16(0.f);
  }
  const int vec_per_row = row_elems / 8;                     // W*3*2 bytes is a multiple of 16 for W % 8 == 0
  for (int i = threadIdx.x; i < 7 * vec_per_row; i += THREADS) {
    const int r = i / vec_per_row, v = i % vec_per_row;
    const int ih = oh * 2 - 3 + r;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (ih >= 0 && ih < H)
      val = reinterpret_cast<const uint4*>(x + ((size_t)n * H + ih) * row_elems)[v];
    // destination starts at element 9 of the row (2-byte aligned only): 2-byte stores
    __nv_bfloat16* d = rows + r * pitch + 9 + v * 8;
    const __nv_bfloat16* sv = reinterpret_cast<const __nv_bfloat16*>(&val);
#pragma unroll
    for (int e = 0; e < 8; ++e) d[e] = sv[e];
  }
  __syncthreads();
  constexpr int UPR = STEM_KP / 8;                           // 21 16-byte units per output row
  uint4* dst = out + ((size_t)n * OH + oh) * OW * UPR;
  const uint32_t* rows32 = reinterpret_cast<const uint32_t*>(rows);
  const int pitch32 = pitch / 2;
  for (int i = threadIdx.x; i < OW * UPR; i += THREADS) {
    const int ow = i / UPR, u = i % UPR;
    const int kh = u / 3, part = u % 3;
    const uint32_t* src = rows32 + kh * pitch32 + ow * 3 + part * 4;   // element 6*ow + part*8 of row kh
    dst[i] = make_uint4(src[0], src[1], src[2], src[3]);
  }
}


// ---- global average pool over the HW positions of an NHWC bf16 tensor ------------------------------------
// forward: y[n][c] = mean_hw x[n][hw][c]; backward: dx[n][hw][c] = dy[n][c] / HW (ATen's expand + mul + layout
// copy for the same thing are 2 kernels / 120 us at [256, 2048, 7, 7]; this is one 51 MB write).
__global__ void __launch_bounds__(THREADS) avgpool_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y,
                                                              int HW, int V, long long total, float inv) {
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long n = i / V;
    const int v = (int)(i % V);
    const uint4* src = x + n * HW * V + v;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int h = 0; h < HW; ++h) {
      float f[8];
      unpack8(src[(long long)h * V], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    y[i] = pack8(acc);
  }
}
__global__ void __launch_bounds__(THREADS) avgpool_bwd_kernel(const uint4* __restrict__ dy, uint4* __restrict__ dx,
                                                              int HW, int V, long long total, float inv) {
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long n = i / ((long long)HW * V);
    const int v = (int)(i % V);
    float f[8];
    unpack8(dy[n * V + v], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= inv;
    dx[i] = pack8(f);
  }
}

thread_local char g_err[256];
int fail(const char* what, cudaError_t e) {
  snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
  return -1;
}

int g_sms = 0;
int reduce_grid() {
  if (g_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_sms <= 0) g_sms = 132;
    if (g_sms > RED_MAX_BLOCKS) g_sms = RED_MAX_BLOCKS;   // one reduction slot per block
  }
  return g_sms;
}

int grid_for(long long nvec, int V) {
  // streaming kernels: 64 registers x 256 threads -> 4 resident blocks per SM.  1.5 waves (888 blocks)
  // measured ~1.5 % faster end-to-end than exactly one wave (592): the second half-wave evens out
  // the per-SM HBM-channel imbalance of the first.
  long long blocks = (nvec + THREADS * 8 - 1) / (THREADS * 8);
  if (blocks > (long long)reduce_grid() * 6) blocks = (long long)reduce_grid() * 6;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// fp32 accumulator -> gradient tensor (the attention dQ): dst (bf16 or fp32) = (accumulate ? dst : 0) + src,
// and the accumulator is re-zeroed in the same pass so the next backward, which adds to it, starts from zero
// without a memset.
template <bool OUT_BF16>
__global__ void cast_acc_zero_kernel(float* __restrict__ src, void* __restrict__ dst, long long n4,
                                     int accumulate, int zero_src) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 v = reinterpret_cast<float4*>(src)[i];
    if (zero_src) reinterpret_cast<float4*>(src)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (OUT_BF16) {
      uint2* d = reinterpret_cast<uint2*>(dst) + i;
      if (accumulate) {
        const uint2 o = *d;
        v.x += __uint_as_float(o.x << 16); v.y += __uint_as_float(o.x & 0xffff0000u);
        v.z += __uint_as_float(o.y << 16); v.w += __uint_as_float(o.y & 0xffff0000u);
      }
      __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
      *d = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
    } else {
      float4* d = reinterpret_cast<float4*>(dst) + i;
      if (accumulate) { const float4 o = *d; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
      *d = v;
    }
  }
}

// Dropout + residual add (bf16, memory-bound, one 16-byte vector of 8 elements per thread and step):
//   out = residual + keep * y * (2^16 / t)      (residual == nullptr: plain dropout)
// each product is rounded to fp32 and then added in fp32 (no fma), then rounded to bf16 once.  The keep bit of
// element e is a pure function of the seed and e (philox.cuh for t and its resolution):
//   u    = Philox4x32-10(key = (seed[0] mod 2^32, seed[0] / 2^32),
//                        counter = ((e / 8) mod 2^32, (e / 8) / 2^32, seed[1] mod 2^32, seed[1] / 2^32))
//   bits = (e mod 2) ? u[(e mod 8) / 2] >> 16 : u[(e mod 8) / 2] mod 2^16,   keep = bits < t
// so one Philox call serves exactly one vector.  The backward is the same kernel on dout without a residual
// (dy = keep * dout * 2^16 / t): the bits are drawn again from the seed rather than saved.
__global__ void __launch_bounds__(THREADS) dropout_add_kernel(const uint4* __restrict__ y,
                                                              const uint4* __restrict__ res, uint4* __restrict__ out,
                                                              long long nvec, const unsigned long long* __restrict__ seed,
                                                              uint32_t thr, float scale) {
  const unsigned long long k = seed[0], off = seed[1];
  const uint2 key = make_uint2((uint32_t)k, (uint32_t)(k >> 32));
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const uint4 u = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)((unsigned long long)i >> 32), (uint32_t)off,
                                             (uint32_t)(off >> 32)), key);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float f[8], r[8];
    unpack8(ldg_stream(y + i), f);
    if (res != nullptr) unpack8(ldg_stream(res + i), r);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t bits = (j & 1) ? w[j >> 1] >> 16 : w[j >> 1] & 0xffffu;
      const float d = bits < thr ? __fmul_rn(f[j], scale) : 0.f;
      f[j] = res != nullptr ? __fadd_rn(r[j], d) : d;
    }
    out[i] = pack8(f);
  }
}

bool shape_ok(int C) {
  const int V = C / 8;
  return C % 8 == 0 && V >= 1 && V <= THREADS && (THREADS % V) == 0;   // V | 256 | 1024
}

// The activation tensors of the BatchNorm and LayerNorm kernels are read and written as 16-byte vectors (uint4):
// -1 with a message naming `what` unless every pointer given is 16-byte aligned (nullptr: absent, accepted).
int check_vec16(const char* what, std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if ((uintptr_t)p & 15) {
      snprintf(g_err, sizeof(g_err), "%s: every activation tensor must be 16-byte aligned", what);
      return -1;
    }
  return 0;
}

}  // namespace

extern "C" {

const char* b200dp_ew_last_error() { return g_err; }

// dst[n] (bf16 if out_bf16 else fp32) (+)= src[n] (fp32); optionally re-zero src.  n % 4 == 0.
int b200dp_cast_acc_zero(void* src, void* dst, long long n, int out_bf16, int accumulate, int zero_src,
                         unsigned long long stream) {
  if (n % 4) {
    snprintf(g_err, sizeof(g_err), "cast_acc_zero: n must be a multiple of 4");
    return -1;
  }
  const long long n4 = n / 4;
  int grid = (int)((n4 + 255) / 256);
  if (grid > reduce_grid() * 8) grid = reduce_grid() * 8;
  if (grid < 1) grid = 1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  if (out_bf16) cast_acc_zero_kernel<true><<<grid, 256, 0, st>>>((float*)src, dst, n4, accumulate, zero_src);
  else cast_acc_zero_kernel<false><<<grid, 256, 0, st>>>((float*)src, dst, n4, accumulate, zero_src);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("cast_acc_zero launch", e);
  return 0;
}

// out[n] = res[n] + dropout(y[n], p) for bf16 tensors (res == nullptr: out = dropout(y, p)); n % 8 == 0, all
// three 16-byte aligned; 0 < p <= 1; seed: 2 words in device memory (Philox key, offset).  out may alias res.
int b200dp_dropout_add(const void* y, const void* res, void* out, long long n, const unsigned long long* seed,
                       float p, unsigned long long stream) {
  if (n < 0 || n % 8 || ((uintptr_t)y & 15) || ((uintptr_t)res & 15) || ((uintptr_t)out & 15)) {
    snprintf(g_err, sizeof(g_err), "dropout_add: n must be a multiple of 8 and every tensor 16-byte aligned");
    return -1;
  }
  if (!(p > 0.f && p <= 1.f) || seed == nullptr) {
    snprintf(g_err, sizeof(g_err), "dropout_add: needs 0 < p <= 1 and a seed");
    return -1;
  }
  if (n == 0) return 0;
  const uint32_t thr = dropout_thr16(p);
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  long long grid = (n / 8 + THREADS - 1) / THREADS;
  if (grid > reduce_grid() * 8) grid = reduce_grid() * 8;
  dropout_add_kernel<<<(unsigned)grid, THREADS, 0, st>>>((const uint4*)y, (const uint4*)res, (uint4*)out, n / 8,
                                                             seed, thr, dropout_scale16(thr));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("dropout_add launch", e);
  return 0;
}

int b200dp_bn_supported(int C) { return shape_ok(C) ? 1 : 0; }

// stats: [2*C] fp32, zeroed by this call (have_stats == 0), or provided by the producing GEMM / conv epilogue
// (have_stats == 1; == 2: a persistent accumulator that the finalize kernel re-zeroes after reading).
// Writes mean/invstd/a/b ([C] fp32 each); updates running stats.
int b200dp_bn_fwd(const void* x, const void* res, void* y, const void* gamma, const void* beta,
                  float* stats, float* mean, float* invstd, float* a, float* b, void* running_mean,
                  void* running_var, long long M, int C, float eps, float momentum, int relu,
                  int param_bf16, int have_stats, void* relu_mask, void* num_batches_tracked,
                  unsigned long long stream) {
  if (!shape_ok(C)) {
    snprintf(g_err, sizeof(g_err), "unsupported channel count %d", C);
    return -1;
  }
  if (M < 1) {   // the batch statistics of no rows are undefined, and the running statistics must not take them
    snprintf(g_err, sizeof(g_err), "bn_fwd: needs at least one row");
    return -1;
  }
  if (check_vec16("bn_fwd", {x, res, y})) return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int V = C / 8;
  const long long nvec = M * V;
  cudaError_t e = cudaSuccess;
  const int grid = grid_for(nvec, V);
  if (!have_stats) {   // otherwise `stats` was accumulated by the producing GEMM's epilogue
    e = cudaMemsetAsync(stats, 0, sizeof(float) * 2 * C, st);
    if (e != cudaSuccess) return fail("memset", e);
    bn_stats_kernel<<<reduce_grid(), RTHREADS, 0, st>>>((const uint4*)x, stats, stats + C, nvec, V);
  }
  bn_finalize_kernel<false><<<(C + 127) / 128, 128, 0, st>>>(stats, stats + C, gamma, beta, mean, invstd, a, b,
                                                      running_mean, running_var, (float)M, eps, momentum, C,
                                                      param_bf16, have_stats == 2 ? 1 : 0,
                                                      (long long*)num_batches_tracked);
  bn_apply_kernel<<<grid, THREADS, 0, st>>>((const uint4*)x, (const uint4*)res, (uint4*)y, a, b, nvec, V,
                                            relu, (uint8_t*)relu_mask);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("bn_fwd launch", e);
  return 0;
}

// ---- SyncBatchNorm building blocks: the same kernels with the cross-rank reduction between the passes ----
// local statistics only: stats[2*C] = sum | sum of squares over this rank's M rows
int b200dp_bn_stats(const void* x, float* stats, long long M, int C, unsigned long long stream) {
  if (!shape_ok(C) || check_vec16("bn_stats", {x})) return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(float) * 2 * C, st);
  if (e != cudaSuccess) return fail("memset", e);
  bn_stats_kernel<<<reduce_grid(), RTHREADS, 0, st>>>((const uint4*)x, stats, stats + C, (long long)M * (C / 8),
                                                      C / 8);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("bn_stats launch", e);
  return 0;
}

// finalize + apply with statistics that were summed over all ranks: `count` = the global number of rows, a
// device fp32 (the all-reduced stats[2*C]), so ranks may hold different numbers of rows, none included
int b200dp_bn_fwd_sync(const void* x, const void* res, void* y, const void* gamma, const void* beta,
                       const float* stats, float* mean, float* invstd, float* a, float* b, void* running_mean,
                       void* running_var, long long M_local, const float* count, int C, float eps, float momentum,
                       int relu, int param_bf16, void* relu_mask, unsigned long long stream) {
  if (!shape_ok(C) || check_vec16("bn_fwd_sync", {x, res, y})) return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int V = C / 8;
  const long long nvec = M_local * V;
  bn_finalize_kernel<true><<<(C + 127) / 128, 128, 0, st>>>(const_cast<float*>(stats), const_cast<float*>(stats) + C, gamma,
                                                      beta, mean, invstd, a, b, running_mean, running_var,
                                                      0.f, eps, momentum, C, param_bf16, 0, nullptr, count);
  bn_apply_kernel<<<grid_for(nvec, V), THREADS, 0, st>>>((const uint4*)x, (const uint4*)res, (uint4*)y, a, b, nvec,
                                                         V, relu, (uint8_t*)relu_mask);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("bn_fwd_sync launch", e);
  return 0;
}

// backward, pass 1: local sums[2*C] = sum dz | sum dz*(x - mean)     (dz = dy masked by the ReLU)
int b200dp_bn_bwd_reduce(const void* dy, const void* x, const void* relu_mask, const float* mean, float* sums,
                         long long M, int C, int relu, unsigned long long stream) {
  if (!shape_ok(C) || check_vec16("bn_bwd_reduce", {dy, x})) return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  cudaError_t e = cudaMemsetAsync(sums, 0, sizeof(float) * 2 * C, st);
  if (e != cudaSuccess) return fail("memset", e);
  bn_bwd_reduce_kernel<<<reduce_grid(), RTHREADS, 0, st>>>((const uint4*)dy, (const uint4*)x,
                                                           (const uint8_t*)relu_mask, mean, sums, sums + C,
                                                           (long long)M * (C / 8), C / 8, relu);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("bn_bwd_reduce launch", e);
  return 0;
}

// backward, pass 2 with globally summed `sums` and the global row count (device fp32, as in b200dp_bn_fwd_sync)
int b200dp_bn_bwd_apply(const void* dy, const void* x, const void* relu_mask, void* dx, void* dres,
                        const float* scale_a, const float* mean, const float* invstd, const float* sums,
                        const float* count, long long M, int C, int relu, unsigned long long stream) {
  if (!shape_ok(C) || check_vec16("bn_bwd_apply", {dy, x, dx, dres})) return -1;
  const int V = C / 8;
  const long long nvec = M * V;
  bn_bwd_apply_kernel<true><<<grid_for(nvec, V), THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>(
      (const uint4*)dy, (const uint4*)x, (const uint8_t*)relu_mask, (uint4*)dx, (uint4*)dres, mean, invstd, scale_a,
      sums, sums + C, 0.f, nvec, V, relu, nullptr, nullptr, 0, count);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("bn_bwd_apply launch", e);
  return 0;
}

// Inference / frozen-statistics apply: y = relu(x*a + b + res) with caller-provided a, b.
int b200dp_bn_apply(const void* x, const void* res, void* y, const float* a, const float* b, long long M,
                    int C, int relu, unsigned long long stream) {
  if (!shape_ok(C) || check_vec16("bn_apply", {x, res, y})) return -1;
  if (M == 0) return 0;
  const int V = C / 8;
  const long long nvec = M * V;
  bn_apply_kernel<<<grid_for(nvec, V), THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>(
      (const uint4*)x, (const uint4*)res, (uint4*)y, a, b, nvec, V, relu, nullptr);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("bn_apply launch", e);
  return 0;
}

// sums: [2*C] fp32 (zeroed here): sum_dy | sum_dy_xhat  (== dbeta | dgamma).
// `relu_mask`: the byte-per-8-channels mask written by b200dp_bn_fwd (required when relu != 0).
int b200dp_bn_bwd(const void* dy, const void* x, const void* relu_mask, void* dx, void* dres, const float* scale_a,
                  const float* mean, const float* invstd, float* sums, void* dgamma, void* dbeta,
                  int param_bf16, long long M, int C, int relu, unsigned long long stream) {
  if (!shape_ok(C) || check_vec16("bn_bwd", {dy, x, dx, dres})) return -1;
  if (M < 1) {
    snprintf(g_err, sizeof(g_err), "bn_bwd: needs at least one row");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int V = C / 8;
  const long long nvec = M * V;
  cudaError_t e = cudaMemsetAsync(sums, 0, sizeof(float) * 2 * C, st);
  if (e != cudaSuccess) return fail("memset", e);
  const int grid = grid_for(nvec, V);
  bn_bwd_reduce_kernel<<<reduce_grid(), RTHREADS, 0, st>>>((const uint4*)dy, (const uint4*)x,
                                                           (const uint8_t*)relu_mask, mean, sums, sums + C,
                                                           nvec, V, relu);
  bn_bwd_apply_kernel<false><<<grid, THREADS, 0, st>>>((const uint4*)dy, (const uint4*)x, (const uint8_t*)relu_mask,
                                                (uint4*)dx, (uint4*)dres, mean, invstd, scale_a, sums,
                                                sums + C, 1.0f / (float)M, nvec, V, relu, dgamma, dbeta,
                                                param_bf16);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("bn_bwd launch", e);
  return 0;
}

// 3x3/s2/p1 max-pool over NHWC bf16; idx: [N*OH*OW*C] bytes (arg-max tap per output element).
int b200dp_maxpool_fwd(const void* x, void* y, void* idx, int N, int H, int W, int C,
                       unsigned long long stream) {
  if (C % 8) return -1;
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1, V = C / 8;
  const long long total = (long long)N * OH * OW * V;
  int grid = (int)((total + THREADS - 1) / THREADS);
  if (grid > reduce_grid() * 16) grid = reduce_grid() * 16;
  maxpool_fwd_kernel<<<grid, THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>((const uint4*)x, (uint4*)y,
                                                                             (uint2*)idx, N, H, W, OH, OW, V);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("maxpool_fwd launch", e);
  return 0;
}

int b200dp_maxpool_bwd(const void* dy, const void* idx, void* dx, int N, int H, int W, int C,
                       unsigned long long stream) {
  if (C % 8) return -1;
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1, V = C / 8;
  if (H % 2 == 0 && W % 2 == 0) {
    const long long patches = (long long)N * (H / 2) * (W / 2) * V;
    int pgrid = (int)((patches + THREADS - 1) / THREADS);
    if (pgrid > reduce_grid() * 16) pgrid = reduce_grid() * 16;
    maxpool_bwd_patch_kernel<<<pgrid, THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>(
        (const uint4*)dy, (const uint2*)idx, (uint4*)dx, N, H, W, OH, OW, V);
    cudaError_t pe = cudaGetLastError();
    if (pe != cudaSuccess) return fail("maxpool_bwd launch", pe);
    return 0;
  }
  const long long total = (long long)N * H * W * V;
  int grid = (int)((total + THREADS - 1) / THREADS);
  if (grid > reduce_grid() * 16) grid = reduce_grid() * 16;
  maxpool_bwd_kernel<<<grid, THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>((const uint4*)dy, (const uint2*)idx,
                                                                             (uint4*)dx, N, H, W, OH, OW, V);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("maxpool_bwd launch", e);
  return 0;
}

// x: NHWC bf16 [N, HW, C] -> y [N, C] (C % 8 == 0)
int b200dp_avgpool_fwd(const void* x, void* y, long long N, int HW, int C, unsigned long long stream) {
  if (C % 8) return -1;
  const int V = C / 8;
  const long long total = N * V;
  int grid = (int)((total + THREADS - 1) / THREADS);
  if (grid > reduce_grid() * 8) grid = reduce_grid() * 8;
  avgpool_fwd_kernel<<<grid, THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>((const uint4*)x, (uint4*)y, HW, V, total,
                                                                             1.0f / (float)HW);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("avgpool_fwd launch", e);
  return 0;
}

int b200dp_avgpool_bwd(const void* dy, void* dx, long long N, int HW, int C, unsigned long long stream) {
  if (C % 8) return -1;
  const int V = C / 8;
  const long long total = N * HW * V;
  int grid = (int)((total + THREADS - 1) / THREADS);
  if (grid > reduce_grid() * 8) grid = reduce_grid() * 8;
  avgpool_bwd_kernel<<<grid, THREADS, 0, (cudaStream_t)(uintptr_t)stream>>>((const uint4*)dy, (uint4*)dx, HW, V, total,
                                                                             1.0f / (float)HW);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("avgpool_bwd launch", e);
  return 0;
}

// x: NHWC bf16 [N,H,W,3] (H, W multiples of 8); out: [N*OH*OW, 168] bf16, OH = H/2, OW = W/2.
int b200dp_stem_im2col(const void* x, void* out, int N, int H, int W, unsigned long long stream) {
  if ((W % 8) || (H % 2)) return -1;
  const int OH = H / 2, OW = W / 2;
  const size_t smem = (size_t)7 * ((9 + W * 3 + 15 + 7) & ~7) * sizeof(__nv_bfloat16);
  stem_im2col_kernel<<<N * OH, THREADS, smem, (cudaStream_t)(uintptr_t)stream>>>(
      (const __nv_bfloat16*)x, (uint4*)out, H, W, OH, OW);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("stem_im2col launch", e);
  return 0;
}

int b200dp_ln_supported(int C) { return (C % 256 == 0 && C / 256 >= 1 && C / 256 <= 4) ? 1 : 0; }

int b200dp_ln_fwd(const void* x, void* y, const void* gamma, const void* beta, float* mean, float* rstd,
                  long long rows, int C, float eps, int param_bf16, unsigned long long stream) {
  if (!b200dp_ln_supported(C) || check_vec16("ln_fwd", {x, y})) return -1;
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  long long blocks = (rows + LN_WARPS - 1) / LN_WARPS;
  if (blocks > reduce_grid() * 4) blocks = reduce_grid() * 4;
#define LN_FWD(V) ln_fwd_kernel<V><<<(int)blocks, LN_WARPS * 32, 0, st>>>((const uint4*)x, (uint4*)y, gamma, beta, mean, rstd, rows, eps, param_bf16)
  switch (C / 256) { case 1: LN_FWD(1); break; case 2: LN_FWD(2); break; case 3: LN_FWD(3); break; default: LN_FWD(4); }
#undef LN_FWD
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("ln_fwd launch", e);
  return 0;
}

// sums: [2*C] fp32 scratch (zeroed here); dgamma/dbeta written in the parameter dtype.
int b200dp_ln_bwd(const void* dy, const void* x, void* dx, const void* gamma, const float* mean,
                  const float* rstd, float* sums, void* dgamma, void* dbeta, long long rows, int C,
                  int param_bf16, unsigned long long stream) {
  if (!b200dp_ln_supported(C) || check_vec16("ln_bwd", {dy, x, dx})) return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  cudaError_t e = cudaMemsetAsync(sums, 0, sizeof(float) * 2 * C, st);
  if (e != cudaSuccess) return fail("memset", e);
  if (rows == 0) {   // no rows: zero parameter gradients, no row kernel
    ln_param_grad_kernel<<<(C + 255) / 256, 256, 0, st>>>(sums, dgamma, dbeta, C, param_bf16);
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail("ln_bwd launch", e);
  }
  long long blocks = (rows + LN_WARPS - 1) / LN_WARPS;
  if (blocks > reduce_grid() * 2) blocks = reduce_grid() * 2;
  const size_t smem = sizeof(float) * LN_WARPS * C;
#define LN_BWD(V)                                                                                      \
  do {                                                                                                 \
    static bool attr = false;                                                                          \
    if (!attr) {                                                                                       \
      cudaFuncSetAttribute(ln_bwd_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  \
      attr = true;                                                                                     \
    }                                                                                                  \
    ln_bwd_kernel<V><<<(int)blocks, LN_WARPS * 32, smem, st>>>((const uint4*)dy, (const uint4*)x,      \
                                                               (uint4*)dx, gamma, mean, rstd, sums,    \
                                                               rows, param_bf16);                      \
  } while (0)
  switch (C / 256) { case 1: LN_BWD(1); break; case 2: LN_BWD(2); break; case 3: LN_BWD(3); break; default: LN_BWD(4); }
#undef LN_BWD
  ln_param_grad_kernel<<<(C + 255) / 256, 256, 0, st>>>(sums, dgamma, dbeta, C, param_bf16);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("ln_bwd launch", e);
  return 0;
}

}  // extern "C"

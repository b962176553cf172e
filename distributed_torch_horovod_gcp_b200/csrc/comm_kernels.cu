// sm_90a communication kernels over NVLink / NVSwitch peer memory.
//
// K1 one-shot allreduce  : every rank loads the same 16-byte chunk from all peers (P2P ld over
//                          NVLink), sums in fp32 in fixed rank order (bit-identical on all
//                          ranks) and applies the epilogue locally.  Latency-optimal.
// K2 two-shot allreduce  : rank r reduces slice r from all peers (P2P ld), applies the
//                          epilogue, and pushes the result slice to every peer (P2P st).
// K3 NVLS allreduce      : multimem.ld_reduce on the multicast address (the NVSwitch performs
//                          the reduction), epilogue, multimem.st broadcast of the result.
// K4 broadcast           : root pushes its buffer to all peers (multimem.st or P2P st).
// K7 fused epilogue      : x 1/N (and pre/post-scale), cast, SGD-momentum / Adam / AdamW update
//                          with fp32 master weights + optimizer state, writing the updated
//                          parameters (for K2/K3: *parameters* are broadcast instead of the
//                          reduced gradient, which removes one full pass and shards the state).
//
// These replace Horovod's NCCL allreduce/broadcast ops, its ScaleBuffer kernel and the
// separate optimizer step (SURVEY.md §2.2 N6/N7/N8/N15, §2.6 S8/S9; reference call sites
// app/torch_train.py:259,266,277,280).  No NCCL call is made on this path.
//
// Cross-GPU synchronisation: per-(channel, block, peer) monotonic counters in a symmetric
// "signal pad".  A barrier = red.release.sys +1 into every peer's pad, then spin with
// ld.acquire.sys on the local pad until the peer's counter reaches the locally tracked
// epoch.  Counters live in device memory, so the kernels are CUDA-graph replay safe.  Every
// spin is bounded by %globaltimer: on timeout the kernel records (code, peer, block) in a
// host-mapped mailbox and returns instead of hanging the GPU (SURVEY.md §5.3).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define B200DP_MAX_RANKS 8
#define B200DP_MAX_BLOCKS 128
#define B200DP_NUM_CHANNELS 4

extern "C" {

struct CommCtx {
  uint32_t* sig[B200DP_MAX_RANKS];  // signal pads of every rank (peer-mapped VAs)
  uint32_t* epoch;                  // local counters [channel][block][peer]
  int* err;                         // host-mapped mailbox: {code, peer, block, channel}
  unsigned long long timeout_ns;
  int rank;
  int world;
};

enum { OPT_NONE = 0, OPT_SGD = 1, OPT_ADAM = 2 };

struct OptHyper {
  int kind;        // OPT_*
  int nesterov;
  int adamw;       // decoupled weight decay
  int maximize;
  float lr;
  float momentum;
  float dampening;
  float weight_decay;
  float beta1;
  float beta2;
  float eps;
  float pad_;
};

struct ARArgs {
  const void* in[B200DP_MAX_RANKS];  // gradient bucket on every rank
  void* out[B200DP_MAX_RANKS];       // result / parameter bucket on every rank
  const void* in_mc;                 // multicast VA of the gradient bucket (NVLS)
  void* out_mc;                      // multicast VA of the result bucket (NVLS)
  float* master;                     // fp32 master weights (nullptr: `out` is fp32 and is the master)
  float* s0;                         // momentum buffer | exp_avg
  float* s1;                         // exp_avg_sq
  int* step_ctr;                     // completed optimizer steps for this bucket (device)
  unsigned int* ticket;              // last-block detection (device)
  const float* lr_scale;             // optional device scalar multiplied into lr (graph-safe LR schedules)
  void* scratch;                     // one-shot in-place: local scratch of n elements
  unsigned long long n;              // elements
  float scale;                       // applied to the fp32 sum (1/N, pre*post scale)
  int channel;
  int zero_input;                    // zero the local gradient bucket after the closing barrier
  int copy_back;                     // one-shot in-place: copy scratch -> in[rank] after the barrier
  OptHyper h;
};

// reduce-scatter / all-gather / all-to-all over peer memory (equal chunks of `chunk` elements per rank)
struct CollArgs {
  const void* src[B200DP_MAX_RANKS];  // reduce-scatter: every rank's (symmetric) input; others: [rank] = local input
  void* dst[B200DP_MAX_RANKS];        // all-gather / all-to-all: every rank's (symmetric) output; RS: [rank] = local out
  const void* src_mc;                 // multicast VA of the inputs  (NVLS reduce-scatter)
  void* dst_mc;                       // multicast VA of the outputs (NVLS all-gather)
  unsigned long long chunk;           // elements per rank chunk (16-byte multiple)
  float scale;
  int channel;
  int use_mc;
  int pad_;
};

struct BcastArgs {
  void* buf[B200DP_MAX_RANKS];
  void* buf_mc;
  unsigned long long nbytes;  // multiple of 16
  int root;
  int channel;
  int use_mc;
  int pad_;
};

}  // extern "C"

namespace {

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_peer_v4(const void* p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_peer_v4(void* p, uint4 v) {
  asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void mc_st_v4(void* p, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 mc_ld_reduce_f32(const void* p) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 mc_ld_reduce_bf16(const void* p) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 mc_ld_reduce_f16(const void* p) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ------------------------------------------------------------------ cross-rank block barrier
// Block b of every rank meets block b of every other rank.  acq_rel: writes made by this
// block before the barrier (P2P / multimem stores) are visible to peers after it.
__device__ __forceinline__ bool rank_barrier(const CommCtx& c, int channel) {
  __shared__ int s_failed;
  if (threadIdx.x == 0) s_failed = 0;
  __syncthreads();
  const int t = threadIdx.x;
  if (c.world > 1 && t < c.world && t != c.rank) {
    const int base = (channel * B200DP_MAX_BLOCKS + (int)blockIdx.x) * B200DP_MAX_RANKS;
    const uint32_t e = c.epoch[base + t] + 1u;
    c.epoch[base + t] = e;
    red_add_release_sys(c.sig[t] + base + c.rank, 1u);
    const uint32_t* mine = c.sig[c.rank] + base + t;
    unsigned long long t0 = 0;
    unsigned spins = 0;
    while ((int)(ld_acquire_sys(mine) - e) < 0) {
      if (++spins > 4096u) {
        spins = 0;
        const unsigned long long now = globaltimer_ns();
        if (t0 == 0) {
          t0 = now;
        } else if (now - t0 > c.timeout_ns || *(volatile int*)c.err != 0) {
          volatile int* mb = c.err;     // host-mapped mailbox; benign race between reporters
          if (mb[0] == 0) {
            mb[1] = t;
            mb[2] = (int)blockIdx.x;
            mb[3] = channel;
            __threadfence_system();
            mb[0] = 1;
            __threadfence_system();
          }
          s_failed = 1;
          break;
        }
        __nanosleep(64);
      }
    }
  }
  __syncthreads();
  return s_failed == 0;
}

// After a watchdog expiry the data behind the barrier is incomplete: rank_barrier returns false and the
// kernels return without reducing / writing anything (the host raises HorovodInternalError from the
// mailbox) instead of producing silently wrong results.

// ------------------------------------------------------------------ vector <-> fp32 helpers
template <typename T>
struct Vec;  // 16 bytes of T

template <>
struct Vec<float> {
  static constexpr int N = 4;
  __device__ static void unpack(const uint4& v, float* f) {
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
    f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
  }
  __device__ static uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                      __float_as_uint(f[3]));
  }
  __device__ static uint4 mc_reduce(const void* p) { return mc_ld_reduce_f32(p); }
};

template <>
struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static void unpack(const uint4& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ static uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  __device__ static uint4 mc_reduce(const void* p) { return mc_ld_reduce_bf16(p); }
};

template <>
struct Vec<__half> {
  static constexpr int N = 8;
  __device__ static void unpack(const uint4& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
      float2 x = __half22float2(h);
      f[2 * i] = x.x;
      f[2 * i + 1] = x.y;
    }
  }
  __device__ static uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  __device__ static uint4 mc_reduce(const void* p) { return mc_ld_reduce_f16(p); }
};

// ------------------------------------------------------------------ K7: fused optimizer epilogue
// `g[]` holds the reduced gradient of VN consecutive elements starting at element `idx`.
// Returns the values to store in the result bucket (updated parameters, or the scaled
// gradient when no optimizer is fused) in `o[]`.
struct StepInfo {
  int first;      // first optimizer step (SGD momentum buffer initialisation)
  float bc1;      // Adam bias corrections for this step
  float bc2_sqrt;
  float lr;
};

__device__ __forceinline__ StepInfo make_step(const ARArgs& a) {
  StepInfo s;
  const int t = a.step_ctr ? *a.step_ctr : 0;
  s.first = (t == 0);
  s.lr = a.h.lr * (a.lr_scale ? *a.lr_scale : 1.0f);
  if (a.h.kind == OPT_ADAM) {
    const float tf = (float)(t + 1);
    s.bc1 = 1.0f - powf(a.h.beta1, tf);
    s.bc2_sqrt = sqrtf(1.0f - powf(a.h.beta2, tf));
  } else {
    s.bc1 = 1.0f;
    s.bc2_sqrt = 1.0f;
  }
  return s;
}

template <typename T, int VN>
__device__ __forceinline__ void epilogue(const ARArgs& a, const StepInfo& s, size_t idx, float* g,
                                         const T* out_local, float* o) {
#pragma unroll
  for (int i = 0; i < VN; ++i) g[i] *= a.scale;
  if (a.h.kind == OPT_NONE) {
#pragma unroll
    for (int i = 0; i < VN; ++i) o[i] = g[i];
    return;
  }
  float p[VN];
  if (a.master) {
#pragma unroll
    for (int i = 0; i < VN; i += 4) {
      const float4 m = *reinterpret_cast<const float4*>(a.master + idx + i);
      p[i] = m.x; p[i + 1] = m.y; p[i + 2] = m.z; p[i + 3] = m.w;
    }
  } else {  // the result bucket is fp32 and is the master copy
    const uint4 v = *reinterpret_cast<const uint4*>(out_local + idx);
    Vec<T>::unpack(v, p);
  }
  if (a.h.maximize) {
#pragma unroll
    for (int i = 0; i < VN; ++i) g[i] = -g[i];
  }
  if (a.h.kind == OPT_SGD) {
    if (a.h.weight_decay != 0.0f) {
#pragma unroll
      for (int i = 0; i < VN; ++i) g[i] = fmaf(a.h.weight_decay, p[i], g[i]);
    }
    if (a.h.momentum != 0.0f) {
      float b[VN];
      if (s.first) {
#pragma unroll
        for (int i = 0; i < VN; ++i) b[i] = g[i];
      } else {
#pragma unroll
        for (int i = 0; i < VN; i += 4) {
          const float4 m = *reinterpret_cast<const float4*>(a.s0 + idx + i);
          b[i] = m.x; b[i + 1] = m.y; b[i + 2] = m.z; b[i + 3] = m.w;
        }
#pragma unroll
        for (int i = 0; i < VN; ++i)
          b[i] = fmaf(a.h.momentum, b[i], (1.0f - a.h.dampening) * g[i]);
      }
#pragma unroll
      for (int i = 0; i < VN; i += 4)
        *reinterpret_cast<float4*>(a.s0 + idx + i) = make_float4(b[i], b[i + 1], b[i + 2], b[i + 3]);
#pragma unroll
      for (int i = 0; i < VN; ++i) g[i] = a.h.nesterov ? fmaf(a.h.momentum, b[i], g[i]) : b[i];
    }
#pragma unroll
    for (int i = 0; i < VN; ++i) p[i] = fmaf(-s.lr, g[i], p[i]);
  } else {  // Adam / AdamW (torch.optim semantics, non-amsgrad)
    float m[VN], v[VN];
#pragma unroll
    for (int i = 0; i < VN; i += 4) {
      const float4 a0 = *reinterpret_cast<const float4*>(a.s0 + idx + i);
      const float4 a1 = *reinterpret_cast<const float4*>(a.s1 + idx + i);
      m[i] = a0.x; m[i + 1] = a0.y; m[i + 2] = a0.z; m[i + 3] = a0.w;
      v[i] = a1.x; v[i + 1] = a1.y; v[i + 2] = a1.z; v[i + 3] = a1.w;
    }
#pragma unroll
    for (int i = 0; i < VN; ++i) {
      if (a.h.adamw) {
        p[i] *= (1.0f - s.lr * a.h.weight_decay);
      } else if (a.h.weight_decay != 0.0f) {
        g[i] = fmaf(a.h.weight_decay, p[i], g[i]);
      }
      m[i] = fmaf(a.h.beta1, m[i], (1.0f - a.h.beta1) * g[i]);      // lerp(m, g, 1-b1)
      v[i] = fmaf(a.h.beta2, v[i], (1.0f - a.h.beta2) * g[i] * g[i]);
      const float denom = sqrtf(v[i]) / s.bc2_sqrt + a.h.eps;
      p[i] = fmaf(-(s.lr / s.bc1), m[i] / denom, p[i]);
    }
#pragma unroll
    for (int i = 0; i < VN; i += 4) {
      *reinterpret_cast<float4*>(a.s0 + idx + i) = make_float4(m[i], m[i + 1], m[i + 2], m[i + 3]);
      *reinterpret_cast<float4*>(a.s1 + idx + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
    }
  }
  if (a.master) {
#pragma unroll
    for (int i = 0; i < VN; i += 4)
      *reinterpret_cast<float4*>(a.master + idx + i) = make_float4(p[i], p[i + 1], p[i + 2], p[i + 3]);
  }
#pragma unroll
  for (int i = 0; i < VN; ++i) o[i] = p[i];
}

// The last block to finish bumps the per-bucket step counter (all blocks read it first).
__device__ __forceinline__ void finish_step(const ARArgs& a) {
  if (a.step_ctr == nullptr || a.ticket == nullptr) return;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int t = atomicAdd(a.ticket, 1u);
    if (t == gridDim.x - 1) {
      *a.ticket = 0u;
      *a.step_ctr = *a.step_ctr + 1;
      __threadfence();
    }
  }
}

// ------------------------------------------------------------------ K1: one-shot
template <typename T>
__global__ void __launch_bounds__(512) allreduce_oneshot_kernel(CommCtx c, ARArgs a) {
  constexpr int VN = Vec<T>::N;
  const size_t nvec = a.n / VN;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const StepInfo s = make_step(a);
  T* out_local = reinterpret_cast<T*>(a.copy_back ? a.scratch : a.out[c.rank]);

  if (!rank_barrier(c, a.channel)) return;  // every peer's gradients are complete
  for (size_t v = start; v < nvec; v += stride) {
    uint4 raw[B200DP_MAX_RANKS];
#pragma unroll
    for (int r = 0; r < B200DP_MAX_RANKS; ++r)
      if (r < c.world) raw[r] = ld_peer_v4(reinterpret_cast<const uint4*>(a.in[r]) + v);
    float acc[VN], f[VN];
#pragma unroll
    for (int i = 0; i < VN; ++i) acc[i] = 0.0f;
#pragma unroll
    for (int r = 0; r < B200DP_MAX_RANKS; ++r) {  // fixed order => bit-identical on all ranks
      if (r < c.world) {
        Vec<T>::unpack(raw[r], f);
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[i] += f[i];
      }
    }
    float o[VN];
    epilogue<T, VN>(a, s, v * VN, acc, reinterpret_cast<const T*>(a.out[c.rank]), o);
    reinterpret_cast<uint4*>(out_local)[v] = Vec<T>::pack(o);
  }
  rank_barrier(c, a.channel);  // every peer has finished reading my gradients
  if (a.copy_back | a.zero_input) {
    uint4* mine = reinterpret_cast<uint4*>(const_cast<void*>(a.in[c.rank]));
    for (size_t v = start; v < nvec; v += stride)
      mine[v] = a.copy_back ? reinterpret_cast<const uint4*>(a.scratch)[v] : make_uint4(0, 0, 0, 0);
  }
  finish_step(a);
}

// ------------------------------------------------------------------ K2: two-shot (P2P) and K3: NVLS
template <typename T, bool kNVLS>
__global__ void __launch_bounds__(512) allreduce_sliced_kernel(CommCtx c, ARArgs a) {
  constexpr int VN = Vec<T>::N;
  const size_t nvec = a.n / VN;
  const size_t per = (nvec + c.world - 1) / c.world;
  const size_t lo = min((size_t)c.rank * per, nvec);
  const size_t hi = min(lo + per, nvec);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const StepInfo s = make_step(a);

  if (!rank_barrier(c, a.channel)) return;
  // U independent 16-byte transactions per thread are issued before any is consumed: NVLink
  // round trips are ~2 us, so bytes-in-flight (not instruction count) bounds the bandwidth.
  constexpr int U = kNVLS ? 4 : 2;
  for (size_t v0 = lo + start; v0 < hi; v0 += U * stride) {
    float acc[U][VN];
    if (kNVLS) {
      uint4 red[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = v0 + u * stride;
        if (v < hi) red[u] = Vec<T>::mc_reduce(reinterpret_cast<const uint4*>(a.in_mc) + v);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) Vec<T>::unpack(red[u], acc[u]);
    } else {
      uint4 raw[U][B200DP_MAX_RANKS];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = v0 + u * stride;
#pragma unroll
        for (int r = 0; r < B200DP_MAX_RANKS; ++r)
          if (r < c.world && v < hi) raw[u][r] = ld_peer_v4(reinterpret_cast<const uint4*>(a.in[r]) + v);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float f[VN];
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[u][i] = 0.0f;
#pragma unroll
        for (int r = 0; r < B200DP_MAX_RANKS; ++r) {
          if (r < c.world) {
            Vec<T>::unpack(raw[u][r], f);
#pragma unroll
            for (int i = 0; i < VN; ++i) acc[u][i] += f[i];
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t v = v0 + u * stride;
      if (v >= hi) break;
      float o[VN];
      epilogue<T, VN>(a, s, v * VN, acc[u], reinterpret_cast<const T*>(a.out[c.rank]), o);
      const uint4 packed = Vec<T>::pack(o);
      if (kNVLS) {
        mc_st_v4(reinterpret_cast<uint4*>(a.out_mc) + v, packed);
      } else {
#pragma unroll
        for (int r = 0; r < B200DP_MAX_RANKS; ++r)
          if (r < c.world) st_peer_v4(reinterpret_cast<uint4*>(a.out[r]) + v, packed);
      }
    }
  }
  rank_barrier(c, a.channel);  // pushes visible everywhere; peers done reading my gradients
  if (a.zero_input && a.in[c.rank] != a.out[c.rank]) {
    // mirror the peers' read pattern: peer q's block b read slice q with this block's stride
    uint4* mine = reinterpret_cast<uint4*>(const_cast<void*>(a.in[c.rank]));
    for (int q = 0; q < c.world; ++q) {
      const size_t qlo = min((size_t)q * per, nvec), qhi = min(qlo + per, nvec);
      for (size_t v = qlo + start; v < qhi; v += stride) mine[v] = make_uint4(0, 0, 0, 0);
    }
  }
  finish_step(a);
}

// ------------------------------------------------------------------ reduce-scatter / all-gather / all-to-all
// The two halves of the sliced allreduce as stand-alone collectives, plus the personalised exchange.
// Reduce-scatter: rank r reads chunk r of every peer (P2P loads, or ONE multimem.ld_reduce per 16 bytes when
// the switch does the sum) and keeps scale * sum locally — (N-1)/N * S bytes in per rank instead of the
// 2 * S an allreduce-then-slice moves.  All-gather: rank r pushes its chunk into slot r of every peer
// (one multimem.st per 16 bytes with NVLS).  All-to-all: rank r pushes chunk j into slot r of peer j.
template <typename T, bool kNVLS>
__global__ void __launch_bounds__(512) reducescatter_kernel(CommCtx c, CollArgs a) {
  constexpr int VN = Vec<T>::N;
  const size_t nvec = a.chunk / VN;
  const size_t base = (size_t)c.rank * nvec;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint4* out = reinterpret_cast<uint4*>(a.dst[c.rank]);
  if (!rank_barrier(c, a.channel)) return;
  constexpr int U = kNVLS ? 4 : 2;
  for (size_t v0 = start; v0 < nvec; v0 += U * stride) {
    float acc[U][VN];
    if (kNVLS) {
      uint4 red[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = v0 + u * stride;
        if (v < nvec) red[u] = Vec<T>::mc_reduce(reinterpret_cast<const uint4*>(a.src_mc) + base + v);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) Vec<T>::unpack(red[u], acc[u]);
    } else {
      uint4 raw[U][B200DP_MAX_RANKS];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = v0 + u * stride;
#pragma unroll
        for (int r = 0; r < B200DP_MAX_RANKS; ++r)
          if (r < c.world && v < nvec) raw[u][r] = ld_peer_v4(reinterpret_cast<const uint4*>(a.src[r]) + base + v);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float f[VN];
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[u][i] = 0.0f;
#pragma unroll
        for (int r = 0; r < B200DP_MAX_RANKS; ++r) {   // fixed rank order
          if (r < c.world) {
            Vec<T>::unpack(raw[u][r], f);
#pragma unroll
            for (int i = 0; i < VN; ++i) acc[u][i] += f[i];
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t v = v0 + u * stride;
      if (v >= nvec) break;
#pragma unroll
      for (int i = 0; i < VN; ++i) acc[u][i] *= a.scale;
      out[v] = Vec<T>::pack(acc[u]);
    }
  }
  rank_barrier(c, a.channel);   // peers have finished reading my input
}

__global__ void __launch_bounds__(512) allgather_kernel(CommCtx c, CollArgs a) {
  const size_t nvec = a.chunk;   // chunk is given in 16-byte vectors for the copy collectives
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(a.src[c.rank]);
  const size_t slot = (size_t)c.rank * nvec;
  if (!rank_barrier(c, a.channel)) return;   // every rank's output is free to overwrite
  for (size_t v = start; v < nvec; v += stride) {
    const uint4 x = src[v];
    if (a.use_mc) {
      mc_st_v4(reinterpret_cast<uint4*>(a.dst_mc) + slot + v, x);
    } else {
#pragma unroll
      for (int r = 0; r < B200DP_MAX_RANKS; ++r)
        if (r < c.world) st_peer_v4(reinterpret_cast<uint4*>(a.dst[r]) + slot + v, x);
    }
  }
  rank_barrier(c, a.channel);   // all pushes visible everywhere
}

__global__ void __launch_bounds__(512) alltoall_kernel(CommCtx c, CollArgs a) {
  const size_t nvec = a.chunk;   // 16-byte vectors per (source, destination) pair
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(a.src[c.rank]);
  const size_t slot = (size_t)c.rank * nvec;
  if (!rank_barrier(c, a.channel)) return;
  for (int j = 0; j < c.world; ++j) {
    const int peer = (c.rank + j) % c.world;          // staggered: no two ranks hammer the same peer first
    uint4* dst = reinterpret_cast<uint4*>(a.dst[peer]) + slot;
    const uint4* sp = src + (size_t)peer * nvec;
    for (size_t v = start; v < nvec; v += stride) st_peer_v4(dst + v, sp[v]);
  }
  rank_barrier(c, a.channel);
}

// ------------------------------------------------------------------ K4: broadcast
__global__ void __launch_bounds__(512) broadcast_kernel(CommCtx c, BcastArgs a) {
  const size_t nvec = a.nbytes / 16;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (!rank_barrier(c, a.channel)) return;  // destination buffers are free to overwrite on every rank
  if (c.rank == a.root) {
    const uint4* src = reinterpret_cast<const uint4*>(a.buf[c.rank]);
    for (size_t v = start; v < nvec; v += stride) {
      const uint4 x = src[v];
      if (a.use_mc) {
        mc_st_v4(reinterpret_cast<uint4*>(a.buf_mc) + v, x);   // one store, switch fans out
      } else {
#pragma unroll
        for (int r = 0; r < B200DP_MAX_RANKS; ++r)
          if (r < c.world && r != c.rank) st_peer_v4(reinterpret_cast<uint4*>(a.buf[r]) + v, x);
      }
    }
  }
  rank_barrier(c, a.channel);  // root's stores are visible to every rank
}

// ------------------------------------------------------------------ local helpers
template <typename T>
cudaError_t launch_ar(const CommCtx& c, const ARArgs& a, int algo, int blocks, int threads,
                      cudaStream_t st) {
  if (algo == 0) {
    allreduce_oneshot_kernel<T><<<blocks, threads, 0, st>>>(c, a);
  } else if (algo == 1) {
    allreduce_sliced_kernel<T, false><<<blocks, threads, 0, st>>>(c, a);
  } else {
    allreduce_sliced_kernel<T, true><<<blocks, threads, 0, st>>>(c, a);
  }
  return cudaGetLastError();
}

}  // namespace

extern "C" {

static thread_local char g_comm_err[256];
const char* b200dp_comm_last_error() { return g_comm_err; }

int b200dp_comm_limits(int* max_ranks, int* max_blocks, int* channels, int* ctx_bytes,
                       int* ar_bytes, int* bc_bytes) {
  *max_ranks = B200DP_MAX_RANKS;
  *max_blocks = B200DP_MAX_BLOCKS;
  *channels = B200DP_NUM_CHANNELS;
  *ctx_bytes = (int)sizeof(CommCtx);
  *ar_bytes = (int)sizeof(ARArgs);
  *bc_bytes = (int)sizeof(BcastArgs);
  return 0;
}

// algo: 0 one-shot, 1 two-shot, 2 NVLS.  dtype: 0 fp32, 1 bf16, 2 fp16.
int b200dp_comm_allreduce(const CommCtx* ctx, const ARArgs* args, int algo, int dtype, int blocks,
                          int threads, unsigned long long stream) {
  if (blocks < 1 || blocks > B200DP_MAX_BLOCKS || threads < 32 || threads > 512 ||
      ctx->world > B200DP_MAX_RANKS || args->channel < 0 || args->channel >= B200DP_NUM_CHANNELS) {
    snprintf(g_comm_err, sizeof(g_comm_err), "bad launch config blocks=%d threads=%d world=%d ch=%d",
             blocks, threads, ctx->world, args->channel);
    return -1;
  }
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  cudaError_t e;
  if (dtype == 0) e = launch_ar<float>(*ctx, *args, algo, blocks, threads, st);
  else if (dtype == 1) e = launch_ar<__nv_bfloat16>(*ctx, *args, algo, blocks, threads, st);
  else if (dtype == 2) e = launch_ar<__half>(*ctx, *args, algo, blocks, threads, st);
  else e = cudaErrorInvalidValue;
  if (e != cudaSuccess) {
    snprintf(g_comm_err, sizeof(g_comm_err), "allreduce launch: %s", cudaGetErrorString(e));
    return -1;
  }
  return 0;
}

// mode: 0 reduce-scatter, 1 all-gather, 2 all-to-all.  dtype as in b200dp_comm_allreduce (reduce-scatter only).
int b200dp_comm_collective(const CommCtx* ctx, const CollArgs* args, int mode, int dtype, int blocks, int threads,
                           unsigned long long stream) {
  if (blocks < 1 || blocks > B200DP_MAX_BLOCKS || threads < 32 || threads > 512 ||
      args->channel < 0 || args->channel >= B200DP_NUM_CHANNELS) {
    snprintf(g_comm_err, sizeof(g_comm_err), "bad launch config");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  if (mode == 0) {
    const bool mc = args->use_mc != 0;
    if (dtype == 0) {
      if (mc) reducescatter_kernel<float, true><<<blocks, threads, 0, st>>>(*ctx, *args);
      else reducescatter_kernel<float, false><<<blocks, threads, 0, st>>>(*ctx, *args);
    } else if (dtype == 1) {
      if (mc) reducescatter_kernel<__nv_bfloat16, true><<<blocks, threads, 0, st>>>(*ctx, *args);
      else reducescatter_kernel<__nv_bfloat16, false><<<blocks, threads, 0, st>>>(*ctx, *args);
    } else if (dtype == 2) {
      if (mc) reducescatter_kernel<__half, true><<<blocks, threads, 0, st>>>(*ctx, *args);
      else reducescatter_kernel<__half, false><<<blocks, threads, 0, st>>>(*ctx, *args);
    } else {
      snprintf(g_comm_err, sizeof(g_comm_err), "reduce-scatter: unsupported dtype %d", dtype);
      return -1;
    }
  } else if (mode == 1) {
    allgather_kernel<<<blocks, threads, 0, st>>>(*ctx, *args);
  } else if (mode == 2) {
    alltoall_kernel<<<blocks, threads, 0, st>>>(*ctx, *args);
  } else {
    snprintf(g_comm_err, sizeof(g_comm_err), "unknown collective mode %d", mode);
    return -1;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    snprintf(g_comm_err, sizeof(g_comm_err), "collective launch: %s", cudaGetErrorString(e));
    return -1;
  }
  return 0;
}

int b200dp_comm_coll_bytes() { return (int)sizeof(CollArgs); }

int b200dp_comm_broadcast(const CommCtx* ctx, const BcastArgs* args, int blocks, int threads,
                          unsigned long long stream) {
  if (blocks < 1 || blocks > B200DP_MAX_BLOCKS || threads < 32 || threads > 512) {
    snprintf(g_comm_err, sizeof(g_comm_err), "bad launch config");
    return -1;
  }
  broadcast_kernel<<<blocks, threads, 0, (cudaStream_t)(uintptr_t)stream>>>(*ctx, *args);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    snprintf(g_comm_err, sizeof(g_comm_err), "broadcast launch: %s", cudaGetErrorString(e));
    return -1;
  }
  return 0;
}

}  // extern "C"

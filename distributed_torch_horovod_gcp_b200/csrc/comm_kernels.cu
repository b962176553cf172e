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

enum { OPT_NONE = 0, OPT_SGD = 1, OPT_ADAM = 2, OPT_LARS = 3, OPT_LAMB = 4, OPT_MUON = 5 };

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

// Global-norm gradient clipping on the one-shot path (max_grad_norm=).  The per-bucket kernel is split in
// three: K1c reduces into the fp32 arena `r` and writes one sum-of-squares slot per CTA, K8 folds every
// slot into the norm and the clip coefficient, K9 scales `r` by the coefficient and runs the K7 epilogue.
struct ClipArgs {
  float* r;                // fp32 reduced gradient of this bucket (scale * sum), n elements
  float* slots;            // K1c: this bucket's B200DP_MAX_BLOCKS slots; K8: the first slot of all buckets
  float* norm;             // device scalar: total L2 norm before clipping (K8 writes it)
  float* coef;             // device scalar: min(max_norm / (norm + 1e-6), 1) (K8 writes, K9 reads)
  float max_norm;
  int nslots;              // K8: number of slots (buckets * B200DP_MAX_BLOCKS)
};

// Layer-wise adaptive optimizers (LARS / LAMB, h.kind OPT_LARS / OPT_LAMB) on the one-shot path.  Each tensor's
// update is scaled by a trust ratio built from norms over the whole tensor, so the bucket kernel is split in
// two, both launched from the bucket-ready hook: K10 reduces, forms the update direction into the fp32 arena
// `r` and writes per-chunk partial sums of squares; K11 folds each tensor's partials into its trust ratio and
// applies the update.  A chunk is a fixed-size slice of one tensor (the host builds the table once).
struct LwChunk {
  int first_vec;  // first 16-byte vector of the chunk in the bucket
  int nvec;       // vectors in the chunk
  int tfirst;     // first chunk of the tensor the chunk belongs to (index into this bucket's table)
  int tcount;     // chunks of that tensor
};

// A bucket's slice of the chunk table and of the arrays indexed by it, shared by LARS / LAMB and Muon.
struct ChunkArgs {
  float* r;                // fp32 arena of this bucket: the update direction (K10) or Muon's u (K12)
  float* part;             // per chunk: two fp32 partial sums of squares (K10 / K12 write, K11 / K13 read)
  const LwChunk* chunks;   // this bucket's chunk table
  int nchunks;
  int pad_;
};

struct LwArgs {
  ChunkArgs tab;           // r: LARS g + wd w, LAMB m^/(sqrt(v^)+eps) + wd w; part: {sum of w^2, sum of r^2}
  float* ratio;            // per chunk: the tensor's trust ratio, written at the tensor's first chunk (K11)
  int adaptive;            // 0: trust ratio 1 (biases, norm layers)
  float trust_coef;        // LARS eta; 1 for LAMB
};

// Muon (h.kind OPT_MUON) on the one-shot path.  A bucket of matrices runs in three phases here, all launched from
// the bucket-ready hook, around the Newton-Schulz GEMMs that the host launches on the wgmma kernel between phases 1
// and 2: phase 0 (K12) reduces, updates the momentum buffer in s0, writes u to `r` and per-chunk sums of squares of
// u; phase 1 (K13) folds each matrix's partials into its norm and writes X0 = bf16(u / max(norm, eps)), transposed
// for tall matrices so that every NS operand has rows <= cols; phase 2 (K14) applies the decay and the NS result O.
// `tab` is LARS / LAMB's chunk table (ChunkArgs); `mats` gives the matrix of each chunk.
struct MuonMat {
  int rows;       // the parameter's shape
  int cols;
  int elem0;      // its first element in the bucket
  int x0;         // first element of its NS operand in `x0` / `o`: [min(rows, cols)][max(rows, cols)] bf16
};

struct MuonArgs {
  ChunkArgs tab;             // r: u (nesterov: g.lerp(buf, momentum), else buf); part: {sum of u^2, 0}
  const MuonMat* mats;       // per chunk: the matrix the chunk belongs to
  __nv_bfloat16* x0;         // K13: the bucket's NS inputs
  const __nv_bfloat16* o;    // K14: the bucket's NS results, laid out as x0
  int nesterov;
  int lr_mode;               // learning-rate factor f: 0 sqrt(max(1, rows / cols)), 1 0.2 sqrt(max(rows, cols))
  float eps;                 // clamp of the norm
  int pad_;
};

// reduce-scatter / all-gather among a group of ranks: `coll`'s pointers are indexed by group rank (the index in
// `members`), and multicast is never used (the world's multicast object spans non-members' buffers too).
struct GroupCollArgs {
  CollArgs coll;                    // src[] / dst[] by group rank; use_mc must be 0
  int members[B200DP_MAX_RANKS];    // world ranks of the group, ascending
  int size;                         // ranks in the group
  int index;                        // this rank's group rank: members[index] == CommCtx::rank
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
// Spin until this rank's pad entry `mine` (written by world rank `peer`) reaches epoch `e`.  False after the
// watchdog expires or another block has reported a failure; the first reporter records (1, peer, block, channel)
// in the mailbox.
__device__ __forceinline__ bool wait_for_peer(const CommCtx& c, const uint32_t* mine, uint32_t e, int peer,
                                              int channel) {
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
          mb[1] = peer;
          mb[2] = (int)blockIdx.x;
          mb[3] = channel;
          __threadfence_system();
          mb[0] = 1;
          __threadfence_system();
        }
        return false;
      }
      __nanosleep(64);
    }
  }
  return true;
}

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
    if (!wait_for_peer(c, c.sig[c.rank] + base + t, e, t, channel)) s_failed = 1;
  }
  __syncthreads();
  return s_failed == 0;
}

// The same barrier among the members of a group only.  The pad and epoch entries stay indexed by WORLD rank, so
// the counter of an ordered pair of ranks counts exactly the collectives both took part in, whether world or group
// ones, and a channel can carry both.  (Indexed by group rank, world ranks 0 and 2 would both credit slot 0 of
// rank 3's pad when they lead groups {0, 1, 3} and {2, 3}.)
__device__ __forceinline__ bool group_barrier(const CommCtx& c, const GroupCollArgs& g, int channel) {
  __shared__ int s_failed;
  if (threadIdx.x == 0) s_failed = 0;
  __syncthreads();
  const int t = threadIdx.x;
  if (g.size > 1 && t < g.size && t != g.index) {
    const int peer = g.members[t];
    const int base = (channel * B200DP_MAX_BLOCKS + (int)blockIdx.x) * B200DP_MAX_RANKS;
    const uint32_t e = c.epoch[base + peer] + 1u;
    c.epoch[base + peer] = e;
    red_add_release_sys(c.sig[peer] + base + c.rank, 1u);
    if (!wait_for_peer(c, c.sig[c.rank] + base + peer, e, peer, channel)) s_failed = 1;
  }
  __syncthreads();
  return s_failed == 0;
}

// Who takes part in a collective: `rank()` of `size()` ranks, and their barrier.  The whole world, or a group whose
// data pointers are indexed by group rank.
struct WorldTeam {
  const CommCtx& c;
  __device__ __forceinline__ int rank() const { return c.rank; }
  __device__ __forceinline__ int size() const { return c.world; }
  __device__ __forceinline__ bool barrier(int channel) const { return rank_barrier(c, channel); }
};

struct GroupTeam {
  const CommCtx& c;
  const GroupCollArgs& g;
  __device__ __forceinline__ int rank() const { return g.index; }
  __device__ __forceinline__ int size() const { return g.size; }
  __device__ __forceinline__ bool barrier(int channel) const { return group_barrier(c, g, channel); }
};

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

// ------------------------------------------------------------------ shared kernel pieces
// Zero-on-consume tail of the grid-stride one-shot kernels, run after the closing barrier: every peer has read
// this thread's vectors of the local gradient bucket, so zero them, or, for an in-place one-shot, overwrite them
// with the result kept in `restore`.
__device__ __forceinline__ void release_input(const void* in, const uint4* restore, size_t start, size_t nvec,
                                              size_t stride) {
  uint4* mine = reinterpret_cast<uint4*>(const_cast<void*>(in));
  for (size_t v = start; v < nvec; v += stride) mine[v] = restore ? restore[v] : make_uint4(0, 0, 0, 0);
}

// ------------------------------------------------------------------ fp32 arenas (master, S0, S1, R)
template <int VN>
__device__ __forceinline__ void load_f32(const float* src, float* x) {
#pragma unroll
  for (int i = 0; i < VN; i += 4) {
    const float4 m = *reinterpret_cast<const float4*>(src + i);
    x[i] = m.x; x[i + 1] = m.y; x[i + 2] = m.z; x[i + 3] = m.w;
  }
}

template <int VN>
__device__ __forceinline__ void store_f32(float* dst, const float* x) {
#pragma unroll
  for (int i = 0; i < VN; i += 4)
    *reinterpret_cast<float4*>(dst + i) = make_float4(x[i], x[i + 1], x[i + 2], x[i + 3]);
}

// fp32 master values of VN elements from element `idx`: the master arena, or the fp32 result bucket itself.
// The master load is spelled out rather than taken from load_f32: through load_f32, nvcc 12.9 splits each
// 128-bit master load of the sliced kernels (K2/K3) into four 32-bit loads.
template <typename T, int VN>
__device__ __forceinline__ void load_master(const ARArgs& a, const T* out_local, size_t idx, float* p) {
  if (a.master) {
#pragma unroll
    for (int i = 0; i < VN; i += 4) {
      const float4 m = *reinterpret_cast<const float4*>(a.master + idx + i);
      p[i] = m.x; p[i + 1] = m.y; p[i + 2] = m.z; p[i + 3] = m.w;
    }
  } else {
    const uint4 v = *reinterpret_cast<const uint4*>(out_local + idx);
    Vec<T>::unpack(v, p);
  }
}

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

// Adam / LAMB bias corrections 1 - beta1^t and sqrt(1 - beta2^t) for step t (1-based), each rounded to fp32 once.
// They are formed in double: in fp32, 1 - beta^t cancels for beta near 1 and small t and magnifies the rounding of
// beta^t by beta^t / (1 - beta^t) (about 10^5 for beta2 = 0.99999), far beyond the rest of the update's error.
__device__ __forceinline__ void bias_corrections(float beta1, float beta2, int t, float* bc1, float* bc2_sqrt) {
  const double tf = (double)t;
  *bc1 = (float)(1.0 - pow((double)beta1, tf));
  *bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, tf));
}

__device__ __forceinline__ StepInfo make_step(const ARArgs& a) {
  StepInfo s;
  const int t = a.step_ctr ? *a.step_ctr : 0;
  s.first = (t == 0);
  s.lr = a.h.lr * (a.lr_scale ? *a.lr_scale : 1.0f);
  if (a.h.kind == OPT_ADAM) {
    bias_corrections(a.h.beta1, a.h.beta2, t + 1, &s.bc1, &s.bc2_sqrt);
  } else {
    s.bc1 = 1.0f;
    s.bc2_sqrt = 1.0f;
  }
  return s;
}

// Adam / LAMB update of the moments m and v of one element with gradient g (torch.optim semantics, non-amsgrad);
// returns the denominator sqrt(v^) + eps.  The callers form the update from it differently.
__device__ __forceinline__ float adam_moments(const OptHyper& h, float bc2_sqrt, float g, float& m, float& v) {
  m = fmaf(h.beta1, m, (1.0f - h.beta1) * g);      // lerp(m, g, 1-b1)
  v = fmaf(h.beta2, v, (1.0f - h.beta2) * g * g);
  return sqrtf(v) / bc2_sqrt + h.eps;
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
  load_master<T, VN>(a, out_local, idx, p);
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
        load_f32<VN>(a.s0 + idx, b);
#pragma unroll
        for (int i = 0; i < VN; ++i)
          b[i] = fmaf(a.h.momentum, b[i], (1.0f - a.h.dampening) * g[i]);
      }
      store_f32<VN>(a.s0 + idx, b);
#pragma unroll
      for (int i = 0; i < VN; ++i) g[i] = a.h.nesterov ? fmaf(a.h.momentum, b[i], g[i]) : b[i];
    }
#pragma unroll
    for (int i = 0; i < VN; ++i) p[i] = fmaf(-s.lr, g[i], p[i]);
  } else {  // Adam / AdamW
    float m[VN], v[VN];
    load_f32<VN>(a.s0 + idx, m);
    load_f32<VN>(a.s1 + idx, v);
#pragma unroll
    for (int i = 0; i < VN; ++i) {
      if (a.h.adamw) {
        p[i] *= (1.0f - s.lr * a.h.weight_decay);
      } else if (a.h.weight_decay != 0.0f) {
        g[i] = fmaf(a.h.weight_decay, p[i], g[i]);
      }
      const float denom = adam_moments(a.h, s.bc2_sqrt, g[i], m[i], v[i]);
      p[i] = fmaf(-(s.lr / s.bc1), m[i] / denom, p[i]);
    }
    store_f32<VN>(a.s0 + idx, m);
    store_f32<VN>(a.s1 + idx, v);
  }
  if (a.master) store_f32<VN>(a.master + idx, p);
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
  if (a.copy_back | a.zero_input)
    release_input(a.in[c.rank], a.copy_back ? reinterpret_cast<const uint4*>(a.scratch) : nullptr, start, nvec,
                  stride);
  finish_step(a);
}

// ------------------------------------------------------------------ K1c / K8 / K9: clip by global norm
// Fixed-shape block sum (warp butterfly, then warp 0 over the warp partials) of one value per thread: an fp32
// value, or a pair of fp32 or fp64 values.  The same inputs give the same bits on every rank and every run.
struct DoublePair {
  double x, y;
};
__device__ __forceinline__ float shfl_xor_add(float v, int o) { return v + __shfl_xor_sync(0xffffffffu, v, o); }
__device__ __forceinline__ float2 shfl_xor_add(float2 v, int o) {
  return make_float2(shfl_xor_add(v.x, o), shfl_xor_add(v.y, o));
}
__device__ __forceinline__ DoublePair shfl_xor_add(DoublePair v, int o) {
  return {v.x + __shfl_xor_sync(0xffffffffu, v.x, o), v.y + __shfl_xor_sync(0xffffffffu, v.y, o)};
}

template <typename V>
__device__ __forceinline__ V block_sum_fixed(V v) {
  __shared__ V s_part[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = shfl_xor_add(v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) s_part[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? s_part[lane] : V{};
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = shfl_xor_add(v, o);
  }
  return v;  // valid in thread 0; s_part is free again after the next __syncthreads()
}

// K1c: K1's reduction (same fixed rank order, same `scale * sum`), but the result goes to the fp32 arena
// `k.r` instead of through the optimizer epilogue, and each CTA stores the sum of squares of the values it
// wrote in slot `k.slots[blockIdx.x]`.  Every rank reduces the whole bucket, so every rank holds the same
// bits of `r` and of the slots, and hence computes the same norm.  Step counters are not touched.
template <typename T>
__global__ void __launch_bounds__(512) allreduce_oneshot_clip_kernel(CommCtx c, ARArgs a, ClipArgs k) {
  constexpr int VN = Vec<T>::N;
  const size_t nvec = a.n / VN;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;

  if (!rank_barrier(c, a.channel)) return;
  float sq = 0.0f;
  for (size_t v = start; v < nvec; v += stride) {
    uint4 raw[B200DP_MAX_RANKS];
#pragma unroll
    for (int r = 0; r < B200DP_MAX_RANKS; ++r)
      if (r < c.world) raw[r] = ld_peer_v4(reinterpret_cast<const uint4*>(a.in[r]) + v);
    float acc[VN], f[VN];
#pragma unroll
    for (int i = 0; i < VN; ++i) acc[i] = 0.0f;
#pragma unroll
    for (int r = 0; r < B200DP_MAX_RANKS; ++r) {
      if (r < c.world) {
        Vec<T>::unpack(raw[r], f);
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[i] += f[i];
      }
    }
#pragma unroll
    for (int i = 0; i < VN; ++i) {
      acc[i] *= a.scale;
      sq = fmaf(acc[i], acc[i], sq);
    }
    store_f32<VN>(k.r + v * VN, acc);
  }
  const float total = block_sum_fixed(sq);
  if (threadIdx.x == 0) k.slots[blockIdx.x] = total;  // a CTA without elements writes 0
  rank_barrier(c, a.channel);  // every peer has finished reading my gradients
  if (a.zero_input) release_input(a.in[c.rank], nullptr, start, nvec, stride);
}

// K8: one CTA.  Thread t adds slots t, t + blockDim, ... in double, then a fixed tree in shared memory
// combines the threads, so the order of every addition is fixed.  The coefficient follows
// torch.nn.utils.clip_grad_norm_ in fp32: (1 / (norm + 1e-6)) * max_norm, clamped to at most 1 (NaN stays NaN).
__global__ void __launch_bounds__(256) clip_finalize_kernel(ClipArgs k) {
  __shared__ double s[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < k.nslots; i += blockDim.x) acc += (double)k.slots[i];
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int w = blockDim.x >> 1; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float norm = (float)sqrt(s[0]);
    const float c = __frcp_rn(norm + 1e-6f) * k.max_norm;
    *k.norm = norm;
    *k.coef = c > 1.0f ? 1.0f : c;
  }
}

// K9: purely local.  g = r * coef, then the K7 epilogue with a.scale == 1 (the scale is already in r), so
// with coef == 1 the update is bit-identical to K1's.  Output and state are this rank's own copies.
template <typename T>
__global__ void __launch_bounds__(512) clip_apply_kernel(CommCtx c, ARArgs a, ClipArgs k) {
  constexpr int VN = Vec<T>::N;
  const size_t nvec = a.n / VN;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const StepInfo s = make_step(a);
  const float coef = *k.coef;
  T* out = reinterpret_cast<T*>(a.out[c.rank]);
  for (size_t v = start; v < nvec; v += stride) {
    float g[VN];
    load_f32<VN>(k.r + v * VN, g);
#pragma unroll
    for (int i = 0; i < VN; ++i) g[i] *= coef;
    float o[VN];
    epilogue<T, VN>(a, s, v * VN, g, out, o);
    reinterpret_cast<uint4*>(out)[v] = Vec<T>::pack(o);
  }
  finish_step(a);
}

// ------------------------------------------------------------------ K10 / K11: LARS / LAMB
// The zero-on-consume tail of K10 and K12, after their closing barrier: zero exactly the vectors this thread read
// in the chunk walk.  The CTA of the same index on every peer has read them too, while other CTAs may still be
// reading theirs.  Vectors outside every chunk (bucket padding) are never written, so they stay zero.
__device__ __forceinline__ void zero_chunks(const ChunkArgs& t, const void* in) {
  uint4* mine = reinterpret_cast<uint4*>(const_cast<void*>(in));
  for (int ch = blockIdx.x; ch < t.nchunks; ch += gridDim.x) {
    const LwChunk q = t.chunks[ch];
    for (int v = q.first_vec + (int)threadIdx.x; v < q.first_vec + q.nvec; v += blockDim.x)
      mine[v] = make_uint4(0, 0, 0, 0);
  }
}

// The fold of K11 and K13: the sums of a tensor's partials over chunks [first, first + count) in double (the
// second only if `both`), thread t adding partials t, t + blockDim, ... then a fixed shuffle / warp tree, so every
// CTA that needs them computes the same bits without waiting for another.  Valid in thread 0.
__device__ __forceinline__ DoublePair fold_partials(const float* part, int first, int count, bool both) {
  DoublePair acc = {0.0, 0.0};
  for (int i = threadIdx.x; i < count; i += blockDim.x) {
    acc.x += (double)part[2 * (first + i)];
    if (both) acc.y += (double)part[2 * (first + i) + 1];
  }
  return block_sum_fixed(acc);
}

// K10: K1's reduction (same fixed rank order, same `scale * sum`), then the update direction into `k.r`
// (LAMB also updates exp_avg / exp_avg_sq in s0 / s1) and, per chunk, the fp32 sums of squares of the master
// weights and of the direction.  CTAs walk whole chunks, so every partial covers one tensor only and is added
// in a fixed order; every rank reduces the whole bucket and holds the same bits.  Step counters are read
// (LAMB bias correction), not bumped.
template <typename T>
__global__ void __launch_bounds__(512) allreduce_oneshot_lw_kernel(CommCtx c, ARArgs a, LwArgs k) {
  constexpr int VN = Vec<T>::N;
  const T* out_local = reinterpret_cast<const T*>(a.out[c.rank]);
  const bool lamb = a.h.kind == OPT_LAMB;
  float bc1 = 1.0f, bc2_sqrt = 1.0f;
  if (lamb) bias_corrections(a.h.beta1, a.h.beta2, (a.step_ctr ? *a.step_ctr : 0) + 1, &bc1, &bc2_sqrt);

  if (!rank_barrier(c, a.channel)) return;
  for (int ch = blockIdx.x; ch < k.tab.nchunks; ch += gridDim.x) {
    const LwChunk q = k.tab.chunks[ch];
    float ww = 0.0f, dd = 0.0f;
    for (int v = q.first_vec + (int)threadIdx.x; v < q.first_vec + q.nvec; v += blockDim.x) {
      uint4 raw[B200DP_MAX_RANKS];
#pragma unroll
      for (int r = 0; r < B200DP_MAX_RANKS; ++r)
        if (r < c.world) raw[r] = ld_peer_v4(reinterpret_cast<const uint4*>(a.in[r]) + v);
      float g[VN], f[VN], p[VN];
#pragma unroll
      for (int i = 0; i < VN; ++i) g[i] = 0.0f;
#pragma unroll
      for (int r = 0; r < B200DP_MAX_RANKS; ++r) {
        if (r < c.world) {
          Vec<T>::unpack(raw[r], f);
#pragma unroll
          for (int i = 0; i < VN; ++i) g[i] += f[i];
        }
      }
      const size_t idx = (size_t)v * VN;
      load_master<T, VN>(a, out_local, idx, p);
#pragma unroll
      for (int i = 0; i < VN; ++i) g[i] *= a.scale;
      if (lamb) {
#pragma unroll
        for (int i = 0; i < VN; i += 4) {
          float m[4], s[4];
          load_f32<4>(a.s0 + idx + i, m);
          load_f32<4>(a.s1 + idx + i, s);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float denom = adam_moments(a.h, bc2_sqrt, g[i + j], m[j], s[j]);
            g[i + j] = fmaf(a.h.weight_decay, p[i + j], (m[j] / bc1) / denom);
          }
          store_f32<4>(a.s0 + idx + i, m);
          store_f32<4>(a.s1 + idx + i, s);
        }
      } else {
#pragma unroll
        for (int i = 0; i < VN; ++i) g[i] = fmaf(a.h.weight_decay, p[i], g[i]);
      }
#pragma unroll
      for (int i = 0; i < VN; ++i) {
        ww = fmaf(p[i], p[i], ww);
        dd = fmaf(g[i], g[i], dd);
      }
      store_f32<VN>(k.tab.r + idx, g);
    }
    const float2 s = block_sum_fixed(make_float2(ww, dd));
    __syncthreads();  // the next chunk's sum reuses the block sum's shared memory
    if (threadIdx.x == 0) {
      k.tab.part[2 * ch] = s.x;
      k.tab.part[2 * ch + 1] = s.y;
    }
  }
  rank_barrier(c, a.channel);
  if (a.zero_input) zero_chunks(k.tab, a.in[c.rank]);
}

// Trust ratio of the tensor whose partials are chunks [first, first + count), computed by thread 0 from
// fold_partials and broadcast to the CTA.  1 when the group is not adaptive or either norm is not > 0.
__device__ float lw_trust(const LwArgs& k, int first, int count) {
  __shared__ float s_ratio;
  const DoublePair wd = fold_partials(k.tab.part, first, count, true);
  if (threadIdx.x == 0) {
    const double wn = sqrt(wd.x), dn = sqrt(wd.y);
    s_ratio = (k.adaptive && wn > 0.0 && dn > 0.0) ? (float)((double)k.trust_coef * wn / dn) : 1.0f;
  }
  __syncthreads();
  return s_ratio;
}

// K11: purely local.  LARS: buf = momentum * buf + (lr * trust) * r, w -= buf.  LAMB: w -= (lr * trust) * r.
// Writes master, output and LARS state, then bumps the step counter.  A CTA recomputes the ratio only when its
// next chunk belongs to another tensor.
template <typename T>
__global__ void __launch_bounds__(512) lw_apply_kernel(CommCtx c, ARArgs a, LwArgs k) {
  constexpr int VN = Vec<T>::N;
  const float lr = a.h.lr * (a.lr_scale ? *a.lr_scale : 1.0f);
  const bool lamb = a.h.kind == OPT_LAMB;
  T* out = reinterpret_cast<T*>(a.out[c.rank]);
  int tensor = -1;
  float trust = 1.0f;
  for (int ch = blockIdx.x; ch < k.tab.nchunks; ch += gridDim.x) {
    const LwChunk q = k.tab.chunks[ch];
    if (q.tfirst != tensor) {
      tensor = q.tfirst;
      trust = lw_trust(k, q.tfirst, q.tcount);
      if (ch == q.tfirst && threadIdx.x == 0) k.ratio[ch] = trust;
    }
    const float step = lr * trust;
    for (int v = q.first_vec + (int)threadIdx.x; v < q.first_vec + q.nvec; v += blockDim.x) {
      const size_t idx = (size_t)v * VN;
      float d[VN], p[VN];
      load_f32<VN>(k.tab.r + idx, d);
      load_master<T, VN>(a, out, idx, p);
      if (lamb) {
#pragma unroll
        for (int i = 0; i < VN; ++i) p[i] = fmaf(-step, d[i], p[i]);
      } else {
        float b[VN];
        load_f32<VN>(a.s0 + idx, b);
#pragma unroll
        for (int i = 0; i < VN; ++i) {
          b[i] = fmaf(a.h.momentum, b[i], step * d[i]);
          p[i] -= b[i];
        }
        store_f32<VN>(a.s0 + idx, b);
      }
      if (a.master) store_f32<VN>(a.master + idx, p);
      reinterpret_cast<uint4*>(out)[v] = Vec<T>::pack(p);
    }
  }
  finish_step(a);
}

// ------------------------------------------------------------------ K12 / K13 / K14: Muon
// torch.lerp's formula: s + w (e - s) for |w| < 0.5, else e - (e - s)(1 - w).
__device__ __forceinline__ float lerp_torch(float s, float e, float w) {
  return fabsf(w) < 0.5f ? fmaf(w, e - s, s) : fmaf(-(e - s), 1.0f - w, e);
}

// K12: K1's reduction (same fixed rank order, same `scale * sum`), then buf.lerp_(g, 1 - momentum) into s0, u into
// `k.r` and, per chunk, the fp32 sum of squares of u.  CTAs walk whole chunks as K10 does, so every rank holds the
// same bits of u and of the partials.  Step counters are not touched.
template <typename T>
__global__ void __launch_bounds__(512) allreduce_oneshot_muon_kernel(CommCtx c, ARArgs a, MuonArgs k) {
  constexpr int VN = Vec<T>::N;
  const float mu = a.h.momentum, w = a.h.dampening;  // dampening carries Muon's lerp weight 1 - momentum

  if (!rank_barrier(c, a.channel)) return;
  for (int ch = blockIdx.x; ch < k.tab.nchunks; ch += gridDim.x) {
    const LwChunk q = k.tab.chunks[ch];
    float uu = 0.0f;
    for (int v = q.first_vec + (int)threadIdx.x; v < q.first_vec + q.nvec; v += blockDim.x) {
      uint4 raw[B200DP_MAX_RANKS];
#pragma unroll
      for (int r = 0; r < B200DP_MAX_RANKS; ++r)
        if (r < c.world) raw[r] = ld_peer_v4(reinterpret_cast<const uint4*>(a.in[r]) + v);
      float g[VN], f[VN], b[VN];
#pragma unroll
      for (int i = 0; i < VN; ++i) g[i] = 0.0f;
#pragma unroll
      for (int r = 0; r < B200DP_MAX_RANKS; ++r) {
        if (r < c.world) {
          Vec<T>::unpack(raw[r], f);
#pragma unroll
          for (int i = 0; i < VN; ++i) g[i] += f[i];
        }
      }
      const size_t idx = (size_t)v * VN;
      load_f32<VN>(a.s0 + idx, b);
#pragma unroll
      for (int i = 0; i < VN; ++i) {
        g[i] = __fmul_rn(g[i], a.scale);  // rounded, as K1's scale * sum: never contracted into the lerp's e - s
        b[i] = lerp_torch(b[i], g[i], w);
        g[i] = k.nesterov ? lerp_torch(g[i], b[i], mu) : b[i];
        uu = fmaf(g[i], g[i], uu);
      }
      store_f32<VN>(a.s0 + idx, b);
      store_f32<VN>(k.tab.r + idx, g);
    }
    const float s = block_sum_fixed(uu);
    __syncthreads();  // the next chunk's sum reuses the block sum's shared memory
    if (threadIdx.x == 0) {
      k.tab.part[2 * ch] = s;
      k.tab.part[2 * ch + 1] = 0.0f;
    }
  }
  rank_barrier(c, a.channel);
  if (a.zero_input) zero_chunks(k.tab, a.in[c.rank]);
}

// max(norm, eps) of the matrix whose partials are chunks [first, first + count), from fold_partials (the first
// sums only: K12 writes 0 to the second), rounded to fp32 once by thread 0 and broadcast to the CTA.
__device__ float muon_norm(const MuonArgs& k, int first, int count) {
  __shared__ float s_norm;
  const DoublePair acc = fold_partials(k.tab.part, first, count, false);
  if (threadIdx.x == 0) {
    const float n = (float)sqrt(acc.x);
    s_norm = n > k.eps ? n : k.eps;
  }
  __syncthreads();
  return s_norm;
}

// Position of element e (row-major in the [rows, cols] parameter) in its NS operand: the same place, or for a tall
// matrix (rows > cols) the transposed one.
__device__ __forceinline__ int muon_pos(const MuonMat& m, int e) {
  return m.rows > m.cols ? (e % m.cols) * m.rows + e / m.cols : e;
}

// K13: purely local.  X0 = bf16(u / max(norm, eps)) for every element of every matrix of the bucket.  Elements past
// a matrix's end (the padding of its last vector) are skipped.
template <typename T>
__global__ void __launch_bounds__(512) muon_normalize_kernel(MuonArgs k) {
  constexpr int VN = Vec<T>::N;
  int tensor = -1;
  float nrm = 1.0f;
  for (int ch = blockIdx.x; ch < k.tab.nchunks; ch += gridDim.x) {
    const LwChunk q = k.tab.chunks[ch];
    const MuonMat m = k.mats[ch];
    if (q.tfirst != tensor) {
      tensor = q.tfirst;
      nrm = muon_norm(k, q.tfirst, q.tcount);
    }
    const int numel = m.rows * m.cols;
    for (int v = q.first_vec + (int)threadIdx.x; v < q.first_vec + q.nvec; v += blockDim.x) {
      float u[VN];
      load_f32<VN>(k.tab.r + (size_t)v * VN, u);
#pragma unroll
      for (int i = 0; i < VN; ++i) {
        const int e = v * VN + i - m.elem0;
        if (e < numel) k.x0[m.x0 + muon_pos(m, e)] = __float2bfloat16_rn(__fdiv_rn(u[i], nrm));
      }
    }
  }
}

// K14: purely local.  w = w (1 - lr wd) - (lr f) O on the fp32 master, with lr = h.lr * lr_scale and O read back in
// the parameter's orientation; writes master and output, then bumps the step counter.
template <typename T>
__global__ void __launch_bounds__(512) muon_apply_kernel(CommCtx c, ARArgs a, MuonArgs k) {
  constexpr int VN = Vec<T>::N;
  const float lr = a.h.lr * (a.lr_scale ? *a.lr_scale : 1.0f);
  const float decay = 1.0f - lr * a.h.weight_decay;
  T* out = reinterpret_cast<T*>(a.out[c.rank]);
  for (int ch = blockIdx.x; ch < k.tab.nchunks; ch += gridDim.x) {
    const LwChunk q = k.tab.chunks[ch];
    const MuonMat m = k.mats[ch];
    const double f = k.lr_mode ? 0.2 * sqrt((double)max(m.rows, m.cols))
                               : sqrt(fmax(1.0, (double)m.rows / (double)m.cols));
    const float step = (float)((double)lr * f);
    const int numel = m.rows * m.cols;
    for (int v = q.first_vec + (int)threadIdx.x; v < q.first_vec + q.nvec; v += blockDim.x) {
      const size_t idx = (size_t)v * VN;
      float p[VN];
      load_master<T, VN>(a, out, idx, p);
#pragma unroll
      for (int i = 0; i < VN; ++i) {
        const int e = (int)idx + i - m.elem0;
        if (e < numel) p[i] = fmaf(-step, __bfloat162float(k.o[m.x0 + muon_pos(m, e)]), p[i] * decay);
      }
      if (a.master) store_f32<VN>(a.master + idx, p);
      reinterpret_cast<uint4*>(out)[v] = Vec<T>::pack(p);
    }
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
template <typename T, bool kNVLS, typename Team>
__device__ __forceinline__ void reducescatter_body(const Team& m, const CollArgs& a) {
  constexpr int VN = Vec<T>::N;
  const size_t nvec = a.chunk / VN;
  const size_t base = (size_t)m.rank() * nvec;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint4* out = reinterpret_cast<uint4*>(a.dst[m.rank()]);
  if (!m.barrier(a.channel)) return;
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
          if (r < m.size() && v < nvec) raw[u][r] = ld_peer_v4(reinterpret_cast<const uint4*>(a.src[r]) + base + v);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float f[VN];
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[u][i] = 0.0f;
#pragma unroll
        for (int r = 0; r < B200DP_MAX_RANKS; ++r) {   // fixed rank order
          if (r < m.size()) {
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
  m.barrier(a.channel);   // peers have finished reading my input
}

template <typename T, bool kNVLS>
__global__ void __launch_bounds__(512) reducescatter_kernel(CommCtx c, CollArgs a) {
  reducescatter_body<T, kNVLS>(WorldTeam{c}, a);
}

template <typename T>
__global__ void __launch_bounds__(512) reducescatter_group_kernel(CommCtx c, GroupCollArgs a) {
  reducescatter_body<T, false>(GroupTeam{c, a}, a.coll);
}

// kMC: multicast when the argument block asks for it (world only).
template <bool kMC, typename Team>
__device__ __forceinline__ void allgather_body(const Team& m, const CollArgs& a) {
  const size_t nvec = a.chunk;   // chunk is given in 16-byte vectors for the copy collectives
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(a.src[m.rank()]);
  const size_t slot = (size_t)m.rank() * nvec;
  if (!m.barrier(a.channel)) return;   // every rank's output is free to overwrite
  for (size_t v = start; v < nvec; v += stride) {
    const uint4 x = src[v];
    if (kMC && a.use_mc) {
      mc_st_v4(reinterpret_cast<uint4*>(a.dst_mc) + slot + v, x);
    } else {
#pragma unroll
      for (int r = 0; r < B200DP_MAX_RANKS; ++r)
        if (r < m.size()) st_peer_v4(reinterpret_cast<uint4*>(a.dst[r]) + slot + v, x);
    }
  }
  m.barrier(a.channel);   // all pushes visible everywhere
}

__global__ void __launch_bounds__(512) allgather_kernel(CommCtx c, CollArgs a) {
  allgather_body<true>(WorldTeam{c}, a);
}

__global__ void __launch_bounds__(512) allgather_group_kernel(CommCtx c, GroupCollArgs a) {
  allgather_body<false>(GroupTeam{c, a}, a.coll);
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

// ------------------------------------------------------------------ host launch helpers
template <typename T>
struct TypeTag {
  using type = T;
};

// Calls f(TypeTag<T>{}) with the element type of a dtype code (0 fp32, 1 bf16, 2 fp16).
template <typename F>
cudaError_t with_dtype(int dtype, F&& f) {
  switch (dtype) {
    case 0: return f(TypeTag<float>{});
    case 1: return f(TypeTag<__nv_bfloat16>{});
    case 2: return f(TypeTag<__half>{});
  }
  return cudaErrorInvalidValue;
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

// The launch checks of every entry point.  The grid must fit the per-block barrier counters and slots
// (1..B200DP_MAX_BLOCKS CTAs) and be whole warps of at most 512 threads (the block sums and __launch_bounds__);
// the world and the channel must fit the signal pad, and the rank must lie in the world (it indexes `sig[]`);
// `sel` (algorithm, phase or collective mode) must be below `nsel` and the dtype code known.  Sets the error
// message and returns false otherwise.
static bool launch_ok(const char* what, const CommCtx* ctx, int channel, const char* sel_name, int sel, int nsel,
                      int dtype, int blocks, int threads) {
  if (blocks >= 1 && blocks <= B200DP_MAX_BLOCKS && threads >= 32 && threads <= 512 && (threads & 31) == 0 &&
      ctx->world >= 1 && ctx->world <= B200DP_MAX_RANKS && ctx->rank >= 0 && ctx->rank < ctx->world &&
      channel >= 0 && channel < B200DP_NUM_CHANNELS && sel >= 0 && sel < nsel && dtype >= 0 && dtype <= 2)
    return true;
  snprintf(g_comm_err, sizeof(g_comm_err),
           "bad %s launch: blocks=%d threads=%d rank=%d world=%d channel=%d %s=%d dtype=%d", what, blocks, threads,
           ctx->rank, ctx->world, channel, sel_name, sel, dtype);
  return false;
}

// The kernels walk whole 16-byte vectors (`size / unit`) and would silently drop a tail: a size that is not a
// multiple of `unit` is refused.  Sets the error message and returns false then.
static bool size_ok(const char* what, const char* size_name, unsigned long long size, unsigned long long unit) {
  if (size % unit == 0) return true;
  snprintf(g_comm_err, sizeof(g_comm_err), "bad %s launch: %s=%llu is not a multiple of %llu", what, size_name,
           size, unit);
  return false;
}

// The chunked entry points (LARS / LAMB, Muon) walk the chunk table, not `n`: the optimizer kind must be one of
// the entry point's (`kind_ok`) and the chunk count not negative.  Sets the error message and returns false otherwise.
static bool chunks_ok(const char* what, bool kind_ok, int kind, const ChunkArgs& t) {
  if (kind_ok && t.nchunks >= 0) return true;
  snprintf(g_comm_err, sizeof(g_comm_err), "bad %s launch: kind=%d chunks=%d", what, kind, t.nchunks);
  return false;
}

// Elements of a dtype code per 16-byte vector.
static unsigned long long vec_elems(int dtype) { return dtype == 0 ? 4 : 8; }

// 0, or -1 with the launch error in b200dp_comm_last_error().
static int launched(const char* what, cudaError_t e) {
  if (e == cudaSuccess) return 0;
  snprintf(g_comm_err, sizeof(g_comm_err), "%s launch: %s", what, cudaGetErrorString(e));
  return -1;
}

int b200dp_comm_clip_bytes() { return (int)sizeof(ClipArgs); }

// phase: 0 reduce into k.r + norm slots (K1c), 1 clip + optimizer update from k.r (K9).  dtype as in
// b200dp_comm_allreduce: the dtype of the gradient bucket on the wire and of the parameter output.
int b200dp_comm_clip_bucket(const CommCtx* ctx, const ARArgs* args, const ClipArgs* clip, int phase, int dtype,
                            int blocks, int threads, unsigned long long stream) {
  if (!launch_ok("clip", ctx, args->channel, "phase", phase, 2, dtype, blocks, threads) ||
      !size_ok("clip", "n", args->n, vec_elems(dtype)))
    return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  return launched("clip", with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if (phase == 1) clip_apply_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args, *clip);
    else allreduce_oneshot_clip_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args, *clip);
    return cudaGetLastError();
  }));
}

int b200dp_comm_clip_finalize(const ClipArgs* clip, unsigned long long stream) {
  clip_finalize_kernel<<<1, 256, 0, (cudaStream_t)(uintptr_t)stream>>>(*clip);
  return launched("clip finalize", cudaGetLastError());
}

int b200dp_comm_lw_bytes() { return (int)sizeof(LwArgs); }

// phase: 0 reduce + direction + chunk partials (K10), 1 trust ratios + update + step counter (K11).
// args->h.kind selects LARS or LAMB.  dtype as in b200dp_comm_allreduce.
int b200dp_comm_lw_bucket(const CommCtx* ctx, const ARArgs* args, const LwArgs* lw, int phase, int dtype,
                          int blocks, int threads, unsigned long long stream) {
  if (!launch_ok("layer-wise", ctx, args->channel, "phase", phase, 2, dtype, blocks, threads) ||
      !chunks_ok("layer-wise", args->h.kind == OPT_LARS || args->h.kind == OPT_LAMB, args->h.kind, lw->tab))
    return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  return launched("layer-wise", with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if (phase == 1) lw_apply_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args, *lw);
    else allreduce_oneshot_lw_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args, *lw);
    return cudaGetLastError();
  }));
}

int b200dp_comm_muon_bytes() { return (int)sizeof(MuonArgs); }

// phase: 0 reduce + momentum + u + chunk partials (K12), 1 norms + X0 (K13), 2 decay + NS result + step counter
// (K14).  args->h.kind must be OPT_MUON; dtype as in b200dp_comm_allreduce.
int b200dp_comm_muon_bucket(const CommCtx* ctx, const ARArgs* args, const MuonArgs* mu, int phase, int dtype,
                            int blocks, int threads, unsigned long long stream) {
  if (!launch_ok("muon", ctx, args->channel, "phase", phase, 3, dtype, blocks, threads) ||
      !chunks_ok("muon", args->h.kind == OPT_MUON, args->h.kind, mu->tab))
    return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  return launched("muon", with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if (phase == 0) allreduce_oneshot_muon_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args, *mu);
    else if (phase == 1) muon_normalize_kernel<T><<<blocks, threads, 0, st>>>(*mu);
    else muon_apply_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args, *mu);
    return cudaGetLastError();
  }));
}

// algo: 0 one-shot, 1 two-shot, 2 NVLS.  dtype: 0 fp32, 1 bf16, 2 fp16.
int b200dp_comm_allreduce(const CommCtx* ctx, const ARArgs* args, int algo, int dtype, int blocks,
                          int threads, unsigned long long stream) {
  if (!launch_ok("allreduce", ctx, args->channel, "algo", algo, 3, dtype, blocks, threads) ||
      !size_ok("allreduce", "n", args->n, vec_elems(dtype)))
    return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  return launched("allreduce", with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if (algo == 0) allreduce_oneshot_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args);
    else if (algo == 1) allreduce_sliced_kernel<T, false><<<blocks, threads, 0, st>>>(*ctx, *args);
    else allreduce_sliced_kernel<T, true><<<blocks, threads, 0, st>>>(*ctx, *args);
    return cudaGetLastError();
  }));
}

// mode: 0 reduce-scatter, 1 all-gather, 2 all-to-all.  dtype as in b200dp_comm_allreduce (reduce-scatter only).
int b200dp_comm_collective(const CommCtx* ctx, const CollArgs* args, int mode, int dtype, int blocks, int threads,
                           unsigned long long stream) {
  if (!launch_ok("collective", ctx, args->channel, "mode", mode, 3, dtype, blocks, threads) ||
      (mode == 0 && !size_ok("collective", "chunk", args->chunk, vec_elems(dtype))))
    return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  if (mode == 1) {
    allgather_kernel<<<blocks, threads, 0, st>>>(*ctx, *args);
  } else if (mode == 2) {
    alltoall_kernel<<<blocks, threads, 0, st>>>(*ctx, *args);
  } else {
    return launched("reduce-scatter", with_dtype(dtype, [&](auto tag) {
      using T = typename decltype(tag)::type;
      if (args->use_mc) reducescatter_kernel<T, true><<<blocks, threads, 0, st>>>(*ctx, *args);
      else reducescatter_kernel<T, false><<<blocks, threads, 0, st>>>(*ctx, *args);
      return cudaGetLastError();
    }));
  }
  return launched("collective", cudaGetLastError());
}

int b200dp_comm_coll_bytes() { return (int)sizeof(CollArgs); }

int b200dp_comm_group_coll_bytes() { return (int)sizeof(GroupCollArgs); }

// The member list of a group launch: 1..B200DP_MAX_RANKS world ranks, strictly ascending (sorted, no duplicates),
// inside the world, with the caller at `index`; no multicast.  Sets the error message and returns false otherwise.
static bool group_ok(const CommCtx* ctx, const GroupCollArgs* g) {
  const char* why = nullptr;
  if (g->size < 1 || g->size > B200DP_MAX_RANKS) {
    why = "size";
  } else if (g->index < 0 || g->index >= g->size || g->members[g->index] != ctx->rank) {
    why = "the caller is not members[index]";
  } else if (g->coll.use_mc) {
    why = "multicast";
  } else {
    for (int i = 0; i < g->size && !why; ++i) {
      if (g->members[i] < 0 || g->members[i] >= ctx->world) why = "a member outside the world";
      else if (i > 0 && g->members[i] <= g->members[i - 1]) why = "members not strictly ascending";
    }
  }
  if (!why) return true;
  snprintf(g_comm_err, sizeof(g_comm_err), "bad group collective launch: %s (size=%d index=%d rank=%d world=%d)",
           why, g->size, g->index, ctx->rank, ctx->world);
  return false;
}

// mode: 0 reduce-scatter, 1 all-gather, among the members of `args` (the world collectives' layouts, indexed by
// group rank).  dtype as in b200dp_comm_collective.
int b200dp_comm_group_collective(const CommCtx* ctx, const GroupCollArgs* args, int mode, int dtype, int blocks,
                                 int threads, unsigned long long stream) {
  if (!launch_ok("group collective", ctx, args->coll.channel, "mode", mode, 2, dtype, blocks, threads) ||
      !group_ok(ctx, args) ||
      (mode == 0 && !size_ok("group collective", "chunk", args->coll.chunk, vec_elems(dtype))))
    return -1;
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  if (mode == 1) {
    allgather_group_kernel<<<blocks, threads, 0, st>>>(*ctx, *args);
    return launched("group all-gather", cudaGetLastError());
  }
  return launched("group reduce-scatter", with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    reducescatter_group_kernel<T><<<blocks, threads, 0, st>>>(*ctx, *args);
    return cudaGetLastError();
  }));
}

int b200dp_comm_broadcast(const CommCtx* ctx, const BcastArgs* args, int blocks, int threads,
                          unsigned long long stream) {
  if (!launch_ok("broadcast", ctx, args->channel, "-", 0, 1, 0, blocks, threads) ||
      !size_ok("broadcast", "nbytes", args->nbytes, 16))
    return -1;
  broadcast_kernel<<<blocks, threads, 0, (cudaStream_t)(uintptr_t)stream>>>(*ctx, *args);
  return launched("broadcast", cudaGetLastError());
}

}  // extern "C"

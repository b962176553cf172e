// Implicit-GEMM convolution for sm_90a (NHWC bf16): forward, data gradient and weight gradient of
// 3x3 (stride 1/2, pad 1) and 1x1 (stride 1/2) convolutions on the wgmma mainloop of gemm_sm90.cu.
//
// No im2col matrix is ever materialised.  An NHWC activation is a 4D tensor {C, W, H, N} for the TMA
// unit; the 128 rows of a GEMM M-tile are a {bw, bh, bn} box of output pixels, and the A operand of
// filter tap (r, s) is the SAME box shifted by (s - pad, r - pad) — one cp.async.bulk.tensor.4d per
// tap and 64-channel chunk, with the zero padding produced by the TMA's out-of-bounds fill.  The smem
// image of such a box is exactly the K-major [128 rows][64 k] 128B-swizzled tile the GMMA descriptors
// of the GEMM expect, so the wgmma mainloop and the epilogue are shared with the GEMM.
//
//   fprop  y[p, co]  = sum_{r,s,ci} x[p + (r,s) - pad, ci] * w[co, r, s, ci]      A = x boxes, B = w (K-major)
//   dgrad  dx[p, ci] = sum_{r,s,co} dy[p + pad - (r,s), co] * w[co, r, s, ci]     A = dy boxes, B = w (MN-major)
//   wgrad  dw[co, r, s, ci] = sum_p dy[p, co] * x[p + (r,s) - pad, ci]            A = dy boxes, B = x boxes,
//          both MN-major with K = 64-pixel boxes; split-K over pixels, the partials summed in split order
//          and written to the [Cout][R*S*Cin] weight gradient in its dtype (splitk_finish_tile)
//
// Stride 2 never uses strided gathers: the input (fprop/wgrad) or the output (dgrad) is addressed
// through four parity views {C, W/2, H/2, N} (base offset (ph*W + pw)*C, doubled pitches), so every
// tap is again a dense shifted box of one view; dgrad runs the four output parities as "classes"
// with 1, 2, 2 and 4 taps.  Weights are [Cout][R][S][Cin] (PyTorch channels_last), which is the
// K-major B matrix of fprop and the MN-major B matrix of dgrad without any repacking.
//
// Replaces the cuDNN convolution calls of the ResNet zoo.  The reference application has no convolution
// at all (its whole model is one LSTM).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "sm90_common.cuh"

namespace {

constexpr int MAX_TAPS = 9;
constexpr int MAX_CLASSES = 4;

struct ConvTap {
  int amap;      // which activation view (parity) the tap reads
  int dw, dh;    // box shift in that view
  int wcol;      // fprop/dgrad: column of the [Cout][R*S*Cin] weight matrix; wgrad: output column
};
struct ConvClass {
  int ntaps;
  int out_map;   // which output view (dgrad stride 2: parity of dx)
  ConvTap taps[MAX_TAPS];
};
struct ConvParams {
  GemmParams g;
  int num_classes;
  int kc_per_tap;                 // 64-channel chunks of the reduction dimension per tap (fprop/dgrad)
  int bw, bh, bn;                 // pixel box: 128 rows of an M tile (fprop/dgrad) / 64 rows of a K block (wgrad)
  int sw, sh;                     // fprop/dgrad: {sw, sh, .} pixel box of one 32-row slab of the M tile
  int tiles_w, tiles_h, tiles_n;  // boxes covering the (class) output pixel space
  int num_taps_total;             // wgrad: R*S
  int out_w, out_h, out_n;        // extent of the (class) output pixel space: rows beyond it are clipped / not counted
  ConvClass cls[MAX_CLASSES];
};
struct alignas(64) ConvMaps {
  CUtensorMap a[4];     // activation views read with tap shifts (x for fprop/wgrad, dy for dgrad)
  CUtensorMap b;        // 2D weight matrix (fprop/dgrad); unused by wgrad
  CUtensorMap out[4];   // fprop/dgrad: output views (32-row slab boxes); wgrad: out[0] = dy (64-pixel boxes)
};

enum { MODE_FPROP = 0, MODE_DGRAD = 1, MODE_WGRAD = 2 };

// fprop/dgrad: work = class x pixel tile x n block (n fastest: the A boxes of one pixel tile are re-used from
// L2 by the CTAs working on its other n blocks); K blocks = taps x channel chunks.
// wgrad: work = split x (m block x n block x tap), tap fastest: the dy / x boxes of one pixel range are shared
// through L2 by the CTAs of the same split; K blocks = 64-pixel boxes.
template <int BN, int MODE>
struct ConvWork {
  static constexpr bool kStats = MODE == MODE_FPROP, kSplitK = MODE == MODE_WGRAD;
  static constexpr bool B_MN = MODE != MODE_FPROP;
  const ConvMaps& maps;
  const ConvParams& p;
  int nnb, pix_tiles, tiles, items, kb_per_split;

  __device__ ConvWork(const ConvMaps& maps_, const ConvParams& p_)
      : maps(maps_), p(p_), nnb(p_.g.num_n_blocks), pix_tiles(p_.tiles_w * p_.tiles_h * p_.tiles_n),
        tiles(MODE == MODE_WGRAD ? p_.g.num_m_blocks * nnb * p_.num_taps_total : p_.num_classes * pix_tiles * nnb),
        items(tiles * p_.g.splits),
        kb_per_split(MODE == MODE_WGRAD ? (pix_tiles + p_.g.splits - 1) / p_.g.splits : 0) {}
  __device__ void prefetch() const {
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&maps.a[i]);
    tma_prefetch_desc(&maps.b);
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&maps.out[i]);
  }
  __device__ int num_kb(int w) const {
    if (MODE != MODE_WGRAD) return p.cls[(w / nnb) / pix_tiles].ntaps * p.kc_per_tap;
    const int kb0 = (w / tiles) * kb_per_split;
    return min(kb0 + kb_per_split, pix_tiles) - kb0;
  }
  template <class Next>
  __device__ void load(int w, Next& next) const {
    if (MODE != MODE_WGRAD) {
      const int nt = w % nnb;
      const int rest = w / nnb;
      const int mt = rest % pix_tiles;
      const ConvClass& cl = p.cls[rest / pix_tiles];
      const int w0 = (mt % p.tiles_w) * p.bw;
      const int h0 = ((mt / p.tiles_w) % p.tiles_h) * p.bh;
      const int n0 = (mt / (p.tiles_w * p.tiles_h)) * p.bn;
      const int n_idx = nt * BN;
      for (int t = 0; t < cl.ntaps; ++t) {
        const ConvTap tap = cl.taps[t];
        for (int kc = 0; kc < p.kc_per_tap; ++kc) {
          const Stage s = next();
          tma_load_4d(&maps.a[tap.amap], s.bar, s.a, kc * BLOCK_K, w0 + tap.dw, h0 + tap.dh, n0);
          if (!B_MN) {
            tma_load_2d(&maps.b, s.bar, s.b, tap.wcol + kc * BLOCK_K, n_idx);   // box {64 k, BN co}
          } else {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)                                  // box {64 ci, 64 co}
              tma_load_2d(&maps.b, s.bar, s.b + c * (BLOCK_K * 128), tap.wcol + n_idx + 64 * c, kc * BLOCK_K);
          }
        }
      }
    } else {
      const int tile = w % tiles, split = w / tiles;
      const ConvTap tap = p.cls[0].taps[tile % p.num_taps_total];
      const int mn = tile / p.num_taps_total;
      const int m_idx = (mn / nnb) * BLOCK_M;
      const int n_idx = (mn % nnb) * BN;
      const int kb0 = split * kb_per_split;
      const int kb1 = min(kb0 + kb_per_split, pix_tiles);
      for (int kb = kb0; kb < kb1; ++kb) {
        const int w0 = (kb % p.tiles_w) * p.bw;
        const int h0 = ((kb / p.tiles_w) % p.tiles_h) * p.bh;
        const int n0 = (kb / (p.tiles_w * p.tiles_h)) * p.bn;
        const Stage s = next();
#pragma unroll
        for (int c = 0; c < BLOCK_M / 64; ++c)      // dy: 64 pixels x 64 output channels per box
          tma_load_4d(&maps.out[0], s.bar, s.a + c * (BLOCK_K * 128), m_idx + 64 * c, w0, h0, n0);
#pragma unroll
        for (int c = 0; c < BN / 64; ++c)           // x : the same pixels shifted by the tap
          tma_load_4d(&maps.a[tap.amap], s.bar, s.b + c * (BLOCK_K * 128), n_idx + 64 * c, w0 + tap.dw,
                      h0 + tap.dh, n0);
      }
    }
  }
  __device__ Slab slab(int w, int q) const {
    if (MODE != MODE_WGRAD) {
      const int nt = w % nnb;
      const int rest = w / nnb;
      const int mt = rest % pix_tiles;
      const int r0 = q * 32;                                   // first row of this warp's slab in the box
      StoreAt at;
      at.rank4 = 1;
      at.w = (mt % p.tiles_w) * p.bw + (r0 % p.bw);
      at.h = ((mt / p.tiles_w) % p.tiles_h) * p.bh + (r0 / p.bw) % p.bh;
      at.n = (mt / (p.tiles_w * p.tiles_h)) * p.bn + r0 / (p.bw * p.bh);
      at.sw = p.sw; at.sh = p.sh;
      at.vw = p.out_w - at.w; at.vh = p.out_h - at.h; at.vn = p.out_n - at.n;
      return Slab{&maps.out[p.cls[rest / pix_tiles].out_map], 0, nt * BN, at, 0, 0, 0, 0};
    }
    const int tile = w % tiles;
    const ConvTap tap = p.cls[0].taps[tile % p.num_taps_total];
    const int mn = tile / p.num_taps_total;
    const int m_idx = (mn / nnb) * BLOCK_M;
    return Slab{nullptr, m_idx + q * 32, (mn % nnb) * BN, StoreAt{}, tile, m_idx, tap.wcol, w / tiles};
  }
};

template <int BN, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_bf16_kernel(const __grid_constant__ ConvMaps maps, const __grid_constant__ ConvParams p) {
  persistent_body<BN, MODE == MODE_WGRAD, MODE != MODE_FPROP>(ConvWork<BN, MODE>(maps, p), p.g);
}

// 4D bf16 view {C, Wd, Hd, Nd} of an NHWC tensor (element pitches pw/ph/pn), box {64, bw, bh, bn}.
int make_map4(CUtensorMap* m, const void* ptr, uint64_t C, uint64_t Wd, uint64_t Hd, uint64_t Nd, uint64_t pw,
              uint64_t ph, uint64_t pn, uint32_t bw, uint32_t bh, uint32_t bn) {
  const cuuint64_t dims[4] = {C, Wd, Hd, Nd};
  const cuuint64_t strides[3] = {pw * 2, ph * 2, pn * 2};
  const cuuint32_t box[4] = {64, bw, bh, bn};
  return encode_map(m, ptr, 4, dims, strides, box);
}

// Pixel box {bw, bh, bn} (powers of two, bw*bh*bn == rows) that covers a W x H x N pixel space with the
// least padding; ties go to the widest box (longest contiguous runs in memory).
void choose_box(int W, int H, int N, int rows, int* bw, int* bh, int* bn) {
  double best = 1e30;
  *bw = 1; *bh = 1; *bn = rows;
  for (int w = 1; w <= rows; w <<= 1) {
    for (int h = 1; w * h <= rows; h <<= 1) {
      const int n = rows / (w * h);
      const double covered = (double)((W + w - 1) / w * w) * ((H + h - 1) / h * h) * ((N + n - 1) / n * n);
      const double score = covered - 1e-3 * w - 1e-6 * h;
      if (score < best) { best = score; *bw = w; *bh = h; *bn = n; }
    }
  }
}

int floordiv2(int e) { return (e >= 0) ? e / 2 : -((-e + 1) / 2); }

struct ConvShape {
  int N, H, W, Cin, Cout, R, S, stride, pad, OH, OW;
};

int check_shape(ConvShape& s) {
  if (s.R != s.S || (s.R != 1 && s.R != 3)) return fail("only 1x1 and 3x3 filters");
  if (s.pad != (s.R - 1) / 2) return fail("padding must be (R-1)/2");
  if (s.stride != 1 && s.stride != 2) return fail("stride must be 1 or 2");
  if (s.stride == 2 && ((s.H | s.W) & 1)) return fail("stride 2 needs even H and W");
  if ((s.Cin % 8) || (s.Cout % 8)) return fail("channels must be multiples of 8");
  s.OH = s.H / s.stride;
  s.OW = s.W / s.stride;
  return 0;
}

// parity views of an NHWC tensor with even H, W: a[ph*2+pw] = t[:, ph::2, pw::2, :]
int make_parity_maps(CUtensorMap* maps, const void* base, int C, int W, int H, int N, int bw, int bh, int bn) {
  for (int ph = 0; ph < 2; ++ph)
    for (int pw = 0; pw < 2; ++pw) {
      const __nv_bfloat16* ptr = reinterpret_cast<const __nv_bfloat16*>(base) + ((size_t)ph * W + pw) * C;
      if (make_map4(&maps[ph * 2 + pw], ptr, C, W / 2, H / 2, N, 2 * (uint64_t)C, 2 * (uint64_t)W * C,
                    (uint64_t)H * W * C, bw, bh, bn))
        return -1;
    }
  return 0;
}

// Taps of fprop and wgrad: tap (r, s) reads the input box shifted by (r - pad, s - pad); with stride 2 that is a
// shift inside one of the four parity views of the input.
void forward_taps(ConvClass& cl, int R, int S, int Cin, int stride, int pad) {
  for (int r = 0; r < R; ++r)
    for (int c = 0; c < S; ++c) {
      ConvTap& t = cl.taps[cl.ntaps++];
      const int eh = r - pad, ew = c - pad;
      if (stride == 1) {
        t.amap = 0; t.dh = eh; t.dw = ew;
      } else {
        const int ph = eh & 1, pw = ew & 1;
        t.amap = ph * 2 + pw; t.dh = floordiv2(eh - ph); t.dw = floordiv2(ew - pw);
      }
      t.wcol = (r * S + c) * Cin;
    }
}

// {sw, sh, 32 / (sw * sh)} pixel box of one 32-row slab of the {bw, bh, bn} M tile: the bulk-store box
void slab_box(ConvParams& p) {
  p.sw = p.bw < 32 ? p.bw : 32;
  p.sh = (32 / p.sw) < p.bh ? (32 / p.sw) : p.bh;
}

template <int MODE>
int launch_conv(const ConvMaps& maps, const ConvParams& p, int BN, int work, int max_ctas, cudaStream_t st) {
  if (BN == 64) return launch_persistent<conv_bf16_kernel<64, MODE>, 64>(work, max_ctas, st, maps, p);
  return launch_persistent<conv_bf16_kernel<128, MODE>, 128>(work, max_ctas, st, maps, p);
}

// zeroed parameters of a single-split convolution (no row limit: rows outside the output are clipped by TMA)
ConvParams conv_params() {
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.g.M = INT_MAX;
  p.g.splits = 1;
  p.g.alpha = 1.0f;
  return p;
}

}  // namespace

extern "C" {

const char* b200dp_conv_last_error() { return g_err; }

// y[N, OH, OW, Cout] = conv(x[N, H, W, Cin], w[Cout, R, S, Cin])          (all bf16, NHWC / KRSC)
int b200dp_conv_fprop(const void* x, const void* w, void* y, int N, int H, int W, int Cin, int Cout, int R, int S,
                      int stride, int pad, int block_n, int max_ctas, float* stats, unsigned long long stream) {
  if (ensure_init()) return -1;
  ConvShape s{N, H, W, Cin, Cout, R, S, stride, pad, 0, 0};
  if (check_shape(s)) return -1;
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) return fail("pointers must be 16-byte aligned");
  const int BN = pick_bn(Cout, block_n);
  if (BN < 0) return -1;
  ConvMaps maps;
  ConvParams p = conv_params();
  p.g.N = Cout; p.g.ldc = Cout; p.g.C = y; p.g.out_mode = 0;
  p.g.stats = stats;
  if (stats != nullptr && Cout > STATS_MAX_N) return fail("stats: Cout <= 2048 required");
  p.g.num_n_blocks = (Cout + BN - 1) / BN;
  p.g.num_k_blocks = (Cin + BLOCK_K - 1) / BLOCK_K;
  p.kc_per_tap = p.g.num_k_blocks;
  choose_box(s.OW, s.OH, N, BLOCK_M, &p.bw, &p.bh, &p.bn);
  p.tiles_w = (s.OW + p.bw - 1) / p.bw; p.tiles_h = (s.OH + p.bh - 1) / p.bh; p.tiles_n = (N + p.bn - 1) / p.bn;
  p.num_classes = 1;
  p.num_taps_total = R * S;
  p.out_w = s.OW; p.out_h = s.OH; p.out_n = N;
  forward_taps(p.cls[0], R, S, Cin, stride, pad);
  if (stride == 1) {
    if (make_map4(&maps.a[0], x, Cin, W, H, N, Cin, (uint64_t)W * Cin, (uint64_t)H * W * Cin, p.bw, p.bh, p.bn))
      return -1;
    maps.a[1] = maps.a[2] = maps.a[3] = maps.a[0];
  } else if (make_parity_maps(maps.a, x, Cin, W, H, N, p.bw, p.bh, p.bn)) {
    return -1;
  }
  if (make_map2(&maps.b, w, Cout, (uint64_t)R * S * Cin, (uint64_t)R * S * Cin, BN)) return -1;
  slab_box(p);
  if (make_map4(&maps.out[0], y, Cout, s.OW, s.OH, N, Cout, (uint64_t)s.OW * Cout, (uint64_t)s.OH * s.OW * Cout, p.sw,
                p.sh, 32 / (p.sw * p.sh)))
    return -1;
  maps.out[1] = maps.out[2] = maps.out[3] = maps.out[0];
  const int work = p.tiles_w * p.tiles_h * p.tiles_n * p.g.num_n_blocks;
  return launch_conv<MODE_FPROP>(maps, p, BN, work, max_ctas, (cudaStream_t)(uintptr_t)stream);
}

// dx[N, H, W, Cin] = conv_transpose(dy[N, OH, OW, Cout], w[Cout, R, S, Cin])
int b200dp_conv_dgrad(const void* dy, const void* w, void* dx, int N, int H, int W, int Cin, int Cout, int R, int S,
                      int stride, int pad, int block_n, int max_ctas, unsigned long long stream) {
  if (ensure_init()) return -1;
  ConvShape s{N, H, W, Cin, Cout, R, S, stride, pad, 0, 0};
  if (check_shape(s)) return -1;
  if (((uintptr_t)dy | (uintptr_t)w | (uintptr_t)dx) & 15) return fail("pointers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  const int BN = pick_bn(Cin, block_n);
  if (BN < 0) return -1;
  ConvMaps maps;
  ConvParams p = conv_params();
  p.g.N = Cin; p.g.ldc = Cin; p.g.C = dx; p.g.out_mode = 0;
  p.g.num_n_blocks = (Cin + BN - 1) / BN;
  p.g.num_k_blocks = (Cout + BLOCK_K - 1) / BLOCK_K;
  p.kc_per_tap = p.g.num_k_blocks;
  choose_box(s.OW, s.OH, N, BLOCK_M, &p.bw, &p.bh, &p.bn);   // stride 2: each dx parity view is OW x OH
  p.tiles_w = (s.OW + p.bw - 1) / p.bw; p.tiles_h = (s.OH + p.bh - 1) / p.bh; p.tiles_n = (N + p.bn - 1) / p.bn;
  p.num_taps_total = R * S;
  p.out_w = s.OW; p.out_h = s.OH; p.out_n = N;
  slab_box(p);
  const int sn = 32 / (p.sw * p.sh);
  if (make_map4(&maps.a[0], dy, Cout, s.OW, s.OH, N, Cout, (uint64_t)s.OW * Cout, (uint64_t)s.OH * s.OW * Cout,
                p.bw, p.bh, p.bn))
    return -1;
  maps.a[1] = maps.a[2] = maps.a[3] = maps.a[0];
  if (make_map2(&maps.b, w, Cout, (uint64_t)R * S * Cin, (uint64_t)R * S * Cin, 64)) return -1;
  if (stride == 1) {
    p.num_classes = 1;
    ConvClass& cl = p.cls[0];
    cl.out_map = 0;
    for (int r = 0; r < R; ++r)
      for (int c = 0; c < S; ++c) {
        ConvTap& t = cl.taps[cl.ntaps++];
        t.amap = 0; t.dh = pad - r; t.dw = pad - c; t.wcol = (r * S + c) * Cin;
      }
    if (make_map4(&maps.out[0], dx, Cin, W, H, N, Cin, (uint64_t)W * Cin, (uint64_t)H * W * Cin, p.sw, p.sh, sn))
      return -1;
    maps.out[1] = maps.out[2] = maps.out[3] = maps.out[0];
  } else {
    if (make_parity_maps(maps.out, dx, Cin, W, H, N, p.sw, p.sh, sn)) return -1;
    bool any_empty = false;
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw) {
        ConvClass cl;
        memset(&cl, 0, sizeof(cl));
        cl.out_map = ph * 2 + pw;
        for (int r = 0; r < R; ++r) {
          if ((ph + pad - r) & 1) continue;
          for (int c = 0; c < S; ++c) {
            if ((pw + pad - c) & 1) continue;
            ConvTap& t = cl.taps[cl.ntaps++];
            t.amap = 0; t.dh = floordiv2(ph + pad - r); t.dw = floordiv2(pw + pad - c); t.wcol = (r * S + c) * Cin;
          }
        }
        if (cl.ntaps == 0) { any_empty = true; continue; }
        p.cls[p.num_classes++] = cl;
      }
    if (any_empty) {    // 1x1 stride 2: the odd rows / columns of dx receive no gradient
      cudaError_t e = cudaMemsetAsync(dx, 0, (size_t)N * H * W * Cin * 2, st);
      if (e != cudaSuccess) return fail(cudaGetErrorString(e), (int)e);
    }
  }
  const int work = p.num_classes * p.tiles_w * p.tiles_h * p.tiles_n * p.g.num_n_blocks;
  return launch_conv<MODE_DGRAD>(maps, p, BN, work, max_ctas, st);
}

// dw[Cout][R*S*Cin] (+)= dy^T (*) x   (accumulate: add to dw; out_bf16: dw is bf16, else fp32) — split-K over
// pixels, summed in fp32 in split order and rounded once to dw's dtype.
int b200dp_conv_wgrad(const void* dy, const void* x, void* dw, int N, int H, int W, int Cin, int Cout, int R, int S,
                      int stride, int pad, int splits, int block_n, int max_ctas, int accumulate, int out_bf16,
                      unsigned long long stream) {
  if (ensure_init()) return -1;
  ConvShape s{N, H, W, Cin, Cout, R, S, stride, pad, 0, 0};
  if (check_shape(s)) return -1;
  if (((uintptr_t)dy | (uintptr_t)x | (uintptr_t)dw) & 15) return fail("pointers must be 16-byte aligned");
  const int BN = pick_bn(Cin, block_n);
  if (BN < 0) return -1;
  ConvMaps maps;
  ConvParams p = conv_params();
  p.g.M = Cout; p.g.N = Cin; p.g.ldc = R * S * Cin; p.g.C = dw;
  p.g.out_mode = accumulate ? 1 : 2;
  p.g.c_bf16 = out_bf16 ? 1 : 0;
  p.g.num_m_blocks = (Cout + BLOCK_M - 1) / BLOCK_M;
  p.g.num_n_blocks = (Cin + BN - 1) / BN;
  choose_box(s.OW, s.OH, N, BLOCK_K, &p.bw, &p.bh, &p.bn);     // 64-pixel K blocks
  p.tiles_w = (s.OW + p.bw - 1) / p.bw; p.tiles_h = (s.OH + p.bh - 1) / p.bh; p.tiles_n = (N + p.bn - 1) / p.bn;
  const int kblocks = p.tiles_w * p.tiles_h * p.tiles_n;
  p.num_classes = 1;
  p.num_taps_total = R * S;
  forward_taps(p.cls[0], R, S, Cin, stride, pad);
  const int tiles = p.g.num_m_blocks * p.g.num_n_blocks * R * S;
  if (splits <= 0) {
    splits = g_num_sms / tiles;                          // one wave: never a second, short one
    if (splits < 1) splits = 1;
    const int max_splits = kblocks / 8 > 1 ? kblocks / 8 : 1;
    if (splits > max_splits) splits = max_splits;
  }
  p.g.splits = normalize_splits(splits, kblocks);
  if (stride == 1) {
    if (make_map4(&maps.a[0], x, Cin, W, H, N, Cin, (uint64_t)W * Cin, (uint64_t)H * W * Cin, p.bw, p.bh, p.bn))
      return -1;
    maps.a[1] = maps.a[2] = maps.a[3] = maps.a[0];
  } else if (make_parity_maps(maps.a, x, Cin, W, H, N, p.bw, p.bh, p.bn)) {
    return -1;
  }
  if (make_map4(&maps.out[0], dy, Cout, s.OW, s.OH, N, Cout, (uint64_t)s.OW * Cout, (uint64_t)s.OH * s.OW * Cout,
                p.bw, p.bh, p.bn))
    return -1;
  maps.out[1] = maps.out[2] = maps.out[3] = maps.out[0];
  maps.b = maps.out[0];   // unused
  cudaStream_t st = (cudaStream_t)(uintptr_t)stream;
  if (p.g.splits > 1) p.g.splitk_slice = (long long)Cout * p.g.ldc;
  return run_splitk(p.g, tiles, st,
                    [&] { return launch_conv<MODE_WGRAD>(maps, p, BN, tiles * p.g.splits, max_ctas, st); });
}

}  // extern "C"

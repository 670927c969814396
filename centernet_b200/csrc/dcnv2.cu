// Modulated deformable convolution (DCNv2), im2col-free, fp32.
//
// Replaces dcn_v2_cuda_forward / dcn_v2_cuda_backward of
// src/lib/models/networks/DCNv2/src/dcn_v2_cuda.c:10-241 and the kernels of
// src/cuda/dcn_v2_im2col_cuda.cu:18-312:
//   y[b,o,h,w] = bias[o] + sum_{c,t} W[o,c,t] * mask[b,g*KT+t,h,w] * bilinear(x[b,c], h*s-p+i*d+dy, w*s-p+j*d+dx)
// with offset channel 2t = dy, 2t+1 = dx (:155-159) and the bilinear rule of :18-47 / :165
// (sample only if -1 < h_im < H and -1 < w_im < W; out-of-range corners contribute 0).
//
// The reference materialises a Cin*KT x HW column matrix per sample (37.7 MB for 64ch@128^2) and
// runs one SGEMM per sample.  Here a CTA owns 128 output pixels x (64|128) output channels:
//   1. per (tap, pixel) the 4 bilinear corner offsets + weights (mask folded in) are computed ONCE
//      and kept in shared memory (they are shared by every input channel of the deformable group);
//   2. per chunk of 8 input channels the sampled "column" tile [8*KT][128] is built in shared
//      memory straight from x (gathers hit L1/L2; the column matrix never touches HBM);
//   3. the chunk is contracted against the matching weight slice [8*KT][Cout_tile] with an 8x4
//      register tile per thread (fp32 FMA -- bit-compatible accumulation precision with the
//      reference SGEMM; the tensor-core path is dcnv2_tc.cu);
//   4. bias + store, coalesced along pixels.
// Backward: k_dcn_bwd_data recomputes the sampling per pixel tile, contracts grad_out with W^T
// chunk by chunk and turns the column gradient into dX (atomicAdd scatter, as the reference),
// dOffset and dMask without materialising it; k_dcn_bwd_weight accumulates dW / dBias over a
// range of pixel tiles in registers and adds them to the (accumulating) outputs once per CTA.
#include "dcnv2_tc.cuh"

namespace cnb {

constexpr int DCN_TP = 128;       // output pixels per CTA
constexpr int DCN_CK = 8;         // input channels per chunk
constexpr int DCN_KT_MAX = 9;     // taps (kh*kw)
constexpr int DCN_THREADS = 256;
constexpr int DCN_WPAD = 4;       // padding of the transposed weight tile

struct DcnShape {
  int B, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo;
};

struct TapMeta {   // one (tap, pixel): corner offsets into an input plane (-1: out of range, never read) + weights
  int o[4];
  float w[4];
};

// Bilinear geometry of one sampling point (dcn_v2_im2col_cuda.cu:18-47, :165).
struct Bilin {
  int h_low, w_low;
  float lh, lw;
  bool inside, v1, v2, v3, v4;
};
__device__ __forceinline__ Bilin bilin_setup(float h_im, float w_im, int H, int W) {
  Bilin g;
  g.inside = (h_im > -1.0f) && (w_im > -1.0f) && (h_im < (float)H) && (w_im < (float)W);
  const float hf = floorf(h_im), wf = floorf(w_im);
  g.h_low = (int)hf;
  g.w_low = (int)wf;
  g.lh = h_im - hf;
  g.lw = w_im - wf;
  const int h_high = g.h_low + 1, w_high = g.w_low + 1;
  g.v1 = g.inside && g.h_low >= 0 && g.w_low >= 0;
  g.v2 = g.inside && g.h_low >= 0 && w_high <= W - 1;
  g.v3 = g.inside && h_high <= H - 1 && g.w_low >= 0;
  g.v4 = g.inside && h_high <= H - 1 && w_high <= W - 1;
  return g;
}

__device__ __forceinline__ void sample_point(const DcnShape &s, const float *__restrict__ offset,
                                             const float *__restrict__ mask, int b, int g, int t, int p,
                                             float *h_im, float *w_im, float *m) {
  const int KT = s.kh * s.kw;
  const int ho = p / s.Wo, wo = p - ho * s.Wo;
  const int i = t / s.kw, j = t - i * s.kw;
  const long long HWo = (long long)s.Ho * s.Wo;
  const float *op = offset + ((long long)b * s.dg + g) * 2 * KT * HWo;
  const float dy = __ldg(op + (2 * t) * HWo + p), dx = __ldg(op + (2 * t + 1) * HWo + p);
  *m = __ldg(mask + (((long long)b * s.dg + g) * KT + t) * HWo + p);
  *h_im = (float)(ho * s.sh - s.ph + i * s.dh) + dy;
  *w_im = (float)(wo * s.sw - s.pw + j * s.dw) + dx;
}

// x at corner offset o of plane xp: an out-of-range corner (o < 0) is not read and counts 0, as in the reference
// (dcn_v2_im2col_cuda.cu:31-41), so a NaN / Inf elsewhere in the plane never meets its zero weight
__device__ __forceinline__ float corner_value(const float *__restrict__ xp, int o) {
  return o >= 0 ? __ldg(xp + o) : 0.0f;
}

// Fill meta[t][pp] for the pixel tile (deformable group g).  fold_mask: weights *= mask.
__device__ __forceinline__ void build_meta(const DcnShape &s, const float *offset, const float *mask, int b, int g,
                                           long long p_base, long long HWo, TapMeta *meta, float *mask_out,
                                           bool fold_mask) {
  const int KT = s.kh * s.kw;
  for (int idx = threadIdx.x; idx < KT * DCN_TP; idx += blockDim.x) {
    const int t = idx / DCN_TP, pp = idx - t * DCN_TP;
    const long long p = p_base + pp;
    TapMeta mt;
    float mval = 0.0f;
#pragma unroll
    for (int q = 0; q < 4; ++q) { mt.o[q] = -1; mt.w[q] = 0.0f; }
    if (p < HWo) {
      float h_im, w_im;
      sample_point(s, offset, mask, b, g, t, (int)p, &h_im, &w_im, &mval);
      const Bilin bl = bilin_setup(h_im, w_im, s.H, s.W);
      const float hh = 1.0f - bl.lh, hw = 1.0f - bl.lw;
      const float f = fold_mask ? mval : 1.0f;
      const int base = bl.h_low * s.W + bl.w_low;
      if (!bl.inside) mt.w[0] = 0.0f * f;   // outside: the column value is 0 * mask (:174), NaN for a NaN mask
      if (bl.v1) { mt.o[0] = base; mt.w[0] = hh * hw * f; }
      if (bl.v2) { mt.o[1] = base + 1; mt.w[1] = hh * bl.lw * f; }
      if (bl.v3) { mt.o[2] = base + s.W; mt.w[2] = bl.lh * hw * f; }
      if (bl.v4) { mt.o[3] = base + s.W + 1; mt.w[3] = bl.lh * bl.lw * f; }
    }
    meta[idx] = mt;
    if (mask_out) mask_out[idx] = mval;
  }
}

// ------------------------------------------------------------------ forward
template <int NSETS>
__global__ void __launch_bounds__(DCN_THREADS, 2)
k_dcn_forward(const float *__restrict__ x, const float *__restrict__ offset, const float *__restrict__ mask,
              const float *__restrict__ weight, const float *__restrict__ bias, float *__restrict__ y,
              const DcnShape s) {
  extern __shared__ __align__(16) unsigned char dcn_smem[];
  const int KT = s.kh * s.kw;
  constexpr int CO_T = 64 * NSETS;
  constexpr int WP = CO_T + DCN_WPAD;
  TapMeta *meta = reinterpret_cast<TapMeta *>(dcn_smem);                         // [KT][TP]
  float *col = reinterpret_cast<float *>(meta + DCN_KT_MAX * DCN_TP);            // [CK*KT][TP]
  float *wt = col + DCN_CK * DCN_KT_MAX * DCN_TP;                                // [CK*KT][WP]

  const long long HWo = (long long)s.Ho * s.Wo, HW = (long long)s.H * s.W;
  const int tiles = (int)((HWo + DCN_TP - 1) / DCN_TP);
  const int b = blockIdx.x / tiles;
  const long long p_base = (long long)(blockIdx.x - b * tiles) * DCN_TP;
  const int co_base = blockIdx.y * CO_T;
  const int cpg = s.Cin / s.dg;
  const int og = threadIdx.x >> 5, pg = threadIdx.x & 31;

  float acc[NSETS][8][4];
#pragma unroll
  for (int a = 0; a < NSETS; ++a)
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[a][i][j] = 0.0f;

  for (int g = 0; g < s.dg; ++g) {
    __syncthreads();
    build_meta(s, offset, mask, b, g, p_base, HWo, meta, nullptr, true);
    for (int c0 = g * cpg; c0 < (g + 1) * cpg; c0 += DCN_CK) {
      const int ck = min(DCN_CK, (g + 1) * cpg - c0);
      const int kc = ck * KT;
      __syncthreads();  // meta ready / previous chunk consumed
      // ---- weight slice, transposed: wt[kk][o] = W[co_base+o][c0*KT + kk]
      for (int idx = threadIdx.x; idx < CO_T * kc; idx += DCN_THREADS) {
        const int o = idx / kc, kk = idx - o * kc;
        float v = 0.0f;
        if (co_base + o < s.Cout) v = __ldg(weight + ((long long)(co_base + o) * s.Cin + c0) * KT + kk);
        wt[kk * WP + o] = v;
      }
      // ---- sampled column tile: col[cl*KT + t][pp]
      for (int idx = threadIdx.x; idx < kc * DCN_TP; idx += DCN_THREADS) {
        const int pp = idx & (DCN_TP - 1), r = idx >> 7;  // DCN_TP == 128
        const int cl = r / KT, t = r - cl * KT;
        const TapMeta mt = meta[t * DCN_TP + pp];
        const float *xp = x + ((long long)b * s.Cin + c0 + cl) * HW;
        float v = mt.w[0] * corner_value(xp, mt.o[0]);
        v = fmaf(mt.w[1], corner_value(xp, mt.o[1]), v);
        v = fmaf(mt.w[2], corner_value(xp, mt.o[2]), v);
        v = fmaf(mt.w[3], corner_value(xp, mt.o[3]), v);
        col[r * DCN_TP + pp] = v;
      }
      __syncthreads();
      // ---- contraction: acc[o][p] += wt[kk][o] * col[kk][p]
#pragma unroll 4
      for (int kk = 0; kk < kc; ++kk) {
        const float4 cv = *reinterpret_cast<const float4 *>(col + kk * DCN_TP + pg * 4);
#pragma unroll
        for (int a = 0; a < NSETS; ++a) {
          const float4 w0 = *reinterpret_cast<const float4 *>(wt + kk * WP + a * 64 + og * 8);
          const float4 w1 = *reinterpret_cast<const float4 *>(wt + kk * WP + a * 64 + og * 8 + 4);
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            acc[a][i][0] = fmaf(wv[i], cv.x, acc[a][i][0]);
            acc[a][i][1] = fmaf(wv[i], cv.y, acc[a][i][1]);
            acc[a][i][2] = fmaf(wv[i], cv.z, acc[a][i][2]);
            acc[a][i][3] = fmaf(wv[i], cv.w, acc[a][i][3]);
          }
        }
      }
    }
  }
  // ---- bias + store
  const long long p0 = p_base + pg * 4;
  const bool vec = (HWo % 4 == 0) && ((reinterpret_cast<uintptr_t>(y) & 15u) == 0);
#pragma unroll
  for (int a = 0; a < NSETS; ++a)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int o = co_base + a * 64 + og * 8 + i;
      if (o >= s.Cout) continue;
      const float bv = bias ? __ldg(bias + o) : 0.0f;
      float *yp = y + ((long long)b * s.Cout + o) * HWo;
      if (vec && p0 + 3 < HWo) {
        *reinterpret_cast<float4 *>(yp + p0) =
            make_float4(acc[a][i][0] + bv, acc[a][i][1] + bv, acc[a][i][2] + bv, acc[a][i][3] + bv);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (p0 + j < HWo) yp[p0 + j] = acc[a][i][j] + bv;
      }
    }
}

// ------------------------------------------------------------------ backward: dX, dOffset, dMask
struct BwdMeta {   // one (tap, pixel) of the backward pass: geometry instead of pre-multiplied weights
  int o[4];        // clamped corner offsets
  float lh, lw, m; // bilinear fractions and modulation mask
  int flags;       // bit q: corner q valid; bit 4: sampling point inside (-1,H)x(-1,W)
};

__device__ __forceinline__ void build_bwd_meta(const DcnShape &s, const float *offset, const float *mask, int b,
                                               int g, long long p_base, long long HWo, BwdMeta *meta) {
  const int KT = s.kh * s.kw;
  for (int idx = threadIdx.x; idx < KT * DCN_TP; idx += blockDim.x) {
    const int t = idx / DCN_TP, pp = idx - t * DCN_TP;
    const long long p = p_base + pp;
    BwdMeta mt;
    mt.o[0] = mt.o[1] = mt.o[2] = mt.o[3] = 0;
    mt.lh = mt.lw = mt.m = 0.f;
    mt.flags = 0;
    if (p < HWo) {
      float h_im, w_im, mval;
      sample_point(s, offset, mask, b, g, t, (int)p, &h_im, &w_im, &mval);
      const Bilin bl = bilin_setup(h_im, w_im, s.H, s.W);
      const int base = bl.h_low * s.W + bl.w_low;
      mt.lh = bl.lh; mt.lw = bl.lw; mt.m = mval;
      if (bl.v1) { mt.o[0] = base; mt.flags |= 1; }
      if (bl.v2) { mt.o[1] = base + 1; mt.flags |= 2; }
      if (bl.v3) { mt.o[2] = base + s.W; mt.flags |= 4; }
      if (bl.v4) { mt.o[3] = base + s.W + 1; mt.flags |= 8; }
      if (bl.inside) mt.flags |= 16;
    }
    meta[idx] = mt;
  }
}

// One CTA per (image, 128-pixel tile).  For every chunk of 8 input channels:
//   dcol[kk][p] = sum_o W[o][c0*KT+kk] * dY[o][p]         (contraction over Cout, 64 at a time)
// then per (tap, pixel), looping the chunk's channels in order (deterministic per-CTA sums):
//   dX      += dcol*mask*w_corner   (global atomicAdd, dcn_v2_im2col_cuda.cu:182-239)
//   dMask   += dcol * v             (:297)        v = unmasked bilinear sample
//   dOffset += dcol * mask * dv/d{h,w}   (:75-116, :299-302)
__global__ void __launch_bounds__(DCN_THREADS, 1)
k_dcn_bwd_data(const float *__restrict__ x, const float *__restrict__ offset, const float *__restrict__ mask,
               const float *__restrict__ weight, const float *__restrict__ gy, float *__restrict__ gx,
               float *__restrict__ goff, float *__restrict__ gmask, const DcnShape s, const int csplit) {
  // csplit > 1 (small maps: too few pixel tiles to fill the GPU): blockIdx.y takes every csplit-th channel
  // chunk and dOffset / dMask are accumulated into the outputs with atomics
  extern __shared__ __align__(16) unsigned char dcn_smem[];
  const int KT = s.kh * s.kw;
  constexpr int KC = DCN_CK * DCN_KT_MAX;
  BwdMeta *meta = reinterpret_cast<BwdMeta *>(dcn_smem);                  // [KT][TP]
  float *dcol = reinterpret_cast<float *>(meta + DCN_KT_MAX * DCN_TP);    // [KC][TP]
  float *gyt = dcol + KC * DCN_TP;                                        // [64][TP] grad_out slice
  float *wsl = gyt + 64 * DCN_TP;                                         // [64][KC+1] weight slice
  float *accm = wsl + 64 * (KC + 1);                                      // [KT][TP] dMask
  float *acch = accm + DCN_KT_MAX * DCN_TP;                               // [KT][TP] dOffset (h)
  float *accw = acch + DCN_KT_MAX * DCN_TP;                               // [KT][TP] dOffset (w)

  const long long HWo = (long long)s.Ho * s.Wo, HW = (long long)s.H * s.W;
  const int tiles = (int)((HWo + DCN_TP - 1) / DCN_TP);
  const int b = blockIdx.x / tiles;
  const long long p_base = (long long)(blockIdx.x - b * tiles) * DCN_TP;
  const int cpg = s.Cin / s.dg;
  const int tid = threadIdx.x;
  const int kg = tid >> 5, pg = tid & 31;   // dcol micro-tile: rows kg + 8i (i < 9) x pixels pg*4..+3

  for (int g = 0; g < s.dg; ++g) {
    __syncthreads();
    build_bwd_meta(s, offset, mask, b, g, p_base, HWo, meta);
    for (int idx = tid; idx < KT * DCN_TP; idx += DCN_THREADS) { accm[idx] = 0.f; acch[idx] = 0.f; accw[idx] = 0.f; }
    for (int c0 = g * cpg; c0 < (g + 1) * cpg; c0 += DCN_CK) {
      if (csplit > 1 && ((c0 - g * cpg) / DCN_CK) % csplit != (int)blockIdx.y) continue;   // CTA-uniform
      const int ck = min(DCN_CK, (g + 1) * cpg - c0);
      const int kc = ck * KT;
      float acc[9][4];
#pragma unroll
      for (int i = 0; i < 9; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      for (int o0 = 0; o0 < s.Cout; o0 += 64) {
        const int on = min(64, s.Cout - o0);
        __syncthreads();
        for (int idx = tid; idx < 64 * DCN_TP; idx += DCN_THREADS) {
          const int o = idx >> 7, pp = idx & (DCN_TP - 1);
          float v = 0.f;
          if (o < on && p_base + pp < HWo) v = __ldg(gy + ((long long)b * s.Cout + o0 + o) * HWo + p_base + pp);
          gyt[idx] = v;
        }
        for (int idx = tid; idx < 64 * kc; idx += DCN_THREADS) {
          const int o = idx / kc, kk = idx - o * kc;
          wsl[o * (KC + 1) + kk] = (o < on) ? __ldg(weight + ((long long)(o0 + o) * s.Cin + c0) * KT + kk) : 0.f;
        }
        __syncthreads();
        for (int o = 0; o < on; ++o) {
          const float4 gv = *reinterpret_cast<const float4 *>(gyt + o * DCN_TP + pg * 4);
#pragma unroll
          for (int i = 0; i < 9; ++i) {
            const int kk = kg + 8 * i;
            if (kk < kc) {
              const float wv = wsl[o * (KC + 1) + kk];
              acc[i][0] = fmaf(wv, gv.x, acc[i][0]);
              acc[i][1] = fmaf(wv, gv.y, acc[i][1]);
              acc[i][2] = fmaf(wv, gv.z, acc[i][2]);
              acc[i][3] = fmaf(wv, gv.w, acc[i][3]);
            }
          }
        }
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        const int kk = kg + 8 * i;
        if (kk < kc)
          *reinterpret_cast<float4 *>(dcol + kk * DCN_TP + pg * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      }
      __syncthreads();
      // ---- consume the column gradient: the thread that owns a (tap, pixel) walks the chunk's channels
      for (int idx = tid; idx < KT * DCN_TP; idx += DCN_THREADS) {
        const int t = idx / DCN_TP, pp = idx - t * DCN_TP;
        if (p_base + pp >= HWo) continue;
        const BwdMeta mt = meta[idx];
        if (!(mt.flags & 16)) continue;   // outside: no contribution to any gradient (:286-289)
        const float hh = 1.0f - mt.lh, hw = 1.0f - mt.lw;
        const float w1 = hh * hw, w2 = hh * mt.lw, w3 = mt.lh * hw, w4 = mt.lh * mt.lw;
        const bool f1 = mt.flags & 1, f2 = mt.flags & 2, f3 = mt.flags & 4, f4 = mt.flags & 8;
        float am = accm[idx], ah = acch[idx], aw = accw[idx];
        for (int cl = 0; cl < ck; ++cl) {
          const float d = dcol[(cl * KT + t) * DCN_TP + pp];
          const float *xp = x + ((long long)b * s.Cin + c0 + cl) * HW;
          const float x1 = f1 ? __ldg(xp + mt.o[0]) : 0.f, x2 = f2 ? __ldg(xp + mt.o[1]) : 0.f;
          const float x3 = f3 ? __ldg(xp + mt.o[2]) : 0.f, x4 = f4 ? __ldg(xp + mt.o[3]) : 0.f;
          am = fmaf(d, w1 * x1 + w2 * x2 + w3 * x3 + w4 * x4, am);
          const float dm = d * mt.m;
          ah = fmaf(dm, -hw * x1 - mt.lw * x2 + hw * x3 + mt.lw * x4, ah);
          aw = fmaf(dm, -hh * x1 + hh * x2 - mt.lh * x3 + mt.lh * x4, aw);
          if (gx) {
            float *gxp = gx + ((long long)b * s.Cin + c0 + cl) * HW;
            if (f1 && w1 != 0.f) atomicAdd(gxp + mt.o[0], dm * w1);
            if (f2 && w2 != 0.f) atomicAdd(gxp + mt.o[1], dm * w2);
            if (f3 && w3 != 0.f) atomicAdd(gxp + mt.o[2], dm * w3);
            if (f4 && w4 != 0.f) atomicAdd(gxp + mt.o[3], dm * w4);
          }
        }
        accm[idx] = am; acch[idx] = ah; accw[idx] = aw;
      }
    }
    __syncthreads();
    for (int idx = tid; idx < KT * DCN_TP; idx += DCN_THREADS) {
      const int t = idx / DCN_TP, pp = idx - t * DCN_TP;
      const long long p = p_base + pp;
      if (p >= HWo) continue;
      float *mp = gmask ? gmask + (((long long)b * s.dg + g) * KT + t) * HWo + p : nullptr;
      float *op = goff ? goff + ((long long)b * s.dg + g) * 2 * KT * HWo + p : nullptr;
      if (csplit > 1) {
        if (mp) atomicAdd(mp, accm[idx]);
        if (op) { atomicAdd(op + (2 * t) * HWo, acch[idx]); atomicAdd(op + (2 * t + 1) * HWo, accw[idx]); }
      } else {               // the only writer of this (tap, pixel): accumulate without atomics
        if (mp) *mp += accm[idx];
        if (op) { op[(2 * t) * HWo] += acch[idx]; op[(2 * t + 1) * HWo] += accw[idx]; }
      }
    }
  }
}

// ------------------------------------------------------------------ backward: dW (+= over batch and pixels)
// grid = (channel chunks, Cout/64, pixel-range splits).  Each CTA keeps a [8*KT][64] tile of dW in
// registers (9 x 2 per thread), walks its range of (image, pixel-tile) pairs rebuilding the masked
// column tile, and adds the tile to grad_weight once (atomicAdd: grad_weight accumulates, as in
// dcn_v2_cuda.c:217-220).  wpart != NULL (deterministic mode): the tile is stored as the split's partial
// wpart[split][o][cin][KT] instead (every element has one writer per split) and k_dcn_bwd_wsum adds the partials.
__global__ void __launch_bounds__(DCN_THREADS, 1)
k_dcn_bwd_weight(const float *__restrict__ x, const float *__restrict__ offset, const float *__restrict__ mask,
                 const float *__restrict__ gy, float *__restrict__ gw, float *__restrict__ wpart, const DcnShape s,
                 int splits) {
  extern __shared__ __align__(16) unsigned char dcn_smem[];
  const int KT = s.kh * s.kw;
  constexpr int KC = DCN_CK * DCN_KT_MAX;
  TapMeta *meta = reinterpret_cast<TapMeta *>(dcn_smem);                   // [KT][TP] (mask folded)
  float *col = reinterpret_cast<float *>(meta + DCN_KT_MAX * DCN_TP);      // [KC][TP]
  float *gyt = col + KC * DCN_TP;                                          // [TP][65] grad_out, pixel-major

  const long long HWo = (long long)s.Ho * s.Wo, HW = (long long)s.H * s.W;
  const int tiles = (int)((HWo + DCN_TP - 1) / DCN_TP);
  const int cpg = s.Cin / s.dg;
  const int chunks_per_group = (cpg + DCN_CK - 1) / DCN_CK;
  const int g = blockIdx.x / chunks_per_group;
  const int c0 = g * cpg + (blockIdx.x - g * chunks_per_group) * DCN_CK;
  const int ck = min(DCN_CK, (g + 1) * cpg - c0);
  const int kc = ck * KT;
  const int o0 = blockIdx.y * 64;
  const int on = min(64, s.Cout - o0);
  const int tid = threadIdx.x, kg = tid >> 5, lane = tid & 31;
  const long long work = (long long)s.B * tiles;
  const long long w_begin = work * blockIdx.z / splits, w_end = work * (blockIdx.z + 1) / splits;

  float acc[9][2];
#pragma unroll
  for (int i = 0; i < 9; ++i) acc[i][0] = acc[i][1] = 0.f;

  for (long long wi = w_begin; wi < w_end; ++wi) {
    const int b = (int)(wi / tiles);
    const long long p_base = (wi - (long long)b * tiles) * DCN_TP;
    __syncthreads();
    build_meta(s, offset, mask, b, g, p_base, HWo, meta, nullptr, true);
    for (int idx = tid; idx < 64 * DCN_TP; idx += DCN_THREADS) {
      const int o = idx >> 7, pp = idx & (DCN_TP - 1);
      float v = 0.f;
      if (o < on && p_base + pp < HWo) v = __ldg(gy + ((long long)b * s.Cout + o0 + o) * HWo + p_base + pp);
      gyt[pp * 65 + o] = v;
    }
    __syncthreads();
    for (int idx = tid; idx < kc * DCN_TP; idx += DCN_THREADS) {
      const int pp = idx & (DCN_TP - 1), r = idx >> 7;
      const int cl = r / KT, t = r - cl * KT;
      const TapMeta mt = meta[t * DCN_TP + pp];
      const float *xp = x + ((long long)b * s.Cin + c0 + cl) * HW;
      float v = mt.w[0] * corner_value(xp, mt.o[0]);
      v = fmaf(mt.w[1], corner_value(xp, mt.o[1]), v);
      v = fmaf(mt.w[2], corner_value(xp, mt.o[2]), v);
      v = fmaf(mt.w[3], corner_value(xp, mt.o[3]), v);
      col[r * DCN_TP + pp] = v;
    }
    __syncthreads();
#pragma unroll 2
    for (int pp = 0; pp < DCN_TP; ++pp) {
      const float g0 = gyt[pp * 65 + lane], g1 = gyt[pp * 65 + lane + 32];
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        const int kk = kg + 8 * i;
        const float cv = (kk < kc) ? col[kk * DCN_TP + pp] : 0.f;
        acc[i][0] = fmaf(cv, g0, acc[i][0]);
        acc[i][1] = fmaf(cv, g1, acc[i][1]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int kk = kg + 8 * i;
    if (kk >= kc) continue;
    if (wpart) {
      float *wp = wpart + (long long)blockIdx.z * s.Cout * s.Cin * KT;
      if (lane < on) wp[((long long)(o0 + lane) * s.Cin + c0) * KT + kk] = acc[i][0];
      if (lane + 32 < on) wp[((long long)(o0 + lane + 32) * s.Cin + c0) * KT + kk] = acc[i][1];
      continue;
    }
    if (lane < on) atomicAdd(gw + ((long long)(o0 + lane) * s.Cin + c0) * KT + kk, acc[i][0]);
    if (lane + 32 < on) atomicAdd(gw + ((long long)(o0 + lane + 32) * s.Cin + c0) * KT + kk, acc[i][1]);
  }
}

// gw[i] += sum over splits (ascending) of wpart[split][i]
__global__ void __launch_bounds__(256) k_dcn_bwd_wsum(const float *__restrict__ wpart, float *__restrict__ gw,
                                                      long long n, int splits) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int sp = 0; sp < splits; ++sp) acc += __ldg(wpart + (long long)sp * n + i);
    gw[i] += acc;
  }
}

// pixel-range splits of k_dcn_bwd_weight: about two CTAs per SM
static int fp32_weight_splits(int b, int cin, int cout, int dg, long long tiles) {
  const int cpg = cin / dg;
  const int chunks = dg * ((cpg + DCN_CK - 1) / DCN_CK);
  const int cot = (cout + 63) / 64;
  const long long work = (long long)b * tiles;
  int splits = (int)((2ll * num_sms() + (long long)chunks * cot - 1) / ((long long)chunks * cot));
  if (splits < 1) splits = 1;
  if ((long long)splits > work) splits = (int)work;
  return splits;
}

// dBias[o] += sum_{b,p} dY[b,o,p]   (dcn_v2_cuda.c:225-230)
__global__ void __launch_bounds__(256) k_dcn_bwd_bias(const float *__restrict__ gy, float *__restrict__ gb, int B,
                                                      int Cout, long long HWo) {
  __shared__ float red[8];
  const int o = blockIdx.x;
  float sum = 0.f;
  for (int b = 0; b < B; ++b) {
    const float *p = gy + ((long long)b * Cout + o) * HWo;
    for (long long i = threadIdx.x; i < HWo; i += blockDim.x) sum += __ldg(p + i);
  }
  for (int k = 16; k > 0; k >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, k);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(gb + o, t);
  }
}

// The one validation of every fp32 DCNv2 entry point and workspace query, then the plan of the call (dcnv2_tc.cuh).
// x_cl / gx_cl: the caller's input / grad_input are channels-last.
static int dcn_plan(const char *fn, int b, int cin, int h, int w, int cout, int kh, int kw, int sh, int sw, int ph,
                    int pw, int dh, int dw, int dg, bool det, bool x_cl, bool gx_cl, DcnPlan *p) {
  CNB_REQUIRE(b > 0 && cin > 0 && h > 0 && w > 0 && cout > 0 && kh > 0 && kw > 0, CNB_EINVAL,
              "%s: non-positive dimension", fn);
  CNB_REQUIRE(sh > 0 && sw > 0 && dh > 0 && dw > 0 && ph >= 0 && pw >= 0 && dg > 0, CNB_EINVAL,
              "%s: bad stride/dilation/padding/groups", fn);
  CNB_REQUIRE(cin % dg == 0, CNB_EINVAL, "%s: channels (%d) not divisible by deformable groups (%d)", fn, cin, dg);
  CNB_REQUIRE((long long)kh * kw <= DCN_KT_MAX, CNB_EUNSUPPORTED, "%s: kernel %dx%d has more than %d taps", fn, kh, kw,
              DCN_KT_MAX);
  const int ho = (h + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;   // dcn_v2_cuda.c:40-41
  const int wo = (w + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
  CNB_REQUIRE(ho > 0 && wo > 0, CNB_EINVAL, "%s: empty output", fn);
  CNB_REQUIRE((long long)h * w < (1ll << 31) && (long long)ho * wo < (1ll << 31), CNB_EUNSUPPORTED,
              "%s: plane too large", fn);
  fill_shape(&p->s, b, cin, h, w, cout, kh, kw, sh, sw, ph, pw, dh, dw, dg);
  const bool whole_blocks = (cin / dg) % TC_CB == 0;
  p->det = det;
  p->x_cl = x_cl && whole_blocks;
  p->gx_cl = gx_cl && whole_blocks;
  p->xt_ready = false;
  p->fwd_tc = sh == sw && ph == pw && dh == dw;   // and at most 9 taps, checked above
  p->fp32_dw_splits = fp32_weight_splits(b, cin, cout, dg, ((long long)ho * wo + DCN_TP - 1) / DCN_TP);
  plan_forward_tc(p);
  plan_backward_tc(p);
  return CNB_OK;
}

// the fp32 kernels' view of the validated shape
static DcnShape fp32_shape(const DcnShapeTc &t) {
  return {t.B, t.Cin, t.H, t.W, t.Cout, t.kh, t.kw, t.sh, t.sw, t.ph, t.pw, t.dh, t.dw, t.dg, t.Ho, t.Wo};
}

// fp32 CUDA-core backward of dX, dOffset, dMask
static int fp32_backward_data(const DcnShape &s, const float *input, const float *offset, const float *mask,
                              const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                              float *grad_mask, cudaStream_t stream) {
  constexpr int KC = DCN_CK * DCN_KT_MAX;
  const int tiles = (int)(((long long)s.Ho * s.Wo + DCN_TP - 1) / DCN_TP);
  const size_t smem = sizeof(BwdMeta) * DCN_KT_MAX * DCN_TP + sizeof(float) * KC * DCN_TP +
                      sizeof(float) * 64 * DCN_TP + sizeof(float) * 64 * (KC + 1) +
                      3 * sizeof(float) * DCN_KT_MAX * DCN_TP;
  CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_data, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // small maps: fewer pixel tiles than SMs -> also split the channel chunks over blockIdx.y
  const int chunks_pg = (s.Cin / s.dg + DCN_CK - 1) / DCN_CK;
  int csplit = (int)((2ll * num_sms() + (long long)s.B * tiles - 1) / ((long long)s.B * tiles));
  if (csplit > chunks_pg) csplit = chunks_pg;
  if (csplit < 1 || (long long)s.B * tiles >= num_sms()) csplit = 1;
  dim3 dgrid((unsigned)(s.B * tiles), (unsigned)csplit);
  k_dcn_bwd_data<<<dgrid, DCN_THREADS, smem, stream>>>(input, offset, mask, weight, grad_output, grad_input,
                                                       grad_offset, grad_mask, s, csplit);
  CNB_CHECK_LAUNCH("cnb_dcnv2_backward data");
  count_launch();
  return CNB_OK;
}

// fp32 CUDA-core backward of dW; wpart != NULL (deterministic mode): per-split partials, added in split order
static int fp32_backward_weight(const DcnShape &s, int splits, const float *input, const float *offset,
                                const float *mask, const float *grad_output, float *grad_weight, float *wpart,
                                cudaStream_t stream) {
  constexpr int KC = DCN_CK * DCN_KT_MAX;
  const int cpg = s.Cin / s.dg;
  const int chunks = s.dg * ((cpg + DCN_CK - 1) / DCN_CK);
  const int cot = (s.Cout + 63) / 64;
  const size_t smem = sizeof(TapMeta) * DCN_KT_MAX * DCN_TP + sizeof(float) * KC * DCN_TP +
                      sizeof(float) * DCN_TP * 65;
  CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_weight, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)chunks, (unsigned)cot, (unsigned)splits);
  k_dcn_bwd_weight<<<grid, DCN_THREADS, smem, stream>>>(input, offset, mask, grad_output, grad_weight, wpart, s, splits);
  CNB_CHECK_LAUNCH("cnb_dcnv2_backward weight");
  count_launch();
  if (wpart) {
    const long long n = (long long)s.Cout * s.Cin * s.kh * s.kw;
    k_dcn_bwd_wsum<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(wpart, grad_weight, n, splits);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward weight partials");
    count_launch();
  }
  return CNB_OK;
}

}  // namespace cnb

using namespace cnb;

extern "C" {

// No column / ones scratch (the reference's `columns`, `ones`): the workspace holds the weights re-tiled
// (TF32 hi/lo split, wgmma K-major layout) and a channels-last copy of the input for the tensor-core forward.  Passing workspace == NULL
// (or too small) to cnb_dcnv2_forward selects the fp32 CUDA-core kernel instead.  Every query returns 0 for a shape
// the calls reject.
size_t cnb_dcnv2_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw, int stride, int pad, int dil,
                                 int dg) {
  DcnPlan p;
  if (dcn_plan("cnb_dcnv2_workspace_bytes", b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, dg, false,
               false, false, &p) != CNB_OK)
    return 0;
  return p.fwd.bytes;
}

// Process-wide; every backward call reads it once and hands it down in its plan.
static std::atomic<int> g_dcn_deterministic{0};
void cnb_dcnv2_set_deterministic(int on) { g_dcn_deterministic.store(on ? 1 : 0, std::memory_order_relaxed); }
int cnb_dcnv2_get_deterministic(void) { return g_dcn_deterministic.load(std::memory_order_relaxed); }

size_t cnb_dcnv2_backward_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw, int stride, int pad,
                                          int dil, int dg) {
  DcnPlan p;
  if (dcn_plan("cnb_dcnv2_backward_workspace_bytes", b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, dg,
               cnb_dcnv2_get_deterministic() != 0, false, false, &p) != CNB_OK || !p.bwd_tc)
    return 0;
  return p.bwd.bytes;
}

size_t cnb_dcnv2_backward_bf16_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw, int stride,
                                               int pad, int dil, int dg) {
  DcnPlan p;
  if (dcn_plan("cnb_dcnv2_backward_bf16_workspace_bytes", b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil,
               dg, cnb_dcnv2_get_deterministic() != 0, false, false, &p) != CNB_OK)
    return 0;
  return p.bwd16.bytes;   // 0 where the bf16 backward does not run
}

// Checks in order: pointers, dtype codes, shape (dcn_plan), coverage, layout, workspace, alignment.
int cnb_dcnv2_backward_bf16(const void *input, int input_dtype, int input_channels_last, const float *offset,
                            const float *mask, const float *weight, const void *grad_output, int grad_output_dtype,
                            float *grad_input, int grad_input_channels_last, float *grad_offset, float *grad_mask,
                            float *grad_weight, float *grad_bias, int b, int cin, int h, int w, int cout, int kh,
                            int kw, int stride, int pad, int dil, int deformable_groups, void *workspace,
                            size_t workspace_bytes, void *stream) {
  const char *fn = "cnb_dcnv2_backward_bf16";
  CNB_REQUIRE(input && offset && mask && weight && grad_output && workspace, CNB_EINVAL, "%s: null pointer", fn);
  CNB_REQUIRE((input_dtype == CNB_DTYPE_F32 || input_dtype == CNB_DTYPE_BF16) &&
                  (grad_output_dtype == CNB_DTYPE_F32 || grad_output_dtype == CNB_DTYPE_BF16),
              CNB_EINVAL, "%s: unknown dtype code (input %d, grad_output %d)", fn, input_dtype, grad_output_dtype);
  const bool gx_cl = grad_input_channels_last && grad_input;
  DcnPlan p;
  int rc = dcn_plan(fn, b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, deformable_groups,
                    cnb_dcnv2_get_deterministic() != 0, input_channels_last != 0, gx_cl, &p);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(p.bwd16.bytes > 0, CNB_EUNSUPPORTED,
              "%s: the bf16 backward needs both tensor-core passes (cout <= 256, images within their 32-bit indexing)",
              fn);
  CNB_REQUIRE(!(input_channels_last || gx_cl) || (cin / deformable_groups) % 32 == 0, CNB_EUNSUPPORTED,
              "%s: channels-last tensors need cin / deformable_groups to be a multiple of 32", fn);
  CNB_REQUIRE(workspace_bytes >= p.bwd16.bytes, CNB_EWORKSPACE, "%s: workspace too small (%zu < %zu)", fn,
              workspace_bytes, p.bwd16.bytes);
  CNB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15u) == 0 && (reinterpret_cast<uintptr_t>(input) & 15u) == 0 &&
                  (!gx_cl || (reinterpret_cast<uintptr_t>(grad_input) & 15u) == 0),
              CNB_EINVAL, "%s: buffers must be 16-byte aligned", fn);
  return dcn_backward_bf16(p, input, input_dtype == CNB_DTYPE_BF16, offset, mask, weight, grad_output,
                           grad_output_dtype == CNB_DTYPE_BF16, grad_input, grad_offset, grad_mask, grad_weight,
                           grad_bias, workspace, (cudaStream_t)stream);
}

size_t cnb_dcnv2_wtiles_bytes(int cin, int cout, int kh, int kw, int dg) {
  DcnPlan p;   // the weight tiles do not depend on the image: any one the kernel fits in will do
  if (dcn_plan("cnb_dcnv2_wtiles_bytes", 1, cin, 8, 8, cout, kh, kw, 1, 1, 1, 1, 1, 1, dg, false, false, false, &p) !=
      CNB_OK)
    return 0;
  return p.fwd.wtiles_bytes;
}

int cnb_dcnv2_prepare_weights(const float *weight, int cin, int cout, int kh, int kw, int deformable_groups,
                              void *wtiles, size_t wtiles_bytes, void *stream) {
  CNB_REQUIRE(weight && wtiles, CNB_EINVAL, "cnb_dcnv2_prepare_weights: null pointer");
  CNB_REQUIRE(cin > 0 && cout > 0 && kh > 0 && kw > 0 && deformable_groups > 0 && cin % deformable_groups == 0,
              CNB_EINVAL, "cnb_dcnv2_prepare_weights: bad shape");
  CNB_REQUIRE(kh * kw <= DCN_KT_MAX, CNB_EUNSUPPORTED, "cnb_dcnv2_prepare_weights: more than %d taps", DCN_KT_MAX);
  const size_t need = cnb_dcnv2_wtiles_bytes(cin, cout, kh, kw, deformable_groups);
  CNB_REQUIRE(wtiles_bytes >= need, CNB_EWORKSPACE, "cnb_dcnv2_prepare_weights: buffer %zu < %zu", wtiles_bytes, need);
  CNB_REQUIRE((reinterpret_cast<uintptr_t>(wtiles) & 15u) == 0, CNB_EINVAL,
              "cnb_dcnv2_prepare_weights: buffer must be 16-byte aligned");
  return dcn_prepare_weights_tc(weight, cin, cout, kh, kw, deformable_groups, reinterpret_cast<float *>(wtiles),
                                (cudaStream_t)stream);
}

size_t cnb_dcnv2_prepared_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw, int stride, int pad,
                                          int dil, int dg) {
  DcnPlan p;
  if (dcn_plan("cnb_dcnv2_prepared_workspace_bytes", b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, dg,
               false, false, false, &p) != CNB_OK)
    return 0;
  return p.fwd.prepared_bytes;
}

int cnb_dcnv2_forward_prepared(const float *input, int input_channels_last, const float *offset, const float *mask,
                               const void *wtiles, const float *bias, float *output, int b, int cin, int h, int w,
                               int cout, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                               int dil_w, int deformable_groups, void *workspace, size_t workspace_bytes,
                               void *stream_) {
  CNB_REQUIRE(input && offset && mask && wtiles && output && workspace, CNB_EINVAL,
              "cnb_dcnv2_forward_prepared: null pointer");
  DcnPlan p;
  int rc = dcn_plan("cnb_dcnv2_forward_prepared", b, cin, h, w, cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h,
                    dil_w, deformable_groups, false, input_channels_last != 0, false, &p);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(p.fwd_tc, CNB_EUNSUPPORTED, "cnb_dcnv2_forward_prepared: anisotropic stride/pad/dilation");
  CNB_REQUIRE(workspace_bytes >= p.fwd.prepared_bytes, CNB_EWORKSPACE, "cnb_dcnv2_forward_prepared: workspace too small");
  CNB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15u) == 0 && (reinterpret_cast<uintptr_t>(wtiles) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(input) & 15u) == 0,
              CNB_EINVAL, "cnb_dcnv2_forward_prepared: buffers must be 16-byte aligned");
  return dcn_forward_tc_prepared(p, input, offset, mask, reinterpret_cast<const float *>(wtiles), bias, output,
                                 workspace, (cudaStream_t)stream_, 0, nullptr, nullptr, 0);
}

int cnb_dcnv2_forward_fused(const float *input, int input_channels_last, const float *offset_mask, const void *wtiles,
                            const float *bias, const float *bn_scale, const float *bn_shift, int relu, float *output,
                            int b, int cin, int h, int w, int cout, int kh, int kw, int stride, int pad, int dil,
                            int deformable_groups, void *workspace, size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(input && offset_mask && wtiles && output && workspace, CNB_EINVAL,
              "cnb_dcnv2_forward_fused: null pointer");
  CNB_REQUIRE((bn_scale == nullptr) == (bn_shift == nullptr), CNB_EINVAL,
              "cnb_dcnv2_forward_fused: bn_scale and bn_shift go together");
  DcnPlan p;
  int rc = dcn_plan("cnb_dcnv2_forward_fused", b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil,
                    deformable_groups, false, input_channels_last != 0, false, &p);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(workspace_bytes >= p.fwd.prepared_bytes, CNB_EWORKSPACE, "cnb_dcnv2_forward_fused: workspace too small");
  CNB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15u) == 0 && (reinterpret_cast<uintptr_t>(wtiles) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(input) & 15u) == 0,
              CNB_EINVAL, "cnb_dcnv2_forward_fused: buffers must be 16-byte aligned");
  return dcn_forward_tc_prepared(p, input, offset_mask, nullptr, reinterpret_cast<const float *>(wtiles), bias, output,
                                 workspace, (cudaStream_t)stream_, 1, bn_scale, bn_shift, relu);
}

// ------------------------------------------------------------------ bf16 forward (opt-in; dcnv2_tc.cu)
size_t cnb_dcnv2_wtiles_bf16_bytes(int cin, int cout, int kh, int kw, int dg) {
  DcnPlan p;   // as cnb_dcnv2_wtiles_bytes: any image the kernel fits in will do
  if (dcn_plan("cnb_dcnv2_wtiles_bf16_bytes", 1, cin, 8, 8, cout, kh, kw, 1, 1, 1, 1, 1, 1, dg, false, false, false,
               &p) != CNB_OK)
    return 0;
  return p.bf16.wtiles_bytes;
}

int cnb_dcnv2_prepare_weights_bf16(const float *weight, int cin, int cout, int kh, int kw, int deformable_groups,
                                   void *wtiles, size_t wtiles_bytes, void *stream) {
  CNB_REQUIRE(weight && wtiles, CNB_EINVAL, "cnb_dcnv2_prepare_weights_bf16: null pointer");
  CNB_REQUIRE(cin > 0 && cout > 0 && kh > 0 && kw > 0 && deformable_groups > 0 && cin % deformable_groups == 0,
              CNB_EINVAL, "cnb_dcnv2_prepare_weights_bf16: bad shape");
  CNB_REQUIRE(kh * kw <= DCN_KT_MAX, CNB_EUNSUPPORTED, "cnb_dcnv2_prepare_weights_bf16: more than %d taps", DCN_KT_MAX);
  const size_t need = cnb_dcnv2_wtiles_bf16_bytes(cin, cout, kh, kw, deformable_groups);
  CNB_REQUIRE(wtiles_bytes >= need, CNB_EWORKSPACE, "cnb_dcnv2_prepare_weights_bf16: buffer %zu < %zu", wtiles_bytes,
              need);
  CNB_REQUIRE((reinterpret_cast<uintptr_t>(wtiles) & 15u) == 0, CNB_EINVAL,
              "cnb_dcnv2_prepare_weights_bf16: buffer must be 16-byte aligned");
  return dcn_prepare_weights_bf16(weight, cin, cout, kh, kw, deformable_groups, wtiles, (cudaStream_t)stream);
}

size_t cnb_dcnv2_bf16_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw, int stride, int pad,
                                      int dil, int dg) {
  DcnPlan p;
  if (dcn_plan("cnb_dcnv2_bf16_workspace_bytes", b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, dg,
               false, false, false, &p) != CNB_OK)
    return 0;
  return p.bf16.prepared_bytes;
}

// The checks of both bf16 entry points, in order: pointers, dtype codes, shape (dcn_plan), workspace, alignment.
static int dcn_bf16_call(const char *fn, const void *input, int input_dtype, int input_channels_last,
                         const float *offset, const float *mask, const void *wtiles, const float *bias,
                         const float *bn_scale, const float *bn_shift, int relu, void *output, int output_dtype, int b,
                         int cin, int h, int w, int cout, int kh, int kw, int stride, int pad, int dil, int dg,
                         void *workspace, size_t workspace_bytes, void *stream, int fused) {
  CNB_REQUIRE(input && offset && (mask || fused) && wtiles && output && workspace, CNB_EINVAL, "%s: null pointer", fn);
  CNB_REQUIRE((bn_scale == nullptr) == (bn_shift == nullptr), CNB_EINVAL, "%s: bn_scale and bn_shift go together", fn);
  CNB_REQUIRE((input_dtype == CNB_DTYPE_F32 || input_dtype == CNB_DTYPE_BF16) &&
                  (output_dtype == CNB_DTYPE_F32 || output_dtype == CNB_DTYPE_BF16),
              CNB_EINVAL, "%s: unknown dtype code (input %d, output %d)", fn, input_dtype, output_dtype);
  DcnPlan p;
  int rc = dcn_plan(fn, b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, dg, false,
                    input_channels_last != 0, false, &p);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(workspace_bytes >= p.bf16.prepared_bytes, CNB_EWORKSPACE, "%s: workspace too small (%zu < %zu)", fn,
              workspace_bytes, p.bf16.prepared_bytes);
  CNB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15u) == 0 && (reinterpret_cast<uintptr_t>(wtiles) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(input) & 15u) == 0,
              CNB_EINVAL, "%s: buffers must be 16-byte aligned", fn);
  return dcn_forward_bf16(p, input, input_dtype == CNB_DTYPE_BF16, offset, mask, wtiles, bias, output,
                          output_dtype == CNB_DTYPE_BF16, workspace, (cudaStream_t)stream, fused, bn_scale, bn_shift,
                          relu);
}

int cnb_dcnv2_forward_bf16(const void *input, int input_dtype, int input_channels_last, const float *offset,
                           const float *mask, const void *wtiles, const float *bias, void *output, int output_dtype,
                           int b, int cin, int h, int w, int cout, int kh, int kw, int stride, int pad, int dil,
                           int deformable_groups, void *workspace, size_t workspace_bytes, void *stream) {
  return dcn_bf16_call("cnb_dcnv2_forward_bf16", input, input_dtype, input_channels_last, offset, mask, wtiles, bias,
                       nullptr, nullptr, 0, output, output_dtype, b, cin, h, w, cout, kh, kw, stride, pad, dil,
                       deformable_groups, workspace, workspace_bytes, stream, 0);
}

int cnb_dcnv2_forward_fused_bf16(const void *input, int input_dtype, int input_channels_last,
                                 const float *offset_mask, const void *wtiles, const float *bias,
                                 const float *bn_scale, const float *bn_shift, int relu, void *output,
                                 int output_dtype, int b, int cin, int h, int w, int cout, int kh, int kw, int stride,
                                 int pad, int dil, int deformable_groups, void *workspace, size_t workspace_bytes,
                                 void *stream) {
  return dcn_bf16_call("cnb_dcnv2_forward_fused_bf16", input, input_dtype, input_channels_last, offset_mask, nullptr,
                       wtiles, bias, bn_scale, bn_shift, relu, output, output_dtype, b, cin, h, w, cout, kh, kw,
                       stride, pad, dil, deformable_groups, workspace, workspace_bytes, stream, 1);
}

// ------------------------------------------------------------------ DCN block (opt-in; dcnv2_tc.cu)
// The range of the block kernel: the DCN of dla_34 and resnet_dcn
static int dcn_block_range(const char *fn, int cin, int kh, int kw, int stride, int pad, int dil, int dg) {
  CNB_REQUIRE(kh == 3 && kw == 3 && stride == 1 && pad == 1 && dil == 1 && dg == 1 && cin % TC_CB == 0,
              CNB_EUNSUPPORTED,
              "%s: needs a 3x3 kernel, stride 1, padding 1, dilation 1, one deformable group and cin %% 32 == 0 "
              "(got %dx%d, stride %d, padding %d, dilation %d, %d groups, cin %d)", fn, kh, kw, stride, pad, dil, dg, cin);
  return CNB_OK;
}

size_t cnb_dcnv2_om_tiles_bytes(int cin, int kh, int kw, int dg) {
  const char *fn = "cnb_dcnv2_om_tiles_bytes";
  if (cin <= 0 || dcn_block_range(fn, cin, kh, kw, 1, 1, 1, dg) != CNB_OK) return 0;
  return dcn_om_tiles_bytes(cin);
}

int cnb_dcnv2_prepare_om_weights_bf16(const float *w_om, int cin, int kh, int kw, int dg, void *om_tiles,
                                      size_t om_tiles_bytes, void *stream) {
  const char *fn = "cnb_dcnv2_prepare_om_weights_bf16";
  CNB_REQUIRE(w_om && om_tiles, CNB_EINVAL, "%s: null pointer", fn);
  CNB_REQUIRE(cin > 0 && kh > 0 && kw > 0 && dg > 0, CNB_EINVAL, "%s: bad shape", fn);
  const int rc = dcn_block_range(fn, cin, kh, kw, 1, 1, 1, dg);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(om_tiles_bytes >= dcn_om_tiles_bytes(cin), CNB_EWORKSPACE, "%s: buffer %zu < %zu", fn, om_tiles_bytes,
              dcn_om_tiles_bytes(cin));
  CNB_REQUIRE((reinterpret_cast<uintptr_t>(om_tiles) & 15u) == 0, CNB_EINVAL, "%s: buffer must be 16-byte aligned", fn);
  return dcn_prepare_om_weights_bf16(w_om, cin, om_tiles, (cudaStream_t)stream);
}

size_t cnb_dcnv2_block_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw, int stride, int pad,
                                       int dil, int dg) {
  const char *fn = "cnb_dcnv2_block_workspace_bytes";
  DcnPlan p;
  if (dcn_plan(fn, b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, dg, false, false, false, &p) !=
          CNB_OK ||
      dcn_block_range(fn, cin, kh, kw, stride, pad, dil, dg) != CNB_OK)
    return 0;
  return p.bf16.prepared_bytes;
}

int cnb_dcnv2_forward_block_bf16(const void *input, int input_dtype, int input_channels_last, const void *om_tiles,
                                 const float *om_bias, const void *wtiles, const float *bias, const float *bn_scale,
                                 const float *bn_shift, int relu, void *output, int b, int cin, int h, int w, int cout,
                                 int kh, int kw, int stride, int pad, int dil, int deformable_groups, void *workspace,
                                 size_t workspace_bytes, void *stream) {
  const char *fn = "cnb_dcnv2_forward_block_bf16";
  CNB_REQUIRE(input && om_tiles && wtiles && output && workspace, CNB_EINVAL, "%s: null pointer", fn);
  CNB_REQUIRE((bn_scale == nullptr) == (bn_shift == nullptr), CNB_EINVAL, "%s: bn_scale and bn_shift go together", fn);
  CNB_REQUIRE(input_dtype == CNB_DTYPE_F32 || input_dtype == CNB_DTYPE_BF16, CNB_EINVAL,
              "%s: input dtype must be CNB_DTYPE_F32 or CNB_DTYPE_BF16 (got %d)", fn, input_dtype);
  DcnPlan p;
  int rc = dcn_plan(fn, b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, deformable_groups, false,
                    input_channels_last != 0, false, &p);
  if (rc != CNB_OK) return rc;
  rc = dcn_block_range(fn, cin, kh, kw, stride, pad, dil, deformable_groups);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(workspace_bytes >= p.bf16.prepared_bytes, CNB_EWORKSPACE, "%s: workspace too small (%zu < %zu)", fn,
              workspace_bytes, p.bf16.prepared_bytes);
  CNB_REQUIRE(((reinterpret_cast<uintptr_t>(workspace) | reinterpret_cast<uintptr_t>(wtiles) |
                reinterpret_cast<uintptr_t>(om_tiles) | reinterpret_cast<uintptr_t>(input)) & 15u) == 0,
              CNB_EINVAL, "%s: buffers must be 16-byte aligned", fn);
  return dcn_forward_block_bf16(p, input, input_dtype == CNB_DTYPE_BF16, om_tiles, om_bias, wtiles, bias, output,
                                workspace, (cudaStream_t)stream, bn_scale, bn_shift, relu);
}

int cnb_dcnv2_forward(const float *input, const float *offset, const float *mask, const float *weight,
                      const float *bias, float *output, int b, int cin, int h, int w, int cout, int kh, int kw,
                      int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int deformable_groups,
                      void *workspace, size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(input && offset && mask && weight && output, CNB_EINVAL, "cnb_dcnv2_forward: null pointer");
  DcnPlan p;
  int rc = dcn_plan("cnb_dcnv2_forward", b, cin, h, w, cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w,
                    deformable_groups, false, false, false, &p);
  if (rc != CNB_OK) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (p.fwd_tc && workspace && workspace_bytes >= p.fwd.bytes && (reinterpret_cast<uintptr_t>(workspace) & 15u) == 0) {
    // the weight tiles at the head of the workspace, the prepared forward's workspace behind them
    float *wt = reinterpret_cast<float *>(workspace);
    rc = dcn_prepare_weights_tc(weight, cin, cout, kh, kw, deformable_groups, wt, stream);
    if (rc != CNB_OK) return rc;
    return dcn_forward_tc_prepared(p, input, offset, mask, wt, bias, output,
                                   reinterpret_cast<char *>(workspace) + p.fwd.wtiles_bytes, stream, 0, nullptr,
                                   nullptr, 0);
  }
  const DcnShape s = fp32_shape(p.s);
  const int tiles = (int)(((long long)s.Ho * s.Wo + DCN_TP - 1) / DCN_TP);
  const int nsets = cout > 64 ? 2 : 1;
  const int co_t = 64 * nsets;
  const size_t smem = sizeof(TapMeta) * DCN_KT_MAX * DCN_TP + sizeof(float) * DCN_CK * DCN_KT_MAX * DCN_TP +
                      sizeof(float) * DCN_CK * DCN_KT_MAX * (co_t + DCN_WPAD);
  dim3 grid((unsigned)(b * tiles), (unsigned)((cout + co_t - 1) / co_t));
  if (nsets == 1) {
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_forward<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_dcn_forward<1><<<grid, DCN_THREADS, smem, stream>>>(input, offset, mask, weight, bias, output, s);
  } else {
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_forward<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_dcn_forward<2><<<grid, DCN_THREADS, smem, stream>>>(input, offset, mask, weight, bias, output, s);
  }
  CNB_CHECK_LAUNCH("cnb_dcnv2_forward");
  count_launch();
  return CNB_OK;
}

static int dcnv2_backward_impl(const float *input, const float *offset, const float *mask, const float *weight,
                               const float *grad_output, float *grad_input, float *grad_offset, float *grad_mask,
                               float *grad_weight, float *grad_bias, int b, int cin, int h, int w, int cout, int kh,
                               int kw, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w,
                               int deformable_groups, void *workspace, size_t workspace_bytes, void *stream_,
                               bool input_cl, bool grad_input_cl) {
  CNB_REQUIRE(input && offset && mask && weight && grad_output, CNB_EINVAL, "cnb_dcnv2_backward: null pointer");
  DcnPlan p;
  int rc = dcn_plan("cnb_dcnv2_backward", b, cin, h, w, cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w,
                    deformable_groups, cnb_dcnv2_get_deterministic() != 0, input_cl, grad_input_cl && grad_input, &p);
  if (rc != CNB_OK) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  const bool data = grad_input || grad_offset || grad_mask;
  // tensor-core path (dcnv2_bwd_tc.cu) when the caller provides the workspace; else the fp32 CUDA-core kernels
  const bool tc = p.bwd_tc && workspace && workspace_bytes >= p.bwd.bytes &&
                  (reinterpret_cast<uintptr_t>(workspace) & 15u) == 0;
  // deterministic mode is implemented by the tensor-core backward only (the fp32 kernels scatter with atomics)
  CNB_REQUIRE(!p.det || tc || !(data || grad_weight), CNB_EUNSUPPORTED,
              "cnb_dcnv2_backward: deterministic mode (cnb_dcnv2_set_deterministic) needs the tensor-core backward: a "
              "workspace of cnb_dcnv2_backward_workspace_bytes queried in deterministic mode, at most 9 taps, isotropic "
              "stride/pad/dilation and images within its 32-bit indexing");
  if (input_cl || grad_input_cl) {   // channels-last input / grad_input: tensor-core path only, whole 32-channel blocks, scatter form of dX
    CNB_REQUIRE(tc && p.dw_tc, CNB_EUNSUPPORTED, "cnb_dcnv2_backward_ex: channels-last tensors need the tensor-core path "
                "(workspace of cnb_dcnv2_backward_workspace_bytes, at most 9 taps, isotropic stride/pad/dilation, cout <= 256)");
    CNB_REQUIRE((cin / deformable_groups) % 32 == 0, CNB_EUNSUPPORTED,
                "cnb_dcnv2_backward_ex: channels-last tensors need cin / deformable_groups to be a multiple of 32");
  }
  const DcnShape s = fp32_shape(p.s);
  if (data) {
    rc = tc ? dcn_backward_data_tc(p, input, offset, mask, weight, grad_output, grad_input, grad_offset, grad_mask,
                                   workspace, stream)
            : fp32_backward_data(s, input, offset, mask, weight, grad_output, grad_input, grad_offset, grad_mask, stream);
    if (rc != CNB_OK) return rc;
  }
  if (grad_weight && tc && p.dw_tc) {
    p.xt_ready = data;
    rc = dcn_backward_weight_tc(p, input, offset, mask, grad_output, grad_weight, grad_bias, workspace, stream);
    grad_bias = nullptr;   // done by the weight pass
  } else if (grad_weight) {
    float *wpart = p.det ? reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.bwd.wpart32) : nullptr;
    rc = fp32_backward_weight(s, p.fp32_dw_splits, input, offset, mask, grad_output, grad_weight, wpart, stream);
  }
  if (rc != CNB_OK) return rc;
  if (grad_bias) {
    k_dcn_bwd_bias<<<cout, 256, 0, stream>>>(grad_output, grad_bias, b, cout, (long long)s.Ho * s.Wo);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward bias");
    count_launch();
  }
  return CNB_OK;
}

int cnb_dcnv2_backward(const float *input, const float *offset, const float *mask, const float *weight,
                       const float *grad_output, float *grad_input, float *grad_offset, float *grad_mask,
                       float *grad_weight, float *grad_bias, int b, int cin, int h, int w, int cout, int kh, int kw,
                       int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int deformable_groups,
                       void *workspace, size_t workspace_bytes, void *stream_) {
  return dcnv2_backward_impl(input, offset, mask, weight, grad_output, grad_input, grad_offset, grad_mask, grad_weight,
                             grad_bias, b, cin, h, w, cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w,
                             deformable_groups, workspace, workspace_bytes, stream_, false, false);
}

int cnb_dcnv2_backward_ex(const float *input, int input_channels_last, const float *offset, const float *mask,
                          const float *weight, const float *grad_output, float *grad_input,
                          int grad_input_channels_last, float *grad_offset, float *grad_mask, float *grad_weight,
                          float *grad_bias, int b, int cin, int h, int w, int cout, int kh, int kw, int stride, int pad,
                          int dil, int deformable_groups, void *workspace, size_t workspace_bytes, void *stream_) {
  return dcnv2_backward_impl(input, offset, mask, weight, grad_output, grad_input, grad_offset, grad_mask, grad_weight,
                             grad_bias, b, cin, h, w, cout, kh, kw, stride, stride, pad, pad, dil, dil, deformable_groups,
                             workspace, workspace_bytes, stream_, input_channels_last != 0,
                             grad_input_channels_last != 0);
}

}  // extern "C"

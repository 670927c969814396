// DCNv2 backward with both dense contractions on the Hopper tensor cores (wgmma, 3xTF32).
// Reference: dcn_v2_cuda.c:104-241 (per sample: SGEMM columns = W^T . dY, col2im_coord, col2im, im2col again,
// SGEMM dW += dY . columns^T, SGEMV dBias) and dcn_v2_im2col_cuda.cu:182-312.
//
// The column gradient
//     dcol[b][p][q = (channel block, tap)][32 ch] = sum_o dY[b][o][p] * W[o][ch][tap]
// is a plain GEMM (M = pixels, N = Cin*9, K = Cout).  k_dcn_bwd_dcol_tc runs it as a persistent TMA -> wgmma
// pipeline (both operands arrive pre-split into TF32 hi/lo tiles; no thread touches an operand) and writes
// dcol channels-last, so that everything after it moves whole 128-byte lines:
//   k_dcn_bwd_offmask   one (tap, 4 pixels) per warp, lane = (pixel, 4-channel quad): reads the dcol line and the
//                       four bilinear corner lines of the channels-last input, reduces dMask / dOffset over the
//                       channels in a fixed order (deterministic; dcn_v2_im2col_cuda.cu:241-312) and scatters
//                       dX = dcol * mask * corner weight with 16-byte vector reductions (red.global.add.v4.f32:
//                       a quarter of the reference's per-element atomicAdds, :182-239) into a channels-last dX
//   k_dcn_bwd_dx_nchw   adds the channels-last dX into the caller's NCHW gradient
// Deterministic mode (cnb_dcnv2_set_deterministic) keeps the scatter but makes it order-independent: every dX
// contribution is rounded to a 64-bit fixed-point integer with a per-image power-of-two scale and added with
// red.global.add.u64 (integer addition is associative: any order, grid or batch split gives the same sum);
// k_dcn_bwd_dx_fixed then converts the integers back to fp32 into grad_input (NCHW or channels-last).  The
// scale comes from a bound on |dX| that holds before any contribution is made (see det_scale).
// The weight gradient dW[o][ch][tap] = sum_{b,p} dY[b][o][p] * col[b][p][ch][tap] is a GEMM with K = pixels:
// k_dcn_bwd_weight_tc rebuilds the masked column tile in shared memory exactly as the forward sampler does
// (never in HBM), keeps a [128 rows = 4 chunks x 32 ch] x (64|128 output channels) accumulator in the registers of two
// warpgroups over its whole pixel range and
// writes one partial per CTA; k_dcn_bwd_wreduce adds the partials in a fixed order (deterministic).
// plan_backward_tc lays out every region of the workspace these passes use (DcnPlan::bwd in dcnv2_tc.cuh); the
// hosts below only read their pointers from the plan.
#include <stdlib.h>
#include <algorithm>
#include "dcnv2_tc.cuh"

namespace cnb {

constexpr int BW_STAGES = 3;
constexpr int BW_STAGE_BYTES = 4 * TC_A_BYTES;     // A hi, A lo, B hi, B lo: 4 x (128 rows x 32 k x 4 B) = 64 KB
constexpr int BW_TILE_FLOATS = 2 * TC_TP * TC_K;   // one operand tile, hi + lo
constexpr int BW_THREADS = (4 * TC_MMA_WGS + 1) * 32;   // warps 0-7 two consumer warpgroups (MMA + epilogue), 8 TMA

struct BwdGeom {
  int KS;      // 32-wide slices of Cout (K of the dcol GEMM)
  int Q;       // chunks (channel block, tap) = nb * 9
  int RG;      // groups of 4 chunks = 128 GEMM rows
  int Qp;      // RG * 4: chunk pitch of dcol
  int tiles;   // pixel tiles per image
};
static BwdGeom bwd_geom(const DcnShapeTc &s) {
  BwdGeom g;
  g.KS = (s.Cout + TC_K - 1) / TC_K;
  g.Q = s.nb * TC_NT;
  g.RG = (g.Q + 3) / 4;
  g.Qp = g.RG * 4;
  g.tiles = s.tiles_x * s.tiles_y;
  return g;
}

// Bounds of deterministic mode, as the bits of non-negative floats (integer max of those bits is the float max,
// NaN > inf > finite, and max is order-free): bnd[ks] = max over rows r of sum_{o in slice ks} |W[o][r]|,
// bnd[KS + 2b] = max |dY| of image b, bnd[KS + 2b + 1] = max |mask| of image b.
__device__ __forceinline__ unsigned abs_bits(float v) { return __float_as_uint(v) & 0x7fffffffu; }
__device__ __forceinline__ unsigned warp_max_u32(unsigned v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, d));
  return v;
}

// W[Cout][Cin][KT] -> per (row group rg, slice ks): [128 rows = (chunk ql, ch)][32 k = output channel], hi then lo.
// DET: also bnd[ks] (a warp holds one row's 32 output channels of the slice per iteration: lane = k).
template <bool DET>
__global__ void __launch_bounds__(256) k_bwd_prep_w(const float *__restrict__ w, const DcnShapeTc s, const BwdGeom g,
                                                    float *__restrict__ wtt, unsigned *__restrict__ bnd) {
  const int KT = s.kh * s.kw, cpg = s.Cin / s.dg;
  const int rg = blockIdx.x / g.KS, ks = blockIdx.x - rg * g.KS;
  unsigned char *hi = reinterpret_cast<unsigned char *>(wtt + (size_t)blockIdx.x * BW_TILE_FLOATS);
  unsigned char *lo = hi + TC_A_BYTES;
  unsigned rmax = 0;
  for (int i = threadIdx.x; i < TC_TP * TC_K; i += blockDim.x) {
    const int k = i & (TC_K - 1), row = i >> 5;
    const int q = rg * 4 + (row >> 5), ch = row & 31;
    const int bi = q / TC_NT, tap = q - bi * TC_NT;
    const int gi = bi / s.cbs_pg, cw = (bi - gi * s.cbs_pg) * TC_CB + ch;
    const int o = ks * TC_K + k;
    float v = 0.f;
    if (q < g.Q && o < s.Cout && cw < cpg && tap < KT) v = __ldg(w + ((size_t)o * s.Cin + gi * cpg + cw) * KT + tap);
    const float h = tf32_hi(v);
    *reinterpret_cast<float *>(hi + tc_tile_off(row, k)) = h;
    *reinterpret_cast<float *>(lo + tc_tile_off(row, k)) = v - h;
    if (DET) {
      float sum = fabsf(v);
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
      rmax = max(rmax, abs_bits(sum));
    }
  }
  if (DET && (threadIdx.x & 31) == 0) atomicMax(bnd + ks, rmax);
}

// dY [B][Cout][HWo] -> per (image, pixel tile, slice ks): [128 px][32 k = output channel], hi then lo.  grid (tiles, KS, B)
// DET: also the bounds max |dY| and (blocks of slice 0, over the tile's pixels) max |mask| of each image.
template <bool DET>
__global__ void __launch_bounds__(256) k_bwd_prep_gy(const float *__restrict__ gy, const DcnShapeTc s, const BwdGeom g,
                                                     float *__restrict__ gyt, const float *__restrict__ mask,
                                                     unsigned *__restrict__ bnd_img) {
  const int t = blockIdx.x, ks = blockIdx.y, b = blockIdx.z;
  const int pp = threadIdx.x & (TC_TP - 1), half = threadIdx.x >> 7;
  const int ho = (t / s.tiles_x) * s.th + pp / s.tw, wo = (t % s.tiles_x) * s.tw + pp % s.tw;
  const bool ok = ho < s.Ho && wo < s.Wo;
  const long long HWo = (long long)s.Ho * s.Wo, p = (long long)ho * s.Wo + wo;
  unsigned char *hi = reinterpret_cast<unsigned char *>(gyt + ((size_t)((size_t)b * g.tiles + t) * g.KS + ks) * BW_TILE_FLOATS);
  unsigned char *lo = hi + TC_A_BYTES;
  unsigned ymax = 0;
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    const int kq = half * 4 + kc;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = ks * TC_K + kq * 4 + j;
      v[j] = (ok && o < s.Cout) ? __ldg(gy + ((long long)b * s.Cout + o) * HWo + p) : 0.f;
      if (DET) ymax = max(ymax, abs_bits(v[j]));
    }
    const float4 h4 = make_float4(tf32_hi(v[0]), tf32_hi(v[1]), tf32_hi(v[2]), tf32_hi(v[3]));
    const uint32_t off = tc_tile_off(pp, kq * 4);
    *reinterpret_cast<float4 *>(hi + off) = h4;
    *reinterpret_cast<float4 *>(lo + off) = make_float4(v[0] - h4.x, v[1] - h4.y, v[2] - h4.z, v[3] - h4.w);
  }
  if (DET) {
    unsigned mmax = 0;
    if (ks == 0 && ok) {
      const float *mp = mask + (long long)b * s.mask_bs + p;
      for (int c = half; c < s.dg * s.kh * s.kw; c += 2) mmax = max(mmax, abs_bits(__ldg(mp + (long long)c * HWo)));
    }
    ymax = warp_max_u32(ymax);
    mmax = warp_max_u32(mmax);
    if ((threadIdx.x & 31) == 0) {
      atomicMax(bnd_img + 2 * b, ymax);
      if (mmax) atomicMax(bnd_img + 2 * b + 1, mmax);
    }
  }
}

// Scale of image b's fixed-point dX, or 0 when its bounds are not finite.  A dX element collects at most one
// contribution dcol * mask * w_corner (w_corner <= 1) per sampling point that can reach it: KT * HWo of them, and
//   |dcol[p][c,tap]| <= sum_o |W[o][c][tap]| * max|dY_b| <= A * Y_b,   A = sum_ks bnd[ks],
// so |dX| <= KT * HWo * A * Y_b * M_b = bound.  The scale is the power of two with bound * scale < 2^61: one bit
// below the 2^62 that the int64 sums stay under, as margin for the rounding of dcol (3xTF32), of the float sums
// behind A and of the products.  Resolution: bound * 2^-61 (64@128^2: KT * HWo = 2^17.2, so 2^-43.8 * A * Y_b * M_b).
__device__ __forceinline__ double det_scale(const unsigned *__restrict__ bnd, const DcnShapeTc &s, const BwdGeom &g,
                                            int b) {
  double a = 0.0;
  for (int ks = 0; ks < g.KS; ++ks) a += (double)__uint_as_float(bnd[ks]);
  const double bound = (double)(s.kh * s.kw) * ((double)s.Ho * s.Wo) * a * (double)__uint_as_float(bnd[g.KS + 2 * b]) *
                       (double)__uint_as_float(bnd[g.KS + 2 * b + 1]);
  if (!(bound <= 1e300)) return 0.0;   // inf or NaN in dY, W or the mask
  if (bound == 0.0) return 1.0;        // every contribution is zero
  int ex;
  frexp(bound, &ex);                   // bound < 2^ex
  return ldexp(1.0, 61 - ex);
}

// ------------------------------------------------------------------ dcol = dY^T . W   (item = image, pixel tile, row group)
__global__ void __launch_bounds__(BW_THREADS, 1)
k_dcn_bwd_dcol_tc(const float *__restrict__ gyt, const float *__restrict__ wtt, float *__restrict__ dcol,
                  const DcnShapeTc s, const BwdGeom g, const int n_items) {
  extern __shared__ __align__(128) unsigned char tc_smem[];
  __shared__ __align__(8) uint64_t full[BW_STAGES], empty[BW_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < BW_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TC_MMA_WGS); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == TC_WARP_TMA) {
    if (lane == 0) {
      int stage = 0, ph = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int rg = item % g.RG, bt = item / g.RG;          // bt = image * tiles + tile
        for (int ks = 0; ks < g.KS; ++ks) {
          mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));
          unsigned char *dst = tc_smem + (size_t)stage * BW_STAGE_BYTES;
          const unsigned char *a = reinterpret_cast<const unsigned char *>(gyt + ((size_t)bt * g.KS + ks) * BW_TILE_FLOATS);
          const unsigned char *bsrc = reinterpret_cast<const unsigned char *>(wtt + ((size_t)rg * g.KS + ks) * BW_TILE_FLOATS);
          mbar_expect_tx(&full[stage], (uint32_t)BW_STAGE_BYTES);
          for (uint32_t off = 0; off < 2u * TC_A_BYTES; off += 8192u) bulk_g2s(dst + off, a + off, 8192u, &full[stage]);
          for (uint32_t off = 0; off < 2u * TC_A_BYTES; off += 8192u)
            bulk_g2s(dst + 2 * TC_A_BYTES + off, bsrc + off, 8192u, &full[stage]);
          if (++stage == BW_STAGES) { stage = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp < TC_WARP_TMA) {
    // consumers: warpgroup wgi computes pixels 64 wgi .. 64 wgi + 63 of the tile x the 128 columns (4 chunks x 32 ch)
    // of the row group, then stores them straight from the registers: per row a thread holds 2 adjacent channels of
    // every 8, so a warp's store covers 8 pixels x 32 contiguous bytes
    const int wgi = warp >> 2, wq = warp & 3;
    const long long HWo = (long long)s.Ho * s.Wo;
    int stage = 0, ph = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int rg = item % g.RG, bt = item / g.RG;
      const int t = bt % g.tiles, b = bt / g.tiles;
      const int ty0 = (t / s.tiles_x) * s.th, tx0 = (t % s.tiles_x) * s.tw;
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      for (int ks = 0; ks < g.KS; ++ks) {
        mbar_wait(&full[stage], (uint32_t)ph);
        const uint32_t base = smem_u32(tc_smem + (size_t)stage * BW_STAGE_BYTES);
        const uint32_t ah = base + (uint32_t)wgi * 8u * TC_SBO, al = ah + TC_A_BYTES;
        const uint32_t bh = base + 2u * TC_A_BYTES, bl = bh + TC_A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k8 = 0; k8 < TC_K / 8; ++k8) {
          const uint32_t koff = (uint32_t)k8 * 2u * TC_LBO;
          wgmma_3xtf32<128>(d, tc_desc(ah + koff), tc_desc(al + koff), tc_desc(bh + koff), tc_desc(bl + koff),
                            (ks > 0 || k8 > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        if ((tid & 127) == 0) mbar_arrive_tc(&empty[stage]);
        if (++stage == BW_STAGES) { stage = 0; ph ^= 1; }
      }
      float *dimg = dcol + (long long)b * HWo * g.Qp * TC_CB + (long long)rg * 4 * TC_CB + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pp = wgi * 64 + wq * 16 + (lane >> 2) + 8 * h;
        const int ho = ty0 + pp / s.tw, wo = tx0 + pp % s.tw;
        if (ho >= s.Ho || wo >= s.Wo) continue;
        float *dp = dimg + ((long long)ho * s.Wo + wo) * g.Qp * TC_CB;
#pragma unroll
        for (int j = 0; j < 16; ++j) *reinterpret_cast<float2 *>(dp + 8 * j) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------ dMask / dOffset (+ the dX scatter)
__device__ __forceinline__ void red_add_v4(float *addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d));
}
__device__ __forceinline__ float dot4(const float4 a, const float4 b) {
  return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)));
}

// dX contribution of one corner in deterministic mode: the fp32 products of the default scatter, each rounded to
// the nearest multiple of 1/qs (exact power-of-two scaling in double) and added as a two's-complement integer
__device__ __forceinline__ void red_add_s64(long long *addr, long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ void red_fixed4(long long *addr, const float4 dm, float wgt, double qs) {
  const long long v0 = __double2ll_rn((double)(dm.x * wgt) * qs), v1 = __double2ll_rn((double)(dm.y * wgt) * qs);
  const long long v2 = __double2ll_rn((double)(dm.z * wgt) * qs), v3 = __double2ll_rn((double)(dm.w * wgt) * qs);
  if (v0) red_add_s64(addr, v0);
  if (v1) red_add_s64(addr + 1, v1);
  if (v2) red_add_s64(addr + 2, v2);
  if (v3) red_add_s64(addr + 3, v3);
}

// Geometry of one (tap, pixel): fractional parts, mask and (hl*W + wl + W + 1) << 7 | flags
// (bit 0-3: corner in range, 4: sampling point inside (-1,H)x(-1,W), 5: pixel inside the output map).
struct __align__(16) BwdMetaTc {
  float lh, lw, m;
  int packed;
};
__device__ __forceinline__ BwdMetaTc bwd_meta(const DcnShapeTc &s, const float *__restrict__ off_img,
                                              const float *__restrict__ mask_img, int gi, int tap, int ho, int wo) {
  const int KT = s.kh * s.kw;
  const long long HWo = (long long)s.Ho * s.Wo;
  BwdMetaTc mt;
  mt.lh = mt.lw = mt.m = 0.f;
  mt.packed = 0;
  if (ho < s.Ho && wo < s.Wo && tap < KT) {
    const long long p = (long long)ho * s.Wo + wo;
    const int ki = tap / s.kw, kj = tap - ki * s.kw;
    const float *op = off_img + ((long long)gi * 2 * KT + 2 * tap) * HWo + p;
    const float dy = __ldg(op), dx = __ldg(op + HWo);
    mt.m = __ldg(mask_img + ((long long)gi * KT + tap) * HWo + p);
    const float h_im = (float)(ho * s.sh - s.ph + ki * s.dh) + dy;
    const float w_im = (float)(wo * s.sw - s.pw + kj * s.dw) + dx;
    int flags = 32;
    int base = 0;
    if (h_im > -1.f && w_im > -1.f && h_im < (float)s.H && w_im < (float)s.W) {   // dcn_v2_im2col_cuda.cu:286-289
      const float hf = floorf(h_im), wf = floorf(w_im);
      const int hl = (int)hf, wl = (int)wf;
      mt.lh = h_im - hf;
      mt.lw = w_im - wf;
      flags |= 16;
      if (hl >= 0 && wl >= 0) flags |= 1;
      if (hl >= 0 && wl + 1 <= s.W - 1) flags |= 2;
      if (hl + 1 <= s.H - 1 && wl >= 0) flags |= 4;
      if (hl + 1 <= s.H - 1 && wl + 1 <= s.W - 1) flags |= 8;
      base = hl * s.W + wl + s.W + 1;
    }
    mt.packed = (base << 7) | flags;
  }
  return mt;
}

// grid = images x pixel tiles, 8 warps.  Per deformable group the CTA first lays the geometry of its 9 x 128 sampling
// points into shared memory (every point computed once), then each warp walks (tap, 4 pixels) items with
// lane = (pixel j, 4-channel quad c4): 16-byte loads of the dcol line and of the four corner lines, next channel
// block in flight while the current one is reduced.
template <int MINB>
__global__ void __launch_bounds__(256, MINB)
k_dcn_bwd_offmask(const float *__restrict__ xt, const float *__restrict__ offset, const float *__restrict__ mask,
                  const float *__restrict__ dcol, float *__restrict__ dxt, float *__restrict__ goff,
                  float *__restrict__ gmask, long long *__restrict__ dxi, const unsigned *__restrict__ bnd,
                  const DcnShapeTc s, const BwdGeom g, const int b_first) {
  // dxt != NULL: every sample is scattered into the channels-last dX (16-byte reductions);
  // dxi != NULL (deterministic mode): into the fixed-point dX of the batch chunk [bl][HW][Cp] (scale from bnd)
  __shared__ BwdMetaTc meta[TC_NT * TC_TP];
  const int KT = s.kh * s.kw;
  const long long HWo = (long long)s.Ho * s.Wo, HW = (long long)s.H * s.W;
  const int Cp = s.nb * TC_CB;
  const int t = blockIdx.x % g.tiles, bl = blockIdx.x / g.tiles;   // bl: image within this batch chunk (dcol index)
  const int b = b_first + bl;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = lane >> 3, c4 = lane & 7;
  const int ty0 = (t / s.tiles_x) * s.th, tx0 = (t % s.tiles_x) * s.tw;
  const int tws = s.tw == 16 ? 4 : 3;                               // tile width is 16 or 8 (fill_shape)
  const float *off_img = offset + (long long)b * s.off_bs, *mask_img = mask + (long long)b * s.mask_bs;
  const float *x_img = xt + (long long)b * HW * Cp + c4 * 4;
  float *dx_img = dxt ? dxt + (long long)b * HW * Cp + c4 * 4 : nullptr;
  const double qs = dxi ? det_scale(bnd, s, g, b) : 0.0;     // 0: non-finite bounds, k_dcn_bwd_dx_fixed writes NaN
  long long *dxi_img = qs != 0.0 ? dxi + (long long)bl * HW * Cp + c4 * 4 : nullptr;
  const float *dc_img = dcol + (long long)bl * HWo * g.Qp * TC_CB + c4 * 4;
  float *gmask_img = gmask ? gmask + (long long)b * s.mask_bs : nullptr;
  float *goff_img = goff ? goff + (long long)b * s.off_bs : nullptr;
  const int xs1 = Cp, xs2 = s.W * Cp, xs3 = (s.W + 1) * Cp;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int gi = 0; gi < s.dg; ++gi) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < KT * TC_TP; idx += 256) {
      const int tap = idx >> 7, pp = idx & (TC_TP - 1);
      meta[idx] = bwd_meta(s, off_img, mask_img, gi, tap, ty0 + (pp >> tws), tx0 + (pp & (s.tw - 1)));
    }
    __syncthreads();
    const int cb0 = gi * s.cbs_pg;
    // This warp's items k = 0 .. 4 KT - 1: tap k / 4, pixels (warp + 8 (k % 4)) * 4 + j.  The five 16-byte loads of a
    // (item, channel block) step are issued one step ahead -- across the item boundary too -- so the only exposed
    // latency is the very first step's.
    const int n_items = KT * 4;
    struct Item { BwdMetaTc mt; int p, xo, dco; };
    auto item = [&](int k) {
      Item it;
      const int tap = k >> 2, pp = (warp + 8 * (k & 3)) * 4 + j;
      it.mt = meta[tap * TC_TP + pp];
      it.p = (ty0 + (pp >> tws)) * s.Wo + tx0 + (pp & (s.tw - 1));            // 32-bit offsets within one image (host-checked)
      it.xo = ((it.mt.packed >> 7) - (s.W + 1)) * Cp + cb0 * TC_CB;
      it.dco = (it.p * g.Qp + cb0 * TC_NT + tap) * TC_CB;
      return it;
    };
    float4 d, x1, x2, x3, x4;
    auto issue = [&](int flags, int xo, int dco) {      // a corner out of range (or a sample outside: all flags clear) is not loaded
      d = (flags & 16) ? __ldg(reinterpret_cast<const float4 *>(dc_img + dco)) : z4;
      x1 = (flags & 1) ? __ldg(reinterpret_cast<const float4 *>(x_img + xo)) : z4;
      x2 = (flags & 2) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs1))) : z4;
      x3 = (flags & 4) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs2))) : z4;
      x4 = (flags & 8) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs3))) : z4;
    };
    Item cur = item(0);
    issue(cur.mt.packed, cur.xo, cur.dco);
#pragma unroll 1
    for (int k = 0; k < n_items; ++k) {
      const int tap = k >> 2;
      Item nxt = cur;
      if (k + 1 < n_items) nxt = item(k + 1);
      const int flags = cur.mt.packed & 127;
      const bool f1 = flags & 1, f2 = flags & 2, f3 = flags & 4, f4 = flags & 8;
      const float lh = cur.mt.lh, lw = cur.mt.lw, hh = 1.f - lh, hw = 1.f - lw, m = cur.mt.m;
      const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
      int xo = cur.xo, dco = cur.dco;
      float am = 0.f, ah = 0.f, aw = 0.f;
#pragma unroll 1
      for (int cbi = 0; cbi < s.cbs_pg; ++cbi) {
        const float4 cd = d, c1 = x1, c2 = x2, c3 = x3, c4v = x4;
        if (cbi + 1 < s.cbs_pg) issue(flags, xo + TC_CB, dco + TC_NT * TC_CB);
        else if (k + 1 < n_items) issue(nxt.mt.packed, nxt.xo, nxt.dco);
        if (flags & 16) {
          // dMask (:297): dcol * unmasked bilinear sample
          float4 v;
          v.x = w1 * c1.x + w2 * c2.x + w3 * c3.x + w4 * c4v.x;
          v.y = w1 * c1.y + w2 * c2.y + w3 * c3.y + w4 * c4v.y;
          v.z = w1 * c1.z + w2 * c2.z + w3 * c3.z + w4 * c4v.z;
          v.w = w1 * c1.w + w2 * c2.w + w3 * c3.w + w4 * c4v.w;
          am += dot4(cd, v);
          // dOffset (:75-116, :299-302): dcol * mask * d(sample)/d{h,w}
          const float4 dm = make_float4(cd.x * m, cd.y * m, cd.z * m, cd.w * m);
          float4 gh, gw;
          gh.x = -hw * c1.x - lw * c2.x + hw * c3.x + lw * c4v.x;
          gh.y = -hw * c1.y - lw * c2.y + hw * c3.y + lw * c4v.y;
          gh.z = -hw * c1.z - lw * c2.z + hw * c3.z + lw * c4v.z;
          gh.w = -hw * c1.w - lw * c2.w + hw * c3.w + lw * c4v.w;
          gw.x = -hh * c1.x + hh * c2.x - lh * c3.x + lh * c4v.x;
          gw.y = -hh * c1.y + hh * c2.y - lh * c3.y + lh * c4v.y;
          gw.z = -hh * c1.z + hh * c2.z - lh * c3.z + lh * c4v.z;
          gw.w = -hh * c1.w + hh * c2.w - lh * c3.w + lh * c4v.w;
          ah += dot4(dm, gh);
          aw += dot4(dm, gw);
          // dX (:182-239): the four corners receive dcol * mask * corner weight
          if (dx_img) {
            if (f1 && w1 != 0.f) red_add_v4(dx_img + xo, dm.x * w1, dm.y * w1, dm.z * w1, dm.w * w1);
            if (f2 && w2 != 0.f) red_add_v4(dx_img + (xo + xs1), dm.x * w2, dm.y * w2, dm.z * w2, dm.w * w2);
            if (f3 && w3 != 0.f) red_add_v4(dx_img + (xo + xs2), dm.x * w3, dm.y * w3, dm.z * w3, dm.w * w3);
            if (f4 && w4 != 0.f) red_add_v4(dx_img + (xo + xs3), dm.x * w4, dm.y * w4, dm.z * w4, dm.w * w4);
          } else if (dxi_img) {
            if (f1 && w1 != 0.f) red_fixed4(dxi_img + xo, dm, w1, qs);
            if (f2 && w2 != 0.f) red_fixed4(dxi_img + (xo + xs1), dm, w2, qs);
            if (f3 && w3 != 0.f) red_fixed4(dxi_img + (xo + xs2), dm, w3, qs);
            if (f4 && w4 != 0.f) red_fixed4(dxi_img + (xo + xs3), dm, w4, qs);
          }
        }
        xo += TC_CB;
        dco += TC_NT * TC_CB;
      }
      // fixed-order reduction over the 8 channel quads of a pixel
#pragma unroll
      for (int sh = 4; sh > 0; sh >>= 1) {
        am += __shfl_xor_sync(0xffffffffu, am, sh);
        ah += __shfl_xor_sync(0xffffffffu, ah, sh);
        aw += __shfl_xor_sync(0xffffffffu, aw, sh);
      }
      // the gradients arrive zero-filled (dcn_v2_func.py:44-48) and every (tap, pixel) has exactly one writer:
      // a plain store is the accumulation
      if ((flags & 32) && c4 == 0) {
        const int go = (gi * KT + tap) * (int)HWo + cur.p;
        if (gmask_img) gmask_img[go] = am;
        if (goff_img) {
          goff_img[2 * go - cur.p] = ah;                 // channel 2 * (gi*KT + tap)
          goff_img[2 * go - cur.p + (int)HWo] = aw;
        }
      }
      cur = nxt;
    }
  }
}

// gx[b][ch][pos] += dxt[b][pos][slot(ch)]   (inverse of k_dcn_nhwc).  grid (pixel blocks of 32, channel blocks of 64, B)
__global__ void __launch_bounds__(256) k_dcn_bwd_dx_nchw(const float *__restrict__ dxt, float *__restrict__ gx,
                                                         const DcnShapeTc s) {
  __shared__ float tile[64][33];
  const long long HW = (long long)s.H * s.W;
  const long long p0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 64, b = blockIdx.z;
  const int Cp = s.nb * TC_CB, cpg = s.Cin / s.dg;
  {
    const int c = threadIdx.x & 63, pr = threadIdx.x >> 6;
    const int ch = c0 + c;
    if (ch < s.Cin) {
      const int gi = ch / cpg, within = ch - gi * cpg;
      const int slot = (gi * s.cbs_pg + within / TC_CB) * TC_CB + within % TC_CB;
      for (int px = pr; px < 32; px += 4)
        tile[c][px] = (p0 + px < HW) ? __ldg(dxt + ((long long)b * HW + p0 + px) * Cp + slot) : 0.f;
    }
  }
  __syncthreads();
  {
    const int px = threadIdx.x & 31, cr = threadIdx.x >> 5;
    for (int c = cr; c < 64; c += 8)
      if (c0 + c < s.Cin && p0 + px < HW) gx[((long long)b * s.Cin + c0 + c) * HW + p0 + px] += tile[c][px];
  }
}

// Deterministic mode: gx[b] += dxi[bl] / scale (fixed point -> fp32) for the images b = b_first + bl of a batch
// chunk; all NaN for an image whose bounds are not finite.  NCHW: as k_dcn_bwd_dx_nchw, grid (pixel blocks of 32,
// channel blocks of 64, images).  CL (channels-last grad_input, cin/dg % 32 == 0 so slot == channel): grid
// (pixel blocks of 32, 1, images), 8 warps x 4 pixels of whole channel lines.
template <bool CL>
__global__ void __launch_bounds__(256) k_dcn_bwd_dx_fixed(const long long *__restrict__ dxi,
                                                          const unsigned *__restrict__ bnd, float *__restrict__ gx,
                                                          const DcnShapeTc s, const BwdGeom g, const int b_first) {
  const long long HW = (long long)s.H * s.W;
  const long long p0 = (long long)blockIdx.x * 32;
  const int bl = blockIdx.z, b = b_first + bl;
  const int Cp = s.nb * TC_CB, cpg = s.Cin / s.dg;
  const double qs = det_scale(bnd, s, g, b);
  const double inv = qs != 0.0 ? 1.0 / qs : __longlong_as_double(0x7ff8000000000000ll);
  const long long *src = dxi + (long long)bl * HW * Cp;
  if (CL) {
    for (int i = threadIdx.x; i < 32 * Cp; i += 256) {
      const long long p = p0 + i / Cp;
      const int ch = i % Cp;
      if (p < HW) gx[((long long)b * HW + p) * Cp + ch] += (float)((double)__ldg(src + p * Cp + ch) * inv);
    }
    return;
  }
  __shared__ float tile[64][33];
  const int c0 = blockIdx.y * 64;
  {
    const int c = threadIdx.x & 63, pr = threadIdx.x >> 6;
    const int ch = c0 + c;
    if (ch < s.Cin) {
      const int gi = ch / cpg, within = ch - gi * cpg;
      const int slot = (gi * s.cbs_pg + within / TC_CB) * TC_CB + within % TC_CB;
      for (int px = pr; px < 32; px += 4)
        tile[c][px] = (p0 + px < HW) ? (float)((double)__ldg(src + (p0 + px) * Cp + slot) * inv) : 0.f;
    }
  }
  __syncthreads();
  {
    const int px = threadIdx.x & 31, cr = threadIdx.x >> 5;
    for (int c = cr; c < 64; c += 8)
      if (c0 + c < s.Cin && p0 + px < HW) gx[((long long)b * s.Cin + c0 + c) * HW + p0 + px] += tile[c][px];
  }
}

// ------------------------------------------------------------------ dW = dY . col^T   (K = pixels)
constexpr int WG_SAMPLERS = 8;                                // sampler warps, 4 tasks each (2 rounds of 2)
constexpr int WG_TASKS = 32 / WG_SAMPLERS;
constexpr int WG_GEOM = 4;                                    // warps 0-3: geometry producers (4 taps x 32 pixels per slice)
constexpr int WG_MR = 4;                                      // slices of geometry in flight
constexpr int WG_WARP_C0 = 4;                                 // warps 4-11: two consumer warpgroups (MMA + epilogue)
constexpr int WG_WARP_S0 = WG_WARP_C0 + 4 * TC_MMA_WGS;       // warps 12-19: samplers; lane 0 of warp 12 also issues the
                                                              // dY tile copies (TMA) of each stage it has seen drained
constexpr int WG_THREADS = (WG_WARP_S0 + WG_SAMPLERS) * 32;   // 640: leaves the consumers 96+ registers
constexpr uint32_t WG_SBO = 1040;                             // pitch of the A tile's 8-row groups (bank-conflict-free scalar stores)
constexpr int WG_A_BYTES = (TC_TP / 8) * WG_SBO;              // 16640 per hi / lo tile
constexpr int WG_STAGES = 3;

struct WgGeom {
  int co_r;          // Cout rounded up to 64, or to 128 above 64: a whole number of N tiles
  int nt;            // output channels per CTA (wgmma N): 64 or 128
  int n_nt;          // N tiles (CTAs per row group and split)
  int spi;           // 32-pixel slices per image
  int n_slices;      // B * spi
  int splits;        // pixel-range splits (CTAs per row group)
  int stages;
  int stage_bytes;   // 2 * WG_A_BYTES + 2 * nt * 128
  unsigned wo_magic; // floor(2^32 / Wo) + 1: p / Wo == umulhi(p, magic) for p < 2^32 / Wo; 0 = divide
};
static WgGeom wg_geom(const DcnShapeTc &s, const BwdGeom &g) {
  WgGeom w;
  w.co_r = s.Cout <= 64 ? 64 : (s.Cout + 127) / 128 * 128;
  w.nt = w.co_r == 64 ? 64 : 128;
  w.n_nt = w.co_r / w.nt;
  w.spi = (int)(((long long)s.Ho * s.Wo + TC_K - 1) / TC_K);
  w.n_slices = s.B * w.spi;
  int splits = num_sms() / (g.RG * w.n_nt);   // one CTA per SM at most (a CTA owns ~200 KB of shared memory): no second wave
  if (splits > w.n_slices) splits = w.n_slices;
  if (splits < 1) splits = 1;
  w.splits = splits;
  w.stage_bytes = 2 * WG_A_BYTES + 2 * w.nt * TC_K * 4;
  w.stages = WG_STAGES;
  w.wo_magic = ((unsigned long long)s.Ho * s.Wo * s.Wo < (1ull << 32)) ? (unsigned)((1ull << 32) / (unsigned)s.Wo + 1) : 0u;
  return w;
}

// dY [B][Cout][HWo] -> per (image, 32-pixel slice): [co_r rows = output channel][32 k = pixel], hi then lo.  grid (spi, B)
// A warp owns one output channel of the slice at a time, so the bias gradient's partial sums (dcn_v2_cuda.c:225-230)
// fall out of the same pass: bpart[slice][o] = sum of the 32 pixels, fixed shuffle order.
__global__ void __launch_bounds__(256) k_bwd_prep_gyk(const float *__restrict__ gy, const DcnShapeTc s, const WgGeom wg,
                                                      float *__restrict__ gyk, float *__restrict__ bpart) {
  const int sl = blockIdx.x, b = blockIdx.y;
  const long long HWo = (long long)s.Ho * s.Wo, p0 = (long long)sl * TC_K;
  const size_t tile = (size_t)wg.co_r * TC_K;
  unsigned char *hi = reinterpret_cast<unsigned char *>(gyk + ((size_t)b * wg.spi + sl) * 2 * tile);
  unsigned char *lo = hi + tile * 4;
  for (int i = threadIdx.x; i < wg.co_r * TC_K; i += blockDim.x) {
    const int k = i & (TC_K - 1), o = i >> 5;
    const float v = (o < s.Cout && p0 + k < HWo) ? __ldg(gy + ((long long)b * s.Cout + o) * HWo + p0 + k) : 0.f;
    const float h = tf32_hi(v);
    *reinterpret_cast<float *>(hi + tc_tile_off(o, k)) = h;
    *reinterpret_cast<float *>(lo + tc_tile_off(o, k)) = v - h;
    if (bpart) {
      float sum = v;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
      if (k == 0) bpart[((size_t)b * wg.spi + sl) * wg.co_r + o] = sum;
    }
  }
}

// gb[o] += sum over slices of bpart[slice][o]: strided per-thread sums, then a fixed tree.  grid = Cout
__global__ void __launch_bounds__(256) k_dcn_bwd_bias_reduce(const float *__restrict__ bpart, float *__restrict__ gb,
                                                             const WgGeom wg) {
  __shared__ float red[256];
  const int o = blockIdx.x;
  float sum = 0.f;
  for (int i = threadIdx.x; i < wg.n_slices; i += 256) sum += __ldg(bpart + (size_t)i * wg.co_r + o);
  red[threadIdx.x] = sum;
  __syncthreads();
  for (int d = 128; d > 0; d >>= 1) {
    if (threadIdx.x < d) red[threadIdx.x] += red[threadIdx.x + d];
    __syncthreads();
  }
  if (threadIdx.x == 0) gb[o] += red[0];
}

// CTA = (row group rg = 4 chunks x 32 channels, N tile, split): D[128 rows][NT output channels] accumulates over the
// CTA's slices in the registers of two consumer warpgroups (64 rows each).
template <int NT>
__global__ void __launch_bounds__(WG_THREADS, 1)
k_dcn_bwd_weight_tc(const float *__restrict__ xt, const float *__restrict__ offset, const float *__restrict__ mask,
                    const float *__restrict__ gyk, float *__restrict__ wpart, const DcnShapeTc s, const BwdGeom g,
                    const WgGeom wg) {
  extern __shared__ __align__(128) unsigned char tc_smem[];
  __shared__ __align__(8) uint64_t a_full[WG_STAGES], b_full[WG_STAGES], empty[WG_STAGES], m_full[WG_MR], m_empty[WG_MR];
  __shared__ BwdMetaTc wmeta[WG_MR][128];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rg = blockIdx.x % g.RG, nti = (blockIdx.x / g.RG) % wg.n_nt, split = blockIdx.x / g.RG / wg.n_nt;
  const int sl0 = (int)((long long)split * wg.n_slices / wg.splits), sl1 = (int)((long long)(split + 1) * wg.n_slices / wg.splits);
  const int KT = s.kh * s.kw;
  const long long HWo = (long long)s.Ho * s.Wo, HW = (long long)s.H * s.W;
  const int Cp = s.nb * TC_CB;
  const int b_bytes = NT * TC_K * 4;                 // the CTA's N tile of one hi or lo dY tile

  if (tid == 0) {
    for (int i = 0; i < WG_STAGES; ++i) {
      mbar_init(&a_full[i], WG_SAMPLERS);
      mbar_init(&b_full[i], 1);
      mbar_init(&empty[i], TC_MMA_WGS);
    }
    for (int i = 0; i < WG_MR; ++i) { mbar_init(&m_full[i], WG_GEOM); mbar_init(&m_empty[i], WG_SAMPLERS); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= WG_WARP_S0) {
    // =========================================================== samplers: the masked column tile, rows = channels
    // task = (chunk ql, 4 pixels): lane = (pixel j, channel quad c4) gathers 4 corners x 16 bytes and stores its
    // 4 channels x 1 pixel as scalars -- the 8-row groups of the A tile are pitched WG_SBO = 1040 bytes so that the 32
    // lanes of a store hit 32 different banks.  Warps run free of each other: the geometry comes through a ring, the
    // tile goes out through the 3-stage A ring.  A warp's WG_TASKS tasks run in rounds of two.
    const int sw = warp - WG_WARP_S0;
    const int j = lane >> 3, c4 = lane & 7;
    int t_meta[WG_TASKS], t_xc[WG_TASKS];
    uint32_t t_dst[WG_TASKS];
#pragma unroll
    for (int it = 0; it < WG_TASKS; ++it) {
      const int task = sw + it * WG_SAMPLERS;      // chunk ql = task / 8, pixel group pg = task % 8
      const int ql = task >> 3, pg = task & 7;
      const int q = rg * 4 + ql;
      const int bi = q < g.Q ? q / TC_NT : 0;
      t_meta[it] = ql * 32 + pg * 4 + j;
      t_xc[it] = bi * TC_CB + c4 * 4;
      const int row = ql * 32 + c4 * 4;            // + i (i < 4 stays inside one 8-row group)
      t_dst[it] = (uint32_t)(row >> 3) * WG_SBO + (uint32_t)pg * TC_LBO + (uint32_t)(row & 7) * 16u + (uint32_t)j * 4u;
    }
    const int xs1 = Cp, xs2 = s.W * Cp, xs3 = (s.W + 1) * Cp;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    int stage = 0, ph = 0, ms = 0, mph = 0;
    int b = sl0 / wg.spi, sll = sl0 - b * wg.spi;      // image and slice within the image
    const size_t tile_bytes = (size_t)wg.co_r * TC_K * 4;          // one hi or lo dY tile, all output channels
    for (int sl = sl0; sl < sl1; ++sl) {
      // take the geometry of the slice from the ring (a corner that is out of range, or a sample that is outside
      // altogether -- all four flags clear, weights zero -- is simply not loaded)
      mbar_wait(&m_full[ms], (uint32_t)mph);
      BwdMetaTc mt[WG_TASKS];
#pragma unroll
      for (int it = 0; it < WG_TASKS; ++it) mt[it] = wmeta[ms][t_meta[it]];
      __syncwarp();
      if (lane == 0) mbar_arrive_tc(&m_empty[ms]);
      if (++ms == WG_MR) { ms = 0; mph ^= 1; }
      const float *x_img = xt + (long long)b * HW * Cp;
      unsigned char *a_hi = tc_smem + (size_t)stage * wg.stage_bytes;
      unsigned char *a_lo = a_hi + WG_A_BYTES;
#pragma unroll
      for (int r = 0; r < WG_TASKS; r += 2) {
        float4 xc[2][4];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int flags = mt[r + u].packed;
          const int xo = ((flags >> 7) - (s.W + 1)) * Cp + t_xc[r + u];
          xc[u][0] = (flags & 1) ? __ldg(reinterpret_cast<const float4 *>(x_img + xo)) : z4;
          xc[u][1] = (flags & 2) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs1))) : z4;
          xc[u][2] = (flags & 4) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs2))) : z4;
          xc[u][3] = (flags & 8) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs3))) : z4;
        }
        if (r == 0) {
          mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));
          if (sw == 0 && lane == 0) {
            // B operand: rows nti*NT .. nti*NT + NT - 1 of the slice's hi and lo dY tiles (8-row groups are contiguous,
            // 128 bytes a row)
            unsigned char *dst = a_hi + 2 * WG_A_BYTES;
            const unsigned char *src = reinterpret_cast<const unsigned char *>(gyk) + (size_t)sl * 2 * tile_bytes +
                                       (size_t)nti * NT * TC_K * 4;
            mbar_expect_tx(&b_full[stage], 2u * (uint32_t)b_bytes);
            for (uint32_t off = 0; off < (uint32_t)b_bytes; off += 2048u) {
              bulk_g2s(dst + off, src + off, 2048u, &b_full[stage]);
              bulk_g2s(dst + b_bytes + off, src + tile_bytes + off, 2048u, &b_full[stage]);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const BwdMetaTc &m = mt[r + u];
          const float lh = m.lh, lw = m.lw, mm = m.m, hh = 1.f - lh, hw = 1.f - lw;
          const float w1 = hh * hw * mm, w2 = hh * lw * mm, w3 = lh * hw * mm, w4 = lh * lw * mm;   // as the forward sampler
          const float4 x1 = xc[u][0], x2 = xc[u][1], x3 = xc[u][2], x4 = xc[u][3];
          float4 v;
          v.x = fmaf(w4, x4.x, fmaf(w3, x3.x, fmaf(w2, x2.x, w1 * x1.x)));
          v.y = fmaf(w4, x4.y, fmaf(w3, x3.y, fmaf(w2, x2.y, w1 * x1.y)));
          v.z = fmaf(w4, x4.z, fmaf(w3, x3.z, fmaf(w2, x2.z, w1 * x1.z)));
          v.w = fmaf(w4, x4.w, fmaf(w3, x3.w, fmaf(w2, x2.w, w1 * x1.w)));
          const float4 h4 = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
          float *dh = reinterpret_cast<float *>(a_hi + t_dst[r + u]), *dl = reinterpret_cast<float *>(a_lo + t_dst[r + u]);
          dh[0] = h4.x; dh[4] = h4.y; dh[8] = h4.z; dh[12] = h4.w;                          // rows c4*4 + 0..3: 16 bytes apart
          dl[0] = v.x - h4.x; dl[4] = v.y - h4.y; dl[8] = v.z - h4.z; dl[12] = v.w - h4.w;
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive_tc(&a_full[stage]);
      if (++stage == wg.stages) { stage = 0; ph ^= 1; }
      if (++sll == wg.spi) { sll = 0; ++b; }
    }
  } else if (warp >= WG_WARP_C0) {
    // =========================================================== consumers: warpgroup cw accumulates rows 64 cw .. 64 cw + 63
    const int cw = (warp - WG_WARP_C0) >> 2, wq = warp & 3;
    float d[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) d[i] = 0.f;
    int stage = 0, ph = 0;
    for (int sl = sl0; sl < sl1; ++sl) {
      mbar_wait(&a_full[stage], (uint32_t)ph);
      mbar_wait(&b_full[stage], (uint32_t)ph);
      const uint32_t base = smem_u32(tc_smem + (size_t)stage * wg.stage_bytes);
      const uint32_t ah = base + (uint32_t)cw * 8u * WG_SBO, al = ah + WG_A_BYTES;
      const uint32_t bh = base + 2u * WG_A_BYTES, bl = bh + (uint32_t)b_bytes;
      wgmma_fence();
#pragma unroll
      for (int k8 = 0; k8 < TC_K / 8; ++k8) {
        const uint32_t koff = (uint32_t)k8 * 2u * TC_LBO;
        wgmma_3xtf32<NT>(d, wg_desc(ah + koff, TC_LBO, WG_SBO), wg_desc(al + koff, TC_LBO, WG_SBO), tc_desc(bh + koff),
                         tc_desc(bl + koff), (sl > sl0 || k8 > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait_all();
      if (((tid - WG_WARP_C0 * 32) & 127) == 0) mbar_arrive_tc(&empty[stage]);
      if (++stage == wg.stages) { stage = 0; ph ^= 1; }
    }
    // epilogue: wpart[split][rg][row][co_r], columns nti*NT .. nti*NT + NT - 1 (zeros for a CTA without slices)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
      float *dst = wpart + (((size_t)split * g.RG + rg) * 128 + row) * wg.co_r + nti * NT + 2 * (lane & 3);
#pragma unroll
      for (int jj = 0; jj < NT / 8; ++jj)
        *reinterpret_cast<float2 *>(dst + 8 * jj) = make_float2(d[4 * jj + 2 * h], d[4 * jj + 2 * h + 1]);
    }
  } else {
    // =========================================================== warps 0-3 produce the geometry: 4 taps x 32 pixels of a slice, one
    // entry per thread, WG_MR slices ahead of the samplers (ring in shared memory, mbarrier hand-over); the offsets and
    // mask of the next slice are fetched before the current entry is finished
    const int st = tid;
    const int m_q = rg * 4 + (st >> 5);
    const int m_bi = m_q / TC_NT, m_tap = m_q < g.Q ? m_q - m_bi * TC_NT : TC_NT;     // TC_NT = "no such tap"
    const int m_gi = m_bi / s.cbs_pg;
    const bool m_ok = m_tap < KT;
    const int ki = m_ok ? m_tap / s.kw : 0, kj = m_tap - ki * s.kw;
    const int hb = ki * s.dh - s.ph, wb = kj * s.dw - s.pw;
    const long long o_dy = ((long long)m_gi * 2 * KT + 2 * (m_ok ? m_tap : 0)) * HWo, o_m = ((long long)m_gi * KT + (m_ok ? m_tap : 0)) * HWo;
    const int HWo_i = (int)HWo;
    int b = sl0 / wg.spi, sll = sl0 - b * wg.spi;
    float dy = 0.f, dx = 0.f, mk = 0.f;
    auto fetch = [&](int bb, int sl_local) {
      const int p = sl_local * TC_K + (st & 31);
      dy = dx = mk = 0.f;
      if (m_ok && p < HWo_i) {
        const float *op = offset + (long long)bb * s.off_bs + o_dy + p;
        dy = __ldg(op);
        dx = __ldg(op + HWo);
        mk = __ldg(mask + (long long)bb * s.mask_bs + o_m + p);
      }
    };
    if (sl0 < sl1) fetch(b, sll);
    int ms = 0, mph = 0;
    for (int sl = sl0; sl < sl1; ++sl) {
      const float cdy = dy, cdx = dx, cm = mk;
      const int p = sll * TC_K + (st & 31);
      int nb_ = b, nsl = sll + 1;
      if (nsl == wg.spi) { nsl = 0; ++nb_; }
      if (sl + 1 < sl1) fetch(nb_, nsl);
      BwdMetaTc mt;
      mt.lh = mt.lw = mt.m = 0.f;
      mt.packed = 0;
      if (m_ok && p < HWo_i) {
        const int ho = wg.wo_magic ? (int)__umulhi((unsigned)p, wg.wo_magic) : p / s.Wo;
        const int wo = p - ho * s.Wo;
        const float h_im = (float)(ho * s.sh + hb) + cdy, w_im = (float)(wo * s.sw + wb) + cdx;
        if (h_im > -1.f && w_im > -1.f && h_im < (float)s.H && w_im < (float)s.W) {     // dcn_v2_im2col_cuda.cu:165
          const float hf = floorf(h_im), wf = floorf(w_im);
          const int hl = (int)hf, wl = (int)wf;
          int flags = 16;
          if (hl >= 0 && wl >= 0) flags |= 1;
          if (hl >= 0 && wl + 1 <= s.W - 1) flags |= 2;
          if (hl + 1 <= s.H - 1 && wl >= 0) flags |= 4;
          if (hl + 1 <= s.H - 1 && wl + 1 <= s.W - 1) flags |= 8;
          mt.lh = h_im - hf;
          mt.lw = w_im - wf;
          mt.m = cm;
          mt.packed = ((hl * s.W + wl + s.W + 1) << 7) | flags;
        }
      }
      mbar_wait(&m_empty[ms], (uint32_t)(mph ^ 1));
      wmeta[ms][st] = mt;
      __syncwarp();
      if (lane == 0) mbar_arrive_tc(&m_full[ms]);
      if (++ms == WG_MR) { ms = 0; mph ^= 1; }
      b = nb_;
      sll = nsl;
    }
  }
}

// gw[o][ch][tap] += sum over splits (ascending) of wpart[split][rg][row][o]
__global__ void __launch_bounds__(256) k_dcn_bwd_wreduce(const float *__restrict__ wpart, float *__restrict__ gw,
                                                         const DcnShapeTc s, const BwdGeom g, const WgGeom wg) {
  const int KT = s.kh * s.kw, cpg = s.Cin / s.dg;
  const long long total = (long long)g.RG * 128 * wg.co_r;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i % wg.co_r);
    const int row = (int)((i / wg.co_r) % 128), rg = (int)(i / ((long long)wg.co_r * 128));
    const int q = rg * 4 + (row >> 5), ch = row & 31;
    const int bi = q / TC_NT, tap = q - bi * TC_NT;
    const int gi = bi / s.cbs_pg, cw = (bi - gi * s.cbs_pg) * TC_CB + ch;
    if (q >= g.Q || o >= s.Cout || cw >= cpg || tap >= KT) continue;
    float acc = 0.f;
    for (int sp = 0; sp < wg.splits; ++sp) acc += __ldg(wpart + (size_t)sp * total + i);
    gw[((size_t)o * s.Cin + gi * cpg + cw) * KT + tap] += acc;
  }
}

// =====================================================================================================================
// bf16 backward (opt-in, cnb_dcnv2_backward_bf16): both contractions on wgmma m64nNk16 .f32.bf16.bf16, one bf16 tile
// per operand where the passes above use a TF32 hi/lo pair.  With W_b = bf16(W) and dY_b = bf16(dY) (RN; exact for a
// bf16 grad_output):
//   dcol = sum_o W_b dY_b  (exact products, fp32 sums), stored fp32 in the layout above, so that k_dcn_bwd_offmask, the
//          dX scatter (atomics or fixed point), k_dcn_bwd_dx_nchw and k_dcn_bwd_dx_fixed run unchanged;
//   dW   = sum_p bf16(col) dY_b, col the masked bilinear value of the forward sampler (same fmaf chain) rounded RN as
//          k_dcn_forward_bf16 rounds it; per-CTA partials added by k_dcn_bwd_wreduce in split order;
//   dBias  sums grad_output as given, in the order of k_bwd_prep_gyk and k_dcn_bwd_bias_reduce.
constexpr int BB_TILE_BYTES = TC_TP * TC_K * 2;    // one bf16 tile [128 rows][32 k], dense K-major (bf_tile_off): 8 KB
constexpr int BB_STAGES = 4;
constexpr int BB_STAGE_BYTES = 2 * BB_TILE_BYTES;  // column-gradient stage: dY tile + W tile, 16 KB
constexpr uint32_t WB_SBO = 528;                   // weight pass A tile: 8-row groups 512 + 16 bytes apart (DESIGN 4.4.3)
constexpr int WB_A_BYTES = (TC_TP / 8) * WB_SBO;   // 8448
constexpr int WB_STAGES = 4;

__device__ __forceinline__ float ld_f32(const float *p) { return __ldg(p); }
__device__ __forceinline__ float ld_f32(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }

// W -> per (row group rg, slice ks) one bf16 tile [128 rows = (chunk ql, ch)][32 k = output channel], the rows and
// zero fill of k_bwd_prep_w.  DET: bnd[ks] from |W_b|.
template <bool DET>
__global__ void __launch_bounds__(256) k_bwd_prep_w_bf16(const float *__restrict__ w, const DcnShapeTc s,
                                                         const BwdGeom g, unsigned char *__restrict__ wtb,
                                                         unsigned *__restrict__ bnd) {
  const int KT = s.kh * s.kw, cpg = s.Cin / s.dg;
  const int rg = blockIdx.x / g.KS, ks = blockIdx.x - rg * g.KS;
  unsigned char *tile = wtb + (size_t)blockIdx.x * BB_TILE_BYTES;
  unsigned rmax = 0;
  for (int i = threadIdx.x; i < TC_TP * TC_K; i += blockDim.x) {
    const int k = i & (TC_K - 1), row = i >> 5;
    const int q = rg * 4 + (row >> 5), ch = row & 31;
    const int bi = q / TC_NT, tap = q - bi * TC_NT;
    const int gi = bi / s.cbs_pg, cw = (bi - gi * s.cbs_pg) * TC_CB + ch;
    const int o = ks * TC_K + k;
    float v = 0.f;
    if (q < g.Q && o < s.Cout && cw < cpg && tap < KT) v = __ldg(w + ((size_t)o * s.Cin + gi * cpg + cw) * KT + tap);
    const __nv_bfloat16 vb = __float2bfloat16_rn(v);
    *reinterpret_cast<__nv_bfloat16 *>(tile + bf_tile_off(row, k)) = vb;
    if (DET) {
      float sum = fabsf(__bfloat162float(vb));
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
      rmax = max(rmax, abs_bits(sum));
    }
  }
  if (DET && (threadIdx.x & 31) == 0) atomicMax(bnd + ks, rmax);
}

// dY [B][Cout][HWo] (fp32 or bf16) -> per (image, pixel tile, slice ks) one bf16 tile [128 px][32 k = output channel].
// grid (tiles, KS, B); a thread rounds 16 output channels of one pixel into two 16-byte k-chunks.  DET: the bounds of
// k_bwd_prep_gy, max |dY_b| and max |mask|.
template <typename T, bool DET>
__global__ void __launch_bounds__(256) k_bwd_prep_gy_bf16(const T *__restrict__ gy, const DcnShapeTc s, const BwdGeom g,
                                                          unsigned char *__restrict__ gyt, const float *__restrict__ mask,
                                                          unsigned *__restrict__ bnd_img) {
  const int t = blockIdx.x, ks = blockIdx.y, b = blockIdx.z;
  const int pp = threadIdx.x & (TC_TP - 1), half = threadIdx.x >> 7;
  const int ho = (t / s.tiles_x) * s.th + pp / s.tw, wo = (t % s.tiles_x) * s.tw + pp % s.tw;
  const bool ok = ho < s.Ho && wo < s.Wo;
  const long long HWo = (long long)s.Ho * s.Wo, p = (long long)ho * s.Wo + wo;
  unsigned char *tile = gyt + ((size_t)((size_t)b * g.tiles + t) * g.KS + ks) * BB_TILE_BYTES;
  unsigned ymax = 0;
#pragma unroll
  for (int kc = 0; kc < 2; ++kc) {
    const int k0 = half * 16 + kc * 8;
    uint32_t r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = ks * TC_K + k0 + 2 * j;
      const float v0 = (ok && o < s.Cout) ? ld_f32(gy + ((long long)b * s.Cout + o) * HWo + p) : 0.f;
      const float v1 = (ok && o + 1 < s.Cout) ? ld_f32(gy + ((long long)b * s.Cout + o + 1) * HWo + p) : 0.f;
      const __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1);   // v0 at the lower address
      r[j] = *reinterpret_cast<const uint32_t *>(&h);
      if (DET) ymax = max(ymax, max(abs_bits(__low2float(h)), abs_bits(__high2float(h))));
    }
    *reinterpret_cast<uint4 *>(tile + bf_tile_off(pp, k0)) = make_uint4(r[0], r[1], r[2], r[3]);
  }
  if (DET) {
    unsigned mmax = 0;
    if (ks == 0 && ok) {
      const float *mp = mask + (long long)b * s.mask_bs + p;
      for (int c = half; c < s.dg * s.kh * s.kw; c += 2) mmax = max(mmax, abs_bits(__ldg(mp + (long long)c * HWo)));
    }
    ymax = warp_max_u32(ymax);
    mmax = warp_max_u32(mmax);
    if ((threadIdx.x & 31) == 0) {
      atomicMax(bnd_img + 2 * b, ymax);
      if (mmax) atomicMax(bnd_img + 2 * b + 1, mmax);
    }
  }
}

// dcol = dY_b^T . W_b: k_dcn_bwd_dcol_tc with a 16 KB stage (one bf16 tile each of dY and W) and two k16 steps a slice
__global__ void __launch_bounds__(BW_THREADS, 1)
k_dcn_bwd_dcol_bf16(const unsigned char *__restrict__ gyt, const unsigned char *__restrict__ wtb,
                    float *__restrict__ dcol, const DcnShapeTc s, const BwdGeom g, const int n_items) {
  extern __shared__ __align__(128) unsigned char tc_smem[];
  __shared__ __align__(8) uint64_t full[BB_STAGES], empty[BB_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < BB_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TC_MMA_WGS); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == TC_WARP_TMA) {
    if (lane == 0) {
      int stage = 0, ph = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int rg = item % g.RG, bt = item / g.RG;          // bt = image * tiles + tile
        for (int ks = 0; ks < g.KS; ++ks) {
          mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));
          unsigned char *dst = tc_smem + (size_t)stage * BB_STAGE_BYTES;
          mbar_expect_tx(&full[stage], (uint32_t)BB_STAGE_BYTES);
          bulk_g2s(dst, gyt + ((size_t)bt * g.KS + ks) * BB_TILE_BYTES, (uint32_t)BB_TILE_BYTES, &full[stage]);
          bulk_g2s(dst + BB_TILE_BYTES, wtb + ((size_t)rg * g.KS + ks) * BB_TILE_BYTES, (uint32_t)BB_TILE_BYTES,
                   &full[stage]);
          if (++stage == BB_STAGES) { stage = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp < TC_WARP_TMA) {
    // consumers and epilogue as k_dcn_bwd_dcol_tc: warpgroup wgi owns pixels 64 wgi .. 64 wgi + 63 of the tile
    const int wgi = warp >> 2, wq = warp & 3;
    const long long HWo = (long long)s.Ho * s.Wo;
    int stage = 0, ph = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int rg = item % g.RG, bt = item / g.RG;
      const int t = bt % g.tiles, b = bt / g.tiles;
      const int ty0 = (t / s.tiles_x) * s.th, tx0 = (t % s.tiles_x) * s.tw;
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      for (int ks = 0; ks < g.KS; ++ks) {
        mbar_wait(&full[stage], (uint32_t)ph);
        const uint32_t base = smem_u32(tc_smem + (size_t)stage * BB_STAGE_BYTES);
        const uint32_t a = base + (uint32_t)wgi * 8u * BF_B_SBO, bw = base + (uint32_t)BB_TILE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < TC_K / 16; ++kk) {   // one k16 step = two 16-byte k-chunks
          const uint32_t koff = (uint32_t)kk * 2u * BF_B_LBO;
          wgmma_bf16<128>(d, wg_desc(a + koff, BF_B_LBO, BF_B_SBO), wg_desc(bw + koff, BF_B_LBO, BF_B_SBO),
                          (ks > 0 || kk > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        if ((tid & 127) == 0) mbar_arrive_tc(&empty[stage]);
        if (++stage == BB_STAGES) { stage = 0; ph ^= 1; }
      }
      float *dimg = dcol + (long long)b * HWo * g.Qp * TC_CB + (long long)rg * 4 * TC_CB + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pp = wgi * 64 + wq * 16 + (lane >> 2) + 8 * h;
        const int ho = ty0 + pp / s.tw, wo = tx0 + pp % s.tw;
        if (ho >= s.Ho || wo >= s.Wo) continue;
        float *dp = dimg + ((long long)ho * s.Wo + wo) * g.Qp * TC_CB;
#pragma unroll
        for (int j = 0; j < 16; ++j) *reinterpret_cast<float2 *>(dp + 8 * j) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
      }
    }
  }
}

// dY (fp32 or bf16) -> per (image, 32-pixel slice) one bf16 tile [co_r rows = output channel][32 k = pixel]; the bias
// partials bpart exactly as k_bwd_prep_gyk makes them (the same values, lanes and shuffle order).  grid (spi, B)
template <typename T>
__global__ void __launch_bounds__(256) k_bwd_prep_gyk_bf16(const T *__restrict__ gy, const DcnShapeTc s,
                                                           const WgGeom wg, unsigned char *__restrict__ gyk,
                                                           float *__restrict__ bpart) {
  const int sl = blockIdx.x, b = blockIdx.y;
  const long long HWo = (long long)s.Ho * s.Wo, p0 = (long long)sl * TC_K;
  unsigned char *tile = gyk + ((size_t)b * wg.spi + sl) * wg.co_r * TC_K * 2;
  for (int i = threadIdx.x; i < wg.co_r * TC_K; i += blockDim.x) {
    const int k = i & (TC_K - 1), o = i >> 5;
    const float v = (o < s.Cout && p0 + k < HWo) ? ld_f32(gy + ((long long)b * s.Cout + o) * HWo + p0 + k) : 0.f;
    *reinterpret_cast<__nv_bfloat16 *>(tile + bf_tile_off(o, k)) = __float2bfloat16_rn(v);
    if (bpart) {
      float sum = v;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
      if (k == 0) bpart[((size_t)b * wg.spi + sl) * wg.co_r + o] = sum;
    }
  }
}

// The geometry warps of the bf16 weight pass: the producer loop of k_dcn_bwd_weight_tc (which keeps it inline -- called
// through this function, that kernel's registers are allocated differently), 4 taps x 32 pixels of a slice, one entry
// per thread, WG_MR slices ahead of the samplers
__device__ __forceinline__ void wg_geometry(const DcnShapeTc &s, const BwdGeom &g, const WgGeom &wg, int rg, int sl0,
                                            int sl1, const float *__restrict__ offset, const float *__restrict__ mask,
                                            int st, BwdMetaTc (*wmeta)[128], uint64_t *m_full, uint64_t *m_empty) {
  const int KT = s.kh * s.kw, lane = st & 31;
  const long long HWo = (long long)s.Ho * s.Wo;
  const int m_q = rg * 4 + (st >> 5);
  const int m_bi = m_q / TC_NT, m_tap = m_q < g.Q ? m_q - m_bi * TC_NT : TC_NT;     // TC_NT = "no such tap"
  const int m_gi = m_bi / s.cbs_pg;
  const bool m_ok = m_tap < KT;
  const int ki = m_ok ? m_tap / s.kw : 0, kj = m_tap - ki * s.kw;
  const int hb = ki * s.dh - s.ph, wb = kj * s.dw - s.pw;
  const long long o_dy = ((long long)m_gi * 2 * KT + 2 * (m_ok ? m_tap : 0)) * HWo;
  const long long o_m = ((long long)m_gi * KT + (m_ok ? m_tap : 0)) * HWo;
  const int HWo_i = (int)HWo;
  int b = sl0 / wg.spi, sll = sl0 - b * wg.spi;
  float dy = 0.f, dx = 0.f, mk = 0.f;
  auto fetch = [&](int bb, int sl_local) {
    const int p = sl_local * TC_K + lane;
    dy = dx = mk = 0.f;
    if (m_ok && p < HWo_i) {
      const float *op = offset + (long long)bb * s.off_bs + o_dy + p;
      dy = __ldg(op);
      dx = __ldg(op + HWo);
      mk = __ldg(mask + (long long)bb * s.mask_bs + o_m + p);
    }
  };
  if (sl0 < sl1) fetch(b, sll);
  int ms = 0, mph = 0;
  for (int sl = sl0; sl < sl1; ++sl) {
    const float cdy = dy, cdx = dx, cm = mk;
    const int p = sll * TC_K + lane;
    int nb_ = b, nsl = sll + 1;
    if (nsl == wg.spi) { nsl = 0; ++nb_; }
    if (sl + 1 < sl1) fetch(nb_, nsl);
    BwdMetaTc mt;
    mt.lh = mt.lw = mt.m = 0.f;
    mt.packed = 0;
    if (m_ok && p < HWo_i) {
      const int ho = wg.wo_magic ? (int)__umulhi((unsigned)p, wg.wo_magic) : p / s.Wo;
      const int wo = p - ho * s.Wo;
      const float h_im = (float)(ho * s.sh + hb) + cdy, w_im = (float)(wo * s.sw + wb) + cdx;
      if (h_im > -1.f && w_im > -1.f && h_im < (float)s.H && w_im < (float)s.W) {
        const float hf = floorf(h_im), wf = floorf(w_im);
        const int hl = (int)hf, wl = (int)wf;
        int flags = 16;
        if (hl >= 0 && wl >= 0) flags |= 1;
        if (hl >= 0 && wl + 1 <= s.W - 1) flags |= 2;
        if (hl + 1 <= s.H - 1 && wl >= 0) flags |= 4;
        if (hl + 1 <= s.H - 1 && wl + 1 <= s.W - 1) flags |= 8;
        mt.lh = h_im - hf;
        mt.lw = w_im - wf;
        mt.m = cm;
        mt.packed = ((hl * s.W + wl + s.W + 1) << 7) | flags;
      }
    }
    mbar_wait(&m_empty[ms], (uint32_t)(mph ^ 1));
    wmeta[ms][st] = mt;
    __syncwarp();
    if (lane == 0) mbar_arrive_tc(&m_full[ms]);
    if (++ms == WG_MR) { ms = 0; mph ^= 1; }
    b = nb_;
    sll = nsl;
  }
}

// dW = dY_b . bf16(col)^T: the warp roles, work split and epilogue of k_dcn_bwd_weight_tc.  The samplers round each
// interpolated value once to bf16 and store it as a 2-byte scalar into the K-major A tile [128 rows = channels][32 k =
// pixels]; its 8-row groups are pitched WB_SBO = 528 bytes so that the 32 lanes of a store (4 pixels x 8 channel
// quads) hit 16 different 4-byte words, two lanes each (DESIGN 4.4.3).  The B tile (NT rows of the slice's dY tile) is
// dense and arrives by TMA.
template <int NT>
__global__ void __launch_bounds__(WG_THREADS, 1)
k_dcn_bwd_weight_bf16(const float *__restrict__ xt, const float *__restrict__ offset, const float *__restrict__ mask,
                      const unsigned char *__restrict__ gyk, float *__restrict__ wpart, const DcnShapeTc s,
                      const BwdGeom g, const WgGeom wg) {
  constexpr int B_BYTES = NT * TC_K * 2;
  constexpr int STAGE_BYTES = WB_A_BYTES + B_BYTES;
  extern __shared__ __align__(128) unsigned char tc_smem[];
  __shared__ __align__(8) uint64_t a_full[WB_STAGES], b_full[WB_STAGES], empty[WB_STAGES], m_full[WG_MR], m_empty[WG_MR];
  __shared__ BwdMetaTc wmeta[WG_MR][128];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rg = blockIdx.x % g.RG, nti = (blockIdx.x / g.RG) % wg.n_nt, split = blockIdx.x / g.RG / wg.n_nt;
  const int sl0 = (int)((long long)split * wg.n_slices / wg.splits), sl1 = (int)((long long)(split + 1) * wg.n_slices / wg.splits);
  const long long HW = (long long)s.H * s.W;
  const int Cp = s.nb * TC_CB;

  if (tid == 0) {
    for (int i = 0; i < WB_STAGES; ++i) {
      mbar_init(&a_full[i], WG_SAMPLERS);
      mbar_init(&b_full[i], 1);
      mbar_init(&empty[i], TC_MMA_WGS);
    }
    for (int i = 0; i < WG_MR; ++i) { mbar_init(&m_full[i], WG_GEOM); mbar_init(&m_empty[i], WG_SAMPLERS); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= WG_WARP_S0) {
    // =========================================================== samplers: task = (chunk ql, 4 pixels), lane = (pixel j,
    // channel quad c4), as in k_dcn_bwd_weight_tc
    const int sw = warp - WG_WARP_S0;
    const int j = lane >> 3, c4 = lane & 7;
    int t_meta[WG_TASKS], t_xc[WG_TASKS];
    uint32_t t_dst[WG_TASKS];
#pragma unroll
    for (int it = 0; it < WG_TASKS; ++it) {
      const int task = sw + it * WG_SAMPLERS;
      const int ql = task >> 3, pg = task & 7;
      const int q = rg * 4 + ql;
      const int bi = q < g.Q ? q / TC_NT : 0;
      t_meta[it] = ql * 32 + pg * 4 + j;
      t_xc[it] = bi * TC_CB + c4 * 4;
      const int row = ql * 32 + c4 * 4, k = pg * 4 + j;     // + i for channel i < 4: the next 16 bytes, same row group
      t_dst[it] = (uint32_t)(row >> 3) * WB_SBO + (uint32_t)(k >> 3) * BF_B_LBO + (uint32_t)(row & 7) * 16u +
                  (uint32_t)(k & 7) * 2u;
    }
    const int xs1 = Cp, xs2 = s.W * Cp, xs3 = (s.W + 1) * Cp;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    int stage = 0, ph = 0, ms = 0, mph = 0;
    int b = sl0 / wg.spi, sll = sl0 - b * wg.spi;
    const size_t tile_bytes = (size_t)wg.co_r * TC_K * 2;          // one dY tile, all output channels
    for (int sl = sl0; sl < sl1; ++sl) {
      mbar_wait(&m_full[ms], (uint32_t)mph);
      BwdMetaTc mt[WG_TASKS];
#pragma unroll
      for (int it = 0; it < WG_TASKS; ++it) mt[it] = wmeta[ms][t_meta[it]];
      __syncwarp();
      if (lane == 0) mbar_arrive_tc(&m_empty[ms]);
      if (++ms == WG_MR) { ms = 0; mph ^= 1; }
      const float *x_img = xt + (long long)b * HW * Cp;
      unsigned char *a = tc_smem + (size_t)stage * STAGE_BYTES;
#pragma unroll
      for (int r = 0; r < WG_TASKS; r += 2) {
        float4 xc[2][4];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int flags = mt[r + u].packed;
          const int xo = ((flags >> 7) - (s.W + 1)) * Cp + t_xc[r + u];
          xc[u][0] = (flags & 1) ? __ldg(reinterpret_cast<const float4 *>(x_img + xo)) : z4;
          xc[u][1] = (flags & 2) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs1))) : z4;
          xc[u][2] = (flags & 4) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs2))) : z4;
          xc[u][3] = (flags & 8) ? __ldg(reinterpret_cast<const float4 *>(x_img + (xo + xs3))) : z4;
        }
        if (r == 0) {
          mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));
          if (sw == 0 && lane == 0) {
            // B operand: rows nti*NT .. nti*NT + NT - 1 of the slice's dY tile (contiguous 8-row groups)
            mbar_expect_tx(&b_full[stage], (uint32_t)B_BYTES);
            bulk_g2s(a + WB_A_BYTES, gyk + (size_t)sl * tile_bytes + (size_t)nti * B_BYTES, (uint32_t)B_BYTES,
                     &b_full[stage]);
          }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const BwdMetaTc &m = mt[r + u];
          const float lh = m.lh, lw = m.lw, mm = m.m, hh = 1.f - lh, hw = 1.f - lw;
          const float w1 = hh * hw * mm, w2 = hh * lw * mm, w3 = lh * hw * mm, w4 = lh * lw * mm;   // as the forward sampler
          const float4 x1 = xc[u][0], x2 = xc[u][1], x3 = xc[u][2], x4 = xc[u][3];
          __nv_bfloat16 *dst = reinterpret_cast<__nv_bfloat16 *>(a + t_dst[r + u]);
          dst[0] = __float2bfloat16_rn(fmaf(w4, x4.x, fmaf(w3, x3.x, fmaf(w2, x2.x, w1 * x1.x))));
          dst[8] = __float2bfloat16_rn(fmaf(w4, x4.y, fmaf(w3, x3.y, fmaf(w2, x2.y, w1 * x1.y))));    // rows c4*4 + 0..3:
          dst[16] = __float2bfloat16_rn(fmaf(w4, x4.z, fmaf(w3, x3.z, fmaf(w2, x2.z, w1 * x1.z))));   // 16 bytes apart
          dst[24] = __float2bfloat16_rn(fmaf(w4, x4.w, fmaf(w3, x3.w, fmaf(w2, x2.w, w1 * x1.w))));
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive_tc(&a_full[stage]);
      if (++stage == WB_STAGES) { stage = 0; ph ^= 1; }
      if (++sll == wg.spi) { sll = 0; ++b; }
    }
  } else if (warp >= WG_WARP_C0) {
    // =========================================================== consumers: warpgroup cw accumulates rows 64 cw .. 64 cw + 63
    const int cw = (warp - WG_WARP_C0) >> 2, wq = warp & 3;
    float d[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) d[i] = 0.f;
    int stage = 0, ph = 0;
    for (int sl = sl0; sl < sl1; ++sl) {
      mbar_wait(&a_full[stage], (uint32_t)ph);
      mbar_wait(&b_full[stage], (uint32_t)ph);
      const uint32_t base = smem_u32(tc_smem + (size_t)stage * STAGE_BYTES);
      const uint32_t a = base + (uint32_t)cw * 8u * WB_SBO, bw = base + (uint32_t)WB_A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < TC_K / 16; ++kk) {
        const uint32_t koff = (uint32_t)kk * 2u * BF_B_LBO;
        wgmma_bf16<NT>(d, wg_desc(a + koff, BF_B_LBO, WB_SBO), wg_desc(bw + koff, BF_B_LBO, BF_B_SBO),
                       (sl > sl0 || kk > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait_all();
      if (((tid - WG_WARP_C0 * 32) & 127) == 0) mbar_arrive_tc(&empty[stage]);
      if (++stage == WB_STAGES) { stage = 0; ph ^= 1; }
    }
    // epilogue: wpart[split][rg][row][co_r], columns nti*NT .. nti*NT + NT - 1 (zeros for a CTA without slices)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
      float *dst = wpart + (((size_t)split * g.RG + rg) * 128 + row) * wg.co_r + nti * NT + 2 * (lane & 3);
#pragma unroll
      for (int jj = 0; jj < NT / 8; ++jj)
        *reinterpret_cast<float2 *>(dst + 8 * jj) = make_float2(d[4 * jj + 2 * h], d[4 * jj + 2 * h + 1]);
    }
  } else {
    wg_geometry(s, g, wg, rg, sl0, sl1, offset, mask, tid, wmeta, m_full, m_empty);
  }
}

// ------------------------------------------------------------------ host
void plan_backward_tc(DcnPlan *p) {
  const DcnShapeTc &s = p->s;
  const BwdGeom g = bwd_geom(s);
  // the kernels index within one image with 32 bits (and pack hl*W+wl into 24): larger images use the fp32 path
  const unsigned long long lim = 1ull << 31, hw2 = (unsigned long long)(s.H + 2) * (s.W + 2);
  p->bwd_tc = p->fwd_tc && hw2 < (1ull << 24) && hw2 * s.nb * TC_CB < lim &&
              (unsigned long long)s.Ho * s.Wo * g.Qp * TC_CB < lim &&
              (unsigned long long)s.Ho * s.Wo * s.dg * 2 * s.kh * s.kw < lim;
  p->dw_tc = p->bwd_tc && s.Cout <= 256;
  p->bwd = {};
  if (!p->bwd_tc) return;
  const WgGeom wg = wg_geom(s, g);
  const size_t gyt_img = (size_t)g.tiles * g.KS * BW_TILE_FLOATS * 4;
  const size_t dcol_img = align_up((size_t)s.Ho * s.Wo * g.Qp * TC_CB * 4, 256);
  // images per pass: the column gradient of a pass is held to ~1.5 GiB (B=16 of the largest dla_34 layer is 0.67 GB)
  long long bc = (long long)((1536ull << 20) / (dcol_img + gyt_img));
  if (bc < 1) bc = 1;
  if (bc > s.B) bc = s.B;
  auto &l = p->bwd;
  l.chunk = (int)bc;
  l.xt = 0;
  l.dxt = l.xt + p->xt_bytes;
  l.wtt = l.dxt + p->xt_bytes;
  l.gyt = l.wtt + align_up((size_t)g.RG * g.KS * BW_TILE_FLOATS * 4, 256);
  l.dcol = l.gyt + align_up((size_t)bc * gyt_img, 256);
  const size_t data_end = l.dcol + (size_t)bc * dcol_img;
  l.gyk = l.gyt;
  l.wpart = l.gyk + align_up((size_t)wg.n_slices * 2 * wg.co_r * TC_K * 4, 256);
  l.bpart = l.wpart + align_up((size_t)wg.splits * g.RG * 128 * wg.co_r * 4, 256);
  const size_t weight_end = l.bpart + align_up((size_t)wg.n_slices * wg.co_r * 4, 256);
  const size_t end = std::max(data_end, weight_end);
  // deterministic mode: [bounds: KS + 2B uint32][fixed-point dX of one batch chunk: bc x HW x Cp int64], or the
  // per-split dW partials of the fp32 kernel (cout > 256) in the same place, whichever is larger
  l.bnd = end;
  l.dxi = l.bnd + align_up((size_t)(g.KS + 2 * s.B) * 4, 256);
  const size_t dxi_end = l.dxi + align_up((size_t)bc * s.H * s.W * s.nb * TC_CB * 8, 256);
  l.wpart32 = end;
  const size_t wpart32_end =
      s.Cout > 256 ? l.wpart32 + align_up((size_t)p->fp32_dw_splits * s.Cout * s.Cin * s.kh * s.kw * 4, 256) : 0;
  l.bytes = p->det ? std::max(dxi_end, wpart32_end) : end;
}

// dX, dOffset, dMask (each nullable; accumulated into, as cnb_dcnv2_backward documents).  p.det: dX in fixed point
// (order-independent) in the regions bnd and dxi.
int dcn_backward_data_tc(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                         const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                         float *grad_mask, void *workspace, cudaStream_t stream) {
  // p.x_cl / p.gx_cl: `input` / grad_input already are channels-last [b][h*w][cin]: the layout passes and the
  // channels-last scratch copies are skipped
  const DcnShapeTc &s = p.s;
  const BwdGeom g = bwd_geom(s);
  const int b = s.B, cin = s.Cin, cout = s.Cout, bc = p.bwd.chunk;
  char *ws = reinterpret_cast<char *>(workspace);
  float *xt = reinterpret_cast<float *>(ws + p.bwd.xt);
  float *dxt = p.gx_cl ? grad_input : reinterpret_cast<float *>(ws + p.bwd.dxt);
  const float *xsrc = p.x_cl ? input : xt;
  float *wtt = reinterpret_cast<float *>(ws + p.bwd.wtt);
  float *gyt = reinterpret_cast<float *>(ws + p.bwd.gyt);
  float *dcol = reinterpret_cast<float *>(ws + p.bwd.dcol);
  const long long HW = (long long)s.H * s.W, HWo = (long long)s.Ho * s.Wo;
  // default: every sample is scattered into a channels-last dX (16-byte vector reductions) and added to grad_input at
  // the end; deterministic mode: into the fixed-point dX of the batch chunk, converted into grad_input per chunk
  const bool det = grad_input && p.det;
  unsigned *bnd = nullptr;
  long long *dxi = nullptr;
  if (det) {
    bnd = reinterpret_cast<unsigned *>(ws + p.bwd.bnd);
    dxi = reinterpret_cast<long long *>(ws + p.bwd.dxi);
    CNB_CUDA(cudaMemsetAsync(bnd, 0, (size_t)(g.KS + 2 * b) * 4, stream));
  }

  int rc = CNB_OK;
  if (!p.x_cl) rc = dcn_to_channels_last(input, xt, s, stream);
  if (rc != CNB_OK) return rc;
  if (grad_input && !det && !p.gx_cl) CNB_CUDA(cudaMemsetAsync(dxt, 0, (size_t)b * HW * s.nb * TC_CB * 4, stream));
  if (det) k_bwd_prep_w<true><<<g.RG * g.KS, 256, 0, stream>>>(weight, s, g, wtt, bnd);
  else k_bwd_prep_w<false><<<g.RG * g.KS, 256, 0, stream>>>(weight, s, g, wtt, nullptr);
  CNB_CHECK_LAUNCH("cnb_dcnv2_backward weight tiles");
  count_launch();
  const size_t smem = (size_t)BW_STAGES * BW_STAGE_BYTES;     // operand ring
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_dcol_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dev_done = dev;
  }
  for (int b0 = 0; b0 < b; b0 += bc) {
    const int nbimg = (b - b0 < bc) ? b - b0 : bc;
    dim3 pgrid((unsigned)g.tiles, (unsigned)g.KS, (unsigned)nbimg);
    if (det) {
      CNB_CUDA(cudaMemsetAsync(dxi, 0, (size_t)nbimg * HW * s.nb * TC_CB * 8, stream));
      k_bwd_prep_gy<true><<<pgrid, 256, 0, stream>>>(grad_output + (long long)b0 * cout * HWo, s, g, gyt,
                                                      mask + (long long)b0 * s.mask_bs, bnd + g.KS + 2 * b0);
    } else {
      k_bwd_prep_gy<false><<<pgrid, 256, 0, stream>>>(grad_output + (long long)b0 * cout * HWo, s, g, gyt, nullptr, nullptr);
    }
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward grad_output tiles");
    const int n_items = nbimg * g.tiles * g.RG;
    const int grid = n_items < num_sms() ? n_items : num_sms();
    k_dcn_bwd_dcol_tc<<<grid, BW_THREADS, smem, stream>>>(gyt, wtt, dcol, s, g, n_items);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward column gradient (wgmma)");
    k_dcn_bwd_offmask<3><<<nbimg * g.tiles, 256, 0, stream>>>(xsrc, offset, mask, dcol, (grad_input && !det) ? dxt : nullptr,
                                                              grad_offset, grad_mask, dxi, bnd, s, g, b0);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward offset/mask gradient");
    count_launch(3);
    if (det) {
      if (p.gx_cl) {
        k_dcn_bwd_dx_fixed<true><<<dim3((unsigned)((HW + 31) / 32), 1u, (unsigned)nbimg), 256, 0, stream>>>(
            dxi, bnd, grad_input, s, g, b0);
      } else {
        dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((cin + 63) / 64), (unsigned)nbimg);
        k_dcn_bwd_dx_fixed<false><<<tgrid, 256, 0, stream>>>(dxi, bnd, grad_input, s, g, b0);
      }
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward input gradient (fixed point)");
      count_launch();
    }
  }
  if (grad_input && !det && !p.gx_cl) {
    dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((cin + 63) / 64), (unsigned)b);
    k_dcn_bwd_dx_nchw<<<tgrid, 256, 0, stream>>>(dxt, grad_input, s);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward input gradient");
    count_launch();
  }
  return CNB_OK;
}

// dW and dBias (accumulated into grad_weight / grad_bias; grad_bias nullable).  p.xt_ready: the channels-last input
// copy was already written by dcn_backward_data_tc on this stream.
int dcn_backward_weight_tc(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                           const float *grad_output, float *grad_weight, float *grad_bias, void *workspace,
                           cudaStream_t stream) {
  const DcnShapeTc &s = p.s;
  const BwdGeom g = bwd_geom(s);
  const WgGeom wg = wg_geom(s, g);
  char *ws = reinterpret_cast<char *>(workspace);
  float *xt = reinterpret_cast<float *>(ws + p.bwd.xt);
  float *gyk = reinterpret_cast<float *>(ws + p.bwd.gyk);
  float *wpart = reinterpret_cast<float *>(ws + p.bwd.wpart);
  float *bpart = reinterpret_cast<float *>(ws + p.bwd.bpart);
  const float *xsrc = p.x_cl ? input : xt;
  if (!p.xt_ready && !p.x_cl) {
    const int rc = dcn_to_channels_last(input, xt, s, stream);
    if (rc != CNB_OK) return rc;
  }
  dim3 pgrid((unsigned)wg.spi, (unsigned)s.B);
  k_bwd_prep_gyk<<<pgrid, 256, 0, stream>>>(grad_output, s, wg, gyk, grad_bias ? bpart : nullptr);
  CNB_CHECK_LAUNCH("cnb_dcnv2_backward grad_output tiles (weight pass)");
  const size_t smem = (size_t)wg.stages * wg.stage_bytes;
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_weight_tc<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  WG_STAGES * (2 * WG_A_BYTES + 2 * 64 * TC_K * 4)));
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_weight_tc<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  WG_STAGES * (2 * WG_A_BYTES + 2 * 128 * TC_K * 4)));
    dev_done = dev;
  }
  const unsigned wgrid = (unsigned)(g.RG * wg.n_nt * wg.splits);
  if (wg.nt == 64) k_dcn_bwd_weight_tc<64><<<wgrid, WG_THREADS, smem, stream>>>(xsrc, offset, mask, gyk, wpart, s, g, wg);
  else k_dcn_bwd_weight_tc<128><<<wgrid, WG_THREADS, smem, stream>>>(xsrc, offset, mask, gyk, wpart, s, g, wg);
  CNB_CHECK_LAUNCH("cnb_dcnv2_backward weight gradient (wgmma)");
  const long long total = (long long)g.RG * 128 * wg.co_r;
  k_dcn_bwd_wreduce<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(wpart, grad_weight, s, g, wg);
  CNB_CHECK_LAUNCH("cnb_dcnv2_backward weight gradient reduce");
  count_launch(3);
  if (grad_bias) {
    k_dcn_bwd_bias_reduce<<<s.Cout, 256, 0, stream>>>(bpart, grad_bias, wg);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward bias gradient reduce");
    count_launch();
  }
  return CNB_OK;
}

// The bf16 backward's workspace: plan_backward_tc's regions with bf16 tiles.  It needs both tensor-core passes (the
// weight pass covers cout <= 256): elsewhere bytes stays 0 and cnb_dcnv2_backward_bf16 returns CNB_EUNSUPPORTED.
void plan_backward_bf16(DcnPlan *p) {
  const DcnShapeTc &s = p->s;
  p->bwd16 = {};
  if (!p->bwd_tc || !p->dw_tc) return;
  const BwdGeom g = bwd_geom(s);
  const WgGeom wg = wg_geom(s, g);
  const size_t gyt_img = (size_t)g.tiles * g.KS * BB_TILE_BYTES;
  const size_t dcol_img = align_up((size_t)s.Ho * s.Wo * g.Qp * TC_CB * 4, 256);
  long long bc = (long long)((1536ull << 20) / (dcol_img + gyt_img));   // as plan_backward_tc: ~1.5 GiB a pass
  if (bc < 1) bc = 1;
  if (bc > s.B) bc = s.B;
  auto &l = p->bwd16;
  l.chunk = (int)bc;
  l.xt = 0;
  l.dxt = l.xt + p->xt_bytes;
  l.wtb = l.dxt + p->xt_bytes;
  l.gyt = l.wtb + align_up((size_t)g.RG * g.KS * BB_TILE_BYTES, 256);
  l.dcol = l.gyt + align_up((size_t)bc * gyt_img, 256);
  const size_t data_end = l.dcol + (size_t)bc * dcol_img;
  l.gyk = l.gyt;
  l.wpart = l.gyk + align_up((size_t)wg.n_slices * wg.co_r * TC_K * 2, 256);
  l.bpart = l.wpart + align_up((size_t)wg.splits * g.RG * 128 * wg.co_r * 4, 256);
  const size_t weight_end = l.bpart + align_up((size_t)wg.n_slices * wg.co_r * 4, 256);
  const size_t end = std::max(data_end, weight_end);
  l.bnd = end;
  l.dxi = l.bnd + align_up((size_t)(g.KS + 2 * s.B) * 4, 256);
  l.bytes = p->det ? l.dxi + align_up((size_t)bc * s.H * s.W * s.nb * TC_CB * 8, 256) : end;
}

int dcn_backward_bf16(const DcnPlan &p, const void *input, bool in_bf16, const float *offset, const float *mask,
                      const float *weight, const void *grad_output, bool gy_bf16, float *grad_input, float *grad_offset,
                      float *grad_mask, float *grad_weight, float *grad_bias, void *workspace, cudaStream_t stream) {
  const DcnShapeTc &s = p.s;
  const BwdGeom g = bwd_geom(s);
  const WgGeom wg = wg_geom(s, g);
  const auto &l = p.bwd16;
  const int b = s.B, cin = s.Cin, bc = l.chunk;
  const long long HW = (long long)s.H * s.W, HWo = (long long)s.Ho * s.Wo;
  char *ws = reinterpret_cast<char *>(workspace);
  float *xt = reinterpret_cast<float *>(ws + l.xt);
  const float *gy32 = reinterpret_cast<const float *>(grad_output);
  const __nv_bfloat16 *gy16 = reinterpret_cast<const __nv_bfloat16 *>(grad_output);
  const bool data = grad_input || grad_offset || grad_mask;
  int rc = CNB_OK;
  // the samplers read an fp32 channels-last input: an fp32 channels-last one in place, else the copy xt
  const float *xsrc = xt;
  if (data || grad_weight) {
    if (in_bf16) rc = dcn_to_channels_last(reinterpret_cast<const __nv_bfloat16 *>(input), p.x_cl, xt, s, stream);
    else if (p.x_cl) xsrc = reinterpret_cast<const float *>(input);
    else rc = dcn_to_channels_last(reinterpret_cast<const float *>(input), xt, s, stream);
    if (rc != CNB_OK) return rc;
  }

  if (data) {
    // the data pass of dcn_backward_data_tc with bf16 operand tiles and k_dcn_bwd_dcol_bf16
    float *dxt = p.gx_cl ? grad_input : reinterpret_cast<float *>(ws + l.dxt);
    unsigned char *wtb = reinterpret_cast<unsigned char *>(ws + l.wtb);
    unsigned char *gyt = reinterpret_cast<unsigned char *>(ws + l.gyt);
    float *dcol = reinterpret_cast<float *>(ws + l.dcol);
    const bool det = grad_input && p.det;
    unsigned *bnd = nullptr;
    long long *dxi = nullptr;
    if (det) {
      bnd = reinterpret_cast<unsigned *>(ws + l.bnd);
      dxi = reinterpret_cast<long long *>(ws + l.dxi);
      CNB_CUDA(cudaMemsetAsync(bnd, 0, (size_t)(g.KS + 2 * b) * 4, stream));
    }
    if (grad_input && !det && !p.gx_cl) CNB_CUDA(cudaMemsetAsync(dxt, 0, (size_t)b * HW * s.nb * TC_CB * 4, stream));
    if (det) k_bwd_prep_w_bf16<true><<<g.RG * g.KS, 256, 0, stream>>>(weight, s, g, wtb, bnd);
    else k_bwd_prep_w_bf16<false><<<g.RG * g.KS, 256, 0, stream>>>(weight, s, g, wtb, nullptr);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 weight tiles");
    count_launch();
    const size_t smem = (size_t)BB_STAGES * BB_STAGE_BYTES;
    static thread_local int dev_done = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev_done != dev) {
      CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_dcol_bf16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      dev_done = dev;
    }
    for (int b0 = 0; b0 < b; b0 += bc) {
      const int nbimg = (b - b0 < bc) ? b - b0 : bc;
      const dim3 pgrid((unsigned)g.tiles, (unsigned)g.KS, (unsigned)nbimg);
      const long long go = (long long)b0 * s.Cout * HWo;
      if (det) {
        CNB_CUDA(cudaMemsetAsync(dxi, 0, (size_t)nbimg * HW * s.nb * TC_CB * 8, stream));
        const float *mk = mask + (long long)b0 * s.mask_bs;
        if (gy_bf16) k_bwd_prep_gy_bf16<__nv_bfloat16, true><<<pgrid, 256, 0, stream>>>(gy16 + go, s, g, gyt, mk, bnd + g.KS + 2 * b0);
        else k_bwd_prep_gy_bf16<float, true><<<pgrid, 256, 0, stream>>>(gy32 + go, s, g, gyt, mk, bnd + g.KS + 2 * b0);
      } else {
        if (gy_bf16) k_bwd_prep_gy_bf16<__nv_bfloat16, false><<<pgrid, 256, 0, stream>>>(gy16 + go, s, g, gyt, nullptr, nullptr);
        else k_bwd_prep_gy_bf16<float, false><<<pgrid, 256, 0, stream>>>(gy32 + go, s, g, gyt, nullptr, nullptr);
      }
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 grad_output tiles");
      const int n_items = nbimg * g.tiles * g.RG;
      const int grid = n_items < num_sms() ? n_items : num_sms();
      k_dcn_bwd_dcol_bf16<<<grid, BW_THREADS, smem, stream>>>(gyt, wtb, dcol, s, g, n_items);
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 column gradient (wgmma bf16)");
      k_dcn_bwd_offmask<3><<<nbimg * g.tiles, 256, 0, stream>>>(xsrc, offset, mask, dcol, (grad_input && !det) ? dxt : nullptr,
                                                                grad_offset, grad_mask, dxi, bnd, s, g, b0);
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 offset/mask gradient");
      count_launch(3);
      if (det) {
        if (p.gx_cl) {
          k_dcn_bwd_dx_fixed<true><<<dim3((unsigned)((HW + 31) / 32), 1u, (unsigned)nbimg), 256, 0, stream>>>(
              dxi, bnd, grad_input, s, g, b0);
        } else {
          dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((cin + 63) / 64), (unsigned)nbimg);
          k_dcn_bwd_dx_fixed<false><<<tgrid, 256, 0, stream>>>(dxi, bnd, grad_input, s, g, b0);
        }
        CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 input gradient (fixed point)");
        count_launch();
      }
    }
    if (grad_input && !det && !p.gx_cl) {
      dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((cin + 63) / 64), (unsigned)b);
      k_dcn_bwd_dx_nchw<<<tgrid, 256, 0, stream>>>(dxt, grad_input, s);
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 input gradient");
      count_launch();
    }
  }

  if (grad_weight || grad_bias) {
    // the weight pass of dcn_backward_weight_tc; the bias partials come from the same grad_output pass either way
    unsigned char *gyk = reinterpret_cast<unsigned char *>(ws + l.gyk);
    float *wpart = reinterpret_cast<float *>(ws + l.wpart);
    float *bpart = grad_bias ? reinterpret_cast<float *>(ws + l.bpart) : nullptr;
    const dim3 pgrid((unsigned)wg.spi, (unsigned)b);
    if (gy_bf16) k_bwd_prep_gyk_bf16<__nv_bfloat16><<<pgrid, 256, 0, stream>>>(gy16, s, wg, gyk, bpart);
    else k_bwd_prep_gyk_bf16<float><<<pgrid, 256, 0, stream>>>(gy32, s, wg, gyk, bpart);
    CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 grad_output tiles (weight pass)");
    count_launch();
    if (grad_weight) {
      const size_t smem = (size_t)WB_STAGES * (WB_A_BYTES + wg.nt * TC_K * 2);
      static thread_local int dev_done = -1;
      int dev = 0;
      cudaGetDevice(&dev);
      if (dev_done != dev) {
        CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_weight_bf16<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      WB_STAGES * (WB_A_BYTES + 64 * TC_K * 2)));
        CNB_CUDA(cudaFuncSetAttribute(k_dcn_bwd_weight_bf16<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      WB_STAGES * (WB_A_BYTES + 128 * TC_K * 2)));
        dev_done = dev;
      }
      const unsigned wgrid = (unsigned)(g.RG * wg.n_nt * wg.splits);
      if (wg.nt == 64)
        k_dcn_bwd_weight_bf16<64><<<wgrid, WG_THREADS, smem, stream>>>(xsrc, offset, mask, gyk, wpart, s, g, wg);
      else
        k_dcn_bwd_weight_bf16<128><<<wgrid, WG_THREADS, smem, stream>>>(xsrc, offset, mask, gyk, wpart, s, g, wg);
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 weight gradient (wgmma bf16)");
      const long long total = (long long)g.RG * 128 * wg.co_r;
      k_dcn_bwd_wreduce<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(wpart, grad_weight, s, g, wg);
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 weight gradient reduce");
      count_launch(2);
    }
    if (grad_bias) {
      k_dcn_bwd_bias_reduce<<<s.Cout, 256, 0, stream>>>(bpart, grad_bias, wg);
      CNB_CHECK_LAUNCH("cnb_dcnv2_backward_bf16 bias gradient reduce");
      count_launch();
    }
  }
  return CNB_OK;
}

}  // namespace cnb

// Float64 DCNv2 (the reference's second build, _ext.dcn_v2_double: dcn_v2_cuda_double.c and
// dcn_v2_im2col_cuda_double.cu) on the FP64 tensor cores.
//
// Every contraction is one block GEMM on mma.sync.m16n8k16.f64 (DMMA.16x8x16 on sm_90a): 128 threads, a 64x64
// tile, K in steps of 16, fed through shared memory by loaders that build their operand on the fly.  The deformable
// columns are never written to memory: the forward and the weight gradient sample them straight into the shared
// tile, following modulated_deformable_im2col_gpu_kernel (:132-194) step for step in double.
//
// Backward, and why every gradient is bit-reproducible:
//   dcol = W^T . dY      DMMA GEMM into the workspace, a chunk of images at a time (plain stores);
//   dOffset / dMask      one thread per (image, group, tap, pixel) walks its channels in order
//                        (modulated_deformable_col2im_coord_gpu_kernel :255-326), one writer per output;
//   dX                   the same thread scatters dcol * mask * corner weight (col2im :196-253) into a two-limb
//                        fixed-point accumulator with integer atomics; integer addition is associative, so the
//                        sum does not depend on the order the adds land (fx64.cuh);
//   dW = dY . col^T      DMMA GEMM over fixed pixel ranges, one partial per range, the partials added in range
//                        order;
//   dBias                one block per output channel, fixed per-thread strides and a fixed tree.
#include <algorithm>
#include "fx64.cuh"

namespace cnb {

namespace {

constexpr int G_BM = 64, G_BN = 64, G_BK = 16, G_THREADS = 128;
constexpr int G_LDA = G_BK + 4;   // As[m][k] row stride (doubles): conflict-free fragment reads
constexpr int G_LDB = G_BN + 4;   // Bs[k][n]
constexpr long long DCOL_CHUNK_BYTES = 3ll << 29;   // column gradient of up to 1.5 GiB of images at a time
constexpr long long DW_RANGE = 2048;                 // pixel range of one weight-gradient partial (times a factor)
constexpr int DW_MAX_PARTIALS = 64;

struct Dcn64 {
  const double *x, *off, *msk;
  int B, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg;
  int Ho, Wo, KT, K, HWo, cpg;
};

__device__ __forceinline__ void dmma(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
        "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// C[m][n] = sum_k A[m][k] B[k][n] over k in [0, nk) for one 64x64 tile.  fa(m, k) / fb(k, n) return the operand
// (0 outside the problem), store(m, n, v) writes a result.  A_KFAST / B_KFAST: the operand's source is contiguous
// along k (else along m / n), which decides how the 128 threads split the tile's loads so that neighbouring
// threads read neighbouring addresses.  The next step's operands are loaded into registers
// while the tensor cores work on the current one.
template <bool A_KFAST, bool B_KFAST, class FA, class FB, class FS>
__device__ __forceinline__ void block_gemm(int nk, FA fa, FB fb, FS store) {
  __shared__ double As[G_BM * G_LDA];
  __shared__ double Bs[G_BK * G_LDB];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.0;
  double ra[8], rb[8];
  auto load = [&](int k0) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int e = tid + r * G_THREADS;
      ra[r] = A_KFAST ? fa(e >> 4, k0 + (e & 15)) : fa(e & 63, k0 + (e >> 6));
      rb[r] = B_KFAST ? fb(k0 + (e & 15), e >> 4) : fb(k0 + (e >> 6), e & 63);
    }
  };
  load(0);
  for (int k0 = 0; k0 < nk; k0 += G_BK) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int e = tid + r * G_THREADS;
      if (A_KFAST) As[(e >> 4) * G_LDA + (e & 15)] = ra[r];
      else As[(e & 63) * G_LDA + (e >> 6)] = ra[r];
      if (B_KFAST) Bs[(e & 15) * G_LDB + (e >> 4)] = rb[r];
      else Bs[(e >> 6) * G_LDB + (e & 63)] = rb[r];
    }
    __syncthreads();
    if (k0 + G_BK < nk) load(k0 + G_BK);
    double af[2][8], bf[4][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int i = 0; i < 8; ++i) af[mi][i] = As[(wm + mi * 16 + g + 8 * (i & 1)) * G_LDA + tq + 4 * (i >> 1)];
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) bf[ni][i] = Bs[(tq + 4 * i) * G_LDB + wn + ni * 8 + g];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) dmma(acc[mi][ni], af[mi], bf[ni]);
    __syncthreads();
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int r = 0; r < 4; ++r)
        store(wm + mi * 16 + g + 8 * (r >> 1), wn + ni * 8 + 2 * tq + (r & 1), acc[mi][ni][r]);
}

// dmcn_im2col_bilinear (:32-61)
__device__ __forceinline__ double bilinear64(const double *im, int H, int W, double h, double w) {
  const int h_low = (int)floor(h), w_low = (int)floor(w), h_high = h_low + 1, w_high = w_low + 1;
  const double lh = h - h_low, lw = w - w_low, hh = 1 - lh, hw = 1 - lw;
  double v1 = 0, v2 = 0, v3 = 0, v4 = 0;
  if (h_low >= 0 && w_low >= 0) v1 = im[h_low * W + w_low];
  if (h_low >= 0 && w_high <= W - 1) v2 = im[h_low * W + w_high];
  if (h_high <= H - 1 && w_low >= 0) v3 = im[h_high * W + w_low];
  if (h_high <= H - 1 && w_high <= W - 1) v4 = im[h_high * W + w_high];
  const double w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
  return w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4;
}

// Sampling position of tap t at output pixel p of image b, group g (:155-177); false outside (-1, H) x (-1, W).
__device__ __forceinline__ bool sample_pos(const Dcn64 &a, int b, int g, int t, int p, double *h_im, double *w_im,
                                           double *mask) {
  const int ho = p / a.Wo, wo = p - ho * a.Wo, i = t / a.kw, j = t - i * a.kw;
  const long long ob = (long long)(b * a.dg + g) * a.KT + t;
  const double oh = a.off[(2 * ob) * a.HWo + p], ow = a.off[(2 * ob + 1) * a.HWo + p];
  *mask = a.msk[ob * a.HWo + p];
  *h_im = (ho * a.sh - a.ph + i * a.dh) + oh;
  *w_im = (wo * a.sw - a.pw + j * a.dw) + ow;
  return *h_im > -1 && *w_im > -1 && *h_im < a.H && *w_im < a.W;
}

// column entry k = ci * KT + t (the weight's (cin, kh, kw) order) at pixel p: mask * bilinear sample
__device__ __forceinline__ double col64(const Dcn64 &a, int b, int k, int p) {
  const int ci = k / a.KT, t = k - ci * a.KT;
  double h, w, m;
  double val = 0;
  if (sample_pos(a, b, ci / a.cpg, t, p, &h, &w, &m))
    val = bilinear64(a.x + ((long long)b * a.Cin + ci) * a.H * a.W, a.H, a.W, h, w);
  return val * m;
}

__global__ void __launch_bounds__(G_THREADS) k_dcn64_forward(const Dcn64 a, const double *__restrict__ wt,
                                                             const double *__restrict__ bias, double *out) {
  const int p0 = blockIdx.x * G_BN, co0 = blockIdx.y * G_BM, b = blockIdx.z;
  block_gemm<true, false>(
      a.K,
      [&](int m, int k) { return (co0 + m < a.Cout && k < a.K) ? wt[(long long)(co0 + m) * a.K + k] : 0.0; },
      [&](int k, int n) { return (k < a.K && p0 + n < a.HWo) ? col64(a, b, k, p0 + n) : 0.0; },
      [&](int m, int n, double v) {
        const int co = co0 + m, p = p0 + n;
        if (co < a.Cout && p < a.HWo) out[((long long)b * a.Cout + co) * a.HWo + p] = v + (bias ? bias[co] : 0.0);
      });
}

// dcol[bl][k][p] = sum_co W[co][k] dY[b0 + bl][co][p]
__global__ void __launch_bounds__(G_THREADS) k_dcn64_dcol(const Dcn64 a, const double *__restrict__ wt,
                                                          const double *__restrict__ gy, int b0, double *dcol) {
  const int p0 = blockIdx.x * G_BN, k0 = blockIdx.y * G_BM, bl = blockIdx.z, b = b0 + bl;
  const double *gyb = gy + (long long)b * a.Cout * a.HWo;
  block_gemm<false, false>(
      a.Cout,
      [&](int m, int co) { return (k0 + m < a.K && co < a.Cout) ? wt[(long long)co * a.K + k0 + m] : 0.0; },
      [&](int co, int n) { return (co < a.Cout && p0 + n < a.HWo) ? gyb[(long long)co * a.HWo + p0 + n] : 0.0; },
      [&](int m, int n, double v) {
        if (k0 + m < a.K && p0 + n < a.HWo) dcol[((long long)bl * a.K + k0 + m) * a.HWo + p0 + n] = v;
      });
}

// partial s of dW over the flattened pixels q = b * HWo + p in [s * range, (s + 1) * range)
__global__ void __launch_bounds__(G_THREADS) k_dcn64_dw(const Dcn64 a, const double *__restrict__ gy, long long range,
                                                        double *part) {
  const int k0 = blockIdx.x * G_BN, co0 = blockIdx.y * G_BM, s = blockIdx.z;
  const long long q0 = (long long)s * range, total = (long long)a.B * a.HWo;
  const int nq = (int)min(range, total - q0);
  block_gemm<true, true>(
      nq,
      [&](int m, int kk) {
        if (co0 + m >= a.Cout || kk >= nq) return 0.0;
        const long long q = q0 + kk;
        const int b = (int)(q / a.HWo), p = (int)(q - (long long)b * a.HWo);
        return gy[((long long)b * a.Cout + co0 + m) * a.HWo + p];
      },
      [&](int kk, int n) {
        if (kk >= nq || k0 + n >= a.K) return 0.0;
        const long long q = q0 + kk;
        const int b = (int)(q / a.HWo), p = (int)(q - (long long)b * a.HWo);
        return col64(a, b, k0 + n, p);
      },
      [&](int m, int n, double v) {
        if (co0 + m < a.Cout && k0 + n < a.K) part[((long long)s * a.Cout + co0 + m) * a.K + k0 + n] = v;
      });
}

__global__ void k_dcn64_dw_sum(const double *__restrict__ part, int nparts, long long n, double *gw) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0;
  for (int j = 0; j < nparts; ++j) s += part[(long long)j * n + i];
  gw[i] += s;
}

__global__ void __launch_bounds__(256) k_dcn64_dbias(const double *__restrict__ gy, int B, int Cout, int HWo,
                                                     double *gb) {
  __shared__ double red[256];
  const int co = blockIdx.x;
  double s = 0;
  for (int b = 0; b < B; ++b) {
    const double *p = gy + ((long long)b * Cout + co) * HWo;
    for (int i = threadIdx.x; i < HWo; i += 256) s += p[i];
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) gb[co] += red[0];
}

// ------------------------------------------------------------------ fixed-point dX (fx64.cuh)
__global__ void k_fx_finish(const unsigned long long *__restrict__ hi, const unsigned long long *__restrict__ lo,
                            const FxParam *__restrict__ prm, long long per_img, long long n, double *out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const FxParam f = prm[i / per_img];
  if (f.bad) {
    out[i] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  const unsigned long long l = lo[i];
  const long long h = (long long)hi[i] + (long long)(l >> f.L);
  const double r = (double)h + scalbn((double)(l & ((1ull << f.L) - 1)), -f.L);
  out[i] += scalbn(r, -f.e);
}

// bounds of the dX accumulator: bits of max |W col sum| (slot 2B), per image max |dY| (slot b), max |mask| (B + b)
__global__ void k_dcn64_wbound(const double *__restrict__ wt, int Cout, int K, unsigned long long *bits) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  double s = 0;
  for (int co = 0; co < Cout; ++co) s += fabs(wt[(long long)co * K + k]);
  atomicMax(bits, abs_bits64(s));
}

__global__ void k_absmax_per_image(const double *__restrict__ v, long long per_img, unsigned long long *bits) {
  const int b = blockIdx.y;
  const double *p = v + (long long)b * per_img;
  unsigned long long m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_img; i += (long long)gridDim.x * blockDim.x)
    m = max(m, abs_bits64(p[i]));
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(bits + b, m);
}

__global__ void k_dcn64_params(const unsigned long long *__restrict__ bits, int B, double count, FxParam *prm) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const unsigned long long ba = bits[2 * B], by = bits[b], bm = bits[B + b];
  const bool finite = ba < kInfBits64 && by < kInfBits64 && bm < kInfBits64;
  const double bound = count * __longlong_as_double(ba) * __longlong_as_double(by) * __longlong_as_double(bm);
  prm[b] = fx_param(bound, count, finite);
}

// one thread per (image bl of the chunk, group, tap, pixel): dOffset / dMask in channel order, and the dX scatter
__global__ void __launch_bounds__(256) k_dcn64_coord(const Dcn64 a, const double *__restrict__ dcol, int b0, int nb,
                                                     const FxParam *__restrict__ prm, double *goff, double *gmsk,
                                                     unsigned long long *fx_hi, unsigned long long *fx_lo) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)nb * a.dg * a.KT * a.HWo;
  if (idx >= n) return;
  const int p = (int)(idx % a.HWo);
  long long r = idx / a.HWo;
  const int t = (int)(r % a.KT);
  r /= a.KT;
  const int g = (int)(r % a.dg), bl = (int)(r / a.dg), b = b0 + bl;
  double inv_h, inv_w, mask;
  const bool valid = sample_pos(a, b, g, t, p, &inv_h, &inv_w, &mask);
  const FxParam f = prm[b];
  const int H = a.H, W = a.W;
  const int h_low = (int)floor(inv_h), w_low = (int)floor(inv_w), h_high = h_low + 1, w_high = w_low + 1;
  const bool c1 = h_low >= 0 && w_low >= 0, c2 = h_low >= 0 && w_high <= W - 1;
  const bool c3 = h_high <= H - 1 && w_low >= 0, c4 = h_high <= H - 1 && w_high <= W - 1;
  const double lh = inv_h - h_low, lw = inv_w - w_low, hh = 1 - lh, hw = 1 - lw;
  // dmcn_get_coordinate_weight (:89-130) and dmcn_get_gradient_weight (:63-87) factors
  const double ah = h_low + 1 - inv_h, bh = inv_h - h_low, aw = w_low + 1 - inv_w, bw = inv_w - w_low;
  const double q1 = (h_low + 1 - inv_h) * (w_low + 1 - inv_w), q2 = (h_low + 1 - inv_h) * (inv_w + 1 - w_high);
  const double q3 = (inv_h + 1 - h_high) * (w_low + 1 - inv_w), q4 = (inv_h + 1 - h_high) * (inv_w + 1 - w_high);
  const long long HW = (long long)H * W;
  double val_h = 0, val_w = 0, mval = 0;
  const int ci0 = g * a.cpg;
  for (int c = 0; c < a.cpg; ++c) {
    const int ci = ci0 + c;
    const double dc = dcol[((long long)bl * a.K + (long long)ci * a.KT + t) * a.HWo + p];
    if (!valid) continue;   // inv_h = inv_w = -2 in the reference: every weight is 0
    const long long pl = ((long long)b * a.Cin + ci) * HW;
    const double *im = a.x + pl;
    const double v1 = c1 ? im[h_low * W + w_low] : 0.0, v2 = c2 ? im[h_low * W + w_high] : 0.0;
    const double v3 = c3 ? im[h_high * W + w_low] : 0.0, v4 = c4 ? im[h_high * W + w_high] : 0.0;
    mval += dc * (hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4);
    const double wy = -1 * aw * v1 + -1 * bw * v2 + aw * v3 + bw * v4;
    const double wx = -1 * ah * v1 + ah * v2 + -1 * bh * v3 + bh * v4;
    val_h += wy * dc * mask;
    val_w += wx * dc * mask;
    if (f.bad) continue;
    const double top = dc * mask;
    if (c1) fx_add(fx_hi, fx_lo, pl + h_low * W + w_low, q1 * top, f);
    if (c2) fx_add(fx_hi, fx_lo, pl + h_low * W + w_high, q2 * top, f);
    if (c3) fx_add(fx_hi, fx_lo, pl + h_high * W + w_low, q3 * top, f);
    if (c4) fx_add(fx_hi, fx_lo, pl + h_high * W + w_high, q4 * top, f);
  }
  const long long ob = (long long)(b * a.dg + g) * a.KT + t;
  goff[(2 * ob) * a.HWo + p] += val_h;
  goff[(2 * ob + 1) * a.HWo + p] += val_w;
  gmsk[ob * a.HWo + p] += mval;
}

// ------------------------------------------------------------------ host side
int fill_dcn64(const char *who, Dcn64 *a, const double *x, const double *off, const double *msk, const double *w,
               int b, int cin, int h, int wd, int cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
               int dg) {
  CNB_REQUIRE(x && off && msk && w, CNB_EINVAL, "%s: null pointer", who);
  CNB_REQUIRE(b > 0 && b <= 65535 && cin > 0 && h > 0 && wd > 0 && cout > 0 && kh > 0 && kw > 0, CNB_EINVAL,
              "%s: bad shape", who);
  CNB_REQUIRE(sh > 0 && sw > 0 && dh > 0 && dw > 0 && ph >= 0 && pw >= 0, CNB_EINVAL,
              "%s: bad stride / padding / dilation", who);
  CNB_REQUIRE(dg > 0 && cin % dg == 0, CNB_EINVAL, "%s: deformable_groups %d must divide cin %d", who, dg, cin);
  const long long ho = ((long long)h + 2 * ph - ((long long)dh * (kh - 1) + 1)) / sh + 1;
  const long long wo = ((long long)wd + 2 * pw - ((long long)dw * (kw - 1) + 1)) / sw + 1;
  CNB_REQUIRE(ho > 0 && wo > 0, CNB_EINVAL, "%s: empty output grid", who);
  const long long kt = (long long)kh * kw, k = (long long)cin * kt;
  CNB_REQUIRE(ho * wo < (1ll << 31) && k < (1ll << 31) && kt * dg * 2 * ho * wo < (1ll << 31) &&
                  (long long)h * wd < (1ll << 31),
              CNB_EINVAL, "%s: shape exceeds 32-bit in-image indexing", who);
  a->x = x; a->off = off; a->msk = msk;
  a->B = b; a->Cin = cin; a->H = h; a->W = wd; a->Cout = cout; a->kh = kh; a->kw = kw;
  a->sh = sh; a->sw = sw; a->ph = ph; a->pw = pw; a->dh = dh; a->dw = dw; a->dg = dg;
  a->Ho = (int)ho; a->Wo = (int)wo; a->KT = (int)kt; a->K = (int)k; a->HWo = (int)(ho * wo); a->cpg = cin / dg;
  return CNB_OK;
}

struct Bwd64Layout {
  size_t bits, prm, hi, lo, part, dcol, total;
  int nbc, nparts;
  long long range;
};

Bwd64Layout bwd64_layout(const Dcn64 &a) {
  Bwd64Layout l;
  const long long total_q = (long long)a.B * a.HWo;
  long long range = DW_RANGE * ((total_q + DW_RANGE * DW_MAX_PARTIALS - 1) / (DW_RANGE * DW_MAX_PARTIALS));
  l.range = range;
  l.nparts = (int)((total_q + range - 1) / range);
  const long long per_img_dcol = (long long)a.K * a.HWo * 8;
  l.nbc = (int)std::max(1ll, std::min((long long)a.B, DCOL_CHUNK_BYTES / per_img_dcol));
  const size_t nx = (size_t)a.B * a.Cin * a.H * a.W;
  size_t o = 0;
  l.bits = o; o = align_up(o + (size_t)(2 * a.B + 1) * 8, 256);
  l.prm = o; o = align_up(o + (size_t)a.B * sizeof(FxParam), 256);
  l.hi = o; o = align_up(o + nx * 8, 256);
  l.lo = o; o = align_up(o + nx * 8, 256);
  l.part = o; o = align_up(o + (size_t)l.nparts * a.Cout * a.K * 8, 256);
  l.dcol = o; o = align_up(o + (size_t)l.nbc * per_img_dcol, 256);
  l.total = o;
  return l;
}

unsigned grid1(long long n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

// shared with the float64 PSROI pooling backward (psroi.cu)
void absmax_bits_launch(const double *v, long long per_img, int nimg, unsigned long long *bits, cudaStream_t st) {
  if (per_img <= 0 || nimg <= 0) return;
  k_absmax_per_image<<<dim3((unsigned)std::min(grid1(per_img, 256), 64u), nimg), 256, 0, st>>>(v, per_img, bits);
  count_launch();
}

int fx_finish_launch(const unsigned long long *hi, const unsigned long long *lo, const FxParam *prm,
                     long long per_img, long long n, double *out, cudaStream_t st) {
  if (n == 0) return CNB_OK;
  k_fx_finish<<<grid1(n, 256), 256, 0, st>>>(hi, lo, prm, per_img, n, out);
  CNB_CHECK_LAUNCH("fx_finish");
  count_launch();
  return CNB_OK;
}

}  // namespace cnb

using namespace cnb;

extern "C" {

size_t cnb_dcnv2_f64_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw, int stride, int pad,
                                     int dil, int dg) {
  static const double dummy = 0;
  Dcn64 a;
  if (fill_dcn64("cnb_dcnv2_f64_workspace_bytes", &a, &dummy, &dummy, &dummy, &dummy, b, cin, h, w, cout, kh, kw,
                 stride, stride, pad, pad, dil, dil, dg) != CNB_OK)
    return 0;
  return bwd64_layout(a).total;
}

int cnb_dcnv2_forward_f64(const double *input, const double *offset, const double *mask, const double *weight,
                          const double *bias, double *output, int b, int cin, int h, int w, int cout, int kh, int kw,
                          int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w,
                          int deformable_groups, void *stream) {
  Dcn64 a;
  int rc = fill_dcn64("cnb_dcnv2_forward_f64", &a, input, offset, mask, weight, b, cin, h, w, cout, kh, kw, stride_h,
                      stride_w, pad_h, pad_w, dil_h, dil_w, deformable_groups);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(output, CNB_EINVAL, "cnb_dcnv2_forward_f64: null pointer");
  const dim3 grid((a.HWo + G_BN - 1) / G_BN, (cout + G_BM - 1) / G_BM, b);
  CNB_REQUIRE(grid.y <= 65535, CNB_EINVAL, "cnb_dcnv2_forward_f64: bad shape");
  k_dcn64_forward<<<grid, G_THREADS, 0, (cudaStream_t)stream>>>(a, weight, bias, output);
  CNB_CHECK_LAUNCH("cnb_dcnv2_forward_f64");
  count_launch();
  return CNB_OK;
}

int cnb_dcnv2_backward_f64(const double *input, const double *offset, const double *mask, const double *weight,
                           const double *grad_output, double *grad_input, double *grad_offset, double *grad_mask,
                           double *grad_weight, double *grad_bias, int b, int cin, int h, int w, int cout, int kh,
                           int kw, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w,
                           int deformable_groups, void *workspace, size_t workspace_bytes, void *stream) {
  const char *who = "cnb_dcnv2_backward_f64";
  Dcn64 a;
  int rc = fill_dcn64(who, &a, input, offset, mask, weight, b, cin, h, w, cout, kh, kw, stride_h, stride_w, pad_h,
                      pad_w, dil_h, dil_w, deformable_groups);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(grad_output && grad_input && grad_offset && grad_mask && grad_weight, CNB_EINVAL, "%s: null pointer",
              who);
  const Bwd64Layout l = bwd64_layout(a);
  CNB_REQUIRE(workspace && workspace_bytes >= l.total, CNB_EINVAL,
              "%s: workspace of %zu bytes is smaller than the %zu cnb_dcnv2_f64_workspace_bytes asks for", who,
              workspace_bytes, l.total);
  CNB_REQUIRE(((uintptr_t)workspace & 15) == 0, CNB_EINVAL, "%s: workspace must be 16-byte aligned", who);
  CNB_REQUIRE((unsigned)((a.K + G_BM - 1) / G_BM) <= 65535 && (unsigned)((cout + G_BM - 1) / G_BM) <= 65535,
              CNB_EINVAL, "%s: bad shape", who);
  cudaStream_t st = (cudaStream_t)stream;
  char *ws = (char *)workspace;
  unsigned long long *bits = (unsigned long long *)(ws + l.bits);
  FxParam *prm = (FxParam *)(ws + l.prm);
  unsigned long long *hi = (unsigned long long *)(ws + l.hi), *lo = (unsigned long long *)(ws + l.lo);
  double *part = (double *)(ws + l.part), *dcol = (double *)(ws + l.dcol);
  const long long nx = (long long)b * cin * h * w;
  CNB_CUDA(cudaMemsetAsync(ws + l.bits, 0, l.hi - l.bits, st));
  CNB_CUDA(cudaMemsetAsync(hi, 0, (size_t)nx * 8, st));
  CNB_CUDA(cudaMemsetAsync(lo, 0, (size_t)nx * 8, st));
  // bound of |dX| per image: KT * HWo contributions of at most max|W col sum| * max|dY_b| * max|mask_b| each
  k_dcn64_wbound<<<grid1(a.K, 256), 256, 0, st>>>(weight, cout, a.K, bits + 2 * b);
  const long long ny = (long long)cout * a.HWo, nm = (long long)deformable_groups * a.KT * a.HWo;
  absmax_bits_launch(grad_output, ny, b, bits, st);
  absmax_bits_launch(mask, nm, b, bits + b, st);
  k_dcn64_params<<<grid1(b, 128), 128, 0, st>>>(bits, b, (double)a.KT * a.HWo, prm);
  CNB_CHECK_LAUNCH(who);
  count_launch(2);
  for (int b0 = 0; b0 < b; b0 += l.nbc) {
    const int nb = std::min(l.nbc, b - b0);
    k_dcn64_dcol<<<dim3((a.HWo + G_BN - 1) / G_BN, (a.K + G_BM - 1) / G_BM, nb), G_THREADS, 0, st>>>(
        a, weight, grad_output, b0, dcol);
    const long long nc = (long long)nb * deformable_groups * a.KT * a.HWo;
    k_dcn64_coord<<<grid1(nc, 256), 256, 0, st>>>(a, dcol, b0, nb, prm, grad_offset, grad_mask, hi, lo);
    CNB_CHECK_LAUNCH(who);
    count_launch(2);
  }
  rc = fx_finish_launch(hi, lo, prm, (long long)cin * h * w, nx, grad_input, st);
  if (rc != CNB_OK) return rc;
  k_dcn64_dw<<<dim3((a.K + G_BN - 1) / G_BN, (cout + G_BM - 1) / G_BM, l.nparts), G_THREADS, 0, st>>>(
      a, grad_output, l.range, part);
  const long long nw = (long long)cout * a.K;
  k_dcn64_dw_sum<<<grid1(nw, 256), 256, 0, st>>>(part, l.nparts, nw, grad_weight);
  count_launch(2);
  if (grad_bias) {
    k_dcn64_dbias<<<cout, 256, 0, st>>>(grad_output, b, cout, a.HWo, grad_bias);
    count_launch();
  }
  CNB_CHECK_LAUNCH(who);
  return CNB_OK;
}

}  // extern "C"

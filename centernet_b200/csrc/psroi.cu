// Deformable PSROI pooling, forward and backward (DCNv2 package surface: DCNv2Pooling / DCNPooling,
// SURVEY.md section 8f N4).  Semantics of
//   src/lib/models/networks/DCNv2/src/cuda/dcn_v2_psroi_pooling_cuda.cu:47-139 (forward), :141-255 (backward):
// every output bin (roi n, channel ctop, ph, pw) averages sample_per_part^2 bilinear samples of one
// position-sensitive input channel, the bin window optionally shifted by a learned (class, part) offset.
// No CenterNet network instantiates it, so this is a plain one-thread-per-bin kernel (the op is tiny:
// N * output_dim * P * P bins x <= 16 samples); the arithmetic follows the reference expression by
// expression, including its float/double mixing in the window geometry, so bins land on the same pixels.
#include <algorithm>
#include "fx64.cuh"

namespace cnb {

struct PsroiArgs {
  const float *data, *rois, *trans;   // trans == nullptr when no_trans
  int B, C, H, W, N;
  int no_trans, output_dim, group_size, P, part_size, spp, num_classes, ch_each;
  float spatial_scale, trans_std;
};

struct PsroiBin {
  int n, ctop, ph, pw, batch, c, cls, part_h, part_w;
  float wstart, hstart, sub_w, sub_h, roi_w, roi_h;
};

// window geometry of one bin (:66-108): float arithmetic with the double literals of the source
__device__ __forceinline__ PsroiBin psroi_bin(const PsroiArgs &a, long long index) {
  PsroiBin b;
  const int P = a.P;
  b.pw = (int)(index % P);
  b.ph = (int)((index / P) % P);
  b.ctop = (int)((index / P / P) % a.output_dim);
  b.n = (int)(index / P / P / a.output_dim);
  const float *r = a.rois + (long long)b.n * 5;
  b.batch = (int)r[0];
  const float start_w = (float)((double)((float)round((double)r[1]) * a.spatial_scale) - 0.5);
  const float start_h = (float)((double)((float)round((double)r[2]) * a.spatial_scale) - 0.5);
  const float end_w = (float)((double)((float)(round((double)r[3]) + 1.) * a.spatial_scale) - 0.5);
  const float end_h = (float)((double)((float)(round((double)r[4]) + 1.) * a.spatial_scale) - 0.5);
  b.roi_w = (float)fmax((double)(end_w - start_w), 0.1);   // avoid 0
  b.roi_h = (float)fmax((double)(end_h - start_h), 0.1);
  const float bin_h = b.roi_h / (float)P, bin_w = b.roi_w / (float)P;
  b.sub_h = bin_h / (float)a.spp;
  b.sub_w = bin_w / (float)a.spp;
  b.part_h = (int)floorf((float)b.ph / (float)P * (float)a.part_size);
  b.part_w = (int)floorf((float)b.pw / (float)P * (float)a.part_size);
  b.cls = b.ctop / a.ch_each;
  float tx = 0.f, ty = 0.f;
  if (!a.no_trans) {
    const long long t0 = (((long long)b.n * a.num_classes + b.cls) * 2) * a.part_size;
    tx = a.trans[(t0 + b.part_h) * a.part_size + b.part_w] * a.trans_std;
    ty = a.trans[(t0 + a.part_size + b.part_h) * a.part_size + b.part_w] * a.trans_std;
  }
  b.wstart = __fadd_rn(__fadd_rn(__fmul_rn((float)b.pw, bin_w), start_w), __fmul_rn(tx, b.roi_w));
  b.hstart = __fadd_rn(__fadd_rn(__fmul_rn((float)b.ph, bin_h), start_h), __fmul_rn(ty, b.roi_h));
  int gw = (int)floorf((float)b.pw * (float)a.group_size / (float)P);
  int gh = (int)floorf((float)b.ph * (float)a.group_size / (float)P);
  gw = min(max(gw, 0), a.group_size - 1);
  gh = min(max(gh, 0), a.group_size - 1);
  b.c = (b.ctop * a.group_size + gh) * a.group_size + gw;
  return b;
}

// sample position (iw, ih) of a bin; false when it falls outside the map (:113-121)
__device__ __forceinline__ bool psroi_sample(const PsroiArgs &a, const PsroiBin &b, int iw, int ih, float *w, float *h) {
  float ww = __fadd_rn(b.wstart, __fmul_rn((float)iw, b.sub_w));
  float hh = __fadd_rn(b.hstart, __fmul_rn((float)ih, b.sub_h));
  if ((double)ww < -0.5 || (double)ww > (double)a.W - 0.5 || (double)hh < -0.5 || (double)hh > (double)a.H - 0.5) return false;
  *w = (float)fmin(fmax((double)ww, 0.), (double)a.W - 1.);
  *h = (float)fmin(fmax((double)hh, 0.), (double)a.H - 1.);
  return true;
}

__global__ void __launch_bounds__(256) k_psroi_forward(const PsroiArgs a, long long count, float *__restrict__ out,
                                                       float *__restrict__ top_count) {
  const long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (index >= count) return;
  const PsroiBin b = psroi_bin(a, index);
  if (b.batch < 0 || b.batch >= a.B) {   // roi names an image that does not exist: empty bin instead of a wild read
    out[index] = 0.f;
    top_count[index] = 0.f;
    return;
  }
  const float *pl = a.data + ((long long)b.batch * a.C + b.c) * a.H * a.W;
  float sum = 0.f;
  int cnt = 0;
  for (int ih = 0; ih < a.spp; ++ih)
    for (int iw = 0; iw < a.spp; ++iw) {
      float w, h;
      if (!psroi_sample(a, b, iw, ih, &w, &h)) continue;
      const int x1 = (int)floorf(w), x2 = (int)ceilf(w), y1 = (int)floorf(h), y2 = (int)ceilf(h);   // :24-45
      const float dx = w - (float)x1, dy = h - (float)y1;
      const float v11 = pl[y1 * a.W + x1], v12 = pl[y2 * a.W + x1], v21 = pl[y1 * a.W + x2], v22 = pl[y2 * a.W + x2];
      const float val = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(1.f - dx, 1.f - dy), v11),
                                                       __fmul_rn(__fmul_rn(1.f - dx, dy), v12)),
                                            __fmul_rn(__fmul_rn(dx, 1.f - dy), v21)),
                                  __fmul_rn(__fmul_rn(dx, dy), v22));
      sum = __fadd_rn(sum, val);
      ++cnt;
    }
  out[index] = cnt == 0 ? 0.f : sum / (float)cnt;
  top_count[index] = (float)cnt;
}

__global__ void __launch_bounds__(256) k_psroi_backward(const PsroiArgs a, long long count,
                                                        const float *__restrict__ top_diff,
                                                        const float *__restrict__ top_count, float *grad_data,
                                                        float *grad_trans) {
  const long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (index >= count) return;
  if (top_count[index] <= 0.f) return;
  const PsroiBin b = psroi_bin(a, index);
  if (b.batch < 0 || b.batch >= a.B) return;
  const float dv = top_diff[index] / top_count[index];
  const long long plane = ((long long)b.batch * a.C + b.c) * a.H * a.W;
  const float *pl = a.data + plane;
  float *gp = grad_data + plane;
  float gx = 0.f, gy = 0.f;
  for (int ih = 0; ih < a.spp; ++ih)
    for (int iw = 0; iw < a.spp; ++iw) {
      float w, h;
      if (!psroi_sample(a, b, iw, ih, &w, &h)) continue;
      const int x0 = (int)floorf(w), x1 = (int)ceilf(w), y0 = (int)floorf(h), y1 = (int)ceilf(h);
      const float dx = w - (float)x0, dy = h - (float)y0;
      atomicAdd(gp + y0 * a.W + x0, (1.f - dx) * (1.f - dy) * dv);   // :223-231
      atomicAdd(gp + y1 * a.W + x0, (1.f - dx) * dy * dv);
      atomicAdd(gp + y0 * a.W + x1, dx * (1.f - dy) * dv);
      atomicAdd(gp + y1 * a.W + x1, dx * dy * dv);
      if (a.no_trans) continue;
      const float u00 = pl[y0 * a.W + x0], u01 = pl[y1 * a.W + x0], u10 = pl[y0 * a.W + x1], u11 = pl[y1 * a.W + x1];
      gx += (u11 * dy + u10 * (1.f - dy) - u01 * dy - u00 * (1.f - dy)) * a.trans_std * dv * b.roi_w;   // :241-246
      gy += (u11 * dx + u01 * (1.f - dx) - u10 * dx - u00 * (1.f - dx)) * a.trans_std * dv * b.roi_h;
    }
  if (!a.no_trans) {  // one atomic per bin and direction (the reference issues one per sample)
    const long long t0 = (((long long)b.n * a.num_classes + b.cls) * 2) * a.part_size;
    atomicAdd(grad_trans + (t0 + b.part_h) * a.part_size + b.part_w, gx);
    atomicAdd(grad_trans + (t0 + a.part_size + b.part_h) * a.part_size + b.part_w, gy);
  }
}

static int fill_args(const char *who, PsroiArgs *a, const float *data, const float *rois, const float *trans, int b,
                     int c, int h, int w, int num_rois, int channels_trans, int no_trans, float spatial_scale,
                     int output_dim, int group_size, int pooled_size, int part_size, int sample_per_part,
                     float trans_std) {
  CNB_REQUIRE(data && rois, CNB_EINVAL, "%s: null pointer", who);
  CNB_REQUIRE(b > 0 && c > 0 && h > 0 && w > 0 && num_rois >= 0, CNB_EINVAL, "%s: bad shape", who);
  CNB_REQUIRE(output_dim > 0 && group_size > 0 && pooled_size > 0 && part_size > 0 && sample_per_part > 0, CNB_EINVAL,
              "%s: non-positive pooling parameter", who);
  CNB_REQUIRE(c >= output_dim * group_size * group_size, CNB_EINVAL,
              "%s: input has %d channels, output_dim * group_size^2 = %d needed", who, c,
              output_dim * group_size * group_size);
  CNB_REQUIRE(no_trans || (trans && channels_trans >= 2 && channels_trans % 2 == 0), CNB_EINVAL,
              "%s: offsets need an even, positive channel count (got %d)", who, channels_trans);
  a->data = data; a->rois = rois; a->trans = no_trans ? nullptr : trans;
  a->B = b; a->C = c; a->H = h; a->W = w; a->N = num_rois;
  a->no_trans = no_trans; a->output_dim = output_dim; a->group_size = group_size; a->P = pooled_size;
  a->part_size = part_size; a->spp = sample_per_part; a->spatial_scale = spatial_scale; a->trans_std = trans_std;
  a->num_classes = no_trans ? 1 : channels_trans / 2;                     // :282-283
  a->ch_each = no_trans ? output_dim : output_dim / a->num_classes;
  CNB_REQUIRE(a->ch_each > 0, CNB_EINVAL, "%s: output_dim %d < number of offset classes %d", who, output_dim,
              a->num_classes);
  return CNB_OK;
}

// ------------------------------------------------------------------ float64 (dcn_v2_psroi_pooling_cuda_double.cu)
// The double source computes the window geometry in double throughout (:88-116), so these kernels do too.  The
// backward is bit-reproducible: grad_data goes through the fixed-point accumulator of fx64.cuh, and each grad_trans
// element has one writer that walks the bins and samples of its (roi, class, part) in a fixed order.
struct Psroi64Args {
  const double *data, *rois, *trans;
  int B, C, H, W, N, no_trans, output_dim, group_size, P, part_size, spp, num_classes, ch_each;
  double spatial_scale, trans_std;
};

struct Bin64 {
  int batch, c, cls, part_h, part_w;
  double wstart, hstart, sub_w, sub_h, roi_w, roi_h;
};

__device__ __forceinline__ Bin64 psroi_bin64(const Psroi64Args &a, int n, int ctop, int ph, int pw) {
  Bin64 b;
  const int P = a.P;
  const double *r = a.rois + (long long)n * 5;
  b.batch = (int)r[0];
  const double start_w = (double)(round(r[1])) * a.spatial_scale - 0.5;
  const double start_h = (double)(round(r[2])) * a.spatial_scale - 0.5;
  const double end_w = (double)(round(r[3]) + 1.) * a.spatial_scale - 0.5;
  const double end_h = (double)(round(r[4]) + 1.) * a.spatial_scale - 0.5;
  b.roi_w = fmax(end_w - start_w, 0.1);
  b.roi_h = fmax(end_h - start_h, 0.1);
  const double bin_h = b.roi_h / (double)P, bin_w = b.roi_w / (double)P;
  b.sub_h = bin_h / (double)a.spp;
  b.sub_w = bin_w / (double)a.spp;
  b.part_h = (int)floor((double)ph / P * a.part_size);
  b.part_w = (int)floor((double)pw / P * a.part_size);
  b.cls = ctop / a.ch_each;
  double tx = 0, ty = 0;
  if (!a.no_trans) {
    tx = a.trans[(((long long)(n * a.num_classes + b.cls) * 2) * a.part_size + b.part_h) * a.part_size + b.part_w] *
         a.trans_std;
    ty = a.trans[(((long long)(n * a.num_classes + b.cls) * 2 + 1) * a.part_size + b.part_h) * a.part_size +
                 b.part_w] *
         a.trans_std;
  }
  b.wstart = (double)pw * bin_w + start_w;
  b.wstart += tx * b.roi_w;
  b.hstart = (double)ph * bin_h + start_h;
  b.hstart += ty * b.roi_h;
  int gw = (int)floor((double)pw * a.group_size / P), gh = (int)floor((double)ph * a.group_size / P);
  gw = min(max(gw, 0), a.group_size - 1);
  gh = min(max(gh, 0), a.group_size - 1);
  b.c = (ctop * a.group_size + gh) * a.group_size + gw;
  return b;
}

__device__ __forceinline__ bool psroi_sample64(const Psroi64Args &a, const Bin64 &b, int iw, int ih, double *w,
                                               double *h) {
  double ww = b.wstart + iw * b.sub_w, hh = b.hstart + ih * b.sub_h;
  if (ww < -0.5 || ww > a.W - 0.5 || hh < -0.5 || hh > a.H - 0.5) return false;
  *w = fmin(fmax(ww, 0.), a.W - 1.);
  *h = fmin(fmax(hh, 0.), a.H - 1.);
  return true;
}

__global__ void __launch_bounds__(256) k_psroi64_forward(const Psroi64Args a, long long count, double *out,
                                                         double *top_count) {
  const long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (index >= count) return;
  const int P = a.P, pw = (int)(index % P), ph = (int)((index / P) % P);
  const int ctop = (int)((index / P / P) % a.output_dim), n = (int)(index / P / P / a.output_dim);
  const Bin64 b = psroi_bin64(a, n, ctop, ph, pw);
  if (b.batch < 0 || b.batch >= a.B) {
    out[index] = 0;
    top_count[index] = 0;
    return;
  }
  const double *pl = a.data + ((long long)b.batch * a.C + b.c) * a.H * a.W;
  double sum = 0;
  int cnt = 0;
  for (int ih = 0; ih < a.spp; ++ih)
    for (int iw = 0; iw < a.spp; ++iw) {
      double w, h;
      if (!psroi_sample64(a, b, iw, ih, &w, &h)) continue;
      const int x1 = (int)floor(w), x2 = (int)ceil(w), y1 = (int)floor(h), y2 = (int)ceil(h);   // bilinear_interp
      const double dx = w - x1, dy = h - y1;
      sum += (1 - dx) * (1 - dy) * pl[y1 * a.W + x1] + (1 - dx) * dy * pl[y2 * a.W + x1] +
             dx * (1 - dy) * pl[y1 * a.W + x2] + dx * dy * pl[y2 * a.W + x2];
      ++cnt;
    }
  out[index] = cnt == 0 ? 0.0 : sum / cnt;
  top_count[index] = cnt;
}

// grad_data: every sample of a bin scatters its four bilinear weights * top_diff / count
__global__ void __launch_bounds__(256) k_psroi64_backward_data(const Psroi64Args a, long long count,
                                                               const double *__restrict__ top_diff,
                                                               const double *__restrict__ top_count,
                                                               const FxParam *__restrict__ prm,
                                                               unsigned long long *hi, unsigned long long *lo) {
  const long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (index >= count || top_count[index] <= 0) return;
  const FxParam f = prm[0];
  if (f.bad) return;
  const int P = a.P, pw = (int)(index % P), ph = (int)((index / P) % P);
  const int ctop = (int)((index / P / P) % a.output_dim), n = (int)(index / P / P / a.output_dim);
  const Bin64 b = psroi_bin64(a, n, ctop, ph, pw);
  if (b.batch < 0 || b.batch >= a.B) return;
  const double dv = top_diff[index] / top_count[index];
  const long long plane = ((long long)b.batch * a.C + b.c) * a.H * a.W;
  for (int ih = 0; ih < a.spp; ++ih)
    for (int iw = 0; iw < a.spp; ++iw) {
      double w, h;
      if (!psroi_sample64(a, b, iw, ih, &w, &h)) continue;
      const int x0 = (int)floor(w), x1 = (int)ceil(w), y0 = (int)floor(h), y1 = (int)ceil(h);
      const double dx = w - x0, dy = h - y0;
      fx_add(hi, lo, plane + y0 * a.W + x0, (1 - dx) * (1 - dy) * dv, f);
      fx_add(hi, lo, plane + y1 * a.W + x0, (1 - dx) * dy * dv, f);
      fx_add(hi, lo, plane + y0 * a.W + x1, dx * (1 - dy) * dv, f);
      fx_add(hi, lo, plane + y1 * a.W + x1, dx * dy * dv, f);
    }
}

// grad_trans: one thread per (roi, class, part_h, part_w) walks the bins (ctop, ph, pw) of that part and their
// samples in order, adding both directions' terms (:256-266)
__global__ void __launch_bounds__(128) k_psroi64_backward_trans(const Psroi64Args a, long long count,
                                                                const double *__restrict__ top_diff,
                                                                const double *__restrict__ top_count,
                                                                double *grad_trans) {
  const long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (index >= count) return;
  const int PS = a.part_size, part_w = (int)(index % PS), part_h = (int)((index / PS) % PS);
  const int cls = (int)((index / PS / PS) % a.num_classes), n = (int)(index / PS / PS / a.num_classes);
  const int P = a.P;
  double gx = 0, gy = 0;
  for (int j = 0; j < a.ch_each * P * P; ++j) {   // bins (ctop, ph, pw) of the class in row-major order
    const int pw = j % P, ph = (j / P) % P, ctop = cls * a.ch_each + j / (P * P);
    if ((int)floor((double)ph / P * PS) != part_h || (int)floor((double)pw / P * PS) != part_w) continue;
    const long long bin = (((long long)n * a.output_dim + ctop) * P + ph) * P + pw;
    if (top_count[bin] <= 0) continue;
    const Bin64 b = psroi_bin64(a, n, ctop, ph, pw);
    if (b.batch < 0 || b.batch >= a.B) continue;
    const double dv = top_diff[bin] / top_count[bin];
    const double *pl = a.data + ((long long)b.batch * a.C + b.c) * a.H * a.W;
    for (int s = 0; s < a.spp * a.spp; ++s) {
      const int ih = s / a.spp, iw = s - ih * a.spp;
      double w, h;
      if (!psroi_sample64(a, b, iw, ih, &w, &h)) continue;
      const int x0 = (int)floor(w), x1 = (int)ceil(w), y0 = (int)floor(h), y1 = (int)ceil(h);
      const double dx = w - x0, dy = h - y0;
      const double u00 = pl[y0 * a.W + x0], u01 = pl[y1 * a.W + x0], u10 = pl[y0 * a.W + x1], u11 = pl[y1 * a.W + x1];
      double diff_x = (u11 * dy + u10 * (1 - dy) - u01 * dy - u00 * (1 - dy)) * a.trans_std * dv;
      diff_x *= b.roi_w;
      double diff_y = (u11 * dx + u01 * (1 - dx) - u10 * dx - u00 * (1 - dx)) * a.trans_std * dv;
      diff_y *= b.roi_h;
      gx += diff_x;
      gy += diff_y;
    }
  }
  const long long t0 = (((long long)n * a.num_classes + cls) * 2) * PS;
  grad_trans[(t0 + part_h) * PS + part_w] += gx;
  grad_trans[(t0 + PS + part_h) * PS + part_w] += gy;
}

// |grad_data| <= N * P^2 * max|top_diff|: an element of channel c only receives from the N * P^2 bins that read c,
// and a bin's samples add at most count * |top_diff| / count to it
__global__ void k_psroi64_params(const unsigned long long *__restrict__ bits, double nbins_per_channel, double count,
                                 FxParam *prm) {
  const unsigned long long m = bits[0];
  prm[0] = fx_param(nbins_per_channel * __longlong_as_double(m), count, m < kInfBits64);
}

static int fill_args64(const char *who, Psroi64Args *a, const double *data, const double *rois, const double *trans,
                       int b, int c, int h, int w, int num_rois, int channels_trans, int no_trans,
                       double spatial_scale, int output_dim, int group_size, int pooled_size, int part_size,
                       int sample_per_part, double trans_std) {
  CNB_REQUIRE(data && rois, CNB_EINVAL, "%s: null pointer", who);
  CNB_REQUIRE(b > 0 && c > 0 && h > 0 && w > 0 && num_rois >= 0 && (long long)h * w < (1ll << 31), CNB_EINVAL,
              "%s: bad shape", who);
  CNB_REQUIRE(output_dim > 0 && group_size > 0 && pooled_size > 0 && part_size > 0 && sample_per_part > 0, CNB_EINVAL,
              "%s: non-positive pooling parameter", who);
  CNB_REQUIRE(c >= output_dim * group_size * group_size, CNB_EINVAL,
              "%s: input has %d channels, output_dim * group_size^2 = %d needed", who, c,
              output_dim * group_size * group_size);
  CNB_REQUIRE(no_trans || (trans && channels_trans >= 2 && channels_trans % 2 == 0), CNB_EINVAL,
              "%s: offsets need an even, positive channel count (got %d)", who, channels_trans);
  a->data = data; a->rois = rois; a->trans = no_trans ? nullptr : trans;
  a->B = b; a->C = c; a->H = h; a->W = w; a->N = num_rois;
  a->no_trans = no_trans; a->output_dim = output_dim; a->group_size = group_size; a->P = pooled_size;
  a->part_size = part_size; a->spp = sample_per_part; a->spatial_scale = spatial_scale; a->trans_std = trans_std;
  a->num_classes = no_trans ? 1 : channels_trans / 2;
  a->ch_each = no_trans ? output_dim : output_dim / a->num_classes;
  // a remainder would make the reference index offsets of a class that does not exist
  CNB_REQUIRE(a->ch_each > 0 && output_dim % a->num_classes == 0, CNB_EINVAL,
              "%s: output_dim %d is not a multiple of the number of offset classes %d", who, output_dim,
              a->num_classes);
  return CNB_OK;
}

static size_t psroi64_ws(int b, int c, int h, int w) {
  return 256 + 256 + 2 * align_up((size_t)b * c * h * w * 8, 256);
}

}  // namespace cnb

using namespace cnb;

extern "C" {

int cnb_psroi_pooling_forward(const float *data, const float *rois, const float *trans, float *out, float *top_count,
                              int b, int c, int h, int w, int num_rois, int channels_trans, int no_trans,
                              float spatial_scale, int output_dim, int group_size, int pooled_size, int part_size,
                              int sample_per_part, float trans_std, void *stream) {
  PsroiArgs a;
  int rc = fill_args("cnb_psroi_pooling_forward", &a, data, rois, trans, b, c, h, w, num_rois, channels_trans, no_trans,
                     spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part, trans_std);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(out && top_count, CNB_EINVAL, "cnb_psroi_pooling_forward: null output");
  const long long count = (long long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return CNB_OK;
  k_psroi_forward<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, count, out, top_count);
  CNB_CHECK_LAUNCH("cnb_psroi_pooling_forward");
  count_launch();
  return CNB_OK;
}

int cnb_psroi_pooling_backward(const float *grad_out, const float *data, const float *rois, const float *trans,
                               const float *top_count, float *grad_data, float *grad_trans, int b, int c, int h, int w,
                               int num_rois, int channels_trans, int no_trans, float spatial_scale, int output_dim,
                               int group_size, int pooled_size, int part_size, int sample_per_part, float trans_std,
                               void *stream) {
  PsroiArgs a;
  int rc = fill_args("cnb_psroi_pooling_backward", &a, data, rois, trans, b, c, h, w, num_rois, channels_trans,
                     no_trans, spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part, trans_std);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(grad_out && top_count && grad_data && (no_trans || grad_trans), CNB_EINVAL,
              "cnb_psroi_pooling_backward: null pointer");
  const long long count = (long long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return CNB_OK;
  k_psroi_backward<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, count, grad_out, top_count,
                                                                                      grad_data, grad_trans);
  CNB_CHECK_LAUNCH("cnb_psroi_pooling_backward");
  count_launch();
  return CNB_OK;
}

size_t cnb_psroi_pooling_f64_workspace_bytes(int b, int c, int h, int w) {
  if (b <= 0 || c <= 0 || h <= 0 || w <= 0) return 0;
  return psroi64_ws(b, c, h, w);
}

int cnb_psroi_pooling_forward_f64(const double *data, const double *rois, const double *trans, double *out,
                                  double *top_count, int b, int c, int h, int w, int num_rois, int channels_trans,
                                  int no_trans, double spatial_scale, int output_dim, int group_size, int pooled_size,
                                  int part_size, int sample_per_part, double trans_std, void *stream) {
  Psroi64Args a;
  int rc = fill_args64("cnb_psroi_pooling_forward_f64", &a, data, rois, trans, b, c, h, w, num_rois, channels_trans,
                       no_trans, spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part,
                       trans_std);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(out && top_count, CNB_EINVAL, "cnb_psroi_pooling_forward_f64: null output");
  const long long count = (long long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return CNB_OK;
  k_psroi64_forward<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, count, out, top_count);
  CNB_CHECK_LAUNCH("cnb_psroi_pooling_forward_f64");
  count_launch();
  return CNB_OK;
}

int cnb_psroi_pooling_backward_f64(const double *grad_out, const double *data, const double *rois,
                                   const double *trans, const double *top_count, double *grad_data,
                                   double *grad_trans, int b, int c, int h, int w, int num_rois, int channels_trans,
                                   int no_trans, double spatial_scale, int output_dim, int group_size,
                                   int pooled_size, int part_size, int sample_per_part, double trans_std,
                                   void *workspace, size_t workspace_bytes, void *stream) {
  const char *who = "cnb_psroi_pooling_backward_f64";
  Psroi64Args a;
  int rc = fill_args64(who, &a, data, rois, trans, b, c, h, w, num_rois, channels_trans, no_trans, spatial_scale,
                       output_dim, group_size, pooled_size, part_size, sample_per_part, trans_std);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(grad_out && top_count && grad_data && (no_trans || grad_trans), CNB_EINVAL, "%s: null pointer", who);
  const size_t need = psroi64_ws(b, c, h, w);
  CNB_REQUIRE(workspace && workspace_bytes >= need, CNB_EINVAL,
              "%s: workspace of %zu bytes is smaller than the %zu cnb_psroi_pooling_f64_workspace_bytes asks for", who,
              workspace_bytes, need);
  CNB_REQUIRE(((uintptr_t)workspace & 15) == 0, CNB_EINVAL, "%s: workspace must be 16-byte aligned", who);
  const long long count = (long long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return CNB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  char *ws = (char *)workspace;
  unsigned long long *bits = (unsigned long long *)ws;
  FxParam *prm = (FxParam *)(ws + 256);
  const long long nd = (long long)b * c * h * w;
  const size_t limb = align_up((size_t)nd * 8, 256);
  unsigned long long *hi = (unsigned long long *)(ws + 512), *lo = (unsigned long long *)(ws + 512 + limb);
  CNB_CUDA(cudaMemsetAsync(ws, 0, 512 + 2 * limb, st));
  absmax_bits_launch(grad_out, count, 1, bits, st);
  const double per_channel = (double)num_rois * pooled_size * pooled_size;
  k_psroi64_params<<<1, 1, 0, st>>>(bits, per_channel, 4.0 * per_channel * sample_per_part * sample_per_part, prm);
  k_psroi64_backward_data<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(a, count, grad_out, top_count, prm, hi,
                                                                           lo);
  CNB_CHECK_LAUNCH(who);
  count_launch(2);
  rc = fx_finish_launch(hi, lo, prm, nd, nd, grad_data, st);
  if (rc != CNB_OK) return rc;
  if (!no_trans) {
    const long long nt = (long long)num_rois * a.num_classes * part_size * part_size;
    k_psroi64_backward_trans<<<(unsigned)((nt + 127) / 128), 128, 0, st>>>(a, nt, grad_out, top_count, grad_trans);
    CNB_CHECK_LAUNCH(who);
    count_launch();
  }
  return CNB_OK;
}

}  // extern "C"

// Training input of the ctdet sampler on the device (datasets/sample/ctdet.py:29-145, utils/image.py:198-230):
// the random crop / flip warp, /255, color_aug, the normalisation and the layout change of a whole batch of
// ragged uint8 sources, and the ctdet regression targets plus the object lists of FocalSplatLoss.  Every value
// is the one the reference's loader computes for the same drawn parameters, bit for bit; no atomics, so the
// output is also identical run to run.  The numeric contract is DESIGN.md section 4.9.
#include <map>

#include "common.cuh"
#include "warp.cuh"

namespace cnb {
namespace {

constexpr int kThreads = 256;
constexpr int kLeafLog = 8;        // depth-D slots per block of the grey pass (a subtree of 256 slots)
constexpr int kMaxTopLog = 8;      // the top of the tree, combined by every block of the image pass
constexpr int kPairwiseLeaf = 128; // numpy's PW_BLOCKSIZE

// ---------------------------------------------------------------- numpy's pairwise float32 sum (gs.mean())
// sum(a[0:n]): n < 8 sequentially; n <= 128 eight strided accumulators, ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)),
// then the n % 8 tail in order; n > 128 sum(a[:n2]) + sum(a[n2:]) with n2 = n/2 - (n/2) % 8.  The tree depends
// on n alone.  Node j at depth d is addressed by the bits of j (MSB first: 0 = left); its value is kept in
// slot j << (D - d) of an array over the depth-D nodes, D the depth of the deepest leaf.

// 0: node (d, j) does not exist (below a leaf), 1: leaf, 2: internal.  *start / *len: its element range.
__host__ __device__ __forceinline__ int pw_node(long long n, int d, long long j, long long *start, long long *len) {
  long long s = 0, l = n;
  for (int i = d - 1; i >= 0; --i) {
    if (l <= kPairwiseLeaf) return 0;
    long long h = l / 2;
    h -= h % 8;
    if ((j >> i) & 1) {
      s += h;
      l -= h;
    } else {
      l = h;
    }
  }
  *start = s;
  *len = l;
  return l <= kPairwiseLeaf ? 1 : 2;
}

int pw_depth(long long n, std::map<long long, int> &memo) {
  if (n <= kPairwiseLeaf) return 0;
  auto it = memo.find(n);
  if (it != memo.end()) return it->second;
  long long h = n / 2;
  h -= h % 8;
  const int d = 1 + std::max(pw_depth(h, memo), pw_depth(n - h, memo));
  memo[n] = d;
  return d;
}

int pw_depth(long long n) {
  std::map<long long, int> memo;
  return pw_depth(n, memo);
}

// v[j - j0] holds the values of the depth-dbot nodes j0 .. j0 + 2^(dbot - dtop) - 1 (j0 aligned); combines the
// levels dbot - 1 .. dtop in place, so that v[0] ends up holding node (dtop, j0 >> (dbot - dtop)).
__device__ void pw_combine(float *v, long long n, int dbot, int dtop, long long j0) {
  for (int lvl = dbot - 1; lvl >= dtop; --lvl) {
    const int sh = dbot - lvl;
    const int cnt = 1 << (lvl - dtop);
    for (int u = threadIdx.x; u < cnt; u += blockDim.x) {
      long long s, l;
      if (pw_node(n, lvl, (j0 >> sh) + u, &s, &l) == 2) v[u << sh] = __fadd_rn(v[u << sh], v[(u << sh) + (1 << (sh - 1))]);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- per-image records
struct ImageRec {
  const unsigned char *img;
  int H, W, flip, order;
  bool ok;
};

// Blend orders of color_aug's random.shuffle over [brightness_, contrast_, saturation_] (kinds 0, 1, 2), the six
// permutations in lexicographic order.
__constant__ unsigned char kOrders[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};

__device__ __forceinline__ ImageRec load_rec(const unsigned char *src, const long long *src_off, const int *src_hw,
                                             const unsigned char *flip, const int *order, int b) {
  ImageRec r;
  r.img = src + src_off[b];
  r.H = src_hw[2 * b];
  r.W = src_hw[2 * b + 1];
  r.flip = flip[b] ? 1 : 0;
  r.order = order ? order[b] : -1;
  r.ok = r.H >= 1 && r.H <= 32767 && r.W >= 1 && r.W <= 32767 && r.order >= -1 && r.order < 6;
  return r;
}

// cv2.warpAffine of the (optionally mirrored, img[:, ::-1]) source at output pixel (x, y): the mirrored image is
// sampled at mirrored columns, never materialised.
__device__ __forceinline__ void warp_px(const ImageRec &r, const double *__restrict__ minv, int x, int y, int v[3]) {
  const WarpTaps t = warp_taps(minv, x, y, r.H, r.W);
  const int c0 = r.flip ? r.W - 1 - t.sx : t.sx, c1 = r.flip ? r.W - 2 - t.sx : t.sx + 1;
  const bool k00 = t.y0ok && t.x0ok, k01 = t.y0ok && t.x1ok, k10 = t.y1ok && t.x0ok, k11 = t.y1ok && t.x1ok;
  const unsigned char *row0 = r.img + (size_t)t.sy * r.W * 3, *row1 = row0 + (size_t)r.W * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int p00 = k00 ? row0[(size_t)c0 * 3 + c] : 0;
    const int p01 = k01 ? row0[(size_t)c1 * 3 + c] : 0;
    const int p10 = k10 ? row1[(size_t)c0 * 3 + c] : 0;
    const int p11 = k11 ? row1[(size_t)c1 * 3 + c] : 0;
    const int s = (p00 * t.w0 + p01 * t.w1 + p10 * t.w2 + p11 * t.w3 + (1 << 14)) >> 15;
    v[c] = min(max(s, 0), 255);
  }
}

// cv2.cvtColor(float32 BGR -> GRAY) of the /255 image.
__device__ __forceinline__ float grey(const float x[3]) {
  return __fmaf_rn(x[2], 0.299f, __fmaf_rn(x[0], 0.114f, __fmul_rn(x[1], 0.587f)));
}

__device__ __forceinline__ float grey_at(const ImageRec &r, const double *minv, long long p, int ow) {
  int v[3];
  warp_px(r, minv, (int)(p % ow), (int)(p / ow), v);
  float x[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) x[c] = __fdiv_rn((float)v[c], 255.f);
  return grey(x);
}

// Phase 1: one thread per depth-D slot; the thread that owns a leaf sums its grey values as numpy does, then each
// block combines its 2^kLeafLog slots up to depth D - kLeafLog and stores that node's partial sum.
__global__ void __launch_bounds__(kThreads) k_train_grey(const unsigned char *__restrict__ src,
                                                          const long long *__restrict__ src_off,
                                                          const int *__restrict__ src_hw,
                                                          const double *__restrict__ minv,
                                                          const unsigned char *__restrict__ flip,
                                                          const int *__restrict__ order, int oh, int ow, int depth,
                                                          int leaf_log, float *__restrict__ top) {
  __shared__ float v[1 << kLeafLog];
  const int b = blockIdx.y;
  const ImageRec r = load_rec(src, src_off, src_hw, flip, order, b);
  if (!r.ok || r.order < 0) return;   // uniform per block
  const double *mv = minv + 6 * b;
  const long long n = (long long)oh * ow;
  const long long slot = ((long long)blockIdx.x << leaf_log) + threadIdx.x;
  // the leaf above this slot, and whether the slot is its leftmost (owning) one
  long long s = 0, l = n;
  int dl = 0;
  while (dl < depth && l > kPairwiseLeaf) {
    long long h = l / 2;
    h -= h % 8;
    if ((slot >> (depth - 1 - dl)) & 1) {
      s += h;
      l -= h;
    } else {
      l = h;
    }
    ++dl;
  }
  const bool owner = (slot & ((1ll << (depth - dl)) - 1)) == 0;
  if (owner) {
    float acc;
    if (l < 8) {
      acc = 0.f;
      for (long long i = 0; i < l; ++i) acc = __fadd_rn(acc, grey_at(r, mv, s + i, ow));
    } else {
      float a[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = grey_at(r, mv, s + j, ow);
      long long i = 8;
      for (; i < l - (l % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = __fadd_rn(a[j], grey_at(r, mv, s + i + j, ow));
      }
      acc = __fadd_rn(__fadd_rn(__fadd_rn(a[0], a[1]), __fadd_rn(a[2], a[3])),
                      __fadd_rn(__fadd_rn(a[4], a[5]), __fadd_rn(a[6], a[7])));
      for (; i < l; ++i) acc = __fadd_rn(acc, grey_at(r, mv, s + i, ow));
    }
    v[threadIdx.x] = acc;
  }
  __syncthreads();
  pw_combine(v, n, depth, depth - leaf_log, (long long)blockIdx.x << leaf_log);
  if (threadIdx.x == 0) top[((size_t)b << (depth - leaf_log)) + blockIdx.x] = v[0];
}

template <typename T>
__device__ __forceinline__ T from_f32(float f);
template <>
__device__ __forceinline__ float from_f32<float>(float f) { return f; }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float f) { return __float2bfloat16_rn(f); }
template <>
__device__ __forceinline__ __half from_f32<__half>(float f) { return __float2half_rn(f); }

// Phase 2: warp again, /255, the three blends in the drawn order, the lighting, (x - mean) / std, one store per
// channel.  Grid (x tiles, rows, images).
template <typename T>
__global__ void __launch_bounds__(kThreads) k_train_images(const unsigned char *__restrict__ src,
                                                            const long long *__restrict__ src_off,
                                                            const int *__restrict__ src_hw,
                                                            const double *__restrict__ minv,
                                                            const unsigned char *__restrict__ flip,
                                                            const int *__restrict__ order,
                                                            const float *__restrict__ blend,
                                                            const double *__restrict__ light,
                                                            const float *__restrict__ mean,
                                                            const float *__restrict__ stdv, int oh, int ow, int depth,
                                                            int top_log, const float *__restrict__ top,
                                                            int channels_last, T *__restrict__ out) {
  __shared__ float v[1 << kMaxTopLog];
  const int b = blockIdx.z, y = blockIdx.y, x = blockIdx.x * blockDim.x + threadIdx.x;
  const ImageRec r = load_rec(src, src_off, src_hw, flip, order, b);
  float mb = 0.f;   // f32(gs_mean * (1 - alpha)) of contrast_
  if (r.ok && r.order >= 0) {
    const long long n = (long long)oh * ow;
    for (int i = threadIdx.x; i < (1 << top_log); i += blockDim.x) v[i] = top[((size_t)b << top_log) + i];
    __syncthreads();
    pw_combine(v, n, top_log, 0, 0);
    mb = __fmul_rn(__fdiv_rn(v[0], (float)n), blend[6 * b + 3]);
  }
  if (x >= ow) return;
  float f[3];
  if (!r.ok) {
    f[0] = f[1] = f[2] = __int_as_float(0x7fc00000);
  } else {
    int px[3];
    warp_px(r, minv + 6 * b, x, y, px);
#pragma unroll
    for (int c = 0; c < 3; ++c) f[c] = __fdiv_rn((float)px[c], 255.f);
    if (r.order >= 0) {
      const float g = grey(f);
      const float *ab = blend + 6 * b;   // (a, b) of brightness_, contrast_, saturation_
      const float gb = __fmul_rn(g, ab[5]);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int kind = kOrders[r.order][k];
        const float a = ab[2 * kind];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float m = __fmul_rn(f[c], a);
          f[c] = kind == 0 ? m : __fadd_rn(m, kind == 1 ? mb : gb);
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) f[c] = __double2float_rn(__dadd_rn((double)f[c], light[3 * b + c]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) f[c] = __fdiv_rn(__fsub_rn(f[c], mean[c]), stdv[c]);
  }
  const size_t plane = (size_t)oh * ow;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const size_t o = channels_last ? ((size_t)b * plane + (size_t)y * ow + x) * 3 + c
                                   : ((size_t)b * 3 + c) * plane + (size_t)y * ow + x;
    out[o] = from_f32<T>(f[c]);
  }
}

// ---------------------------------------------------------------- ctdet targets (ctdet.py:99-127)
// gaussian_radius((ceil(h), ceil(w))) of utils/image.py:95-115 with its Python ints and float64 operations in
// the order the source evaluates them.
__device__ __forceinline__ double gaussian_radius_f64(long long height, long long width) {
  const double mo1 = 0.30000000000000004;   // 1 - 0.7, and -(0.7 - 1)
  const long long b1 = height + width;
  const double c1 = __ddiv_rn(__dmul_rn((double)(width * height), mo1), 1.7);
  const double r1 = __ddiv_rn(__dadd_rn((double)b1, __dsqrt_rn(__dsub_rn((double)(b1 * b1), __dmul_rn(4.0, c1)))), 2.0);
  const long long b2 = 2 * (height + width);
  const double c2 = __dmul_rn(__dmul_rn(mo1, (double)width), (double)height);
  const double r2 = __ddiv_rn(__dadd_rn((double)b2, __dsqrt_rn(__dsub_rn((double)(b2 * b2), __dmul_rn(16.0, c2)))), 2.0);
  const double a3 = 2.8;                    // 4 * 0.7
  const double b3 = __dmul_rn(-1.4, (double)(height + width));
  const double c3 = __dmul_rn(__dmul_rn(-mo1, (double)width), (double)height);
  const double sq3 = __dsqrt_rn(__dsub_rn(__dmul_rn(b3, b3), __dmul_rn(__dmul_rn(4.0, a3), c3)));
  const double r3 = __ddiv_rn(__dadd_rn(b3, sq3), 2.0);
  return fmin(fmin(r1, r2), r3);
}

// affine_transform (utils/image.py:62-65) in the plain float64 order t0 x + t1 y + t2, rounded to float32.
__device__ __forceinline__ float affine_f32(const double *t, float x, float y) {
  return __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(t[0], (double)x), __dmul_rn(t[1], (double)y)), t[2]));
}

__global__ void __launch_bounds__(kThreads) k_ctdet_targets(
    const float *__restrict__ boxes, const int *__restrict__ cls, const int *__restrict__ num_objs,
    const unsigned char *__restrict__ flip, const int *__restrict__ src_hw, const double *__restrict__ trans, int nb,
    int m, int num_classes, int oh, int ow, float *__restrict__ wh, long long *__restrict__ ind,
    float *__restrict__ reg, unsigned char *__restrict__ reg_mask, float *__restrict__ cat_spec_wh,
    unsigned char *__restrict__ cat_spec_mask, int *__restrict__ obj_cls, int *__restrict__ obj_cx,
    int *__restrict__ obj_cy, int *__restrict__ obj_radius, unsigned char *__restrict__ obj_valid) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nb * m) return;
  const int b = (int)(i / m), k = (int)(i % m);
  float w = 0.f, h = 0.f, rx = 0.f, ry = 0.f;
  int c = 0, cx = 0, cy = 0, rad = 0;
  bool valid = false;
  if (k < min(num_objs[b], m)) {
    const float *bb = boxes + i * 4;
    float x0 = bb[0], y0 = bb[1], x1 = bb[2], y1 = bb[3];
    if (flip[b]) {   // bbox[[0, 2]] = width - bbox[[2, 0]] - 1 in float32
      const float wd = (float)src_hw[2 * b + 1];
      const float nx0 = __fsub_rn(__fsub_rn(wd, x1), 1.f), nx1 = __fsub_rn(__fsub_rn(wd, x0), 1.f);
      x0 = nx0;
      x1 = nx1;
    }
    const double *t = trans + 6 * b;
    float p0 = affine_f32(t, x0, y0), q0 = affine_f32(t + 3, x0, y0);
    float p1 = affine_f32(t, x1, y1), q1 = affine_f32(t + 3, x1, y1);
    const float xm = (float)(ow - 1), ym = (float)(oh - 1);
    p0 = fminf(fmaxf(p0, 0.f), xm);
    p1 = fminf(fmaxf(p1, 0.f), xm);
    q0 = fminf(fmaxf(q0, 0.f), ym);
    q1 = fminf(fmaxf(q1, 0.f), ym);
    h = __fsub_rn(q1, q0);
    w = __fsub_rn(p1, p0);
    if (h > 0.f && w > 0.f) {
      const double r = gaussian_radius_f64((long long)ceilf(h), (long long)ceilf(w));
      rad = r > 0.0 ? (int)r : 0;   // max(0, int(radius))
      const float ctx = __fdiv_rn(__fadd_rn(p0, p1), 2.f), cty = __fdiv_rn(__fadd_rn(q0, q1), 2.f);
      cx = (int)ctx;
      cy = (int)cty;
      rx = __fsub_rn(ctx, (float)cx);
      ry = __fsub_rn(cty, (float)cy);
      c = cls[i];
      valid = true;
    } else {
      w = h = 0.f;
    }
  }
  wh[2 * i] = w;
  wh[2 * i + 1] = h;
  reg[2 * i] = rx;
  reg[2 * i + 1] = ry;
  ind[i] = valid ? (long long)cy * ow + cx : 0;
  reg_mask[i] = valid ? 1 : 0;
  obj_cls[i] = c;
  obj_cx[i] = cx;
  obj_cy[i] = cy;
  obj_radius[i] = rad;
  obj_valid[i] = valid ? 1 : 0;
  if (cat_spec_wh) {
    float *sw = cat_spec_wh + i * 2 * num_classes;
    unsigned char *sm = cat_spec_mask + i * 2 * num_classes;
    for (int j = 0; j < num_classes; ++j) {
      const bool on = valid && j == c;
      sw[2 * j] = on ? w : 0.f;
      sw[2 * j + 1] = on ? h : 0.f;
      sm[2 * j] = sm[2 * j + 1] = on ? 1 : 0;
    }
  }
}

// ---------------------------------------------------------------- multi_pose targets (multi_pose.py:104-160)
// One thread per (image, slot), looping over the joints; the box half is k_ctdet_targets' arithmetic.  A slot gets
// targets when (h > 0 && w > 0) || rotated; reg_mask is 1 only when it has a visible joint (num_kpts != 0: the
// visibilities are finite and >= 0, checked on the host, so the float32 sum is 0 exactly when all are) and the
// image is not rotated.  The centre list is "got targets": hm[cls, ct] = 0.9999 for num_kpts == 0 is overwritten
// by the Gaussian's peak of 1 on the next line of the reference.
__global__ void __launch_bounds__(kThreads) k_multi_pose_targets(
    const float *__restrict__ boxes, const int *__restrict__ cls, const int *__restrict__ num_objs,
    const float *__restrict__ kps, const unsigned char *__restrict__ flip, const unsigned char *__restrict__ rotated,
    const int *__restrict__ src_hw, const double *__restrict__ trans, const double *__restrict__ trans_rot,
    const int *__restrict__ perm, int nb, int m, int nj, int res, float *__restrict__ wh, long long *__restrict__ ind,
    float *__restrict__ reg, unsigned char *__restrict__ reg_mask, float *__restrict__ hps,
    unsigned char *__restrict__ hps_mask, float *__restrict__ hp_offset, long long *__restrict__ hp_ind,
    long long *__restrict__ hp_mask, int *__restrict__ obj_cls, int *__restrict__ obj_cx, int *__restrict__ obj_cy,
    int *__restrict__ obj_radius, unsigned char *__restrict__ obj_valid, int *__restrict__ hp_cx,
    int *__restrict__ hp_cy, int *__restrict__ hp_radius, unsigned char *__restrict__ hp_valid) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nb * m) return;
  const int b = (int)(i / m), k = (int)(i % m);
  const bool rot = rotated[b] != 0, fl = flip[b] != 0;
  const float wd = (float)src_hw[2 * b + 1];
  float w = 0.f, h = 0.f, rx = 0.f, ry = 0.f;
  int c = 0, cx = 0, cy = 0, rad = 0;
  bool valid = false, any_kpt = false;
  if (k < min(num_objs[b], m)) {
    const float *bb = boxes + i * 4;
    float x0 = bb[0], y0 = bb[1], x1 = bb[2], y1 = bb[3];
    if (fl) {   // bbox[[0, 2]] = width - bbox[[2, 0]] - 1 in float32
      const float nx0 = __fsub_rn(__fsub_rn(wd, x1), 1.f), nx1 = __fsub_rn(__fsub_rn(wd, x0), 1.f);
      x0 = nx0;
      x1 = nx1;
    }
    const double *t = trans + 6 * b;
    float p0 = affine_f32(t, x0, y0), q0 = affine_f32(t + 3, x0, y0);
    float p1 = affine_f32(t, x1, y1), q1 = affine_f32(t + 3, x1, y1);
    const float mx = (float)(res - 1);
    p0 = fminf(fmaxf(p0, 0.f), mx);
    p1 = fminf(fmaxf(p1, 0.f), mx);
    q0 = fminf(fmaxf(q0, 0.f), mx);
    q1 = fminf(fmaxf(q1, 0.f), mx);
    h = __fsub_rn(q1, q0);
    w = __fsub_rn(p1, p0);
    if ((h > 0.f && w > 0.f) || rot) {
      const double r = gaussian_radius_f64((long long)ceilf(h), (long long)ceilf(w));
      rad = r > 0.0 ? (int)r : 0;   // max(0, int(radius))
      const float ctx = __fdiv_rn(__fadd_rn(p0, p1), 2.f), cty = __fdiv_rn(__fadd_rn(q0, q1), 2.f);
      cx = (int)ctx;
      cy = (int)cty;
      rx = __fsub_rn(ctx, (float)cx);
      ry = __fsub_rn(cty, (float)cy);
      c = cls[i];
      valid = true;
    } else {
      w = h = 0.f;
    }
  }
  const float *pk = kps + i * nj * 3;
  const double *tr = trans_rot + 6 * b;
  for (int j = 0; j < nj; ++j) {
    const long long o = i * nj + j;                     // [b, k * nj + j] of hp_*, [b, k, j] of hps
    const long long l = ((long long)b * nj + j) * m + k; // [b, j, k] of the joint lists
    float hx = 0.f, hy = 0.f, ox = 0.f, oy = 0.f;
    int jx = 0, jy = 0;
    bool in = false;
    if (valid) {
      const float *q = pk + 3 * (fl ? perm[j] : j);
      const float v = q[2];
      any_kpt = any_kpt || v != 0.f;
      if (v > 0.f) {
        const float x = fl ? __fsub_rn(__fsub_rn(wd, q[0]), 1.f) : q[0];
        const float px = affine_f32(tr, x, q[1]), py = affine_f32(tr + 3, x, q[1]);
        if (px >= 0.f && px < (float)res && py >= 0.f && py < (float)res) {
          in = true;
          jx = (int)px;
          jy = (int)py;
          hx = __fsub_rn(px, (float)cx);
          hy = __fsub_rn(py, (float)cy);
          ox = __fsub_rn(px, (float)jx);
          oy = __fsub_rn(py, (float)jy);
        }
      }
    }
    hps[2 * o] = hx;
    hps[2 * o + 1] = hy;
    hps_mask[2 * o] = hps_mask[2 * o + 1] = (in && !rot) ? 1 : 0;
    hp_offset[2 * o] = ox;
    hp_offset[2 * o + 1] = oy;
    hp_ind[o] = in ? (long long)jy * res + jx : 0;
    hp_mask[o] = in ? 1 : 0;
    hp_cx[l] = jx;
    hp_cy[l] = jy;
    hp_radius[l] = in ? rad : 0;
    hp_valid[l] = in ? 1 : 0;
  }
  wh[2 * i] = w;
  wh[2 * i + 1] = h;
  reg[2 * i] = rx;
  reg[2 * i + 1] = ry;
  ind[i] = valid ? (long long)cy * res + cx : 0;
  reg_mask[i] = (valid && any_kpt && !rot) ? 1 : 0;
  obj_cls[i] = c;
  obj_cx[i] = cx;
  obj_cy[i] = cy;
  obj_radius[i] = rad;
  obj_valid[i] = valid ? 1 : 0;
}

// Depth of the grey tree and the number of its levels combined per block of the grey pass.
void grey_plan(int out_h, int out_w, int *depth, int *leaf_log) {
  *depth = pw_depth((long long)out_h * out_w);
  *leaf_log = std::min(*depth, kLeafLog);
}

}  // namespace
}  // namespace cnb

extern "C" size_t cnb_train_images_workspace_bytes(int b, int out_h, int out_w) {
  if (b <= 0 || out_h <= 0 || out_w <= 0 || (long long)out_h * out_w > CNB_TRAIN_MAX_PIXELS) return 0;
  int depth, leaf_log;
  cnb::grey_plan(out_h, out_w, &depth, &leaf_log);
  return (size_t)b * ((size_t)1 << (depth - leaf_log)) * sizeof(float);
}

extern "C" int cnb_train_images(const uint8_t *src, const int64_t *src_off, const int32_t *src_hw,
                                const double *minv6, const uint8_t *flip, const int32_t *order, const float *blend,
                                const double *light, const float *mean3, const float *std3, int b, int out_h,
                                int out_w, void *out, int out_dtype, int channels_last, void *workspace,
                                size_t workspace_bytes, void *stream) {
  CNB_REQUIRE(src && src_off && src_hw && minv6 && flip && mean3 && std3 && out, CNB_EINVAL,
              "cnb_train_images: null pointer");
  CNB_REQUIRE(!order || (blend && light), CNB_EINVAL, "cnb_train_images: colour augmentation needs blend and light");
  CNB_REQUIRE(b > 0 && b <= 65535 && out_h > 0 && out_h <= 65535 && out_w > 0, CNB_EINVAL,
              "cnb_train_images: bad shape (b = %d, out %d x %d)", b, out_h, out_w);
  CNB_REQUIRE(cnb::dtype_known(out_dtype), CNB_EINVAL, "cnb_train_images: unknown dtype code %d", out_dtype);
  CNB_REQUIRE(channels_last == 0 || channels_last == 1, CNB_EINVAL, "cnb_train_images: channels_last must be 0 or 1");
  CNB_REQUIRE((long long)out_h * out_w <= CNB_TRAIN_MAX_PIXELS, CNB_EUNSUPPORTED,
              "cnb_train_images: at most %d output pixels per image (got %d x %d)", CNB_TRAIN_MAX_PIXELS, out_h, out_w);
  int depth = 0, leaf_log = 0;
  if (order) {
    CNB_REQUIRE(workspace, CNB_EINVAL, "cnb_train_images: null workspace");
    const size_t need = cnb_train_images_workspace_bytes(b, out_h, out_w);
    CNB_REQUIRE(workspace_bytes >= need, CNB_EWORKSPACE, "cnb_train_images: workspace %zu < %zu bytes",
                workspace_bytes, need);
    cnb::grey_plan(out_h, out_w, &depth, &leaf_log);
    CNB_REQUIRE(depth - leaf_log <= cnb::kMaxTopLog, CNB_EUNSUPPORTED, "cnb_train_images: grey tree too deep");
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int top_log = depth - leaf_log;
  float *top = (float *)workspace;
  const long long *off = (const long long *)src_off;
  if (order) {
    dim3 g1((unsigned)(1u << top_log), (unsigned)b);
    cnb::k_train_grey<<<g1, 1 << leaf_log, 0, st>>>(src, off, src_hw, minv6, flip, order, out_h, out_w, depth, leaf_log,
                                                    top);
    CNB_CHECK_LAUNCH("cnb_train_images (grey)");
    cnb::count_launch();
  }
  dim3 g2((unsigned)((out_w + cnb::kThreads - 1) / cnb::kThreads), (unsigned)out_h, (unsigned)b);
#define CNB_TRAIN_LAUNCH(T)                                                                                        \
  cnb::k_train_images<T><<<g2, cnb::kThreads, 0, st>>>(src, off, src_hw, minv6, flip, order, blend, light, mean3,  \
                                                       std3, out_h, out_w, depth, top_log, top, channels_last,    \
                                                       (T *)out)
  if (out_dtype == CNB_DTYPE_F32)
    CNB_TRAIN_LAUNCH(float);
  else if (out_dtype == CNB_DTYPE_BF16)
    CNB_TRAIN_LAUNCH(__nv_bfloat16);
  else
    CNB_TRAIN_LAUNCH(__half);
#undef CNB_TRAIN_LAUNCH
  CNB_CHECK_LAUNCH("cnb_train_images");
  cnb::count_launch();
  return CNB_OK;
}

extern "C" int cnb_ctdet_targets(const float *boxes, const int32_t *cls, const int32_t *num_objs, const uint8_t *flip,
                                 const int32_t *src_hw, const double *trans6, int b, int m, int num_classes, int out_h,
                                 int out_w, float *wh, int64_t *ind, float *reg, uint8_t *reg_mask, float *cat_spec_wh,
                                 uint8_t *cat_spec_mask, int32_t *obj_cls, int32_t *obj_cx, int32_t *obj_cy,
                                 int32_t *obj_radius, uint8_t *obj_valid, void *stream) {
  CNB_REQUIRE(boxes && cls && num_objs && flip && src_hw && trans6 && wh && ind && reg && reg_mask && obj_cls &&
                  obj_cx && obj_cy && obj_radius && obj_valid,
              CNB_EINVAL, "cnb_ctdet_targets: null pointer");
  CNB_REQUIRE(!cat_spec_wh == !cat_spec_mask, CNB_EINVAL,
              "cnb_ctdet_targets: cat_spec_wh and cat_spec_mask are both given or both NULL");
  CNB_REQUIRE(b > 0 && m > 0 && num_classes > 0 && out_h > 0 && out_w > 0 && (long long)out_h * out_w <= INT32_MAX,
              CNB_EINVAL, "cnb_ctdet_targets: bad shape");
  const long long n = (long long)b * m;
  cnb::k_ctdet_targets<<<(unsigned)((n + cnb::kThreads - 1) / cnb::kThreads), cnb::kThreads, 0,
                         (cudaStream_t)stream>>>(boxes, cls, num_objs, flip, src_hw, trans6, b, m, num_classes, out_h,
                                                 out_w, wh, (long long *)ind, reg, reg_mask, cat_spec_wh, cat_spec_mask,
                                                 obj_cls, obj_cx, obj_cy, obj_radius, obj_valid);
  CNB_CHECK_LAUNCH("cnb_ctdet_targets");
  cnb::count_launch();
  return CNB_OK;
}

extern "C" int cnb_multi_pose_targets(const float *boxes, const int32_t *cls, const int32_t *num_objs,
                                      const float *kps, const uint8_t *flip, const uint8_t *rotated,
                                      const int32_t *src_hw, const double *trans6, const double *trans_rot6,
                                      const int32_t *flip_perm, int b, int m, int num_joints, int out_res, float *wh,
                                      int64_t *ind, float *reg, uint8_t *reg_mask, float *hps, uint8_t *hps_mask,
                                      float *hp_offset, int64_t *hp_ind, int64_t *hp_mask, int32_t *obj_cls,
                                      int32_t *obj_cx, int32_t *obj_cy, int32_t *obj_radius, uint8_t *obj_valid,
                                      int32_t *hp_cx, int32_t *hp_cy, int32_t *hp_radius, uint8_t *hp_valid,
                                      void *stream) {
  CNB_REQUIRE(boxes && cls && num_objs && kps && flip && rotated && src_hw && trans6 && trans_rot6 && flip_perm &&
                  wh && ind && reg && reg_mask && hps && hps_mask && hp_offset && hp_ind && hp_mask && obj_cls &&
                  obj_cx && obj_cy && obj_radius && obj_valid && hp_cx && hp_cy && hp_radius && hp_valid,
              CNB_EINVAL, "cnb_multi_pose_targets: null pointer");
  CNB_REQUIRE(b > 0 && m > 0 && num_joints > 0 && out_res > 0 && (long long)out_res * out_res <= INT32_MAX &&
                  (long long)b * m * num_joints <= INT32_MAX,
              CNB_EINVAL, "cnb_multi_pose_targets: bad shape (b = %d, m = %d, joints = %d, out_res = %d)", b, m,
              num_joints, out_res);
  const long long n = (long long)b * m;
  cnb::k_multi_pose_targets<<<(unsigned)((n + cnb::kThreads - 1) / cnb::kThreads), cnb::kThreads, 0,
                              (cudaStream_t)stream>>>(
      boxes, cls, num_objs, kps, flip, rotated, src_hw, trans6, trans_rot6, flip_perm, b, m, num_joints, out_res, wh,
      (long long *)ind, reg, reg_mask, hps, hps_mask, hp_offset, (long long *)hp_ind, (long long *)hp_mask, obj_cls,
      obj_cx, obj_cy, obj_radius, obj_valid, hp_cx, hp_cy, hp_radius, hp_valid);
  CNB_CHECK_LAUNCH("cnb_multi_pose_targets");
  cnb::count_launch();
  return CNB_OK;
}

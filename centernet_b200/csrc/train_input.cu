// Training input of the ctdet sampler on the device (datasets/sample/ctdet.py:29-145, utils/image.py:198-230):
// the random crop / flip warp, /255, color_aug, the normalisation and the layout change of a whole batch of
// ragged uint8 sources, and the ctdet regression targets plus the object lists of FocalSplatLoss.  Every value
// is the one the reference's loader computes for the same drawn parameters, bit for bit; no atomics, so the
// output is also identical run to run.  The numeric contract is DESIGN.md section 4.9.  The multi_pose, ddd and
// exdet targets (sections 4.10 to 4.12) reuse the warp and the box arithmetic.
#include <map>

#include "common.cuh"
#include "gauss.cuh"
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

// max(0, int(gaussian_radius((ceil(h), ceil(w))))) of ctdet, multi_pose and exdet.
__device__ __forceinline__ int radius_f64(float h, float w) {
  const double r = gaussian_radius_f64((long long)ceilf(h), (long long)ceilf(w));
  return r > 0.0 ? (int)r : 0;
}

// affine_transform (utils/image.py:62-65) in the plain float64 order t0 x + t1 y + t2, rounded to float32.
__device__ __forceinline__ float affine_f32(const double *t, float x, float y) {
  return __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(t[0], (double)x), __dmul_rn(t[1], (double)y)), t[2]));
}

// A box [x0, y0, x1, y1] on the output map, as ctdet, multi_pose and ddd place it.
// Every field but the corners is 0 unless the box is placed (ok).
struct MapBox {
  bool ok;                 // h > 0 && w > 0, or forced
  float w, h;
  float p0, q0, p1, q1;    // the clipped corners
  int r;                   // the sampler's radius
  int cx, cy;              // ct_int
  float rx, ry;            // ct - ct_int
};

// With a non-null width the box is mirrored first (bbox[[0, 2]] = width - bbox[[2, 0]] - 1 in float32).  Both
// corners go through affine_transform and np.clip to [0, xm] x [0, ym]; h = q1 - q0 and w = p1 - p0.  A box with
// h > 0 and w > 0, or any box under `force` (multi_pose's rotated images), is placed: Radius(h, w), then
// ct = (p0 + p1) / 2, ct_int and the offset, all in float32.
template <int (*Radius)(float, float)>
__device__ __forceinline__ MapBox map_box(const float *bb, const int *width, const double *t, float xm, float ym,
                                          bool force) {
  float x0 = bb[0], y0 = bb[1], x1 = bb[2], y1 = bb[3];
  if (width) {
    const float wd = (float)*width;
    const float nx0 = __fsub_rn(__fsub_rn(wd, x1), 1.f), nx1 = __fsub_rn(__fsub_rn(wd, x0), 1.f);
    x0 = nx0;
    x1 = nx1;
  }
  MapBox g = {};
  g.p0 = fminf(fmaxf(affine_f32(t, x0, y0), 0.f), xm);
  g.q0 = fminf(fmaxf(affine_f32(t + 3, x0, y0), 0.f), ym);
  g.p1 = fminf(fmaxf(affine_f32(t, x1, y1), 0.f), xm);
  g.q1 = fminf(fmaxf(affine_f32(t + 3, x1, y1), 0.f), ym);
  g.h = __fsub_rn(g.q1, g.q0);
  g.w = __fsub_rn(g.p1, g.p0);
  g.ok = (g.h > 0.f && g.w > 0.f) || force;
  if (g.ok) {
    g.r = Radius(g.h, g.w);
    const float ctx = __fdiv_rn(__fadd_rn(g.p0, g.p1), 2.f), cty = __fdiv_rn(__fadd_rn(g.q0, g.q1), 2.f);
    g.cx = (int)ctx;
    g.cy = (int)cty;
    g.rx = __fsub_rn(ctx, (float)g.cx);
    g.ry = __fsub_rn(cty, (float)g.cy);
  } else {
    g.w = g.h = 0.f;
  }
  return g;
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
  MapBox g = {};
  if (k < min(num_objs[b], m))
    g = map_box<radius_f64>(boxes + i * 4, flip[b] ? src_hw + 2 * b + 1 : nullptr, trans + 6 * b, (float)(ow - 1),
                            (float)(oh - 1), false);
  const bool valid = g.ok;
  const int c = valid ? cls[i] : 0;
  wh[2 * i] = g.w;
  wh[2 * i + 1] = g.h;
  reg[2 * i] = g.rx;
  reg[2 * i + 1] = g.ry;
  ind[i] = (long long)g.cy * ow + g.cx;
  reg_mask[i] = valid ? 1 : 0;
  obj_cls[i] = c;
  obj_cx[i] = g.cx;
  obj_cy[i] = g.cy;
  obj_radius[i] = g.r;
  obj_valid[i] = valid ? 1 : 0;
  if (cat_spec_wh) {
    float *sw = cat_spec_wh + i * 2 * num_classes;
    unsigned char *sm = cat_spec_mask + i * 2 * num_classes;
    for (int j = 0; j < num_classes; ++j) {
      const bool on = valid && j == c;
      sw[2 * j] = on ? g.w : 0.f;
      sw[2 * j + 1] = on ? g.h : 0.f;
      sm[2 * j] = sm[2 * j + 1] = on ? 1 : 0;
    }
  }
}

// ---------------------------------------------------------------- multi_pose targets (multi_pose.py:104-160)
// One thread per (image, slot), looping over the joints; the box half is k_ctdet_targets' map_box.  A slot gets
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
  MapBox g = {};
  if (k < min(num_objs[b], m))
    g = map_box<radius_f64>(boxes + i * 4, fl ? src_hw + 2 * b + 1 : nullptr, trans + 6 * b, (float)(res - 1),
                            (float)(res - 1), rot);
  const bool valid = g.ok;
  bool any_kpt = false;
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
          hx = __fsub_rn(px, (float)g.cx);
          hy = __fsub_rn(py, (float)g.cy);
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
    hp_radius[l] = in ? g.r : 0;
    hp_valid[l] = in ? 1 : 0;
  }
  wh[2 * i] = g.w;
  wh[2 * i + 1] = g.h;
  reg[2 * i] = g.rx;
  reg[2 * i + 1] = g.ry;
  ind[i] = (long long)g.cy * res + g.cx;
  reg_mask[i] = (valid && any_kpt && !rot) ? 1 : 0;
  obj_cls[i] = valid ? cls[i] : 0;
  obj_cx[i] = g.cx;
  obj_cy[i] = g.cy;
  obj_radius[i] = g.r;
  obj_valid[i] = valid ? 1 : 0;
}

// ---------------------------------------------------------------- ddd targets and heat map (ddd.py:86-140)
// ddd calls gaussian_radius((h, w)) on float32 numpy scalars: every operation is float32 (NEP 50), the Python
// constants rounded to float32 at each use, and b ** 2 is numpy's float32 scalar power, i.e. the C library's
// powf(b, 2), which is NOT always the rounded b * b.  powf_sq restates glibc's powf (ARM optimized-routines: a
// 16-entry log2 table and a degree-5 polynomial, then a 32-entry exp2 table and a cubic, in float64 with the fused
// multiply-adds of its FMA build) for y = 2.
__constant__ double kPowfInvc[16] = {
    0x1.661ec79f8f3bep+0, 0x1.571ed4aaf883dp+0, 0x1.49539f0f010b0p+0, 0x1.3c995b0b80385p+0,
    0x1.30d190c8864a5p+0, 0x1.25e227b0b8ea0p+0, 0x1.1bb4a4a1a343fp+0, 0x1.12358f08ae5bap+0,
    0x1.0953f419900a7p+0, 0x1.0000000000000p+0, 0x1.e608cfd9a47acp-1, 0x1.ca4b31f026aa0p-1,
    0x1.b2036576afce6p-1, 0x1.9c2d163a1aa2dp-1, 0x1.886e6037841edp-1, 0x1.767dcf5534862p-1};
__constant__ double kPowfLogc[16] = {
    -0x1.efec65b963019p-2, -0x1.b0b6832d4fca4p-2, -0x1.7418b0a1fb77bp-2, -0x1.39de91a6dcf7bp-2,
    -0x1.01d9bf3f2b631p-2, -0x1.97c1d1b3b7af0p-3, -0x1.2f9e393af3c9fp-3, -0x1.960cbbf788d5cp-4,
    -0x1.a6f9db6475fcep-5, 0x0.0p+0,               0x1.338ca9f24f53dp-4,  0x1.476a9543891bap-3,
    0x1.e840b4ac4e4d2p-3,  0x1.40645f0c6651cp-2,  0x1.88e9c2c1b9ff8p-2,  0x1.ce0a44eb17bccp-2};
__constant__ unsigned long long kExp2fTab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};

__device__ __forceinline__ float powf_sq(float x) {
  unsigned int ix = __float_as_uint(x) & 0x7fffffffu;   // (-x) ** 2 == x ** 2: the even-integer y path
  if (ix == 0u) return 0.f;
  if (ix < 0x00800000u) ix = (__float_as_uint(__fmul_rn(__uint_as_float(ix), 0x1p23f)) & 0x7fffffffu) - (23u << 23);
  // log2(x): x = 2^k z with z in [0x3f330000, 2 * 0x3f330000), log2(z) = log2(c) + log2(z / c)
  const unsigned int tmp = ix - 0x3f330000u;
  const int i = (int)((tmp >> 19) & 15u);
  const unsigned int top = tmp & 0xff800000u;
  const int k = (int)top >> 23;
  const double z = (double)__uint_as_float(ix - top);
  const double r = __fma_rn(z, kPowfInvc[i], -1.0);
  const double y0 = __dadd_rn(kPowfLogc[i], (double)k);
  const double r2 = __dmul_rn(r, r);
  double y = __fma_rn(0x1.27616c9496e0bp-2, r, -0x1.71969a075c67ap-2);
  const double p = __fma_rn(0x1.ec70a6ca7baddp-2, r, -0x1.7154748bef6c8p-1);
  const double r4 = __dmul_rn(r2, r2);
  double q = __fma_rn(0x1.71547652ab82bp+0, r, y0);
  q = __fma_rn(p, r2, q);
  y = __fma_rn(y, r4, q);
  const double xd = __dmul_rn(2.0, y);   // y * log2(x)
  if (xd > 0x1.fffffffd1d571p+6) return __int_as_float(0x7f800000);
  if (xd <= -150.0) return 0.f;
  // exp2(xd) = 2^(ki / 32) 2^rr
  double kd = __dadd_rn(xd, 0x1.8p+47);
  const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
  kd = __dsub_rn(kd, 0x1.8p+47);
  const double rr = __dsub_rn(xd, kd);
  const double s = __longlong_as_double((long long)(kExp2fTab[ki & 31] + (ki << 47)));
  const double zz = __fma_rn(0x1.c6af84b912394p-5, rr, 0x1.ebfce50fac4f3p-3);
  const double rr2 = __dmul_rn(rr, rr);
  double e = __fma_rn(0x1.62e42ff0c52d6p-1, rr, 1.0);
  e = __fma_rn(zz, rr2, e);
  return __double2float_rn(__dmul_rn(e, s));
}

// gaussian_radius((h, w)) of utils/image.py:95-115 on float32 h, w, in numpy's left-to-right order; min(r1, r2, r3)
// is Python's min (the first smallest).
__device__ __forceinline__ float gaussian_radius_f32(float h, float w) {
  const float b1 = __fadd_rn(h, w);
  const float c1 = __fdiv_rn(__fmul_rn(__fmul_rn(w, h), 0.3f), 1.7f);
  const float r1 = __fdiv_rn(__fadd_rn(b1, __fsqrt_rn(__fsub_rn(powf_sq(b1), __fmul_rn(4.f, c1)))), 2.f);
  const float b2 = __fmul_rn(2.f, __fadd_rn(h, w));
  const float c2 = __fmul_rn(__fmul_rn(0.3f, w), h);
  const float r2 = __fdiv_rn(__fadd_rn(b2, __fsqrt_rn(__fsub_rn(powf_sq(b2), __fmul_rn(16.f, c2)))), 2.f);
  const float b3 = __fmul_rn(-1.4f, __fadd_rn(h, w));
  const float c3 = __fmul_rn(__fmul_rn(-0.3f, w), h);
  const float r3 = __fdiv_rn(__fadd_rn(b3, __fsqrt_rn(__fsub_rn(powf_sq(b3), __fmul_rn(11.2f, c3)))), 2.f);
  float m = r1;
  if (r2 < m) m = r2;
  if (r3 < m) m = r3;
  return m;
}

// max(0, int(radius)); NaN (never for h, w > 0) gives 0.
__device__ __forceinline__ int ddd_radius(float h, float w) {
  const float r = gaussian_radius_f32(h, w);
  return r >= 1.f ? (int)r : 0;
}

// One slot of ddd.py:86-140 for an image: what the targets and hm both read, so they cannot disagree.
struct DddSlot {
  int kind;                 // 0 nothing (empty, cls <= -99, h or w <= 0), 1 positive, 2 ignore
  int cls;                  // the positive class, the ignore class, or -1 for all classes
  bool gauss;               // draws draw_umich_gaussian(hm[cls], ct, r)
  int cx, cy, r;            // ct_int and the radius
  int ox0, oy0, ox1, oy1;   // then hm[cls, oy0:oy1 + 1, ox0:ox1 + 1] = 0.9999 (empty when ox0 > ox1)
  float rx, ry, w, h;       // the offset ct - ct_int, and the box's size on the map
};

__device__ __forceinline__ DddSlot ddd_slot(const float *bb, int cls, const double *t, int num_classes, int oh, int ow,
                                            bool rect_mask) {
  DddSlot s;
  s.kind = 0;
  s.cls = 0;
  s.gauss = false;
  s.cx = s.cy = s.r = 0;
  s.ox0 = 0;
  s.ox1 = -1;
  s.oy0 = 0;
  s.oy1 = -1;
  s.rx = s.ry = s.w = s.h = 0.f;
  const bool pos = cls >= 0 && cls < num_classes;
  const bool ign = cls == -1 || (cls <= -2 && cls >= -num_classes - 1);
  if (!pos && !ign) return s;
  const MapBox g = map_box<ddd_radius>(bb, nullptr, t, (float)(ow - 1), (float)(oh - 1), false);
  if (!g.ok) return s;
  s.h = g.h;
  s.w = g.w;
  s.r = g.r;
  s.rx = g.rx;
  s.ry = g.ry;
  s.cx = g.cx;
  s.cy = g.cy;
  if (pos) {
    s.kind = 1;
    s.cls = cls;
    s.gauss = true;
  } else {
    s.kind = 2;
    s.cls = cls == -1 ? -1 : -cls - 2;
    if (rect_mask) {   // hm[ignore_id, int(y0):int(y1) + 1, int(x0):int(x1) + 1] = 0.9999
      s.ox0 = (int)g.p0;
      s.ox1 = (int)g.p1;
      s.oy0 = (int)g.q0;
      s.oy1 = (int)g.q1;
    } else {           // the Gaussian, then hm[ignore_id, ct_int.y, ct_int.x] = 0.9999
      s.gauss = true;
      s.ox0 = s.ox1 = s.cx;
      s.oy0 = s.oy1 = s.cy;
    }
  }
  return s;
}

constexpr double kPi = 3.141592653589793;

__global__ void __launch_bounds__(kThreads) k_ddd_targets(
    const float *__restrict__ boxes, const int *__restrict__ cls, const int *__restrict__ num_objs,
    const double *__restrict__ alpha, const float *__restrict__ depth, const float *__restrict__ dim,
    const unsigned char *__restrict__ aug, const double *__restrict__ trans, int nb, int m, int num_classes, int oh,
    int ow, int rect_mask, float *__restrict__ dep, float *__restrict__ dim_out,
    long long *__restrict__ ind, long long *__restrict__ rotbin, float *__restrict__ rotres,
    unsigned char *__restrict__ reg_mask, unsigned char *__restrict__ rot_mask, float *__restrict__ wh,
    float *__restrict__ reg) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nb * m) return;
  const int b = (int)(i / m), k = (int)(i % m);
  DddSlot s;
  s.kind = 0;
  if (k < min(num_objs[b], m))
    s = ddd_slot(boxes + i * 4, cls[i], trans + 6 * b, num_classes, oh, ow, rect_mask != 0);
  const bool on = s.kind == 1;
  long long bin0 = 0, bin1 = 0;
  float res0 = 0.f, res1 = 0.f;
  if (on) {   // _convert_alpha(alpha) in float64; rotres f32(alpha -/+ pi / 2)
    const double a = alpha[i];
    if (a < kPi / 6. || a > 5 * kPi / 6.) {
      bin0 = 1;
      res0 = __double2float_rn(__dsub_rn(a, -0.5 * kPi));
    }
    if (a > -kPi / 6. || a < -5 * kPi / 6.) {
      bin1 = 1;
      res1 = __double2float_rn(__dsub_rn(a, 0.5 * kPi));
    }
  }
  wh[2 * i] = on ? s.w : 0.f;
  wh[2 * i + 1] = on ? s.h : 0.f;
  reg[2 * i] = on ? s.rx : 0.f;
  reg[2 * i + 1] = on ? s.ry : 0.f;
  ind[i] = on ? (long long)s.cy * ow + s.cx : 0;
  dep[i] = on ? depth[i] : 0.f;
  dim_out[3 * i] = on ? dim[3 * i] : 0.f;
  dim_out[3 * i + 1] = on ? dim[3 * i + 1] : 0.f;
  dim_out[3 * i + 2] = on ? dim[3 * i + 2] : 0.f;
  rotbin[2 * i] = bin0;
  rotbin[2 * i + 1] = bin1;
  rotres[2 * i] = res0;
  rotres[2 * i + 1] = res1;
  reg_mask[i] = (on && !aug[b]) ? 1 : 0;
  rot_mask[i] = on ? 1 : 0;
}

constexpr int kDddMaxSlots = 128;
constexpr int kDddRows = 4;   // output rows per CTA of the heat map

// The slots of one image as the heat map reads them: class (-1 all), the Gaussian's window and the overwrite
// rectangle, both clipped to the map, and ct_int / r for the Gaussian's value.
struct DddRec {
  int cls, cx, cy, r;
  int gx0, gy0, gx1, gy1;   // Gaussian window on the map (empty when gx0 > gx1)
  int ox0, oy0, ox1, oy1;   // overwrite rectangle
};

// hm [b, C, oh, ow]: each CTA covers kDddRows rows of one image for every class.  It rebuilds the image's slot
// records in shared memory, keeps those (in slot order) that touch its rows, and per pixel and class scans them
// backwards: the max of the Gaussians up to the first slot whose overwrite covers the pixel, then max(that, 0.9999)
// -- the value of the reference's in-order np.maximum / assignment sequence.
__global__ void __launch_bounds__(kThreads) k_ddd_heatmap(const float *__restrict__ boxes,
                                                           const int *__restrict__ cls,
                                                           const int *__restrict__ num_objs,
                                                           const double *__restrict__ trans, int m, int num_classes,
                                                           int oh, int ow, int rect_mask, float *__restrict__ hm) {
  __shared__ DddRec all[kDddMaxSlots];
  __shared__ unsigned char keep[kDddMaxSlots];
  __shared__ DddRec recs[kDddMaxSlots];
  __shared__ int s_n;
  const int b = blockIdx.y;
  const int y0 = blockIdx.x * kDddRows, y1 = min(y0 + kDddRows, oh) - 1;
  const int n = min(num_objs[b], m);
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const long long i = (long long)b * m + k;
    const DddSlot s = ddd_slot(boxes + i * 4, cls[i], trans + 6 * b, num_classes, oh, ow, rect_mask != 0);
    DddRec r;
    r.cls = s.cls;
    r.cx = s.cx;
    r.cy = s.cy;
    r.r = s.r;
    r.gx0 = s.gauss ? max(s.cx - s.r, 0) : 0;
    r.gx1 = s.gauss ? min(s.cx + s.r, ow - 1) : -1;
    r.gy0 = s.gauss ? max(s.cy - s.r, 0) : 0;
    r.gy1 = s.gauss ? min(s.cy + s.r, oh - 1) : -1;
    r.ox0 = s.ox0;
    r.ox1 = s.ox1;
    r.oy0 = s.oy0;
    r.oy1 = s.oy1;
    all[k] = r;
    const bool g_rows = r.gx0 <= r.gx1 && r.gy0 <= y1 && r.gy1 >= y0;
    const bool o_rows = r.ox0 <= r.ox1 && r.oy0 <= y1 && r.oy1 >= y0;
    keep[k] = s.kind != 0 && (g_rows || o_rows);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int c = 0;
    for (int k = 0; k < n; ++k)
      if (keep[k]) recs[c++] = all[k];
    s_n = c;
  }
  __syncthreads();
  const int nr = s_n;
  const size_t plane = (size_t)oh * ow;
  const int npx = (y1 - y0 + 1) * ow;
  for (int p = threadIdx.x; p < npx * num_classes; p += blockDim.x) {
    const int c = p / npx, q = p % npx;
    const int y = y0 + q / ow, x = q % ow;
    float acc = 0.f;
    for (int k = nr - 1; k >= 0; --k) {
      const DddRec &r = recs[k];
      if (r.cls != c && r.cls != -1) continue;
      if (x >= r.ox0 && x <= r.ox1 && y >= r.oy0 && y <= r.oy1) {
        acc = fmaxf(acc, 0.9999f);
        break;
      }
      if (x >= r.gx0 && x <= r.gx1 && y >= r.gy0 && y <= r.gy1) acc = fmaxf(acc, gauss_value(x - r.cx, y - r.cy, r.r));
    }
    hm[((size_t)b * num_classes + c) * plane + (size_t)y * ow + x] = acc;
  }
}

__global__ void __launch_bounds__(kThreads) k_ddd_radius(const float *__restrict__ h, const float *__restrict__ w,
                                                          int n, int *__restrict__ radius) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) radius[i] = h[i] > 0.f && w[i] > 0.f ? ddd_radius(h[i], w[i]) : 0;
}

// ---------------------------------------------------------------- exdet targets (exdet.py:95-129)
constexpr int kExdetMaxSlots = 128;

// np.clip(x, 0, hi) of a float32: a bound replaces x only when x lies strictly outside it, so -0 stays -0 as there
// (and reaches reg as -0 - 0 = -0).
__device__ __forceinline__ float clip_f32(float x, float hi) {
  x = x < 0.f ? 0.f : x;
  return x > hi ? hi : x;
}

// One thread per (image, slot).  Slot k < min(num_objs[b], m) holds the extreme points pts[b, k] [4, 2] (t, l, b, r)
// and the class cls[b, k].  Part p's outputs live at [p, b, k]: reg [4, nb, m, 2], ind [4, nb, m] and the lists
// ex_* [4, nb, m]; the centre lists obj_* and reg_mask are [nb, m].
__global__ void __launch_bounds__(kThreads) k_exdet_targets(
    const float *__restrict__ pts, const int *__restrict__ cls, const int *__restrict__ num_objs,
    const unsigned char *__restrict__ flip, const int *__restrict__ src_hw, const double *__restrict__ trans, int nb,
    int m, int res, int agnostic, float *__restrict__ reg, long long *__restrict__ ind,
    unsigned char *__restrict__ reg_mask, int *__restrict__ obj_cls, int *__restrict__ obj_cx,
    int *__restrict__ obj_cy, int *__restrict__ obj_radius, unsigned char *__restrict__ obj_valid,
    int *__restrict__ ex_cls, int *__restrict__ ex_cx, int *__restrict__ ex_cy, int *__restrict__ ex_radius,
    unsigned char *__restrict__ ex_valid) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nb * m) return;
  const int b = (int)(i / m), k = (int)(i % m);
  float px[4] = {0.f, 0.f, 0.f, 0.f}, py[4] = {0.f, 0.f, 0.f, 0.f};
  int c = 0, rad = 0, cx = 0, cy = 0;
  bool valid = false;
  if (k < min(num_objs[b], m)) {
    const float *q = pts + i * 8;
    const bool fl = flip[b] != 0;
    const float wd = (float)src_hw[2 * b + 1];
    const double *t = trans + 6 * b;
    const float hi = (float)(res - 1);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      // pts[:, 0] = width - pts[:, 0] - 1 in float32, then pts[1] <-> pts[3]
      const int s = fl && (j & 1) ? 4 - j : j;
      const float x = fl ? __fsub_rn(__fsub_rn(wd, q[2 * s]), 1.f) : q[2 * s], y = q[2 * s + 1];
      px[j] = clip_f32(affine_f32(t, x, y), hi);
      py[j] = clip_f32(affine_f32(t + 3, x, y), hi);
    }
    const float h = __fsub_rn(py[2], py[0]), w = __fsub_rn(px[3], px[1]);
    valid = h > 0.f && w > 0.f;
    if (valid) {
      rad = radius_f64(h, w);
      cx = (int)__fdiv_rn(__fadd_rn(px[3], px[1]), 2.f);
      cy = (int)__fdiv_rn(__fadd_rn(py[0], py[2]), 2.f);
      c = cls[i];
    }
  }
  const long long plane = (long long)nb * m;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long o = j * plane + i;
    const int ix = valid ? (int)px[j] : 0, iy = valid ? (int)py[j] : 0;   // the clip makes both >= 0
    reg[2 * o] = valid ? __fsub_rn(px[j], (float)ix) : 0.f;
    reg[2 * o + 1] = valid ? __fsub_rn(py[j], (float)iy) : 0.f;
    ind[o] = (long long)iy * res + ix;
    ex_cls[o] = agnostic ? 0 : c;
    ex_cx[o] = ix;
    ex_cy[o] = iy;
    ex_radius[o] = rad;
    ex_valid[o] = valid ? 1 : 0;
  }
  reg_mask[i] = valid ? 1 : 0;
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

extern "C" int cnb_ddd_targets(const float *boxes, const int32_t *cls, const int32_t *num_objs, const double *alpha,
                               const float *depth, const float *dim, const uint8_t *aug, const double *trans6, int b,
                               int m, int num_classes, int out_h, int out_w, int rect_mask, float *hm, float *dep,
                               float *dim_out, int64_t *ind, int64_t *rotbin, float *rotres, uint8_t *reg_mask,
                               uint8_t *rot_mask, float *wh, float *reg, void *stream) {
  CNB_REQUIRE(boxes && cls && num_objs && alpha && depth && dim && aug && trans6 && hm && dep && dim_out && ind &&
                  rotbin && rotres && reg_mask && rot_mask && wh && reg,
              CNB_EINVAL, "cnb_ddd_targets: null pointer");
  CNB_REQUIRE(b > 0 && b <= 65535 && m > 0 && num_classes > 0 && out_h > 0 && out_w > 0 &&
                  (long long)out_h * out_w <= INT32_MAX && (long long)num_classes * out_h * out_w <= INT32_MAX &&
                  (rect_mask == 0 || rect_mask == 1),
              CNB_EINVAL, "cnb_ddd_targets: bad shape (b = %d, m = %d, classes = %d, out %d x %d, rect_mask %d)", b, m,
              num_classes, out_h, out_w, rect_mask);
  CNB_REQUIRE(m <= cnb::kDddMaxSlots, CNB_EUNSUPPORTED, "cnb_ddd_targets: at most %d slots per image (got %d)",
              cnb::kDddMaxSlots, m);
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)b * m;
  cnb::k_ddd_targets<<<(unsigned)((n + cnb::kThreads - 1) / cnb::kThreads), cnb::kThreads, 0, st>>>(
      boxes, cls, num_objs, alpha, depth, dim, aug, trans6, b, m, num_classes, out_h, out_w, rect_mask, dep, dim_out,
      (long long *)ind, (long long *)rotbin, rotres, reg_mask, rot_mask, wh, reg);
  CNB_CHECK_LAUNCH("cnb_ddd_targets");
  cnb::count_launch();
  dim3 g((unsigned)((out_h + cnb::kDddRows - 1) / cnb::kDddRows), (unsigned)b);
  cnb::k_ddd_heatmap<<<g, cnb::kThreads, 0, st>>>(boxes, cls, num_objs, trans6, m, num_classes, out_h, out_w,
                                                   rect_mask, hm);
  CNB_CHECK_LAUNCH("cnb_ddd_targets (hm)");
  cnb::count_launch();
  return CNB_OK;
}

extern "C" int cnb_ddd_gaussian_radius(const float *h, const float *w, int n, int32_t *radius, void *stream) {
  CNB_REQUIRE(h && w && radius, CNB_EINVAL, "cnb_ddd_gaussian_radius: null pointer");
  CNB_REQUIRE(n > 0, CNB_EINVAL, "cnb_ddd_gaussian_radius: bad length %d", n);
  cnb::k_ddd_radius<<<(unsigned)((n + cnb::kThreads - 1) / cnb::kThreads), cnb::kThreads, 0, (cudaStream_t)stream>>>(
      h, w, n, radius);
  CNB_CHECK_LAUNCH("cnb_ddd_gaussian_radius");
  cnb::count_launch();
  return CNB_OK;
}

extern "C" int cnb_exdet_targets(const float *pts, const int32_t *cls, const int32_t *num_objs, const uint8_t *flip,
                                 const int32_t *src_hw, const double *trans6, int b, int m, int out_res, int agnostic_ex,
                                 float *reg, int64_t *ind, uint8_t *reg_mask, int32_t *obj_cls, int32_t *obj_cx,
                                 int32_t *obj_cy, int32_t *obj_radius, uint8_t *obj_valid, int32_t *ex_cls,
                                 int32_t *ex_cx, int32_t *ex_cy, int32_t *ex_radius, uint8_t *ex_valid, void *stream) {
  CNB_REQUIRE(pts && cls && num_objs && flip && src_hw && trans6 && reg && ind && reg_mask && obj_cls && obj_cx &&
                  obj_cy && obj_radius && obj_valid && ex_cls && ex_cx && ex_cy && ex_radius && ex_valid,
              CNB_EINVAL, "cnb_exdet_targets: null pointer");
  CNB_REQUIRE(b > 0 && m > 0 && out_res > 0 && (long long)out_res * out_res <= INT32_MAX &&
                  (agnostic_ex == 0 || agnostic_ex == 1),
              CNB_EINVAL, "cnb_exdet_targets: bad shape (b = %d, m = %d, out_res = %d, agnostic_ex %d)", b, m, out_res,
              agnostic_ex);
  CNB_REQUIRE(m <= cnb::kExdetMaxSlots, CNB_EUNSUPPORTED, "cnb_exdet_targets: at most %d slots per image (got %d)",
              cnb::kExdetMaxSlots, m);
  const long long n = (long long)b * m;
  cnb::k_exdet_targets<<<(unsigned)((n + cnb::kThreads - 1) / cnb::kThreads), cnb::kThreads, 0,
                         (cudaStream_t)stream>>>(pts, cls, num_objs, flip, src_hw, trans6, b, m, out_res, agnostic_ex,
                                                 reg, (long long *)ind, reg_mask, obj_cls, obj_cx, obj_cy, obj_radius,
                                                 obj_valid, ex_cls, ex_cx, ex_cy, ex_radius, ex_valid);
  CNB_CHECK_LAUNCH("cnb_exdet_targets");
  cnb::count_launch();
  return CNB_OK;
}

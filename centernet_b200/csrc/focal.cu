// Training-side kernels: _sigmoid + penalty-reduced focal loss (+ gradient) with the
// Gaussian target splat fused in, the standalone splat, and the Reg*Loss family.
//
//   _sigmoid            models/utils.py:8-10     clamp(sigmoid(x), 1e-4, 1-1e-4)
//   _neg_loss           models/losses.py:42-67   pos = gt==1, neg = gt<1,
//        L = -(sum log(p)(1-p)^2 pos + sum log(1-p) p^2 (1-gt)^4 neg) / num_pos   (un-normalised if 0)
//   draw_umich_gaussian utils/image.py:126-141   gt = max over objects of exp(-(dx^2+dy^2)/(2 sigma^2)),
//        sigma = (2r+1)/6, window |dx|,|dy| <= r, evaluated in float64 and stored as fp32
//   Reg*Loss            models/losses.py:98-175
//
// The fused kernel streams pred once and writes the gradient once (10.49 MB/image): the
// dense target map of the reference (built on the CPU, copied H2D, read by ~12 ATen kernels)
// is never materialised.  num_pos -- needed to normalise the gradient in the same pass -- is
// known up front from the object lists (one positive per distinct valid centre).
#include <stdlib.h>
#include "common.cuh"

namespace cnb {

constexpr int FOCAL_THREADS = 256;
constexpr int MAX_OBJ_PER_PLANE = 128;
constexpr int FOCAL_MAX_CTAS = 16384;   // grid cap of the loss kernels: one (pos, neg) partial per CTA
constexpr size_t FOCAL_PART_OFF = 256;  // partials start here in the workspace

struct FocalAcc {       // lives at the start of the workspace, zeroed per call
  double num_pos;
  unsigned int done;
  unsigned int pad;
};
// The per-CTA loss sums are stored, not atomically added: the last CTA adds them in CTA order, so the loss is
// bit-identical run to run.  num_pos is a count (exact in double) and keeps its atomics.
__device__ __forceinline__ double2 *focal_partials(FocalAcc *acc) {
  return reinterpret_cast<double2 *>(reinterpret_cast<char *>(acc) + FOCAL_PART_OFF);
}

struct Obj { int x, y, r; };

__device__ __forceinline__ float gauss_value(int dx, int dy, int r) {
  // gaussian2D (utils/image.py:118-124) in float64, cast to fp32 like np.maximum(..., out=fp32 map)
  const double sigma = (double)(2 * r + 1) / 6.0;
  return (float)exp(-(double)(dx * dx + dy * dy) / (2.0 * sigma * sigma));
}

// Gaussian tables (shared memory).  exp(-(dx^2+dy^2)/(2 sigma^2)) depends on d2 = dx^2 + dy^2 only, so every
// object gets a table over d2 in [0, 2 r^2] -- about half the size of its (2r+1)^2 window -- filled once per
// plane by all threads (one float64 exp per ENTRY, no divergence) instead of one exp per covered pixel inside
// a divergent warp.  Same expression, same float64 -> fp32 rounding: bit-identical targets.  Objects whose
// table does not fit keep the direct evaluation.
constexpr int GAUSS_TAB_FLOATS = 6144;   // 24 KB
struct ObjTab { int off; };              // table start, or -1 (direct evaluation)

__device__ __forceinline__ void build_tables(const Obj *objs, int n, ObjTab *tabs, float *tab, int *s_total) {
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < n; ++i) {
      const long long sz = 2ll * objs[i].r * objs[i].r + 1;
      if (run + sz <= GAUSS_TAB_FLOATS) { tabs[i].off = run; run += (int)sz; }
      else tabs[i].off = -1;
    }
    *s_total = run;
  }
  __syncthreads();
  for (int i = 0; i < n; ++i) {
    const int off = tabs[i].off;
    if (off < 0) continue;
    const int r = objs[i].r, sz = 2 * r * r + 1;
    const double sigma = (double)(2 * r + 1) / 6.0;
    const double den = 2.0 * sigma * sigma;
    for (int d2 = threadIdx.x; d2 < sz; d2 += blockDim.x) tab[off + d2] = (float)exp(-(double)d2 / den);
  }
  __syncthreads();
}

// targets of the 4 pixels (x..x+3, y): objects are first rejected by row, then by column
__device__ __forceinline__ float4 target_at4(const Obj *objs, const ObjTab *tabs, const float *tab, int n, int x, int y) {
  float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;
  for (int i = 0; i < n; ++i) {
    const int r = objs[i].r, dy = y - objs[i].y;
    if (dy < -r || dy > r) continue;
    const int dx0 = x - objs[i].x;
    if (dx0 > r || dx0 + 3 < -r) continue;
    const int off = tabs[i].off, dy2 = dy * dy;
#define CNB_TAP(G, J)                                                                              \
    {                                                                                              \
      const int dx = dx0 + (J);                                                                    \
      if (dx >= -r && dx <= r) G = fmaxf(G, (off >= 0) ? tab[off + dx * dx + dy2] : gauss_value(dx, dy, r)); \
    }
    CNB_TAP(g0, 0) CNB_TAP(g1, 1) CNB_TAP(g2, 2) CNB_TAP(g3, 3)
#undef CNB_TAP
  }
  return make_float4(g0, g1, g2, g3);
}
__device__ __forceinline__ float target_at(const Obj *objs, const ObjTab *tabs, const float *tab, int n, int x, int y) {
  float g = 0.0f;
  for (int i = 0; i < n; ++i) {
    const int dx = x - objs[i].x, dy = y - objs[i].y, r = objs[i].r;
    if (dx >= -r && dx <= r && dy >= -r && dy <= r) {
      const int off = tabs[i].off;
      g = fmaxf(g, (off >= 0) ? tab[off + dx * dx + dy * dy] : gauss_value(dx, dy, r));
    }
  }
  return g;
}

// Collect the valid objects of image b that belong to class c (block-wide, order-free: max is commutative).
__device__ __forceinline__ int gather_objects(const int32_t *cls, const int32_t *cx, const int32_t *cy,
                                              const int32_t *rad, const uint8_t *valid, int b, int M, int c, int H,
                                              int W, Obj *s_obj, int *s_n, int y0 = 0, int y1 = 0x7fffffff) {
  if (threadIdx.x == 0) *s_n = 0;
  __syncthreads();
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    const size_t o = (size_t)b * M + m;
    if (valid[o] && cls[o] == c) {
      const int x = cx[o], y = cy[o];
      if (x >= 0 && x < W && y >= 0 && y < H && rad[o] >= 0 && y + rad[o] >= y0 && y - rad[o] < y1) {   // rows [y0, y1) of this CTA
        const int slot = atomicAdd(s_n, 1);
        if (slot < MAX_OBJ_PER_PLANE) s_obj[slot] = Obj{x, y, rad[o]};
      }
    }
  }
  __syncthreads();
  return min(*s_n, MAX_OBJ_PER_PLANE);
}

struct Elem { float loss_pos, loss_neg, grad, is_pos; };

// One element of _neg_loss (+ its gradient w.r.t. pred or, when LOGITS, w.r.t. the logit).
template <bool LOGITS>
__device__ __forceinline__ Elem focal_elem(float v, float gt, float inv_norm) {
  float p = v, chain = 1.0f;
  if (LOGITS) {  // _sigmoid: in-place sigmoid, clamp; clamp passes gradient only inside [min, max]
    const float s = 1.0f / (1.0f + expf(-v));
    p = fminf(fmaxf(s, 1e-4f), 1.0f - 1e-4f);
    chain = (s >= 1e-4f && s <= 1.0f - 1e-4f) ? s * (1.0f - s) : 0.0f;
  }
  Elem e;
  const float omp = 1.0f - p;
  if (gt == 1.0f) {
    const float lg = logf(p);
    e.loss_pos = lg * (omp * omp);
    e.loss_neg = 0.0f;
    e.is_pos = 1.0f;
    e.grad = -((omp * omp) / p - 2.0f * omp * lg) * inv_norm * chain;
  } else if (gt < 1.0f) {
    const float lg = logf(omp);
    const float w1 = 1.0f - gt, w2 = w1 * w1, w4 = w2 * w2;
    e.loss_pos = 0.0f;
    e.loss_neg = lg * (p * p) * w4;
    e.is_pos = 0.0f;
    e.grad = -(w4 * (2.0f * p * lg - (p * p) / omp)) * inv_norm * chain;
  } else {  // gt > 1 or NaN: neither mask fires in the reference
    e.loss_pos = e.loss_neg = e.is_pos = e.grad = 0.0f;
  }
  return e;
}

// the CTA's (pos, neg) sums (fixed shuffle / warp order) -> its partial
__device__ __forceinline__ void block_accumulate(double pos, double neg, FocalAcc *acc) {
  __shared__ double red[2][FOCAL_THREADS / 32];
  for (int o = 16; o > 0; o >>= 1) {
    pos += __shfl_xor_sync(0xffffffffu, pos, o);
    neg += __shfl_xor_sync(0xffffffffu, neg, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { red[0][warp] = pos; red[1][warp] = neg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0;
    for (int i = 0; i < FOCAL_THREADS / 32; ++i) { a += red[0][i]; b += red[1][i]; }
    focal_partials(acc)[blockIdx.x] = make_double2(a, b);
  }
}

// The last CTA to finish adds the partials in CTA order (thread t takes CTAs t, t + 256, ..., then a fixed tree) and
// turns them into (loss, num_pos): losses.py:59-66.
__device__ __forceinline__ void finish_loss(FocalAcc *acc, unsigned int total_blocks, float *out2) {
  __shared__ bool last;
  __shared__ double red[2][FOCAL_THREADS];
  __threadfence();
  if (threadIdx.x == 0) last = (atomicAdd(&acc->done, 1u) == total_blocks - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();
  const double2 *part = focal_partials(acc);
  double ps = 0.0, ns = 0.0;
  for (unsigned i = threadIdx.x; i < total_blocks; i += FOCAL_THREADS) {
    const double2 v = __ldcg(part + i);
    ps += v.x;
    ns += v.y;
  }
  red[0][threadIdx.x] = ps;
  red[1][threadIdx.x] = ns;
  __syncthreads();
  for (int d = FOCAL_THREADS / 2; d > 0; d >>= 1) {
    if ((int)threadIdx.x < d) {
      red[0][threadIdx.x] += red[0][threadIdx.x + d];
      red[1][threadIdx.x] += red[1][threadIdx.x + d];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double np_ = *((volatile double *)&acc->num_pos);
    out2[0] = (np_ == 0.0) ? (float)(-red[1][0]) : (float)(-(red[0][0] + red[1][0]) / np_);
    out2[1] = (float)np_;
  }
}

// ---- pass 0 (dense target): count positives so the gradient can be normalised in the main pass
__global__ void __launch_bounds__(FOCAL_THREADS) k_count_pos_dense(const float *__restrict__ gt, long long n,
                                                                   FocalAcc *acc) {
  double c = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    c += (gt[i] == 1.0f) ? 1.0 : 0.0;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c != 0.0) atomicAdd(&acc->num_pos, c);
}

// ---- pass 0 (object lists): one positive per distinct valid in-bounds (cls, cx, cy)
__global__ void __launch_bounds__(128) k_count_pos_objects(const int32_t *cls, const int32_t *cx, const int32_t *cy,
                                                           const int32_t *rad, const uint8_t *valid, int M, int C,
                                                           int H, int W, FocalAcc *acc) {
  extern __shared__ int cp_sm[];   // per object: packed key (cls, cy, cx) or -1 when it cannot produce a positive
  const int b = blockIdx.x;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    const size_t o = (size_t)b * M + m;
    const bool ok = valid[o] && cls[o] >= 0 && cls[o] < C && cx[o] >= 0 && cx[o] < W && cy[o] >= 0 && cy[o] < H &&
                    rad[o] >= 0;
    cp_sm[m] = ok ? ((cls[o] * H + cy[o]) * W + cx[o]) : -1;
  }
  __syncthreads();
  int cnt = 0;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    const int key = cp_sm[m];
    bool first = key >= 0;
    for (int q = 0; first && q < m; ++q) first = (cp_sm[q] != key);   // shared memory: cheap O(M^2)
    cnt += first ? 1 : 0;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&acc->num_pos, (double)cnt);
}

// ---- main pass, dense target
template <bool LOGITS>
__global__ void __launch_bounds__(FOCAL_THREADS) k_focal_dense(const float *__restrict__ pred,
                                                               const float *__restrict__ gt, long long n,
                                                               float grad_scale, float *__restrict__ grad,
                                                               FocalAcc *acc, float *out2) {
  const double np_ = acc->num_pos;  // written by pass 0 (previous kernel on the stream)
  const float inv_norm = grad_scale / (np_ > 0.0 ? (float)np_ : 1.0f);
  double pos = 0, neg = 0;
  const long long n4 = n >> 2;
  const bool vec = ((((uintptr_t)pred | (uintptr_t)gt | (uintptr_t)grad) & 15u) == 0);
  if (vec) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
         i += (long long)gridDim.x * blockDim.x) {
      const float4 p = __ldg(reinterpret_cast<const float4 *>(pred) + i);
      const float4 g = __ldg(reinterpret_cast<const float4 *>(gt) + i);
      const Elem e0 = focal_elem<LOGITS>(p.x, g.x, inv_norm), e1 = focal_elem<LOGITS>(p.y, g.y, inv_norm);
      const Elem e2 = focal_elem<LOGITS>(p.z, g.z, inv_norm), e3 = focal_elem<LOGITS>(p.w, g.w, inv_norm);
      pos += (double)((e0.loss_pos + e1.loss_pos) + (e2.loss_pos + e3.loss_pos));
      neg += (double)((e0.loss_neg + e1.loss_neg) + (e2.loss_neg + e3.loss_neg));
      if (grad) reinterpret_cast<float4 *>(grad)[i] = make_float4(e0.grad, e1.grad, e2.grad, e3.grad);
    }
  }
  for (long long i = (vec ? (n4 << 2) : 0) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const Elem e = focal_elem<LOGITS>(pred[i], gt[i], inv_norm);
    pos += e.loss_pos; neg += e.loss_neg;
    if (grad) grad[i] = e.grad;
  }
  block_accumulate(pos, neg, acc);
  finish_loss(acc, gridDim.x, out2);
}

// ---- main pass, target rebuilt from object lists: one CTA per (image, class) plane
template <bool LOGITS, bool WRITE_HM>
__global__ void __launch_bounds__(FOCAL_THREADS) k_focal_splat(const float *__restrict__ pred, const int32_t *cls,
                                                               const int32_t *cx, const int32_t *cy,
                                                               const int32_t *rad, const uint8_t *valid, int M, int C,
                                                               int H, int W, float grad_scale,
                                                               float *__restrict__ grad, float *__restrict__ hm,
                                                               FocalAcc *acc, float *out2, int parts, int B) {
  // one CTA per (image, class plane, band of H / parts rows): more, shorter CTAs fill the last wave better.  Grids are
  // capped at FOCAL_MAX_CTAS (one loss partial per CTA): a CTA then takes items blockIdx.x, + gridDim.x, ...
  __shared__ Obj s_obj[MAX_OBJ_PER_PLANE];
  __shared__ ObjTab s_tab[MAX_OBJ_PER_PLANE];
  __shared__ float s_gauss[GAUSS_TAB_FLOATS];
  __shared__ int s_n, s_total;
  float inv_norm = 0.0f;
  if (!WRITE_HM) {
    const double np_ = acc->num_pos;
    inv_norm = grad_scale / (np_ > 0.0 ? (float)np_ : 1.0f);
  }
  double pos = 0, neg = 0;
  const int n_items = B * C * parts;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
  __syncthreads();   // the previous item's objects and tables are no longer read
  const int plane = item / parts, part = item - plane * parts;
  const int b = plane / C, c = plane - b * C;
  const int y_lo = (int)((long long)H * part / parts), y_hi = (int)((long long)H * (part + 1) / parts);
  const int nobj = gather_objects(cls, cx, cy, rad, valid, b, M, c, H, W, s_obj, &s_n, y_lo, y_hi);
  if (nobj) build_tables(s_obj, nobj, s_tab, s_gauss, &s_total);
  const long long base = (long long)plane * H * W;
  const bool vec = (W % 4 == 0) && ((((uintptr_t)pred | (uintptr_t)grad | (uintptr_t)hm) & 15u) == 0);
  if (vec) {
    // (x, y) of the thread's float4 advance incrementally: no division in the loop (the kernel is issue-bound)
    const int w4 = W / 4;
    int y = y_lo + (int)threadIdx.x / w4, x = ((int)threadIdx.x - ((int)threadIdx.x / w4) * w4) * 4;
    const int dyq = (int)blockDim.x / w4, dxq = ((int)blockDim.x - dyq * w4) * 4;
    for (int i = y_lo * w4 + threadIdx.x; i < y_hi * w4; i += blockDim.x, y += dyq, x += dxq) {
      if (x >= W) { x -= W; ++y; }
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
      if (nobj) g = target_at4(s_obj, s_tab, s_gauss, nobj, x, y);
      if (WRITE_HM) {
        reinterpret_cast<float4 *>(hm + base)[i] = g;
      } else {
        const float4 p = __ldg(reinterpret_cast<const float4 *>(pred + base) + i);
        const Elem e0 = focal_elem<LOGITS>(p.x, g.x, inv_norm), e1 = focal_elem<LOGITS>(p.y, g.y, inv_norm);
        const Elem e2 = focal_elem<LOGITS>(p.z, g.z, inv_norm), e3 = focal_elem<LOGITS>(p.w, g.w, inv_norm);
        pos += (double)((e0.loss_pos + e1.loss_pos) + (e2.loss_pos + e3.loss_pos));
        neg += (double)((e0.loss_neg + e1.loss_neg) + (e2.loss_neg + e3.loss_neg));
        if (grad) reinterpret_cast<float4 *>(grad + base)[i] = make_float4(e0.grad, e1.grad, e2.grad, e3.grad);
      }
    }
  } else {
    for (int i = y_lo * W + threadIdx.x; i < y_hi * W; i += blockDim.x) {
      const int y = i / W, x = i - y * W;
      const float g = nobj ? target_at(s_obj, s_tab, s_gauss, nobj, x, y) : 0.0f;
      if (WRITE_HM) {
        hm[base + i] = g;
      } else {
        const Elem e = focal_elem<LOGITS>(pred[base + i], g, inv_norm);
        pos += e.loss_pos; neg += e.loss_neg;
        if (grad) grad[base + i] = e.grad;
      }
    }
  }
  }
  if (!WRITE_HM) {
    block_accumulate(pos, neg, acc);
    finish_loss(acc, gridDim.x, out2);
  }
}

// ---- Reg*Loss: B*M*D is tiny (e.g. 64*128*2); one CTA does sums, loss and the scatter of the gradient.
__global__ void __launch_bounds__(1024) k_reg_loss(const float *__restrict__ output, const void *mask_,
                                                   const int64_t *__restrict__ ind, const float *__restrict__ target,
                                                   int B, int D, long long HW, int M, int mode, float grad_scale,
                                                   float *out1, float *grad_output) {
  __shared__ double red[2][32];
  __shared__ double s_tot[2];
  const long long n = (long long)B * M * D;
  const uint8_t *mask_u8 = reinterpret_cast<const uint8_t *>(mask_);
  const float *mask_f = reinterpret_cast<const float *>(mask_);
  double loss = 0, msum = 0;
  // pass 0: the sums (strided per thread, fixed tree); pass 1: the gradient, one thread per (image, channel) plane
  // walking m in ascending order, so repeated indices add up in a fixed order without atomics
  for (int pass = 0; pass < 2; ++pass) {
    const double denom = pass ? (s_tot[1] + 1e-4) : 1.0;
    const long long n_it = pass ? (long long)B * D : n;
    for (long long it = threadIdx.x; it < n_it; it += blockDim.x) {
      if (pass && !grad_output) break;
      for (int mm = 0; mm < (pass ? M : 1); ++mm) {
        const long long i = pass ? ((it / D) * M + mm) * D + it % D : it;
        const int d = (int)(i % D);
        const long long bm = i / D;
        const int b = (int)(bm / M);
        const long long sp = ind[bm];
        if (sp < 0 || sp >= HW) continue;   // torch's gather raises on such an index; never read or write outside the map
        const float m = (mode == 3) ? mask_f[i] : (float)mask_u8[bm];
        float pred = output[((long long)b * D + d) * HW + sp];
        float tgt = target[i];
        float scale = 1.0f;
        if (mode == 2) {  // NormRegL1Loss: pred / (target + 1e-4) against 1
          scale = 1.0f / (tgt + 1e-4f);
          pred = pred / (tgt + 1e-4f);
          tgt = tgt * 0.0f + 1.0f;
        }
        const float diff = pred * m - tgt * m;
        if (pass == 0) {
          const float ad = fabsf(diff);
          loss += (mode == 1) ? (ad < 1.0f ? 0.5 * (double)ad * ad : (double)ad - 0.5) : (double)ad;
          msum += (mode == 1) ? ((d == 0) ? (double)m : 0.0) : (double)m;  // RegLoss divides by mask.sum() un-expanded
        } else {
          float g = (diff > 0.0f) ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
          if (mode == 1 && fabsf(diff) < 1.0f) g = diff;
          g = g * m * scale * grad_scale / (float)denom;
          if (g != 0.0f) grad_output[((long long)b * D + d) * HW + sp] += g;
        }
      }
    }
    if (pass == 0) {
      for (int o = 16; o > 0; o >>= 1) {
        loss += __shfl_xor_sync(0xffffffffu, loss, o);
        msum += __shfl_xor_sync(0xffffffffu, msum, o);
      }
      if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = loss; red[1][threadIdx.x >> 5] = msum; }
      __syncthreads();
      if (threadIdx.x == 0) {
        double a = 0, c = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += red[0][i]; c += red[1][i]; }
        s_tot[0] = a; s_tot[1] = c;
        out1[0] = (float)(a / (c + 1e-4));
      }
      __syncthreads();
    }
  }
}

static int focal_grid(long long n4) {
  long long g = (n4 + FOCAL_THREADS - 1) / FOCAL_THREADS;
  long long cap = (long long)num_sms() * 8;
  if (cap > FOCAL_MAX_CTAS) cap = FOCAL_MAX_CTAS;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}
static int splat_grid(long long items) { return (int)(items < FOCAL_MAX_CTAS ? items : FOCAL_MAX_CTAS); }

}  // namespace cnb

using namespace cnb;

// bands per plane of the splat kernels (CNB_FOCAL_PARTS overrides, for tuning)
static int focal_parts(int h) {
  static const int env = [] { const char *e = getenv("CNB_FOCAL_PARTS"); return e ? atoi(e) : 0; }();
  int p = env > 0 ? env : 1;
  if (p > h) p = h;
  return p < 1 ? 1 : p;
}

extern "C" {

size_t cnb_focal_workspace_bytes(long long) { return FOCAL_PART_OFF + (size_t)FOCAL_MAX_CTAS * sizeof(double2); }

int cnb_focal_loss(const float *pred, const float *gt, long long n, int logits, float grad_scale, float *out2,
                   float *grad, void *workspace, size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(pred && gt && out2 && workspace, CNB_EINVAL, "cnb_focal_loss: null pointer");
  CNB_REQUIRE(n > 0, CNB_EINVAL, "cnb_focal_loss: n=%lld", n);
  CNB_REQUIRE(workspace_bytes >= cnb_focal_workspace_bytes(n), CNB_EWORKSPACE, "cnb_focal_loss: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  FocalAcc *acc = reinterpret_cast<FocalAcc *>(workspace);
  CNB_CUDA(cudaMemsetAsync(acc, 0, sizeof(FocalAcc), stream));
  const int grid = focal_grid(n / 4 + 1);
  k_count_pos_dense<<<grid, FOCAL_THREADS, 0, stream>>>(gt, n, acc);
  CNB_CHECK_LAUNCH("cnb_focal_loss count");
  if (logits)
    k_focal_dense<true><<<grid, FOCAL_THREADS, 0, stream>>>(pred, gt, n, grad_scale, grad, acc, out2);
  else
    k_focal_dense<false><<<grid, FOCAL_THREADS, 0, stream>>>(pred, gt, n, grad_scale, grad, acc, out2);
  CNB_CHECK_LAUNCH("cnb_focal_loss");
  count_launch(2);
  return CNB_OK;
}

int cnb_splat_gaussian(const int32_t *obj_cls, const int32_t *obj_cx, const int32_t *obj_cy,
                       const int32_t *obj_radius, const uint8_t *obj_valid, int b, int m, int c, int h, int w,
                       float *hm, void *stream_) {
  CNB_REQUIRE(obj_cls && obj_cx && obj_cy && obj_radius && obj_valid && hm, CNB_EINVAL,
              "cnb_splat_gaussian: null pointer");
  CNB_REQUIRE(b > 0 && m > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "cnb_splat_gaussian: non-positive dimension");
  CNB_REQUIRE(m <= MAX_OBJ_PER_PLANE, CNB_EUNSUPPORTED, "cnb_splat_gaussian: at most %d objects per image (got %d)",
              MAX_OBJ_PER_PLANE, m);
  const int parts = focal_parts(h);
  k_focal_splat<false, true><<<splat_grid((long long)b * c * parts), FOCAL_THREADS, 0, (cudaStream_t)stream_>>>(
      nullptr, obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, m, c, h, w, 0.0f, nullptr, hm, nullptr, nullptr, parts, b);
  CNB_CHECK_LAUNCH("cnb_splat_gaussian");
  count_launch();
  return CNB_OK;
}

int cnb_focal_splat_loss(const float *pred, const int32_t *obj_cls, const int32_t *obj_cx, const int32_t *obj_cy,
                         const int32_t *obj_radius, const uint8_t *obj_valid, int b, int m, int c, int h, int w,
                         int logits, float grad_scale, float *out2, float *grad, void *workspace,
                         size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(pred && obj_cls && obj_cx && obj_cy && obj_radius && obj_valid && out2 && workspace, CNB_EINVAL,
              "cnb_focal_splat_loss: null pointer");
  CNB_REQUIRE(b > 0 && m > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "cnb_focal_splat_loss: non-positive dimension");
  CNB_REQUIRE(m <= MAX_OBJ_PER_PLANE, CNB_EUNSUPPORTED, "cnb_focal_splat_loss: at most %d objects per image (got %d)",
              MAX_OBJ_PER_PLANE, m);
  CNB_REQUIRE(workspace_bytes >= cnb_focal_workspace_bytes((long long)b * c * h * w), CNB_EWORKSPACE,
              "cnb_focal_splat_loss: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  FocalAcc *acc = reinterpret_cast<FocalAcc *>(workspace);
  CNB_CUDA(cudaMemsetAsync(acc, 0, sizeof(FocalAcc), stream));
  CNB_REQUIRE((long long)c * h * w < (1ll << 31), CNB_EUNSUPPORTED, "cnb_focal_splat_loss: c*h*w must be < 2^31");
  k_count_pos_objects<<<b, 128, (size_t)m * sizeof(int), stream>>>(obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, m, c, h,
                                                                    w, acc);
  CNB_CHECK_LAUNCH("cnb_focal_splat_loss count");
  const int parts = focal_parts(h);
  if (logits)
    k_focal_splat<true, false><<<splat_grid((long long)b * c * parts), FOCAL_THREADS, 0, stream>>>(pred, obj_cls, obj_cx, obj_cy, obj_radius,
                                                                             obj_valid, m, c, h, w, grad_scale, grad,
                                                                             nullptr, acc, out2, parts, b);
  else
    k_focal_splat<false, false><<<splat_grid((long long)b * c * parts), FOCAL_THREADS, 0, stream>>>(pred, obj_cls, obj_cx, obj_cy, obj_radius,
                                                                              obj_valid, m, c, h, w, grad_scale, grad,
                                                                              nullptr, acc, out2, parts, b);
  CNB_CHECK_LAUNCH("cnb_focal_splat_loss");
  count_launch(2);
  return CNB_OK;
}

int cnb_reg_loss(const float *output, const void *mask, const int64_t *ind, const float *target, int b, int d, int hw,
                 int m, int mode, float grad_scale, float *out1, float *grad_output, void *stream_) {
  CNB_REQUIRE(output && mask && ind && target && out1, CNB_EINVAL, "cnb_reg_loss: null pointer");
  CNB_REQUIRE(b > 0 && d > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_reg_loss: non-positive dimension");
  CNB_REQUIRE(mode >= 0 && mode <= 3, CNB_EINVAL, "cnb_reg_loss: mode %d", mode);
  k_reg_loss<<<1, 1024, 0, (cudaStream_t)stream_>>>(output, mask, ind, target, b, d, hw, m, mode, grad_scale, out1,
                                                    grad_output);
  CNB_CHECK_LAUNCH("cnb_reg_loss");
  count_launch();
  return CNB_OK;
}

}  // extern "C"

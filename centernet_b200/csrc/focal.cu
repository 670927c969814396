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
// known up front from the object lists (one positive per distinct valid centre inside the map).
//
// pred may be fp32, bf16 or fp16; each loss has one kernel body, templated on pred's type T.  Both half formats widen
// to fp32 exactly (to_f32) and everything after the load is the fp32 arithmetic, with the same grid, elements per
// thread, (e0 + e1) + (e2 + e3) groups and partials, so a half pred gives bit for bit the loss of the T = float
// instance on its .float() upcast.
#include <stdlib.h>
#include <type_traits>
#include "common.cuh"
#include "gauss.cuh"

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
      // draw_umich_gaussian clips the window to the map: a centre outside it still paints the overlap
      const long long x = cx[o], y = cy[o], r = rad[o];
      if (r >= 0 && x + r >= 0 && x - r < W && y + r >= 0 && y - r < H && y + r >= y0 && y - r < y1) {   // rows [y0, y1) of this CTA
        const int slot = atomicAdd(s_n, 1);
        if (slot < MAX_OBJ_PER_PLANE) s_obj[slot] = Obj{(int)x, (int)y, (int)r};
      }
    }
  }
  __syncthreads();
  return min(*s_n, MAX_OBJ_PER_PLANE);
}

struct Elem { float loss_pos, loss_neg, grad, is_pos; };

// One element of _neg_loss outside the fast path's assumptions (p or gt NaN, p outside (0, 1), gt outside [0, 1]):
// the reference's masked products as IEEE fp32 evaluates them, pos_loss = log(p) (1-p)^2 [gt == 1] and
// neg_loss = log(1-p) p^2 (1-gt)^4 [gt < 1], with the gradient autograd takes through them factor by factor.  A mask
// of 0 times an infinite or NaN factor is NaN, so the loss and the gradient are NaN or inf exactly where the
// reference's are (a NaN target: (1-gt)^4 = NaN times 0; p = 1 at a positive: log(0) times 0).
template <bool LOGITS>
__device__ __forceinline__ Elem focal_elem_ieee(float p, float s, bool in_clamp, float gt, float inv_norm,
                                                bool pos_live) {
  const float pos = (gt == 1.0f) ? 1.0f : 0.0f, neg = (gt < 1.0f) ? 1.0f : 0.0f;
  const float omp = 1.0f - p, w1 = 1.0f - gt, w = (w1 * w1) * (w1 * w1);
  const float lp = logf(p), lq = logf(omp);
  Elem e;
  e.loss_pos = lp * (omp * omp) * pos;
  e.loss_neg = lq * (p * p) * w * neg;
  e.is_pos = pos;
  // with num_pos == 0 the reference returns -neg_loss: the positive terms are not in its graph
  const float dpos = pos_live ? (pos * (omp * omp)) / p - (pos * lp) * (2.0f * omp) : 0.0f;
  const float dneg = (neg * w * lq) * (2.0f * p) - (neg * w * (p * p)) / omp;
  const float g = -(dpos + dneg) * inv_norm;
  // clamp's backward selects (0 outside [min, max], whatever flows in); sigmoid's then multiplies by s (1 - s)
  e.grad = LOGITS ? (in_clamp ? g * (s * (1.0f - s)) : 0.0f * s) : g;
  return e;
}

// One element of _neg_loss (+ its gradient w.r.t. pred or, when LOGITS, w.r.t. the logit).  pos_live: num_pos > 0.
template <bool LOGITS>
__device__ __forceinline__ Elem focal_elem(float v, float gt, float inv_norm, bool pos_live) {
  float p = v, s = v, chain = 1.0f;
  bool in_clamp = true;
  if (LOGITS) {  // _sigmoid: in-place sigmoid, clamp; clamp passes gradient only inside [min, max]
    s = 1.0f / (1.0f + expf(-v));
    p = s < 1e-4f ? 1e-4f : (s > 1.0f - 1e-4f ? 1.0f - 1e-4f : s);   // NaN stays NaN, as in torch.clamp
    in_clamp = (s >= 1e-4f && s <= 1.0f - 1e-4f);
    chain = in_clamp ? s * (1.0f - s) : 0.0f;
  }
  // p in (0, 1) and gt in [+0, 1] as two unsigned compares of the bit patterns (NaN and negatives fail both)
  const bool fast = (__float_as_uint(p) - 1u < 0x3f7fffffu) & (__float_as_uint(gt) <= 0x3f800000u);
  if (!fast) return focal_elem_ieee<LOGITS>(p, s, in_clamp, gt, inv_norm, pos_live);
  Elem e;
  const float omp = 1.0f - p;
  if (gt == 1.0f) {
    const float lg = logf(p);
    e.loss_pos = lg * (omp * omp);
    e.loss_neg = 0.0f;
    e.is_pos = 1.0f;
    e.grad = -((omp * omp) / p - 2.0f * omp * lg) * inv_norm * chain;
  } else {
    const float lg = logf(omp);
    const float w1 = 1.0f - gt, w2 = w1 * w1, w4 = w2 * w2;
    e.loss_pos = 0.0f;
    e.loss_neg = lg * (p * p) * w4;
    e.is_pos = 0.0f;
    e.grad = -(w4 * (2.0f * p * lg - (p * p) / omp)) * inv_norm * chain;
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

template <typename T> __device__ __forceinline__ T narrow(float v);   // round to nearest even; fp16 overflows to inf
template <> __device__ __forceinline__ float narrow<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 narrow<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half narrow<__half>(float v) { return __float2half_rn(v); }

template <typename T> union Pack4 { uint2 u; T t[4]; };
// Elements 4i .. 4i+3 of p.  bf16 / fp16: one 8-byte access when p is 8-byte aligned (al8), else four 2-byte ones.
// fp32: one 16-byte access, al8 unused (the fp32 kernels group by four only when p is 16-byte aligned).
template <typename T>
__device__ __forceinline__ float4 load4(const T *p, long long i, bool al8) {
  Pack4<T> r;
  p += 4 * i;
  if (al8) {
    r.u = __ldg(reinterpret_cast<const uint2 *>(p));
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) r.t[j] = __ldg(p + j);
  }
  return make_float4(to_f32(r.t[0]), to_f32(r.t[1]), to_f32(r.t[2]), to_f32(r.t[3]));
}
template <> __device__ __forceinline__ float4 load4<float>(const float *p, long long i, bool) {
  return __ldg(reinterpret_cast<const float4 *>(p) + i);
}
template <typename T>
__device__ __forceinline__ void store4(T *p, long long i, bool al8, float a, float b, float c, float d) {
  Pack4<T> r;
  r.t[0] = narrow<T>(a); r.t[1] = narrow<T>(b); r.t[2] = narrow<T>(c); r.t[3] = narrow<T>(d);
  p += 4 * i;
  if (al8) {
    *reinterpret_cast<uint2 *>(p) = r.u;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) p[j] = r.t[j];
  }
}
template <> __device__ __forceinline__ void store4<float>(float *p, long long i, bool, float a, float b, float c,
                                                          float d) {
  reinterpret_cast<float4 *>(p)[i] = make_float4(a, b, c, d);
}
__device__ __forceinline__ float incoming_grad(const float *grad_out) { return grad_out ? __ldg(grad_out) : 1.0f; }

// ---- main pass, dense target.  One body, three uses:
//   fp32 forward  (T = float, BWD = false): the loss, and the gradient, scaled by grad_scale, into grad (nullable);
//   half forward  (BWD = false, grad_scale = 1, grad null): the loss only;
//   half backward (BWD = true, acc null): out2 holds the forward's (loss, num_pos); stores T(grad * *grad_out).
// A half gradient cannot be finished in the forward pass as the fp32 one is: it has to be rounded to T once, AFTER
// the scale by the loss's incoming gradient, which only backward knows.  So backward evaluates focal_elem again, and
// __fmul_rn keeps that product out of any contraction with focal_elem's last multiply.
template <typename T, bool LOGITS, bool BWD>
__global__ void __launch_bounds__(FOCAL_THREADS) k_focal_dense(const T *__restrict__ pred,
                                                               const float *__restrict__ gt, long long n,
                                                               float grad_scale, T *__restrict__ grad,
                                                               FocalAcc *acc, float *out2,
                                                               const float *__restrict__ grad_out) {
  // num_pos: written by pass 0 (previous kernel on the stream), or in backward by the forward
  const double np_ = BWD ? (double)out2[1] : acc->num_pos;
  const float inv_norm = grad_scale / (np_ > 0.0 ? (float)np_ : 1.0f);
  const bool pos_live = np_ > 0.0;
  constexpr bool F32 = std::is_same<T, float>::value;
  constexpr bool STORE = F32 || BWD;   // a half forward computes no gradient
  const float go = BWD ? incoming_grad(grad_out) : 1.0f;
  auto scaled = [go](float g) { return BWD ? __fmul_rn(g, go) : g; };
  double pos = 0, neg = 0;
  const long long n4 = n >> 2;
  // fp32 groups by four when pred, gt and grad are 16-byte aligned.  A half pred groups as the fp32 kernel does on
  // its .float() upcast and that gradient, fresh allocations: by gt's alignment alone.
  const bool group4 = F32 ? ((((uintptr_t)pred | (uintptr_t)gt | (uintptr_t)grad) & 15u) == 0)
                          : (((uintptr_t)gt & 15u) == 0);
  const bool al8 = ((((uintptr_t)pred | (uintptr_t)grad) & 7u) == 0);
  if (group4) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
         i += (long long)gridDim.x * blockDim.x) {
      const float4 p = load4<T>(pred, i, al8);
      const float4 g = __ldg(reinterpret_cast<const float4 *>(gt) + i);
      const Elem e0 = focal_elem<LOGITS>(p.x, g.x, inv_norm, pos_live), e1 = focal_elem<LOGITS>(p.y, g.y, inv_norm, pos_live);
      const Elem e2 = focal_elem<LOGITS>(p.z, g.z, inv_norm, pos_live), e3 = focal_elem<LOGITS>(p.w, g.w, inv_norm, pos_live);
      if (!BWD) {
        pos += (double)((e0.loss_pos + e1.loss_pos) + (e2.loss_pos + e3.loss_pos));
        neg += (double)((e0.loss_neg + e1.loss_neg) + (e2.loss_neg + e3.loss_neg));
      }
      if (STORE && grad) store4<T>(grad, i, al8, scaled(e0.grad), scaled(e1.grad), scaled(e2.grad), scaled(e3.grad));
    }
  }
  for (long long i = (group4 ? (n4 << 2) : 0) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const Elem e = focal_elem<LOGITS>(to_f32(pred[i]), gt[i], inv_norm, pos_live);
    if (!BWD) { pos += e.loss_pos; neg += e.loss_neg; }
    if (STORE && grad) grad[i] = narrow<T>(scaled(e.grad));
  }
  if (!BWD) {
    block_accumulate(pos, neg, acc);
    finish_loss(acc, gridDim.x, out2);
  }
}

// ---- main pass, target rebuilt from object lists: one CTA per (image, class) plane.  The gradient is stored in fp32,
// scaled by grad_scale, into grad (nullable).  With a half pred (grad_scale = 1) that is the unscaled fp32 gradient
// k_scale_round turns into T: this kernel is issue-bound, and evaluating the tables and focal_elem a second time in
// backward measured slower than storing the gradient (DESIGN 4.3.1).  WRITE_HM (T = float): only the target, to hm.
template <typename T, bool LOGITS, bool WRITE_HM>
__global__ void __launch_bounds__(FOCAL_THREADS) k_focal_splat(const T *__restrict__ pred, const int32_t *cls,
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
  bool pos_live = false;
  if (!WRITE_HM) {
    const double np_ = acc->num_pos;
    inv_norm = grad_scale / (np_ > 0.0 ? (float)np_ : 1.0f);
    pos_live = np_ > 0.0;
  }
  double pos = 0, neg = 0;
  const int n_items = B * C * parts;
  // Groups of four need W % 4 == 0; fp32 also needs pred, grad and hm 16-byte aligned.  A half pred groups as the
  // fp32 kernel does on its .float() upcast and that gradient, fresh allocations: whenever W % 4 == 0 (its plane bases
  // are then 8-byte multiples).  A half pred's fp32 gradient group is one 16-byte store when grad is so aligned.
  constexpr bool F32 = std::is_same<T, float>::value;
  const bool al8 = (((uintptr_t)pred & 7u) == 0), g_al16 = F32 || (((uintptr_t)grad & 15u) == 0);
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
  __syncthreads();   // the previous item's objects and tables are no longer read
  const int plane = item / parts, part = item - plane * parts;
  const int b = plane / C, c = plane - b * C;
  const int y_lo = (int)((long long)H * part / parts), y_hi = (int)((long long)H * (part + 1) / parts);
  const int nobj = gather_objects(cls, cx, cy, rad, valid, b, M, c, H, W, s_obj, &s_n, y_lo, y_hi);
  if (nobj) build_tables(s_obj, nobj, s_tab, s_gauss, &s_total);
  const long long base = (long long)plane * H * W;
  const bool vec = (W % 4 == 0) && (!F32 || ((((uintptr_t)pred | (uintptr_t)grad | (uintptr_t)hm) & 15u) == 0));
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
        const float4 p = load4<T>(pred + base, i, al8);
        const Elem e0 = focal_elem<LOGITS>(p.x, g.x, inv_norm, pos_live), e1 = focal_elem<LOGITS>(p.y, g.y, inv_norm, pos_live);
        const Elem e2 = focal_elem<LOGITS>(p.z, g.z, inv_norm, pos_live), e3 = focal_elem<LOGITS>(p.w, g.w, inv_norm, pos_live);
        pos += (double)((e0.loss_pos + e1.loss_pos) + (e2.loss_pos + e3.loss_pos));
        neg += (double)((e0.loss_neg + e1.loss_neg) + (e2.loss_neg + e3.loss_neg));
        if (grad && g_al16) {
          reinterpret_cast<float4 *>(grad + base)[i] = make_float4(e0.grad, e1.grad, e2.grad, e3.grad);
        } else if (grad) {
          float *gp = grad + base + 4ll * i;
          gp[0] = e0.grad; gp[1] = e1.grad; gp[2] = e2.grad; gp[3] = e3.grad;
        }
      }
    }
  } else {
    for (int i = y_lo * W + threadIdx.x; i < y_hi * W; i += blockDim.x) {
      const int y = i / W, x = i - y * W;
      const float g = nobj ? target_at(s_obj, s_tab, s_gauss, nobj, x, y) : 0.0f;
      if (WRITE_HM) {
        hm[base + i] = g;
      } else {
        const Elem e = focal_elem<LOGITS>(to_f32(pred[base + i]), g, inv_norm, pos_live);
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
// One (image, object, channel) element i and its offset `at` in the output map: false when its index is outside the
// map (torch's gather raises on such an index; never read or write outside the map).
template <typename T>
__device__ __forceinline__ bool reg_elem(const T *__restrict__ output, const float *mask_f,
                                         const int64_t *__restrict__ ind, const float *__restrict__ target, int D,
                                         long long HW, int M, int mode, long long i, float *diff, float *m,
                                         float *scale, long long *at) {
  const int d = (int)(i % D);
  const long long bm = i / D;
  const int b = (int)(bm / M);
  const long long sp = ind[bm];
  if (sp < 0 || sp >= HW) return false;
  *m = mask_f[(mode == 3) ? i : bm];   // mask.float(): fractional weights stay fractional
  *at = ((long long)b * D + d) * HW + sp;
  float pred = to_f32(output[*at]);
  float tgt = target[i];
  *scale = 1.0f;
  if (mode == 2) {  // NormRegL1Loss: pred / (target + 1e-4) against 1
    *scale = 1.0f / (tgt + 1e-4f);
    pred = pred / (tgt + 1e-4f);
    tgt = tgt * 0.0f + 1.0f;
  }
  *diff = pred * *m - tgt * *m;
  return true;
}

// out[0] = the loss.  A half output (read at the gathered positions only) also gets out[1] = (float)(mask sum + 1e-4),
// the denominator k_reg_grad_half divides its gradient by; an fp32 output gets its gradient here instead (grad_output,
// nullable), which half leaves null.
template <typename T>
__global__ void __launch_bounds__(1024) k_reg_loss(const T *__restrict__ output, const float *mask_f,
                                                   const int64_t *__restrict__ ind, const float *__restrict__ target,
                                                   int B, int D, long long HW, int M, int mode, float grad_scale,
                                                   float *out, float *grad_output) {
  constexpr bool F32 = std::is_same<T, float>::value;
  __shared__ double red[2][32];
  __shared__ double s_tot[2];
  const long long n = (long long)B * M * D;
  double loss = 0, msum = 0;
  // pass 0: the sums (strided per thread, fixed tree); pass 1: the gradient, one thread per (image, channel) plane
  // walking m in ascending order, so repeated indices add up in a fixed order without atomics
  for (int pass = 0; pass < (F32 ? 2 : 1); ++pass) {
    const double denom = pass ? (s_tot[1] + 1e-4) : 1.0;
    const long long n_it = pass ? (long long)B * D : n;
    for (long long it = threadIdx.x; it < n_it; it += blockDim.x) {
      if (pass && !grad_output) break;
      for (int mm = 0; mm < (pass ? M : 1); ++mm) {
        const long long i = pass ? ((it / D) * M + mm) * D + it % D : it;
        float diff, m, scale;
        long long at;
        if (!reg_elem<T>(output, mask_f, ind, target, D, HW, M, mode, i, &diff, &m, &scale, &at)) continue;
        if (pass == 0) {
          const float ad = fabsf(diff);
          loss += (mode == 1) ? (ad < 1.0f ? 0.5 * (double)ad * ad : (double)ad - 0.5) : (double)ad;
          msum += (mode == 1) ? (((int)(i % D) == 0) ? (double)m : 0.0) : (double)m;  // RegLoss divides by mask.sum() un-expanded
        } else {
          float g = (diff > 0.0f) ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
          if (mode == 1 && fabsf(diff) < 1.0f) g = diff;
          g = g * m * scale * grad_scale / (float)denom;
          if (g != 0.0f) grad_output[at] += g;
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
        out[0] = (float)(a / (c + 1e-4));
        if (!F32) out[1] = (float)(c + 1e-4);
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------ bf16 / fp16 gradients, no fp32 counterpart
// out = T(g32 * *grad_out): the scale by the loss's incoming gradient, then the one rounding
template <typename T>
__global__ void __launch_bounds__(256) k_scale_round(const float *__restrict__ g32, long long n,
                                                     const float *__restrict__ grad_out, T *__restrict__ out) {
  const float go = incoming_grad(grad_out);
  const bool vec = ((((uintptr_t)g32 & 15u) | ((uintptr_t)out & 7u)) == 0);
  const long long n4 = vec ? (n >> 2) : 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 g = __ldg(reinterpret_cast<const float4 *>(g32) + i);
    store4<T>(out, i, true, __fmul_rn(g.x, go), __fmul_rn(g.y, go), __fmul_rn(g.z, go), __fmul_rn(g.w, go));
  }
  for (long long i = (n4 << 2) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    out[i] = narrow<T>(__fmul_rn(g32[i], go));
}

// Every element of the fp32 gradient map that no index selects is +0, and autograd's scale makes it 0 * grad_out
// (-0 for a negative grad_out): the fill of the half map.
template <typename T>
__global__ void __launch_bounds__(256) k_fill_scaled_zero(T *__restrict__ p, long long n,
                                                          const float *__restrict__ grad_out) {
  const T z = narrow<T>(__fmul_rn(0.0f, incoming_grad(grad_out)));
  const bool al8 = (((uintptr_t)p & 7u) == 0);
  Pack4<T> r;
  r.t[0] = r.t[1] = r.t[2] = r.t[3] = z;
  const long long n4 = al8 ? (n >> 2) : 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
    reinterpret_cast<uint2 *>(p)[i] = r.u;
  for (long long i = (n4 << 2) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    p[i] = z;
}

// The gradient k_reg_loss's pass 1 leaves in an fp32 map, scaled and rounded once.  One thread per (image, object,
// channel); the thread of the first m that holds a map index is that element's only writer: it adds the
// contributions of every m with the same index in fp32 in ascending m, as pass 1 does in the map, multiplies the sum
// by *grad_out and rounds it to T.  Nothing is accumulated in the half map and there are no atomics.
template <typename T>
__global__ void __launch_bounds__(256) k_reg_grad_half(const T *__restrict__ output, const float *mask_f,
                                                       const int64_t *__restrict__ ind,
                                                       const float *__restrict__ target, int B, int D, long long HW,
                                                       int M, int mode, const float *__restrict__ loss_den,
                                                       const float *__restrict__ grad_out, T *__restrict__ grad) {
  const long long n = (long long)B * M * D;
  const float den = loss_den[1], go = incoming_grad(grad_out);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(i % D);
    const long long bm = i / D;
    const int b = (int)(bm / M), m0 = (int)(bm % M);
    const int64_t *row = ind + (long long)b * M;
    const long long sp = row[m0];
    if (sp < 0 || sp >= HW) continue;
    bool first = true;
    for (int q = 0; first && q < m0; ++q) first = (row[q] != sp);
    if (!first) continue;
    float sum = 0.0f;
    for (int q = m0; q < M; ++q) {
      if (row[q] != sp) continue;
      float diff, m, scale;
      long long at;
      reg_elem<T>(output, mask_f, ind, target, D, HW, M, mode, ((long long)b * M + q) * D + d, &diff, &m, &scale,
                  &at);
      float g = (diff > 0.0f) ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
      if (mode == 1 && fabsf(diff) < 1.0f) g = diff;
      g = g * m * scale / den;
      if (g != 0.0f) sum += g;
    }
    grad[((long long)b * D + d) * HW + sp] = narrow<T>(__fmul_rn(sum, go));
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

// The dense focal loss of cnb_focal_loss (T = float) and cnb_focal_loss_ex (bf16 / fp16: grad_scale = 1, grad null).
// Errors name `who`, the entry point the caller used.
template <typename T>
static int focal_loss(const char *who, const T *pred, const float *gt, long long n, int logits, float grad_scale,
                      float *out2, T *grad, void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  CNB_REQUIRE(pred && gt && out2 && workspace, CNB_EINVAL, "%s: null pointer", who);
  CNB_REQUIRE(n > 0, CNB_EINVAL, "%s: n=%lld", who, n);
  CNB_REQUIRE(workspace_bytes >= cnb_focal_workspace_bytes(n), CNB_EWORKSPACE, "%s: workspace too small", who);
  FocalAcc *acc = reinterpret_cast<FocalAcc *>(workspace);
  CNB_CUDA(cudaMemsetAsync(acc, 0, sizeof(FocalAcc), stream));
  const int grid = focal_grid(n / 4 + 1);
  k_count_pos_dense<<<grid, FOCAL_THREADS, 0, stream>>>(gt, n, acc);
  const cudaError_t e = cudaGetLastError();
  CNB_REQUIRE(e == cudaSuccess, CNB_ECUDA, "%s count: CUDA error: %s", who, cudaGetErrorString(e));
  if (logits)
    k_focal_dense<T, true, false><<<grid, FOCAL_THREADS, 0, stream>>>(pred, gt, n, grad_scale, grad, acc, out2, nullptr);
  else
    k_focal_dense<T, false, false><<<grid, FOCAL_THREADS, 0, stream>>>(pred, gt, n, grad_scale, grad, acc, out2, nullptr);
  CNB_CHECK_LAUNCH(who);
  count_launch(2);
  return CNB_OK;
}

// The fused splat loss of cnb_focal_splat_loss (T = float) and cnb_focal_splat_loss_ex (bf16 / fp16: grad_scale = 1,
// grad the unscaled fp32 gradient).  Errors name `who`, the entry point the caller used.
template <typename T>
static int focal_splat_loss(const char *who, const T *pred, const int32_t *obj_cls, const int32_t *obj_cx,
                            const int32_t *obj_cy, const int32_t *obj_radius, const uint8_t *obj_valid, int b, int m,
                            int c, int h, int w, int logits, float grad_scale, float *out2, float *grad,
                            void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  CNB_REQUIRE(pred && obj_cls && obj_cx && obj_cy && obj_radius && obj_valid && out2 && workspace, CNB_EINVAL,
              "%s: null pointer", who);
  CNB_REQUIRE(b > 0 && m > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "%s: non-positive dimension", who);
  CNB_REQUIRE(m <= MAX_OBJ_PER_PLANE, CNB_EUNSUPPORTED, "%s: at most %d objects per image (got %d)", who,
              MAX_OBJ_PER_PLANE, m);
  CNB_REQUIRE(workspace_bytes >= cnb_focal_workspace_bytes((long long)b * c * h * w), CNB_EWORKSPACE,
              "%s: workspace too small", who);
  CNB_REQUIRE((long long)c * h * w < (1ll << 31), CNB_EUNSUPPORTED, "%s: c*h*w must be < 2^31", who);
  FocalAcc *acc = reinterpret_cast<FocalAcc *>(workspace);
  CNB_CUDA(cudaMemsetAsync(acc, 0, sizeof(FocalAcc), stream));
  k_count_pos_objects<<<b, 128, (size_t)m * sizeof(int), stream>>>(obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, m, c, h,
                                                                    w, acc);
  const cudaError_t e = cudaGetLastError();
  CNB_REQUIRE(e == cudaSuccess, CNB_ECUDA, "%s count: CUDA error: %s", who, cudaGetErrorString(e));
  const int parts = focal_parts(h), grid = splat_grid((long long)b * c * parts);
  if (logits)
    k_focal_splat<T, true, false><<<grid, FOCAL_THREADS, 0, stream>>>(pred, obj_cls, obj_cx, obj_cy, obj_radius,
                                                                      obj_valid, m, c, h, w, grad_scale, grad,
                                                                      nullptr, acc, out2, parts, b);
  else
    k_focal_splat<T, false, false><<<grid, FOCAL_THREADS, 0, stream>>>(pred, obj_cls, obj_cx, obj_cy, obj_radius,
                                                                       obj_valid, m, c, h, w, grad_scale, grad,
                                                                       nullptr, acc, out2, parts, b);
  CNB_CHECK_LAUNCH(who);
  count_launch(2);
  return CNB_OK;
}

extern "C" {

size_t cnb_focal_workspace_bytes(long long) { return FOCAL_PART_OFF + (size_t)FOCAL_MAX_CTAS * sizeof(double2); }

int cnb_focal_loss(const float *pred, const float *gt, long long n, int logits, float grad_scale, float *out2,
                   float *grad, void *workspace, size_t workspace_bytes, void *stream_) {
  return focal_loss("cnb_focal_loss", pred, gt, n, logits, grad_scale, out2, grad, workspace, workspace_bytes,
                    (cudaStream_t)stream_);
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
  k_focal_splat<float, false, true><<<splat_grid((long long)b * c * parts), FOCAL_THREADS, 0, (cudaStream_t)stream_>>>(
      nullptr, obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, m, c, h, w, 0.0f, nullptr, hm, nullptr, nullptr, parts, b);
  CNB_CHECK_LAUNCH("cnb_splat_gaussian");
  count_launch();
  return CNB_OK;
}

int cnb_focal_splat_loss(const float *pred, const int32_t *obj_cls, const int32_t *obj_cx, const int32_t *obj_cy,
                         const int32_t *obj_radius, const uint8_t *obj_valid, int b, int m, int c, int h, int w,
                         int logits, float grad_scale, float *out2, float *grad, void *workspace,
                         size_t workspace_bytes, void *stream_) {
  return focal_splat_loss("cnb_focal_splat_loss", pred, obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, b, m, c, h, w,
                          logits, grad_scale, out2, grad, workspace, workspace_bytes, (cudaStream_t)stream_);
}

int cnb_reg_loss(const float *output, const void *mask, const int64_t *ind, const float *target, int b, int d, int hw,
                 int m, int mode, float grad_scale, float *out1, float *grad_output, void *stream_) {
  CNB_REQUIRE(output && mask && ind && target && out1, CNB_EINVAL, "cnb_reg_loss: null pointer");
  CNB_REQUIRE(b > 0 && d > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_reg_loss: non-positive dimension");
  CNB_REQUIRE(mode >= 0 && mode <= 3, CNB_EINVAL, "cnb_reg_loss: mode %d", mode);
  k_reg_loss<<<1, 1024, 0, (cudaStream_t)stream_>>>(output, static_cast<const float *>(mask), ind, target, b, d, hw, m, mode, grad_scale, out1,
                                                    grad_output);
  CNB_CHECK_LAUNCH("cnb_reg_loss");
  count_launch();
  return CNB_OK;
}

// ---- bf16 / fp16 pred: forward (loss) and backward (gradient in pred's dtype) as two calls.  An fp32 code given to a
// call that has an fp32 form is that call.

int cnb_focal_loss_ex(const void *pred, int pred_dtype, const float *gt, long long n, int logits, float *out2,
                      void *workspace, size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(dtype_known(pred_dtype), CNB_EINVAL, "cnb_focal_loss_ex: unknown dtype code %d", pred_dtype);
  if (pred_dtype == CNB_DTYPE_F32)
    return cnb_focal_loss(static_cast<const float *>(pred), gt, n, logits, 1.0f, out2, nullptr, workspace,
                          workspace_bytes, stream_);
  cudaStream_t stream = (cudaStream_t)stream_;
  if (pred_dtype == CNB_DTYPE_BF16)
    return focal_loss<__nv_bfloat16>("cnb_focal_loss_ex", static_cast<const __nv_bfloat16 *>(pred), gt, n, logits,
                                     1.0f, out2, nullptr, workspace, workspace_bytes, stream);
  return focal_loss<__half>("cnb_focal_loss_ex", static_cast<const __half *>(pred), gt, n, logits, 1.0f, out2, nullptr,
                            workspace, workspace_bytes, stream);
}

int cnb_focal_grad_ex(const void *pred, int pred_dtype, const float *gt, long long n, int logits,
                      const float *loss_num_pos, const float *grad_out, void *grad, void *stream_) {
  CNB_REQUIRE(dtype_known(pred_dtype), CNB_EINVAL, "cnb_focal_grad_ex: unknown dtype code %d", pred_dtype);
  CNB_REQUIRE(pred_dtype != CNB_DTYPE_F32, CNB_EUNSUPPORTED,
              "cnb_focal_grad_ex: bf16 / fp16 only (cnb_focal_loss writes the fp32 gradient in its one pass)");
  CNB_REQUIRE(pred && gt && loss_num_pos && grad, CNB_EINVAL, "cnb_focal_grad_ex: null pointer");
  CNB_REQUIRE(n > 0, CNB_EINVAL, "cnb_focal_grad_ex: n=%lld", n);
  cudaStream_t stream = (cudaStream_t)stream_;
  const int grid = focal_grid(n / 4 + 1);
  float *out2 = const_cast<float *>(loss_num_pos);   // read only when BWD
  const auto *pb = static_cast<const __nv_bfloat16 *>(pred);
  const auto *ph = static_cast<const __half *>(pred);
  auto *gb = static_cast<__nv_bfloat16 *>(grad);
  auto *gh = static_cast<__half *>(grad);
  if (pred_dtype == CNB_DTYPE_BF16 && logits)
    k_focal_dense<__nv_bfloat16, true, true><<<grid, FOCAL_THREADS, 0, stream>>>(pb, gt, n, 1.0f, gb, nullptr, out2, grad_out);
  else if (pred_dtype == CNB_DTYPE_BF16)
    k_focal_dense<__nv_bfloat16, false, true><<<grid, FOCAL_THREADS, 0, stream>>>(pb, gt, n, 1.0f, gb, nullptr, out2, grad_out);
  else if (logits)
    k_focal_dense<__half, true, true><<<grid, FOCAL_THREADS, 0, stream>>>(ph, gt, n, 1.0f, gh, nullptr, out2, grad_out);
  else
    k_focal_dense<__half, false, true><<<grid, FOCAL_THREADS, 0, stream>>>(ph, gt, n, 1.0f, gh, nullptr, out2, grad_out);
  CNB_CHECK_LAUNCH("cnb_focal_grad_ex");
  count_launch();
  return CNB_OK;
}

int cnb_focal_splat_loss_ex(const void *pred, int pred_dtype, const int32_t *obj_cls, const int32_t *obj_cx,
                            const int32_t *obj_cy, const int32_t *obj_radius, const uint8_t *obj_valid, int b, int m,
                            int c, int h, int w, int logits, float *out2, float *grad32, void *workspace,
                            size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(dtype_known(pred_dtype), CNB_EINVAL, "cnb_focal_splat_loss_ex: unknown dtype code %d", pred_dtype);
  if (pred_dtype == CNB_DTYPE_F32)
    return cnb_focal_splat_loss(static_cast<const float *>(pred), obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, b, m,
                                c, h, w, logits, 1.0f, out2, grad32, workspace, workspace_bytes, stream_);
  cudaStream_t stream = (cudaStream_t)stream_;
  if (pred_dtype == CNB_DTYPE_BF16)
    return focal_splat_loss("cnb_focal_splat_loss_ex", static_cast<const __nv_bfloat16 *>(pred), obj_cls, obj_cx,
                            obj_cy, obj_radius, obj_valid, b, m, c, h, w, logits, 1.0f, out2, grad32, workspace,
                            workspace_bytes, stream);
  return focal_splat_loss("cnb_focal_splat_loss_ex", static_cast<const __half *>(pred), obj_cls, obj_cx, obj_cy,
                          obj_radius, obj_valid, b, m, c, h, w, logits, 1.0f, out2, grad32, workspace, workspace_bytes,
                          stream);
}

int cnb_focal_splat_grad_ex(const float *grad32, long long n, const float *grad_out, void *grad, int grad_dtype,
                            void *stream_) {
  CNB_REQUIRE(dtype_known(grad_dtype), CNB_EINVAL, "cnb_focal_splat_grad_ex: unknown dtype code %d", grad_dtype);
  CNB_REQUIRE(grad_dtype != CNB_DTYPE_F32, CNB_EUNSUPPORTED,
              "cnb_focal_splat_grad_ex: bf16 / fp16 only (an fp32 gradient is grad32 times grad_out)");
  CNB_REQUIRE(grad32 && grad, CNB_EINVAL, "cnb_focal_splat_grad_ex: null pointer");
  CNB_REQUIRE(n > 0, CNB_EINVAL, "cnb_focal_splat_grad_ex: n=%lld", n);
  cudaStream_t stream = (cudaStream_t)stream_;
  const long long ctas = (n / 4 + 255) / 256 + 1, cap = (long long)num_sms() * 16;
  const int grid = (int)(ctas < cap ? ctas : cap);
  if (grad_dtype == CNB_DTYPE_BF16)
    k_scale_round<<<grid, 256, 0, stream>>>(grad32, n, grad_out, static_cast<__nv_bfloat16 *>(grad));
  else
    k_scale_round<<<grid, 256, 0, stream>>>(grad32, n, grad_out, static_cast<__half *>(grad));
  CNB_CHECK_LAUNCH("cnb_focal_splat_grad_ex");
  count_launch();
  return CNB_OK;
}

int cnb_reg_loss_ex(const void *output, int output_dtype, const void *mask, const int64_t *ind, const float *target,
                    int b, int d, int hw, int m, int mode, float *out2, void *stream_) {
  CNB_REQUIRE(dtype_known(output_dtype), CNB_EINVAL, "cnb_reg_loss_ex: unknown dtype code %d", output_dtype);
  CNB_REQUIRE(output_dtype != CNB_DTYPE_F32, CNB_EUNSUPPORTED, "cnb_reg_loss_ex: bf16 / fp16 only (fp32: cnb_reg_loss)");
  CNB_REQUIRE(output && mask && ind && target && out2, CNB_EINVAL, "cnb_reg_loss_ex: null pointer");
  CNB_REQUIRE(b > 0 && d > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_reg_loss_ex: non-positive dimension");
  CNB_REQUIRE(mode >= 0 && mode <= 3, CNB_EINVAL, "cnb_reg_loss_ex: mode %d", mode);
  cudaStream_t stream = (cudaStream_t)stream_;
  const float *mask_f = static_cast<const float *>(mask);
  if (output_dtype == CNB_DTYPE_BF16)
    k_reg_loss<<<1, 1024, 0, stream>>>(static_cast<const __nv_bfloat16 *>(output), mask_f, ind, target, b, d,
                                       (long long)hw, m, mode, 1.0f, out2, nullptr);
  else
    k_reg_loss<<<1, 1024, 0, stream>>>(static_cast<const __half *>(output), mask_f, ind, target, b, d, (long long)hw,
                                       m, mode, 1.0f, out2, nullptr);
  CNB_CHECK_LAUNCH("cnb_reg_loss_ex");
  count_launch();
  return CNB_OK;
}

int cnb_reg_loss_grad_ex(const void *output, int output_dtype, const void *mask, const int64_t *ind,
                         const float *target, int b, int d, int hw, int m, int mode, const float *loss_den,
                         const float *grad_out, void *grad_output, void *stream_) {
  CNB_REQUIRE(dtype_known(output_dtype), CNB_EINVAL, "cnb_reg_loss_grad_ex: unknown dtype code %d", output_dtype);
  CNB_REQUIRE(output_dtype != CNB_DTYPE_F32, CNB_EUNSUPPORTED,
              "cnb_reg_loss_grad_ex: bf16 / fp16 only (cnb_reg_loss writes the fp32 gradient in its one pass)");
  CNB_REQUIRE(output && mask && ind && target && loss_den && grad_output, CNB_EINVAL,
              "cnb_reg_loss_grad_ex: null pointer");
  CNB_REQUIRE(b > 0 && d > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_reg_loss_grad_ex: non-positive dimension");
  CNB_REQUIRE(mode >= 0 && mode <= 3, CNB_EINVAL, "cnb_reg_loss_grad_ex: mode %d", mode);
  cudaStream_t stream = (cudaStream_t)stream_;
  const float *mask_f = static_cast<const float *>(mask);
  const long long total = (long long)b * d * hw, work = (long long)b * m * d;
  const long long fill_ctas = (total / 4 + 255) / 256 + 1, cap = (long long)num_sms() * 16;
  const int fill_grid = (int)(fill_ctas < cap ? fill_ctas : cap);
  const int grid = (int)((work + 255) / 256 < cap ? (work + 255) / 256 : cap);
  if (output_dtype == CNB_DTYPE_BF16) {
    auto *g = static_cast<__nv_bfloat16 *>(grad_output);
    k_fill_scaled_zero<<<fill_grid, 256, 0, stream>>>(g, total, grad_out);
    k_reg_grad_half<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16 *>(output), mask_f, ind, target, b, d,
                                              (long long)hw, m, mode, loss_den, grad_out, g);
  } else {
    auto *g = static_cast<__half *>(grad_output);
    k_fill_scaled_zero<<<fill_grid, 256, 0, stream>>>(g, total, grad_out);
    k_reg_grad_half<<<grid, 256, 0, stream>>>(static_cast<const __half *>(output), mask_f, ind, target, b, d,
                                              (long long)hw, m, mode, loss_den, grad_out, g);
  }
  CNB_CHECK_LAUNCH("cnb_reg_loss_grad_ex");
  count_launch(2);
  return CNB_OK;
}

}  // extern "C"

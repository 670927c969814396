// C-ABI entry points of the heat-map decode family (models/decode.py, models/utils.py).
#include "select.cuh"

namespace cnb {

// ------------------------------------------------------------------ A1: standalone _nms
// One thread per 4 consecutive pixels; neighbours come through L1/L2 so DRAM sees one
// read and one write of the map.  models/decode.py:9-15.
template <bool VEC>
__global__ void __launch_bounds__(256) k_nms(const float *__restrict__ heat, float *__restrict__ out,
                                             long long planes, int H, int W) {
  const int Wq = VEC ? W / 4 : W;
  const long long total = planes * H * Wq;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int xq = (int)(i % Wq);
    const long long t = i / Wq;
    const int y = (int)(t % H);
    const float *pl = heat + (t / H) * (long long)H * W;
    const float NI = CNB_NEG_INF;
    if (VEC) {
      const int x0 = xq * 4;
      float v[6] = {NI, NI, NI, NI, NI, NI};  // vertical max of columns x0-1 .. x0+4
      float4 ctr = make_float4(0, 0, 0, 0);
      for (int dy = -1; dy <= 1; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;
        const float *row = pl + (long long)yy * W;
        const float4 q = __ldg(reinterpret_cast<const float4 *>(row + x0));
        if (dy == 0) ctr = q;
        v[1] = fmaxf(v[1], q.x); v[2] = fmaxf(v[2], q.y); v[3] = fmaxf(v[3], q.z); v[4] = fmaxf(v[4], q.w);
        if (x0 > 0) v[0] = fmaxf(v[0], __ldg(row + x0 - 1));
        if (x0 + 4 < W) v[5] = fmaxf(v[5], __ldg(row + x0 + 4));
      }
      float4 o;
      o.x = ctr.x * ((fmax3(v[0], v[1], v[2]) == ctr.x) ? 1.0f : 0.0f);
      o.y = ctr.y * ((fmax3(v[1], v[2], v[3]) == ctr.y) ? 1.0f : 0.0f);
      o.z = ctr.z * ((fmax3(v[2], v[3], v[4]) == ctr.z) ? 1.0f : 0.0f);
      o.w = ctr.w * ((fmax3(v[3], v[4], v[5]) == ctr.w) ? 1.0f : 0.0f);
      *reinterpret_cast<float4 *>(out + (t * W) + x0) = o;
    } else {
      const int x = xq;
      const float c = pl[(long long)y * W + x];
      float m = c;
      for (int dy = -1; dy <= 1; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;
        for (int dx = -1; dx <= 1; ++dx) {
          const int xx = x + dx;
          if (xx < 0 || xx >= W) continue;
          m = fmaxf(m, __ldg(pl + (long long)yy * W + xx));
        }
      }
      out[t * W + x] = c * ((m == c) ? 1.0f : 0.0f);
    }
  }
}

// ------------------------------------------------------------------ A4: gather
// out[b, m, ch] = feat[b, ch, ind[b, m]]   (models/utils.py:12-26 without the transpose copy)
__global__ void __launch_bounds__(256) k_gather_feat(const float *__restrict__ feat,
                                                     const int64_t *__restrict__ ind, float *__restrict__ out,
                                                     int B, int C, long long HW, int M) {
  const long long total = (long long)B * M * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C);
    const long long bm = i / C;
    const int b = (int)(bm / M);
    const long long sp = ind[bm];
    float v = 0.0f;
    if (sp >= 0 && sp < HW) v = __ldg(feat + ((long long)b * C + ch) * HW + sp);
    out[i] = v;
  }
}

// grad_feat[b, ch, ind[b, m]] += grad_out[b, m, ch]: the adjoint of the gather (autograd of `feat.gather(1, ind)`,
// models/utils.py:15).  An index may repeat inside an image: one thread per (image, channel) plane adds the plane's M
// values in ascending m, so repeats sum in a fixed order without atomics.  grad_feat arrives zero-filled.
__global__ void __launch_bounds__(256) k_gather_feat_bwd(const float *__restrict__ grad_out,
                                                         const int64_t *__restrict__ ind,
                                                         float *__restrict__ grad_feat, int B, int C, long long HW,
                                                         int M) {
  const long long planes = (long long)B * C;
  for (long long pl = blockIdx.x * (long long)blockDim.x + threadIdx.x; pl < planes;
       pl += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(pl / C), ch = (int)(pl % C);
    float *gp = grad_feat + pl * HW;
    for (int m = 0; m < M; ++m) {
      const long long sp = __ldg(ind + (long long)b * M + m);
      if (sp >= 0 && sp < HW) gp[sp] += __ldg(grad_out + ((long long)b * M + m) * C + ch);
    }
  }
}

// The gather of a bf16 / fp16 feat read in place: each value widens exactly, so out is the gather of the upcast.
template <typename T>
__global__ void __launch_bounds__(256) k_gather_feat_half(const T *__restrict__ feat, const int64_t *__restrict__ ind,
                                                          float *__restrict__ out, int B, int C, long long HW, int M) {
  const long long total = (long long)B * M * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C);
    const long long bm = i / C;
    const int b = (int)(bm / M);
    const long long sp = ind[bm];
    float v = 0.0f;
    if (sp >= 0 && sp < HW) v = (float)__ldg(feat + ((long long)b * C + ch) * HW + sp);
    out[i] = v;
  }
}

// Its adjoint into a zero-filled bf16 / fp16 grad_feat.  One thread per (image, m, channel); the thread of the first
// m that holds a map index is that element's only writer: it adds the rows of every m with the same index in fp32 in
// ascending m, starting from the map's 0 as k_gather_feat_bwd does, and rounds the sum once.
template <typename T>
__global__ void __launch_bounds__(256) k_gather_feat_bwd_half(const float *__restrict__ grad_out,
                                                              const int64_t *__restrict__ ind,
                                                              T *__restrict__ grad_feat, int B, int C, long long HW,
                                                              int M) {
  const long long total = (long long)B * M * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C);
    const long long bm = i / C;
    const int b = (int)(bm / M), m0 = (int)(bm % M);
    const int64_t *row = ind + (long long)b * M;
    const long long sp = __ldg(row + m0);
    if (sp < 0 || sp >= HW) continue;
    bool first = true;
    for (int q = 0; first && q < m0; ++q) first = (__ldg(row + q) != sp);
    if (!first) continue;
    float sum = 0.0f;
    for (int q = m0; q < M; ++q)
      if (__ldg(row + q) == sp) sum += __ldg(grad_out + ((long long)b * M + q) * C + ch);
    grad_feat[((long long)b * C + ch) * HW + sp] = T(sum);
  }
}

// ------------------------------------------------------------------ A9: ddd epilogue
// models/decode.py:432-460: [xs, ys, score, rot(8), depth, dim(3), (wh(2)), cls]
__global__ void __launch_bounds__(128) k_ddd_epilogue(const float *__restrict__ scores,
                                                      const int64_t *__restrict__ inds,
                                                      const int32_t *__restrict__ clses,
                                                      const float *__restrict__ ys, const float *__restrict__ xs,
                                                      const float *__restrict__ rot, const float *__restrict__ depth,
                                                      const float *__restrict__ dim, const float *__restrict__ wh,
                                                      const float *__restrict__ reg, int B, int K, long long HW,
                                                      float *__restrict__ dets) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * K) return;
  const int b = i / K;
  const long long sp = inds[i];
  const int D = wh ? 18 : 16;
  float *d = dets + (size_t)i * D;
  float x = xs[i], y = ys[i];
  if (reg) {
    x += reg[((long long)b * 2) * HW + sp];
    y += reg[((long long)b * 2 + 1) * HW + sp];
  } else {
    x += 0.5f;
    y += 0.5f;
  }
  d[0] = x; d[1] = y; d[2] = scores[i];
  for (int r = 0; r < 8; ++r) d[3 + r] = rot[((long long)b * 8 + r) * HW + sp];
  d[11] = depth[(long long)b * HW + sp];
  for (int r = 0; r < 3; ++r) d[12 + r] = dim[((long long)b * 3 + r) * HW + sp];
  int o = 15;
  if (wh) {
    d[15] = wh[((long long)b * 2) * HW + sp];
    d[16] = wh[((long long)b * 2 + 1) * HW + sp];
    o = 17;
  }
  d[o] = (float)clses[i];
}

// k_ddd_epilogue for cnb_ddd_decode_ex: each head of its own dtype code in h, widened exactly; with h.logits the
// depth head holds the raw `dep` output and goes through ddd_depth at the K gathered positions only.
struct DddHeads {
  int rot, depth, dim, wh, reg;  // CNB_DTYPE_* codes
  int logits;
};

// `1. / (dep.sigmoid() + 1e-6) - 1.` (detectors/ddd.py:62) in torch's op order on fp32 CUDA tensors: sigmoid,
// add(1e-6), reciprocal and mul(1.0) (Tensor.__rtruediv__ is `reciprocal() * other`), sub(1.0), every step rounded to
// fp32.  The _rn intrinsics keep nvcc from contracting or reordering them.
__device__ __forceinline__ float ddd_depth(float x) {
  const float s = 1.0f / (1.0f + expf(-x));  // torch's CUDA sigmoid (k_sigmoid)
  return __fsub_rn(__fmul_rn(__frcp_rn(__fadd_rn(s, 1e-6f)), 1.0f), 1.0f);
}

// v[r] = head[i + r * HW], r < N.  One dtype switch per head, so that its N loads are in flight together.
template <int N>
__device__ __forceinline__ void ld_rows(float (&v)[N], const void *__restrict__ p, int dt, long long i, long long HW) {
  if (dt == CNB_DTYPE_F32) {
#pragma unroll
    for (int r = 0; r < N; ++r) v[r] = __ldg(reinterpret_cast<const float *>(p) + i + r * HW);
  } else if (dt == CNB_DTYPE_BF16) {
#pragma unroll
    for (int r = 0; r < N; ++r)
      v[r] = __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16 *>(p) + i + r * HW));
  } else {
#pragma unroll
    for (int r = 0; r < N; ++r) v[r] = __half2float(__ldg(reinterpret_cast<const __half *>(p) + i + r * HW));
  }
}

__global__ void __launch_bounds__(128) k_ddd_epilogue_ex(const float *__restrict__ scores,
                                                         const int64_t *__restrict__ inds,
                                                         const int32_t *__restrict__ clses,
                                                         const float *__restrict__ ys, const float *__restrict__ xs,
                                                         const void *__restrict__ rot, const void *__restrict__ depth,
                                                         const void *__restrict__ dim, const void *__restrict__ wh,
                                                         const void *__restrict__ reg, DddHeads h, int B, int K,
                                                         long long HW, float *__restrict__ dets) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * K) return;
  const int b = i / K;
  const long long sp = inds[i];
  const int D = wh ? 18 : 16;
  float *d = dets + (size_t)i * D;
  float x = xs[i], y = ys[i];
  if (reg) {
    float rg[2];
    ld_rows(rg, reg, h.reg, ((long long)b * 2) * HW + sp, HW);
    x += rg[0];
    y += rg[1];
  } else {
    x += 0.5f;
    y += 0.5f;
  }
  d[0] = x; d[1] = y; d[2] = scores[i];
  float rt[8], dp[1], dm[3];
  ld_rows(rt, rot, h.rot, ((long long)b * 8) * HW + sp, HW);
  ld_rows(dp, depth, h.depth, (long long)b * HW + sp, HW);
  ld_rows(dm, dim, h.dim, ((long long)b * 3) * HW + sp, HW);
  for (int r = 0; r < 8; ++r) d[3 + r] = rt[r];
  d[11] = h.logits ? ddd_depth(dp[0]) : dp[0];
  for (int r = 0; r < 3; ++r) d[12 + r] = dm[r];
  int o = 15;
  if (wh) {
    float wv[2];
    ld_rows(wv, wh, h.wh, ((long long)b * 2) * HW + sp, HW);
    d[15] = wv[0];
    d[16] = wv[1];
    o = 17;
  }
  d[o] = (float)clses[i];
}

struct RawTopk {
  float *scores;
  int64_t *inds;
  int32_t *clses;
  float *ys;
  float *xs;
};

static size_t raw_bytes(long long n) {  // n = n_img * K entries
  return align_up((size_t)n * 8, 256) + 4 * align_up((size_t)n * 4, 256);
}
static RawTopk carve_raw(char *p, long long n) {
  RawTopk r;
  r.inds = reinterpret_cast<int64_t *>(p); p += align_up((size_t)n * 8, 256);
  r.scores = reinterpret_cast<float *>(p); p += align_up((size_t)n * 4, 256);
  r.clses = reinterpret_cast<int32_t *>(p); p += align_up((size_t)n * 4, 256);
  r.ys = reinterpret_cast<float *>(p); p += align_up((size_t)n * 4, 256);
  r.xs = reinterpret_cast<float *>(p);
  return r;
}

}  // namespace cnb

using namespace cnb;

// out = 1 / (1 + exp(-x)), the expression of torch's CUDA sigmoid (4 elements per thread); a 16-bit x is widened
// to fp32 first, exactly
template <typename T>
__global__ void __launch_bounds__(256) k_sigmoid(const T *__restrict__ x, float *__restrict__ out, long long n) {
  const long long i0 = ((long long)blockIdx.x * 256 + threadIdx.x) * 4;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (i0 + j < n) out[i0 + j] = 1.0f / (1.0f + expf(-to_f32(x[i0 + j])));
}

// out = x widened to fp32 (what torch's .float() gives), 4 elements per thread
template <typename T>
__global__ void __launch_bounds__(256) k_widen(const T *__restrict__ x, float *__restrict__ out, long long n) {
  const long long i0 = ((long long)blockIdx.x * 256 + threadIdx.x) * 4;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (i0 + j < n) out[i0 + j] = to_f32(x[i0 + j]);
}

// fp32 heat map (sigmoid of the logits, or the widened map) of a 16-bit or fp32 src, n elements
int cnb::launch_to_f32(const void *src, int dt, bool sigmoid, float *out, long long n, cudaStream_t stream) {
  const unsigned grid = (unsigned)((n + 1023) / 1024);
  if (sigmoid) {
    if (dt == CNB_DTYPE_BF16) k_sigmoid<<<grid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16 *>(src), out, n);
    else if (dt == CNB_DTYPE_F16) k_sigmoid<<<grid, 256, 0, stream>>>(reinterpret_cast<const __half *>(src), out, n);
    else k_sigmoid<<<grid, 256, 0, stream>>>(reinterpret_cast<const float *>(src), out, n);
  } else {
    if (dt == CNB_DTYPE_BF16) k_widen<<<grid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16 *>(src), out, n);
    else k_widen<<<grid, 256, 0, stream>>>(reinterpret_cast<const __half *>(src), out, n);
  }
  CNB_CHECK_LAUNCH(sigmoid ? "decode sigmoid pass" : "decode widening pass");
  count_launch();
  return CNB_OK;
}

int cnb::plan_map_select(const void *src, int dt, int logits, int n_img, int C, int H, int W, int K,
                         const float *copy, MapSelect *m) {
  int rc = make_select_plan(src, n_img, C, H, W, K, 1, &m->pl, dtype_bytes(dt));
  if (rc != CNB_OK) return rc;
  m->widen = !m->pl.hot && (dt != CNB_DTYPE_F32 || logits);
  m->map_bytes = 0;
  if (m->widen) {
    rc = make_select_plan(copy, n_img, C, H, W, K, 1, &m->pl);
    if (rc != CNB_OK) return rc;
    m->map_bytes = align_up((size_t)n_img * C * H * W * 4, 256);
  }
  m->pl.logits = (logits && !m->widen) ? 1 : 0;  // a widened map holds the sigmoid already
  m->sel_bytes = select_workspace_bytes(m->pl);
  return CNB_OK;
}

int cnb::run_map_select(const void *src, int dt, int logits, const MapSelect &m, float *copy, const FinalizeOut &out,
                        void *ws, cudaStream_t stream) {
  if (!m.widen) return run_select(src, m.pl, out, ws, stream, dt);
  const int rc = launch_to_f32(src, dt, logits != 0, copy, (long long)m.pl.n_img * m.pl.C * m.pl.H * m.pl.W, stream);
  if (rc != CNB_OK) return rc;
  return run_select(copy, m.pl, out, ws, stream);
}

// Flip-test merge (detectors/ctdet.py:34-37, detectors/multi_pose.py:43-51): src [2n, c, h, w] holds the heads
// of n images followed by those of their horizontally flipped copies; dst [n, c, h, w] =
//   ( f(src[i, ch]) + sign[ch] * f(flip_w(src[n + i, perm[ch]])) ) / 2,     f = sigmoid (mode 1) or identity.
// perm / sign (nullable) express flip_lr (joint swap, models/utils.py:33-39) and flip_lr_off (joint swap + negated
// x offsets, :41-50); null = flip_tensor (:28-29).  One pass instead of the reference's sigmoid_, slices, host
// round trip through numpy, add and divide.
template <typename T>
__global__ void __launch_bounds__(256) k_flip_merge(const T *__restrict__ src, float *__restrict__ dst, int n, int c,
                                                    int h, int w, int mode, const int *__restrict__ perm,
                                                    const float *__restrict__ sign) {
  const long long total = (long long)n * c * h * w;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % w);
    long long r = i / w;
    const int y = (int)(r % h);
    r /= h;
    const int ch = (int)(r % c), img = (int)(r / c);
    const int pc = perm ? perm[ch] : ch;
    float a = to_f32(src[i]);
    float b = to_f32(src[(((long long)(n + img) * c + pc) * h + y) * w + (w - 1 - x)]);
    if (mode == 1) {
      a = 1.0f / (1.0f + expf(-a));
      b = 1.0f / (1.0f + expf(-b));
    }
    if (sign) b = __fmul_rn(b, sign[ch]);
    dst[i] = __fadd_rn(a, b) / 2.0f;
  }
}

extern "C" {

int cnb_flip_merge(const float *src, float *dst, int n, int c, int h, int w, int apply_sigmoid, const int32_t *perm,
                   const float *sign, void *stream) {
  CNB_REQUIRE(src && dst, CNB_EINVAL, "cnb_flip_merge: null pointer");
  CNB_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "cnb_flip_merge: non-positive dimension");
  const long long total = (long long)n * c * h * w;
  const int grid = (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736);
  k_flip_merge<<<grid, 256, 0, (cudaStream_t)stream>>>(src, dst, n, c, h, w, apply_sigmoid ? 1 : 0, perm, sign);
  CNB_CHECK_LAUNCH("cnb_flip_merge");
  count_launch();
  return CNB_OK;
}

int cnb_flip_merge_ex(const void *src, int src_dtype, float *dst, int n, int c, int h, int w, int apply_sigmoid,
                      const int32_t *perm, const float *sign, void *stream) {
  CNB_REQUIRE(dtype_known(src_dtype), CNB_EINVAL, "cnb_flip_merge_ex: unknown dtype code %d", src_dtype);
  if (src_dtype == CNB_DTYPE_F32)
    return cnb_flip_merge(reinterpret_cast<const float *>(src), dst, n, c, h, w, apply_sigmoid, perm, sign, stream);
  CNB_REQUIRE(src && dst, CNB_EINVAL, "cnb_flip_merge_ex: null pointer");
  CNB_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "cnb_flip_merge_ex: non-positive dimension");
  const long long total = (long long)n * c * h * w;
  const int grid = (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736);
  const int mode = apply_sigmoid ? 1 : 0;
  if (src_dtype == CNB_DTYPE_BF16)
    k_flip_merge<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16 *>(src), dst, n, c, h,
                                                         w, mode, perm, sign);
  else
    k_flip_merge<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half *>(src), dst, n, c, h, w, mode,
                                                         perm, sign);
  CNB_CHECK_LAUNCH("cnb_flip_merge_ex");
  count_launch();
  return CNB_OK;
}

int cnb_nms(const float *heat, float *out, int n, int c, int h, int w, void *stream) {
  CNB_REQUIRE(heat && out, CNB_EINVAL, "cnb_nms: null pointer");
  CNB_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "cnb_nms: non-positive dimension");
  const long long planes = (long long)n * c;
  const bool vec = (w % 4 == 0) && (((uintptr_t)heat | (uintptr_t)out) & 15u) == 0;
  const long long work = planes * h * (vec ? w / 4 : w);
  const int grid = (int)((work + 255) / 256 < (long long)num_sms() * 16 ? (work + 255) / 256 : (long long)num_sms() * 16);
  if (vec)
    k_nms<true><<<grid, 256, 0, (cudaStream_t)stream>>>(heat, out, planes, h, w);
  else
    k_nms<false><<<grid, 256, 0, (cudaStream_t)stream>>>(heat, out, planes, h, w);
  CNB_CHECK_LAUNCH("cnb_nms");
  count_launch();
  return CNB_OK;
}

int cnb_gather_feat_backward(const float *grad_out, const int64_t *ind, float *grad_feat, int b, int c, int hw, int m,
                             void *stream) {
  CNB_REQUIRE(grad_out && ind && grad_feat, CNB_EINVAL, "cnb_gather_feat_backward: null pointer");
  CNB_REQUIRE(b > 0 && c > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_gather_feat_backward: non-positive dimension");
  const long long planes = (long long)b * c;
  const int grid = (int)((planes + 255) / 256 < 65535 ? (planes + 255) / 256 : 65535);
  k_gather_feat_bwd<<<grid, 256, 0, (cudaStream_t)stream>>>(grad_out, ind, grad_feat, b, c, hw, m);
  CNB_CHECK_LAUNCH("cnb_gather_feat_backward");
  count_launch();
  return CNB_OK;
}

int cnb_gather_feat(const float *feat, const int64_t *ind, float *out, int b, int c, int hw, int m, void *stream) {
  CNB_REQUIRE(feat && ind && out, CNB_EINVAL, "cnb_gather_feat: null pointer");
  CNB_REQUIRE(b > 0 && c > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_gather_feat: non-positive dimension");
  const long long total = (long long)b * m * c;
  const int grid = (int)((total + 255) / 256 < 65535 ? (total + 255) / 256 : 65535);
  k_gather_feat<<<grid, 256, 0, (cudaStream_t)stream>>>(feat, ind, out, b, c, hw, m);
  CNB_CHECK_LAUNCH("cnb_gather_feat");
  count_launch();
  return CNB_OK;
}

int cnb_gather_feat_ex(const void *feat, int feat_dtype, const int64_t *ind, float *out, int b, int c, int hw, int m,
                       void *stream) {
  CNB_REQUIRE(dtype_known(feat_dtype), CNB_EINVAL, "cnb_gather_feat_ex: unknown dtype code %d", feat_dtype);
  if (feat_dtype == CNB_DTYPE_F32) return cnb_gather_feat(reinterpret_cast<const float *>(feat), ind, out, b, c, hw, m, stream);
  CNB_REQUIRE(feat && ind && out, CNB_EINVAL, "cnb_gather_feat_ex: null pointer");
  CNB_REQUIRE(b > 0 && c > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_gather_feat_ex: non-positive dimension");
  const long long total = (long long)b * m * c;
  const int grid = (int)((total + 255) / 256 < 65535 ? (total + 255) / 256 : 65535);
  if (feat_dtype == CNB_DTYPE_BF16)
    k_gather_feat_half<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16 *>(feat), ind, out,
                                                               b, c, hw, m);
  else
    k_gather_feat_half<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half *>(feat), ind, out, b, c,
                                                               hw, m);
  CNB_CHECK_LAUNCH("cnb_gather_feat_ex");
  count_launch();
  return CNB_OK;
}

int cnb_gather_feat_backward_ex(const float *grad_out, const int64_t *ind, void *grad_feat, int feat_dtype, int b,
                                int c, int hw, int m, void *stream) {
  CNB_REQUIRE(dtype_known(feat_dtype), CNB_EINVAL, "cnb_gather_feat_backward_ex: unknown dtype code %d", feat_dtype);
  CNB_REQUIRE(grad_out && ind && grad_feat, CNB_EINVAL, "cnb_gather_feat_backward_ex: null pointer");
  CNB_REQUIRE(b > 0 && c > 0 && hw > 0 && m > 0, CNB_EINVAL, "cnb_gather_feat_backward_ex: non-positive dimension");
  const size_t elem = feat_dtype == CNB_DTYPE_F32 ? 4 : 2;
  CNB_CUDA(cudaMemsetAsync(grad_feat, 0, (size_t)b * c * hw * elem, (cudaStream_t)stream));
  if (feat_dtype == CNB_DTYPE_F32)
    return cnb_gather_feat_backward(grad_out, ind, reinterpret_cast<float *>(grad_feat), b, c, hw, m, stream);
  const long long total = (long long)b * m * c;
  const int grid = (int)((total + 255) / 256 < 65535 ? (total + 255) / 256 : 65535);
  if (feat_dtype == CNB_DTYPE_BF16)
    k_gather_feat_bwd_half<<<grid, 256, 0, (cudaStream_t)stream>>>(grad_out, ind,
                                                                   reinterpret_cast<__nv_bfloat16 *>(grad_feat), b, c,
                                                                   hw, m);
  else
    k_gather_feat_bwd_half<<<grid, 256, 0, (cudaStream_t)stream>>>(grad_out, ind, reinterpret_cast<__half *>(grad_feat),
                                                                   b, c, hw, m);
  CNB_CHECK_LAUNCH("cnb_gather_feat_backward_ex");
  count_launch();
  return CNB_OK;
}

size_t cnb_topk_workspace_bytes(int n_img, int c, int h, int w, int k) {
  SelectPlan pl;
  // worst case over alignment: the non-TMA plan has the same grid / slot count
  if (make_select_plan(nullptr, n_img, c, h, w, k, 1, &pl) != CNB_OK) return 0;
  return select_workspace_bytes(pl) + raw_bytes((long long)n_img * k);
}

int cnb_topk(const float *scores, int b, int c, int h, int w, int k, int fuse_nms, float *out_scores,
             int64_t *out_inds, int32_t *out_clses, float *out_ys, float *out_xs, void *workspace,
             size_t workspace_bytes, void *stream) {
  CNB_REQUIRE(scores && workspace, CNB_EINVAL, "cnb_topk: null pointer");
  SelectPlan pl;
  int rc = make_select_plan(scores, b, c, h, w, k, fuse_nms, &pl);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(workspace_bytes >= select_workspace_bytes(pl), CNB_EWORKSPACE,
              "cnb_topk: workspace %zu < %zu", workspace_bytes, select_workspace_bytes(pl));
  FinalizeOut out = {out_scores, out_inds, out_clses, out_ys, out_xs, nullptr, nullptr, 0, nullptr};
  return run_select(scores, pl, out, workspace, (cudaStream_t)stream);
}

int cnb_topk_channel(const float *scores, int b, int c, int h, int w, int k, int fuse_nms, float *out_scores,
                     int64_t *out_inds, float *out_ys, float *out_xs, void *workspace, size_t workspace_bytes,
                     void *stream) {
  CNB_REQUIRE(scores && workspace, CNB_EINVAL, "cnb_topk_channel: null pointer");
  CNB_REQUIRE(b > 0 && c > 0, CNB_EINVAL, "cnb_topk_channel: non-positive dimension");
  SelectPlan pl;  // every (b, channel) plane is its own "image" with one class
  int rc = make_select_plan(scores, b * c, 1, h, w, k, fuse_nms, &pl);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(workspace_bytes >= select_workspace_bytes(pl), CNB_EWORKSPACE,
              "cnb_topk_channel: workspace %zu < %zu", workspace_bytes, select_workspace_bytes(pl));
  FinalizeOut out = {out_scores, out_inds, nullptr, out_ys, out_xs, nullptr, nullptr, 0, nullptr};
  return run_select(scores, pl, out, workspace, (cudaStream_t)stream);
}

int cnb_ctdet_decode(const float *heat, const float *wh, const float *reg, int cat_spec_wh, int b, int c, int h,
                     int w, int k, float *dets, void *workspace, size_t workspace_bytes, void *stream) {
  CNB_REQUIRE(heat && wh && dets && workspace, CNB_EINVAL, "cnb_ctdet_decode: null pointer");
  SelectPlan pl;
  int rc = make_select_plan(heat, b, c, h, w, k, 1, &pl);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(workspace_bytes >= select_workspace_bytes(pl), CNB_EWORKSPACE,
              "cnb_ctdet_decode: workspace %zu < %zu", workspace_bytes, select_workspace_bytes(pl));
  FinalizeOut out = {nullptr, nullptr, nullptr, nullptr, nullptr, wh, reg, cat_spec_wh, dets};
  return run_select(heat, pl, out, workspace, (cudaStream_t)stream);
}

/* N1 (SURVEY 8f): ctdet_decode on the head's raw logits, sigmoid fused (detectors/ctdet.py:31 +
 * models/decode.py:464-495).  Hot geometry: the selection kernel works in logit space and applies
 * the sigmoid only to the few candidates; other geometries materialise the heat map once in the
 * workspace and take the normal path. */
size_t cnb_ctdet_logits_workspace_bytes(const float *hm_logits, int b, int c, int h, int w, int k) {
  SelectPlan pl;
  if (make_select_plan(hm_logits, b, c, h, w, k, 1, &pl) != CNB_OK) return 0;
  size_t n = select_workspace_bytes(pl);
  if (!pl.hot) n = align_up(n, 256) + align_up((size_t)b * c * h * w * 4, 256);
  return n;
}

int cnb_ctdet_decode_logits(const float *hm_logits, const float *wh, const float *reg, int cat_spec_wh, int b, int c,
                            int h, int w, int k, float *dets, void *workspace, size_t workspace_bytes, void *stream) {
  CNB_REQUIRE(hm_logits && wh && dets && workspace, CNB_EINVAL, "cnb_ctdet_decode_logits: null pointer");
  SelectPlan pl;
  int rc = make_select_plan(hm_logits, b, c, h, w, k, 1, &pl);
  if (rc != CNB_OK) return rc;
  const size_t need = cnb_ctdet_logits_workspace_bytes(hm_logits, b, c, h, w, k);
  CNB_REQUIRE(workspace_bytes >= need, CNB_EWORKSPACE, "cnb_ctdet_decode_logits: workspace %zu < %zu", workspace_bytes,
              need);
  FinalizeOut out = {nullptr, nullptr, nullptr, nullptr, nullptr, wh, reg, cat_spec_wh, dets};
  if (pl.hot) {
    pl.logits = 1;
    return run_select(hm_logits, pl, out, workspace, (cudaStream_t)stream);
  }
  float *heat = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + align_up(select_workspace_bytes(pl), 256));
  const long long n = (long long)b * c * h * w;
  k_sigmoid<<<(unsigned)((n + 1023) / 1024), 256, 0, (cudaStream_t)stream>>>(hm_logits, heat, n);
  CNB_CHECK_LAUNCH("cnb_ctdet_decode_logits sigmoid");
  count_launch();
  rc = make_select_plan(heat, b, c, h, w, k, 1, &pl);
  if (rc != CNB_OK) return rc;
  return run_select(heat, pl, out, workspace, (cudaStream_t)stream);
}

/* fp32, fp16 or bf16 heads (see the header): the hot geometry reads a 16-bit map in the selection kernel itself;
 * other geometries widen it (or take its sigmoid) into the workspace, after the selection scratch, and run the fp32
 * path.  Layout: [selection scratch | fp32 heat map], the map at the fp32 query's size (logits == 0) or at the
 * aligned selection scratch of the plan (logits != 0, as cnb_ctdet_decode_logits). */
size_t cnb_ctdet_decode_ex_workspace_bytes(const void *heat, int heat_dtype, int logits, int b, int c, int h, int w,
                                           int k) {
  if (!dtype_known(heat_dtype)) return 0;
  SelectPlan pl;
  if (make_select_plan(heat, b, c, h, w, k, 1, &pl, dtype_bytes(heat_dtype)) != CNB_OK) return 0;
  const size_t map = align_up((size_t)b * c * h * w * 4, 256);
  if (logits) return pl.hot ? select_workspace_bytes(pl) : align_up(select_workspace_bytes(pl), 256) + map;
  const size_t base = cnb_topk_workspace_bytes(b, c, h, w, k);
  return (heat_dtype == CNB_DTYPE_F32 || pl.hot) ? base : base + map;
}

int cnb_ctdet_decode_ex(const void *heat, int heat_dtype, int logits, const void *wh, int wh_dtype, const void *reg,
                        int reg_dtype, int cat_spec_wh, int b, int c, int h, int w, int k, float *dets,
                        void *workspace, size_t workspace_bytes, void *stream) {
  CNB_REQUIRE(dtype_known(heat_dtype) && dtype_known(wh_dtype) && dtype_known(reg_dtype), CNB_EINVAL,
              "cnb_ctdet_decode_ex: unknown dtype code (heat %d, wh %d, reg %d)", heat_dtype, wh_dtype, reg_dtype);
  CNB_REQUIRE(heat && wh && dets && workspace, CNB_EINVAL, "cnb_ctdet_decode_ex: null pointer");
  SelectPlan pl;
  int rc = make_select_plan(heat, b, c, h, w, k, 1, &pl, dtype_bytes(heat_dtype));
  if (rc != CNB_OK) return rc;
  const size_t need = cnb_ctdet_decode_ex_workspace_bytes(heat, heat_dtype, logits, b, c, h, w, k);
  CNB_REQUIRE(workspace_bytes >= need, CNB_EWORKSPACE, "cnb_ctdet_decode_ex: workspace %zu < %zu", workspace_bytes,
              need);
  FinalizeOut out = {nullptr, nullptr, nullptr, nullptr, nullptr, wh, reg, cat_spec_wh, dets, wh_dtype, reg_dtype};
  const cudaStream_t st = (cudaStream_t)stream;
  if (pl.hot) {
    pl.logits = logits ? 1 : 0;
    return run_select(heat, pl, out, workspace, st, heat_dtype);
  }
  if (!logits && heat_dtype == CNB_DTYPE_F32) return run_select(heat, pl, out, workspace, st);
  const size_t off = logits ? align_up(select_workspace_bytes(pl), 256) : cnb_topk_workspace_bytes(b, c, h, w, k);
  float *heat32 = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + off);
  SelectPlan pf;
  rc = make_select_plan(heat32, b, c, h, w, k, 1, &pf);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(select_workspace_bytes(pf) <= off, CNB_EWORKSPACE, "cnb_ctdet_decode_ex: selection scratch %zu > %zu",
              select_workspace_bytes(pf), off);
  rc = launch_to_f32(heat, heat_dtype, logits != 0, heat32, (long long)b * c * h * w, st);
  if (rc != CNB_OK) return rc;
  return run_select(heat32, pf, out, workspace, st);
}

int cnb_sigmoid(const float *x, float *out, long long n, void *stream) {
  CNB_REQUIRE(x && out && n >= 0, CNB_EINVAL, "cnb_sigmoid: bad argument");
  if (n == 0) return CNB_OK;
  k_sigmoid<<<(unsigned)((n + 1023) / 1024), 256, 0, (cudaStream_t)stream>>>(x, out, n);
  CNB_CHECK_LAUNCH("cnb_sigmoid");
  count_launch();
  return CNB_OK;
}

int cnb_ddd_decode(const float *heat, const float *rot, const float *depth, const float *dim, const float *wh,
                   const float *reg, int b, int c, int h, int w, int k, float *dets, void *workspace,
                   size_t workspace_bytes, void *stream) {
  CNB_REQUIRE(heat && rot && depth && dim && dets && workspace, CNB_EINVAL, "cnb_ddd_decode: null pointer");
  SelectPlan pl;
  int rc = make_select_plan(heat, b, c, h, w, k, 1, &pl);
  if (rc != CNB_OK) return rc;
  const size_t sel = select_workspace_bytes(pl);
  CNB_REQUIRE(workspace_bytes >= sel + raw_bytes((long long)b * k), CNB_EWORKSPACE,
              "cnb_ddd_decode: workspace %zu < %zu", workspace_bytes, sel + raw_bytes((long long)b * k));
  RawTopk r = carve_raw(reinterpret_cast<char *>(workspace) + sel, (long long)b * k);
  FinalizeOut out = {r.scores, r.inds, r.clses, r.ys, r.xs, nullptr, nullptr, 0, nullptr};
  rc = run_select(heat, pl, out, workspace, (cudaStream_t)stream);
  if (rc != CNB_OK) return rc;
  k_ddd_epilogue<<<(b * k + 127) / 128, 128, 0, (cudaStream_t)stream>>>(r.scores, r.inds, r.clses, r.ys, r.xs, rot,
                                                                         depth, dim, wh, reg, b, k,
                                                                         (long long)h * w, dets);
  CNB_CHECK_LAUNCH("cnb_ddd_decode epilogue");
  count_launch();
  return CNB_OK;
}

/* cnb_ddd_decode of fp32, fp16 or bf16 heads, the heat map or its logits (see the header).  Layout:
 * [selection scratch | raw top-K | fp32 copy of the heat map (only when it is widened)]. */
size_t cnb_ddd_decode_ex_workspace_bytes(const void *heat, int heat_dtype, int logits, int b, int c, int h, int w,
                                         int k) {
  if (!dtype_known(heat_dtype)) return 0;
  MapSelect m;
  if (plan_map_select(heat, heat_dtype, logits, b, c, h, w, k, nullptr, &m) != CNB_OK) return 0;
  return m.sel_bytes + raw_bytes((long long)b * k) + m.map_bytes;
}

int cnb_ddd_decode_ex(const void *heat, int heat_dtype, int logits, const void *rot, int rot_dtype, const void *depth,
                      int depth_dtype, const void *dim, int dim_dtype, const void *wh, int wh_dtype, const void *reg,
                      int reg_dtype, int b, int c, int h, int w, int k, float *dets, void *workspace,
                      size_t workspace_bytes, void *stream) {
  CNB_REQUIRE(dtype_known(heat_dtype) && dtype_known(rot_dtype) && dtype_known(depth_dtype) && dtype_known(dim_dtype) &&
                  dtype_known(wh_dtype) && dtype_known(reg_dtype),
              CNB_EINVAL, "cnb_ddd_decode_ex: unknown dtype code (heat %d, rot %d, depth %d, dim %d, wh %d, reg %d)",
              heat_dtype, rot_dtype, depth_dtype, dim_dtype, wh_dtype, reg_dtype);
  CNB_REQUIRE(heat && rot && depth && dim && dets && workspace, CNB_EINVAL, "cnb_ddd_decode_ex: null pointer");
  MapSelect m;
  int rc = plan_map_select(heat, heat_dtype, logits, b, c, h, w, k, nullptr, &m);
  if (rc != CNB_OK) return rc;
  const size_t sel = m.sel_bytes, raw = raw_bytes((long long)b * k);
  CNB_REQUIRE(workspace_bytes >= sel + raw + m.map_bytes, CNB_EWORKSPACE, "cnb_ddd_decode_ex: workspace %zu < %zu",
              workspace_bytes, sel + raw + m.map_bytes);
  char *p = reinterpret_cast<char *>(workspace);
  RawTopk r = carve_raw(p + sel, (long long)b * k);
  float *copy = reinterpret_cast<float *>(p + sel + raw);
  if (m.widen) {  // the plan of the copy where it really lies (a workspace that is not 16-byte aligned loses TMA)
    rc = plan_map_select(heat, heat_dtype, logits, b, c, h, w, k, copy, &m);
    if (rc != CNB_OK) return rc;
    CNB_REQUIRE(m.sel_bytes <= sel, CNB_EWORKSPACE, "cnb_ddd_decode_ex: selection scratch %zu > %zu", m.sel_bytes,
                sel);
  }
  const cudaStream_t st = (cudaStream_t)stream;
  FinalizeOut out = {r.scores, r.inds, r.clses, r.ys, r.xs, nullptr, nullptr, 0, nullptr};
  rc = run_map_select(heat, heat_dtype, logits, m, copy, out, workspace, st);
  if (rc != CNB_OK) return rc;
  const DddHeads hd = {rot_dtype, depth_dtype, dim_dtype, wh_dtype, reg_dtype, logits ? 1 : 0};
  k_ddd_epilogue_ex<<<(b * k + 127) / 128, 128, 0, st>>>(r.scores, r.inds, r.clses, r.ys, r.xs, rot, depth, dim, wh,
                                                         reg, hd, b, k, (long long)h * w, dets);
  CNB_CHECK_LAUNCH("cnb_ddd_decode_ex epilogue");
  count_launch();
  return CNB_OK;
}

}  // extern "C"

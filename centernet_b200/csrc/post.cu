// Detection post-processing on the device (SURVEY 8f N2): removes the per-scale D2H round trip of
//   utils/post_process.py:83-114   ctdet_post_process / multi_pose_post_process  (affine back-projection)
//   external/nms.pyx:77-275        soft_nms / soft_nms_39
//   detectors/ctdet.py:76-92       merge_outputs (concat over scales, per-class soft-NMS, top max_per_image)
// The detections stay on the GPU from decode to the final per-class lists; the host reads ONE packed result.
//
// Arithmetic follows the reference to the bit where it is defined: the affine map is applied in float64
// to float32 points (np.dot of the float64 cv2 matrix with a float32 point, utils/image.py:63-66), the
// soft-NMS overlaps use the float32 storage / float64 intermediates of the Cython-generated C (integer
// literals become the double 1.0) and the Gaussian weight goes through a float64 exp.
#include "common.cuh"
#include "warp.cuh"

namespace cnb {

// One row of np.dot(t, [x, y, 1.]) (utils/image.py:63-66): the float64 2x3 matrix row t times a float32 point,
// (t0 * x + t1 * y) + t2 with no fused multiply-add, stored to float32 as the reference's float32 arrays store it.
__device__ __forceinline__ float affine_row(const double *__restrict__ t, float x, float y) {
  return (float)__dadd_rn(__dadd_rn(__dmul_rn(t[0], (double)x), __dmul_rn(t[1], (double)y)), t[2]);
}

// rows [b][n][d] -> out (same shape): columns copied, the point pairs (x, y) at columns
// [a0, a0 + 2 na) and [b0, b0 + 2 nb) mapped through the image's 2x3 float64 matrix.
__global__ void __launch_bounds__(256) k_post_transform(const float *__restrict__ in, float *__restrict__ out,
                                                        const double *__restrict__ trans, int b, int n, int d,
                                                        int a0, int na, int b0, int nb) {
  const long long total = (long long)b * n * d;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % d);
    const long long row = i / d;
    const int img = (int)(row / n);
    float v = in[i];
    int rel = -1;
    if (col >= a0 && col < a0 + 2 * na) rel = col - a0;
    else if (col >= b0 && col < b0 + 2 * nb) rel = col - b0;
    if (rel >= 0) {
      const int isy = rel & 1;
      const float x = in[i - isy], y = in[i - isy + 1];
      v = affine_row(trans + (size_t)img * 6 + isy * 3, x, y);
    }
    out[i] = v;
  }
}

// exdet post_process (detectors/exdet.py:85-95) of one scale: rows [b][n][d], image i = rows [i*n, (i+1)*n) split in
// two equal halves as reshape(2, -1, 14) splits them.  In the second half x1 <- out_w - x2 and x2 <- out_w - x1
// (float32), then the point pairs (0,1) and (2,3) are mapped through the image's matrix as k_post_transform maps
// them; every other column is copied.
__global__ void __launch_bounds__(256) k_exdet_transform(const float *__restrict__ in, float *__restrict__ out,
                                                         const double *__restrict__ trans, int b, int n, int d,
                                                         float out_w) {
  const long long total = (long long)b * n * d;
  const int half = n >> 1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % d);
    const long long row = i / d;
    const int img = (int)(row / n);
    float v = in[i];
    if (col < 4) {
      const float *p = in + row * d;
      const bool mirrored = (int)(row - (long long)img * n) >= half;
      const int isy = col & 1;
      float x = p[col - isy];
      if (mirrored) x = __fsub_rn(out_w, p[2 - (col - isy)]);
      const float y = p[col - isy + 1];
      v = affine_row(trans + (size_t)img * 6 + isy * 3, x, y);
    }
    out[i] = v;
  }
}

// One CTA per image.  dets [n][dw] with a float class id in column cls_col -> rows [n][Rows::kWidth] grouped by class
// in class order, input order kept inside a class (boolean-mask indexing of post_process.py:93-97), and offsets
// [num_classes + 1].  Rows whose class id is outside [0, num_classes) are dropped (as the mask does), and so are
// rows the policy's keep() refuses; emit() writes a kept row's output columns.
template <class Rows>
__device__ __forceinline__ void group_rows(const float *__restrict__ dets, int n, int dw, int cls_col, int num_classes,
                                           float *__restrict__ rows, int *__restrict__ offsets, const Rows &rw) {
  extern __shared__ int gsm[];
  int *cnt = gsm;                    // [num_classes + 1] counts -> running offsets
  int *cls_chunk = gsm + num_classes + 1;   // [256]
  const int img = blockIdx.x, tid = threadIdx.x;
  const float *d = dets + (size_t)img * n * dw;
  float *r = rows + (size_t)img * n * Rows::kWidth;
  int *off = offsets + (size_t)img * (num_classes + 1);
  auto in_class = [&](int i, int &c) {   // c = the row's class id; false when the row is dropped
    const float cf = d[(size_t)i * dw + cls_col];
    c = (int)cf;
    if (!rw.keep(d + (size_t)i * dw)) return false;
    return (float)c == cf && c >= 0 && c < num_classes;
  };
  for (int c = tid; c <= num_classes; c += blockDim.x) cnt[c] = 0;
  __syncthreads();
  for (int i = tid; i < n; i += blockDim.x) {
    int c;
    if (in_class(i, c)) atomicAdd(&cnt[c + 1], 1);
  }
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int c = 0; c <= num_classes; ++c) { run += cnt[c]; cnt[c] = run; }   // cnt[c] = first row of class c
  }
  __syncthreads();
  for (int c = tid; c <= num_classes; c += blockDim.x) off[c] = cnt[c];
  __syncthreads();
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + tid;
    int c = -1;
    if (i < n) {
      int ci;
      if (in_class(i, ci)) c = ci;
    }
    cls_chunk[tid] = c;
    __syncthreads();
    int before = 0;
    if (c >= 0)
      for (int t = 0; t < tid; ++t) before += (cls_chunk[t] == c) ? 1 : 0;
    int dst = -1;
    if (c >= 0) dst = cnt[c] + before;
    __syncthreads();
    if (c >= 0) {
      atomicAdd(&cnt[c], 1);          // running offset for the next chunk (all adds of a chunk land before the next read)
      rw.emit(d + (size_t)i * dw, r + (size_t)dst * Rows::kWidth);
    }
    __syncthreads();
  }
}

// x1,y1,x2,y2,score of columns 0-4; with kPositive only rows whose score is > 0 (NaN dropped).
template <bool kPositive>
struct BoxRows {
  static constexpr int kWidth = 5;
  __device__ __forceinline__ bool keep(const float *__restrict__ row) const { return !kPositive || row[4] > 0.f; }
  __device__ __forceinline__ void emit(const float *__restrict__ row, float *__restrict__ out) const {
#pragma unroll
    for (int k = 0; k < 5; ++k) out[k] = row[k];
  }
};

// ctdet rows: [n][6] = x1,y1,x2,y2,score,class.
__global__ void __launch_bounds__(256) k_group_by_class(const float *__restrict__ dets, int n, int num_classes,
                                                        float *__restrict__ rows, int *__restrict__ offsets) {
  group_rows(dets, n, 6, 5, num_classes, rows, offsets, BoxRows<false>());
}

// Rows of any width, class in column cls_col, only rows with score > 0 (exdet merge_outputs, detectors/exdet.py:99-108).
__global__ void __launch_bounds__(256) k_group_positive_by_class(const float *__restrict__ dets, int n, int d,
                                                                 int cls_col, int num_classes, float *__restrict__ rows,
                                                                 int *__restrict__ offsets) {
  group_rows(dets, n, d, cls_col, num_classes, rows, offsets, BoxRows<true>());
}

// The ddd tail of one row: ddd_post_process (utils/post_process.py:13-80 with ddd2locrot, utils/ddd_utils.py:66-111)
// of a ddd_decode row [18] = x, y, score, rot[8], depth, dim[3], w, h, class -> [13] = alpha, x1, y1, x2, y2,
// dim[3], X, Y, Z, rot_y, score.  Every step is the reference's float32 (or, for the affine, float64) operation,
// rounded where numpy rounds it; nothing is contracted into a fused multiply-add.
//   * (x, y) and (w, h) both go through the full inverse affine, translation included (the reference transforms
//     wh with transform_preds), and the box is centre -+ transformed wh / 2;
//   * get_alpha: bin 1 when rot[1] > rot[5] (NaN and ties: bin 2), atan2(sin, cos) -+ float32(pi / 2) in float32;
//     alpha1 * idx + alpha2 * (1 - idx) is float64, so a NaN in either bin makes alpha NaN;
//   * unproject_2d_to_3d, left to right in float32, then Y += dim0 / 2;
//   * alpha2rot_y: alpha + atan2(u - P[0,2], P[0,0]), wrapped once each way against float32(pi) (numpy 2 compares a
//     float32 scalar with a Python float in float32).
// atan2 is evaluated in float64 and rounded, the closest float32 to the angle; numpy's float32 arctan2 is within
// a few ulp of it.
struct DddRows {
  static constexpr int kWidth = 13;
  const double *t;   // the image's 2x3 inverse affine
  const float *P;    // the image's 3x4 calibration, row major
  bool cut;          // merge_outputs: keep score > thresh (NaN dropped); post_process: keep every row
  float thresh;
  __device__ __forceinline__ bool keep(const float *__restrict__ row) const { return !cut || row[2] > thresh; }
  __device__ __forceinline__ void emit(const float *__restrict__ r, float *__restrict__ o) const {
    const float kHalfPi = 1.57079632679489661923f, kPi = 3.14159265358979323846f, kTwoPi = 6.28318530717958647692f;
    const float cx = affine_row(t, r[0], r[1]), cy = affine_row(t + 3, r[0], r[1]);
    const float tw = affine_row(t, r[15], r[16]), th = affine_row(t + 3, r[15], r[16]);
    const float a1 = __fadd_rn((float)atan2((double)r[5], (double)r[6]), -kHalfPi);
    const float a2 = __fadd_rn((float)atan2((double)r[9], (double)r[10]), kHalfPi);
    float alpha = (r[4] > r[8]) ? a1 : a2;
    if (a1 != a1 || a2 != a2) alpha = __int_as_float(0x7fffffff);
    const float depth = r[11], dim0 = r[12];
    const float z = __fsub_rn(depth, P[11]);
    const float X = __fdiv_rn(__fsub_rn(__fsub_rn(__fmul_rn(cx, depth), P[3]), __fmul_rn(P[2], z)), P[0]);
    const float Y = __fdiv_rn(__fsub_rn(__fsub_rn(__fmul_rn(cy, depth), P[7]), __fmul_rn(P[6], z)), P[5]);
    float ry = __fadd_rn(alpha, (float)atan2((double)__fsub_rn(cx, P[2]), (double)P[0]));
    if (ry > kPi) ry = __fsub_rn(ry, kTwoPi);
    if (ry < -kPi) ry = __fadd_rn(ry, kTwoPi);
    const float hw = __fdiv_rn(tw, 2.f), hh = __fdiv_rn(th, 2.f);
    o[0] = alpha;
    o[1] = __fsub_rn(cx, hw); o[2] = __fsub_rn(cy, hh); o[3] = __fadd_rn(cx, hw); o[4] = __fadd_rn(cy, hh);
    o[5] = dim0; o[6] = r[13]; o[7] = r[14];
    o[8] = X; o[9] = __fadd_rn(Y, __fdiv_rn(dim0, 2.f)); o[10] = z;
    o[11] = ry;
    o[12] = r[2];
  }
};

// ddd rows [n][18] (class in column 17) -> rows [n][13] grouped by class and offsets, the score cut applied when
// `cut` is set.  seen (nullable) [num_classes]: 1 where the class has a row before the cut, else 0 -- what tells
// merge_outputs' untouched empty list (shape (0,)) from a list the cut emptied (shape (0, 13)).
__global__ void __launch_bounds__(256) k_ddd_tail(const float *__restrict__ dets, int n, const double *__restrict__ trans,
                                                  const float *__restrict__ calib, int num_classes, int cut, float thresh,
                                                  float *__restrict__ rows, int *__restrict__ offsets,
                                                  unsigned char *__restrict__ seen) {
  const int img = blockIdx.x;
  if (seen) {
    unsigned char *sn = seen + (size_t)img * num_classes;
    for (int c = threadIdx.x; c < num_classes; c += blockDim.x) sn[c] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const float cf = dets[((size_t)img * n + i) * 18 + 17];
      const int c = (int)cf;
      if ((float)c == cf && c >= 0 && c < num_classes) sn[c] = 1;
    }
  }
  group_rows(dets, n, 18, 17, num_classes, rows, offsets,
             DddRows{trans + (size_t)img * 6, calib + (size_t)img * 12, cut != 0, thresh});
}

// Rows of one list held in shared memory: 5 floats + new score + perm + flags = 27 B per row.  The launch sizes its
// shared memory from n_cap (the longest list possible), so 4096 rows take 110.6 KB of the 227 KB opt-in and a
// typical merge (n = 200-500) a few KB.
constexpr int NMS_MAX_ROWS = 4096;
constexpr size_t NMS_ROW_BYTES = 5 * 4 + 4 + 2 + 1;

// nms.pyx:18-22: `a if a <= b else b` / `a if a >= b else b` -- a NaN second operand is returned, a NaN first
// operand is not (fminf / fmaxf would return the non-NaN operand in both cases)
__device__ __forceinline__ float pyx_min(float a, float b) { return a <= b ? a : b; }
__device__ __forceinline__ float pyx_max(float a, float b) { return a >= b ? a : b; }

// One warp per list.  List l = (image l / lists_per_img, class l % lists_per_img) covers rows
// image * img_stride + [offsets[image][class], offsets[image][class + 1]) of `in` ([*, d] floats; columns 0-4 =
// x1,y1,x2,y2,score; d = 5 or 39).  Result written to `out` (may alias `in` when d == 5).  The whole array --
// rows beyond the final N included -- ends up exactly as the reference's in-place routine leaves it.  Shared
// memory holds list_cap rows; a longer list is left untouched and flagged.
__device__ __forceinline__ void soft_nms_list(const float *__restrict__ in, float *__restrict__ out,
                                              const int *__restrict__ offsets, int lists_per_img, int img_stride,
                                              int n_cap, int d, float sigma, float Nt, float threshold, int method,
                                              int *__restrict__ final_n) {
  extern __shared__ __align__(16) unsigned char nsm[];
  float *bx = reinterpret_cast<float *>(nsm);                 // [n_cap][5]
  float *ns = bx + (size_t)n_cap * 5;                         // new score of the current iteration
  unsigned short *perm = reinterpret_cast<unsigned short *>(ns + n_cap);   // original row of the extra columns
  unsigned char *flag = reinterpret_cast<unsigned char *>(perm + n_cap);   // bit0: overlapped, bit1: below threshold
  const int lane = threadIdx.x;
  const int l = blockIdx.x;
  const int img = l / lists_per_img, cls = l - img * lists_per_img;
  const int *off = offsets + (size_t)img * (lists_per_img + 1) + cls;
  const int r0 = img * img_stride + off[0];
  int N = off[1] - off[0];
  if (N <= 0) {
    if (final_n && lane == 0) final_n[l] = 0;
    return;
  }
  if (N > n_cap) {   // a list longer than the shared-memory capacity: leave it untouched, flag it
    for (int i = lane; i < N * d; i += 32) out[(size_t)r0 * d + i] = in[(size_t)r0 * d + i];
    if (final_n && lane == 0) final_n[l] = -N;
    return;
  }
  const int N0 = N;
  for (int i = lane; i < N; i += 32) {
#pragma unroll
    for (int k = 0; k < 5; ++k) bx[i * 5 + k] = in[(size_t)(r0 + i) * d + k];
    perm[i] = (unsigned short)i;
  }
  __syncwarp();
  for (int i = 0; i < N; ++i) {
    // ---- first maximum of the scores in [i, N)   (nms.pyx:95-101: strict '<' scan)
    float best = -__int_as_float(0x7f800000);
    int bpos = 0x7fffffff;
    for (int p = i + lane; p < N; p += 32) {
      const float s = bx[p * 5 + 4];
      if (s > best) { best = s; bpos = p; }       // ascending p per lane: first maximum kept
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int op = __shfl_xor_sync(0xffffffffu, bpos, o);
      if (ob > best || (ob == best && op < bpos)) { best = ob; bpos = op; }
    }
    // a list whose scores are all NaN / -inf never updates maxpos in the reference: it stays at i
    if (bpos == 0x7fffffff || !(best > bx[i * 5 + 4])) bpos = i;
    if (lane == 0 && bpos != i) {     // swap box i <-> maxpos (:104-115), extra columns follow (soft_nms_39 :204-207)
#pragma unroll
      for (int k = 0; k < 5; ++k) { const float t = bx[i * 5 + k]; bx[i * 5 + k] = bx[bpos * 5 + k]; bx[bpos * 5 + k] = t; }
      const unsigned short t = perm[i]; perm[i] = perm[bpos]; perm[bpos] = t;
    }
    __syncwarp();
    const float tx1 = bx[i * 5 + 0], ty1 = bx[i * 5 + 1], tx2 = bx[i * 5 + 2], ty2 = bx[i * 5 + 3];
    // ---- new scores of every later box against box i (:125-153), in parallel
    for (int p = i + 1 + lane; p < N; p += 32) {
      const float x1 = bx[p * 5 + 0], y1 = bx[p * 5 + 1], x2 = bx[p * 5 + 2], y2 = bx[p * 5 + 3], s = bx[p * 5 + 4];
      const float area = (float)__dmul_rn(__dadd_rn((double)(x2 - x1), 1.0), __dadd_rn((double)(y2 - y1), 1.0));
      const float iw = (float)__dadd_rn((double)(pyx_min(tx2, x2) - pyx_max(tx1, x1)), 1.0);
      float nsv = s;
      unsigned char f = 0;
      if (iw > 0.f) {
        const float ih = (float)__dadd_rn((double)(pyx_min(ty2, y2) - pyx_max(ty1, y1)), 1.0);
        if (ih > 0.f) {
          const float inter = __fmul_rn(iw, ih);
          const double u = __dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)(tx2 - tx1), 1.0), __dadd_rn((double)(ty2 - ty1), 1.0)),
                                               (double)area), -(double)inter);
          const float ua = (float)u;
          const float ov = __fdiv_rn(inter, ua);
          float weight;
          if (method == 1) weight = (ov > Nt) ? (float)__dadd_rn(1.0, -(double)ov) : 1.0f;
          else if (method == 2) weight = (float)exp((double)__fdiv_rn(-__fmul_rn(ov, ov), sigma));
          else weight = (ov > Nt) ? 0.0f : 1.0f;
          nsv = __fmul_rn(weight, s);
          f = 1 | ((nsv < threshold) ? 2 : 0);
        }
      }
      ns[p] = nsv;
      flag[p] = f;
    }
    __syncwarp();
    // ---- apply + swap-with-last discard, in the reference's order (:153-166); one lane, shared memory only
    if (lane == 0) {
      int p = i + 1;
      while (p < N) {
        bx[p * 5 + 4] = ns[p];
        if (flag[p] & 2) {
#pragma unroll
          for (int k = 0; k < 5; ++k) bx[p * 5 + k] = bx[(N - 1) * 5 + k];     // COPY of the five box columns
          ns[p] = ns[N - 1];
          flag[p] = flag[N - 1];
          const unsigned short t = perm[p]; perm[p] = perm[N - 1]; perm[N - 1] = t;   // extra columns SWAP (:262-265)
          --N;
        } else {
          ++p;
        }
      }
      ns[0] = __int_as_float(N);
    }
    __syncwarp();
    N = __float_as_int(ns[0]);
    __syncwarp();
  }
  for (int i = lane; i < N0; i += 32) {
#pragma unroll
    for (int k = 0; k < 5; ++k) out[(size_t)(r0 + i) * d + k] = bx[i * 5 + k];
  }
  if (d > 5) {
    for (int i = lane; i < N0 * (d - 5); i += 32) {
      const int row = i / (d - 5), k = 5 + i - row * (d - 5);
      out[(size_t)(r0 + row) * d + k] = in[(size_t)(r0 + perm[row]) * d + k];
    }
  }
  if (final_n && lane == 0) final_n[l] = N;
}

// Images of n_cap rows, lists of at most n_cap rows (offsets from k_group_by_class are never longer).
__global__ void __launch_bounds__(32) k_soft_nms(const float *__restrict__ in, float *__restrict__ out,
                                                 const int *__restrict__ offsets, int lists_per_img, int n_cap,
                                                 int d, float sigma, float Nt, float threshold, int method,
                                                 int *__restrict__ final_n) {
  soft_nms_list(in, out, offsets, lists_per_img, n_cap, n_cap, d, sigma, Nt, threshold, method, final_n);
}

// Images of img_stride rows (up to TOPK_WIDE_MAX_ROWS), lists of at most list_cap <= NMS_MAX_ROWS rows.
__global__ void __launch_bounds__(32) k_soft_nms_strided(const float *__restrict__ in, float *__restrict__ out,
                                                         const int *__restrict__ offsets, int lists_per_img,
                                                         int img_stride, int list_cap, int d, float sigma, float Nt,
                                                         float threshold, int method, int *__restrict__ final_n) {
  soft_nms_list(in, out, offsets, lists_per_img, img_stride, list_cap, d, sigma, Nt, threshold, method, final_n);
}

// One CTA per image: threshold = max_per_image-th largest score of the image's n rows (np.partition(scores,
// kth)[kth], detectors/ctdet.py:85-88), keep[i] = score >= threshold.  n <= 4096.  No cut when n <= max_per_image.
// NaN of either sign orders above +inf, as np.partition sorts it.
__global__ void __launch_bounds__(1024) k_topk_keep(const float *__restrict__ rows, int d, const int *__restrict__ offsets,
                                                    int num_classes, int n_cap, int max_per_image,
                                                    unsigned char *__restrict__ keep, float *__restrict__ thresh_out) {
  extern __shared__ float ksm[];   // [4096] sortable keys
  const int img = blockIdx.x, tid = threadIdx.x;
  const int n = offsets[(size_t)img * (num_classes + 1) + num_classes];
  const float *r = rows + (size_t)img * n_cap * d;
  unsigned char *kp = keep + (size_t)img * n_cap;
  if (n <= max_per_image) {
    for (int i = tid; i < n; i += blockDim.x) kp[i] = 1;
    if (tid == 0 && thresh_out) thresh_out[img] = -__int_as_float(0x7f800000);
    return;
  }
  int m = 2;
  while (m < n) m <<= 1;
  uint32_t *key = reinterpret_cast<uint32_t *>(ksm);
  for (int i = tid; i < m; i += blockDim.x) {
    uint32_t k = 0u;   // pads sort below every real score
    if (i < n) {
      uint32_t u = __float_as_uint(r[(size_t)i * d + 4]);
      if ((u & 0x7fffffffu) > 0x7f800000u) u &= 0x7fffffffu;   // NaN: sign bit cleared, above +inf
      k = (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // order-preserving float -> uint, >= ~(-inf) > 0
    }
    key[i] = k;
  }
  __syncthreads();
  for (int k2 = 2; k2 <= m; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (m >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const uint32_t a = key[i], b = key[i + j];
        const bool desc = (i & k2) == 0;
        if ((a < b) == desc) { key[i] = b; key[i + j] = a; }
      }
      __syncthreads();
    }
  }
  const uint32_t tk = key[max_per_image - 1];
  const float thr = __uint_as_float((tk & 0x80000000u) ? (tk & 0x7fffffffu) : ~tk);
  for (int i = tid; i < n; i += blockDim.x) kp[i] = (r[(size_t)i * d + 4] >= thr) ? 1 : 0;
  if (tid == 0 && thresh_out) thresh_out[img] = thr;
}

// k_topk_keep's cut for images of up to TOPK_WIDE_MAX_ROWS rows: the same sortable keys, held in shared memory
// (4 B per row), and the max_per_image-th largest found by a most-significant-digit-first radix select (four 8-bit
// digits) instead of a full sort.
constexpr int TOPK_WIDE_MAX_ROWS = 32768;

__global__ void __launch_bounds__(1024) k_topk_keep_wide(const float *__restrict__ rows, int d,
                                                         const int *__restrict__ offsets, int num_classes, int n_cap,
                                                         int max_per_image, unsigned char *__restrict__ keep,
                                                         float *__restrict__ thresh_out) {
  extern __shared__ uint32_t wsm[];
  uint32_t *hist = wsm;              // [256]
  uint32_t *sel = wsm + 256;         // [0] prefix of the selected key, [1] rank still to find inside that prefix
  uint32_t *key = wsm + 260;         // [n]
  const int img = blockIdx.x, tid = threadIdx.x;
  const int n = offsets[(size_t)img * (num_classes + 1) + num_classes];
  const float *r = rows + (size_t)img * n_cap * d;
  unsigned char *kp = keep + (size_t)img * n_cap;
  if (n <= max_per_image) {
    for (int i = tid; i < n; i += blockDim.x) kp[i] = 1;
    if (tid == 0 && thresh_out) thresh_out[img] = -__int_as_float(0x7f800000);
    return;
  }
  for (int i = tid; i < n; i += blockDim.x) {
    uint32_t u = __float_as_uint(r[(size_t)i * d + 4]);
    if ((u & 0x7fffffffu) > 0x7f800000u) u &= 0x7fffffffu;   // NaN: sign bit cleared, above +inf
    key[i] = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  }
  if (tid == 0) { sel[0] = 0u; sel[1] = (uint32_t)max_per_image; }
  uint32_t mask = 0u;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = tid; b < 256; b += blockDim.x) hist[b] = 0u;
    __syncthreads();
    const uint32_t prefix = sel[0];
    for (int i = tid; i < n; i += blockDim.x) {
      const uint32_t k = key[i];
      if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid < 32) {   // lane l holds digits 255 - 8l down to 248 - 8l: the lanes cover the digits from the top
      uint32_t c[8], sum = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) { c[q] = hist[255 - 8 * tid - q]; sum += c[q]; }
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (tid >= o) incl += v;
      }
      uint32_t rank = sel[1];
      const uint32_t before = incl - sum;
      __syncwarp();
      if (before < rank && rank <= incl) {   // exactly one lane: the digit holding the rank-th largest key
        rank -= before;
        int q = 0;
        while (rank > c[q]) { rank -= c[q]; ++q; }
        sel[0] = prefix | ((uint32_t)(255 - 8 * tid - q) << shift);
        sel[1] = rank;
      }
    }
    mask |= 255u << shift;
    __syncthreads();
  }
  const uint32_t tk = sel[0];
  const float thr = __uint_as_float((tk & 0x80000000u) ? (tk & 0x7fffffffu) : ~tk);
  for (int i = tid; i < n; i += blockDim.x) kp[i] = (r[(size_t)i * d + 4] >= thr) ? 1 : 0;
  if (tid == 0 && thresh_out) thresh_out[img] = thr;
}

}  // namespace cnb

using namespace cnb;

extern "C" {

int cnb_post_transform(const float *rows, float *out, const double *trans, int b, int n, int d, int a0, int na, int b0,
                       int nb, void *stream) {
  CNB_REQUIRE(rows && out && trans, CNB_EINVAL, "cnb_post_transform: null pointer");
  CNB_REQUIRE(b > 0 && n > 0 && d > 0 && na >= 0 && nb >= 0 && a0 >= 0 && b0 >= 0 && a0 + 2 * na <= d && b0 + 2 * nb <= d,
              CNB_EINVAL, "cnb_post_transform: bad shape / column ranges");
  const long long total = (long long)b * n * d;
  const int grid = (int)((total + 255) / 256 < 2368 ? (total + 255) / 256 : 2368);
  k_post_transform<<<grid, 256, 0, (cudaStream_t)stream>>>(rows, out, trans, b, n, d, a0, na, b0, nb);
  CNB_CHECK_LAUNCH("cnb_post_transform");
  count_launch();
  return CNB_OK;
}

int cnb_group_by_class(const float *dets, int b, int n, int num_classes, float *rows, int32_t *offsets, void *stream) {
  CNB_REQUIRE(dets && rows && offsets, CNB_EINVAL, "cnb_group_by_class: null pointer");
  CNB_REQUIRE(b > 0 && n > 0 && num_classes > 0 && num_classes <= 8192, CNB_EINVAL, "cnb_group_by_class: bad shape");
  const size_t smem = (size_t)(num_classes + 1 + 256) * 4;
  k_group_by_class<<<b, 256, smem, (cudaStream_t)stream>>>(dets, n, num_classes, rows, offsets);
  CNB_CHECK_LAUNCH("cnb_group_by_class");
  count_launch();
  return CNB_OK;
}

int cnb_soft_nms(const float *rows, float *out, const int32_t *offsets, int n_img, int lists_per_img, int n_cap, int d,
                 float sigma, float nt, float threshold, int method, int32_t *final_n, void *stream) {
  CNB_REQUIRE(rows && out && offsets, CNB_EINVAL, "cnb_soft_nms: null pointer");
  CNB_REQUIRE(n_img > 0 && lists_per_img > 0 && n_cap > 0 && d >= 5 && method >= 0 && method <= 2, CNB_EINVAL,
              "cnb_soft_nms: bad arguments");
  const int n_lists = n_img * lists_per_img;
  CNB_REQUIRE(d == 5 || rows != out, CNB_EINVAL, "cnb_soft_nms: in-place only for 5-column rows");
  CNB_REQUIRE(n_cap <= NMS_MAX_ROWS, CNB_EINVAL, "cnb_soft_nms: at most 4096 rows per image");
  const size_t smem = (size_t)n_cap * NMS_ROW_BYTES + 16;
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev_done != dev) {   // opt in once to the largest launch; each launch asks only for what its n_cap needs
    CNB_CUDA(cudaFuncSetAttribute(k_soft_nms, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(NMS_MAX_ROWS * NMS_ROW_BYTES + 16)));
    dev_done = dev;
  }
  k_soft_nms<<<n_lists, 32, smem, (cudaStream_t)stream>>>(rows, out, offsets, lists_per_img, n_cap, d, sigma, nt, threshold,
                                                            method, final_n);
  CNB_CHECK_LAUNCH("cnb_soft_nms");
  count_launch();
  return CNB_OK;
}

int cnb_topk_keep(const float *rows, int b, int n_cap, int d, const int32_t *offsets, int num_classes,
                  int max_per_image, uint8_t *keep, float *thresh, void *stream) {
  CNB_REQUIRE(rows && offsets && keep, CNB_EINVAL, "cnb_topk_keep: null pointer");
  CNB_REQUIRE(b > 0 && n_cap > 0 && n_cap <= 4096 && d >= 5 && max_per_image > 0, CNB_EINVAL,
              "cnb_topk_keep: bad shape (at most 4096 rows per image)");
  k_topk_keep<<<b, 1024, 4096 * 4, (cudaStream_t)stream>>>(rows, d, offsets, num_classes, n_cap, max_per_image, keep,
                                                            thresh);
  CNB_CHECK_LAUNCH("cnb_topk_keep");
  count_launch();
  return CNB_OK;
}

int cnb_exdet_transform(const float *rows, float *out, const double *trans, int b, int n, int d, float out_width,
                        void *stream) {
  CNB_REQUIRE(rows && out && trans, CNB_EINVAL, "cnb_exdet_transform: null pointer");
  CNB_REQUIRE(rows != out, CNB_EINVAL, "cnb_exdet_transform: out must not alias rows");
  CNB_REQUIRE(b > 0 && n > 0 && d >= 4, CNB_EINVAL, "cnb_exdet_transform: bad shape");
  CNB_REQUIRE(n % 2 == 0, CNB_EINVAL, "cnb_exdet_transform: an image's rows split into two equal halves (n even)");
  const long long total = (long long)b * n * d;
  const int grid = (int)((total + 255) / 256 < 2368 ? (total + 255) / 256 : 2368);
  k_exdet_transform<<<grid, 256, 0, (cudaStream_t)stream>>>(rows, out, trans, b, n, d, out_width);
  CNB_CHECK_LAUNCH("cnb_exdet_transform");
  count_launch();
  return CNB_OK;
}

int cnb_group_positive_by_class(const float *dets, int b, int n, int d, int cls_col, int num_classes, float *rows,
                                int32_t *offsets, void *stream) {
  CNB_REQUIRE(dets && rows && offsets, CNB_EINVAL, "cnb_group_positive_by_class: null pointer");
  CNB_REQUIRE(b > 0 && n > 0 && d >= 5 && cls_col >= 0 && cls_col < d && num_classes > 0 && num_classes <= 8192,
              CNB_EINVAL, "cnb_group_positive_by_class: bad shape");
  const size_t smem = (size_t)(num_classes + 1 + 256) * 4;
  k_group_positive_by_class<<<b, 256, smem, (cudaStream_t)stream>>>(dets, n, d, cls_col, num_classes, rows, offsets);
  CNB_CHECK_LAUNCH("cnb_group_positive_by_class");
  count_launch();
  return CNB_OK;
}

int cnb_soft_nms_strided(const float *rows, float *out, const int32_t *offsets, int n_img, int lists_per_img,
                         int img_stride, int list_cap, int d, float sigma, float nt, float threshold, int method,
                         int32_t *final_n, void *stream) {
  CNB_REQUIRE(rows && out && offsets, CNB_EINVAL, "cnb_soft_nms_strided: null pointer");
  CNB_REQUIRE(n_img > 0 && lists_per_img > 0 && img_stride > 0 && list_cap > 0 && d >= 5 && method >= 0 &&
                  method <= 2 && (long long)n_img * lists_per_img <= 0x7fffffffll,
              CNB_EINVAL, "cnb_soft_nms_strided: bad arguments");
  CNB_REQUIRE(d == 5 || rows != out, CNB_EINVAL, "cnb_soft_nms_strided: in-place only for 5-column rows");
  CNB_REQUIRE(img_stride <= TOPK_WIDE_MAX_ROWS, CNB_EUNSUPPORTED, "cnb_soft_nms_strided: at most 32768 rows per image");
  CNB_REQUIRE(list_cap <= NMS_MAX_ROWS, CNB_EUNSUPPORTED, "cnb_soft_nms_strided: at most 4096 rows per list");
  const size_t smem = (size_t)list_cap * NMS_ROW_BYTES + 16;
  static thread_local int dev_done = -1;
  int dev = 0;
  CNB_CUDA(cudaGetDevice(&dev));
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_soft_nms_strided, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(NMS_MAX_ROWS * NMS_ROW_BYTES + 16)));
    dev_done = dev;
  }
  k_soft_nms_strided<<<n_img * lists_per_img, 32, smem, (cudaStream_t)stream>>>(
      rows, out, offsets, lists_per_img, img_stride, list_cap, d, sigma, nt, threshold, method, final_n);
  CNB_CHECK_LAUNCH("cnb_soft_nms_strided");
  count_launch();
  return CNB_OK;
}

int cnb_topk_keep_wide(const float *rows, int b, int n_cap, int d, const int32_t *offsets, int num_classes,
                       int max_per_image, uint8_t *keep, float *thresh, void *stream) {
  CNB_REQUIRE(rows && offsets && keep, CNB_EINVAL, "cnb_topk_keep_wide: null pointer");
  CNB_REQUIRE(b > 0 && n_cap > 0 && d >= 5 && num_classes > 0 && max_per_image > 0, CNB_EINVAL,
              "cnb_topk_keep_wide: bad shape");
  CNB_REQUIRE(n_cap <= TOPK_WIDE_MAX_ROWS, CNB_EUNSUPPORTED, "cnb_topk_keep_wide: at most 32768 rows per image");
  const size_t smem = (size_t)(260 + n_cap) * 4;
  static thread_local int dev_done = -1;
  int dev = 0;
  CNB_CUDA(cudaGetDevice(&dev));
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_topk_keep_wide, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)((260 + TOPK_WIDE_MAX_ROWS) * 4)));
    dev_done = dev;
  }
  k_topk_keep_wide<<<b, 1024, smem, (cudaStream_t)stream>>>(rows, d, offsets, num_classes, n_cap, max_per_image, keep,
                                                            thresh);
  CNB_CHECK_LAUNCH("cnb_topk_keep_wide");
  count_launch();
  return CNB_OK;
}

int cnb_ddd_tail(const float *dets, int b, int n, int d, const double *trans, const float *calib, int num_classes,
                 int cut, float thresh, float *rows, int32_t *offsets, uint8_t *seen, void *stream) {
  CNB_REQUIRE(dets && trans && calib && rows && offsets, CNB_EINVAL, "cnb_ddd_tail: null pointer");
  CNB_REQUIRE(d == 18, CNB_EINVAL,
              "cnb_ddd_tail: rows must have the 18 columns of ddd_decode with wh (x, y, score, rot[8], depth, dim[3], "
              "w, h, class)");
  CNB_REQUIRE(b > 0 && n > 0 && num_classes > 0 && num_classes <= 8192, CNB_EINVAL, "cnb_ddd_tail: bad shape");
  // every output range disjoint from every other buffer
  const char *in_p[3] = {(const char *)dets, (const char *)trans, (const char *)calib};
  const size_t in_n[3] = {(size_t)b * n * 18 * 4, (size_t)b * 6 * 8, (size_t)b * 12 * 4};
  const char *out_p[3] = {(const char *)rows, (const char *)offsets, (const char *)seen};
  const size_t out_n[3] = {(size_t)b * n * 13 * 4, (size_t)b * (num_classes + 1) * 4, (size_t)b * num_classes};
  auto overlap = [](const char *p, size_t pn, const char *q, size_t qn) { return p && q && p < q + qn && q < p + pn; };
  for (int o = 0; o < 3; ++o) {
    for (int i = 0; i < 3; ++i)
      CNB_REQUIRE(!overlap(out_p[o], out_n[o], in_p[i], in_n[i]), CNB_EINVAL, "cnb_ddd_tail: an output aliases an input");
    for (int k = o + 1; k < 3; ++k)
      CNB_REQUIRE(!overlap(out_p[o], out_n[o], out_p[k], out_n[k]), CNB_EINVAL, "cnb_ddd_tail: outputs alias each other");
  }
  const size_t smem = (size_t)(num_classes + 1 + 256) * 4;
  k_ddd_tail<<<b, 256, smem, (cudaStream_t)stream>>>(dets, n, trans, calib, num_classes, cut ? 1 : 0, thresh, rows,
                                                     offsets, seen);
  CNB_CHECK_LAUNCH("cnb_ddd_tail");
  count_launch();
  return CNB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ N4: detector input pre-processing
// detectors/base_detector.py:37-65: cv2.warpAffine(INTER_LINEAR, BORDER_CONSTANT 0) of the uint8 HWC image,
// (x / 255 - mean) / std in float64, HWC -> CHW fp32, optional mirrored copy (flip test) -- one pass, the image
// crosses PCIe as uint8 (3 B / pixel instead of 12-24).  The warp is OpenCV's fixed-point algorithm (warp.cuh).
// kF32: DddDetector.pre_process's normalisation (detectors/ddd.py:50-51), x.astype(float32) / 255. then
// (x - mean) / std all in float32, instead of base_detector's float64 -- the warp is the same.
namespace cnb {
template <bool kF32>
__device__ __forceinline__ void preprocess_px(const unsigned char *__restrict__ img, int H, int W,
                                              const double *__restrict__ minv, const float *__restrict__ mean,
                                              const float *__restrict__ stdv, float *__restrict__ out, int oh, int ow,
                                              int flip) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= ow) return;
  const WarpTaps t = warp_taps(minv, x, y, H, W);
  const int sx = t.sx, sy = t.sy, w0 = t.w0, w1 = t.w1, w2 = t.w2, w3 = t.w3;
  const bool y0ok = t.y0ok, y1ok = t.y1ok, x0ok = t.x0ok, x1ok = t.x1ok;
  const size_t plane = (size_t)oh * ow;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int p00 = (y0ok && x0ok) ? img[((size_t)sy * W + sx) * 3 + c] : 0;
    const int p01 = (y0ok && x1ok) ? img[((size_t)sy * W + sx + 1) * 3 + c] : 0;
    const int p10 = (y1ok && x0ok) ? img[((size_t)(sy + 1) * W + sx) * 3 + c] : 0;
    const int p11 = (y1ok && x1ok) ? img[((size_t)(sy + 1) * W + sx + 1) * 3 + c] : 0;
    int v = (p00 * w0 + p01 * w1 + p10 * w2 + p11 * w3 + (1 << 14)) >> 15;
    v = min(max(v, 0), 255);
    float f;
    if (kF32) {
      f = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), mean[c]), stdv[c]);
    } else {
      const double r = __ddiv_rn(__dadd_rn(__ddiv_rn((double)v, 255.0), -(double)mean[c]), (double)stdv[c]);
      f = (float)r;
    }
    out[c * plane + (size_t)y * ow + x] = f;
    if (flip) out[(3 + c) * plane + (size_t)y * ow + (ow - 1 - x)] = f;
  }
}

__global__ void __launch_bounds__(256) k_preprocess(const unsigned char *__restrict__ img, int H, int W,
                                                    const double *__restrict__ minv, const float *__restrict__ mean,
                                                    const float *__restrict__ stdv, float *__restrict__ out, int oh,
                                                    int ow, int flip) {
  preprocess_px<false>(img, H, W, minv, mean, stdv, out, oh, ow, flip);
}

__global__ void __launch_bounds__(256) k_preprocess_f32(const unsigned char *__restrict__ img, int H, int W,
                                                        const double *__restrict__ minv, const float *__restrict__ mean,
                                                        const float *__restrict__ stdv, float *__restrict__ out, int oh,
                                                        int ow, int flip) {
  preprocess_px<true>(img, H, W, minv, mean, stdv, out, oh, ow, flip);
}
}  // namespace cnb

// cv2.resize(INTER_LINEAR) of a uint8 HWC image (base_detector.py:55 at test scales != 1): OpenCV's 11-bit
// separable fixed point (resize.cpp) -- horizontal pass S = p0 * a0 + p1 * a1 with the source index clamped and
// the phase zeroed at the borders, vertical pass ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2 >> 2 with
// only the row indices clamped; coefficients = cvRound(float phase * 2048).
namespace cnb {
__global__ void __launch_bounds__(256) k_resize_u8(const unsigned char *__restrict__ src, int H, int W,
                                                   unsigned char *__restrict__ dst, int dh, int dw) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  const double sc_x = (double)W / (double)dw, sc_y = (double)H / (double)dh;
  float fx = (float)__dadd_rn(__dmul_rn(__dadd_rn((double)x, 0.5), sc_x), -0.5);
  int sx = (int)floorf(fx);
  fx -= (float)sx;
  if (sx < 0) { fx = 0.f; sx = 0; }
  if (sx >= W - 1) { fx = 0.f; sx = W - 1; }
  const int a0 = __float2int_rn(__fmul_rn(1.0f - fx, 2048.0f)), a1 = __float2int_rn(__fmul_rn(fx, 2048.0f));
  const int sx1 = min(sx + 1, W - 1);
  float fy = (float)__dadd_rn(__dmul_rn(__dadd_rn((double)y, 0.5), sc_y), -0.5);
  const int sy = (int)floorf(fy);
  fy -= (float)sy;
  const int b0 = __float2int_rn(__fmul_rn(1.0f - fy, 2048.0f)), b1 = __float2int_rn(__fmul_rn(fy, 2048.0f));
  const int r0 = min(max(sy, 0), H - 1), r1 = min(max(sy + 1, 0), H - 1);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s0 = src[((size_t)r0 * W + sx) * 3 + c] * a0 + src[((size_t)r0 * W + sx1) * 3 + c] * a1;
    const int s1 = src[((size_t)r1 * W + sx) * 3 + c] * a0 + src[((size_t)r1 * W + sx1) * 3 + c] * a1;
    int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
    dst[((size_t)y * dw + x) * 3 + c] = (unsigned char)min(max(v, 0), 255);
  }
}
}  // namespace cnb

extern "C" int cnb_resize_image(const uint8_t *image_hwc, int h, int w, uint8_t *out_hwc, int out_h, int out_w,
                                void *stream) {
  CNB_REQUIRE(image_hwc && out_hwc, CNB_EINVAL, "cnb_resize_image: null pointer");
  CNB_REQUIRE(h > 0 && w > 0 && out_h > 0 && out_w > 0 && h < 32768 && w < 32768, CNB_EINVAL, "cnb_resize_image: bad shape");
  dim3 grid((unsigned)((out_w + 255) / 256), (unsigned)out_h);
  cnb::k_resize_u8<<<grid, 256, 0, (cudaStream_t)stream>>>(image_hwc, h, w, out_hwc, out_h, out_w);
  CNB_CHECK_LAUNCH("cnb_resize_image");
  cnb::count_launch();
  return CNB_OK;
}

extern "C" int cnb_preprocess_image(const uint8_t *image_hwc, int h, int w, const double *minv6, const float *mean3,
                                    const float *std3, float *out, int out_h, int out_w, int flip_test, void *stream) {
  CNB_REQUIRE(image_hwc && minv6 && mean3 && std3 && out, CNB_EINVAL, "cnb_preprocess_image: null pointer");
  CNB_REQUIRE(h > 0 && w > 0 && out_h > 0 && out_w > 0 && h < 32768 && w < 32768, CNB_EINVAL,
              "cnb_preprocess_image: bad shape");
  dim3 grid((unsigned)((out_w + 255) / 256), (unsigned)out_h);
  cnb::k_preprocess<<<grid, 256, 0, (cudaStream_t)stream>>>(image_hwc, h, w, minv6, mean3, std3, out, out_h, out_w,
                                                            flip_test ? 1 : 0);
  CNB_CHECK_LAUNCH("cnb_preprocess_image");
  cnb::count_launch();
  return CNB_OK;
}

extern "C" int cnb_preprocess_image_f32(const uint8_t *image_hwc, int h, int w, const double *minv6, const float *mean3,
                                        const float *std3, float *out, int out_h, int out_w, int flip_test,
                                        void *stream) {
  CNB_REQUIRE(image_hwc && minv6 && mean3 && std3 && out, CNB_EINVAL, "cnb_preprocess_image_f32: null pointer");
  CNB_REQUIRE(h > 0 && w > 0 && out_h > 0 && out_w > 0 && h < 32768 && w < 32768, CNB_EINVAL,
              "cnb_preprocess_image_f32: bad shape");
  dim3 grid((unsigned)((out_w + 255) / 256), (unsigned)out_h);
  cnb::k_preprocess_f32<<<grid, 256, 0, (cudaStream_t)stream>>>(image_hwc, h, w, minv6, mean3, std3, out, out_h, out_w,
                                                                flip_test ? 1 : 0);
  CNB_CHECK_LAUNCH("cnb_preprocess_image_f32");
  cnb::count_launch();
  return CNB_OK;
}

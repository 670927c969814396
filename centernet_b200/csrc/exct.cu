// exct_decode / agnex_ct_decode (models/decode.py:273-424, :122-271) -- ExtremeNet grouping.
//
//   1. optional edge aggregation of the t,l,b,r maps (:287-291, aggregate.cu)
//   2. fused NMS + clamp-to-1 + top-K on each of the four maps (:294-307, select.cu)
//   3. k_exct_tuples: every (t_i, l_j, b_k, r_m) tuple is scored in registers
//        score = (ts+ls+bs+rs+2*ct)/6 - [score/centre thresholds] - [class mismatch]
//                - [top] - [left] - [bottom] - [right geometry]            (:333-360)
//      and streamed through an exact top-`num_dets` selection (64-bit keys: order-preserving
//      score bits | ~tuple index, candidate buffer + bitonic prune) -- the reference
//      materialises ~30 [B, K^4] tensors instead (10 MB each at K=40, 400 MB at K=100);
//   4. k_exct_merge: merges the per-group segments of an image, adds the regression offsets
//      (or 0.5) and writes the 14-column rows (:366-421).
// Tie order: score desc, tuple index ((i*K+j)*K+k)*K+m asc (torch.topk leaves it open).
//
// cnb_exct_decode_ex reads the nine inputs as fp32, fp16 or bf16, the five maps optionally as logits, and returns
// what the fp32 call returns for the .float() upcast (after torch's CUDA sigmoid, with logits).  Only the steps that
// read an input change: the selections (plan_map_select: in place in the hot geometry, else one widening / sigmoid
// pass), the edge aggregation (score_f32 on load), the centre map (k_ct_agnostic / k_ct_scores write its fp32
// scores) and the regression gathers of k_exct_merge<true>.  k_exct_tuples and the fp32 instances are unchanged.
#include "select.cuh"

namespace cnb {

typedef unsigned long long u64;
int launch_edge_aggregate_ex(const void *heat, int dt, bool sigmoid, float *out, int n, int c, int h, int w,
                             float weight, int horizontal, cudaStream_t stream);

constexpr int EX_THREADS = 512;
constexpr int EX_CAP = 4096;       // candidate keys per CTA
constexpr int EX_STEP = 2048;      // tuples scored between two capacity checks
constexpr int EX_MAX_DETS = 2048;  // num_dets limit (CAP - STEP)
constexpr int EX_MAX_GROUPS = 16;  // segments per image
constexpr int EX_MERGE_KEYS = 16384;  // the merge sorts np2(groups * num_dets) keys in shared memory: 128 KiB at most

struct RawList {
  float *scores; int64_t *inds; int32_t *clses; float *ys; float *xs;
};

struct ExctArgs {
  RawList t, l, b, r;
  const float *ct_heat;     // [B, CC, H, W]   (non-agnostic: CC == C)
  const float *ct_agn;      // [B, H*W] max over classes (agnostic)
  const int32_t *ct_cls;    // [B, H*W] argmax over classes (agnostic)
  const float *t_regr, *l_regr, *b_regr, *r_regr;
  int B, CC, H, W, K, num_dets, groups, agnostic;
  float scores_thresh, center_thresh;
  const uint32_t *ct_max;   // [B] order-preserving bits of the largest centre-map value of the image (pruning bound)
  u64 *gthr;                // [B] best num_dets-th key any group of the image has reached (shared pruning threshold)
  u64 *seg;                 // [B, groups, num_dets]
  int *seg_cnt;             // [B, groups]
  float *dets;              // [B, num_dets, 14]
};

__device__ __forceinline__ uint32_t mono_bits(float v) {  // order-preserving map of any float
  const uint32_t b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float mono_inv(uint32_t m) {
  return __uint_as_float((m & 0x80000000u) ? (m & 0x7fffffffu) : ~m);
}
// mono_bits for the centre-map bound of the pruning test: a NaN of either sign is the top value, because a tuple
// that reads it scores the device's positive NaN, whose key lies above +inf (mono_bits puts a sign-bit NaN below
// every number)
__device__ __forceinline__ uint32_t bound_bits(float v) { return v != v ? 0xffffffffu : mono_bits(v); }

__device__ __forceinline__ void sort_desc(u64 *buf, int n) {
  for (int k = 2; k <= n; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const u64 a = buf[i], b = buf[i + j];
        if ((a < b) == ((i & k) == 0)) { buf[i] = b; buf[i + j] = a; }
      }
      __syncthreads();
    }
}
__device__ __forceinline__ int np2(int v) { int n = 2; while (n < v) n <<= 1; return n; }

// max / argmax over classes of the centre map (decode.py:159), compared as fp32 scores: with SIG the sigmoids,
// not the logits, so classes whose sigmoids tie (e.g. both saturate to 1) yield the first one, as torch.max does.
// As torch.max, a NaN wins over every number and the first NaN class is taken.
template <typename T, bool SIG>
__global__ void __launch_bounds__(256) k_ct_agnostic(const T *__restrict__ ct, int B, int CC, long long HW,
                                                     float *__restrict__ agn, int32_t *__restrict__ cls) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * HW) return;
  const long long b = i / HW, sp = i - b * HW;
  const T *p = ct + b * CC * HW + sp;
  float best = score_f32<SIG>(p[0]);
  int arg = 0, nan_arg = best != best ? 0 : CC;
  for (int c = 1; c < CC; ++c) {
    const float v = score_f32<SIG>(p[(long long)c * HW]);
    if (v > best) { best = v; arg = c; }
    if (v != v) nan_arg = min(nan_arg, c);   // a chain of its own: the max above does not wait for it
  }
  if (nan_arg < CC) { arg = nan_arg; best = score_f32<SIG>(p[(long long)nan_arg * HW]); }
  agn[i] = best;
  cls[i] = arg;
}

// out[b] = max over the image's centre map, as bound_bits (out zero-filled: below every float)
__global__ void __launch_bounds__(256) k_ct_max(const float *__restrict__ ct, long long per_image, uint32_t *__restrict__ out) {
  __shared__ uint32_t red[8];
  const float *p = ct + (long long)blockIdx.y * per_image;
  uint32_t best = 0u;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < per_image; i += (long long)gridDim.x * blockDim.x)
    best = max(best, bound_bits(__ldg(p + i)));
  for (int k = 16; k > 0; k >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, k));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) best = max(best, red[i]);
    atomicMax(out + blockIdx.y, best);
  }
}

// k_ct_max for a centre map that is not an fp32 heat map: also writes its fp32 scores (widened, or the sigmoid of
// the widened logit) to sc, the map k_exct_tuples then reads
template <typename T, bool SIG>
__global__ void __launch_bounds__(256) k_ct_scores(const T *__restrict__ ct, long long per_image, float *__restrict__ sc,
                                                   uint32_t *__restrict__ out) {
  __shared__ uint32_t red[8];
  const long long base = (long long)blockIdx.y * per_image;
  uint32_t best = 0u;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < per_image; i += (long long)gridDim.x * blockDim.x) {
    const float v = score_f32<SIG>(__ldg(ct + base + i));
    sc[base + i] = v;
    best = max(best, bound_bits(v));
  }
  for (int k = 16; k > 0; k >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, k));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) best = max(best, red[i]);
    atomicMax(out + blockIdx.y, best);
  }
}

__global__ void __launch_bounds__(EX_THREADS, 1) k_exct_tuples(const ExctArgs a) {
  extern __shared__ __align__(16) unsigned char ex_smem[];
  u64 *buf = reinterpret_cast<u64 *>(ex_smem);                     // [EX_CAP]
  float *ls = reinterpret_cast<float *>(buf + EX_CAP);             // 4 lists x (score, y, x, cls) x K
  __shared__ int s_cnt;
  __shared__ u64 s_g;
  const int K = a.K, b = blockIdx.x / a.groups, grp = blockIdx.x - b * a.groups;
  const int tid = threadIdx.x;
  float *S[4], *Y[4], *X[4];
  int *CL[4];
  for (int q = 0; q < 4; ++q) {
    S[q] = ls + (q * 4 + 0) * K; Y[q] = ls + (q * 4 + 1) * K; X[q] = ls + (q * 4 + 2) * K;
    CL[q] = reinterpret_cast<int *>(ls + (q * 4 + 3) * K);
  }
  const RawList *L[4] = {&a.t, &a.l, &a.b, &a.r};
  for (int idx = tid; idx < 4 * K; idx += blockDim.x) {
    const int q = idx / K, i = idx - q * K;
    const size_t o = (size_t)b * K + i;
    S[q][i] = L[q]->scores[o]; Y[q][i] = L[q]->ys[o]; X[q][i] = L[q]->xs[o]; CL[q][i] = L[q]->clses[o];
  }
  if (tid == 0) s_cnt = 0;
  __syncthreads();

  const long long HW = (long long)a.H * a.W;
  const int K2 = K * K;
  const long long K3 = (long long)K2 * K;
  const int nd = a.num_dets;
  // upper bounds for the pruning test: the best bottom / right scores and the largest centre value of the image
  float bmax = S[2][0], rmax = S[3][0];
  for (int q = 1; q < K; ++q) { bmax = fmaxf(bmax, S[2][q]); rmax = fmaxf(rmax, S[3][q]); }
  const float ctmax = mono_inv(a.ct_max[b]);
  u64 thr = 0ull;
  // the groups of an image take the top candidates round-robin (every group gets the same mix of strong and weak ones)
  // and share their thresholds through gthr, so they finish together; the merge orders the keys, not the groups
  for (int i = grp; i < K; i += a.groups) {
    const float ts = S[0][i], ty = Y[0][i], tx = X[0][i];
    const int ci = CL[0][i];
    for (int j = 0; j < K; ++j) {
      const float lsx = S[1][j], ly = Y[1][j], lx = X[1][j];
      // Exact pruning of the whole (i, j, *, *) block: every penalty already decided by (i, j) costs 1.0, the score
      // before penalties is at most the same expression over the best bottom / right / centre values, and every step
      // of the computation is monotone in fp32 -- so if even that bound cannot beat the current num_dets-th key the
      // K^2 tuples need not be scored (CTA-uniform: no barrier is skipped by only some threads).
      {
        int lb = 0;
        lb += ((ts < a.scores_thresh) || (lsx < a.scores_thresh)) ? 1 : 0;
        lb += (!a.agnostic && ci != CL[1][j]) ? 1 : 0;
        lb += (ty > ly) ? 1 : 0;
        lb += (lx > tx) ? 1 : 0;
        float ub = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(ts, lsx), bmax), rmax), __fmul_rn(2.0f, ctmax));
        ub = __fdiv_rn(ub, 6.0f);
        for (int q = 0; q < lb; ++q) ub = __fsub_rn(ub, 1.0f);
        ub = __fadd_rn(ub, 0.0f);      // -0 -> +0: the key order puts -0 below +0
        // The list scores are never NaN and at most 1 (the clamp), so besides a NaN centre value (which bound_bits
        // makes the bound) only 2*ct = +inf meeting a -inf sum of the four scores makes a tuple NaN, ranked first:
        // such a block is not pruned.  The block's smallest sum takes the last (lowest) bottom and right scores of
        // the descending lists, fp32 addition being monotone; tested only for a block about to be pruned.
        if (mono_bits(ub) < (uint32_t)(thr >> 32)) {
          if (__fmul_rn(2.0f, ctmax) < INFINITY) continue;
          if (__fadd_rn(__fadd_rn(__fadd_rn(ts, lsx), S[2][K - 1]), S[3][K - 1]) != -INFINITY) continue;
        }
      }
      for (int base = 0; base < K2; base += EX_STEP) {
        // the num_dets-th key of ANY group of the image bounds the result from below: adopt the best one published
        if (tid == 0) s_g = *reinterpret_cast<volatile u64 *>(a.gthr + b);
        __syncthreads();
        const int cnt = s_cnt;           // every push of the previous step is in
        const u64 gth = s_g;
        __syncthreads();                 // nobody pushes before everyone has read: the branches are uniform
        if (gth > thr) thr = gth;
        if (cnt + EX_STEP > EX_CAP) {    // sort, keep the num_dets best, raise the threshold
          const int n = np2(cnt);
          for (int t = cnt + tid; t < n; t += blockDim.x) buf[t] = 0ull;
          __syncthreads();
          sort_desc(buf, n);
          if (cnt >= nd && buf[nd - 1] > thr) thr = buf[nd - 1];
          __syncthreads();
          if (tid == 0) {
            if (cnt > nd) s_cnt = nd;
            if (cnt >= nd) atomicMax(a.gthr + b, thr);
          }
          __syncthreads();
        }
        for (int e = base + tid; e < min(base + EX_STEP, K2); e += blockDim.x) {
          const int k = e / K, m = e - k * K;
          const float bs = S[2][k], rs = S[3][m];
          const float by = Y[2][k], bx = X[2][k], ry = Y[3][m], rx = X[3][m];
          const int cx = ((int)lx + (int)rx) >> 1;   // ((l_x + r_x + 0.5) / 2).long(), decode.py:322
          const int cy = ((int)ty + (int)by) >> 1;   // :323
          float ct;
          if (a.agnostic) ct = __ldg(a.ct_agn + (long long)b * HW + cy * a.W + cx);
          else ct = __ldg(a.ct_heat + ((long long)b * a.CC + ci) * HW + cy * a.W + cx);
          float sc = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(ts, lsx), bs), rs), __fmul_rn(2.0f, ct));
          sc = __fdiv_rn(sc, 6.0f);                                                            // :333
          const bool sc_bad = (ts < a.scores_thresh) || (lsx < a.scores_thresh) || (bs < a.scores_thresh) ||
                              (rs < a.scores_thresh) || (ct < a.center_thresh);                // :350-355
          const bool top_bad = (ty > ly) || (ty > by) || (ty > ry);                            // :341-348
          const bool left_bad = (lx > tx) || (lx > bx) || (lx > rx);
          const bool bot_bad = (by < ty) || (by < ly) || (by < ry);
          const bool right_bad = (rx < tx) || (rx < lx) || (rx < bx);
          sc = __fsub_rn(sc, sc_bad ? 1.0f : 0.0f);                                            // :355-360 order
          if (!a.agnostic) {
            const bool cls_bad = (ci != CL[1][j]) || (ci != CL[2][k]) || (ci != CL[3][m]);
            sc = __fsub_rn(sc, cls_bad ? 1.0f : 0.0f);
          }
          sc = __fsub_rn(sc, top_bad ? 1.0f : 0.0f);
          sc = __fsub_rn(sc, left_bad ? 1.0f : 0.0f);
          sc = __fsub_rn(sc, bot_bad ? 1.0f : 0.0f);
          // sc - 1 as sc + (-1), the same rounding; sc + 0 folds -0 to +0: one value, ordered by tuple index (a
          // negative subnormal sum / 6 rounds to -0)
          sc = __fadd_rn(sc, right_bad ? -1.0f : 0.0f);
          const uint32_t tuple = (uint32_t)((long long)i * K3 + (long long)j * K2 + e);
          const u64 key = ((u64)mono_bits(sc) << 32) | (u64)(0xffffffffu - tuple);
          if (key > thr) buf[atomicAdd(&s_cnt, 1)] = key;
        }
      }
    }
  }
  // final cut of this group's segment
  __syncthreads();
  const int cnt = s_cnt;
  const int n = np2(cnt);
  for (int t = cnt + tid; t < n; t += blockDim.x) buf[t] = 0ull;
  __syncthreads();
  sort_desc(buf, n);
  const int n_out = min(cnt, nd);
  u64 *dst = a.seg + ((size_t)b * a.groups + grp) * nd;
  for (int t = tid; t < n_out; t += blockDim.x) dst[t] = buf[t];
  if (tid == 0) a.seg_cnt[(size_t)b * a.groups + grp] = n_out;
}

// EX: the regression maps are read by their CNB_DTYPE_* codes rdt (t, l, b, r in x, y, z, w), widened exactly; the
// regression pointers of `a` are then untyped
template <bool EX>
__global__ void __launch_bounds__(1024, 1) k_exct_merge(const ExctArgs a, const int4 rdt) {
  extern __shared__ __align__(16) unsigned char ex_smem[];
  u64 *sbuf = reinterpret_cast<u64 *>(ex_smem);
  const int b = blockIdx.x, tid = threadIdx.x, K = a.K, nd = a.num_dets;
  int total = 0;
  for (int g = 0; g < a.groups; ++g) {
    const int n = a.seg_cnt[(size_t)b * a.groups + g];
    const u64 *seg = a.seg + ((size_t)b * a.groups + g) * nd;
    for (int t = tid; t < n; t += blockDim.x) sbuf[total + t] = seg[t];
    total += n;
  }
  const int n = np2(total);
  for (int t = total + tid; t < n; t += blockDim.x) sbuf[t] = 0ull;
  __syncthreads();
  if (a.groups > 1) sort_desc(sbuf, n);
  const long long HW = (long long)a.H * a.W;
  const bool has_reg = a.t_regr && a.l_regr && a.b_regr && a.r_regr;   // decode.py:366-367
  for (int r = tid; r < nd; r += blockDim.x) {
    const u64 key = sbuf[r];
    const float score = mono_inv((uint32_t)(key >> 32));
    const uint32_t tuple = 0xffffffffu - (uint32_t)key;
    const int m = tuple % K, k = (tuple / K) % K, j = (tuple / (K * K)) % K, i = tuple / (K * K * K);
    const size_t oi = (size_t)b * K + i, oj = (size_t)b * K + j, ok = (size_t)b * K + k, om = (size_t)b * K + m;
    float tx = a.t.xs[oi], ty = a.t.ys[oi], lx = a.l.xs[oj], ly = a.l.ys[oj];
    float bx = a.b.xs[ok], by = a.b.ys[ok], rx = a.r.xs[om], ry = a.r.ys[om];
    float cls;
    if (a.agnostic) {
      const int cx = ((int)lx + (int)rx) >> 1, cy = ((int)ty + (int)by) >> 1;
      cls = (float)a.ct_cls[(long long)b * HW + cy * a.W + cx];
    } else {
      cls = (float)a.t.clses[oi];
    }
    if (EX && has_reg) {
      const long long st = a.t.inds[oi], sl = a.l.inds[oj], sb = a.b.inds[ok], sr = a.r.inds[om];
      const long long x0 = (long long)b * 2 * HW, y0 = ((long long)b * 2 + 1) * HW;
      tx += ld_head(a.t_regr, rdt.x, x0 + st); ty += ld_head(a.t_regr, rdt.x, y0 + st);
      lx += ld_head(a.l_regr, rdt.y, x0 + sl); ly += ld_head(a.l_regr, rdt.y, y0 + sl);
      bx += ld_head(a.b_regr, rdt.z, x0 + sb); by += ld_head(a.b_regr, rdt.z, y0 + sb);
      rx += ld_head(a.r_regr, rdt.w, x0 + sr); ry += ld_head(a.r_regr, rdt.w, y0 + sr);
    } else if (has_reg) {  // :366-384
      const long long st = a.t.inds[oi], sl = a.l.inds[oj], sb = a.b.inds[ok], sr = a.r.inds[om];
      tx += a.t_regr[((long long)b * 2) * HW + st]; ty += a.t_regr[((long long)b * 2 + 1) * HW + st];
      lx += a.l_regr[((long long)b * 2) * HW + sl]; ly += a.l_regr[((long long)b * 2 + 1) * HW + sl];
      bx += a.b_regr[((long long)b * 2) * HW + sb]; by += a.b_regr[((long long)b * 2 + 1) * HW + sb];
      rx += a.r_regr[((long long)b * 2) * HW + sr]; ry += a.r_regr[((long long)b * 2 + 1) * HW + sr];
    } else {        // :385-393
      tx += 0.5f; ty += 0.5f; lx += 0.5f; ly += 0.5f; bx += 0.5f; by += 0.5f; rx += 0.5f; ry += 0.5f;
    }
    float *d = a.dets + ((size_t)b * nd + r) * 14;   // :395-421
    d[0] = lx; d[1] = ty; d[2] = rx; d[3] = by; d[4] = score;
    d[5] = tx; d[6] = ty; d[7] = lx; d[8] = ly; d[9] = bx; d[10] = by; d[11] = rx; d[12] = ry; d[13] = cls;
  }
}

static size_t raw_sz(long long n) { return align_up((size_t)n * 8, 256) + 4 * align_up((size_t)n * 4, 256); }
static RawList carve(char *&p, long long n) {
  RawList r;
  r.inds = reinterpret_cast<int64_t *>(p); p += align_up((size_t)n * 8, 256);
  r.scores = reinterpret_cast<float *>(p); p += align_up((size_t)n * 4, 256);
  r.clses = reinterpret_cast<int32_t *>(p); p += align_up((size_t)n * 4, 256);
  r.ys = reinterpret_cast<float *>(p); p += align_up((size_t)n * 4, 256);
  r.xs = reinterpret_cast<float *>(p); p += align_up((size_t)n * 4, 256);
  return r;
}
// CTAs per image of k_exct_tuples: two CTAs per SM over the batch, at most 16, one per top index, and no more
// segments than the merge can sort (at the default num_dets = 1000, 16)
static int exct_groups(int b, int k, int num_dets) {
  if (b < 1 || k < 1 || num_dets < 1) return 1;   // sizes a workspace query on arguments the call then rejects
  int g = (2 * num_sms() + b - 1) / b;
  if (g > EX_MAX_GROUPS) g = EX_MAX_GROUPS;
  if (g > k) g = k;
  if (g > EX_MERGE_KEYS / num_dets) g = EX_MERGE_KEYS / num_dets;
  return g < 1 ? 1 : g;
}

// The nine inputs of an exct decode with their CNB_DTYPE_* codes.  `logits`: the five maps hold pre-sigmoid logits.
struct ExctIn {
  const void *map[4];   // t, l, b, r
  const void *ct;
  const void *regr[4];  // all four or none
  int map_dt[4], ct_dt, regr_dt[4];
  int logits;
};

// every map and regression head fp32, no logits: the fp32 call, its plan, workspace and launches
static bool exct_plain(const ExctIn &x) {
  bool f32 = x.ct_dt == CNB_DTYPE_F32 && !x.logits;
  for (int q = 0; q < 4; ++q) f32 = f32 && x.map_dt[q] == CNB_DTYPE_F32 && x.regr_dt[q] == CNB_DTYPE_F32;
  return f32;
}

// everything after the selection scratch: raw lists, aggregated maps, agnostic centre map, segments, bounds
static size_t exct_tail_bytes(int b, int c, int h, int w, int k, int num_dets) {
  const int g = exct_groups(b, k, num_dets);
  const size_t maps = 4 * align_up((size_t)b * c * h * w * 4, 256);       // aggregated maps (aggr_weight > 0)
  const size_t agn = 2 * align_up((size_t)b * h * w * 4, 256);            // class-agnostic centre map
  return 4 * raw_sz((long long)b * k) + maps + agn + align_up((size_t)b * g * num_dets * 8, 256) +
         align_up((size_t)b * g * 4, 256) + align_up((size_t)b * 4, 256) + align_up((size_t)b * 8, 256);
}

// Argument checks shared by the calls and the dtype-generic query (no CUDA call)
static int exct_check(const char *fn, const ExctIn &x, int b, int c, int cc, int h, int w, int k, int num_dets,
                      int agnostic) {
  bool known = dtype_known(x.ct_dt);
  for (int q = 0; q < 4; ++q) known = known && dtype_known(x.map_dt[q]) && dtype_known(x.regr_dt[q]);
  CNB_REQUIRE(known, CNB_EINVAL, "%s: unknown dtype code (t %d, l %d, b %d, r %d, ct %d, regr %d %d %d %d)", fn,
              x.map_dt[0], x.map_dt[1], x.map_dt[2], x.map_dt[3], x.ct_dt, x.regr_dt[0], x.regr_dt[1], x.regr_dt[2],
              x.regr_dt[3]);
  CNB_REQUIRE(x.map[0] && x.map[1] && x.map[2] && x.map[3] && x.ct, CNB_EINVAL, "%s: null pointer", fn);
  CNB_REQUIRE(b > 0 && c > 0 && cc > 0 && h > 0 && w > 0 && k > 0 && num_dets > 0, CNB_EINVAL,
              "%s: non-positive dimension", fn);
  CNB_REQUIRE(agnostic || cc == c, CNB_EINVAL, "%s: centre map has %d classes, extreme maps %d", fn, cc, c);
  CNB_REQUIRE(k <= 255, CNB_EUNSUPPORTED, "%s: k=%d (k^4 must fit 32 bits)", fn, k);
  const long long k4 = (long long)k * k * k * k;
  CNB_REQUIRE(num_dets <= k4, CNB_EINVAL, "%s: num_dets=%d exceeds k^4=%lld (torch.topk would raise)", fn, num_dets,
              k4);
  CNB_REQUIRE(num_dets <= EX_MAX_DETS, CNB_EUNSUPPORTED, "%s: num_dets=%d > %d", fn, num_dets, EX_MAX_DETS);
  return CNB_OK;
}

// Plans of the four selections of a non-plain decode and the largest scratch they need.  Each selection reads its
// map (in place, or through the fp32 copy at `copy`), or with aggregation the fp32 aggregated map agg[q].  The query
// passes null agg / copy: 16-byte aligned places.
static int exct_plans(const ExctIn &x, bool aggr, float *const agg[4], const float *copy, int b, int c, int h, int w,
                      int k, MapSelect m[4], size_t *sel) {
  *sel = 0;
  for (int q = 0; q < 4; ++q) {
    const int rc = aggr ? plan_map_select(agg[q], CNB_DTYPE_F32, 0, b, c, h, w, k, copy, &m[q])
                        : plan_map_select(x.map[q], x.map_dt[q], x.logits, b, c, h, w, k, copy, &m[q]);
    if (rc != CNB_OK) return rc;
    m[q].pl.clamp_one = 1;   // decode.py:299-302: values above 1 are clamped before _topk
    if (m[q].sel_bytes > *sel) *sel = m[q].sel_bytes;
  }
  return CNB_OK;
}

template <typename T>
static void launch_ct_agnostic(const void *ct, bool sig, int b, int cc, long long hw, float *agn, int32_t *cls,
                               cudaStream_t stream) {
  const long long n = (long long)b * hw;
  const T *p = reinterpret_cast<const T *>(ct);
  if (sig) k_ct_agnostic<T, true><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p, b, cc, hw, agn, cls);
  else k_ct_agnostic<T, false><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p, b, cc, hw, agn, cls);
}

template <typename T>
static void launch_ct_scores(const void *ct, bool sig, dim3 grid, long long per, float *sc, uint32_t *mx,
                             cudaStream_t stream) {
  const T *p = reinterpret_cast<const T *>(ct);
  if (sig) k_ct_scores<T, true><<<grid, 256, 0, stream>>>(p, per, sc, mx);
  else k_ct_scores<T, false><<<grid, 256, 0, stream>>>(p, per, sc, mx);
}

// The host body of cnb_exct_decode (exct_plain(x): its fp32 plan, workspace and launches) and cnb_exct_decode_ex
static int exct_decode(const char *fn, const ExctIn &x, int b, int c, int cc, int h, int w, int k, float scores_thresh,
                       float center_thresh, float aggr_weight, int num_dets, int agnostic, float *dets, void *workspace,
                       size_t workspace_bytes, cudaStream_t stream) {
  int rc = exct_check(fn, x, b, c, cc, h, w, k, num_dets, agnostic);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(dets && workspace, CNB_EINVAL, "%s: null pointer", fn);
  const bool plain = exct_plain(x), aggr = aggr_weight > 0.0f;
  SelectPlan pl;
  MapSelect ms[4];
  size_t sel = 0;
  if (plain) {
    CNB_REQUIRE(workspace_bytes >= cnb_exct_workspace_bytes(b, c, cc, h, w, k, num_dets), CNB_EWORKSPACE,
                "%s: workspace %zu < %zu", fn, workspace_bytes, cnb_exct_workspace_bytes(b, c, cc, h, w, k, num_dets));
    rc = make_select_plan(x.map[0], b, c, h, w, k, 1, &pl);
    if (rc != CNB_OK) return rc;
    pl.clamp_one = 1;   // decode.py:299-302: values above 1 are clamped before _topk
    sel = select_workspace_bytes(pl);
  } else {
    float *const none[4] = {nullptr, nullptr, nullptr, nullptr};
    rc = exct_plans(x, aggr, none, nullptr, b, c, h, w, k, ms, &sel);
    if (rc != CNB_OK) return rc;
    const size_t need = sel + exct_tail_bytes(b, c, h, w, k, num_dets);
    CNB_REQUIRE(workspace_bytes >= need, CNB_EWORKSPACE, "%s: workspace %zu < %zu", fn, workspace_bytes, need);
  }
  char *p = reinterpret_cast<char *>(workspace);
  void *sel_ws = p; p += sel;
  ExctArgs a;
  a.t = carve(p, (long long)b * k); a.l = carve(p, (long long)b * k);
  a.b = carve(p, (long long)b * k); a.r = carve(p, (long long)b * k);
  const size_t map_bytes = align_up((size_t)b * c * h * w * 4, 256);
  float *agg[4];
  for (int q = 0; q < 4; ++q) { agg[q] = reinterpret_cast<float *>(p); p += map_bytes; }
  float *agn = reinterpret_cast<float *>(p); p += align_up((size_t)b * h * w * 4, 256);
  int32_t *agn_cls = reinterpret_cast<int32_t *>(p); p += align_up((size_t)b * h * w * 4, 256);
  const int groups = exct_groups(b, k, num_dets);
  a.seg = reinterpret_cast<u64 *>(p); p += align_up((size_t)b * groups * num_dets * 8, 256);
  a.seg_cnt = reinterpret_cast<int *>(p); p += align_up((size_t)b * groups * 4, 256);
  uint32_t *ct_max = reinterpret_cast<uint32_t *>(p); p += align_up((size_t)b * 4, 256);
  a.ct_max = ct_max;
  a.gthr = reinterpret_cast<u64 *>(p);
  if (!plain) {   // the plans where the aggregated maps and the fp32 copy (agg[0], free without aggregation) really lie
    size_t sel2 = 0;
    rc = exct_plans(x, aggr, agg, agg[0], b, c, h, w, k, ms, &sel2);
    if (rc != CNB_OK) return rc;
    CNB_REQUIRE(sel2 <= sel, CNB_EWORKSPACE, "%s: selection scratch %zu > %zu", fn, sel2, sel);
  }
  CNB_CUDA(cudaMemsetAsync(a.gthr, 0, (size_t)b * 8, stream));

  const void *maps[4] = {x.map[0], x.map[1], x.map[2], x.map[3]};
  if (aggr) {   // :287-291: t,b horizontal; l,r vertical
    const int horiz[4] = {1, 0, 1, 0};
    for (int q = 0; q < 4; ++q) {
      rc = launch_edge_aggregate_ex(maps[q], x.map_dt[q], x.logits != 0, agg[q], b, c, h, w, aggr_weight, horiz[q],
                                    stream);
      if (rc != CNB_OK) return rc;
      maps[q] = agg[q];
    }
  }
  RawList *lists[4] = {&a.t, &a.l, &a.b, &a.r};
  for (int q = 0; q < 4; ++q) {
    FinalizeOut o = {lists[q]->scores, lists[q]->inds, lists[q]->clses, lists[q]->ys, lists[q]->xs,
                     nullptr, nullptr, 0, nullptr};
    if (plain) {
      SelectPlan pq = pl;
      pq.use_tma = pq.use_tma && ((reinterpret_cast<uintptr_t>(maps[q]) & 15u) == 0);
      if (!pq.use_tma) { pq.hot = 0; pq.seg_cap = pq.K; }
      rc = run_select(maps[q], pq, o, sel_ws, stream);
    } else {   // stream order: each selection is done with the scratch and the copy before the next one starts
      rc = aggr ? run_map_select(maps[q], CNB_DTYPE_F32, 0, ms[q], agg[0], o, sel_ws, stream)
                : run_map_select(maps[q], x.map_dt[q], x.logits, ms[q], agg[0], o, sel_ws, stream);
    }
    if (rc != CNB_OK) return rc;
  }
  // centre map; the selections are done with agg[0], which may now hold its fp32 scores
  const bool sig = x.logits != 0;
  a.ct_heat = reinterpret_cast<const float *>(x.ct); a.ct_agn = nullptr; a.ct_cls = nullptr;
  if (agnostic) {
    if (x.ct_dt == CNB_DTYPE_BF16) launch_ct_agnostic<__nv_bfloat16>(x.ct, sig, b, cc, (long long)h * w, agn, agn_cls, stream);
    else if (x.ct_dt == CNB_DTYPE_F16) launch_ct_agnostic<__half>(x.ct, sig, b, cc, (long long)h * w, agn, agn_cls, stream);
    else launch_ct_agnostic<float>(x.ct, sig, b, cc, (long long)h * w, agn, agn_cls, stream);
    CNB_CHECK_LAUNCH("cnb_exct_decode agnostic centre");
    count_launch();
    a.ct_agn = agn; a.ct_cls = agn_cls;
  }
  {   // largest centre value per image: the pruning bound of k_exct_tuples
    CNB_CUDA(cudaMemsetAsync(ct_max, 0, (size_t)b * 4, stream));
    const long long per = agnostic ? (long long)h * w : (long long)cc * h * w;
    int blocks = (int)((per + 256 * 8 - 1) / (256 * 8));
    if (blocks > 64) blocks = 64;
    if (blocks < 1) blocks = 1;
    const dim3 grid((unsigned)blocks, (unsigned)b);
    if (agnostic || (x.ct_dt == CNB_DTYPE_F32 && !sig)) {
      k_ct_max<<<grid, 256, 0, stream>>>(agnostic ? agn : a.ct_heat, per, ct_max);
    } else {   // one pass: the fp32 scores of the centre map (into agg[0]) and their maximum
      if (x.ct_dt == CNB_DTYPE_BF16) launch_ct_scores<__nv_bfloat16>(x.ct, sig, grid, per, agg[0], ct_max, stream);
      else if (x.ct_dt == CNB_DTYPE_F16) launch_ct_scores<__half>(x.ct, sig, grid, per, agg[0], ct_max, stream);
      else launch_ct_scores<float>(x.ct, sig, grid, per, agg[0], ct_max, stream);
      a.ct_heat = agg[0];
    }
    CNB_CHECK_LAUNCH("cnb_exct_decode centre maximum");
    count_launch();
  }
  const bool has_reg = x.regr[0] && x.regr[1] && x.regr[2] && x.regr[3];
  a.t_regr = reinterpret_cast<const float *>(x.regr[0]); a.l_regr = reinterpret_cast<const float *>(x.regr[1]);
  a.b_regr = reinterpret_cast<const float *>(x.regr[2]); a.r_regr = reinterpret_cast<const float *>(x.regr[3]);
  a.B = b; a.CC = cc; a.H = h; a.W = w; a.K = k; a.num_dets = num_dets; a.groups = groups; a.agnostic = agnostic;
  a.scores_thresh = scores_thresh; a.center_thresh = center_thresh; a.dets = dets;
  const size_t smem1 = (size_t)EX_CAP * 8 + (size_t)16 * k * 4;
  CNB_CUDA(cudaFuncSetAttribute(k_exct_tuples, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
  k_exct_tuples<<<b * groups, EX_THREADS, smem1, stream>>>(a);
  CNB_CHECK_LAUNCH("cnb_exct_decode tuples");
  int n2 = 2;
  while (n2 < groups * num_dets) n2 <<= 1;
  const size_t smem2 = (size_t)n2 * 8;
  // fp32 regression maps (or none) take the fp32 merge
  const bool typed = has_reg && !(x.regr_dt[0] == CNB_DTYPE_F32 && x.regr_dt[1] == CNB_DTYPE_F32 &&
                                  x.regr_dt[2] == CNB_DTYPE_F32 && x.regr_dt[3] == CNB_DTYPE_F32);
  if (typed) {
    CNB_CUDA(cudaFuncSetAttribute(k_exct_merge<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    k_exct_merge<true><<<b, 1024, smem2, stream>>>(a, make_int4(x.regr_dt[0], x.regr_dt[1], x.regr_dt[2], x.regr_dt[3]));
  } else {
    CNB_CUDA(cudaFuncSetAttribute(k_exct_merge<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    k_exct_merge<false><<<b, 1024, smem2, stream>>>(a, make_int4(0, 0, 0, 0));
  }
  CNB_CHECK_LAUNCH("cnb_exct_decode merge");
  count_launch(2);
  return CNB_OK;
}

}  // namespace cnb

using namespace cnb;

extern "C" {

size_t cnb_exct_workspace_bytes(int b, int c, int cc, int h, int w, int k, int num_dets) {
  const size_t sel = select_workspace_bytes_any_align(b, c, h, w, k);
  if (sel == 0) return 0;
  (void)cc;
  return sel + exct_tail_bytes(b, c, h, w, k, num_dets);
}

int cnb_exct_groups(int b, int k, int num_dets) {
  if (b < 1 || k < 1 || num_dets < 1) return 0;
  return exct_groups(b, k, num_dets);
}

int cnb_exct_decode(const float *t_heat, const float *l_heat, const float *b_heat, const float *r_heat,
                    const float *ct_heat, const float *t_regr, const float *l_regr, const float *b_regr,
                    const float *r_regr, int b, int c, int cc, int h, int w, int k, float scores_thresh,
                    float center_thresh, float aggr_weight, int num_dets, int agnostic, float *dets, void *workspace,
                    size_t workspace_bytes, void *stream) {
  const int f = CNB_DTYPE_F32;
  const ExctIn x = {{t_heat, l_heat, b_heat, r_heat}, ct_heat, {t_regr, l_regr, b_regr, r_regr}, {f, f, f, f}, f,
                    {f, f, f, f}, 0};
  return exct_decode("cnb_exct_decode", x, b, c, cc, h, w, k, scores_thresh, center_thresh, aggr_weight, num_dets,
                     agnostic, dets, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t cnb_exct_decode_ex_workspace_bytes(const void *t_heat, const void *l_heat, const void *b_heat,
                                          const void *r_heat, int t_dtype, int l_dtype, int b_dtype, int r_dtype,
                                          int ct_dtype, int t_regr_dtype, int l_regr_dtype, int b_regr_dtype,
                                          int r_regr_dtype, int logits, int b, int c, int cc, int h, int w, int k,
                                          float aggr_weight, int num_dets, int agnostic) {
  const int one = 1;   // the centre map's pointer does not enter the workspace: any non-null value
  const ExctIn x = {{t_heat, l_heat, b_heat, r_heat}, &one, {nullptr, nullptr, nullptr, nullptr},
                    {t_dtype, l_dtype, b_dtype, r_dtype}, ct_dtype,
                    {t_regr_dtype, l_regr_dtype, b_regr_dtype, r_regr_dtype}, logits ? 1 : 0};
  if (exct_check("cnb_exct_decode_ex", x, b, c, cc, h, w, k, num_dets, agnostic) != CNB_OK) return 0;
  if (exct_plain(x)) return cnb_exct_workspace_bytes(b, c, cc, h, w, k, num_dets);
  MapSelect m[4];
  size_t sel = 0;
  float *const none[4] = {nullptr, nullptr, nullptr, nullptr};
  if (exct_plans(x, aggr_weight > 0.0f, none, nullptr, b, c, h, w, k, m, &sel) != CNB_OK) return 0;
  return sel + exct_tail_bytes(b, c, h, w, k, num_dets);
}

int cnb_exct_decode_ex(const void *t_heat, int t_dtype, const void *l_heat, int l_dtype, const void *b_heat,
                       int b_dtype, const void *r_heat, int r_dtype, const void *ct_heat, int ct_dtype,
                       const void *t_regr, int t_regr_dtype, const void *l_regr, int l_regr_dtype, const void *b_regr,
                       int b_regr_dtype, const void *r_regr, int r_regr_dtype, int logits, int b, int c, int cc,
                       int h, int w, int k, float scores_thresh, float center_thresh, float aggr_weight,
                       int num_dets, int agnostic, float *dets, void *workspace, size_t workspace_bytes,
                       void *stream) {
  const ExctIn x = {{t_heat, l_heat, b_heat, r_heat}, ct_heat, {t_regr, l_regr, b_regr, r_regr},
                    {t_dtype, l_dtype, b_dtype, r_dtype}, ct_dtype,
                    {t_regr_dtype, l_regr_dtype, b_regr_dtype, r_regr_dtype}, logits ? 1 : 0};
  return exct_decode("cnb_exct_decode_ex", x, b, c, cc, h, w, k, scores_thresh, center_thresh, aggr_weight, num_dets,
                     agnostic, dets, workspace, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"

// Fused 3x3 peak-NMS + exact top-K (score desc, flat index asc) for sm_90a.
//
// Reference semantics (models/decode.py):
//   _nms   :9-15     keep = (maxpool3x3(heat) == heat); heat*keep
//   _topk  :103-119  per-class top-K, then top-K over the C*K survivors
// Under the total order (score desc, flat index asc) the two-stage top-K equals ONE
// global top-K over the NMS'd map, so the kernel streams every plane exactly once:
//
//   stage 1 (persistent, one CTA per SM, 1024 threads)
//     * the B*C planes are cut into n_cta contiguous, equal ranges (perfect balance);
//     * a 3-deep ring of 64 KiB shared-memory stages is filled by TMA bulk copies
//       (cp.async.bulk + mbarrier, UBLKCP in SASS) -- a 128x128 fp32 plane is one stage;
//     * phase A: each warp sweeps rows with a 3-row register window: vertical max3 on
//       float4, horizontal neighbours by warp shuffle, `==` peak test, running-threshold
//       test, and a ballot bitmask of the qualifying pixels (no per-pixel atomics);
//     * phase B: the few set bits are expanded into a 4096-entry key buffer; when it is
//       half full it is bitonic-sorted and cut to K, which raises the threshold so later
//       planes of the same image contribute only a handful of candidates.  The first
//       unit of an image is expanded a quarter at a time so the threshold exists early;
//     * at an image boundary the CTA's best <=K keys go to that image's segment, and the
//       LAST CTA to deliver a segment (atomic ticket) merges the <=max_slots segments,
//       sorts and emits the K best with the ctdet gathers / box assembly fused
//       (decode.py:472-493).  Tiny batches whose segments do not fit the key buffer use
//       the separate finalize kernel instead.
//
// Non-positive scores (zero fillers, negative peaks) only matter when an image has < K
// positive peaks; finalize handles that exactly with an ordered rescan (rare slow path).
//
// The hot kernel also reads fp16 / bf16 maps (k_select_hot<__half | __nv_bfloat16, LOGITS>): 32 KiB planes in the
// same 3-deep ring, each element widened exactly to fp32 in registers, so the result is bit for bit that of the
// .float() upcast (DESIGN 4.1).  Other stage-1 kernels read fp32 only.
#include "select.cuh"
#include <stdlib.h>
#include <algorithm>
#include <map>
#include <mutex>
#include <utility>

namespace cnb {

typedef unsigned long long u64;

// Contiguous partition of the B*C planes over n_cta CTAs.  Planes cost 1, every image boundary costs
// `wb` extra planes (the CTA that crosses it pays a flush, a bootstrap and usually the finalize), so
// ranges that contain a boundary get correspondingly fewer planes.  wb = 0 is the plain equal split.
struct Part {
  long long P;
  int n_cta, C, wb;
};
__host__ __device__ __forceinline__ long long cta_first_plane(long long cta, const Part &q) {
  const long long blk = (long long)q.C + q.wb;
  const long long ftot = (q.P / q.C) * blk;
  const long long T = cta * ftot / q.n_cta;
  const long long m = T / blk, rem = T - m * blk;
  return m * q.C + (rem < q.C ? rem : q.C);
}
// CTA whose range contains plane p: largest i with cta_first_plane(i) <= p.
__host__ __device__ __forceinline__ int cta_of_plane(long long p, const Part &q) {
  int lo = 0, hi = q.n_cta - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cta_first_plane(mid, q) <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}
// Device side: the host-computed table (no 64-bit divisions on the GPU).
__device__ __forceinline__ long long plan_first_plane(const SelectPlan &pl, int cta) { return pl.cta_start[cta]; }
__device__ __forceinline__ int plan_cta_of_plane(const SelectPlan &pl, long long p) {
  int lo = 0, hi = pl.n_cta - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((long long)pl.cta_start[mid] <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ------------------------------------------------------------------ cooperating-thread groups
// The helpers below run either on the whole CTA (generic kernel, separate finalize kernel) or on a
// single warp (the warp-asynchronous hot kernel, where one warp at a time owns the selection state).
struct CtaGroup {
  static __device__ __forceinline__ int tid() { return threadIdx.x; }
  static __device__ __forceinline__ int n() { return blockDim.x; }
  static __device__ __forceinline__ void sync() { __syncthreads(); }
};
struct WarpGroup {
  static __device__ __forceinline__ int tid() { return threadIdx.x & 31; }
  static __device__ __forceinline__ int n() { return 32; }
  static __device__ __forceinline__ void sync() { __syncwarp(); }
};

// ------------------------------------------------------------------ bitonic sort
// Sorts buf[0..n) descending; n is a power of two; all threads of the group must call.
template <typename G>
__device__ __forceinline__ void group_sort_desc(u64 *buf, int n) {
  const int tid = G::tid(), nt = G::n();
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (n >> 1); t += nt) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const u64 a = buf[i], b = buf[i + j];
        const bool desc = (i & k) == 0;
        if ((a < b) == desc) {
          buf[i] = b;
          buf[i + j] = a;
        }
      }
      G::sync();
    }
  }
}
// CTA-wide bitonic sort for n <= blockDim.x: one key per thread in a register; compare-exchange
// partners closer than a warp come by shuffle (no barrier), only the strides >= 32 go through
// shared memory (15 of the 55 stages at n = 1024).
__device__ __forceinline__ void cta_sort_desc_reg(u64 *buf, int n) {
  const int i = threadIdx.x;
  const bool part = (i >> 5) < ((n + 31) >> 5);   // warps that hold keys; the others only keep the barriers company
  u64 v = (i < n) ? buf[i] : 0ull;
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      u64 p = 0ull;
      if (j >= 32) {
        __syncthreads();
        if (i < n) buf[i] = v;
        __syncthreads();
        if (i < n) p = buf[i ^ j];
      } else if (part) {
        const uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)v, j);
        const uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(v >> 32), j);
        p = ((u64)hi << 32) | lo;
      }
      if (part) {
        const bool take_max = (((i & k) == 0) == ((i & j) == 0));
        v = take_max ? (v > p ? v : p) : (v < p ? v : p);
      }
    }
  }
  __syncthreads();
  if (i < n) buf[i] = v;
  __syncthreads();
}
__device__ __forceinline__ void cta_sort_desc(u64 *buf, int n) {
  if (n <= (int)blockDim.x && blockDim.x >= 64) cta_sort_desc_reg(buf, n);
  else group_sort_desc<CtaGroup>(buf, n);
}
template <typename G>
__device__ __forceinline__ void sort_desc_best(u64 *buf, int n) { group_sort_desc<G>(buf, n); }
template <>
__device__ __forceinline__ void sort_desc_best<CtaGroup>(u64 *buf, int n) { cta_sort_desc(buf, n); }

__host__ __device__ __forceinline__ int next_pow2(int v) {
  int n = 2;
  while (n < v) n <<= 1;
  return n;
}

// Sort the candidate buffer and keep the K best.  Returns the new 64-bit threshold
// (key of the K-th best, or 0 when fewer than K are known).  CTA-uniform.
template <typename G>
__device__ __forceinline__ u64 group_prune(u64 *buf, int *s_cnt, int K) {
  G::sync();
  const int cnt = *(volatile int *)s_cnt;
  const int n = next_pow2(cnt);
  for (int t = cnt + G::tid(); t < n; t += G::n()) buf[t] = 0ull;
  G::sync();
  sort_desc_best<G>(buf, n);
  u64 thr = 0ull;
  if (cnt >= K) thr = buf[K - 1];
  G::sync();
  if (G::tid() == 0 && cnt > K) *s_cnt = K;
  G::sync();
  return thr;
}
__device__ __forceinline__ u64 cta_prune(u64 *buf, int *s_cnt, int K) { return group_prune<CtaGroup>(buf, s_cnt, K); }

// ---- running threshold: 2-level histogram of the pushed scores (128 bins per octave over
// [2^-16, 1), 32 coarse x 64 fine).  The lower edge of the highest bin whose suffix count reaches
// K is a valid lower bound of the image's K-th best score: at least K real candidates lie above it.
__device__ __forceinline__ int hist_bin(uint32_t bits) {
  const int e = (int)(bits >> 16) - ((127 - 16) << 7);
  return min(max(e, 0), SEL_HIST_FINE - 1);
}
__device__ __forceinline__ uint32_t bin_lower_bits(int b) {
  return b <= 0 ? 1u : ((uint32_t)(b + ((127 - 16) << 7)) << 16);
}
// Highest of 64 bins whose suffix count is >= need (or -1); *rem = need - (count strictly above it).
__device__ __forceinline__ int warp_suffix_pick(const int *bins, int lane, int need, int *rem) {
  const int c0 = bins[2 * lane], c1 = bins[2 * lane + 1];
  const int s = c0 + c1;
  int suf = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_down_sync(0xffffffffu, suf, o);
    if (lane + o < 32) suf += t;
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, suf >= need);
  if (!bal) return -1;
  const int L = 31 - __clz(bal);
  const int above = __shfl_sync(0xffffffffu, suf - s, L);
  const int c1L = __shfl_sync(0xffffffffu, c1, L);
  if (above + c1L >= need) {
    *rem = need - above;
    return 2 * L + 1;
  }
  *rem = need - above - c1L;
  return 2 * L;
}
// warp 0 only
__device__ __forceinline__ void update_threshold(const int *fine, const int *coarse, int lane, int K,
                                                 uint32_t *s_thr) {
  int rem = 0, rem2 = 0;
  const int cb = warp_suffix_pick(coarse, lane, K, &rem);
  uint32_t bits = 0u;
  if (cb >= 0) {
    const int fb = warp_suffix_pick(fine + cb * 64, lane, rem, &rem2);
    bits = bin_lower_bits(cb * 64 + max(fb, 0));
  }
  if (lane == 0) *s_thr = bits;
}

// ------------------------------------------------------------------ logits input (fused sigmoid)
// The same expression torch's CUDA sigmoid evaluates for float (1 / (1 + exp(-x)), libdevice expf,
// IEEE division; this library is built without fast-math), so scores are bit-identical to
// `hm.sigmoid_()` (detectors/ctdet.py:31).  tests/test_logits_gpu.py checks both the bit identity
// and that the function is monotone non-decreasing over every float - the property the logits path
// relies on: the 3x3 maximum of the heat map is the sigmoid of the 3x3 maximum of the logits.
__device__ __forceinline__ float sigmoid_ref(float x) { return 1.0f / (1.0f + expf(-x)); }

// Conservative lower bound (in logit space) of a score threshold given as fp32 bits.
__device__ __forceinline__ float logit_lower_bound(uint32_t score_bits) {
  if (score_bits == 0u) return CNB_NEG_INF;
  const float t = __uint_as_float(score_bits);
  if (!(t >= 1e-30f)) return CNB_NEG_INF;
  const float l = __logf(t) - __logf(fmaxf(1.0f - t, 1e-8f));
  return l - (0.002f + 0.002f * fabsf(l));
}
// How far below the 3x3 logit maximum M a pixel can sit and still share M's fp32 sigmoid (8 ulp of
// slack on top of the derivative bound; saturated / denormal ends: always compare).
__device__ __forceinline__ float collide_margin(float M) {
  if (M > 12.0f || M < -80.0f) return __int_as_float(0x7f800000);
  if (M > 8.0f) return 0.25f;
  if (M > 4.0f) return 4e-3f;
  if (M > 0.0f) return 1e-4f;
  return 7.62939453125e-6f;  // 2^-17
}

// ------------------------------------------------------------------ finalize (shared by both paths)
// v'(i): the reference's heat*keep value of flat pixel i (keep only in NMS mode); T = map element type.
template <bool NMS, typename T>
__device__ __forceinline__ float nms_value(const T *__restrict__ img, int C, int H, int W, long long i,
                                           bool logits = false) {
  const float v = to_f32(img[i]);
  if (!NMS) return logits ? sigmoid_ref(v) : v;
  const long long HW = (long long)H * W;
  const long long c = i / HW, sp = i - c * HW;
  const int y = (int)(sp / W), x = (int)(sp - (long long)y * W);
  const T *pl = img + c * HW;
  float m = v;
  for (int dy = -1; dy <= 1; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -1; dx <= 1; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W) continue;
      m = fmaxf(m, to_f32(pl[(long long)yy * W + xx]));
    }
  }
  if (logits) {  // monotone sigmoid: max of the heat neighbourhood == sigmoid(max of the logits)
    const float sv = sigmoid_ref(v);
    return (m == v || sigmoid_ref(m) == sv) ? sv : 0.0f;
  }
  return (m == v) ? v : 0.0f;
}

template <bool NMS, typename G, typename T>
__device__ void finalize_fill(const T *__restrict__ img, const SelectPlan &pl, u64 *sbuf, int have, int K,
                              int *s_tmp, u64 *s_red) {
  // Need K-have more entries ranked (value desc, index asc) among NON-positive v'.
  const int tid = G::tid(), lane = tid & 31, warp = tid >> 5, nw = G::n() >> 5;
  const long long N = (long long)pl.C * pl.H * pl.W;
  int found = 0;
  const int need = K - have;
  // step 1: zeros, in index order
  for (long long base = 0; base < N && found < need; base += G::n()) {
    const long long i = base + tid;
    bool pred = false;
    if (i < N) pred = (nms_value<NMS>(img, pl.C, pl.H, pl.W, i, pl.logits != 0) == 0.0f);
    const uint32_t bal = __ballot_sync(0xffffffffu, pred);
    if (lane == 0) s_tmp[warp] = __popc(bal);
    G::sync();
    int before = 0, total = 0;
    for (int w2 = 0; w2 < nw; ++w2) {
      const int cw = s_tmp[w2];
      if (w2 < warp) before += cw;
      total += cw;
    }
    const int pos = found + before + __popc(bal & ((1u << lane) - 1u));
    if (pred && pos < need) sbuf[have + pos] = make_key(0u, (uint32_t)i);
    found += total;
    G::sync();
  }
  found = min(found, need);
  // step 2: negative values, largest first (brute force; pathological inputs only)
  u64 prev = ~0ull;
  while (found < need) {
    u64 best = 0ull;
    for (long long i = tid; i < N; i += G::n()) {
      const float v = nms_value<NMS>(img, pl.C, pl.H, pl.W, i, pl.logits != 0);
      if (v < 0.0f) {
        const u64 key = ((u64)(~__float_as_uint(v)) << 32) | (u64)(0xffffffffu - (uint32_t)i);
        if (key < prev && key > best) best = key;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const u64 other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other > best ? other : best;
    }
    if (lane == 0) s_red[warp] = best;
    G::sync();
    best = 0ull;
    for (int w2 = 0; w2 < nw; ++w2) best = s_red[w2] > best ? s_red[w2] : best;
    G::sync();
    if (best == 0ull) {  // nothing left (NaNs only): pad with pixel 0 / score 0
      if (tid == 0) sbuf[have + found] = make_key(0u, 0u);
    } else {
      if (tid == 0) sbuf[have + found] = make_key(~(uint32_t)(best >> 32), key_idx(best));
      prev = best;
    }
    ++found;
  }
  G::sync();
}

// Row k of image b from its key (raw top-K outputs and/or the fused ctdet epilogue, models/decode.py:472-493).
// The four gathered values (reg x, reg y, wh w, wh h) may come pre-loaded (gath != nullptr).
struct RowGather { float rx, ry, ww, wh_; };
__device__ __forceinline__ RowGather gather_row(const SelectPlan &pl, int b, u64 key, const FinalizeOut &out) {
  RowGather g = {0.5f, 0.5f, 0.f, 0.f};
  if (!out.dets) return g;
  const long long HW = (long long)pl.H * pl.W;
  const uint32_t flat = key_idx(key);
  const int cls = (int)(flat / (uint32_t)HW);
  const int sp = (int)(flat - (uint32_t)cls * (uint32_t)HW);
  if (out.reg) {  // decode.py:472-476
    const size_t r = (size_t)b * 2 * HW + sp;
    g.rx = ld_head(out.reg, out.reg_dtype, r);
    g.ry = ld_head(out.reg, out.reg_dtype, r + HW);
  }
  const int whc = out.cat_spec_wh ? 2 * pl.C : 2;  // :480-486
  const size_t wp = ((size_t)b * whc + (out.cat_spec_wh ? 2 * cls : 0)) * HW + sp;
  g.ww = ld_head(out.wh, out.wh_dtype, wp);
  g.wh_ = ld_head(out.wh, out.wh_dtype, wp + HW);
  return g;
}
__device__ __forceinline__ void emit_one(const SelectPlan &pl, int b, int k, u64 key, const FinalizeOut &out,
                                         const RowGather &g) {
  const int K = pl.K;
  const long long HW = (long long)pl.H * pl.W;
  const float score = __uint_as_float(key_bits(key));
  const uint32_t flat = key_idx(key);
  const int cls = (int)(flat / (uint32_t)HW);
  const int sp = (int)(flat - (uint32_t)cls * (uint32_t)HW);
  const int yi = sp / pl.W, xi = sp - yi * pl.W;
  const size_t o = (size_t)b * K + k;
  if (out.scores) out.scores[o] = score;
  if (out.inds) out.inds[o] = (int64_t)sp;
  if (out.clses) out.clses[o] = cls;
  if (out.ys) out.ys[o] = (float)yi;
  if (out.xs) out.xs[o] = (float)xi;
  if (out.dets) {
    const float xs = (float)xi + g.rx, ys = (float)yi + g.ry;   // reg offsets, or +0.5 when there is no reg head (:477-479)
    const float hw_ = g.ww * 0.5f, hh_ = g.wh_ * 0.5f;
    float *d = out.dets + o * 6;  // :487-493
    d[0] = xs - hw_;
    d[1] = ys - hh_;
    d[2] = xs + hw_;
    d[3] = ys + hh_;
    d[4] = score;
    d[5] = (float)cls;
  }
}
// Write the K rows of image b from its sorted keys.
template <typename G>
__device__ __forceinline__ void emit_rows(const SelectPlan &pl, int b, const u64 *sbuf, const FinalizeOut &out) {
  for (int k = G::tid(); k < pl.K; k += G::n()) {
    const u64 key = sbuf[k];
    emit_one(pl, b, k, key, out, gather_row(pl, b, key, out));
  }
}

// Merge the segments of image b (written by the stage-1 CTAs i0..i1), sort, emit.
// sbuf must hold next_pow2(max(max_slots*K, K)) keys.  All threads of the CTA call.
template <bool NMS, typename G>
__device__ void finalize_image(const float *__restrict__ src, const SelectPlan &pl, int b,
                               const u64 *__restrict__ cand, const int *__restrict__ cand_cnt,
                               const FinalizeOut &out, u64 *sbuf, int *s_tmp, u64 *s_red,
                               const uint32_t *cand_thr = nullptr) {
  const int tid = G::tid(), K = pl.K;
  if (tid == 0) {  // the binary search costs ~1k instructions: one thread does it
    s_tmp[30] = plan_cta_of_plane(pl, (long long)b * pl.C);
    s_tmp[31] = plan_cta_of_plane(pl, (long long)(b + 1) * pl.C - 1);
  }
  G::sync();
  const int i0 = s_tmp[30], i1 = s_tmp[31];
  int total = 0;
  for (int slot = 0; slot <= i1 - i0; ++slot) {
    const int n = __ldcg(cand_cnt + (size_t)b * pl.max_slots + slot);
    const u64 *seg = cand + ((size_t)b * pl.max_slots + slot) * pl.seg_cap;
    for (int t = tid; t < n; t += G::n()) sbuf[total + t] = __ldcg(seg + t);
    total += n;
  }
  G::sync();
  if (cand_thr != nullptr && total > 2 * K && total <= 2 * G::n()) {
    // every segment comes with a valid lower bound of the image's K-th best score (the K-th best of
    // a subset never exceeds the K-th best of the whole), so the largest of them is one too: drop
    // everything below it before sorting (>= K survive, usually ~1.2 K; <= 2 keys per thread here)
    uint32_t tb = 0u;
    for (int slot = 0; slot <= i1 - i0; ++slot) tb = max(tb, __ldcg(cand_thr + (size_t)b * pl.max_slots + slot));
    if (tid == 0) s_tmp[0] = 0;
    const u64 mine0 = (tid < total) ? sbuf[tid] : 0ull;
    const u64 mine1 = (tid + G::n() < total) ? sbuf[tid + G::n()] : 0ull;
    G::sync();
    if (mine0 != 0ull && key_bits(mine0) >= tb) sbuf[atomicAdd(&s_tmp[0], 1)] = mine0;
    if (mine1 != 0ull && key_bits(mine1) >= tb) sbuf[atomicAdd(&s_tmp[0], 1)] = mine1;
    G::sync();
    total = s_tmp[0];
    G::sync();
  }
  if (total <= 256 && total <= G::n() && G::n() >= 256) {
    // few survivors: rank sort (every key counts the keys above it; no dependent network stages)
    const u64 mine = (tid < total) ? sbuf[tid] : 0ull;
    int rank = 0;
    if (tid < total)
      for (int t = 0; t < total; ++t) rank += (sbuf[t] > mine) ? 1 : 0;
    G::sync();
    const int n2 = max(total, K);
    for (int t = total + tid; t < n2; t += G::n()) sbuf[t] = 0ull;
    if (tid < total) sbuf[rank] = mine;
    G::sync();
  } else {
    const int n = next_pow2(max(total, K));
    for (int t = total + tid; t < n; t += G::n()) sbuf[t] = 0ull;
    G::sync();
    sort_desc_best<G>(sbuf, n);  // segments may be unsorted supersets (hot kernel)
  }
  if (total < K) {
    const long long N = (long long)pl.C * pl.H * pl.W;
    finalize_fill<NMS, G>(src + (long long)b * N, pl, sbuf, total, K, s_tmp, s_red);
  }
  emit_rows<G>(pl, b, sbuf, out);
  G::sync();
}

// ------------------------------------------------------------------ stage 1
struct UnitGeom {
  long long plane;
  int img, c;
  int r0, r1;  // rows owned by the unit
  int ra, rb;  // rows resident in the stage (halo included)
};

__device__ __forceinline__ UnitGeom unit_geom(const SelectPlan &pl, long long p_begin, int u) {
  UnitGeom g;
  const int pi = u / pl.upp, strip = u - pi * pl.upp;
  g.plane = p_begin + pi;
  g.img = (int)(g.plane / pl.C);
  g.c = (int)(g.plane - (long long)g.img * pl.C);
  g.r0 = strip * pl.rb;
  g.r1 = min(pl.H, g.r0 + pl.rb);
  g.ra = max(g.r0 - 1, 0);
  g.rb = min(g.r1 + 1, pl.H);
  return g;
}

// MODE 0: generic geometry; 1: one 128-column block per row (W <= 128, W % 4 == 0, TMA);
// MODE 2: the hot geometry, whole 128x128 planes (4 rows per warp, fully unrolled).
template <bool NMS, bool TMA, int MODE>
__global__ void __launch_bounds__(SEL_THREADS, 1)
k_select_stage1(const float *__restrict__ src, const SelectPlan pl, u64 *__restrict__ cand,
                int *__restrict__ cand_cnt, int *__restrict__ img_done, const FinalizeOut fout) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float *stages = reinterpret_cast<float *>(smem_raw);
  u64 *buf = reinterpret_cast<u64 *>(smem_raw + (size_t)SEL_STAGES * SEL_STAGE_BYTES);
  int *fine = reinterpret_cast<int *>(buf + SEL_CAP);
  int *coarse = fine + SEL_HIST_FINE;
  uint32_t *masks = reinterpret_cast<uint32_t *>(coarse + SEL_HIST_COARSE);
  uint64_t *full = reinterpret_cast<uint64_t *>(masks + SEL_MASK_WORDS);
  // [0] buffer count, [1] overflow flag, [2] last-CTA flag, [3] compaction count, [4] threshold bits, [5] count at last update
  int *s_cnt = reinterpret_cast<int *>(full + SEL_STAGES);
  uint32_t *s_thr = reinterpret_cast<uint32_t *>(s_cnt + 4);
  __shared__ int s_tmp[32];
  __shared__ u64 s_red[32];
  constexpr bool FAST = (MODE >= 1);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int H = pl.H, W = pl.W, Wp = pl.Wp, ncb = pl.ncb, K = pl.K;
  const long long HW = (long long)H * W;
  const long long p_begin = plan_first_plane(pl, blockIdx.x);
  const long long p_end = plan_first_plane(pl, blockIdx.x + 1);
  const int total_units = (int)(p_end - p_begin) * pl.upp;
  const float NI = CNB_NEG_INF;

  auto issue = [&](int u) {  // thread 0 only (TMA path)
    const UnitGeom g = unit_geom(pl, p_begin, u);
    const int s = u % SEL_STAGES;
    const uint32_t bytes = (uint32_t)(g.rb - g.ra) * (uint32_t)W * 4u;
    const char *gsrc = reinterpret_cast<const char *>(src + (g.plane * H + g.ra) * (long long)W);
    char *dst = reinterpret_cast<char *>(stages) + (size_t)s * SEL_STAGE_BYTES;
    mbar_expect_tx(&full[s], bytes);
    for (uint32_t off = 0; off < bytes; off += 16384u)
      bulk_g2s(dst + off, gsrc + off, min(16384u, bytes - off), &full[s]);
  };
  auto clear_hist = [&]() {
    for (int i = tid; i < SEL_HIST_FINE + SEL_HIST_COARSE; i += SEL_THREADS) fine[i] = 0;  // coarse follows fine
    if (tid == 0) {
      s_cnt[0] = 0; s_cnt[1] = 0; s_cnt[3] = 0; s_cnt[5] = 0;
      *s_thr = 0u;
    }
  };

  if (tid == 0 && TMA) {
    for (int s = 0; s < SEL_STAGES; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  clear_hist();
  __syncthreads();
  if (TMA && tid == 0) {
    for (int u = 0; u < SEL_STAGES && u < total_units; ++u) issue(u);
  }

  u64 thr64 = 0ull;  // exact key threshold; non-zero only after a sort-prune (overflow fallback)
  int cur_img = -1;

  auto flush = [&](int img) {
    __syncthreads();
    const int cnt = s_cnt[0];
    const u64 *outp = buf;
    int n_out = min(cnt, K);
    if (cnt > K && cnt <= SEL_CAP / 2) {
      // cut with the histogram threshold, sort only the survivors (>= K of them, see header)
      if (warp == 0) update_threshold(fine, coarse, lane, K, s_thr);
      __syncthreads();
      const uint32_t tb = *s_thr;
      u64 *hi = buf + SEL_CAP / 2;
      for (int t = tid; t < cnt; t += SEL_THREADS) {
        const u64 key = buf[t];
        if (key_bits(key) >= tb) hi[atomicAdd(&s_cnt[3], 1)] = key;
      }
      __syncthreads();
      const int m = s_cnt[3];
      const int n = next_pow2(m);
      for (int t = m + tid; t < n; t += SEL_THREADS) hi[t] = 0ull;
      __syncthreads();
      cta_sort_desc(hi, n);
      outp = hi;
      n_out = min(m, K);
    } else {
      cta_prune(buf, s_cnt, K);
    }
    if (tid == 0) s_tmp[28] = plan_cta_of_plane(pl, (long long)img * pl.C);
    __syncthreads();
    const int i0 = s_tmp[28];
    const int slot = (int)blockIdx.x - i0;
    u64 *dst = cand + ((size_t)img * pl.max_slots + slot) * pl.seg_cap;
    for (int t = tid; t < n_out; t += SEL_THREADS) dst[t] = outp[t];
    if (tid == 0) cand_cnt[(size_t)img * pl.max_slots + slot] = n_out;
    if (pl.fused_finalize) {
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        const int i1 = plan_cta_of_plane(pl, (long long)(img + 1) * pl.C - 1);
        const int ticket = atomicAdd(&img_done[img], 1);
        s_cnt[2] = (ticket == i1 - i0) ? 1 : 0;
      }
      __syncthreads();
      if (s_cnt[2]) {  // every segment of this image is in global memory: merge + emit here
        __threadfence();
        finalize_image<NMS, CtaGroup>(src, pl, img, cand, cand_cnt, fout, buf, s_tmp, s_red);
      }
    }
    __syncthreads();
    clear_hist();
    __syncthreads();
  };

  for (int u = 0; u < total_units; ++u) {
    const UnitGeom g = unit_geom(pl, p_begin, u);
    const int s = TMA ? (u % SEL_STAGES) : 0;
    float *st = stages + (size_t)s * (SEL_STAGE_BYTES / 4);
    if (g.img != cur_img) {
      if (cur_img >= 0) flush(cur_img);
      cur_img = g.img;
      thr64 = 0ull;
    }
    if (TMA) {
      mbar_wait(&full[s], (uint32_t)((u / SEL_STAGES) & 1));
    } else {
      // generic loader (W % 4 != 0 or unaligned base): pad columns are -inf
      const int nrow = g.rb - g.ra;
      const float *gsrc = src + (g.plane * H + g.ra) * (long long)W;
      for (int i = tid; i < nrow * Wp; i += SEL_THREADS) {
        const int r = i / Wp, col = i - r * Wp;
        st[i] = (col < W) ? __ldg(gsrc + (long long)r * W + col) : NI;
      }
      __syncthreads();
    }

    // ---------------- phase A: peak + threshold test -> bitmask of qualifying pixels
    // thr_f >= smallest positive float, so b == max(hmax, thr_f) also rejects b <= 0
    const uint32_t thr_bits = max(max(*s_thr, key_bits(thr64)), 1u);
    const float thr_f = __uint_as_float(thr_bits);
    const int rows = g.r1 - g.r0;
    if (MODE == 2) {
      // whole 128x128 plane: warp w owns rows 4w..4w+3, lane l columns 4l..4l+3
      const int y0 = warp * 4;
      const float *p = st + (size_t)y0 * 128 + lane * 4;
      const float4 ninf = make_float4(NI, NI, NI, NI);
      float4 r_[6];
      r_[0] = (y0 > 0) ? *reinterpret_cast<const float4 *>(p - 128) : ninf;
#pragma unroll
      for (int i = 0; i < 4; ++i) r_[i + 1] = *reinterpret_cast<const float4 *>(p + i * 128);
      r_[5] = (y0 + 4 < 128) ? *reinterpret_cast<const float4 *>(p + 4 * 128) : ninf;
      uint4 *mrow = reinterpret_cast<uint4 *>(masks) + y0;
      const bool first = (lane == 0), last = (lane == 31);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 a = r_[i], b = r_[i + 1], c = r_[i + 2];
        const float v0 = fmax3(a.x, b.x, c.x), v1 = fmax3(a.y, b.y, c.y);
        const float v2 = fmax3(a.z, b.z, c.z), v3 = fmax3(a.w, b.w, c.w);
        float l = __shfl_up_sync(0xffffffffu, v3, 1);
        float r = __shfl_down_sync(0xffffffffu, v0, 1);
        l = first ? NI : l;
        r = last ? NI : r;
        const float m01 = fmaxf(v0, v1), m23 = fmaxf(v2, v3);
        const bool q0 = (b.x == fmax3(l, m01, thr_f));
        const bool q1 = (b.y == fmax3(m01, v2, thr_f));
        const bool q2 = (b.z == fmax3(v1, m23, thr_f));
        const bool q3 = (b.w == fmax3(m23, r, thr_f));
        const uint32_t m0 = __ballot_sync(0xffffffffu, q0), m1 = __ballot_sync(0xffffffffu, q1);
        const uint32_t m2 = __ballot_sync(0xffffffffu, q2), m3 = __ballot_sync(0xffffffffu, q3);
        if (first) mrow[i] = make_uint4(m0, m1, m2, m3);
      }
    } else if (MODE == 1) {
      const int thr_s = (int)thr_bits;
      const int rw = (rows + SEL_WARPS - 1) / SEL_WARPS;
      const int y0 = g.r0 + warp * rw, yend = min(y0 + rw, g.r1);
      if (y0 < yend) {
        const bool xin = lane * 4 < W;
        const float *p = st + (size_t)(y0 - g.ra) * Wp + lane * 4;
        const float4 ninf = make_float4(NI, NI, NI, NI);
        float4 a = (NMS && y0 > 0 && xin) ? *reinterpret_cast<const float4 *>(p - Wp) : ninf;
        float4 b = xin ? *reinterpret_cast<const float4 *>(p) : ninf;
        uint4 *mrow = reinterpret_cast<uint4 *>(masks) + (y0 - g.r0);
#pragma unroll 4
        for (int y = y0; y < yend; ++y, p += Wp, ++mrow) {
          const float4 c = (y + 1 < H && xin) ? *reinterpret_cast<const float4 *>(p + Wp) : ninf;
          bool q0 = __float_as_int(b.x) >= thr_s, q1 = __float_as_int(b.y) >= thr_s;
          bool q2 = __float_as_int(b.z) >= thr_s, q3 = __float_as_int(b.w) >= thr_s;
          if (NMS) {
            const float v0 = fmax3(a.x, b.x, c.x), v1 = fmax3(a.y, b.y, c.y);
            const float v2 = fmax3(a.z, b.z, c.z), v3 = fmax3(a.w, b.w, c.w);
            float l = __shfl_up_sync(0xffffffffu, v3, 1);
            float r = __shfl_down_sync(0xffffffffu, v0, 1);
            l = (lane == 0) ? NI : l;
            r = (lane == 31) ? NI : r;
            q0 = q0 && (b.x == fmax3(l, v0, v1));
            q1 = q1 && (b.y == fmax3(v0, v1, v2));
            q2 = q2 && (b.z == fmax3(v1, v2, v3));
            q3 = q3 && (b.w == fmax3(v2, v3, r));
          } else {  // no peak test: NaN/inf bit patterns above +inf must not pass
            q0 = q0 && (__float_as_uint(b.x) <= 0x7f800000u);
            q1 = q1 && (__float_as_uint(b.y) <= 0x7f800000u);
            q2 = q2 && (__float_as_uint(b.z) <= 0x7f800000u);
            q3 = q3 && (__float_as_uint(b.w) <= 0x7f800000u);
          }
          const uint32_t m0 = __ballot_sync(0xffffffffu, q0), m1 = __ballot_sync(0xffffffffu, q1);
          const uint32_t m2 = __ballot_sync(0xffffffffu, q2), m3 = __ballot_sync(0xffffffffu, q3);
          if (lane == 0) *mrow = make_uint4(m0, m1, m2, m3);
          a = b;
          b = c;
        }
      }
    } else {
      const int thr_s = (int)thr_bits;
      const int ngroups = (rows + SEL_RW - 1) / SEL_RW;
      for (int item = warp; item < ngroups * ncb; item += SEL_WARPS) {
        const int grp = item / ncb, cb = item - grp * ncb;
        const int y0 = g.r0 + grp * SEL_RW, yend = min(y0 + SEL_RW, g.r1);
        const int x0 = cb * 128 + lane * 4;
        const bool xin = x0 < Wp;
        auto ldrow = [&](int y) -> float4 {
          if (y < 0 || y >= H || !xin) return make_float4(NI, NI, NI, NI);
          return *reinterpret_cast<const float4 *>(st + (size_t)(y - g.ra) * Wp + x0);
        };
        auto vcol = [&](int y, int x) -> float {  // vertical max3 of one column (warp-edge lanes)
          float m = st[(size_t)(y - g.ra) * Wp + x];
          if (y - 1 >= 0) m = fmaxf(m, st[(size_t)(y - 1 - g.ra) * Wp + x]);
          if (y + 1 < H) m = fmaxf(m, st[(size_t)(y + 1 - g.ra) * Wp + x]);
          return m;
        };
        float4 a = NMS ? ldrow(y0 - 1) : make_float4(NI, NI, NI, NI);
        float4 b = ldrow(y0);
        for (int y = y0; y < yend; ++y) {
          bool q0 = __float_as_int(b.x) >= thr_s, q1 = __float_as_int(b.y) >= thr_s;
          bool q2 = __float_as_int(b.z) >= thr_s, q3 = __float_as_int(b.w) >= thr_s;
          float4 c = make_float4(NI, NI, NI, NI);
          if (NMS) {
            c = ldrow(y + 1);
            const float v0 = fmax3(a.x, b.x, c.x), v1 = fmax3(a.y, b.y, c.y);
            const float v2 = fmax3(a.z, b.z, c.z), v3 = fmax3(a.w, b.w, c.w);
            float l = __shfl_up_sync(0xffffffffu, v3, 1);
            float r = __shfl_down_sync(0xffffffffu, v0, 1);
            if (lane == 0) l = (cb > 0) ? vcol(y, x0 - 1) : NI;
            if (lane == 31) r = (x0 + 4 < Wp) ? vcol(y, x0 + 4) : NI;
            q0 = q0 && (b.x == fmax3(l, v0, v1));
            q1 = q1 && (b.y == fmax3(v0, v1, v2));
            q2 = q2 && (b.z == fmax3(v1, v2, v3));
            q3 = q3 && (b.w == fmax3(v2, v3, r));
          } else {
            q0 = q0 && (__float_as_uint(b.x) <= 0x7f800000u);
            q1 = q1 && (__float_as_uint(b.y) <= 0x7f800000u);
            q2 = q2 && (__float_as_uint(b.z) <= 0x7f800000u);
            q3 = q3 && (__float_as_uint(b.w) <= 0x7f800000u);
          }
          const uint32_t m0 = __ballot_sync(0xffffffffu, q0), m1 = __ballot_sync(0xffffffffu, q1);
          const uint32_t m2 = __ballot_sync(0xffffffffu, q2), m3 = __ballot_sync(0xffffffffu, q3);
          if (lane == 0)
            *reinterpret_cast<uint4 *>(masks + ((y - g.r0) * ncb + cb) * 4) = make_uint4(m0, m1, m2, m3);
          a = b;
          b = NMS ? c : ldrow(y + 1);
        }
      }
    }

    // ---------------- phase B: expand bitmasks into the key buffer (+ histogram)
    const int words = rows * ncb * 4;
    const uint32_t cbase = (uint32_t)((long long)g.c * HW);
    auto make = [&](int word, int bit) -> u64 {
      const int j = word & 3, rc = word >> 2;
      const int row = FAST ? rc : rc / ncb, cb = FAST ? 0 : rc - row * ncb;
      const int y = g.r0 + row, x = cb * 128 + bit * 4 + j;
      float v = st[(size_t)(y - g.ra) * Wp + x];
      if (pl.clamp_one) v = fminf(v, 1.0f);
      return make_key(__float_as_uint(v), cbase + (uint32_t)(y * W + x));
    };
    // while no threshold exists yet, expand an eighth of the unit at a time so it appears early
    const int wpr = (*s_thr == 0u && thr64 == 0ull) ? max((words + 7) >> 3, 16) : words;
    for (int base = 0; base < words; base += wpr) {
      const int end = min(base + wpr, words);
      __syncthreads();  // masks complete / previous round (and its threshold update) done
      const int n0 = s_cnt[0];
      const uint32_t tb = *s_thr;
      for (int t = base + tid; t < end; t += SEL_THREADS) {
        uint32_t m = masks[t];
        while (m) {
          const int bit = __ffs(m) - 1;
          m &= m - 1;
          const u64 key = make(t, bit);
          if (key_bits(key) >= tb && key > thr64) {
            const int hb = hist_bin(key_bits(key));
            atomicAdd(&fine[hb], 1);      // every qualifying candidate is counted exactly once
            atomicAdd(&coarse[hb >> 6], 1);
            const int slot = atomicAdd(&s_cnt[0], 1);
            if (slot < SEL_CAP) buf[slot] = key;
            else s_cnt[1] = 1;
          }
        }
      }
      __syncthreads();
      if (s_cnt[1]) {
        // overflow: drop this round's partial pushes and redo it exactly, in <=1024-candidate steps,
        // sort-pruning whenever a full step would not fit (K <= 1024 = CAP - 1024)
        __syncthreads();
        if (tid == 0) {
          s_cnt[0] = n0;
          s_cnt[1] = 0;
        }
        __syncthreads();
        for (int b2 = base; b2 < end; b2 += 32) {
          const bool full_soon = s_cnt[0] + 1024 > SEL_CAP;   // pushes of the previous step are complete
          __syncthreads();                                     // ...and none of this step start before all have read
          if (full_soon) thr64 = cta_prune(buf, s_cnt, K);
          const int word = b2 + (tid >> 5);
          if (word < end && ((masks[word] >> (tid & 31)) & 1u)) {
            const u64 key = make(word, tid & 31);
            if (key_bits(key) >= tb && key > thr64) buf[atomicAdd(&s_cnt[0], 1)] = key;
          }
          __syncthreads();
        }
      }
      if (warp == 0 && s_cnt[0] != s_cnt[5]) {  // new candidates: refresh the running threshold
        update_threshold(fine, coarse, lane, K, s_thr);
        if (lane == 0) s_cnt[5] = s_cnt[0];
      }
    }
    __syncthreads();  // everyone is done with this stage, the masks and the threshold update
    // the stage is free again: prefetch the unit that will reuse it
    if (TMA && tid == 0 && u + SEL_STAGES < total_units) issue(u + SEL_STAGES);
  }
  if (cur_img >= 0) flush(cur_img);
}

// ------------------------------------------------------------------ stage 1, hot geometry, warp-asynchronous
// Whole 128x128 planes, TMA, NMS, fused finalize, any batch size.  Within an image there is NO CTA-wide
// barrier:
//   * every warp waits for the plane (mbarrier), sweeps its 4 rows (phase A) and pushes its own
//     qualifying pixels straight from registers into the shared key buffer + histogram (atomics;
//     ~20-100 pushes per plane in steady state), then arrives on s_arr[stage];
//   * warp (u mod 32) additionally refreshes the histogram threshold and the LAST warp to finish unit u
//     re-arms the stage with the TMA load of unit u+3.
// Warps therefore drift apart by up to the depth of the stage ring and hide each other's latencies.
// CTA barriers exist only at image boundaries:
//   * bootstrap of the first plane of an image: pass 1 sweeps the plane WITHOUT a threshold and only
//     histograms its ~1.8 k peaks (one spread shared-memory atomic each, no key stores); the K-th best of
//     the plane becomes the threshold; pass 2 sweeps the (still resident) plane again and pushes the
//     ~1.0-1.3 K keys above it.  Two register-only sweeps instead of ~750 three-atomic pushes.
//   * flush: the buffer is cut against the final threshold and delivered UNSORTED (<= seg_cap keys) with
//     that threshold; the last CTA to deliver an image (atomic ticket) finalizes it.  An image that lies
//     entirely inside one CTA skips the global round trip and is finalized straight from shared memory
//     (_topk_channel planes, C = 1).
//   * finalize (finalize_hot): counts, thresholds and keys of all segments are fetched in ONE round of
//     independent L2 loads, cut with the largest segment threshold (a valid lower bound of the K-th
//     best), rank-sorted by 4 threads per key and emitted with the ctdet gathers fused.
// If the key buffer ever overflows (plateaus, very dense peaks) the CTA re-derives its segment of that
// image exactly from global memory at flush time (slow path, sort-prune).
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

#ifdef CNB_SELECT_STATS
// tuning build only (tools/select_stats.py rebuilds the library with -DCNB_SELECT_STATS): per CTA
// [total, wait, bootstrap, flush, finalize] cycles and [units, bootstraps, flushes, finalizes] counts
__device__ unsigned long long g_select_stats[SEL_MAX_CTA][10];
// per call (ring of SEL_TIME_CALLS launches, indexed by SelectPlan::stat_call) and CTA: %globaltimer (ns) at
// [entry, first stage ready, last plane swept, exit]; tools/decode_junction_time.py reads it
constexpr int SEL_TIME_CALLS = 64;
__device__ unsigned long long g_select_times[SEL_TIME_CALLS][SEL_MAX_CTA][4];
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define CNB_STAT(x) x
#else
#define CNB_STAT(x)
#endif

enum { SW_BOTH = 0, SW_HIST = 1, SW_KEYS = 2 };  // what a qualifying pixel updates: histogram and/or key buffer

// Finalize image b inside the hot kernel (all SEL_THREADS threads).  `local`: the keys are already in
// sbuf[0..n_local) (image owned by this CTA alone); otherwise they are merged from the `nslots` segments.
// sbuf holds SEL_CAP keys; s_fcnt holds >= nslots ints.
template <typename MapT>
__device__ void finalize_hot(const MapT *__restrict__ src, const SelectPlan &pl, int b, int nslots, bool local,
                             int n_local, const u64 *__restrict__ cand, const int *__restrict__ cand_cnt,
                             const uint32_t *__restrict__ cand_thr, const FinalizeOut &out, u64 *sbuf, int *s_fcnt,
                             int *s_tmp, u64 *s_red, int *fine, int *coarse) {
  const int tid = threadIdx.x, K = pl.K, cap = pl.seg_cap;
  int total;
  bool sorted = false;
  CNB_STAT(long long ph[6]; ph[0] = clock64(); ph[1] = ph[2] = ph[3] = ph[4] = ph[5] = ph[0];)
  if (local) {
    total = n_local;
  } else {
    const size_t base = (size_t)b * pl.max_slots;
    const u64 *keys = cand + base * (size_t)cap;   // the segments of one image are contiguous
    const int items = nslots * cap;
    // speculative key loads (independent of the counts, so counts + thresholds + keys cost ONE L2 round
    // trip; slots beyond a segment's count hold stale workspace bytes that are never used)
    u64 k0 = 0ull, k1 = 0ull;
    if (tid < items) k0 = __ldcg(keys + tid);
    if (tid + SEL_THREADS < items) k1 = __ldcg(keys + tid + SEL_THREADS);
    if (tid == 0) { s_tmp[0] = 0; s_tmp[1] = 0; s_tmp[2] = 0; }
    __syncthreads();
    for (int s = tid; s < nslots; s += SEL_THREADS) {
      s_fcnt[s] = __ldcg(cand_cnt + base + s);
      atomicMax(reinterpret_cast<unsigned int *>(&s_tmp[1]), __ldcg(cand_thr + base + s));
    }
    __syncthreads();
    // every segment threshold is a valid lower bound of the image's K-th best score (the K-th best of a
    // subset never exceeds the K-th best of the whole), hence so is the largest of them
    uint32_t T = (uint32_t)s_tmp[1];
    if (nslots > 8) {
      // small batches: an image is spread over many one-plane segments whose thresholds are all alike, so the
      // cut above still leaves thousands of keys.  One histogram pass over the (L2-resident) keys gives the
      // K-th best of the union to 1/128 octave; the second pass then keeps ~1.0-1.3 K keys.
      for (int i = tid; i < SEL_HIST_FINE + SEL_HIST_COARSE; i += SEL_THREADS) fine[i] = 0;
      __syncthreads();
      for (int it0 = 0; it0 < items; it0 += 4 * SEL_THREADS) {
        u64 kk[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int it = it0 + q * SEL_THREADS + tid;
          kk[q] = (it < items) ? __ldcg(keys + it) : 0ull;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int it = it0 + q * SEL_THREADS + tid;
          if (it < items) {
            const int slot = it / cap, j = it - slot * cap;
            if (j < s_fcnt[slot] && key_bits(kk[q]) >= T) atomicAdd(&fine[hist_bin(key_bits(kk[q]))], 1);
          }
        }
      }
      __syncthreads();
      {
        const int warp = tid >> 5, lane = tid & 31;
        int sum = fine[warp * 64 + lane] + fine[warp * 64 + 32 + lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) coarse[warp] = sum;
      }
      __syncthreads();
      if (tid < 32) update_threshold(fine, coarse, tid, K, reinterpret_cast<uint32_t *>(&s_tmp[3]));
      __syncthreads();
      T = max(T, (uint32_t)s_tmp[3]);
      __syncthreads();
    }
    auto take = [&](u64 key, int it) {   // called by whole warps: one shared-memory atomic per warp, not per key
      const int slot = it / cap, j = it - slot * cap;
      const bool ok = it < items && j < s_fcnt[slot] && key_bits(key) >= T;
      const uint32_t bal = __ballot_sync(0xffffffffu, ok);
      if (bal) {
        const int lane_ = tid & 31, leader = __ffs(bal) - 1;
        int base_pos = 0;
        if (lane_ == leader) base_pos = atomicAdd(&s_tmp[0], __popc(bal));
        base_pos = __shfl_sync(0xffffffffu, base_pos, leader);
        if (ok) {
          const int pos = base_pos + __popc(bal & ((1u << lane_) - 1u));
          if (pos < SEL_CAP) sbuf[pos] = key;
          else s_tmp[2] = 1;
        }
      }
    };
    CNB_STAT(ph[1] = clock64();)
    take(k0, tid);
    take(k1, tid + SEL_THREADS);
    for (int it0 = 2 * SEL_THREADS; it0 < items; it0 += 4 * SEL_THREADS) {   // small batches: many slots
      u64 kk[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int it = it0 + q * SEL_THREADS + tid;
        kk[q] = (it < items) ? __ldcg(keys + it) : 0ull;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) take(kk[q], it0 + q * SEL_THREADS + tid);
    }
    __syncthreads();
    total = s_tmp[0];
    if (s_tmp[2]) {
      // more than SEL_CAP keys above the cut (plateaus spanning many segments): exact chunked sort-prune
      __syncthreads();
      if (tid == 0) s_tmp[0] = 0;
      __syncthreads();
      u64 thr64 = 0ull;
      const int per = max(1, (SEL_CAP / 2) / cap);   // slots per step: <= CAP/2 new keys + <= K kept
      for (int s0 = 0; s0 < nslots; s0 += per) {
        const int s1 = min(nslots, s0 + per);
        for (int it = s0 * cap + tid; it < s1 * cap; it += SEL_THREADS) {
          const int slot = it / cap, j = it - slot * cap;
          if (j < s_fcnt[slot]) {
            const u64 key = __ldcg(keys + it);
            if (key > thr64) sbuf[atomicAdd(&s_tmp[0], 1)] = key;
          }
        }
        thr64 = cta_prune(sbuf, &s_tmp[0], K);
      }
      total = min(s_tmp[0], K);
      sorted = true;
    }
  }
  CNB_STAT(ph[2] = clock64();)
  const u64 *res = sbuf;
  if (!sorted && total > 256 && total <= SEL_CAP / 2) {
    // too many for the rank sort: one more cut, by a histogram of the keys already in shared memory (the K-th
    // best to 1/128 octave leaves ~1.0-1.3 K keys); far cheaper than a 512- or 1024-key bitonic sort
    for (int i = tid; i < SEL_HIST_FINE + SEL_HIST_COARSE; i += SEL_THREADS) fine[i] = 0;
    __syncthreads();
    for (int t = tid; t < total; t += SEL_THREADS) atomicAdd(&fine[hist_bin(key_bits(sbuf[t]))], 1);
    __syncthreads();
    {
      const int warp = tid >> 5, lane = tid & 31;
      int sum = fine[warp * 64 + lane] + fine[warp * 64 + 32 + lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      if (lane == 0) coarse[warp] = sum;
    }
    if (tid == 0) s_tmp[0] = 0;
    __syncthreads();
    if (tid < 32) update_threshold(fine, coarse, tid, K, reinterpret_cast<uint32_t *>(&s_tmp[3]));
    __syncthreads();
    const uint32_t t2 = (uint32_t)s_tmp[3];
    u64 *dst = sbuf + SEL_CAP / 2;
    for (int t = tid; t < total; t += SEL_THREADS) {
      const u64 key = sbuf[t];
      if (key_bits(key) >= t2) dst[atomicAdd(&s_tmp[0], 1)] = key;
    }
    __syncthreads();
    total = s_tmp[0];
    for (int t = tid; t < total; t += SEL_THREADS) sbuf[t] = dst[t];
    __syncthreads();
  }
  if (!sorted) {
    if (total <= 256) {
      // few survivors: rank sort, 4 threads per key (every key counts the keys above it; keys are unique).  The
      // key's owner issues its reg / wh gathers BEFORE counting -- they depend on the key, not on its rank -- so
      // the L2 round trip runs under the sort, and the owner of a key ranked < K writes its row directly.
      u64 *dst = sbuf + SEL_CAP / 2;
      const int q = tid >> 2, part = tid & 3;
      const u64 mine = (q < total) ? sbuf[q] : 0ull;
      RowGather rg = {0.5f, 0.5f, 0.f, 0.f};
      if (q < total && part == 0 && total >= K) rg = gather_row(pl, b, mine, out);
      int r0 = 0, r1 = 0, r2 = 0, r3 = 0;
      if (q < total) {
        int t = part;
        for (; t + 12 < total; t += 16) {
          r0 += (sbuf[t] > mine) ? 1 : 0;
          r1 += (sbuf[t + 4] > mine) ? 1 : 0;
          r2 += (sbuf[t + 8] > mine) ? 1 : 0;
          r3 += (sbuf[t + 12] > mine) ? 1 : 0;
        }
        for (; t < total; t += 4) r0 += (sbuf[t] > mine) ? 1 : 0;
      }
      int rank = (r0 + r1) + (r2 + r3);
      rank += __shfl_xor_sync(0xffffffffu, rank, 1);
      rank += __shfl_xor_sync(0xffffffffu, rank, 2);
      if (total >= K) {
        if (q < total && part == 0 && rank < K) emit_one(pl, b, rank, mine, out, rg);
        __syncthreads();
        return;
      }
      for (int t = total + tid; t < max(total, K); t += SEL_THREADS) dst[t] = 0ull;
      if (q < total && part == 0) dst[rank] = mine;
      __syncthreads();
      res = dst;
    } else {
      const int n = next_pow2(max(total, K));
      for (int t = total + tid; t < n; t += SEL_THREADS) sbuf[t] = 0ull;
      __syncthreads();
      cta_sort_desc(sbuf, n);
    }
  }
  CNB_STAT(ph[3] = clock64();)
  if (total < K) {
    const long long N = (long long)pl.C * pl.H * pl.W;
    finalize_fill<true, CtaGroup>(src + (long long)b * N, pl, const_cast<u64 *>(res), total, K, s_tmp, s_red);
  }
  CNB_STAT(ph[4] = clock64();)
  emit_rows<CtaGroup>(pl, b, res, out);
  __syncthreads();
#ifdef CNB_SELECT_STATS
  if (tid == 0 && !local && b == 7) {
    unsigned long long *d = g_select_stats[SEL_MAX_CTA - 1];
    ph[5] = clock64();
    d[0] = ph[1] - ph[0]; d[1] = ph[2] - ph[1]; d[2] = ph[3] - ph[2]; d[3] = ph[4] - ph[3]; d[4] = ph[5] - ph[4];
    d[5] = (unsigned long long)total; d[6] = (unsigned long long)nslots;
  }
#endif
}

// Stage ring of the hot kernel for map element type T: SEL_STAGES stages of one whole 128x128 plane each (64 KiB
// for fp32, 32 KiB for fp16 / bf16; DESIGN 4.1 has the measurement behind 3 half-size stages rather than 6).
template <typename T>
constexpr size_t hot_smem_bytes() {
  return (size_t)SEL_STAGES * (128 * 128 * sizeof(T)) + (size_t)SEL_CAP * 8 +
         (size_t)(SEL_HIST_FINE + SEL_HIST_COARSE) * 4 + (size_t)SEL_MASK_WORDS * 4 + SEL_STAGES * 8 + 32;
}

template <typename T, bool LOGITS>
__global__ void __launch_bounds__(SEL_THREADS, 1)
k_select_hot(const T *__restrict__ src, const SelectPlan pl, u64 *__restrict__ cand, int *__restrict__ cand_cnt,
             int *__restrict__ img_done, uint32_t *__restrict__ cand_thr, const FinalizeOut fout) {
  constexpr uint32_t PLANE_BYTES = 128 * 128 * sizeof(T);
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T *stages = reinterpret_cast<T *>(smem_raw);
  u64 *buf = reinterpret_cast<u64 *>(smem_raw + (size_t)SEL_STAGES * PLANE_BYTES);
  int *fine = reinterpret_cast<int *>(buf + SEL_CAP);
  int *coarse = fine + SEL_HIST_FINE;
  int *s_fcnt = reinterpret_cast<int *>(coarse + SEL_HIST_COARSE);   // SEL_MASK_WORDS (512) ints >= SEL_MAX_CTA
  uint64_t *full = reinterpret_cast<uint64_t *>(s_fcnt + SEL_MASK_WORDS);
  int *s_cnt = reinterpret_cast<int *>(full + SEL_STAGES);   // [0] count [1] overflow [2] last flag [3] compaction
  uint32_t *s_thr = reinterpret_cast<uint32_t *>(s_cnt + 4);
  float *s_tl = reinterpret_cast<float *>(s_cnt + 5);        // LOGITS: logit-space lower bound of *s_thr
  __shared__ int s_arr[SEL_STAGES];                          // warps done with the stage (last one re-arms it)
  __shared__ int s_flag[4];                                  // compaction rendezvous requested for unit (u & 3)
  __shared__ uint32_t s_exact;                               // score bits of an exact K-th best (0: none yet)
  __shared__ int s_tmp[32];
  __shared__ u64 s_red[32];
  static_assert(SEL_MASK_WORDS >= SEL_MAX_CTA, "s_fcnt must hold one count per candidate segment");
  static_assert(SEL_HIST_FINE == 64 * SEL_WARPS, "bootstrap derives one coarse bin per warp");

  CNB_STAT(unsigned long long tm[4]; tm[0] = global_ns(); tm[1] = tm[2] = tm[3] = 0ull;)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = pl.K, C = pl.C;
  constexpr int HW = 128 * 128;
  const int me = (int)blockIdx.x;
  const long long p_begin = plan_first_plane(pl, me);
  const long long p_end = plan_first_plane(pl, me + 1);
  const int total_units = (int)(p_end - p_begin);
  const float NI = CNB_NEG_INF;

  auto issue = [&](int u) {  // one lane
    const int s = u % SEL_STAGES;
    const char *gsrc = reinterpret_cast<const char *>(src + (p_begin + u) * (long long)HW);
    char *dst = reinterpret_cast<char *>(stages) + (size_t)s * PLANE_BYTES;
    mbar_expect_tx(&full[s], PLANE_BYTES);
#pragma unroll
    for (uint32_t off = 0; off < PLANE_BYTES; off += 16384u)
      bulk_g2s(dst + off, gsrc + off, 16384u, &full[s]);
  };
  auto clear_hist = [&]() {
    for (int i = tid; i < SEL_HIST_FINE + SEL_HIST_COARSE; i += SEL_THREADS) fine[i] = 0;
  };
  auto clear_scalars = [&]() {  // tid 0
    s_cnt[0] = 0; s_cnt[1] = 0; s_cnt[2] = 0; s_cnt[3] = 0;
    *s_thr = 0u;
    *s_tl = CNB_NEG_INF;
    s_exact = 0u;
  };
  // one warp: refresh the histogram threshold (and its logit-space image)
  auto refresh_thr = [&]() {
    update_threshold(fine, coarse, lane, K, s_thr);
    if (lane == 0) {
      const uint32_t ex = *(volatile uint32_t *)&s_exact;      // exact K-th best of an earlier sort-prune, if any
      if (ex > *s_thr) *s_thr = ex;
      if (LOGITS) *s_tl = logit_lower_bound(*s_thr);
    }
  };

  // Programmatic dependent launch (launch_hot): the next launch on the stream may start as soon as every CTA of this
  // one is resident; each of its CTAs then takes an SM as one of ours leaves it.  Before griddepcontrol.wait (in
  // flush) a CTA only issues TMA loads of its map and sweeps them in shared memory: the map is never written by this
  // kernel, and any other kernel between two hot launches does not trigger early, so plain stream order holds across
  // it.  Segments, counts, thresholds, tickets and dets are touched only after the wait, i.e. after the previous
  // launch has completed and its writes (its ticket resets included) are visible.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (tid == 0) {
    s_flag[0] = s_flag[1] = s_flag[2] = s_flag[3] = 0;
    for (int s = 0; s < SEL_STAGES; ++s) {
      mbar_init(&full[s], 1);
      s_arr[s] = 0;
    }
    mbar_fence_init();
    clear_scalars();
    for (int u = 0; u < SEL_STAGES && u < total_units; ++u) issue(u);
  }
  clear_hist();
  // First / last CTA of the first / last image this CTA touches (every image in between starts and ends
  // inside this CTA's range): two binary searches over the plan, hidden behind the first TMA load.
  const int img_lo = (int)(p_begin / C), img_hi = (int)((p_end - 1) / C);
  if (tid == 32) s_tmp[26] = plan_cta_of_plane(pl, (long long)img_lo * C);
  if (tid == 64) s_tmp[27] = plan_cta_of_plane(pl, (long long)(img_hi + 1) * C - 1);
  __syncthreads();
  const int i0_first = s_tmp[26], i1_last = s_tmp[27];
  CNB_STAT(if (tid == 0) { s_tmp[24] = 0; s_tmp[25] = 0; })

  // one qualifying pixel (any lane of any warp, concurrently)
  auto push = [&](float v, uint32_t flat, int mode) {
    if (pl.clamp_one) v = fminf(v, 1.0f);
    const uint32_t bits = __float_as_uint(v);
    if (mode != SW_KEYS) {
      const int hb = hist_bin(bits);
      atomicAdd(&fine[hb], 1);
      if (mode == SW_BOTH) atomicAdd(&coarse[hb >> 6], 1);
    }
    if (mode != SW_HIST) {
      const int slot = atomicAdd(&s_cnt[0], 1);
      if (slot < SEL_CAP) buf[slot] = make_key(bits, flat);
      else s_cnt[1] = 1;
    }
  };

  // LOGITS: pixel with logit b whose 3x3 logit maximum is M
  auto try_push_logit = [&](float b, float M, uint32_t flat, int mode) {
    bool pk = (b == M);
    if (!pk && (M - b) <= collide_margin(M)) pk = (sigmoid_ref(b) == sigmoid_ref(M));
    if (pk) {
      const float sv = sigmoid_ref(b);
      if (sv > 0.0f) push(sv, flat, mode);
    }
  };

  // ---- CTA-wide compaction of the key buffer against the current threshold (rendezvous, rare)
  auto compact = [&](int slot_idx) {
    __syncthreads();
    if (slot_idx >= 0) {     // mid-stream rendezvous: bring the threshold up to date first (flush: already is)
      if (warp == 0) refresh_thr();
      __syncthreads();
    }
    const uint32_t tb = *s_thr;
    const bool fits = s_cnt[0] <= SEL_CAP;       // read once here, while nobody modifies it
    const int cnt = min(s_cnt[0], SEL_CAP);
    u64 mine[SEL_CAP / SEL_THREADS];
#pragma unroll
    for (int j = 0; j < SEL_CAP / SEL_THREADS; ++j) {
      const int t = tid + j * SEL_THREADS;
      mine[j] = (t < cnt) ? buf[t] : 0ull;
    }
    __syncthreads();
    if (tid == 0) {
      if (fits) s_cnt[0] = 0;                  // an overflowed buffer stays flagged; flush rescans
      if (slot_idx >= 0) s_flag[slot_idx] = 0;
    }
    __syncthreads();
    if (fits) {
#pragma unroll
      for (int j = 0; j < SEL_CAP / SEL_THREADS; ++j) {   // warp-aggregated append: one shared atomic per warp
        const bool ok = mine[j] != 0ull && key_bits(mine[j]) >= tb;
        const uint32_t bal = __ballot_sync(0xffffffffu, ok);
        if (bal) {
          const int leader = __ffs(bal) - 1;
          int base_pos = 0;
          if (lane == leader) base_pos = atomicAdd(&s_cnt[0], __popc(bal));
          base_pos = __shfl_sync(0xffffffffu, base_pos, leader);
          if (ok) buf[base_pos + __popc(bal & ((1u << lane) - 1u))] = mine[j];
        }
      }
    }
    __syncthreads();
    if (fits && s_cnt[0] > SEL_CAP / 2) {
      // the histogram cannot separate them (many candidates inside one 1/128-octave bin: flat noise floors,
      // plateaus): cut exactly -- sort, keep the K best, and raise the threshold to the K-th best score itself
      const u64 kth = cta_prune(buf, s_cnt, K);
      if (tid == 0 && kth != 0ull) {
        s_exact = max(s_exact, key_bits(kth));
        *s_thr = max(*s_thr, s_exact);
        if (LOGITS) *s_tl = logit_lower_bound(*s_thr);
      }
      __syncthreads();
    }
  };

  // ---- CTA-wide flush of image `img` (all threads; called at image boundaries only)
  auto flush = [&](int img) {
    // before the CTA's first global write or workspace read (see the launch note above); returns at once after the
    // first flush
    asm volatile("griddepcontrol.wait;" ::: "memory");
    __syncthreads();
    int n_out;
    if (s_cnt[1]) {
      // the buffer overflowed at some point: rebuild this CTA's segment exactly from global memory
      __syncthreads();
      if (tid == 0) s_cnt[0] = 0;
      __syncthreads();
      u64 thr64 = 0ull;
      const long long lo = max(p_begin, (long long)img * C), hi = min(p_end, (long long)(img + 1) * C);
      const T *ibase = src + (long long)img * C * HW;
      for (long long p = lo; p < hi; ++p) {
        const int c = (int)(p - (long long)img * C);
        for (int base = 0; base < HW; base += SEL_THREADS) {
          const bool full_soon = s_cnt[0] + SEL_THREADS > SEL_CAP;   // previous step's pushes are complete
          __syncthreads();                                            // uniform branch: no push before all have read
          if (full_soon) thr64 = cta_prune(buf, s_cnt, K);
          const long long flat = (long long)c * HW + base + tid;
          float v = nms_value<true>(ibase, C, 128, 128, flat, LOGITS);
          if (pl.clamp_one) v = fminf(v, 1.0f);
          if (v > 0.0f) {
            const u64 key = make_key(__float_as_uint(v), (uint32_t)flat);
            if (key > thr64) buf[atomicAdd(&s_cnt[0], 1)] = key;
          }
          __syncthreads();
        }
      }
      cta_prune(buf, s_cnt, K);
      n_out = min(s_cnt[0], K);
    } else {
      if (s_cnt[0] > pl.seg_cap) compact(-1);     // drop everything below the histogram threshold (>= K survive)
      else {
        if (warp == 0) refresh_thr();
        __syncthreads();
      }
      const int cnt = s_cnt[0];
      n_out = cnt;                                  // deliver unsorted: finalize sorts anyway
      if (cnt > pl.seg_cap) {                       // still too many (ties in the threshold bin): exact cut
        cta_prune(buf, s_cnt, K);
        n_out = min(cnt, K);
      }
    }
    const int i0 = (img == img_lo) ? i0_first : me;
    const int i1 = (img == img_hi) ? i1_last : me;
    if (i0 == i1) {
      // the image lies entirely in this CTA: no segment, no ticket -- finalize from shared memory
      finalize_hot(src, pl, img, 1, true, n_out, cand, cand_cnt, cand_thr, fout, buf, s_fcnt, s_tmp, s_red, fine, coarse);
      clear_hist();
      if (tid == 0) clear_scalars();
      __syncthreads();
      return;
    }
    const int slot = me - i0;
    u64 *dst = cand + ((size_t)img * pl.max_slots + slot) * pl.seg_cap;
    for (int t = tid; t < n_out; t += SEL_THREADS) dst[t] = buf[t];
    if (tid == 0) {
      cand_cnt[(size_t)img * pl.max_slots + slot] = n_out;
      // histogram threshold = valid lower bound of the image's K-th best (0 after an exact rebuild)
      cand_thr[(size_t)img * pl.max_slots + slot] = s_cnt[1] ? 0u : *s_thr;
    }
    __threadfence();
    __syncthreads();
    int ticket = 0;
    if (tid == 0) ticket = atomicAdd(&img_done[img], 1);   // in flight while the histogram is cleared
    clear_hist();
    if (tid == 0) {
      s_cnt[2] = (ticket == i1 - i0) ? 1 : 0;
      // last ticket: every other CTA of this image has drawn its own, so the ticket is free again for the next launch
      if (s_cnt[2]) img_done[img] = 0;
    }
    __syncthreads();
    if (s_cnt[2]) {  // every segment of this image is in global memory: merge + emit here
      __threadfence();
      CNB_STAT(const long long fq = clock64();)
      CNB_STAT(if (tid == 0) { s_tmp[24] += 1; })
      finalize_hot(src, pl, img, i1 - i0 + 1, false, 0, cand, cand_cnt, cand_thr, fout, buf, s_fcnt, s_tmp, s_red, fine,
                   coarse);
      clear_hist();   // the many-segment finalize borrows the histogram
      CNB_STAT(if (tid == 0) { s_tmp[25] += (int)(clock64() - fq); })
    }
    if (tid == 0) clear_scalars();
    __syncthreads();
  };

  // ---- phase A + push of rows [y0, y0 + 4) of the plane in stage `st`
  // Per row: 4 vertical FMNMX3, 2 SHFL, 2 FADD (lane-edge -inf, keeps the ALU pipe free), the
  // horizontal max with the running threshold folded in, 4 compares and one (rarely taken) branch.
  const float edge_l = (lane == 0) ? NI : 0.0f, edge_r = (lane == 31) ? NI : 0.0f;
  // T = fp16 / bf16: a lane loads 4 elements (8 bytes) per row and widens them; everything after the load is the
  // fp32 sweep.
  auto sweep = [&](const T *st, int c, int mode) {
    const bool use_thr = (mode != SW_HIST);
    const int y0 = warp * 4;
    const T *p = st + (size_t)y0 * 128 + lane * 4;
    typename Raw4<T>::type r_[6];
    r_[0] = (y0 > 0) ? ld_raw4(p - 128) : raw4_ninf<T>();
#pragma unroll
    for (int i = 0; i < 4; ++i) r_[i + 1] = ld_raw4(p + i * 128);
    r_[5] = (y0 + 4 < 128) ? ld_raw4(p + 4 * 128) : raw4_ninf<T>();
    const uint32_t fbase = (uint32_t)c * (uint32_t)HW + (uint32_t)(y0 * 128 + lane * 4);
    float lane_best = LOGITS ? NI : 0.0f;   // SW_HIST: best peak among this lane's 16 pixels
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // threshold >= smallest positive float, so `b == max(.., thr)` also rejects b <= 0; it is
      // re-read per row (one broadcast LDS): fresher threshold = fewer pushes
      const float4 a = widen4<T>(r_[i]), b = widen4<T>(r_[i + 1]), cc = widen4<T>(r_[i + 2]);
      const float v0 = fmax3(a.x, b.x, cc.x), v1 = fmax3(a.y, b.y, cc.y);
      const float v2 = fmax3(a.z, b.z, cc.z), v3 = fmax3(a.w, b.w, cc.w);
      const float l = __shfl_up_sync(0xffffffffu, v3, 1) + edge_l;
      const float r = __shfl_down_sync(0xffffffffu, v0, 1) + edge_r;
      if (mode == SW_HIST) {
        // bootstrap pass 1: no pushes, no divergence -- every lane just remembers its best peak (a logit peak is
        // a heat peak: the sigmoid is monotone)
        const float m01 = fmaxf(v0, v1), m23 = fmaxf(v2, v3);
        const float floor_ = LOGITS ? NI : 0.0f;
        const float c0 = (b.x == fmax3(l, m01, b.x)) ? b.x : floor_;
        const float c1 = (b.y == fmax3(m01, v2, b.y)) ? b.y : floor_;
        const float c2 = (b.z == fmax3(v1, m23, b.z)) ? b.z : floor_;
        const float c3 = (b.w == fmax3(m23, r, b.w)) ? b.w : floor_;
        lane_best = fmaxf(lane_best, fmaxf(fmaxf(c0, c1), fmaxf(c2, c3)));
        continue;
      }
      if (LOGITS) {
        // logit space: one compare per pixel against the logit image of the threshold; the (rare)
        // survivors are peak-tested exactly: b is a heat peak iff sigmoid(b) == sigmoid(3x3 max)
        const float tl = use_thr ? *(volatile float *)s_tl : NI;
        const bool q0 = b.x >= tl, q1 = b.y >= tl, q2 = b.z >= tl, q3 = b.w >= tl;
        if (q0 | q1 | q2 | q3) {
          const uint32_t f = fbase + (uint32_t)(i * 128);
          if (q0) try_push_logit(b.x, fmax3(l, v0, v1), f, mode);
          if (q1) try_push_logit(b.y, fmax3(v0, v1, v2), f + 1, mode);
          if (q2) try_push_logit(b.z, fmax3(v1, v2, v3), f + 2, mode);
          if (q3) try_push_logit(b.w, fmax3(v2, v3, r), f + 3, mode);
        }
        continue;
      }
      const float thr_f = __uint_as_float(use_thr ? max(*(volatile uint32_t *)s_thr, 1u) : 1u);
      const float m01 = fmaxf(v0, v1), m23 = fmaxf(v2, v3);
      const bool q0 = (b.x == fmax3(l, m01, thr_f));
      const bool q1 = (b.y == fmax3(m01, v2, thr_f));
      const bool q2 = (b.z == fmax3(v1, m23, thr_f));
      const bool q3 = (b.w == fmax3(m23, r, thr_f));
      if (q0 | q1 | q2 | q3) {  // rare: a few pixels per plane once the threshold exists
        const uint32_t f = fbase + (uint32_t)(i * 128);
        if (q0) push(b.x, f, mode);
        if (q1) push(b.y, f + 1, mode);
        if (q2) push(b.z, f + 2, mode);
        if (q3) push(b.w, f + 3, mode);
      }
    }
    if (mode == SW_HIST) {
      // one histogram entry per lane: the K-th largest of these <= 1024 lane maxima is a valid lower bound of the
      // plane's K-th best peak (each is a distinct real peak), about the top 7 % of its ~1.8 k peaks
      float v = LOGITS ? sigmoid_ref(lane_best) : lane_best;
      if (pl.clamp_one) v = fminf(v, 1.0f);
      if (v > 0.0f) atomicAdd(&fine[hist_bin(__float_as_uint(v))], 1);
    }
  };

  int img = img_lo, c = (int)(p_begin - (long long)img * C);
  int stage = 0, par = 0;
  bool fresh = true;  // first unit of an image in this CTA (CTA-uniform)
  CNB_STAT(long long st_t0 = clock64(); long long st_wait = 0; long long st_boot = 0; long long st_flush = 0;
           int st_nboot = 0; int st_nflush = 0; long long st_q;)
  for (int u = 0; u < total_units; ++u) {
    const T *st = stages + (size_t)stage * (128 * 128);
    CNB_STAT(st_q = clock64();)
    mbar_wait(&full[stage], (uint32_t)par);
    CNB_STAT(st_wait += clock64() - st_q; st_q = clock64(); if (u == 0) tm[1] = global_ns();)
    if (*(volatile int *)&s_flag[u & 3]) compact(u & 3);   // set 3 units ago, before this plane's TMA was issued
    if (fresh) {
      // bootstrap (see header): histogram-only pass, K-th best of the plane, key pass
      sweep(st, c, SW_HIST);
      __syncthreads();
      {  // one coarse bin per warp: sum of its 64 fine bins
        int sum = fine[warp * 64 + lane] + fine[warp * 64 + 32 + lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) coarse[warp] = sum;
      }
      __syncthreads();
      if (warp == 0) refresh_thr();
      __syncthreads();
      sweep(st, c, SW_KEYS);
      fresh = false;
      CNB_STAT(st_boot += clock64() - st_q; ++st_nboot;)
    } else {
      sweep(st, c, SW_BOTH);
      if (warp == (u & (SEL_WARPS - 1))) refresh_thr();  // partial counts are valid too
    }
    __syncwarp();
    if (lane == 0) {
      // last warp to finish this stage re-arms it (no waiting): TMA load of unit u+3
      __threadfence_block();
      if (atomicAdd(&s_arr[stage], 1) == SEL_WARPS - 1) {
        s_arr[stage] = 0;
        if (u + SEL_STAGES < total_units) {
          // buffer half full: ask every warp to rendezvous at unit u+3 (nobody can start it before
          // the TMA below is issued, so all of them will see the flag)
          if (*(volatile int *)&s_cnt[0] > SEL_CAP / 2) s_flag[(u + SEL_STAGES) & 3] = 1;
          issue(u + SEL_STAGES);
        }
      }
    }
    // next unit
    CNB_STAT(st_q = clock64(); if (u == total_units - 1) tm[2] = global_ns();)
    if (++c == C) {
      flush(img);
      c = 0;
      ++img;
      fresh = true;
      CNB_STAT(st_flush += clock64() - st_q; ++st_nflush;)
    } else if (u == total_units - 1) {
      flush(img);
      CNB_STAT(st_flush += clock64() - st_q; ++st_nflush;)
    }
    if (++stage == SEL_STAGES) { stage = 0; par ^= 1; }
  }
#ifdef CNB_SELECT_STATS
  if (tid == 0) {
    unsigned long long *d = g_select_stats[me];
    d[0] = (unsigned long long)(clock64() - st_t0); d[1] = (unsigned long long)st_wait; d[2] = (unsigned long long)st_boot;
    d[3] = (unsigned long long)st_flush; d[4] = (unsigned long long)s_tmp[25]; d[5] = (unsigned long long)total_units;
    d[6] = (unsigned long long)st_nboot; d[7] = (unsigned long long)st_nflush; d[8] = (unsigned long long)s_tmp[24];
    unsigned int smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    d[9] = smid;
    tm[3] = global_ns();
    unsigned long long *t = g_select_times[pl.stat_call % SEL_TIME_CALLS][me];
    t[0] = tm[0]; t[1] = tm[1]; t[2] = tm[2]; t[3] = tm[3];
  }
#endif
}

// ------------------------------------------------------------------ separate finalize kernel
template <bool NMS>
__global__ void __launch_bounds__(1024, 1)
k_select_finalize(const float *__restrict__ src, const SelectPlan pl, const u64 *__restrict__ cand,
                  const int *__restrict__ cand_cnt, const FinalizeOut out) {
  extern __shared__ __align__(16) unsigned char fin_raw[];
  u64 *sbuf = reinterpret_cast<u64 *>(fin_raw);
  __shared__ int s_tmp[32];
  __shared__ u64 s_red[32];
  finalize_image<NMS, CtaGroup>(src, pl, blockIdx.x, cand, cand_cnt, out, sbuf, s_tmp, s_red);
}

// ------------------------------------------------------------------ host
static size_t stage1_smem_bytes() {
  return (size_t)SEL_STAGES * SEL_STAGE_BYTES + (size_t)SEL_CAP * 8 +
         (size_t)(SEL_HIST_FINE + SEL_HIST_COARSE) * 4 + (size_t)SEL_MASK_WORDS * 4 + SEL_STAGES * 8 + 32;
}


int make_select_plan(const void *src, int n_img, int C, int H, int W, int K, int nms, SelectPlan *pl, int elem_size) {
  CNB_REQUIRE(n_img > 0 && C > 0 && H > 0 && W > 0 && K > 0, CNB_EINVAL,
              "top-k: non-positive dimension (n_img=%d c=%d h=%d w=%d k=%d)", n_img, C, H, W, K);
  CNB_REQUIRE((long long)K <= (long long)H * W, CNB_EINVAL,
              "top-k: k=%d exceeds h*w=%lld (torch.topk would raise, decode.py:106)", K, (long long)H * W);
  CNB_REQUIRE(K <= SEL_MAX_K, CNB_EUNSUPPORTED, "top-k: k=%d > %d not implemented", K, SEL_MAX_K);
  CNB_REQUIRE((long long)C * H * W < (1ll << 32), CNB_EUNSUPPORTED, "top-k: c*h*w must be < 2^32");
  pl->n_img = n_img; pl->C = C; pl->H = H; pl->W = W; pl->K = K; pl->nms = nms;
  pl->clamp_one = 0;
  pl->logits = 0;
  pl->Wp = (W + 3) / 4 * 4;
  pl->ncb = (W + 127) / 128;
  pl->P = (long long)n_img * C;
  // rows of whole 16-byte chunks from a 16-byte aligned base
  pl->use_tma = ((long long)W * elem_size % 16 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0);
  const int max_rows = SEL_STAGE_BYTES / (pl->Wp * 4);
  CNB_REQUIRE(max_rows >= 3 && pl->ncb <= 32, CNB_EUNSUPPORTED, "top-k: w=%d too wide for a 64 KiB stage", W);
  int rb_cap = SEL_MASK_WORDS / (4 * pl->ncb);
  if (H <= max_rows && H <= rb_cap) {
    pl->rb = H;
  } else {
    pl->rb = max_rows - 2 < rb_cap ? max_rows - 2 : rb_cap;
  }
  pl->upp = (H + pl->rb - 1) / pl->rb;
  int n_cta = num_sms();
  if (n_cta > SEL_MAX_CTA) n_cta = SEL_MAX_CTA;
  if ((long long)n_cta > pl->P) n_cta = (int)pl->P;
  // hot geometry: whole 128x128 planes through the warp-asynchronous kernel with its own fused finalize
  // (any number of segments per image, so no grid shrinking).  An image boundary costs the crossing CTA a
  // flush + a bootstrap, about 2 planes' worth of cycles; only worth modelling when ranges are long.
  const bool hot_geom = nms && pl->use_tma && W == 128 && H == 128 && pl->rb == 128 && K <= 256;
  // small batches: a one-plane segment per CTA means ~80 loose segments per image for the finalizing CTA to merge;
  // three planes per CTA cost ~3 us more streaming and save more than that in the merge
  if (hot_geom && C > 1 && pl->P < 3ll * n_cta) n_cta = (int)((pl->P + 2) / 3);
  // An image boundary costs the crossing CTA a flush + a bootstrap (~12 k cycles), and -- being the slower one --
  // it usually is the last to deliver the image that ENDS in it, i.e. it also runs that image's finalize
  // (~10 k): 4 planes' worth of cycles balances best (swept 0..10 with tools/select_stats.py); long ranges only.
  int wb = 0;
  if (hot_geom && C > 1 && pl->P / n_cta >= 8) wb = 4;
#ifdef CNB_SELECT_STATS
  if (getenv("CNB_SELECT_WB") && hot_geom && C > 1 && pl->P / n_cta >= 8) wb = atoi(getenv("CNB_SELECT_WB"));
#endif
  for (;;) {
    Part q;
    q.P = pl->P; q.n_cta = n_cta; q.C = C; q.wb = wb;
    bool ok = true;
    for (int i = 0; i < n_cta && ok; ++i) ok = cta_first_plane(i + 1, q) > cta_first_plane(i, q);
    if (!ok) {  // weighted split produced an empty range: fall back to the plain split
      wb = 0;
      continue;
    }
    // segments an image can receive = CTAs whose range touches it; one sweep over the (monotone) ranges
    int ms = 1;
    {
      long long run_img = -1;
      int run_len = 0;
      for (int i = 0; i < n_cta; ++i) {
        const long long lo = cta_first_plane(i, q) / C, hi = (cta_first_plane(i + 1, q) - 1) / C;
        if (lo == run_img) ++run_len; else { run_img = lo; run_len = 1; }
        if (run_len > ms) ms = run_len;
        if (hi != lo) { run_img = hi; run_len = 1; }
      }
    }
    if (hot_geom || (long long)ms * K <= SEL_FIN_MAX || n_cta == 1) {
      pl->max_slots = ms;
      break;
    }
    n_cta = (n_cta * 3) / 4 > 0 ? (n_cta * 3) / 4 : 1;
  }
  pl->n_cta = n_cta;
  pl->wb = wb;
  {
    Part q;
    q.P = pl->P; q.n_cta = n_cta; q.C = C; q.wb = wb;
    for (int i = 0; i <= n_cta; ++i) pl->cta_start[i] = (int)cta_first_plane(i, q);
  }
  pl->fused_finalize = ((long long)pl->max_slots * K <= SEL_CAP) ? 1 : 0;
  pl->seg_cap = K;
  pl->hot = 0;
  if (hot_geom) {
    pl->hot = 1;
    pl->fused_finalize = 1;
    if (K <= 128) pl->seg_cap = 256;
  }
  return CNB_OK;
}

size_t select_workspace_bytes(const SelectPlan &pl) {
  const size_t keys = align_up((size_t)pl.n_img * pl.max_slots * (pl.seg_cap > 256 ? pl.seg_cap : 256) * 8, 256);
  const size_t cnts = align_up((size_t)pl.n_img * pl.max_slots * 4, 256);
  const size_t done = align_up((size_t)pl.n_img * 4, 256);
  return keys + cnts + done + cnts;  // + per-segment thresholds
}

size_t select_workspace_bytes_any_align(int n_img, int C, int H, int W, int K) {
  SelectPlan aligned, misaligned;
  if (make_select_plan(nullptr, n_img, C, H, W, K, 1, &aligned) != CNB_OK) return 0;
  if (make_select_plan(reinterpret_cast<const void *>(4), n_img, C, H, W, K, 1, &misaligned) != CNB_OK) return 0;
  const size_t a = select_workspace_bytes(aligned), m = select_workspace_bytes(misaligned);
  return a > m ? a : m;
}

template <bool NMS, bool TMA, int MODE>
static int launch_stage1(const float *src, const SelectPlan &pl, const FinalizeOut &out, u64 *cand, int *cnt,
                         int *done, cudaStream_t stream) {
  const size_t smem1 = stage1_smem_bytes();
  static thread_local int configured_dev = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (configured_dev != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_select_stage1<NMS, TMA, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem1));
    configured_dev = dev;
  }
  k_select_stage1<NMS, TMA, MODE><<<pl.n_cta, SEL_THREADS, smem1, stream>>>(src, pl, cand, cnt, done, out);
  CNB_CHECK_LAUNCH("select stage 1");
  count_launch();
  return CNB_OK;
}

// Tickets of the hot kernel: one int per image, owned by the library per (device, stream) and zero between launches.
// The CTA that draws an image's last ticket puts it back to 0, so every launch leaves the array as it found it and
// the next launch on the stream needs no memset.  The array is made (and zeroed) on first use and replaced by a
// larger zeroed one when a launch has more images; the old one is freed in stream order, so a launch still in flight
// keeps its tickets.  Keyed by cudaStreamGetId, not the handle: the legacy and per-thread default streams have
// fixed handles.
static std::mutex g_ticket_mu;
static std::map<std::pair<int, unsigned long long>, std::pair<int *, int>> g_tickets;   // -> (array, images)

static int hot_tickets(int n_img, cudaStream_t stream, int **out) {
  int dev = 0;
  unsigned long long sid = 0;
  CNB_CUDA(cudaGetDevice(&dev));
  CNB_CUDA(cudaStreamGetId(stream, &sid));
  std::lock_guard<std::mutex> lock(g_ticket_mu);
  std::pair<int *, int> &t = g_tickets[std::make_pair(dev, sid)];
  if (t.second < n_img) {
    const int n = std::max(n_img, std::max(2 * t.second, 256));
    int *p = nullptr;
    CNB_CUDA(cudaMallocAsync(reinterpret_cast<void **>(&p), (size_t)n * 4, stream));
    CNB_CUDA(cudaMemsetAsync(p, 0, (size_t)n * 4, stream));
    if (t.first) CNB_CUDA(cudaFreeAsync(t.first, stream));
    t = std::make_pair(p, n);
  }
  *out = t.first;
  return CNB_OK;
}

#ifdef CNB_SELECT_STATS
static std::atomic<int> g_hot_calls{0};   // hot launches so far (slot of the next one's timestamps)
#endif

// Launched with programmatic stream serialization: the kernel triggers its dependents at entry and waits for its
// predecessor grid before its first global write or workspace read (k_select_hot), so the next call's CTAs take
// each SM as this call's CTA leaves it and stream their planes under this call's tail.
template <typename T>
static int launch_hot(const void *src, const SelectPlan &pl, const FinalizeOut &out, u64 *cand, int *cnt,
                      uint32_t *thr, cudaStream_t stream) {
  constexpr size_t smem1 = hot_smem_bytes<T>();
  static thread_local int hot_dev = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (hot_dev != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_select_hot<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
    CNB_CUDA(cudaFuncSetAttribute(k_select_hot<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
    hot_dev = dev;
  }
  int *tickets = nullptr;
  const int rc = hot_tickets(pl.n_img, stream, &tickets);
  if (rc != CNB_OK) return rc;
  const T *s = reinterpret_cast<const T *>(src);
#ifdef CNB_SELECT_STATS
  SelectPlan pl_ = pl;
  pl_.stat_call = g_hot_calls.fetch_add(1);
  const SelectPlan &plx = pl_;
#else
  const SelectPlan &plx = pl;
#endif
  void (*kern)(const T *, SelectPlan, u64 *, int *, int *, uint32_t *, FinalizeOut) =
      pl.logits ? k_select_hot<T, true> : k_select_hot<T, false>;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(pl.n_cta);
  cfg.blockDim = dim3(SEL_THREADS);
  cfg.dynamicSmemBytes = smem1;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CNB_CUDA(cudaLaunchKernelEx(&cfg, kern, s, plx, cand, cnt, tickets, thr, out));
  CNB_CHECK_LAUNCH("select stage 1 (hot)");
  count_launch();
  return CNB_OK;
}

template <bool NMS>
static int launch_select(const void *src_v, int src_dtype, const SelectPlan &pl, const FinalizeOut &out, u64 *cand,
                         int *cnt, int *done, uint32_t *thr, cudaStream_t stream) {
  const float *src = reinterpret_cast<const float *>(src_v);   // every path but the hot one reads fp32
  const bool hot = NMS && pl.hot;
  if (pl.fused_finalize && !hot) CNB_CUDA(cudaMemsetAsync(done, 0, (size_t)pl.n_img * 4, stream));
  int rc;
  if (hot) {
    if (src_dtype == CNB_DTYPE_BF16) rc = launch_hot<__nv_bfloat16>(src_v, pl, out, cand, cnt, thr, stream);
    else if (src_dtype == CNB_DTYPE_F16) rc = launch_hot<__half>(src_v, pl, out, cand, cnt, thr, stream);
    else rc = launch_hot<float>(src_v, pl, out, cand, cnt, thr, stream);
  } else if (NMS && pl.use_tma && pl.W == 128 && pl.H == 128 && pl.rb == 128)
    rc = launch_stage1<NMS, true, 2>(src, pl, out, cand, cnt, done, stream);
  else if (pl.use_tma && pl.ncb == 1)
    rc = launch_stage1<NMS, true, 1>(src, pl, out, cand, cnt, done, stream);
  else if (pl.use_tma)
    rc = launch_stage1<NMS, true, 0>(src, pl, out, cand, cnt, done, stream);
  else
    rc = launch_stage1<NMS, false, 0>(src, pl, out, cand, cnt, done, stream);
  if (rc != CNB_OK) return rc;
  if (!pl.fused_finalize) {
    const size_t smem2 = (size_t)next_pow2(pl.max_slots * pl.seg_cap > pl.K ? pl.max_slots * pl.seg_cap : pl.K) * 8;
    CNB_CUDA(cudaFuncSetAttribute(k_select_finalize<NMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    k_select_finalize<NMS><<<pl.n_img, 1024, smem2, stream>>>(src, pl, cand, cnt, out);
    CNB_CHECK_LAUNCH("select finalize");
    count_launch();
  }
  return CNB_OK;
}

int run_select(const void *src, const SelectPlan &pl, const FinalizeOut &out, void *ws, cudaStream_t stream,
               int src_dtype) {
  CNB_REQUIRE(src_dtype == CNB_DTYPE_F32 || (pl.hot && pl.nms), CNB_EINVAL,
              "select: a 16-bit map needs the hot geometry (128x128 planes, k <= 256, 16-byte aligned)");
  char *p = reinterpret_cast<char *>(ws);
  u64 *cand = reinterpret_cast<u64 *>(p);
  p += align_up((size_t)pl.n_img * pl.max_slots * (pl.seg_cap > 256 ? pl.seg_cap : 256) * 8, 256);
  int *cnt = reinterpret_cast<int *>(p);
  p += align_up((size_t)pl.n_img * pl.max_slots * 4, 256);
  int *done = reinterpret_cast<int *>(p);
  p += align_up((size_t)pl.n_img * 4, 256);
  uint32_t *thr = reinterpret_cast<uint32_t *>(p);
  return pl.nms ? launch_select<true>(src, src_dtype, pl, out, cand, cnt, done, thr, stream)
                : launch_select<false>(src, src_dtype, pl, out, cand, cnt, done, thr, stream);
}

#ifdef CNB_SELECT_STATS
extern "C" int cnb_debug_select_stats(unsigned long long *out, int n_cta) {
  return cudaMemcpyFromSymbol(out, g_select_stats, sizeof(unsigned long long) * 10 * n_cta) == cudaSuccess ? 0 : 1;
}
// the whole timestamp ring, [SEL_TIME_CALLS][SEL_MAX_CTA][4]; returns the number of launches so far in *n_calls
extern "C" int cnb_debug_select_times(unsigned long long *out, int *n_calls, int *ring, int *max_cta) {
  *ring = SEL_TIME_CALLS;
  *max_cta = SEL_MAX_CTA;
  *n_calls = g_hot_calls.load();
  if (out == nullptr) return 0;
  return cudaMemcpyFromSymbol(out, g_select_times, sizeof(g_select_times)) == cudaSuccess ? 0 : 1;
}
#endif

}  // namespace cnb

extern "C" int cnb_select_plan_info(const void *src, int n_img, int C, int H, int W, int K, int nms, int elem_size,
                                    int *out, int n_out) {
  CNB_REQUIRE(out != nullptr && n_out >= 0, CNB_EINVAL, "cnb_select_plan_info: null pointer");
  CNB_REQUIRE(elem_size == 4 || elem_size == 2, CNB_EINVAL, "cnb_select_plan_info: elem_size %d", elem_size);
  cnb::SelectPlan pl;
  const int rc = cnb::make_select_plan(src, n_img, C, H, W, K, nms, &pl, elem_size);
  if (rc != CNB_OK) return rc;
  // some image lies inside one CTA's range: that CTA finalizes it without a global segment
  int local_img = 0;
  for (int i = 0; i < pl.n_cta && !local_img; ++i) {
    const long long lo = pl.cta_start[i], hi = pl.cta_start[i + 1];
    const long long first = (lo + C - 1) / C * C;   // first image boundary at or after lo
    local_img = (first + C <= hi) ? 1 : 0;
  }
  const int v[CNB_SELECT_PLAN_FIELDS] = {pl.hot, pl.n_cta, pl.wb, pl.max_slots, pl.seg_cap, pl.fused_finalize,
                                         pl.use_tma, pl.rb, local_img};
  for (int i = 0; i < n_out && i < CNB_SELECT_PLAN_FIELDS; ++i) out[i] = v[i];
  return CNB_OK;
}

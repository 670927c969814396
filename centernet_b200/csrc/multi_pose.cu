// multi_pose_decode (models/decode.py:497-571) on top of the fused NMS+top-K selection:
//   select(heat)  -> K centres per image         (decode.py:503-504)
//   select(hm_hp) -> K peaks per (image, joint)  (:528-533, _topk_channel on _nms(hm_hp))
//   k_pose_assemble: one CTA per (image, joint), one thread per detection; the joint's K
//   heat-map candidates live in shared memory; each thread does the gathers, the nearest-
//   candidate search and the reject tests of :534-566 and writes its slice of the 40-column row.
#include <climits>
#include "select.cuh"

namespace cnb {

struct PoseArgs {
  // centre top-K (per image)
  const float *c_scores; const int64_t *c_inds; const int32_t *c_clses; const float *c_ys; const float *c_xs;
  // joint top-K (per image*joint), null when hm_hp is absent
  const float *j_scores; const int64_t *j_inds; const float *j_ys; const float *j_xs;
  const void *wh, *kps, *reg, *hp_offset;  // fp32, or (EX) of the dtype codes below
  int wh_dt, kps_dt, reg_dt, off_dt;
  int B, J, H, W, K;
  float *dets;  // [B, K, 4 + 1 + 2J + 1]
};

// Element i of a head: fp32 (the cnb_multi_pose_decode instance), or of its dtype code, widened exactly (EX)
template <bool EX>
__device__ __forceinline__ float ld_pose(const void *p, int dt, long long i) {
  if (EX) return ld_head(p, dt, (size_t)i);
  return reinterpret_cast<const float *>(p)[i];
}

template <bool EX>
__global__ void __launch_bounds__(1024) k_pose_assemble(const PoseArgs a) {
  extern __shared__ float sm[];  // [3][K]: candidate x, y, score of this (image, joint)
  const int b = blockIdx.x / a.J, j = blockIdx.x - b * a.J;
  const int K = a.K, D = 4 + 1 + 2 * a.J + 1;
  const long long HW = (long long)a.H * a.W;
  float *cx = sm, *cy = sm + K, *cs = sm + 2 * K;
  const bool has_hp = a.j_scores != nullptr;
  if (has_hp) {
    for (int m = threadIdx.x; m < K; m += blockDim.x) {
      const size_t o = ((size_t)b * a.J + j) * K + m;
      float s = a.j_scores[o], x = a.j_xs[o], y = a.j_ys[o];
      if (a.hp_offset) {  // :534-539
        const long long sp = a.j_inds[o];
        x += ld_pose<EX>(a.hp_offset, a.off_dt, ((long long)b * 2) * HW + sp);
        y += ld_pose<EX>(a.hp_offset, a.off_dt, ((long long)b * 2 + 1) * HW + sp);
      } else {  // :540-542
        x += 0.5f;
        y += 0.5f;
      }
      if (!(s > 0.1f)) {  // :544-547  mask = (hm_score > thresh)
        s = -1.0f;
        x = -10000.0f;
        y = -10000.0f;
      }
      cx[m] = x; cy[m] = y; cs[m] = s;
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const size_t o = (size_t)b * K + k;
    const long long sp = a.c_inds[o];
    const float xi = a.c_xs[o], yi = a.c_ys[o];
    // regressed joint location uses the INTEGER centre (:506-509)
    float kx = ld_pose<EX>(a.kps, a.kps_dt, ((long long)b * 2 * a.J + 2 * j) * HW + sp) + xi;
    float ky = ld_pose<EX>(a.kps, a.kps_dt, ((long long)b * 2 * a.J + 2 * j + 1) * HW + sp) + yi;
    float xs = xi, ys = yi;
    if (a.reg) {
      xs += ld_pose<EX>(a.reg, a.reg_dt, ((long long)b * 2) * HW + sp);
      ys += ld_pose<EX>(a.reg, a.reg_dt, ((long long)b * 2 + 1) * HW + sp);
    } else {
      xs += 0.5f;
      ys += 0.5f;
    }
    const float hw_ = ld_pose<EX>(a.wh, a.wh_dt, ((long long)b * 2) * HW + sp) * 0.5f;
    const float hh_ = ld_pose<EX>(a.wh, a.wh_dt, ((long long)b * 2 + 1) * HW + sp) * 0.5f;
    const float l = xs - hw_, t = ys - hh_, r = xs + hw_, bt = ys + hh_;
    float *d = a.dets + o * D;
    if (j == 0) {
      d[0] = l; d[1] = t; d[2] = r; d[3] = bt;
      d[4] = a.c_scores[o];
      d[D - 1] = (float)a.c_clses[o];
    }
    if (has_hp) {
      // :548-551: first minimum of the L2 distance over the non-NaN distances (candidate 0 when all are NaN)
      float best = 0.0f, bx = 0.0f, by = 0.0f, bs = 0.0f;
      for (int m = 0; m < K; ++m) {
        const float dx = kx - cx[m], dy = ky - cy[m];
        const float dist = sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
        if (m == 0 || dist < best || (isnan(best) && !isnan(dist))) {
          best = dist; bx = cx[m]; by = cy[m]; bs = cs[m];
        }
      }
      // :558-565; torch.max propagates NaN (fmaxf would drop it), and a NaN limit rejects nothing
      const float bh = bt - t, bw = r - l;
      const float lim = ((isnan(bh) || isnan(bw)) ? bh + bw : fmaxf(bh, bw)) * 0.3f;
      const bool reject = (bx < l) || (bx > r) || (by < t) || (by > bt) || (bs < 0.1f) || (best > lim);
      // :566-567: the reference's blend (1 - mask) * hm_kps + mask * kps, not a select, so that a NaN or infinite
      // keypoint regression gives what the reference gives (0 * inf is NaN)
      const float m = reject ? 1.0f : 0.0f;
      kx = __fadd_rn(__fmul_rn(1.0f - m, bx), __fmul_rn(m, kx));
      ky = __fadd_rn(__fmul_rn(1.0f - m, by), __fmul_rn(m, ky));
    }
    d[5 + 2 * j] = kx;
    d[5 + 2 * j + 1] = ky;
  }
}

static size_t raw_bytes_(long long n) { return align_up((size_t)n * 8, 256) + 4 * align_up((size_t)n * 4, 256); }

}  // namespace cnb

using namespace cnb;

extern "C" {

size_t cnb_multi_pose_workspace_bytes(int b, int c, int j, int h, int w, int k) {
  size_t sel = select_workspace_bytes_any_align(b, c, h, w, k);
  if (sel == 0) return 0;
  if (j > 0) {
    const size_t s2 = select_workspace_bytes_any_align(b * j, 1, h, w, k);
    if (s2 == 0) return 0;
    sel = s2 > sel ? s2 : sel;
  }
  return sel + raw_bytes_((long long)b * k) + raw_bytes_((long long)b * j * k);
}

int cnb_multi_pose_decode(const float *heat, const float *wh, const float *kps, const float *reg, const float *hm_hp,
                          const float *hp_offset, int b, int c, int j, int h, int w, int k, float *dets,
                          void *workspace, size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(heat && wh && kps && dets && workspace, CNB_EINVAL, "cnb_multi_pose_decode: null pointer");
  CNB_REQUIRE(j > 0, CNB_EINVAL, "cnb_multi_pose_decode: j=%d", j);
  CNB_REQUIRE(hm_hp || !hp_offset, CNB_EINVAL, "cnb_multi_pose_decode: hp_offset without hm_hp");
  cudaStream_t stream = (cudaStream_t)stream_;
  SelectPlan p1, p2;
  int rc = make_select_plan(heat, b, c, h, w, k, 1, &p1);
  if (rc != CNB_OK) return rc;
  size_t sel = select_workspace_bytes(p1);
  if (hm_hp) {
    rc = make_select_plan(hm_hp, b * j, 1, h, w, k, 1, &p2);
    if (rc != CNB_OK) return rc;
    const size_t s2 = select_workspace_bytes(p2);
    sel = s2 > sel ? s2 : sel;
  }
  const size_t need = sel + raw_bytes_((long long)b * k) + raw_bytes_((long long)b * j * k);
  CNB_REQUIRE(workspace_bytes >= need, CNB_EWORKSPACE, "cnb_multi_pose_decode: workspace %zu < %zu",
              workspace_bytes, need);
  char *p = reinterpret_cast<char *>(workspace) + sel;
  const long long n1 = (long long)b * k, n2 = (long long)b * j * k;
  int64_t *c_inds = reinterpret_cast<int64_t *>(p); p += align_up((size_t)n1 * 8, 256);
  float *c_scores = reinterpret_cast<float *>(p); p += align_up((size_t)n1 * 4, 256);
  int32_t *c_clses = reinterpret_cast<int32_t *>(p); p += align_up((size_t)n1 * 4, 256);
  float *c_ys = reinterpret_cast<float *>(p); p += align_up((size_t)n1 * 4, 256);
  float *c_xs = reinterpret_cast<float *>(p); p += align_up((size_t)n1 * 4, 256);
  int64_t *j_inds = reinterpret_cast<int64_t *>(p); p += align_up((size_t)n2 * 8, 256);
  float *j_scores = reinterpret_cast<float *>(p); p += align_up((size_t)n2 * 4, 256);
  p += align_up((size_t)n2 * 4, 256);  // (unused class slot keeps the raw layout uniform)
  float *j_ys = reinterpret_cast<float *>(p); p += align_up((size_t)n2 * 4, 256);
  float *j_xs = reinterpret_cast<float *>(p);

  FinalizeOut o1 = {c_scores, c_inds, c_clses, c_ys, c_xs, nullptr, nullptr, 0, nullptr};
  rc = run_select(heat, p1, o1, workspace, stream);
  if (rc != CNB_OK) return rc;
  if (hm_hp) {
    FinalizeOut o2 = {j_scores, j_inds, nullptr, j_ys, j_xs, nullptr, nullptr, 0, nullptr};
    rc = run_select(hm_hp, p2, o2, workspace, stream);
    if (rc != CNB_OK) return rc;
  }
  PoseArgs a;
  a.c_scores = c_scores; a.c_inds = c_inds; a.c_clses = c_clses; a.c_ys = c_ys; a.c_xs = c_xs;
  a.j_scores = hm_hp ? j_scores : nullptr; a.j_inds = j_inds; a.j_ys = j_ys; a.j_xs = j_xs;
  a.wh = wh; a.kps = kps; a.reg = reg; a.hp_offset = hp_offset;
  a.wh_dt = a.kps_dt = a.reg_dt = a.off_dt = CNB_DTYPE_F32;
  a.B = b; a.J = j; a.H = h; a.W = w; a.K = k; a.dets = dets;
  const int threads = k < 1024 ? ((k + 31) / 32) * 32 : 1024;
  k_pose_assemble<false><<<b * j, threads, (size_t)3 * k * sizeof(float), stream>>>(a);
  CNB_CHECK_LAUNCH("cnb_multi_pose_decode assemble");
  count_launch();
  return CNB_OK;
}

/* cnb_multi_pose_decode of fp32, fp16 or bf16 heads, the heat maps or their logits (see the header).  Layout:
 * [selection scratch, shared by both selections | raw top-K of the centres | of the joints |
 *  one fp32 map copy, shared by both selections (only when a map is widened)]. */
size_t cnb_multi_pose_decode_ex_workspace_bytes(const void *heat, int heat_dtype, const void *hm_hp, int hm_hp_dtype,
                                                int logits, int b, int c, int j, int h, int w, int k) {
  if (!dtype_known(heat_dtype) || !dtype_known(hm_hp_dtype) || j <= 0) return 0;
  MapSelect m1, m2;
  if (plan_map_select(heat, heat_dtype, logits, b, c, h, w, k, nullptr, &m1) != CNB_OK) return 0;
  size_t sel = m1.sel_bytes, map = m1.map_bytes;
  if (hm_hp) {
    if ((long long)b * j > INT_MAX) return 0;
    if (plan_map_select(hm_hp, hm_hp_dtype, logits, b * j, 1, h, w, k, nullptr, &m2) != CNB_OK) return 0;
    sel = m2.sel_bytes > sel ? m2.sel_bytes : sel;
    map = m2.map_bytes > map ? m2.map_bytes : map;
  }
  return sel + raw_bytes_((long long)b * k) + raw_bytes_((long long)b * j * k) + map;
}

int cnb_multi_pose_decode_ex(const void *heat, int heat_dtype, int logits, const void *wh, int wh_dtype,
                             const void *kps, int kps_dtype, const void *reg, int reg_dtype, const void *hm_hp,
                             int hm_hp_dtype, const void *hp_offset, int hp_offset_dtype, int b, int c, int j, int h,
                             int w, int k, float *dets, void *workspace, size_t workspace_bytes, void *stream_) {
  CNB_REQUIRE(dtype_known(heat_dtype) && dtype_known(wh_dtype) && dtype_known(kps_dtype) && dtype_known(reg_dtype) &&
                  dtype_known(hm_hp_dtype) && dtype_known(hp_offset_dtype),
              CNB_EINVAL,
              "cnb_multi_pose_decode_ex: unknown dtype code (heat %d, wh %d, kps %d, reg %d, hm_hp %d, hp_offset %d)",
              heat_dtype, wh_dtype, kps_dtype, reg_dtype, hm_hp_dtype, hp_offset_dtype);
  CNB_REQUIRE(heat && wh && kps && dets && workspace, CNB_EINVAL, "cnb_multi_pose_decode_ex: null pointer");
  CNB_REQUIRE(j > 0, CNB_EINVAL, "cnb_multi_pose_decode_ex: j=%d", j);
  CNB_REQUIRE(hm_hp || !hp_offset, CNB_EINVAL, "cnb_multi_pose_decode_ex: hp_offset without hm_hp");
  CNB_REQUIRE((long long)b * j <= INT_MAX, CNB_EUNSUPPORTED, "cnb_multi_pose_decode_ex: b*j=%lld", (long long)b * j);
  MapSelect m1, m2;
  int rc = plan_map_select(heat, heat_dtype, logits, b, c, h, w, k, nullptr, &m1);
  if (rc != CNB_OK) return rc;
  size_t sel = m1.sel_bytes, map = m1.map_bytes;
  if (hm_hp) {
    rc = plan_map_select(hm_hp, hm_hp_dtype, logits, b * j, 1, h, w, k, nullptr, &m2);
    if (rc != CNB_OK) return rc;
    sel = m2.sel_bytes > sel ? m2.sel_bytes : sel;
    map = m2.map_bytes > map ? m2.map_bytes : map;
  }
  const long long n1 = (long long)b * k, n2 = (long long)b * j * k;
  const size_t need = sel + raw_bytes_(n1) + raw_bytes_(n2) + map;
  CNB_REQUIRE(workspace_bytes >= need, CNB_EWORKSPACE, "cnb_multi_pose_decode_ex: workspace %zu < %zu",
              workspace_bytes, need);
  char *p = reinterpret_cast<char *>(workspace) + sel;
  int64_t *c_inds = reinterpret_cast<int64_t *>(p); p += align_up((size_t)n1 * 8, 256);
  float *c_scores = reinterpret_cast<float *>(p); p += align_up((size_t)n1 * 4, 256);
  int32_t *c_clses = reinterpret_cast<int32_t *>(p); p += align_up((size_t)n1 * 4, 256);
  float *c_ys = reinterpret_cast<float *>(p); p += align_up((size_t)n1 * 4, 256);
  float *c_xs = reinterpret_cast<float *>(p); p += align_up((size_t)n1 * 4, 256);
  int64_t *j_inds = reinterpret_cast<int64_t *>(p); p += align_up((size_t)n2 * 8, 256);
  float *j_scores = reinterpret_cast<float *>(p); p += align_up((size_t)n2 * 4, 256);
  p += align_up((size_t)n2 * 4, 256);  // (unused class slot keeps the raw layout uniform)
  float *j_ys = reinterpret_cast<float *>(p); p += align_up((size_t)n2 * 4, 256);
  float *j_xs = reinterpret_cast<float *>(p); p += align_up((size_t)n2 * 4, 256);
  float *copy = reinterpret_cast<float *>(p);
  // the plans of widened maps where their copy really lies (a workspace that is not 16-byte aligned loses TMA)
  if (m1.widen) {
    rc = plan_map_select(heat, heat_dtype, logits, b, c, h, w, k, copy, &m1);
    if (rc != CNB_OK) return rc;
  }
  if (hm_hp && m2.widen) {
    rc = plan_map_select(hm_hp, hm_hp_dtype, logits, b * j, 1, h, w, k, copy, &m2);
    if (rc != CNB_OK) return rc;
  }
  CNB_REQUIRE(m1.sel_bytes <= sel && (!hm_hp || m2.sel_bytes <= sel), CNB_EWORKSPACE,
              "cnb_multi_pose_decode_ex: selection scratch exceeds %zu", sel);

  const cudaStream_t stream = (cudaStream_t)stream_;
  FinalizeOut o1 = {c_scores, c_inds, c_clses, c_ys, c_xs, nullptr, nullptr, 0, nullptr};
  rc = run_map_select(heat, heat_dtype, logits, m1, copy, o1, workspace, stream);
  if (rc != CNB_OK) return rc;
  if (hm_hp) {  // stream order: the heat selection is done with the scratch and the copy
    FinalizeOut o2 = {j_scores, j_inds, nullptr, j_ys, j_xs, nullptr, nullptr, 0, nullptr};
    rc = run_map_select(hm_hp, hm_hp_dtype, logits, m2, copy, o2, workspace, stream);
    if (rc != CNB_OK) return rc;
  }
  PoseArgs a;
  a.c_scores = c_scores; a.c_inds = c_inds; a.c_clses = c_clses; a.c_ys = c_ys; a.c_xs = c_xs;
  a.j_scores = hm_hp ? j_scores : nullptr; a.j_inds = j_inds; a.j_ys = j_ys; a.j_xs = j_xs;
  a.wh = wh; a.kps = kps; a.reg = reg; a.hp_offset = hp_offset;
  a.wh_dt = wh_dtype; a.kps_dt = kps_dtype; a.reg_dt = reg_dtype; a.off_dt = hp_offset_dtype;
  a.B = b; a.J = j; a.H = h; a.W = w; a.K = k; a.dets = dets;
  const int threads = k < 1024 ? ((k + 31) / 32) * 32 : 1024;
  k_pose_assemble<true><<<b * j, threads, (size_t)3 * k * sizeof(float), stream>>>(a);
  CNB_CHECK_LAUNCH("cnb_multi_pose_decode_ex assemble");
  count_launch();
  return CNB_OK;
}

}  // extern "C"

/*
 * centernet_b200 -- C ABI of the H100-native CenterNet heat-map hot path.
 *
 * This is the drop-in boundary: plain device pointers, explicit sizes and a
 * CUDA stream handle; no torch types.  The reference has two bindings on this
 * path and both are replaced here:
 *
 *   (1) the Python ATen-op functions of src/lib/models/decode.py,
 *       src/lib/models/utils.py and src/lib/models/losses.py (no FFI of their
 *       own -- each cnb_* entry below names the function it replaces), and
 *   (2) the cffi module `_ext.dcn_v2` declared in
 *       src/lib/models/networks/DCNv2/src/dcn_v2_cuda.h:9-55
 *       (dcn_v2_cuda_forward / dcn_v2_cuda_backward / dcn_v2_psroi_pooling_*).
 *
 * Conventions
 *   - every tensor is fp32 (double in the *_f64 entry points; fp32, fp16 or bf16 where a dtype code is passed), NCHW,
 *     contiguous, resident on the current device;
 *     index outputs use the reference's dtypes (int64 indices, int32 classes);
 *   - the caller owns every buffer, including the scratch `workspace`
 *     (size from the matching cnb_*_workspace_bytes); the library never calls
 *     cudaMalloc and keeps no global mutable state, so it may be called from
 *     one thread per GPU concurrently (torch DataParallel style);
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*);
 *     nothing synchronises the host;
 *   - return value: CNB_OK or an error code; cnb_last_error() gives a
 *     thread-local description.  The reference's THArgCheck/THError
 *     (dcn_v2_cuda.c:20-38) map to CNB_EINVAL.
 */
#ifndef CENTERNET_B200_H_
#define CENTERNET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CNB_OK 0
#define CNB_EINVAL 1       /* bad shape / null pointer / misaligned buffer        */
#define CNB_EUNSUPPORTED 2 /* valid request outside the implemented envelope     */
#define CNB_ECUDA 3        /* CUDA runtime / launch error                        */
#define CNB_EWORKSPACE 4   /* workspace_bytes smaller than cnb_*_workspace_bytes */

/* Element type codes of the entry points that take more than one (cnb_dcnv2_forward_bf16, cnb_ctdet_decode_ex,
 * cnb_flip_merge_ex, cnb_ddd_decode_ex, cnb_multi_pose_decode_ex, cnb_edge_aggregate_ex, cnb_exct_decode_ex,
 * cnb_gather_feat_ex and the loss calls cnb_focal_*_ex / cnb_reg_loss_*ex). */
#define CNB_DTYPE_F32 0
#define CNB_DTYPE_BF16 1
#define CNB_DTYPE_F16 2

/* Library version (major*10000 + minor*100 + patch). */
int cnb_version(void);
/* Thread-local text of the last error returned on this thread ("" if none). */
const char *cnb_last_error(void);
/* Number of kernels launched by this library since process start (all threads);
 * bench.py reports it as `gpu_launches`. */
unsigned long long cnb_launch_count(void);

/* ---------------------------------------------------------------- A1: _nms
 * models/decode.py:9-15.  out = heat * (maxpool3x3(heat) == heat).
 * heat,out: [n, c, h, w]. */
int cnb_nms(const float *heat, float *out, int n, int c, int h, int w, void *stream);

/* ------------------------------------------------------------- A2/A3: top-K
 * Workspace for every selection-based entry point below (depends on the
 * largest (n_img, c, h, w, k) the call processes). */
size_t cnb_topk_workspace_bytes(int n_img, int c, int h, int w, int k);

/* models/decode.py:103-119 (_topk).  scores: [b, c, h, w] (already NMS'd by the
 * caller, as in the reference) -> per image the K best over all classes:
 * out_scores[b,k] f32, out_inds[b,k] i64 (y*w+x), out_clses[b,k] i32,
 * out_ys/out_xs[b,k] f32.  Order: score desc, ties by flat index asc.
 * fuse_nms != 0 applies the 3x3 peak test of _nms first (scores = raw heat). */
int cnb_topk(const float *scores, int b, int c, int h, int w, int k, int fuse_nms,
             float *out_scores, int64_t *out_inds, int32_t *out_clses,
             float *out_ys, float *out_xs,
             void *workspace, size_t workspace_bytes, void *stream);

/* Read-only view of the plan every selection above (and every decode built on it) makes for an
 * [n_img, C, H, W] map at `src` (its alignment and elem_size -- 4, or 2 for fp16 / bf16 -- decide whether
 * TMA can load it) on the current device.  Writes min(n_out, CNB_SELECT_PLAN_FIELDS) ints to out, in this
 * order: hot (warp-asynchronous 128x128 kernel), n_cta (stage-1 grid), wb (planes one image boundary weighs
 * in the partition, 0 = equal split), max_slots (segments one image can receive), seg_cap (keys per
 * segment), fused_finalize (0: the separate finalize kernel runs), use_tma, rb (rows per unit) and
 * local_img (some image lies inside one CTA's range, so that CTA finalizes it from shared memory).
 * Launches nothing; errors are those of the selection itself for the same arguments. */
#define CNB_SELECT_PLAN_FIELDS 9
int cnb_select_plan_info(const void *src, int n_img, int c, int h, int w, int k, int nms, int elem_size,
                         int *out, int n_out);

/* models/decode.py:92-101 (_topk_channel): per (b, channel) top-K.
 * Outputs are [b, c, k]. */
int cnb_topk_channel(const float *scores, int b, int c, int h, int w, int k, int fuse_nms,
                     float *out_scores, int64_t *out_inds, float *out_ys, float *out_xs,
                     void *workspace, size_t workspace_bytes, void *stream);

/* --------------------------------------------------------------- A4: gather
 * models/utils.py:22-26 (_transpose_and_gather_feat) without the transpose
 * copy: out[b, m, ch] = feat[b, ch, ind[b, m]];  feat [b, c, h*w], ind [b, m]. */
int cnb_gather_feat(const float *feat, const int64_t *ind, float *out,
                    int b, int c, int hw, int m, void *stream);
/* Adjoint of cnb_gather_feat (what autograd derives for the reference's
 * permute + gather, models/utils.py:12-26; used by every Reg*Loss, L1Loss and
 * BinRotLoss of models/losses.py through `pred = _transpose_and_gather_feat`):
 * grad_feat[b, ch, ind[b, m]] += grad_out[b, m, ch].  grad_feat must arrive
 * zero-filled; repeated indices accumulate. */
int cnb_gather_feat_backward(const float *grad_out, const int64_t *ind, float *grad_feat,
                             int b, int c, int hw, int m, void *stream);
/* The same pair for a feat of feat_dtype (CNB_DTYPE_F32 / _BF16 / _F16), read and written in place: no fp32 copy
 * of the map is made.  out stays fp32 [b, m, c] and equals cnb_gather_feat of the .float() upcast (both formats
 * widen exactly).  cnb_gather_feat_backward_ex zero-fills grad_feat ([b, c, hw] of feat_dtype) itself and leaves
 * in it, bit for bit, cnb_gather_feat_backward's fp32 map rounded once to feat_dtype: the rows of a repeated
 * index are added in fp32 in ascending m and only the sum is rounded; nothing is accumulated in the half map and
 * there are no atomics, so it is bit-identical run to run.  Indices outside [0, hw) are skipped.  Errors, checked
 * before any CUDA call: CNB_EINVAL for an unknown dtype code, a null pointer or a bad shape. */
int cnb_gather_feat_ex(const void *feat, int feat_dtype, const int64_t *ind, float *out,
                       int b, int c, int hw, int m, void *stream);
int cnb_gather_feat_backward_ex(const float *grad_out, const int64_t *ind, void *grad_feat, int feat_dtype,
                                int b, int c, int hw, int m, void *stream);

/* ---------------------------------------------------------- A5: ctdet_decode
 * models/decode.py:464-495.  heat [b,c,h,w] (post-sigmoid), wh [b,2,h,w] (or
 * [b,2c,h,w] when cat_spec_wh), reg [b,2,h,w] or NULL -> dets [b,k,6] =
 * x1,y1,x2,y2,score,class.  One fused pass: peak-NMS + top-K + gathers. */
int cnb_ctdet_decode(const float *heat, const float *wh, const float *reg, int cat_spec_wh,
                     int b, int c, int h, int w, int k, float *dets,
                     void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------- N1: ctdet_decode with fused sigmoid
 * Replaces `hm = output['hm'].sigmoid_(); ctdet_decode(hm, wh, reg, ...)`
 * (detectors/ctdet.py:30-45): hm_logits [b,c,h,w] is the head's raw output.
 * Scores are bit-identical to torch's CUDA sigmoid of the logits, indices and
 * classes identical to cnb_ctdet_decode on that heat map.  The workspace query
 * takes the logits pointer because its alignment decides the code path. */
size_t cnb_ctdet_logits_workspace_bytes(const float *hm_logits, int b, int c, int h, int w, int k);
int cnb_ctdet_decode_logits(const float *hm_logits, const float *wh, const float *reg, int cat_spec_wh,
                            int b, int c, int h, int w, int k, float *dets,
                            void *workspace, size_t workspace_bytes, void *stream);

/* ----------------------------------- N1: ctdet_decode of fp32, fp16 or bf16 heads
 * cnb_ctdet_decode (logits == 0) or cnb_ctdet_decode_logits (logits != 0) for heads of any of the three float
 * types, each of heat, wh and reg with its own dtype code (CNB_DTYPE_F32 / _F16 / _BF16).  Contract: for fp16 or
 * bf16 tensors the dets, bit for bit, are those the fp32 calls return for the .float() upcast of the same
 * tensors (both widen exactly to fp32; the logits path scores with the fp32 sigmoid of the widened logit).
 * dets stay fp32.  In the hot geometry (h = w = 128, k <= 256, heat 16-byte aligned) the selection kernel reads
 * the 16-bit map itself; any other geometry widens the map once into the workspace (logits: the sigmoid pass reads
 * the 16-bit logits) and runs the fp32 path.  The query takes the heat pointer because its alignment decides the
 * path; with CNB_DTYPE_F32 it equals cnb_topk_workspace_bytes (logits == 0) or cnb_ctdet_logits_workspace_bytes,
 * and it returns 0 for every shape the call rejects.  Errors, checked before any CUDA call: CNB_EINVAL for an
 * unknown dtype code, a null pointer or a bad shape; CNB_EWORKSPACE for too small a workspace. */
size_t cnb_ctdet_decode_ex_workspace_bytes(const void *heat, int heat_dtype, int logits,
                                           int b, int c, int h, int w, int k);
int cnb_ctdet_decode_ex(const void *heat, int heat_dtype, int logits, const void *wh, int wh_dtype,
                        const void *reg, int reg_dtype, int cat_spec_wh, int b, int c, int h, int w, int k,
                        float *dets, void *workspace, size_t workspace_bytes, void *stream);

/* out[i] = 1 / (1 + exp(-x[i])): the bare `sigmoid_()` of detectors/ctdet.py:31, the very expression the
 * fused path applies to its candidates (exposed so tests can pin it against torch and prove it monotone). */
int cnb_sigmoid(const float *x, float *out, long long n, void *stream);

/* ------------------------------------------- N1: flip-test merge of the heads
 * detectors/ctdet.py:34-37 and detectors/multi_pose.py:43-51.  src [2n,c,h,w]:
 * n images followed by their horizontally flipped copies; dst [n,c,h,w] =
 * (f(src[i,ch]) + sign[ch] * f(flip_w(src[n+i, perm[ch]]))) / 2, f = sigmoid when
 * apply_sigmoid.  perm/sign NULL = flip_tensor (models/utils.py:28-29); perm =
 * joint swap for flip_lr (:33-39); perm + sign for flip_lr_off (:41-50). */
int cnb_flip_merge(const float *src, float *dst, int n, int c, int h, int w, int apply_sigmoid,
                   const int32_t *perm, const float *sign, void *stream);
/* The same merge for a src of src_dtype (CNB_DTYPE_F32 / _F16 / _BF16): elements are widened exactly to fp32
 * first, so the fp32 dst equals cnb_flip_merge of the .float() upcast.  CNB_EINVAL for an unknown dtype code, a
 * null pointer or a non-positive dimension, before any CUDA call. */
int cnb_flip_merge_ex(const void *src, int src_dtype, float *dst, int n, int c, int h, int w, int apply_sigmoid,
                      const int32_t *perm, const float *sign, void *stream);

/* ------------------------------------------------------------ A9: ddd_decode
 * models/decode.py:426-462.  rot [b,8,h,w], depth [b,1,h,w], dim [b,3,h,w],
 * wh/reg [b,2,h,w] or NULL -> dets [b,k,18] (16 when wh == NULL). */
int cnb_ddd_decode(const float *heat, const float *rot, const float *depth, const float *dim,
                   const float *wh, const float *reg, int b, int c, int h, int w, int k,
                   float *dets, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------- N1: ddd_decode of fp32, fp16 or bf16 heads, from the logits
 * cnb_ddd_decode for heads of any of the three float types, each of heat, rot, depth, dim, wh and reg with its own
 * dtype code.  logits != 0 replaces `hm.sigmoid_()` and `dep = 1. / (dep.sigmoid() + 1e-6) - 1.`
 * (detectors/ddd.py:61-62): heat holds the hm logits and depth the raw dep output, and the depth transform is
 * evaluated at the k gathered positions only, in torch's op order (sigmoid, add, reciprocal, mul, sub, each rounded
 * to fp32).  Contract: the dets, bit for bit, are those of cnb_ddd_decode on the .float() upcast of the heads (after
 * torch's CUDA sigmoid of heat and the depth transform, with logits).  Half inputs are widened exactly and then
 * processed as fp32; a half-precision `sigmoid_()` would round every intermediate to half instead.  The selection
 * reads the heat map in place in the hot geometry (h = w = 128, k <= 256, 16-byte aligned) and when it is an fp32
 * heat map; otherwise one pass writes its fp32 copy (or sigmoid) into the workspace.  The query takes the heat
 * pointer because its alignment decides the path and returns 0 for every shape or dtype code the call rejects.
 * Errors, checked before any CUDA call: CNB_EINVAL for an unknown dtype code, a null pointer or a bad shape,
 * CNB_EUNSUPPORTED for k > 1024, CNB_EWORKSPACE for too small a workspace. */
size_t cnb_ddd_decode_ex_workspace_bytes(const void *heat, int heat_dtype, int logits,
                                         int b, int c, int h, int w, int k);
int cnb_ddd_decode_ex(const void *heat, int heat_dtype, int logits, const void *rot, int rot_dtype,
                      const void *depth, int depth_dtype, const void *dim, int dim_dtype,
                      const void *wh, int wh_dtype, const void *reg, int reg_dtype,
                      int b, int c, int h, int w, int k, float *dets,
                      void *workspace, size_t workspace_bytes, void *stream);

/* ----------------------------------------------------- A6: multi_pose_decode
 * models/decode.py:497-571.  heat [b,1,h,w]; wh, reg(NULL ok) [b,2,h,w];
 * kps [b,2j,h,w]; hm_hp [b,j,h,w] or NULL; hp_offset [b,2,h,w] or NULL
 * -> dets [b,k,4+1+2j+1]. */
size_t cnb_multi_pose_workspace_bytes(int b, int c, int j, int h, int w, int k);
int cnb_multi_pose_decode(const float *heat, const float *wh, const float *kps, const float *reg,
                          const float *hm_hp, const float *hp_offset,
                          int b, int c, int j, int h, int w, int k, float *dets,
                          void *workspace, size_t workspace_bytes, void *stream);

/* --------------------- N1: multi_pose_decode of fp32, fp16 or bf16 heads, from the logits
 * cnb_multi_pose_decode for heads of any of the three float types, each of heat, wh, kps, reg, hm_hp and hp_offset
 * with its own dtype code (a null head's code must still be a known one).  logits != 0 replaces `hm.sigmoid_()` and
 * `hm_hp.sigmoid_()` (detectors/multi_pose.py:33-35): heat and hm_hp hold logits.  Contract: the dets, bit for bit,
 * are those of cnb_multi_pose_decode on the .float() upcast of the heads (after torch's CUDA sigmoid of heat and hm_hp,
 * with logits).  Half inputs are widened exactly and then processed as fp32.  Each selection (heat as b images,
 * hm_hp as b*j one-plane images) reads its map in place in the hot geometry (h = w = 128, k <= 256, 16-byte aligned)
 * and when it is an fp32 heat map; otherwise one pass writes its fp32 copy (or sigmoid) into the workspace.  The query
 * takes the heat and hm_hp pointers (hm_hp NULL: no joint selection) because their alignment decides the path, and
 * returns 0 for every shape or dtype code the call rejects.  Errors, checked before any CUDA call: CNB_EINVAL for an
 * unknown dtype code, a null pointer, hp_offset without hm_hp or a bad shape, CNB_EUNSUPPORTED for k > 1024,
 * CNB_EWORKSPACE for too small a workspace. */
size_t cnb_multi_pose_decode_ex_workspace_bytes(const void *heat, int heat_dtype, const void *hm_hp,
                                                int hm_hp_dtype, int logits, int b, int c, int j, int h, int w,
                                                int k);
int cnb_multi_pose_decode_ex(const void *heat, int heat_dtype, int logits, const void *wh, int wh_dtype,
                             const void *kps, int kps_dtype, const void *reg, int reg_dtype,
                             const void *hm_hp, int hm_hp_dtype, const void *hp_offset, int hp_offset_dtype,
                             int b, int c, int j, int h, int w, int k, float *dets,
                             void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------ A7: edge aggregation
 * models/decode.py:17-77.  out = heat + weight*(dirA + dirB) with
 * horizontal != 0: _h_aggregate (left+right), else _v_aggregate (top+bottom).
 * Strictly sequential fp32 running sums, as the reference. */
int cnb_edge_aggregate(const float *heat, float *out, int n, int c, int h, int w,
                       float aggr_weight, int horizontal, void *stream);
/* The same for a heat map of dtype code dtype (CNB_DTYPE_F32 / _F16 / _BF16), or for its logits (apply_sigmoid):
 * every element is widened exactly to fp32, then (apply_sigmoid) put through torch's CUDA sigmoid, and the fp32 out
 * equals, bit for bit, cnb_edge_aggregate of the .float() upcast (of torch.sigmoid of it).  horizontal also takes
 * the direction codes 2..5 (left, right, top, bottom: raw ret - heat).  CNB_EINVAL for an unknown dtype code, a
 * null pointer, in-place use, a non-positive dimension or a bad direction code, before any CUDA call. */
int cnb_edge_aggregate_ex(const void *heat, int dtype, int apply_sigmoid, float *out, int n, int c, int h, int w,
                          float aggr_weight, int horizontal, void *stream);

/* ------------------------------------------- A8: exct_decode / agnex_ct_decode
 * models/decode.py:273-424 and :122-271.  t,l,b,r heat [b,c,h,w] (c==1 for
 * agnostic), ct heat [b,cc,h,w]; regr [b,2,h,w] each or all NULL
 * -> dets [b,num_dets,14]. */
size_t cnb_exct_workspace_bytes(int b, int c, int cc, int h, int w, int k, int num_dets);
/* Number of CTAs (groups) per image the tuple kernel of a decode with these sizes launches on the current device:
 * min(16, ceil(2 * SMs / b), k, 16384 / num_dets).  Each group keeps its num_dets best tuples, and the merge sorts
 * the groups' segments of an image in shared memory, which holds at most 16384 keys.  Launches nothing; returns 0
 * when b, k or num_dets is below 1. */
int cnb_exct_groups(int b, int k, int num_dets);
int cnb_exct_decode(const float *t_heat, const float *l_heat, const float *b_heat,
                    const float *r_heat, const float *ct_heat,
                    const float *t_regr, const float *l_regr, const float *b_regr,
                    const float *r_regr, int b, int c, int cc, int h, int w, int k,
                    float scores_thresh, float center_thresh, float aggr_weight,
                    int num_dets, int agnostic, float *dets,
                    void *workspace, size_t workspace_bytes, void *stream);

/* ------------------ N1: exct_decode / agnex_ct_decode of fp32, fp16 or bf16 inputs, from the logits
 * cnb_exct_decode for inputs of any of the three float types, each of the four extreme maps, the centre map and the
 * four regression maps with its own dtype code (a null regression map's code must still be a known one).  logits != 0
 * replaces the `sigmoid_()` of the five maps (detectors/exdet.py:32-36): they hold logits.  Contract: the dets, bit
 * for bit and filler rows included, are those of cnb_exct_decode on the .float() upcast of the inputs (after
 * torch's CUDA sigmoid of the five maps, with logits).  Half inputs are widened exactly and then processed as fp32.
 * Each selection reads its map in place in the hot geometry (h = w = 128, k <= 256, 16-byte aligned) and when it is
 * an fp32 heat map; otherwise one pass writes its fp32 copy (or sigmoid) into the workspace, one copy shared by the
 * four selections.  With aggr_weight > 0 the aggregation reads the maps in their dtype and the selections read the
 * fp32 aggregated maps.  A centre map that is not an fp32 heat map is read in its dtype by the agnostic max /
 * argmax, or written once as fp32 scores into the workspace.  The query takes the four extreme-map pointers because
 * their alignment decides the path; with every code CNB_DTYPE_F32 and logits == 0 it equals
 * cnb_exct_workspace_bytes, and it returns 0 for every argument the call rejects.  Errors, checked before any CUDA
 * call: CNB_EINVAL for an unknown dtype code, a null pointer or a bad shape, CNB_EUNSUPPORTED for k > 255 or
 * num_dets > 2048, CNB_EWORKSPACE for too small a workspace. */
size_t cnb_exct_decode_ex_workspace_bytes(const void *t_heat, const void *l_heat, const void *b_heat,
                                          const void *r_heat, int t_dtype, int l_dtype, int b_dtype, int r_dtype,
                                          int ct_dtype, int t_regr_dtype, int l_regr_dtype, int b_regr_dtype,
                                          int r_regr_dtype, int logits, int b, int c, int cc, int h, int w, int k,
                                          float aggr_weight, int num_dets, int agnostic);
int cnb_exct_decode_ex(const void *t_heat, int t_dtype, const void *l_heat, int l_dtype, const void *b_heat,
                       int b_dtype, const void *r_heat, int r_dtype, const void *ct_heat, int ct_dtype,
                       const void *t_regr, int t_regr_dtype, const void *l_regr, int l_regr_dtype,
                       const void *b_regr, int b_regr_dtype, const void *r_regr, int r_regr_dtype, int logits,
                       int b, int c, int cc, int h, int w, int k, float scores_thresh, float center_thresh,
                       float aggr_weight, int num_dets, int agnostic, float *dets, void *workspace,
                       size_t workspace_bytes, void *stream);

/* ------------------------------------------------- A13/A14/A15: focal + splat
 * _sigmoid (models/utils.py:8-10), _neg_loss (models/losses.py:42-67) and the
 * Gaussian target splat draw_umich_gaussian (utils/image.py:126-141) fused.
 *
 * cnb_focal_loss: pred/gt [n] flat (gt given as a dense map, reference form).
 *   logits != 0: `pred` holds raw logits and _sigmoid (clamped) is applied
 *   first.  Writes out[0]=loss, out[1]=num_pos; grad (nullable) receives
 *   d loss / d pred (or / d logit when logits != 0) scaled by grad_scale.
 * cnb_focal_splat_loss: same loss but the target map is never materialised:
 *   it is rebuilt on the fly from per-image object lists
 *   obj_cls[b,m] i32, obj_cx/obj_cy[b,m] i32 (ct_int), obj_radius[b,m] i32,
 *   obj_valid[b,m] u8 -- exactly the draw_umich_gaussian calls of
 *   datasets/sample/ctdet.py:111-117, so a centre outside the map paints the part
 *   of its window that overlaps it (and is no positive).  Objects with valid = 0,
 *   a negative radius or a class outside [0, c) are skipped.  m <= 128 (the reference's max_objs,
 *   datasets/dataset/coco.py:38); larger lists return CNB_EUNSUPPORTED.
 * Both losses are bit-identical run to run: the workspace (cnb_focal_workspace_bytes) holds one partial sum
 * per CTA, added in CTA order by the last CTA. */
size_t cnb_focal_workspace_bytes(long long n);
int cnb_focal_loss(const float *pred, const float *gt, long long n, int logits,
                   float grad_scale, float *out2, float *grad,
                   void *workspace, size_t workspace_bytes, void *stream);
int cnb_splat_gaussian(const int32_t *obj_cls, const int32_t *obj_cx, const int32_t *obj_cy,
                       const int32_t *obj_radius, const uint8_t *obj_valid, int b, int m,
                       int c, int h, int w, float *hm, void *stream);
int cnb_focal_splat_loss(const float *pred, const int32_t *obj_cls, const int32_t *obj_cx,
                         const int32_t *obj_cy, const int32_t *obj_radius,
                         const uint8_t *obj_valid, int b, int m, int c, int h, int w,
                         int logits, float grad_scale, float *out2, float *grad,
                         void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------ A16: RegL1Loss
 * models/losses.py:139-149 (mode 0), RegLoss smooth-L1 :123-137 (mode 1),
 * NormRegL1Loss :151-163 (mode 2), RegWeightedL1Loss :165-175 (mode 3).  mask is
 * float [b,m] in modes 0-2 (the reference's mask.float(): fractional weights are kept)
 * and float [b,m,d] in mode 3.  output [b,d,h*w], ind [b,m] i64, target [b,m,d].
 * out[0] = loss; grad_output (nullable, [b,d,hw], must be zero-filled) gets
 * d loss/d output * grad_scale; repeated ind entries add up in ascending m (bit-identical run to run). */
int cnb_reg_loss(const float *output, const void *mask, const int64_t *ind, const float *target,
                 int b, int d, int hw, int m, int mode, float grad_scale,
                 float *out1, float *grad_output, void *stream);

/* ------------------------------------- the losses on bf16 / fp16 heads, read in place
 * For a pred / output of dtype code CNB_DTYPE_BF16 or CNB_DTYPE_F16 (gt, mask, target, ind and the object lists
 * as in the fp32 calls above).  No fp32 copy of the map is made.  Contract, with the fp32 call on the .float()
 * upcast as the oracle (the reference evaluated ON half tensors -- log, pow and the sums in bf16 -- is not the
 * target):
 *   1. the loss (and num_pos) are bit for bit what the fp32 call returns for the upcast: both formats widen to
 *      fp32 exactly, and the grid, the elements of each thread, the partials and their order are the fp32 call's;
 *   2. the gradient is bit for bit (g32 * *grad_out) rounded once (to nearest even) to the input's dtype, g32
 *      being the fp32 call's gradient for the upcast with grad_scale = 1: what autograd hands back today for a
 *      half input, for any grad_out (loss weights, AMP scales, 0, negative).  An fp16 overflow becomes inf;
 *   3. the contributions of a repeated ind entry are added in fp32 in ascending m, then scaled, then rounded:
 *      never accumulated in the half map;
 *   4. no atomics on floats: bit-identical run to run.
 * grad_out is only known in backward and must be read on the device, so each loss is two calls:
 *   cnb_*_loss_ex  forward: out2[0] = loss; out2[1] = num_pos (focal) or the fp32 denominator mask sum + 1e-4
 *                  (Reg*Loss).  Same workspace as the fp32 call (cnb_focal_workspace_bytes).
 *   cnb_*_grad_ex  backward: multiplies the gradient by *grad_out (device pointer to one fp32 value; NULL means
 *                  1.0) and writes it in the input's dtype.  cnb_focal_grad_ex and cnb_reg_loss_grad_ex read the
 *                  input again and out2 as the forward left it (device pointer) and evaluate the gradient with
 *                  the forward's arithmetic: no temporary.  cnb_reg_loss_grad_ex fills the whole grad_output map
 *                  itself (elements no index selects get 0 * *grad_out, as in the fp32 path).  The fused splat is
 *                  bound by instruction issue, not by bytes, and evaluating it twice is the slower choice there:
 *                  cnb_focal_splat_loss_ex also stores the unscaled fp32 gradient in grad32 ([b,c,h,w]; NULL when
 *                  no gradient is wanted) and cnb_focal_splat_grad_ex is the scale-and-round pass over those n
 *                  values.
 * CNB_DTYPE_F32: cnb_focal_loss_ex is cnb_focal_loss without a gradient and cnb_focal_splat_loss_ex is
 * cnb_focal_splat_loss with grad_scale = 1; the other four return CNB_EUNSUPPORTED.  Errors, checked before any
 * CUDA call: CNB_EINVAL for an unknown dtype code, a null pointer or a bad shape, CNB_EUNSUPPORTED for m > 128
 * object lists, CNB_EWORKSPACE for too small a workspace. */
int cnb_focal_loss_ex(const void *pred, int pred_dtype, const float *gt, long long n, int logits, float *out2,
                      void *workspace, size_t workspace_bytes, void *stream);
int cnb_focal_grad_ex(const void *pred, int pred_dtype, const float *gt, long long n, int logits,
                      const float *loss_num_pos, const float *grad_out, void *grad, void *stream);
int cnb_focal_splat_loss_ex(const void *pred, int pred_dtype, const int32_t *obj_cls, const int32_t *obj_cx,
                            const int32_t *obj_cy, const int32_t *obj_radius, const uint8_t *obj_valid,
                            int b, int m, int c, int h, int w, int logits, float *out2, float *grad32,
                            void *workspace, size_t workspace_bytes, void *stream);
int cnb_focal_splat_grad_ex(const float *grad32, long long n, const float *grad_out, void *grad, int grad_dtype,
                            void *stream);
int cnb_reg_loss_ex(const void *output, int output_dtype, const void *mask, const int64_t *ind,
                    const float *target, int b, int d, int hw, int m, int mode, float *out2, void *stream);
int cnb_reg_loss_grad_ex(const void *output, int output_dtype, const void *mask, const int64_t *ind,
                         const float *target, int b, int d, int hw, int m, int mode, const float *loss_den,
                         const float *grad_out, void *grad_output, void *stream);

/* ---------------------------------------------------------- A10/A11: DCNv2
 * Replaces dcn_v2_cuda_forward / dcn_v2_cuda_backward
 * (DCNv2/src/dcn_v2_cuda.h:9-33, dcn_v2_cuda.c:10-241).  im2col-free: no
 * `columns` / `ones` scratch.  input [b,cin,h,w], offset [b,2*kh*kw*dg,ho,wo]
 * (channel 2t = dy, 2t+1 = dx of tap t), mask [b,kh*kw*dg,ho,wo],
 * weight [cout,cin,kh,kw], bias [cout] -> output [b,cout,ho,wo].
 * Backward ACCUMULATES into grad_weight/grad_bias and into
 * grad_input/grad_offset/grad_mask on every path (the Python wrapper
 * zero-fills them first, as dcn_v2_func.py:44-48).
 * Forward workspace (cnb_dcnv2_workspace_bytes, 16-byte aligned): the weights
 * re-tiled for the tensor-core path, a channels-last copy of the input and, for
 * maps too small to fill the GPU, split-K partial sums; the query returns 0 for
 * kernels with more than 9 taps.  workspace == NULL (or smaller than the query,
 * or anisotropic stride/pad/dilation) selects the fp32 CUDA-core forward instead.
 * cnb_dcnv2_backward: with a workspace of cnb_dcnv2_backward_workspace_bytes (16-byte aligned; channels-last
 * copies of the input and of dX, TF32 hi/lo tiles of grad_output and of the weights, the column gradient of
 * up to ~1.5 GiB worth of images at a time) the contractions run on the tensor cores; workspace == NULL (or
 * smaller, or anisotropic stride/pad/dilation, or more than 9 taps -- the query then returns 0) selects the
 * fp32 CUDA-core backward. */
size_t cnb_dcnv2_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw,
                                 int stride, int pad, int dil, int dg);
int cnb_dcnv2_forward(const float *input, const float *offset, const float *mask,
                      const float *weight, const float *bias, float *output,
                      int b, int cin, int h, int w, int cout, int kh, int kw,
                      int stride_h, int stride_w, int pad_h, int pad_w,
                      int dil_h, int dil_w, int deformable_groups,
                      void *workspace, size_t workspace_bytes, void *stream);
/* Steady-state form of the forward (what the Python module uses): the weight
 * tiles (TF32 hi/lo split, wgmma K-major layout) are built ONCE per weight version into a
 * caller-owned buffer of cnb_dcnv2_wtiles_bytes and reused by every call;
 * input_channels_last != 0 says `input` already is [b][h*w][cin] (torch
 * channels_last) so no re-layout pass runs (needs cin/dg % 32 == 0, else the flag
 * is ignored and `input` must be NCHW).  workspace: cnb_dcnv2_prepared_workspace_bytes. */
size_t cnb_dcnv2_wtiles_bytes(int cin, int cout, int kh, int kw, int dg);
int cnb_dcnv2_prepare_weights(const float *weight, int cin, int cout, int kh, int kw,
                              int deformable_groups, void *wtiles, size_t wtiles_bytes, void *stream);
size_t cnb_dcnv2_prepared_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw,
                                          int stride, int pad, int dil, int dg);
int cnb_dcnv2_forward_prepared(const float *input, int input_channels_last, const float *offset,
                               const float *mask, const void *wtiles, const float *bias, float *output,
                               int b, int cin, int h, int w, int cout, int kh, int kw,
                               int stride_h, int stride_w, int pad_h, int pad_w,
                               int dil_h, int dil_w, int deformable_groups,
                               void *workspace, size_t workspace_bytes, void *stream);
/* N3 (inference): the DCN module with its prologue and epilogue fused around the tensor-core kernel.
 * offset_mask is the RAW output of DCN.conv_offset_mask, [b, 3*kh*kw*dg, ho, wo]: its first two thirds are
 * read as the offsets and the sigmoid of its last third as the mask inside the sampler (dcn_v2.py:64-70:
 * chunk, cat and sigmoid disappear); bn_scale / bn_shift (nullable, [cout]) are the folded inference
 * BatchNorm that follows the DCN in DeformConv and relu its activation (pose_dla_dcn.py:345-357):
 * y = relu(bn_scale * (dcn + bias) + bn_shift).  Workspace as cnb_dcnv2_forward_prepared. */
int cnb_dcnv2_forward_fused(const float *input, int input_channels_last, const float *offset_mask,
                            const void *wtiles, const float *bias, const float *bn_scale,
                            const float *bn_shift, int relu, float *output,
                            int b, int cin, int h, int w, int cout, int kh, int kw,
                            int stride, int pad, int dil, int deformable_groups,
                            void *workspace, size_t workspace_bytes, void *stream);
/* bf16 forward (opt-in): bf16 operands on the bf16 tensor cores (wgmma k16), fp32 accumulate.
 * Numeric contract:
 *   - activations: a bf16 input is used as it is; an fp32 input is rounded to bf16 (RN) first, so it gives the
 *     result of the same values in bf16;
 *   - geometry: offsets, mask, bilinear weights and the 4-corner interpolation in fp32 with the expressions of the
 *     fp32 kernels (the (-1,H)x(-1,W) test, per-corner zeroing); the interpolated, masked column value is rounded
 *     once to bf16 (RN);
 *   - weights: rounded once to bf16 (RN) by cnb_dcnv2_prepare_weights_bf16 (fp32 weight in), into a buffer of
 *     cnb_dcnv2_wtiles_bf16_bytes (16-byte aligned) that is reused while the weight does not change;
 *   - contraction in fp32 (wgmma ... .f32.bf16.bf16); split-K partials (small maps) are added in a fixed order;
 *     bias, bn_scale / bn_shift and relu in fp32; the output is stored as output_dtype (bf16: RN);
 *   - bit-identical run to run (no atomics).
 * input: [b,cin,h,w] of input_dtype (CNB_DTYPE_F32 or CNB_DTYPE_BF16); input_channels_last != 0 says it is
 * [b][h*w][cin] (torch channels_last): a bf16 one is sampled in place, an fp32 one rounded by one flat pass; needs
 * cin/dg % 32 == 0, else the flag is ignored and input must be NCHW (one re-layout pass).  offset / mask (or the
 * fused form's offset_mask) and bias / bn_scale / bn_shift are fp32; output [b,cout,ho,wo] NCHW of output_dtype.
 * At most 9 taps, one stride / pad / dilation for both axes.  workspace: cnb_dcnv2_bf16_workspace_bytes (16-byte
 * aligned; a bf16 channels-last copy of the input and, on small maps, the fp32 split-K partials); it returns 0 for
 * every shape the calls reject.  Errors, checked before any CUDA call: CNB_EINVAL for a null pointer, an unknown
 * dtype code, a bad shape or a buffer that is not 16-byte aligned; CNB_EWORKSPACE for too small a workspace;
 * CNB_EUNSUPPORTED for more than 9 taps.  cnb_dcnv2_forward_fused_bf16 is cnb_dcnv2_forward_fused in this mode. */
size_t cnb_dcnv2_wtiles_bf16_bytes(int cin, int cout, int kh, int kw, int dg);
int cnb_dcnv2_prepare_weights_bf16(const float *weight, int cin, int cout, int kh, int kw,
                                   int deformable_groups, void *wtiles, size_t wtiles_bytes, void *stream);
size_t cnb_dcnv2_bf16_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw,
                                      int stride, int pad, int dil, int dg);
int cnb_dcnv2_forward_bf16(const void *input, int input_dtype, int input_channels_last,
                           const float *offset, const float *mask, const void *wtiles, const float *bias,
                           void *output, int output_dtype,
                           int b, int cin, int h, int w, int cout, int kh, int kw,
                           int stride, int pad, int dil, int deformable_groups,
                           void *workspace, size_t workspace_bytes, void *stream);
int cnb_dcnv2_forward_fused_bf16(const void *input, int input_dtype, int input_channels_last,
                                 const float *offset_mask, const void *wtiles, const float *bias,
                                 const float *bn_scale, const float *bn_shift, int relu,
                                 void *output, int output_dtype,
                                 int b, int cin, int h, int w, int cout, int kh, int kw,
                                 int stride, int pad, int dil, int deformable_groups,
                                 void *workspace, size_t workspace_bytes, void *stream);
size_t cnb_dcnv2_backward_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw,
                                          int stride, int pad, int dil, int dg);
/* The backward for a channels-last pipeline (torch channels_last): input_channels_last / grad_input_channels_last
 * != 0 say the tensor is [b][h*w][cin]; the re-layout pass of the input, the zero-fill and the final NCHW pass of
 * grad_input disappear (grad_input still arrives zero-filled).  Tensor-core path only: needs the workspace,
 * cin / deformable_groups % 32 == 0, cout <= 256; CNB_EUNSUPPORTED otherwise.  Deterministic mode included. */
int cnb_dcnv2_backward_ex(const float *input, int input_channels_last, const float *offset,
                          const float *mask, const float *weight, const float *grad_output,
                          float *grad_input, int grad_input_channels_last,
                          float *grad_offset, float *grad_mask, float *grad_weight, float *grad_bias,
                          int b, int cin, int h, int w, int cout, int kh, int kw,
                          int stride, int pad, int dil, int deformable_groups,
                          void *workspace, size_t workspace_bytes, void *stream);
/* grad_offset, grad_mask, grad_weight and grad_bias of the tensor-core backward are bit-identical run to run.
 * grad_input is by default scattered with (vector) atomics like the reference's col2im
 * (dcn_v2_im2col_cuda.cu:182-239), i.e. its last bits depend on the order the adds land.  on != 0 (process-wide,
 * default off) makes all five gradients bit-identical for every configuration the tensor-core backward covers
 * (any offsets, stride, dilation, taps <= 9, deformable groups, Cout, channels-last tensors) and independent of
 * the batch size an image is run with: grad_input is summed in 64-bit fixed point (a per-image power-of-two scale
 * from a bound on |grad_input|, integer adds in any order) and converted to fp32 at the end; an image whose
 * grad_output, weight or mask holds an inf or NaN gets an all-NaN grad_input.  While the flag is set:
 *   cnb_dcnv2_backward_workspace_bytes returns the larger size this mode needs (its default-mode value does not
 *   change), so query it after setting the flag;
 *   cnb_dcnv2_backward / _ex return CNB_EUNSUPPORTED for what only the fp32 kernels run (no or too small a
 *   workspace, anisotropic stride/pad/dilation, images beyond the 32-bit in-image indexing);
 *   cnb_dcnv2_backward_ex accepts a channels-last grad_input. */
void cnb_dcnv2_set_deterministic(int on);
int cnb_dcnv2_get_deterministic(void);
int cnb_dcnv2_backward(const float *input, const float *offset, const float *mask,
                       const float *weight, const float *grad_output,
                       float *grad_input, float *grad_offset, float *grad_mask,
                       float *grad_weight, float *grad_bias,
                       int b, int cin, int h, int w, int cout, int kh, int kw,
                       int stride_h, int stride_w, int pad_h, int pad_w,
                       int dil_h, int dil_w, int deformable_groups,
                       void *workspace, size_t workspace_bytes, void *stream);
/* bf16 backward (opt-in, the training counterpart of cnb_dcnv2_forward_bf16): both contractions on bf16 wgmma.
 * With W_b = bf16(weight) and dY_b = bf16(grad_output) (RN; exact when grad_output is bf16):
 *   - column gradient dcol = sum_o W_b * dY_b: exact products, fp32 sums, kept in fp32; grad_offset, grad_mask and
 *     grad_input follow from it with the fp32 backward's kernels (atomics, or the fixed point of deterministic mode);
 *   - grad_weight = sum_p bf16(col) * dY_b, where col is the masked bilinear value exactly as the bf16 forward
 *     computes it and rounds it once (RN): the gradient of the forward as computed, straight through its roundings,
 *     with exact products and fp32 sums;
 *   - grad_bias sums grad_output as given (no rounding) in the fixed order of cnb_dcnv2_backward's tensor-core path;
 *   - grad_offset, grad_mask, grad_weight and grad_bias are bit-identical run to run; grad_input is too while
 *     cnb_dcnv2_set_deterministic is on (the bound behind its scale comes from W_b and dY_b).
 * input: [b,cin,h,w] of input_dtype (CNB_DTYPE_F32 or CNB_DTYPE_BF16), channels-last ([b][h*w][cin]) when
 * input_channels_last != 0; grad_output: [b,cout,ho,wo] NCHW of grad_output_dtype (F32 or BF16); offset, mask and
 * weight are fp32.  The five gradients are fp32, accumulated into (zero-fill them first) and each may be NULL;
 * grad_input is channels-last when grad_input_channels_last != 0.  Channels-last tensors need
 * cin / deformable_groups % 32 == 0.  workspace: cnb_dcnv2_backward_bf16_workspace_bytes (16-byte aligned), which
 * returns 0 for every shape the call rejects and, like cnb_dcnv2_backward_workspace_bytes, more while deterministic
 * mode is on.  The call runs where both tensor-core passes of cnb_dcnv2_backward do: at most 9 taps, one stride /
 * pad / dilation for both axes, cout <= 256 and images within their 32-bit indexing; elsewhere it returns
 * CNB_EUNSUPPORTED (and the query 0) and the caller runs cnb_dcnv2_backward on the upcast operands.  Errors, checked
 * before any CUDA call: CNB_EINVAL for a null input, offset, mask, weight, grad_output or workspace, an unknown dtype
 * code, a bad shape or a buffer (input, workspace, channels-last grad_input) that is not 16-byte aligned;
 * CNB_EUNSUPPORTED as above; CNB_EWORKSPACE for too small a workspace. */
size_t cnb_dcnv2_backward_bf16_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw,
                                               int stride, int pad, int dil, int dg);
int cnb_dcnv2_backward_bf16(const void *input, int input_dtype, int input_channels_last,
                            const float *offset, const float *mask, const float *weight,
                            const void *grad_output, int grad_output_dtype,
                            float *grad_input, int grad_input_channels_last,
                            float *grad_offset, float *grad_mask, float *grad_weight, float *grad_bias,
                            int b, int cin, int h, int w, int cout, int kh, int kw,
                            int stride, int pad, int dil, int deformable_groups,
                            void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------- A10/A11: DCNv2, float64
 * The reference's second build, _ext.dcn_v2_double (dcn_v2_cuda_double.c, dcn_v2_im2col_cuda_double.cu): the
 * same layouts and arguments as the fp32 calls above with double tensors, any kernel size, stride, padding,
 * dilation and deformable_groups dividing cin.  The contractions run on the FP64 tensor cores (DMMA) and no
 * column buffer is written in the forward.  bias may be NULL.  The backward ACCUMULATES into zero-filled
 * gradients (grad_bias may be NULL) and needs a workspace of cnb_dcnv2_f64_workspace_bytes (16-byte aligned;
 * the forward needs none): two 64-bit limbs per grad_input element, one weight-gradient partial per pixel range
 * (at most 64) and the column gradient dcol = W^T . dY of as many images as fit in 1.5 GiB (at least one), e.g.
 * about 1.5 GB in all for B = 16 at 64@128x128 -> 64.
 * Fixed-point contract: all five float64 gradients are bit-identical run to run, whatever the deterministic flag
 * below says, and grad_input, grad_offset and grad_mask of an image do not depend on the batch it runs in.
 * grad_input is summed in two 64-bit integer limbs per element: a contribution v becomes v * 2^(e+L) with a
 * per-image power of two 2^e from the bound |grad_input| <= KT * HWo * max_k sum_co |W[co,k]| * max|grad_output_b|
 * * max|mask_b| (bound * 2^e < 2^60), split exactly into hi = floor(v * 2^e) (signed, two's complement) and
 * lo = floor(frac * 2^L) (L = 40 while KT * HWo < 2^24, fewer bits beyond), both added with integer atomics and
 * converted to double once at the end; the resolution is about bound * 2^-100.  An image with an inf or NaN in
 * grad_output, weight or its mask gets an all-NaN grad_input.  grad_offset / grad_mask have one writer each, dW
 * is added over fixed pixel ranges in range order, grad_bias in a fixed tree.  Errors: CNB_EINVAL (null pointer,
 * bad shape, too small a workspace), checked before any CUDA call. */
size_t cnb_dcnv2_f64_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw,
                                     int stride, int pad, int dil, int dg);
int cnb_dcnv2_forward_f64(const double *input, const double *offset, const double *mask,
                          const double *weight, const double *bias, double *output,
                          int b, int cin, int h, int w, int cout, int kh, int kw,
                          int stride_h, int stride_w, int pad_h, int pad_w,
                          int dil_h, int dil_w, int deformable_groups, void *stream);
int cnb_dcnv2_backward_f64(const double *input, const double *offset, const double *mask,
                           const double *weight, const double *grad_output,
                           double *grad_input, double *grad_offset, double *grad_mask,
                           double *grad_weight, double *grad_bias,
                           int b, int cin, int h, int w, int cout, int kh, int kw,
                           int stride_h, int stride_w, int pad_h, int pad_w,
                           int dil_h, int dil_w, int deformable_groups,
                           void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------- N4: deformable PSROI pooling
 * Replaces dcn_v2_psroi_pooling_cuda_forward / _backward (src/dcn_v2_cuda.h:35-55,
 * src/cuda/dcn_v2_psroi_pooling_cuda.cu:47-255).  data [b,c,h,w]; rois [num_rois,5]
 * = (batch index, x1, y1, x2, y2); trans [num_rois, channels_trans, part, part] or
 * NULL when no_trans; out / top_count [num_rois, output_dim, pooled, pooled].
 * Backward ACCUMULATES into grad_data / grad_trans, which must arrive zero-filled
 * (dcn_v2_func.py:119-120). */
int cnb_psroi_pooling_forward(const float *data, const float *rois, const float *trans,
                              float *out, float *top_count,
                              int b, int c, int h, int w, int num_rois, int channels_trans,
                              int no_trans, float spatial_scale, int output_dim, int group_size,
                              int pooled_size, int part_size, int sample_per_part, float trans_std,
                              void *stream);
int cnb_psroi_pooling_backward(const float *grad_out, const float *data, const float *rois,
                               const float *trans, const float *top_count,
                               float *grad_data, float *grad_trans,
                               int b, int c, int h, int w, int num_rois, int channels_trans,
                               int no_trans, float spatial_scale, int output_dim, int group_size,
                               int pooled_size, int part_size, int sample_per_part, float trans_std,
                               void *stream);
/* float64 (dcn_v2_psroi_pooling_cuda_double.cu): same arguments with double tensors, rois included; with offsets,
 * output_dim must be a multiple of channels_trans / 2.  The backward is bit-identical run to run: grad_data goes
 * through the two-limb fixed-point sum of cnb_dcnv2_backward_f64 (one bound, N * pooled^2 * max|grad_out|, for
 * the whole call; an inf or NaN anywhere in grad_out makes all of grad_data NaN) and each grad_trans element has
 * one writer that adds its bins' samples in order.  It needs a
 * workspace of cnb_psroi_pooling_f64_workspace_bytes (16-byte aligned) and accumulates into zero-filled
 * grad_data / grad_trans. */
size_t cnb_psroi_pooling_f64_workspace_bytes(int b, int c, int h, int w);
int cnb_psroi_pooling_forward_f64(const double *data, const double *rois, const double *trans,
                                  double *out, double *top_count,
                                  int b, int c, int h, int w, int num_rois, int channels_trans,
                                  int no_trans, double spatial_scale, int output_dim, int group_size,
                                  int pooled_size, int part_size, int sample_per_part, double trans_std,
                                  void *stream);
int cnb_psroi_pooling_backward_f64(const double *grad_out, const double *data, const double *rois,
                                   const double *trans, const double *top_count,
                                   double *grad_data, double *grad_trans,
                                   int b, int c, int h, int w, int num_rois, int channels_trans,
                                   int no_trans, double spatial_scale, int output_dim, int group_size,
                                   int pooled_size, int part_size, int sample_per_part, double trans_std,
                                   void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------- N2: detection post-processing
 * Device-side replacements of utils/post_process.py:83-114 (ctdet_post_process,
 * multi_pose_post_process), external/nms.pyx:77-275 (soft_nms, soft_nms_39) and
 * detectors/ctdet.py:76-92 (merge_outputs): the detections stay on the GPU
 * from decode to the final per-class lists.
 *
 * cnb_post_transform: rows [b,n,d] -> out [b,n,d]; the (x,y) pairs at columns
 *   [a0, a0+2*na) and [b0, b0+2*nb) are mapped through the image's 2x3 float64
 *   matrix trans[b][6] (the inverse affine of utils/image.py:27-60, computed by
 *   the caller on the host), every other column is copied.
 * cnb_group_by_class: dets [b,n,6] (x1,y1,x2,y2,score,class) -> rows [b,n,5]
 *   grouped by class, input order kept inside a class; offsets [b,classes+1].
 * cnb_soft_nms: one list per (image, class): rows image*n_cap +
 *   [offsets[image][c], offsets[image][c+1]) of `rows` ([*,d], d = 5 or 39;
 *   extra columns follow soft_nms_39's swap rule).  The array, rows beyond the
 *   final length included, ends exactly as the reference's in-place routine
 *   leaves it; final_n (nullable, [n_img*lists_per_img]) receives len(keep)
 *   (negative: list longer than n_cap rows, left untouched).  n_cap <= 4096;
 *   shared memory is sized from n_cap (27 B per row).  out may alias rows
 *   only when d == 5.  method 0 hard, 1 linear, 2 gaussian.
 * cnb_topk_keep: keep[b,n_cap] = score >= (max_per_image-th largest score of
 *   the image's offsets[b][classes] rows, NaN of either sign ordered above
 *   +inf as np.partition orders it); thresh (nullable) [b]. */
int cnb_post_transform(const float *rows, float *out, const double *trans, int b, int n, int d,
                       int a0, int na, int b0, int nb, void *stream);
int cnb_group_by_class(const float *dets, int b, int n, int num_classes, float *rows,
                       int32_t *offsets, void *stream);
int cnb_soft_nms(const float *rows, float *out, const int32_t *offsets, int n_img, int lists_per_img,
                 int n_cap, int d, float sigma, float nt, float threshold, int method,
                 int32_t *final_n, void *stream);
int cnb_topk_keep(const float *rows, int b, int n_cap, int d, const int32_t *offsets, int num_classes,
                  int max_per_image, uint8_t *keep, float *thresh, void *stream);

/* The exdet tail (detectors/exdet.py:85-122) and images of more than 4096 rows.
 * cnb_exdet_transform: rows [b,n,d] (d >= 4, n even) -> out [b,n,d]; image i's
 *   rows split in two equal halves, in the second x1 <- out_width - x2 and
 *   x2 <- out_width - x1 (float32), then the pairs (0,1) and (2,3) mapped as
 *   cnb_post_transform maps them; other columns copied.  out must not alias rows.
 * cnb_group_positive_by_class: dets [b,n,d] (x1,y1,x2,y2,score in columns 0-4,
 *   float class id in column cls_col) -> rows [b,n,5] and offsets [b,classes+1]
 *   as cnb_group_by_class, keeping only rows whose score is > 0.
 * cnb_soft_nms_strided: cnb_soft_nms with images of img_stride rows
 *   (<= 32768) and lists of at most list_cap rows (<= 4096; shared memory is
 *   sized from list_cap).  A longer list is left untouched, final_n < 0.
 * cnb_topk_keep_wide: cnb_topk_keep for n_cap <= 32768 rows per image (radix
 *   select instead of a sort; the same threshold).
 * Capacities above those bounds return CNB_EUNSUPPORTED. */
int cnb_exdet_transform(const float *rows, float *out, const double *trans, int b, int n, int d,
                        float out_width, void *stream);
int cnb_group_positive_by_class(const float *dets, int b, int n, int d, int cls_col, int num_classes,
                                float *rows, int32_t *offsets, void *stream);
int cnb_soft_nms_strided(const float *rows, float *out, const int32_t *offsets, int n_img,
                         int lists_per_img, int img_stride, int list_cap, int d, float sigma, float nt,
                         float threshold, int method, int32_t *final_n, void *stream);
int cnb_topk_keep_wide(const float *rows, int b, int n_cap, int d, const int32_t *offsets, int num_classes,
                       int max_per_image, uint8_t *keep, float *thresh, void *stream);

/* The ddd tail (utils/post_process.py:13-80 with utils/ddd_utils.py:66-111, and
 * DddDetector.merge_outputs, detectors/ddd.py:82-88).
 * cnb_ddd_tail: dets [b,n,18] (ddd_decode with wh: x, y, score, rot[8], depth,
 *   dim[3], w, h, class) -> rows [b,n,13] = alpha, x1, y1, x2, y2, dim[3], X, Y, Z,
 *   rot_y, score, grouped by class as cnb_group_by_class groups them, and offsets
 *   [b,classes+1].  trans [b][6]: each image's inverse affine (cnb_post_transform);
 *   calib [b][12]: each image's 3x4 float32 projection matrix.  With cut != 0 only
 *   rows with score > thresh are kept (NaN dropped).  seen (nullable) [b,classes]:
 *   1 where the class has a row before the cut.  d must be 18; outputs must not
 *   overlap any other buffer. */
int cnb_ddd_tail(const float *dets, int b, int n, int d, const double *trans, const float *calib, int num_classes,
                 int cut, float thresh, float *rows, int32_t *offsets, uint8_t *seen, void *stream);

/* ------------------------------------------- N4: detector input pre-processing
 * detectors/base_detector.py:37-65 for one image: cv2.warpAffine(INTER_LINEAR,
 * border 0) + (x/255 - mean)/std + HWC->CHW (+ mirrored copy when flip_test).
 * image_hwc: uint8 [h,w,3] on the device; minv6: the INVERTED 2x3 float64 matrix
 * (output pixel -> source coordinates, as cv::warpAffine derives it from its
 * forward matrix); mean3/std3: fp32; out: [1 or 2, 3, out_h, out_w] fp32.
 * Bit-identical to OpenCV's fixed-point bilinear warp. */
/* cv2.resize(image, (out_w, out_h)) with INTER_LINEAR for uint8 [h,w,3] images (the multi-scale test path of
 * base_detector.py:55), bit-identical to OpenCV's fixed-point filter. */
int cnb_resize_image(const uint8_t *image_hwc, int h, int w, uint8_t *out_hwc, int out_h, int out_w,
                     void *stream);
int cnb_preprocess_image(const uint8_t *image_hwc, int h, int w, const double *minv6,
                         const float *mean3, const float *std3, float *out,
                         int out_h, int out_w, int flip_test, void *stream);
/* cnb_preprocess_image with DddDetector.pre_process's normalisation (detectors/ddd.py:50-51):
 * x / 255 then (x - mean) / std in float32 rather than float64; the same warp. */
int cnb_preprocess_image_f32(const uint8_t *image_hwc, int h, int w, const double *minv6,
                             const float *mean3, const float *std3, float *out,
                             int out_h, int out_w, int flip_test, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CENTERNET_B200_H_ */

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
 * cnb_gather_feat_ex, the loss calls cnb_focal_*_ex / cnb_reg_loss_*ex, cnb_head_forward_bf16 and
 * cnb_dcnv2_forward_block_bf16). */
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
/* DCN block, bf16 inference (opt-in): the whole DCN module -- its 3x3 conv_offset_mask, the chunk / cat / sigmoid of
 * dcn_v2.py and the deformable conv -- plus the optional folded BatchNorm + ReLU of DeformConv, in ONE kernel.  The
 * 27 offset / mask values of every pixel are computed on the bf16 tensor cores inside the kernel and never reach
 * global memory.  Numeric contract:
 *   - x and w_om are rounded once to bf16 (RN); om = the exact-product, fp32-accumulated 3x3 conv (zero padding 1)
 *     of them plus om_bias in fp32, kept in fp32 (never rounded to bf16);
 *   - from om on, the result is exactly cnb_dcnv2_forward_fused_bf16 fed that fp32 om as offset_mask: sigmoid,
 *     geometry, bf16 column rounding, bf16 contraction with fp32 accumulate, fp32 epilogue, output rounded to the
 *     input's dtype;
 *   - only the order of the fp32 sums of the two contractions is free; it is fixed (no atomics), so the output is
 *     bit-identical run to run.
 * Range: kh = kw = 3, stride 1, pad 1, dilation 1, deformable_groups 1, cin % 32 == 0, any cout, b, h, w that
 * cnb_dcnv2_forward_bf16 takes.  Outside it every call returns CNB_EUNSUPPORTED and the two size queries return 0;
 * the caller then runs conv_offset_mask itself and cnb_dcnv2_forward_fused_bf16.
 * w_om: [27][cin][3][3] fp32, rounded and tiled once by cnb_dcnv2_prepare_om_weights_bf16 into om_tiles
 * (cnb_dcnv2_om_tiles_bytes, 16-byte aligned), reused while the weight does not change.  om_bias [27] fp32 (NULL: no
 * bias).  wtiles / bias / bn_scale / bn_shift / relu as cnb_dcnv2_forward_fused_bf16.  input: [b,cin,h,w] of
 * input_dtype (CNB_DTYPE_F32 or CNB_DTYPE_BF16), [b][h*w][cin] when input_channels_last != 0 (a bf16 one is read in
 * place); 16-byte aligned.  output: [b,cout,h,w] NCHW of input_dtype.  workspace: cnb_dcnv2_block_workspace_bytes
 * (16-byte aligned).  Errors, checked before any CUDA call: CNB_EINVAL for a null pointer, an unknown dtype code, a
 * bad shape or a misaligned buffer; CNB_EUNSUPPORTED outside the range; CNB_EWORKSPACE for too small a buffer. */
size_t cnb_dcnv2_om_tiles_bytes(int cin, int kh, int kw, int dg);
int cnb_dcnv2_prepare_om_weights_bf16(const float *w_om, int cin, int kh, int kw, int dg,
                                      void *om_tiles, size_t om_tiles_bytes, void *stream);
size_t cnb_dcnv2_block_workspace_bytes(int b, int cin, int cout, int h, int w, int kh, int kw,
                                       int stride, int pad, int dil, int dg);
int cnb_dcnv2_forward_block_bf16(const void *input, int input_dtype, int input_channels_last,
                                 const void *om_tiles, const float *om_bias,
                                 const void *wtiles, const float *bias,
                                 const float *bn_scale, const float *bn_shift, int relu, void *output,
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

/* ------------------------------------- output heads: 3x3 conv, ReLU and 1x1 conv in one bf16 kernel (inference)
 * Every DLASeg / PoseResNet head is nn.Sequential(Conv2d(cin, cmid, 3, padding=1), ReLU, Conv2d(cmid, cout, 1))
 * (pose_dla_dcn.py:448-459, resnet_dcn.py:157-165, msra_resnet.py:135-143).  cnb_head_forward_bf16 runs all three in
 * one kernel on bf16 wgmma; the cmid-channel intermediate stays on chip.  Numeric contract: the result is that of
 *   1. rounding the input, w1 and w2 once to bf16 (RN);
 *   2. an exact-product, fp32-accumulated 3x3 conv (zero padding 1) plus b1;
 *   3. ReLU (NaN stays NaN, as torch.relu), then one rounding to bf16 (RN);
 *   4. a fp32-accumulated 1x1 conv plus b2;
 *   5. rounding to the input's dtype (fp32: none; bf16: RN).
 * Only the order of the fp32 sums is free; it is fixed, so the output is bit-identical run to run (no atomics).
 * Weights: w1 [cmid][cin][3][3] and w2 [cout][cmid] fp32, rounded and tiled once by cnb_head_prepare_weights_bf16 into
 * w1t (cnb_head_w1t_bytes) and w2t (cnb_head_w2t_bytes), both 16-byte aligned, reused while the weights do not change.
 * input: [b,cin,h,w] of input_dtype (CNB_DTYPE_F32 or CNB_DTYPE_BF16), NCHW, or [b][h][w][cin] (torch channels_last)
 * when input_channels_last != 0; 16-byte aligned.  A bf16 channels-last input is read in place, any other is first
 * copied to bf16 channels-last into the workspace (cnb_head_workspace_bytes; 0 when none is needed).  b1 [cmid] and
 * b2 [cout] are fp32.  out: [b,cout,h,w] of input_dtype, in the input's layout.
 * Range: cin and cmid multiples of 32, cmid <= 256, 1 <= cout <= 256, any b, h, w >= 1 within 32-bit indexing; else
 * CNB_EUNSUPPORTED (and the size queries return 0).  Errors, checked before any CUDA call: CNB_EINVAL for a null
 * pointer, an unknown dtype code, a bad shape or a misaligned buffer; CNB_EWORKSPACE for too small a buffer. */
size_t cnb_head_w1t_bytes(int cin, int cmid);
size_t cnb_head_w2t_bytes(int cmid, int cout);
int cnb_head_prepare_weights_bf16(const float *w1, const float *w2, int cin, int cmid, int cout,
                                  void *w1t, size_t w1t_bytes, void *w2t, size_t w2t_bytes, void *stream);
size_t cnb_head_workspace_bytes(int b, int cin, int h, int w, int input_dtype, int input_channels_last);
int cnb_head_forward_bf16(const void *input, int input_dtype, int input_channels_last,
                          const void *w1t, const float *b1, const void *w2t, const float *b2, void *out,
                          int b, int cin, int h, int w, int cmid, int cout,
                          void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------- IDA up-sampling step of DLASeg: depthwise transposed conv + skip add (inference)
 * Every step of pose_dla_dcn's IDAUp is node(up(proj(x)) + skip), with up = ConvTranspose2d(C, C, 2f, stride f,
 * padding f/2, groups C, no bias).  cnb_ida_up_add computes
 *   out = conv_transpose2d(p, w, stride=f, padding=f/2, groups=c) + skip
 * in one pass; the up-sampled map never reaches HBM.  Numeric contract:
 *   1. p and w are widened exactly to fp32;
 *   2. the up value of an output element is an fp32 FMA chain over its valid taps (at most 2 x 2), starting from 0,
 *      in the fixed order (row q-1, column q-1), (q-1, q), (q, q-1), (q, q), q = (y + f/2) / f per axis;
 *   3. skip, widened exactly, is added to it in fp32;
 *   4. the sum is rounded once (RN) to the output dtype.
 * Out-of-range taps are not computed (never multiplied by anything); Inf / NaN propagate through valid taps as in
 * IEEE arithmetic.  The unfused bf16 module rounds twice (after the up and after the add) and cuDNN runs an fp32
 * conv in TF32 by default, so the two differ slightly; this result is the more accurate one.  There are no atomics
 * and no workspace: the output is bit-identical run to run.
 * p: [b,c,hp,wp] and skip: [b,c,f*hp,f*wp], both of dtype (CNB_DTYPE_F32 or CNB_DTYPE_BF16), each NCHW or, when its
 * *_channels_last is 1, [b][h][w][c] (torch channels_last).  w: [c][2f][2f] fp32.  out: [b,c,f*hp,f*wp] of dtype, in
 * the layout out_channels_last picks; it must not overlap p or skip.  skip and out 16-byte aligned.
 * Range: f in {2, 4, 8}, any c >= 1 and b, hp, wp >= 1 within 32-bit indexing; else CNB_EUNSUPPORTED.  Errors,
 * checked before any CUDA call: CNB_EINVAL for a null or misaligned pointer, an unknown dtype code, a channels_last
 * flag other than 0 / 1 or a bad shape. */
int cnb_ida_up_add(const void *p, int dtype, int p_channels_last, const float *w, int f, const void *skip,
                   int skip_channels_last, void *out, int out_channels_last, int b, int c, int hp, int wp,
                   void *stream);

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

/* ------------------------------------------------ training input of the ctdet sampler
 * CTDetDataset.__getitem__ (datasets/sample/ctdet.py:29-145) after the random draws, for a whole batch.
 *
 * cnb_train_images: per image b, the uint8 BGR source [h_b, w_b, 3] at src + src_off[b] (src_hw[b] = (h_b, w_b)),
 * mirrored (img[:, ::-1]) when flip[b] != 0 -- sampled at mirrored columns, never materialised -- and warped with
 * the INVERTED 2x3 float64 matrix minv6[b] (cv2.warpAffine INTER_LINEAR, border 0, OpenCV's fixed point as in
 * cnb_preprocess_image); then x / 255, color_aug (utils/image.py:198-230) and (x - mean) / std, all float32.
 *   order: NULL = no colour augmentation for any image; else order[b] = -1 (off for image b) or the blend order
 *     0..5 = BCS, BSC, CBS, CSB, SBC, SCB (B brightness_, C contrast_, S saturation_, applied left to right);
 *   blend[b, 6] = (a, b) of B, C, S with a = f32(alpha), b = f32(1 - alpha) (the difference in float64);
 *   light[b, 3] = np.dot(eig_vec, eig_val * normal(0.1, 3)) in float64.
 * Per pixel: gs = fma(r, 0.299f, fma(b, 0.114f, g * 0.587f)); gs_mean = numpy's pairwise float32 sum of gs over
 * the out_h * out_w pixels (its exact tree) / n; B: x * a; C: x * a + f32(gs_mean * b); S: x * a + f32(gs * b);
 * lighting f32(f64(x) + light[c]); each step a rounded float32 operation unless stated.
 *   out: [b, 3, out_h, out_w] (channels_last == 0) or [b, out_h, out_w, 3] (channels_last == 1) of out_dtype
 *     (CNB_DTYPE_F32 / _BF16 / _F16; half types are the fp32 value rounded once to nearest even);
 *   mean3 / std3: fp32 on the device.  Every image has the one output size of the batch.
 * With colour augmentation two launches (the grey sums, then the image), else one; the workspace
 * (cnb_train_images_workspace_bytes, 0 for a bad shape) holds the grey partial sums.  No atomics: the output is
 * identical run to run.  Errors, checked before any CUDA call: CNB_EINVAL for a null pointer, a bad shape, an
 * unknown dtype code or a channels_last other than 0 / 1; CNB_EUNSUPPORTED for more than CNB_TRAIN_MAX_PIXELS
 * output pixels; CNB_EWORKSPACE for too small a workspace.  The per-image records live on the device, out of
 * the host's sight: an image whose side lies outside [1, 32767] (the warp clamps source coordinates there) or
 * whose order code is not in -1..5 is written as quiet NaN.  centernet_b200.train_input rejects both first.
 *
 * cnb_ctdet_targets: ctdet.py:99-127 for m = max_objs slots per image, one thread per (image, slot): slot k <
 * min(num_objs[b], m) holds the float32 corners boxes[b, k] = [x, y, x + w, y + h] and the class cls[b, k] in
 * [0, num_classes); they are mirrored when flip[b] != 0 (width src_hw[b][1]), mapped by the FORWARD 2x3 float64
 * trans6[b] (get_affine_transform(c, s, 0, [out_w, out_h]), float64 t0 x + t1 y + t2 rounded to float32),
 * clipped, and a box with h > 0 and w > 0 gets wh [b,m,2] f32, ind [b,m] i64, reg [b,m,2] f32, reg_mask [b,m]
 * u8 = 1, cat_spec_wh [b,m,2*num_classes] f32 / cat_spec_mask u8 (both NULL to skip) and the FocalSplatLoss
 * lists obj_cls / obj_cx / obj_cy / obj_radius i32 and obj_valid u8 [b,m] (ct_int, max(0, int(gaussian_radius(
 * ceil(h), ceil(w)))) in float64, reg_mask); every other slot is zero.  Errors, checked before any CUDA call:
 * CNB_EINVAL for a null pointer, only one of the cat_spec pair or a bad shape.
 *
 * cnb_multi_pose_targets: multi_pose.py:104-160 for m = max_objs slots per image and J = num_joints, one thread per
 * (image, slot) looping over the joints, R = out_res.  Slot k < min(num_objs[b], m) holds the float32 corners
 * boxes[b, k] (as cnb_ctdet_targets), the class cls[b, k] and the keypoints kps[b, k] [J, 3] (x, y, visibility,
 * float32; visibilities finite and >= 0).  When flip[b] != 0 the box and every joint's x are mirrored (width -
 * x - 1 in float32, width src_hw[b][1]) and new joint j is old joint flip_perm[j].  The box goes through the
 * FORWARD trans6[b] (rot 0) and is clipped to [0, R - 1]; the slot gets targets when (h > 0 && w > 0) or
 * rotated[b] != 0: wh [b,m,2] f32, ind [b,m] i64 = ct_int.y R + ct_int.x, reg [b,m,2] f32 = ct - ct_int and the
 * centre lists obj_cls / obj_cx / obj_cy / obj_radius i32 and obj_valid u8 = 1 [b,m] (radius max(0, int(
 * gaussian_radius(ceil(h), ceil(w)))) in float64); reg_mask [b,m] u8 = 1 only when some visibility is non-zero
 * and the image is not rotated.  Each joint with visibility > 0 is mapped by trans_rot6[b] (float64 t0 x + t1 y +
 * t2 rounded to float32) and counts when 0 <= x < R and 0 <= y < R: hps [b,m,2J] f32 = pt - ct_int, hps_mask
 * [b,m,2J] u8 = 1 on both entries unless rotated, hp_offset [b,m*J,2] f32 = pt - pt_int, hp_ind [b,m*J] i64 =
 * pt_int.y R + pt_int.x, hp_mask [b,m*J] i64 = 1 (kept on rotated images, as there), and the joint lists hp_cx /
 * hp_cy / hp_radius i32, hp_valid u8 [b,J,m] (pt_int and the slot's radius), a [b*J, m] list of class 0 that
 * splat_gaussian / FocalSplatLoss read as hm_hp [b*J, 1, R, R].  Differences float32 - int32 are one rounding of
 * the exact difference.  Every other entry is zero.  No atomics: the output is identical run to run.  Errors,
 * checked before any CUDA call: CNB_EINVAL for a null pointer or a bad shape.
 *
 * cnb_ddd_targets: ddd.py:86-140 for m = max_objs slots per image, C = num_classes, and the dense hm; two launches
 * (targets: one thread per (image, slot); hm: one CTA per 4 rows of an image), no atomics, no workspace.  Slot k <
 * min(num_objs[b], m) holds the float32 corners boxes[b, k], the class cls[b, k], alpha[b, k] (float64, after
 * _convert_alpha), depth[b, k] and dim[b, k, 3] (float32).  A class <= -99, or one outside [0, C), -1 and
 * [-C - 1, -2], is skipped.  The box goes through the FORWARD trans6[b] (get_affine_transform(c, s, 0, [out_w,
 * out_h]), float64 t0 x + t1 y + t2 rounded to float32, no flip) and is clipped to [0, out_w - 1] x [0, out_h - 1];
 * nothing happens unless h > 0 and w > 0.  Its radius is max(0, int(gaussian_radius((h, w)))) evaluated on float32
 * h, w as numpy does: every operation float32, b ** 2 the C library's powf(b, 2) (glibc's algorithm, restated) --
 * cnb_ddd_gaussian_radius returns it for n pairs, for testing.  ct = f32((x0 + x1) / 2, (y0 + y1) / 2), ct_int its
 * truncation.
 *   cls in [0, C): draw_umich_gaussian(hm[cls], ct, r) and the targets: wh [b,m,2] f32 = (w, h), rotbin [b,m,2] i64
 *     / rotres [b,m,2] f32 (alpha < pi/6 or > 5pi/6: bin 0, f32(alpha + pi/2); alpha > -pi/6 or < -5pi/6: bin 1,
 *     f32(alpha - pi/2); float64 compares), dep [b,m,1] f32 = depth, dim_out [b,m,3] f32 = dim, ind [b,m] i64 =
 *     ct_int.y out_w + ct_int.x, reg [b,m,2] f32 = ct - ct_int, rot_mask [b,m] u8 = 1, reg_mask [b,m] u8 = 1 only
 *     when aug[b] == 0.
 *   cls < 0 (ignore; classes -cls - 2, or all for -1): no targets.  rect_mask == 1: hm[ignore, int(y0):int(y1) + 1,
 *     int(x0):int(x1) + 1] = f32(0.9999); rect_mask == 0: the Gaussian on each ignore class, then hm[ignore,
 *     ct_int.y, ct_int.x] = f32(0.9999).
 * hm [b,C,out_h,out_w] f32 is the result of doing that in slot order on a zero map (Gaussians as np.maximum of the
 * float64 values rounded to float32, overwrites as assignments), whatever the order.  Every other entry is zero.
 * Errors, checked before any CUDA call: CNB_EINVAL for a null pointer, a bad shape or a rect_mask other than 0 / 1;
 * CNB_EUNSUPPORTED for m > 128.
 *
 * cnb_exdet_targets: exdet.py:95-129 for m = max_objs slots per image, R = out_res; one launch, one thread per
 * (image, slot), no atomics, no workspace.  Slot k < min(num_objs[b], m) holds the float32 extreme points pts[b, k]
 * [4, 2] in the order t, l, b, r (finite) and the class cls[b, k] in [0, C).  When flip[b] != 0 every x becomes
 * width - x - 1 in float32 (width src_hw[b][1]) and points 1 and 3 (l, r) swap.  Each point goes through the
 * FORWARD trans6[b] (get_affine_transform(c, s, 0, [R, R]), float64 t0 x + t1 y + t2 rounded to float32) and is
 * clipped to [0, R - 1] as np.clip does (-0 stays -0).  h = b.y - t.y and w = r.x - l.x in float32; nothing is
 * written unless h > 0 and w > 0.  Then the radius max(0, int(gaussian_radius(ceil(h), ceil(w)))) in float64, shared
 * by all five parts; per part p, pt_int the truncation of the point: reg [4,b,m,2] f32 = pt - pt_int, ind [4,b,m] i64
 * = pt_int.y R + pt_int.x, and the lists ex_cls (cls, or 0 when agnostic_ex == 1) / ex_cx / ex_cy / ex_radius i32
 * and ex_valid u8 [4,b,m], each part a [b, m] list set of splat_gaussian / FocalSplatLoss; the centre ct =
 * (int(f32(r.x + l.x) / 2), int(f32(t.y + b.y) / 2)) goes to obj_cls (cls) / obj_cx / obj_cy / obj_radius i32 and
 * obj_valid u8 [b,m]; reg_mask [b,m] u8 = 1.  Every other entry is zero.  Errors, checked before any CUDA call:
 * CNB_EINVAL for a null pointer, a bad shape or an agnostic_ex other than 0 / 1; CNB_EUNSUPPORTED for m > 128. */
#define CNB_TRAIN_MAX_PIXELS 4194304
size_t cnb_train_images_workspace_bytes(int b, int out_h, int out_w);
int cnb_train_images(const uint8_t *src, const int64_t *src_off, const int32_t *src_hw, const double *minv6,
                     const uint8_t *flip, const int32_t *order, const float *blend, const double *light,
                     const float *mean3, const float *std3, int b, int out_h, int out_w, void *out, int out_dtype,
                     int channels_last, void *workspace, size_t workspace_bytes, void *stream);
int cnb_ctdet_targets(const float *boxes, const int32_t *cls, const int32_t *num_objs, const uint8_t *flip,
                      const int32_t *src_hw, const double *trans6, int b, int m, int num_classes, int out_h,
                      int out_w, float *wh, int64_t *ind, float *reg, uint8_t *reg_mask, float *cat_spec_wh,
                      uint8_t *cat_spec_mask, int32_t *obj_cls, int32_t *obj_cx, int32_t *obj_cy,
                      int32_t *obj_radius, uint8_t *obj_valid, void *stream);
int cnb_multi_pose_targets(const float *boxes, const int32_t *cls, const int32_t *num_objs, const float *kps,
                           const uint8_t *flip, const uint8_t *rotated, const int32_t *src_hw, const double *trans6,
                           const double *trans_rot6, const int32_t *flip_perm, int b, int m, int num_joints,
                           int out_res, float *wh, int64_t *ind, float *reg, uint8_t *reg_mask, float *hps,
                           uint8_t *hps_mask, float *hp_offset, int64_t *hp_ind, int64_t *hp_mask, int32_t *obj_cls,
                           int32_t *obj_cx, int32_t *obj_cy, int32_t *obj_radius, uint8_t *obj_valid, int32_t *hp_cx,
                           int32_t *hp_cy, int32_t *hp_radius, uint8_t *hp_valid, void *stream);
int cnb_ddd_targets(const float *boxes, const int32_t *cls, const int32_t *num_objs, const double *alpha,
                    const float *depth, const float *dim, const uint8_t *aug, const double *trans6, int b, int m,
                    int num_classes, int out_h, int out_w, int rect_mask, float *hm, float *dep, float *dim_out,
                    int64_t *ind, int64_t *rotbin, float *rotres, uint8_t *reg_mask, uint8_t *rot_mask, float *wh,
                    float *reg, void *stream);
int cnb_ddd_gaussian_radius(const float *h, const float *w, int n, int32_t *radius, void *stream);
int cnb_exdet_targets(const float *pts, const int32_t *cls, const int32_t *num_objs, const uint8_t *flip,
                      const int32_t *src_hw, const double *trans6, int b, int m, int out_res, int agnostic_ex,
                      float *reg, int64_t *ind, uint8_t *reg_mask, int32_t *obj_cls, int32_t *obj_cx, int32_t *obj_cy,
                      int32_t *obj_radius, uint8_t *obj_valid, int32_t *ex_cls, int32_t *ex_cx, int32_t *ex_cy,
                      int32_t *ex_radius, uint8_t *ex_valid, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CENTERNET_B200_H_ */

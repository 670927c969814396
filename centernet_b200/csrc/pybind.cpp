// Thin pybind11 layer over the C ABI of include/centernet_b200.h.
// Pointers cross as integers (tensor.data_ptr()); no torch types here, so the module
// builds with g++ alone and the C ABI stays the real boundary.  A non-zero status
// becomes a Python RuntimeError carrying cnb_last_error() -- the counterpart of the
// reference's THError -> RuntimeError path (DCNv2/src/dcn_v2_cuda.c:20-38).
#include <pybind11/pybind11.h>
#include <stdexcept>
#include <string>
#include "../../include/centernet_b200.h"

namespace py = pybind11;
typedef uintptr_t P;

template <typename T>
static inline T *ptr(P p) { return reinterpret_cast<T *>(p); }

static void check(int rc, const char *fn) {
  if (rc == CNB_OK) return;
  std::string msg = std::string(fn) + " failed (status " + std::to_string(rc) + "): " + cnb_last_error();
  if (rc == CNB_EUNSUPPORTED) {  // valid request outside the implemented envelope
    PyErr_SetString(PyExc_NotImplementedError, msg.c_str());
    throw py::error_already_set();
  }
  throw std::runtime_error(msg);
}

PYBIND11_MODULE(_C, m) {
  m.doc() = "centernet_b200 C-ABI bindings (pointers as ints)";
  m.attr("OK") = CNB_OK;
  m.attr("EINVAL") = CNB_EINVAL;
  m.attr("EUNSUPPORTED") = CNB_EUNSUPPORTED;
  m.attr("ECUDA") = CNB_ECUDA;
  m.attr("EWORKSPACE") = CNB_EWORKSPACE;
  m.def("version", &cnb_version);
  m.def("last_error", []() { return std::string(cnb_last_error()); });
  m.def("launch_count", &cnb_launch_count);

  m.def("nms", [](P heat, P out, int n, int c, int h, int w, P stream) {
    check(cnb_nms(ptr<const float>(heat), ptr<float>(out), n, c, h, w, ptr<void>(stream)), "cnb_nms");
  });
  m.def("topk_workspace_bytes", &cnb_topk_workspace_bytes);
  m.def("topk", [](P scores, int b, int c, int h, int w, int k, int fuse_nms, P os, P oi, P oc, P oy, P ox, P ws,
                   size_t wsb, P stream) {
    check(cnb_topk(ptr<const float>(scores), b, c, h, w, k, fuse_nms, ptr<float>(os), ptr<int64_t>(oi),
                   ptr<int32_t>(oc), ptr<float>(oy), ptr<float>(ox), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_topk");
  });
  m.def("select_plan_info", [](P src, int n_img, int c, int h, int w, int k, int nms, int elem_size) {
    int v[CNB_SELECT_PLAN_FIELDS];
    check(cnb_select_plan_info(ptr<const void>(src), n_img, c, h, w, k, nms, elem_size, v, CNB_SELECT_PLAN_FIELDS),
          "cnb_select_plan_info");
    static const char *names[CNB_SELECT_PLAN_FIELDS] = {"hot", "n_cta", "wb", "max_slots", "seg_cap",
                                                         "fused_finalize", "use_tma", "rb", "local_img"};
    py::dict d;
    for (int i = 0; i < CNB_SELECT_PLAN_FIELDS; ++i) d[names[i]] = v[i];
    return d;
  });
  m.def("topk_channel", [](P scores, int b, int c, int h, int w, int k, int fuse_nms, P os, P oi, P oy, P ox, P ws,
                           size_t wsb, P stream) {
    check(cnb_topk_channel(ptr<const float>(scores), b, c, h, w, k, fuse_nms, ptr<float>(os), ptr<int64_t>(oi),
                           ptr<float>(oy), ptr<float>(ox), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_topk_channel");
  });
  m.def("gather_feat", [](P feat, P ind, P out, int b, int c, int hw, int mm, P stream) {
    check(cnb_gather_feat(ptr<const float>(feat), ptr<const int64_t>(ind), ptr<float>(out), b, c, hw, mm,
                          ptr<void>(stream)),
          "cnb_gather_feat");
  });
  m.def("gather_feat_backward", [](P gout, P ind, P gfeat, int b, int c, int hw, int mm, P stream) {
    check(cnb_gather_feat_backward(ptr<const float>(gout), ptr<const int64_t>(ind), ptr<float>(gfeat), b, c, hw, mm,
                                   ptr<void>(stream)),
          "cnb_gather_feat_backward");
  });
  m.def("ctdet_decode", [](P heat, P wh, P reg, int cat, int b, int c, int h, int w, int k, P dets, P ws, size_t wsb,
                           P stream) {
    check(cnb_ctdet_decode(ptr<const float>(heat), ptr<const float>(wh), ptr<const float>(reg), cat, b, c, h, w, k,
                           ptr<float>(dets), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_ctdet_decode");
  });
  m.def("ctdet_logits_workspace_bytes", [](P hm, int b, int c, int h, int w, int k) {
    return cnb_ctdet_logits_workspace_bytes(ptr<const float>(hm), b, c, h, w, k);
  });
  m.def("ctdet_decode_logits", [](P hm, P wh, P reg, int cat, int b, int c, int h, int w, int k, P dets, P ws,
                                  size_t wsb, P stream) {
    check(cnb_ctdet_decode_logits(ptr<const float>(hm), ptr<const float>(wh), ptr<const float>(reg), cat, b, c, h, w,
                                  k, ptr<float>(dets), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_ctdet_decode_logits");
  });
  m.def("ctdet_decode_ex_workspace_bytes", [](P heat, int dt, int logits, int b, int c, int h, int w, int k) {
    return cnb_ctdet_decode_ex_workspace_bytes(ptr<const void>(heat), dt, logits, b, c, h, w, k);
  });
  m.def("ctdet_decode_ex", [](P heat, int heat_dt, int logits, P wh, int wh_dt, P reg, int reg_dt, int cat, int b,
                              int c, int h, int w, int k, P dets, P ws, size_t wsb, P stream) {
    check(cnb_ctdet_decode_ex(ptr<const void>(heat), heat_dt, logits, ptr<const void>(wh), wh_dt, ptr<const void>(reg),
                              reg_dt, cat, b, c, h, w, k, ptr<float>(dets), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_ctdet_decode_ex");
  });
  m.def("flip_merge_ex", [](P src, int dt, P dst, int n, int c, int h, int w, int sig, P perm, P sign, P stream) {
    check(cnb_flip_merge_ex(ptr<const void>(src), dt, ptr<float>(dst), n, c, h, w, sig, ptr<const int32_t>(perm),
                            ptr<const float>(sign), ptr<void>(stream)),
          "cnb_flip_merge_ex");
  });
  m.def("sigmoid", [](P x, P out, long long n, P stream) {
    check(cnb_sigmoid(ptr<const float>(x), ptr<float>(out), n, ptr<void>(stream)), "cnb_sigmoid");
  });
  m.def("flip_merge", [](P src, P dst, int n, int c, int h, int w, int sig, P perm, P sign, P stream) {
    check(cnb_flip_merge(ptr<const float>(src), ptr<float>(dst), n, c, h, w, sig, ptr<const int32_t>(perm),
                         ptr<const float>(sign), ptr<void>(stream)),
          "cnb_flip_merge");
  });
  m.def("psroi_pooling_forward", [](P data, P rois, P trans, P out, P cnt, int b, int c, int h, int w, int n, int ct,
                                    int no_trans, float scale, int od, int gs, int ps, int part, int spp, float tstd,
                                    P stream) {
    check(cnb_psroi_pooling_forward(ptr<const float>(data), ptr<const float>(rois), ptr<const float>(trans),
                                    ptr<float>(out), ptr<float>(cnt), b, c, h, w, n, ct, no_trans, scale, od, gs, ps,
                                    part, spp, tstd, ptr<void>(stream)),
          "cnb_psroi_pooling_forward");
  });
  m.def("psroi_pooling_backward", [](P gout, P data, P rois, P trans, P cnt, P gdata, P gtrans, int b, int c, int h,
                                     int w, int n, int ct, int no_trans, float scale, int od, int gs, int ps, int part,
                                     int spp, float tstd, P stream) {
    check(cnb_psroi_pooling_backward(ptr<const float>(gout), ptr<const float>(data), ptr<const float>(rois),
                                     ptr<const float>(trans), ptr<const float>(cnt), ptr<float>(gdata),
                                     ptr<float>(gtrans), b, c, h, w, n, ct, no_trans, scale, od, gs, ps, part, spp,
                                     tstd, ptr<void>(stream)),
          "cnb_psroi_pooling_backward");
  });
  m.def("psroi_pooling_f64_workspace_bytes", &cnb_psroi_pooling_f64_workspace_bytes);
  m.def("psroi_pooling_forward_f64", [](P data, P rois, P trans, P out, P cnt, int b, int c, int h, int w, int n,
                                        int ct, int no_trans, double scale, int od, int gs, int ps, int part, int spp,
                                        double tstd, P stream) {
    check(cnb_psroi_pooling_forward_f64(ptr<const double>(data), ptr<const double>(rois), ptr<const double>(trans),
                                        ptr<double>(out), ptr<double>(cnt), b, c, h, w, n, ct, no_trans, scale, od, gs,
                                        ps, part, spp, tstd, ptr<void>(stream)),
          "cnb_psroi_pooling_forward_f64");
  });
  m.def("psroi_pooling_backward_f64", [](P gout, P data, P rois, P trans, P cnt, P gdata, P gtrans, int b, int c,
                                         int h, int w, int n, int ct, int no_trans, double scale, int od, int gs,
                                         int ps, int part, int spp, double tstd, P ws, size_t wsb, P stream) {
    check(cnb_psroi_pooling_backward_f64(ptr<const double>(gout), ptr<const double>(data), ptr<const double>(rois),
                                         ptr<const double>(trans), ptr<const double>(cnt), ptr<double>(gdata),
                                         ptr<double>(gtrans), b, c, h, w, n, ct, no_trans, scale, od, gs, ps, part,
                                         spp, tstd, ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_psroi_pooling_backward_f64");
  });
  m.def("dcnv2_f64_workspace_bytes", &cnb_dcnv2_f64_workspace_bytes);
  m.def("dcnv2_forward_f64", [](P input, P offset, P mask, P weight, P bias, P output, int b, int cin, int h, int w,
                                int cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int dg,
                                P stream) {
    check(cnb_dcnv2_forward_f64(ptr<const double>(input), ptr<const double>(offset), ptr<const double>(mask),
                                ptr<const double>(weight), ptr<const double>(bias), ptr<double>(output), b, cin, h, w,
                                cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, ptr<void>(stream)),
          "cnb_dcnv2_forward_f64");
  });
  m.def("dcnv2_backward_f64", [](P input, P offset, P mask, P weight, P gout, P gin, P goff, P gmask, P gw, P gb,
                                 int b, int cin, int h, int w, int cout, int kh, int kw, int sh, int sw, int ph,
                                 int pw, int dh, int dw, int dg, P ws, size_t wsb, P stream) {
    check(cnb_dcnv2_backward_f64(ptr<const double>(input), ptr<const double>(offset), ptr<const double>(mask),
                                 ptr<const double>(weight), ptr<const double>(gout), ptr<double>(gin),
                                 ptr<double>(goff), ptr<double>(gmask), ptr<double>(gw), ptr<double>(gb), b, cin, h, w,
                                 cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_dcnv2_backward_f64");
  });
  m.def("ddd_decode", [](P heat, P rot, P depth, P dim, P wh, P reg, int b, int c, int h, int w, int k, P dets, P ws,
                         size_t wsb, P stream) {
    check(cnb_ddd_decode(ptr<const float>(heat), ptr<const float>(rot), ptr<const float>(depth),
                         ptr<const float>(dim), ptr<const float>(wh), ptr<const float>(reg), b, c, h, w, k,
                         ptr<float>(dets), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_ddd_decode");
  });
  m.def("ddd_decode_ex_workspace_bytes", [](P heat, int dt, int logits, int b, int c, int h, int w, int k) {
    return cnb_ddd_decode_ex_workspace_bytes(ptr<const void>(heat), dt, logits, b, c, h, w, k);
  });
  m.def("ddd_decode_ex", [](P heat, int heat_dt, int logits, P rot, int rot_dt, P depth, int depth_dt, P dim,
                            int dim_dt, P wh, int wh_dt, P reg, int reg_dt, int b, int c, int h, int w, int k, P dets,
                            P ws, size_t wsb, P stream) {
    check(cnb_ddd_decode_ex(ptr<const void>(heat), heat_dt, logits, ptr<const void>(rot), rot_dt,
                            ptr<const void>(depth), depth_dt, ptr<const void>(dim), dim_dt, ptr<const void>(wh), wh_dt,
                            ptr<const void>(reg), reg_dt, b, c, h, w, k, ptr<float>(dets), ptr<void>(ws), wsb,
                            ptr<void>(stream)),
          "cnb_ddd_decode_ex");
  });
  m.def("multi_pose_workspace_bytes", &cnb_multi_pose_workspace_bytes);
  m.def("multi_pose_decode_ex_workspace_bytes", [](P heat, int heat_dt, P hm_hp, int hm_hp_dt, int logits, int b,
                                                   int c, int j, int h, int w, int k) {
    return cnb_multi_pose_decode_ex_workspace_bytes(ptr<const void>(heat), heat_dt, ptr<const void>(hm_hp), hm_hp_dt,
                                                    logits, b, c, j, h, w, k);
  });
  m.def("multi_pose_decode_ex", [](P heat, int heat_dt, int logits, P wh, int wh_dt, P kps, int kps_dt, P reg,
                                   int reg_dt, P hm_hp, int hm_hp_dt, P hp_off, int hp_off_dt, int b, int c, int j,
                                   int h, int w, int k, P dets, P ws, size_t wsb, P stream) {
    check(cnb_multi_pose_decode_ex(ptr<const void>(heat), heat_dt, logits, ptr<const void>(wh), wh_dt,
                                   ptr<const void>(kps), kps_dt, ptr<const void>(reg), reg_dt, ptr<const void>(hm_hp),
                                   hm_hp_dt, ptr<const void>(hp_off), hp_off_dt, b, c, j, h, w, k, ptr<float>(dets),
                                   ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_multi_pose_decode_ex");
  });
  m.def("multi_pose_decode", [](P heat, P wh, P kps, P reg, P hm_hp, P hp_off, int b, int c, int j, int h, int w,
                                int k, P dets, P ws, size_t wsb, P stream) {
    check(cnb_multi_pose_decode(ptr<const float>(heat), ptr<const float>(wh), ptr<const float>(kps),
                                ptr<const float>(reg), ptr<const float>(hm_hp), ptr<const float>(hp_off), b, c, j, h,
                                w, k, ptr<float>(dets), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_multi_pose_decode");
  });
  m.def("edge_aggregate", [](P heat, P out, int n, int c, int h, int w, float wt, int horizontal, P stream) {
    check(cnb_edge_aggregate(ptr<const float>(heat), ptr<float>(out), n, c, h, w, wt, horizontal, ptr<void>(stream)),
          "cnb_edge_aggregate");
  });
  m.def("edge_aggregate_ex", [](P heat, int dt, int sig, P out, int n, int c, int h, int w, float wt, int horizontal,
                                P stream) {
    check(cnb_edge_aggregate_ex(ptr<const void>(heat), dt, sig, ptr<float>(out), n, c, h, w, wt, horizontal,
                                ptr<void>(stream)),
          "cnb_edge_aggregate_ex");
  });
  m.def("exct_workspace_bytes", &cnb_exct_workspace_bytes);
  m.def("exct_groups", &cnb_exct_groups);
  m.def("exct_decode_ex_workspace_bytes", [](P t, P l, P b_, P r, int t_dt, int l_dt, int b_dt, int r_dt, int ct_dt,
                                             int tr_dt, int lr_dt, int br_dt, int rr_dt, int logits, int b, int c,
                                             int cc, int h, int w, int k, float aw, int nd, int agn) {
    return cnb_exct_decode_ex_workspace_bytes(ptr<const void>(t), ptr<const void>(l), ptr<const void>(b_),
                                              ptr<const void>(r), t_dt, l_dt, b_dt, r_dt, ct_dt, tr_dt, lr_dt, br_dt,
                                              rr_dt, logits, b, c, cc, h, w, k, aw, nd, agn);
  });
  m.def("exct_decode_ex", [](P t, int t_dt, P l, int l_dt, P b_, int b_dt, P r, int r_dt, P ct, int ct_dt, P tr,
                             int tr_dt, P lr, int lr_dt, P br, int br_dt, P rr, int rr_dt, int logits, int b, int c,
                             int cc, int h, int w, int k, float st, float cth, float aw, int nd, int agn, P dets, P ws,
                             size_t wsb, P stream) {
    check(cnb_exct_decode_ex(ptr<const void>(t), t_dt, ptr<const void>(l), l_dt, ptr<const void>(b_), b_dt,
                             ptr<const void>(r), r_dt, ptr<const void>(ct), ct_dt, ptr<const void>(tr), tr_dt,
                             ptr<const void>(lr), lr_dt, ptr<const void>(br), br_dt, ptr<const void>(rr), rr_dt,
                             logits, b, c, cc, h, w, k, st, cth, aw, nd, agn, ptr<float>(dets), ptr<void>(ws), wsb,
                             ptr<void>(stream)),
          "cnb_exct_decode_ex");
  });
  m.def("exct_decode", [](P t, P l, P b_, P r, P ct, P tr, P lr, P br, P rr, int b, int c, int cc, int h, int w,
                          int k, float st, float cth, float aw, int nd, int agn, P dets, P ws, size_t wsb, P stream) {
    check(cnb_exct_decode(ptr<const float>(t), ptr<const float>(l), ptr<const float>(b_), ptr<const float>(r),
                          ptr<const float>(ct), ptr<const float>(tr), ptr<const float>(lr), ptr<const float>(br),
                          ptr<const float>(rr), b, c, cc, h, w, k, st, cth, aw, nd, agn, ptr<float>(dets),
                          ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_exct_decode");
  });
  m.def("focal_workspace_bytes", &cnb_focal_workspace_bytes);
  m.def("focal_loss", [](P pred, P gt, long long n, int logits, float gs, P out2, P grad, P ws, size_t wsb, P stream) {
    check(cnb_focal_loss(ptr<const float>(pred), ptr<const float>(gt), n, logits, gs, ptr<float>(out2),
                         ptr<float>(grad), ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_focal_loss");
  });
  m.def("splat_gaussian", [](P cls, P cx, P cy, P rad, P valid, int b, int mm, int c, int h, int w, P hm, P stream) {
    check(cnb_splat_gaussian(ptr<const int32_t>(cls), ptr<const int32_t>(cx), ptr<const int32_t>(cy),
                             ptr<const int32_t>(rad), ptr<const uint8_t>(valid), b, mm, c, h, w, ptr<float>(hm),
                             ptr<void>(stream)),
          "cnb_splat_gaussian");
  });
  m.def("focal_splat_loss", [](P pred, P cls, P cx, P cy, P rad, P valid, int b, int mm, int c, int h, int w,
                               int logits, float gs, P out2, P grad, P ws, size_t wsb, P stream) {
    check(cnb_focal_splat_loss(ptr<const float>(pred), ptr<const int32_t>(cls), ptr<const int32_t>(cx),
                               ptr<const int32_t>(cy), ptr<const int32_t>(rad), ptr<const uint8_t>(valid), b, mm, c,
                               h, w, logits, gs, ptr<float>(out2), ptr<float>(grad), ptr<void>(ws), wsb,
                               ptr<void>(stream)),
          "cnb_focal_splat_loss");
  });
  m.def("reg_loss", [](P output, P mask, P ind, P target, int b, int d, int hw, int mm, int mode, float gs, P out1,
                       P grad, P stream) {
    check(cnb_reg_loss(ptr<const float>(output), ptr<const void>(mask), ptr<const int64_t>(ind),
                       ptr<const float>(target), b, d, hw, mm, mode, gs, ptr<float>(out1), ptr<float>(grad),
                       ptr<void>(stream)),
          "cnb_reg_loss");
  });
  m.def("focal_loss_ex", [](P pred, int dt, P gt, long long n, int logits, P out2, P ws, size_t wsb, P stream) {
    check(cnb_focal_loss_ex(ptr<const void>(pred), dt, ptr<const float>(gt), n, logits, ptr<float>(out2),
                            ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_focal_loss_ex");
  });
  m.def("focal_grad_ex", [](P pred, int dt, P gt, long long n, int logits, P out2, P gout, P grad, P stream) {
    check(cnb_focal_grad_ex(ptr<const void>(pred), dt, ptr<const float>(gt), n, logits, ptr<const float>(out2),
                            ptr<const float>(gout), ptr<void>(grad), ptr<void>(stream)),
          "cnb_focal_grad_ex");
  });
  m.def("focal_splat_loss_ex", [](P pred, int dt, P cls, P cx, P cy, P rad, P valid, int b, int mm, int c, int h,
                                  int w, int logits, P out2, P grad32, P ws, size_t wsb, P stream) {
    check(cnb_focal_splat_loss_ex(ptr<const void>(pred), dt, ptr<const int32_t>(cls), ptr<const int32_t>(cx),
                                  ptr<const int32_t>(cy), ptr<const int32_t>(rad), ptr<const uint8_t>(valid), b, mm,
                                  c, h, w, logits, ptr<float>(out2), ptr<float>(grad32), ptr<void>(ws), wsb,
                                  ptr<void>(stream)),
          "cnb_focal_splat_loss_ex");
  });
  m.def("focal_splat_grad_ex", [](P grad32, long long n, P gout, P grad, int dt, P stream) {
    check(cnb_focal_splat_grad_ex(ptr<const float>(grad32), n, ptr<const float>(gout), ptr<void>(grad), dt,
                                  ptr<void>(stream)),
          "cnb_focal_splat_grad_ex");
  });
  m.def("reg_loss_ex", [](P output, int dt, P mask, P ind, P target, int b, int d, int hw, int mm, int mode, P out2,
                          P stream) {
    check(cnb_reg_loss_ex(ptr<const void>(output), dt, ptr<const void>(mask), ptr<const int64_t>(ind),
                          ptr<const float>(target), b, d, hw, mm, mode, ptr<float>(out2), ptr<void>(stream)),
          "cnb_reg_loss_ex");
  });
  m.def("reg_loss_grad_ex", [](P output, int dt, P mask, P ind, P target, int b, int d, int hw, int mm, int mode,
                               P out2, P gout, P grad, P stream) {
    check(cnb_reg_loss_grad_ex(ptr<const void>(output), dt, ptr<const void>(mask), ptr<const int64_t>(ind),
                               ptr<const float>(target), b, d, hw, mm, mode, ptr<const float>(out2),
                               ptr<const float>(gout), ptr<void>(grad), ptr<void>(stream)),
          "cnb_reg_loss_grad_ex");
  });
  m.def("gather_feat_ex", [](P feat, int dt, P ind, P out, int b, int c, int hw, int mm, P stream) {
    check(cnb_gather_feat_ex(ptr<const void>(feat), dt, ptr<const int64_t>(ind), ptr<float>(out), b, c, hw, mm,
                             ptr<void>(stream)),
          "cnb_gather_feat_ex");
  });
  m.def("gather_feat_backward_ex", [](P gout, P ind, P gfeat, int dt, int b, int c, int hw, int mm, P stream) {
    check(cnb_gather_feat_backward_ex(ptr<const float>(gout), ptr<const int64_t>(ind), ptr<void>(gfeat), dt, b, c, hw,
                                      mm, ptr<void>(stream)),
          "cnb_gather_feat_backward_ex");
  });
  m.def("post_transform", [](P rows, P out, P trans, int b, int n, int d, int a0, int na, int b0, int nb, P stream) {
    check(cnb_post_transform(ptr<const float>(rows), ptr<float>(out), ptr<const double>(trans), b, n, d, a0, na, b0, nb,
                             ptr<void>(stream)),
          "cnb_post_transform");
  });
  m.def("group_by_class", [](P dets, int b, int n, int nc, P rows, P offsets, P stream) {
    check(cnb_group_by_class(ptr<const float>(dets), b, n, nc, ptr<float>(rows), ptr<int32_t>(offsets),
                             ptr<void>(stream)),
          "cnb_group_by_class");
  });
  m.def("soft_nms", [](P rows, P out, P offsets, int n_img, int lists, int n_cap, int d, float sigma, float nt,
                       float thr, int method, P final_n, P stream) {
    check(cnb_soft_nms(ptr<const float>(rows), ptr<float>(out), ptr<const int32_t>(offsets), n_img, lists, n_cap, d,
                       sigma, nt, thr, method, ptr<int32_t>(final_n), ptr<void>(stream)),
          "cnb_soft_nms");
  });
  m.def("topk_keep", [](P rows, int b, int n_cap, int d, P offsets, int nc, int mpi, P keep, P thresh, P stream) {
    check(cnb_topk_keep(ptr<const float>(rows), b, n_cap, d, ptr<const int32_t>(offsets), nc, mpi, ptr<uint8_t>(keep),
                        ptr<float>(thresh), ptr<void>(stream)),
          "cnb_topk_keep");
  });
  m.def("exdet_transform", [](P rows, P out, P trans, int b, int n, int d, float out_w, P stream) {
    check(cnb_exdet_transform(ptr<const float>(rows), ptr<float>(out), ptr<const double>(trans), b, n, d, out_w,
                              ptr<void>(stream)),
          "cnb_exdet_transform");
  });
  m.def("group_positive_by_class", [](P dets, int b, int n, int d, int cls_col, int nc, P rows, P offsets, P stream) {
    check(cnb_group_positive_by_class(ptr<const float>(dets), b, n, d, cls_col, nc, ptr<float>(rows),
                                      ptr<int32_t>(offsets), ptr<void>(stream)),
          "cnb_group_positive_by_class");
  });
  m.def("soft_nms_strided", [](P rows, P out, P offsets, int n_img, int lists, int img_stride, int list_cap, int d,
                               float sigma, float nt, float thr, int method, P final_n, P stream) {
    check(cnb_soft_nms_strided(ptr<const float>(rows), ptr<float>(out), ptr<const int32_t>(offsets), n_img, lists,
                               img_stride, list_cap, d, sigma, nt, thr, method, ptr<int32_t>(final_n),
                               ptr<void>(stream)),
          "cnb_soft_nms_strided");
  });
  m.def("topk_keep_wide", [](P rows, int b, int n_cap, int d, P offsets, int nc, int mpi, P keep, P thresh, P stream) {
    check(cnb_topk_keep_wide(ptr<const float>(rows), b, n_cap, d, ptr<const int32_t>(offsets), nc, mpi,
                             ptr<uint8_t>(keep), ptr<float>(thresh), ptr<void>(stream)),
          "cnb_topk_keep_wide");
  });
  m.def("ddd_tail", [](P dets, int b, int n, int d, P trans, P calib, int nc, int cut, float thresh, P rows, P offsets,
                       P seen, P stream) {
    check(cnb_ddd_tail(ptr<const float>(dets), b, n, d, ptr<const double>(trans), ptr<const float>(calib), nc, cut,
                       thresh, ptr<float>(rows), ptr<int32_t>(offsets), ptr<uint8_t>(seen), ptr<void>(stream)),
          "cnb_ddd_tail");
  });
  m.def("resize_image", [](P img, int h, int w, P out, int oh, int ow, P stream) {
    check(cnb_resize_image(ptr<const uint8_t>(img), h, w, ptr<uint8_t>(out), oh, ow, ptr<void>(stream)),
          "cnb_resize_image");
  });
  m.def("preprocess_image", [](P img, int h, int w, P minv, P mean, P stdv, P out, int oh, int ow, int flip, P stream) {
    check(cnb_preprocess_image(ptr<const uint8_t>(img), h, w, ptr<const double>(minv), ptr<const float>(mean),
                               ptr<const float>(stdv), ptr<float>(out), oh, ow, flip, ptr<void>(stream)),
          "cnb_preprocess_image");
  });
  m.def("preprocess_image_f32", [](P img, int h, int w, P minv, P mean, P stdv, P out, int oh, int ow, int flip,
                                   P stream) {
    check(cnb_preprocess_image_f32(ptr<const uint8_t>(img), h, w, ptr<const double>(minv), ptr<const float>(mean),
                                   ptr<const float>(stdv), ptr<float>(out), oh, ow, flip, ptr<void>(stream)),
          "cnb_preprocess_image_f32");
  });
  m.def("dcnv2_workspace_bytes", &cnb_dcnv2_workspace_bytes);
  m.def("dcnv2_backward_workspace_bytes", &cnb_dcnv2_backward_workspace_bytes);
  m.def("dcnv2_backward_ex", [](P input, int in_cl, P offset, P mask, P weight, P gout, P gin, int gin_cl, P goff, P gmask,
                                P gw, P gb, int b, int cin, int h, int w, int cout, int kh, int kw, int stride, int pad,
                                int dil, int dg, P ws, size_t wsb, P stream) {
    check(cnb_dcnv2_backward_ex(ptr<const float>(input), in_cl, ptr<const float>(offset), ptr<const float>(mask),
                                ptr<const float>(weight), ptr<const float>(gout), ptr<float>(gin), gin_cl,
                                ptr<float>(goff), ptr<float>(gmask), ptr<float>(gw), ptr<float>(gb), b, cin, h, w, cout,
                                kh, kw, stride, pad, dil, dg, ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_dcnv2_backward_ex");
  });
  m.def("dcnv2_backward_bf16_workspace_bytes", &cnb_dcnv2_backward_bf16_workspace_bytes);
  m.def("dcnv2_backward_bf16", [](P input, int in_dt, int in_cl, P offset, P mask, P weight, P gout, int gout_dt, P gin,
                                  int gin_cl, P goff, P gmask, P gw, P gb, int b, int cin, int h, int w, int cout, int kh,
                                  int kw, int stride, int pad, int dil, int dg, P ws, size_t wsb, P stream) {
    check(cnb_dcnv2_backward_bf16(ptr<const void>(input), in_dt, in_cl, ptr<const float>(offset),
                                  ptr<const float>(mask), ptr<const float>(weight), ptr<const void>(gout), gout_dt,
                                  ptr<float>(gin), gin_cl, ptr<float>(goff), ptr<float>(gmask), ptr<float>(gw),
                                  ptr<float>(gb), b, cin, h, w, cout, kh, kw, stride, pad, dil, dg, ptr<void>(ws), wsb,
                                  ptr<void>(stream)),
          "cnb_dcnv2_backward_bf16");
  });
  m.def("dcnv2_set_deterministic", &cnb_dcnv2_set_deterministic);
  m.def("dcnv2_get_deterministic", &cnb_dcnv2_get_deterministic);
  m.def("dcnv2_forward", [](P input, P offset, P mask, P weight, P bias, P output, int b, int cin, int h, int w,
                            int cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int dg, P ws,
                            size_t wsb, P stream) {
    check(cnb_dcnv2_forward(ptr<const float>(input), ptr<const float>(offset), ptr<const float>(mask),
                            ptr<const float>(weight), ptr<const float>(bias), ptr<float>(output), b, cin, h, w, cout,
                            kh, kw, sh, sw, ph, pw, dh, dw, dg, ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_dcnv2_forward");
  });
  m.def("dcnv2_wtiles_bytes", &cnb_dcnv2_wtiles_bytes);
  m.def("dcnv2_prepare_weights", [](P weight, int cin, int cout, int kh, int kw, int dg, P wt, size_t wtb, P stream) {
    check(cnb_dcnv2_prepare_weights(ptr<const float>(weight), cin, cout, kh, kw, dg, ptr<void>(wt), wtb,
                                    ptr<void>(stream)),
          "cnb_dcnv2_prepare_weights");
  });
  m.def("dcnv2_prepared_workspace_bytes", &cnb_dcnv2_prepared_workspace_bytes);
  m.def("dcnv2_forward_prepared", [](P input, int nhwc, P offset, P mask, P wt, P bias, P output, int b, int cin, int h,
                                     int w, int cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                                     int dg, P ws, size_t wsb, P stream) {
    check(cnb_dcnv2_forward_prepared(ptr<const float>(input), nhwc, ptr<const float>(offset), ptr<const float>(mask),
                                     ptr<const void>(wt), ptr<const float>(bias), ptr<float>(output), b, cin, h, w,
                                     cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_dcnv2_forward_prepared");
  });
  m.def("dcnv2_forward_fused", [](P input, int nhwc, P om, P wt, P bias, P sc, P sh_, int relu, P output, int b, int cin,
                                  int h, int w, int cout, int kh, int kw, int stride, int pad, int dil, int dg, P ws,
                                  size_t wsb, P stream) {
    check(cnb_dcnv2_forward_fused(ptr<const float>(input), nhwc, ptr<const float>(om), ptr<const void>(wt),
                                  ptr<const float>(bias), ptr<const float>(sc), ptr<const float>(sh_), relu,
                                  ptr<float>(output), b, cin, h, w, cout, kh, kw, stride, pad, dil, dg, ptr<void>(ws),
                                  wsb, ptr<void>(stream)),
          "cnb_dcnv2_forward_fused");
  });
  m.attr("DTYPE_F32") = CNB_DTYPE_F32;
  m.attr("DTYPE_BF16") = CNB_DTYPE_BF16;
  m.attr("DTYPE_F16") = CNB_DTYPE_F16;
  m.def("dcnv2_wtiles_bf16_bytes", &cnb_dcnv2_wtiles_bf16_bytes);
  m.def("dcnv2_prepare_weights_bf16", [](P weight, int cin, int cout, int kh, int kw, int dg, P wt, size_t wtb,
                                         P stream) {
    check(cnb_dcnv2_prepare_weights_bf16(ptr<const float>(weight), cin, cout, kh, kw, dg, ptr<void>(wt), wtb,
                                         ptr<void>(stream)),
          "cnb_dcnv2_prepare_weights_bf16");
  });
  m.def("dcnv2_bf16_workspace_bytes", &cnb_dcnv2_bf16_workspace_bytes);
  m.def("dcnv2_forward_bf16", [](P input, int in_dt, int nhwc, P offset, P mask, P wt, P bias, P output, int out_dt,
                                 int b, int cin, int h, int w, int cout, int kh, int kw, int stride, int pad, int dil,
                                 int dg, P ws, size_t wsb, P stream) {
    check(cnb_dcnv2_forward_bf16(ptr<const void>(input), in_dt, nhwc, ptr<const float>(offset),
                                 ptr<const float>(mask), ptr<const void>(wt), ptr<const float>(bias), ptr<void>(output),
                                 out_dt, b, cin, h, w, cout, kh, kw, stride, pad, dil, dg, ptr<void>(ws), wsb,
                                 ptr<void>(stream)),
          "cnb_dcnv2_forward_bf16");
  });
  m.def("dcnv2_forward_fused_bf16", [](P input, int in_dt, int nhwc, P om, P wt, P bias, P sc, P sh_, int relu,
                                       P output, int out_dt, int b, int cin, int h, int w, int cout, int kh, int kw,
                                       int stride, int pad, int dil, int dg, P ws, size_t wsb, P stream) {
    check(cnb_dcnv2_forward_fused_bf16(ptr<const void>(input), in_dt, nhwc, ptr<const float>(om), ptr<const void>(wt),
                                       ptr<const float>(bias), ptr<const float>(sc), ptr<const float>(sh_), relu,
                                       ptr<void>(output), out_dt, b, cin, h, w, cout, kh, kw, stride, pad, dil, dg,
                                       ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_dcnv2_forward_fused_bf16");
  });
  m.def("dcnv2_backward", [](P input, P offset, P mask, P weight, P gout, P gin, P goff, P gmask, P gw, P gb, int b,
                             int cin, int h, int w, int cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh,
                             int dw, int dg, P ws, size_t wsb, P stream) {
    check(cnb_dcnv2_backward(ptr<const float>(input), ptr<const float>(offset), ptr<const float>(mask),
                             ptr<const float>(weight), ptr<const float>(gout), ptr<float>(gin), ptr<float>(goff),
                             ptr<float>(gmask), ptr<float>(gw), ptr<float>(gb), b, cin, h, w, cout, kh, kw, sh, sw,
                             ph, pw, dh, dw, dg, ptr<void>(ws), wsb, ptr<void>(stream)),
          "cnb_dcnv2_backward");
  });
}

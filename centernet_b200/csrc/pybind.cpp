// Thin pybind11 layer over the C ABI of include/centernet_b200.h.
// Pointers cross as integers (tensor.data_ptr()); no torch types here, so the module
// builds with g++ alone and the C ABI stays the real boundary.  A non-zero status
// becomes a Python RuntimeError carrying cnb_last_error() -- the counterpart of the
// reference's THError -> RuntimeError path (DCNv2/src/dcn_v2_cuda.c:20-38).
//
// Each entry point is bound from its C type alone: STATUS(name) for a call that returns a
// CNB_* status, VALUE(name) for one whose result is handed back as is.  Every binding is
// positional (arg0, arg1, ...); tests/test_abi.py checks them against the header.
#include <pybind11/pybind11.h>
#include <stdexcept>
#include <string>
#include "../../include/centernet_b200.h"

namespace py = pybind11;

static void check(int rc, const char *fn) {
  if (rc == CNB_OK) return;
  std::string msg = std::string(fn) + " failed (status " + std::to_string(rc) + "): " + cnb_last_error();
  if (rc == CNB_EUNSUPPORTED) {  // valid request outside the implemented envelope
    PyErr_SetString(PyExc_NotImplementedError, msg.c_str());
    throw py::error_already_set();
  }
  throw std::runtime_error(msg);
}

// What a C parameter of type T takes on the Python side: a pointer is an integer address, anything
// else (int, long long, size_t, float, double) itself.
template <typename T>
struct Arg {
  typedef T type;
  static T to_c(T v) { return v; }
};
template <typename T>
struct Arg<T *> {
  typedef uintptr_t type;
  static T *to_c(uintptr_t v) { return reinterpret_cast<T *>(v); }
};

// c_name is a string literal: the error message is only assembled when a call fails.
template <typename... A>
static void def_status(py::module_ &m, const char *py_name, const char *c_name, int (*fn)(A...)) {
  m.def(py_name, [fn, c_name](typename Arg<A>::type... a) { check(fn(Arg<A>::to_c(a)...), c_name); });
}

template <typename R, typename... A>
static void def_value(py::module_ &m, const char *py_name, R (*fn)(A...)) {
  m.def(py_name, [fn](typename Arg<A>::type... a) { return fn(Arg<A>::to_c(a)...); });
}

#define STATUS(name) def_status(m, #name, "cnb_" #name, &cnb_##name)
#define VALUE(name) def_value(m, #name, &cnb_##name)

PYBIND11_MODULE(_C, m) {
  m.doc() = "centernet_b200 C-ABI bindings (pointers as ints)";
  m.attr("OK") = CNB_OK;
  m.attr("EINVAL") = CNB_EINVAL;
  m.attr("EUNSUPPORTED") = CNB_EUNSUPPORTED;
  m.attr("ECUDA") = CNB_ECUDA;
  m.attr("EWORKSPACE") = CNB_EWORKSPACE;
  m.attr("DTYPE_F32") = CNB_DTYPE_F32;
  m.attr("DTYPE_BF16") = CNB_DTYPE_BF16;
  m.attr("DTYPE_F16") = CNB_DTYPE_F16;
  m.attr("TRAIN_MAX_PIXELS") = CNB_TRAIN_MAX_PIXELS;

  VALUE(version);
  m.def("last_error", []() { return std::string(cnb_last_error()); });
  VALUE(launch_count);

  STATUS(nms);
  VALUE(topk_workspace_bytes);
  STATUS(topk);
  m.def("select_plan_info", [](uintptr_t src, int n_img, int c, int h, int w, int k, int nms, int elem_size) {
    int v[CNB_SELECT_PLAN_FIELDS];
    check(cnb_select_plan_info(reinterpret_cast<const void *>(src), n_img, c, h, w, k, nms, elem_size, v,
                               CNB_SELECT_PLAN_FIELDS),
          "cnb_select_plan_info");
    static const char *names[CNB_SELECT_PLAN_FIELDS] = {"hot", "n_cta", "wb", "max_slots", "seg_cap",
                                                         "fused_finalize", "use_tma", "rb", "local_img"};
    py::dict d;
    for (int i = 0; i < CNB_SELECT_PLAN_FIELDS; ++i) d[names[i]] = v[i];
    return d;
  });
  STATUS(topk_channel);
  STATUS(gather_feat);
  STATUS(gather_feat_backward);
  STATUS(gather_feat_ex);
  STATUS(gather_feat_backward_ex);

  STATUS(ctdet_decode);
  VALUE(ctdet_logits_workspace_bytes);
  STATUS(ctdet_decode_logits);
  VALUE(ctdet_decode_ex_workspace_bytes);
  STATUS(ctdet_decode_ex);
  STATUS(sigmoid);
  STATUS(flip_merge);
  STATUS(flip_merge_ex);

  STATUS(ddd_decode);
  VALUE(ddd_decode_ex_workspace_bytes);
  STATUS(ddd_decode_ex);
  VALUE(multi_pose_workspace_bytes);
  STATUS(multi_pose_decode);
  VALUE(multi_pose_decode_ex_workspace_bytes);
  STATUS(multi_pose_decode_ex);
  STATUS(edge_aggregate);
  STATUS(edge_aggregate_ex);
  VALUE(exct_workspace_bytes);
  VALUE(exct_groups);
  STATUS(exct_decode);
  VALUE(exct_decode_ex_workspace_bytes);
  STATUS(exct_decode_ex);

  VALUE(focal_workspace_bytes);
  STATUS(focal_loss);
  STATUS(splat_gaussian);
  STATUS(focal_splat_loss);
  STATUS(reg_loss);
  STATUS(focal_loss_ex);
  STATUS(focal_grad_ex);
  STATUS(focal_splat_loss_ex);
  STATUS(focal_splat_grad_ex);
  STATUS(reg_loss_ex);
  STATUS(reg_loss_grad_ex);

  VALUE(dcnv2_workspace_bytes);
  STATUS(dcnv2_forward);
  VALUE(dcnv2_wtiles_bytes);
  STATUS(dcnv2_prepare_weights);
  VALUE(dcnv2_prepared_workspace_bytes);
  STATUS(dcnv2_forward_prepared);
  STATUS(dcnv2_forward_fused);
  VALUE(dcnv2_wtiles_bf16_bytes);
  STATUS(dcnv2_prepare_weights_bf16);
  VALUE(dcnv2_bf16_workspace_bytes);
  STATUS(dcnv2_forward_bf16);
  STATUS(dcnv2_forward_fused_bf16);
  VALUE(dcnv2_backward_workspace_bytes);
  STATUS(dcnv2_backward_ex);
  VALUE(dcnv2_set_deterministic);
  VALUE(dcnv2_get_deterministic);
  STATUS(dcnv2_backward);
  VALUE(dcnv2_backward_bf16_workspace_bytes);
  STATUS(dcnv2_backward_bf16);

  VALUE(head_w1t_bytes);
  VALUE(head_w2t_bytes);
  STATUS(head_prepare_weights_bf16);
  VALUE(head_workspace_bytes);
  STATUS(head_forward_bf16);

  VALUE(dcnv2_f64_workspace_bytes);
  STATUS(dcnv2_forward_f64);
  STATUS(dcnv2_backward_f64);
  STATUS(psroi_pooling_forward);
  STATUS(psroi_pooling_backward);
  VALUE(psroi_pooling_f64_workspace_bytes);
  STATUS(psroi_pooling_forward_f64);
  STATUS(psroi_pooling_backward_f64);

  STATUS(post_transform);
  STATUS(group_by_class);
  STATUS(soft_nms);
  STATUS(topk_keep);
  STATUS(exdet_transform);
  STATUS(group_positive_by_class);
  STATUS(soft_nms_strided);
  STATUS(topk_keep_wide);
  STATUS(ddd_tail);

  STATUS(resize_image);
  STATUS(preprocess_image);
  STATUS(preprocess_image_f32);

  VALUE(train_images_workspace_bytes);
  STATUS(train_images);
  STATUS(ctdet_targets);
  STATUS(multi_pose_targets);
  STATUS(ddd_targets);
  STATUS(ddd_gaussian_radius);
  STATUS(exdet_targets);
}

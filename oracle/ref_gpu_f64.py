"""ctypes binding of oracle/_ref/libdcnv2_ref_f64.so (TEST INFRASTRUCTURE): the UNMODIFIED reference float64
DCNv2 / deformable-PSROI CUDA kernels (dcn_v2_double) driven by the cuBLAS restatement of their host loop
(oracle/ref_host_f64.cu, recipe oracle/build_ref_f64.py).  Same calls as oracle/ref_gpu.py, but every tensor stays
float64.  tests/golden/make_golden_ref_gpu_f64.py stores its outputs and bench_secondary.py times it.
"""
import ctypes

import torch

from . import build_ref_f64
from .ref_gpu import _out_hw, _p, _stream

_LIB = None
D = torch.float64


def available():
    return build_ref_f64.available()


def lib():
    global _LIB
    if _LIB is None:
        path = build_ref_f64.build()
        if path is None:
            raise RuntimeError("oracle/_ref/libdcnv2_ref_f64.so is missing (build it where /root/reference exists: "
                               "python -m oracle.build_ref_f64)")
        _LIB = ctypes.CDLL(path)
    return _LIB


def _d(*ts):
    return [t.contiguous().to(D) for t in ts]


def dcn_v2_forward(x, offset, mask, weight, bias, stride=1, padding=1, dilation=1, deformable_groups=1):
    x, offset, mask, weight, bias = _d(x, offset, mask, weight, bias)
    B, C, H, W = x.shape
    Co, _, kh, kw = weight.shape
    Ho, Wo = _out_hw(H, W, kh, kw, stride, padding, dilation)
    out = torch.empty(B, Co, Ho, Wo, device=x.device, dtype=D)
    columns = torch.empty(C * kh * kw, Ho * Wo, device=x.device, dtype=D)
    ones = torch.ones(Ho, Wo, device=x.device, dtype=D)
    rc = lib().ref_dcn_v2_forward_f64(_p(x), _p(weight), _p(bias), _p(ones), _p(offset), _p(mask), _p(out),
                                      _p(columns), B, C, H, W, Co, kh, kw, stride, stride, padding, padding, dilation,
                                      dilation, deformable_groups, _stream())
    if rc:
        raise RuntimeError("ref_dcn_v2_forward_f64 failed: %d" % rc)
    return out


def dcn_v2_backward(x, offset, mask, weight, bias, grad_output, stride=1, padding=1, dilation=1,
                    deformable_groups=1):
    """-> (grad_input, grad_offset, grad_mask, grad_weight, grad_bias)."""
    x, offset, mask, weight, grad_output = _d(x, offset, mask, weight, grad_output)
    B, C, H, W = x.shape
    Co, _, kh, kw = weight.shape
    Ho, Wo = _out_hw(H, W, kh, kw, stride, padding, dilation)
    gi = torch.zeros_like(x); go = torch.zeros_like(offset); gm = torch.zeros_like(mask)
    gw = torch.zeros_like(weight); gb = torch.zeros(Co, device=x.device, dtype=D)
    columns = torch.empty(C * kh * kw, Ho * Wo, device=x.device, dtype=D)
    ones = torch.ones(Ho, Wo, device=x.device, dtype=D)
    rc = lib().ref_dcn_v2_backward_f64(_p(x), _p(weight), _p(ones), _p(offset), _p(mask), _p(columns), _p(gi),
                                       _p(gw), _p(gb), _p(go), _p(gm), _p(grad_output), B, C, H, W, Co, kh, kw,
                                       stride, stride, padding, padding, dilation, dilation, deformable_groups,
                                       _stream())
    if rc:
        raise RuntimeError("ref_dcn_v2_backward_f64 failed: %d" % rc)
    return gi, go, gm, gw, gb


def psroi_forward(data, rois, trans, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                  sample_per_part=4, trans_std=0.0):
    """-> (out, top_count)."""
    part_size = pooled_size if part_size is None else part_size
    data, rois, trans = _d(data, rois, trans)
    B, C, H, W = data.shape
    n = rois.shape[0]
    out = torch.zeros(n, output_dim, pooled_size, pooled_size, device=data.device, dtype=D)
    cnt = torch.zeros_like(out)
    ct = 2 if no_trans else trans.shape[1]
    rc = lib().ref_psroi_forward_f64(_p(data), _p(rois), _p(trans), _p(out), _p(cnt), B, C, H, W, n, ct,
                                     int(no_trans), ctypes.c_double(spatial_scale), output_dim, group_size,
                                     pooled_size, part_size, sample_per_part, ctypes.c_double(trans_std), _stream())
    if rc:
        raise RuntimeError("ref_psroi_forward_f64 failed: %d" % rc)
    return out, cnt


def psroi_backward(out_grad, data, rois, trans, top_count, spatial_scale, pooled_size, output_dim, no_trans,
                   group_size=1, part_size=None, sample_per_part=4, trans_std=0.0):
    """-> (grad_input, grad_trans)."""
    part_size = pooled_size if part_size is None else part_size
    out_grad, data, rois, trans, top_count = _d(out_grad, data, rois, trans, top_count)
    B, C, H, W = data.shape
    n = rois.shape[0]
    gi = torch.zeros_like(data); gt = torch.zeros_like(trans)
    ct = 2 if no_trans else trans.shape[1]
    rc = lib().ref_psroi_backward_f64(_p(out_grad), _p(data), _p(rois), _p(trans), _p(top_count), _p(gi), _p(gt), B,
                                      C, H, W, n, ct, int(no_trans), ctypes.c_double(spatial_scale), output_dim,
                                      group_size, pooled_size, part_size, sample_per_part,
                                      ctypes.c_double(trans_std), _stream())
    if rc:
        raise RuntimeError("ref_psroi_backward_f64 failed: %d" % rc)
    return gi, gt

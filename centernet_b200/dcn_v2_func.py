"""Mirror of src/lib/models/networks/DCNv2/dcn_v2_func.py.

``DCNv2Function(stride, padding, dilation=1, deformable_groups=1)`` keeps the reference's
construct-then-call shape (dcn_v2_func.py:13-73, used directly by DCNv2/test.py:88,113) while
delegating to a new-style static autograd Function; the work is done by cnb_dcnv2_forward /
cnb_dcnv2_backward (im2col-free, no `ones`/`columns` scratch).  Non-CUDA tensors raise
NotImplementedError exactly like the reference (:23-24, :41-42).
"""
import os
import warnings
import weakref

import torch
from torch.autograd import Function

from ._lib import C, f32c, ptr, stream_ptr, workspace

# CNB_DCN_FP32=1 selects the fp32 CUDA-core contraction instead of the wgmma (3xTF32) one
_FORCE_FP32 = os.environ.get("CNB_DCN_FP32", "0") == "1"
# CNB_DCN_DETERMINISTIC=1: bit-identical gradients run to run (cnb_dcnv2_set_deterministic); also on under
# torch.use_deterministic_algorithms(True)
_DETERMINISTIC = os.environ.get("CNB_DCN_DETERMINISTIC", "0") == "1"


def _deterministic():
    return bool(_DETERMINISTIC or torch.are_deterministic_algorithms_enabled())


def _alert_not_deterministic(what):
    """torch's rule for an op without a deterministic implementation: raise, or warn and run under warn_only."""
    msg = ("%s does not have a deterministic implementation, but deterministic algorithms were requested "
           "(torch.use_deterministic_algorithms(True) or CNB_DCN_DETERMINISTIC=1)" % what)
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg)
    else:
        raise RuntimeError(msg)


def _f64c(what, *tensors):
    """float64 + contiguous views; the reference's typed backend takes no mixed types, so a float tensor of another
    dtype next to a float64 input is an error rather than a silent cast."""
    out = []
    for t in tensors:
        if t is None:
            out.append(None)
            continue
        if t.dtype != torch.float64:
            raise RuntimeError("%s: the input is float64, so every tensor must be float64 too (got %s)" % (what, t.dtype))
        out.append(t.contiguous())
    return out


def _out_hw(h, w, kh, kw, stride, padding, dilation):
    ho = (h + 2 * padding - (dilation * (kh - 1) + 1)) // stride + 1   # dcn_v2_func.py:64-73
    wo = (w + 2 * padding - (dilation * (kw - 1) + 1)) // stride + 1
    return ho, wo


_WT_CACHE = {}      # (id(weight), bf16) -> (weakref to it, its version when tiled, tiles); evicted when the tensor dies


def _weight_tiles(weight, dg, bf16=False):
    """TF32 hi/lo weight tiles in the wgmma K-major layout (cnb_dcnv2_prepare_weights), or with bf16=True the bf16
    tiles of the bf16 forward (cnb_dcnv2_prepare_weights_bf16), rebuilt only when the parameter changes: torch bumps
    `_version` on every in-place update (optimizer step, load_state_dict), and the entry is tied to the tensor OBJECT
    by a weak reference, so a new tensor that happens to reuse the address never sees stale tiles.  The two kinds of
    tiles of one parameter are cached side by side.  bf16 tiles are cached for a weight of any dtype (a bf16 model's
    parameters are bf16; the tiles are built from its fp32 upcast, which is exact)."""
    w = f32c(weight)
    cout, cin, kh, kw = [int(v) for v in w.shape]
    own = bf16 or w is weight or w.data_ptr() == weight.data_ptr()
    key = (id(weight), bool(bf16))
    ver = weight._version
    hit = _WT_CACHE.get(key) if own else None
    if hit is not None and hit[0]() is weight and hit[1] == ver and hit[2].device == w.device:
        return hit[2]
    if bf16:
        wt = workspace(C.dcnv2_wtiles_bf16_bytes(cin, cout, kh, kw, dg), w.device)
        C.dcnv2_prepare_weights_bf16(ptr(w), cin, cout, kh, kw, dg, ptr(wt), wt.numel(), stream_ptr(w))
    else:
        wt = workspace(C.dcnv2_wtiles_bytes(cin, cout, kh, kw, dg), w.device)
        C.dcnv2_prepare_weights(ptr(w), cin, cout, kh, kw, dg, ptr(wt), wt.numel(), stream_ptr(w))
    if own:
        try:
            _WT_CACHE[key] = (weakref.ref(weight, lambda _r, k=key: _WT_CACHE.pop(k, None)), ver, wt)
        except TypeError:      # not weak-referenceable: do not cache
            pass
    return wt


def _dcn_shapes(x, off, msk, w, stride, padding, dilation, deformable_groups):
    n, cin, h, wd = [int(v) for v in x.shape]
    cout, cin_w, kh, kw = [int(v) for v in w.shape]
    if cin_w != cin:   # dcn_v2_cuda.c:36-38
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (cin, cin_w))
    ho, wo = _out_hw(h, wd, kh, kw, stride, padding, dilation)
    kt = kh * kw
    if tuple(off.shape) != (n, 2 * kt * deformable_groups, ho, wo) or \
            tuple(msk.shape) != (n, kt * deformable_groups, ho, wo):
        raise RuntimeError("DCNv2: offset/mask shape does not match the output grid")
    return n, cin, h, wd, cout, kh, kw, ho, wo


def _dcn_forward_f64(ctx, input, offset, mask, weight, bias, stride, padding, dilation, dg):
    """float64 (the reference's dcn_v2_double build): DMMA kernels, bit-reproducible backward in every mode."""
    x, off, msk, w, b = _f64c("DCNv2", input, offset, mask, weight, bias)
    n, cin, h, wd, cout, kh, kw, ho, wo = _dcn_shapes(x, off, msk, w, stride, padding, dilation, dg)
    out = torch.empty((n, cout, ho, wo), dtype=torch.float64, device=x.device)
    C.dcnv2_forward_f64(ptr(x), ptr(off), ptr(msk), ptr(w), ptr(b), ptr(out), n, cin, h, wd, cout, kh, kw, stride,
                        stride, padding, padding, dilation, dilation, dg, stream_ptr(x))
    ctx.save_for_backward(x, off, msk, w, b)
    ctx.f64 = True
    ctx.cfg = (stride, padding, dilation, dg)
    return out


def _dcn_backward_f64(ctx, grad_output):
    x, off, msk, w, b = ctx.saved_tensors
    stride, padding, dilation, dg = ctx.cfg
    go = grad_output.double().contiguous()
    n, cin, h, wd = [int(v) for v in x.shape]
    cout, _, kh, kw = [int(v) for v in w.shape]
    gx, goff, gmsk, gw = (torch.zeros_like(t) for t in (x, off, msk, w))   # accumulated into (dcn_v2_func.py:44-48)
    gb = torch.zeros_like(b) if b is not None else None
    ws = workspace(C.dcnv2_f64_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding, dilation, dg), x.device)
    C.dcnv2_backward_f64(ptr(x), ptr(off), ptr(msk), ptr(w), ptr(go), ptr(gx), ptr(goff), ptr(gmsk), ptr(gw), ptr(gb),
                         n, cin, h, wd, cout, kh, kw, stride, stride, padding, padding, dilation, dilation, dg, ptr(ws),
                         ws.numel(), stream_ptr(x))
    return gx, goff, gmsk, gw, gb, None, None, None, None


class _DCNv2(Function):
    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups):
        if not input.is_cuda:
            raise NotImplementedError
        ctx.f64 = False
        if input.dtype == torch.float64:   # dtype follows the input, as the reference's typed backend
            return _dcn_forward_f64(ctx, input, offset, mask, weight, bias, stride, padding, dilation,
                                    deformable_groups)
        off, msk, w, b = f32c(offset), f32c(mask), f32c(weight), f32c(bias)
        n, cin, h, wd, cout, kh, kw, ho, wo = _dcn_shapes(input, off, msk, w, stride, padding, dilation,
                                                          deformable_groups)
        kt = kh * kw
        out = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=input.device)
        # a channels_last activation (what cuDNN produces under torch.channels_last) is sampled in place
        nhwc = (not _FORCE_FP32) and kt <= 9 and (cin // deformable_groups) % 32 == 0 and \
            input.dtype == torch.float32 and input.is_contiguous(memory_format=torch.channels_last) and \
            not input.is_contiguous()
        need_grad = any(ctx.needs_input_grad[:5])
        # the backward takes a channels_last input as it is too (cnb_dcnv2_backward_ex): no NCHW copy is kept for it
        x_cl = nhwc and need_grad and cout <= 256 and \
            C.dcnv2_backward_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding, dilation, deformable_groups) > 0
        x = f32c(input) if ((need_grad and not x_cl) or not nhwc) else None      # NCHW copy only when somebody needs it
        if _FORCE_FP32 or kt > 9:
            C.dcnv2_forward(ptr(x), ptr(off), ptr(msk), ptr(w), ptr(b), ptr(out), n, cin, h, wd, cout, kh, kw,
                            stride, stride, padding, padding, dilation, dilation, deformable_groups, 0, 0,
                            stream_ptr(x))
        else:
            # tensor-core path: weight tiles cached per weight version; NCHW inputs go through one re-layout pass
            wt = _weight_tiles(weight, deformable_groups)
            xin = input if nhwc else x
            ws = workspace(C.dcnv2_prepared_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding, dilation,
                                                            deformable_groups), input.device)
            C.dcnv2_forward_prepared(ptr(xin), int(nhwc), ptr(off), ptr(msk), ptr(wt), ptr(b), ptr(out), n, cin, h, wd,
                                     cout, kh, kw, stride, stride, padding, padding, dilation, dilation,
                                     deformable_groups, ptr(ws), ws.numel(), stream_ptr(off))
        if need_grad:
            ctx.save_for_backward(input if x_cl else x, off, msk, w, b)
        ctx.x_cl = bool(x_cl)
        ctx.cfg = (stride, padding, dilation, deformable_groups)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        if not grad_output.is_cuda:
            raise NotImplementedError
        if ctx.f64:
            return _dcn_backward_f64(ctx, grad_output)
        x, off, msk, w, b = ctx.saved_tensors
        return _dcn_backward_f32(x, off, msk, w, b, f32c(grad_output), ctx.cfg, ctx.x_cl) + (None,) * 4


def _dcn_backward_f32(x, off, msk, w, b, go, cfg, x_cl):
    """The fp32 backward (tensor cores when the workspace query allows, else the fp32 kernels): gradients of input,
    offset, mask, weight and bias, all fp32.  x_cl: x is a channels_last input the tensor-core backward reads as is."""
    stride, padding, dilation, dg = cfg
    n, cin, h, wd = [int(v) for v in x.shape]
    cout, _, kh, kw = [int(v) for v in w.shape]
    # order-independent (fixed-point) grad_input when the user asked torch for deterministic algorithms (or
    # CNB_DCN_DETERMINISTIC=1); the workspace query, made after setting the mode, includes what that mode needs
    det = _deterministic()
    C.dcnv2_set_deterministic(int(det))
    wsb = 0 if _FORCE_FP32 else C.dcnv2_backward_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding,
                                                                 dilation, dg)
    if det and wsb == 0:
        C.dcnv2_set_deterministic(0)    # the fp32 kernels run under warn_only; otherwise the alert raises
        _alert_not_deterministic("DCNv2 backward on the fp32 path (CNB_DCN_FP32=1, more than 9 taps or an image "
                                 "beyond the tensor-core kernels' 32-bit indexing)")
    use_cl = x_cl and not _FORCE_FP32
    if x_cl and not use_cl:
        x = x.contiguous()          # the fp32 kernels work on NCHW
    # zero-filled, accumulated into -- dcn_v2_func.py:44-48 (zeros_like keeps a channels_last input's layout)
    gx = torch.zeros_like(x)
    goff = torch.zeros_like(off)
    gmsk = torch.zeros_like(msk)
    gw = torch.zeros_like(w)
    gb = torch.zeros_like(b) if b is not None else None
    wsbuf = workspace(wsb, x.device) if wsb else None
    if use_cl:
        C.dcnv2_backward_ex(ptr(x), 1, ptr(off), ptr(msk), ptr(w), ptr(go), ptr(gx), 1, ptr(goff), ptr(gmsk), ptr(gw),
                            ptr(gb), n, cin, h, wd, cout, kh, kw, stride, padding, dilation, dg, ptr(wsbuf), wsb,
                            stream_ptr(x))
    else:
        C.dcnv2_backward(ptr(x), ptr(off), ptr(msk), ptr(w), ptr(go), ptr(gx), ptr(goff), ptr(gmsk), ptr(gw), ptr(gb),
                         n, cin, h, wd, cout, kh, kw, stride, stride, padding, padding, dilation, dilation, dg,
                         ptr(wsbuf) if wsbuf is not None else 0, wsb, stream_ptr(x))
    return gx, goff, gmsk, gw, gb


# ------------------------------------------------------------------ bf16 forward (opt-in: compute_dtype=torch.bfloat16)
def _check_compute_dtype(compute_dtype):
    if compute_dtype is not None and compute_dtype != torch.bfloat16:
        raise ValueError("compute_dtype must be None (fp32-accurate contraction) or torch.bfloat16, got %r"
                         % (compute_dtype,))
    return compute_dtype


def _check_backward_dtype(compute_dtype, backward_dtype):
    """backward_dtype=torch.bfloat16 (the bf16 backward) goes with compute_dtype=torch.bfloat16 only."""
    if backward_dtype is None:
        return None
    if backward_dtype != torch.bfloat16 or compute_dtype != torch.bfloat16:
        raise ValueError("backward_dtype must be None (the fp32 backward) or torch.bfloat16 together with "
                         "compute_dtype=torch.bfloat16, got backward_dtype=%r with compute_dtype=%r"
                         % (backward_dtype, compute_dtype))
    return backward_dtype


def _bf16_forward(what, input, offset, mask, offset_mask, weight, bias, stride, padding, dilation, dg,
                  bn_scale=None, bn_shift=None, relu=False):
    """One call of cnb_dcnv2_forward_bf16 (or, with offset_mask, cnb_dcnv2_forward_fused_bf16).  The output has the
    input's dtype.  A channels_last input with whole 32-channel blocks is read as it is (a bf16 one in place)."""
    if not input.is_cuda:
        raise NotImplementedError
    if input.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("%s: compute_dtype=torch.bfloat16 takes a float32 or bfloat16 input, got %s"
                           % (what, input.dtype))
    n, cin, h, wd = [int(v) for v in input.shape]
    cout, cin_w, kh, kw = [int(v) for v in weight.shape]
    if cin_w != cin:
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (cin, cin_w))
    if kh * kw > 9:
        raise NotImplementedError("%s: compute_dtype=torch.bfloat16 runs at most 9 taps" % what)
    ho, wo = _out_hw(h, wd, kh, kw, stride, padding, dilation)
    kt = kh * kw
    if offset_mask is not None:
        om = f32c(offset_mask)
        if tuple(om.shape) != (n, 3 * kt * dg, ho, wo):
            raise RuntimeError("%s: offset_mask must be [%d, %d, %d, %d]" % (what, n, 3 * kt * dg, ho, wo))
    else:
        off, msk = f32c(offset), f32c(mask)
        if tuple(off.shape) != (n, 2 * kt * dg, ho, wo) or tuple(msk.shape) != (n, kt * dg, ho, wo):
            raise RuntimeError("DCNv2: offset/mask shape does not match the output grid")
    cl = (cin // dg) % 32 == 0 and input.is_contiguous(memory_format=torch.channels_last) and \
        not input.is_contiguous()
    x = input if cl else input.contiguous()
    if x.data_ptr() % 16:
        x = x.clone()               # the kernels read 16-byte pieces (clone keeps the memory format)
    dt = C.DTYPE_BF16 if x.dtype == torch.bfloat16 else C.DTYPE_F32
    wt = _weight_tiles(weight, dg, bf16=True)
    out = torch.empty((n, cout, ho, wo), dtype=input.dtype, device=input.device)
    ws = workspace(C.dcnv2_bf16_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding, dilation, dg),
                   input.device)
    b = f32c(bias)
    if offset_mask is not None:
        sc, sh = f32c(bn_scale), f32c(bn_shift)
        C.dcnv2_forward_fused_bf16(ptr(x), dt, int(cl), ptr(om), ptr(wt), ptr(b), ptr(sc), ptr(sh), int(bool(relu)),
                                   ptr(out), dt, n, cin, h, wd, cout, kh, kw, stride, padding, dilation, dg, ptr(ws),
                                   ws.numel(), stream_ptr(om))
        return out, None, None
    C.dcnv2_forward_bf16(ptr(x), dt, int(cl), ptr(off), ptr(msk), ptr(wt), ptr(b), ptr(out), dt, n, cin, h, wd, cout,
                         kh, kw, stride, padding, dilation, dg, ptr(ws), ws.numel(), stream_ptr(off))
    return out, off, msk


class _DCNv2BF16(Function):
    """bf16 forward.  bf16_backward=False: the backward is the fp32 one evaluated at the operands the forward used (the
    bf16 activation and weight, upcast exactly); True: the bf16 backward (cnb_dcnv2_backward_bf16) where it runs, that
    fp32 one elsewhere (cout > 256).  Each gradient is returned in its input's dtype; the activation is saved as
    bf16."""

    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups,
                bf16_backward=False):
        out, off, msk = _bf16_forward("DCNv2", input, offset, mask, None, weight, bias, stride, padding, dilation,
                                      deformable_groups)
        if any(ctx.needs_input_grad[:5]):
            xb = input if input.dtype == torch.bfloat16 else input.bfloat16()
            ctx.save_for_backward(xb, off, msk, weight, bias)
        ctx.dtypes = tuple(None if t is None else t.dtype for t in (input, offset, mask, weight, bias))
        ctx.cfg = (stride, padding, dilation, deformable_groups)
        ctx.bf16_backward = bool(bf16_backward)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        if not grad_output.is_cuda:
            raise NotImplementedError
        xb, off, msk, weight, bias = ctx.saved_tensors
        grads = _dcn_backward_bf16(xb, off, msk, weight, bias, grad_output, ctx.cfg) if ctx.bf16_backward else None
        if grads is None:
            x = xb.float().contiguous()
            w = weight.bfloat16().float().contiguous()
            grads = _dcn_backward_f32(x, off, msk, w, f32c(bias), f32c(grad_output), ctx.cfg, False)
        grads = tuple(None if g is None else g.to(dt) for g, dt in zip(grads, ctx.dtypes))
        return grads + (None,) * 5


def _dcn_backward_bf16(xb, off, msk, weight, bias, grad_output, cfg):
    """One call of cnb_dcnv2_backward_bf16 on the saved bf16 activation: the five gradients in fp32, or None where
    that backward does not run (the workspace query returns 0: cout > 256 or an image beyond its 32-bit indexing).
    A channels_last activation with whole 32-channel blocks is read as it is and gets a channels_last grad_input."""
    stride, padding, dilation, dg = cfg
    n, cin, h, wd = [int(v) for v in xb.shape]
    cout, _, kh, kw = [int(v) for v in weight.shape]
    det = _deterministic()
    C.dcnv2_set_deterministic(int(det))
    wsb = C.dcnv2_backward_bf16_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding, dilation, dg)
    if wsb == 0:
        return None
    cl = (cin // dg) % 32 == 0 and xb.is_contiguous(memory_format=torch.channels_last) and not xb.is_contiguous()
    x = xb if cl else xb.contiguous()
    if x.data_ptr() % 16:
        x = x.clone()               # the kernels read 16-byte pieces (clone keeps the memory format)
    go = grad_output if grad_output.dtype == torch.bfloat16 else grad_output.float()
    go = go.contiguous()
    w = f32c(weight)
    gx = torch.zeros_like(x, dtype=torch.float32)     # keeps x's layout: channels_last when cl
    goff, gmsk, gw = torch.zeros_like(off), torch.zeros_like(msk), torch.zeros_like(w)
    gb = torch.zeros(cout, dtype=torch.float32, device=x.device) if bias is not None else None
    ws = workspace(wsb, x.device)
    C.dcnv2_backward_bf16(ptr(x), C.DTYPE_BF16, int(cl), ptr(off), ptr(msk), ptr(w), ptr(go),
                          C.DTYPE_BF16 if go.dtype == torch.bfloat16 else C.DTYPE_F32, ptr(gx), int(cl), ptr(goff),
                          ptr(gmsk), ptr(gw), ptr(gb), n, cin, h, wd, cout, kh, kw, stride, padding, dilation, dg,
                          ptr(ws), ws.numel(), stream_ptr(x))
    return gx, goff, gmsk, gw, gb


def dcn_fused_inference(input, offset_mask, weight, bias, stride, padding, dilation, deformable_groups,
                        bn_scale=None, bn_shift=None, relu=False, compute_dtype=None):
    """Inference form of the whole DCN module around ONE kernel (cnb_dcnv2_forward_fused): `offset_mask` is the raw
    conv_offset_mask output (chunk / cat / sigmoid of dcn_v2.py:64-70 happen inside the sampler), bn_scale /
    bn_shift / relu the folded BatchNorm + ReLU that follow the DCN in DeformConv (pose_dla_dcn.py:345-357).
    compute_dtype=torch.bfloat16: the bf16 forward (cnb_dcnv2_forward_fused_bf16), output in the input's dtype.
    No autograd (use DCNv2Function for training)."""
    if _check_compute_dtype(compute_dtype) is not None:
        return _bf16_forward("dcn_fused_inference", input, None, None, offset_mask, weight, bias, stride, padding,
                             dilation, deformable_groups, bn_scale, bn_shift, relu)[0]
    if not input.is_cuda:
        raise NotImplementedError
    if input.dtype == torch.float64:
        raise NotImplementedError("dcn_fused_inference: float32 only; float64 runs through DCNv2Function")
    n, cin, h, wd = [int(v) for v in input.shape]
    cout, cin_w, kh, kw = [int(v) for v in weight.shape]
    if cin_w != cin:
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (cin, cin_w))
    if kh * kw > 9:
        raise NotImplementedError("dcn_fused_inference: at most 9 taps")
    ho, wo = _out_hw(h, wd, kh, kw, stride, padding, dilation)
    om = f32c(offset_mask)
    if tuple(om.shape) != (n, 3 * kh * kw * deformable_groups, ho, wo):
        raise RuntimeError("dcn_fused_inference: offset_mask must be [%d, %d, %d, %d]" % (n, 3 * kh * kw * deformable_groups, ho, wo))
    nhwc = (cin // deformable_groups) % 32 == 0 and input.dtype == torch.float32 and \
        input.is_contiguous(memory_format=torch.channels_last) and not input.is_contiguous()
    xin = input if nhwc else f32c(input)
    wt = _weight_tiles(weight, deformable_groups)
    out = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=input.device)
    ws = workspace(C.dcnv2_prepared_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding, dilation,
                                                    deformable_groups), input.device)
    b = f32c(bias)
    sc, sh = f32c(bn_scale), f32c(bn_shift)
    C.dcnv2_forward_fused(ptr(xin), int(nhwc), ptr(om), ptr(wt), ptr(b), ptr(sc), ptr(sh), int(bool(relu)), ptr(out),
                          n, cin, h, wd, cout, kh, kw, stride, padding, dilation, deformable_groups, ptr(ws),
                          ws.numel(), stream_ptr(om))
    return out


# ------------------------------------------------------------------ DCN block (opt-in: dcn_v2.fuse_offset_conv)
def _om_tiles(w_om):
    """bf16 tiles of a conv_offset_mask weight (cnb_dcnv2_prepare_om_weights_bf16), cached per weight version next to
    the tiles of _weight_tiles: rebuilt when torch bumps `_version` (optimizer step, load_state_dict), tied to the
    tensor object by a weak reference."""
    key = (id(w_om), "om")
    hit = _WT_CACHE.get(key)
    if hit is not None and hit[0]() is w_om and hit[1] == w_om._version and hit[2].device == w_om.device:
        return hit[2]
    ver = w_om._version
    w = f32c(w_om)
    cin = int(w.shape[1])
    t = workspace(C.dcnv2_om_tiles_bytes(cin, 3, 3, 1), w.device)
    C.dcnv2_prepare_om_weights_bf16(ptr(w), cin, 3, 3, 1, ptr(t), t.numel(), stream_ptr(w))
    try:
        _WT_CACHE[key] = (weakref.ref(w_om, lambda _r, k=key: _WT_CACHE.pop(k, None)), ver, t)
    except TypeError:          # not weak-referenceable: do not cache
        pass
    return t


def dcn_block_inference(input, w_om, b_om, weight, bias, stride, padding, dilation, deformable_groups,
                        bn_scale=None, bn_shift=None, relu=False):
    """Inference form of a whole DCN module in ONE kernel (cnb_dcnv2_forward_block_bf16): conv_offset_mask (w_om,
    b_om), the chunk / cat / sigmoid and the bf16 deformable conv, plus the optional folded BatchNorm + ReLU.  The
    offsets are computed in fp32 from bf16 operands and never leave the chip; from them on the result is
    dcn_fused_inference(..., compute_dtype=torch.bfloat16) fed those offsets.  Output in the input's dtype.  Returns
    None where the kernel does not run (not a CUDA float32 / bfloat16 input, outside its range -- 3x3, stride 1,
    padding 1, dilation 1, one deformable group, input channels a multiple of 32); the caller then runs
    conv_offset_mask and dcn_fused_inference.  No autograd."""
    if not input.is_cuda or input.dtype not in (torch.float32, torch.bfloat16) or input.dim() != 4:
        return None
    n, cin, h, wd = [int(v) for v in input.shape]
    cout, cin_w, kh, kw = [int(v) for v in weight.shape]
    if cin_w != cin or tuple(w_om.shape) != (3 * kh * kw * deformable_groups, cin, kh, kw):
        return None
    wsb = C.dcnv2_block_workspace_bytes(n, cin, cout, h, wd, kh, kw, stride, padding, dilation, deformable_groups)
    if wsb == 0:
        return None
    cl = input.is_contiguous(memory_format=torch.channels_last) and not input.is_contiguous()
    x = input if cl else input.contiguous()
    if x.data_ptr() % 16:
        x = x.clone()               # the kernel reads 16-byte pieces (clone keeps the memory format)
    dt = C.DTYPE_BF16 if x.dtype == torch.bfloat16 else C.DTYPE_F32
    wt = _weight_tiles(weight, deformable_groups, bf16=True)
    omt = _om_tiles(w_om)
    out = torch.empty((n, cout, h, wd), dtype=input.dtype, device=input.device)
    ws = workspace(wsb, input.device)
    bom, b, sc, sh = f32c(b_om), f32c(bias), f32c(bn_scale), f32c(bn_shift)
    C.dcnv2_forward_block_bf16(ptr(x), dt, int(cl), ptr(omt), ptr(bom), ptr(wt), ptr(b), ptr(sc), ptr(sh),
                               int(bool(relu)), ptr(out), n, cin, h, wd, cout, kh, kw, stride, padding, dilation,
                               deformable_groups, ptr(ws), ws.numel(), stream_ptr(x))
    return out


class DCNv2Function(object):
    """Callable instance, same constructor as the reference's old-style Function.  compute_dtype=torch.bfloat16
    selects the bf16 forward (float32 or bfloat16 input, output in the input's dtype); None keeps the default.
    backward_dtype=torch.bfloat16 (with compute_dtype=torch.bfloat16 only) selects the bf16 backward; None keeps the
    fp32 backward at the operands the bf16 forward used."""

    def __init__(self, stride, padding, dilation=1, deformable_groups=1, compute_dtype=None, backward_dtype=None):
        self.stride = stride
        self.padding = padding
        self.dilation = dilation
        self.deformable_groups = deformable_groups
        self.compute_dtype = _check_compute_dtype(compute_dtype)
        self.backward_dtype = _check_backward_dtype(self.compute_dtype, backward_dtype)

    def __call__(self, input, offset, mask, weight, bias):
        if self.compute_dtype is not None:
            return _DCNv2BF16.apply(input, offset, mask, weight, bias, self.stride, self.padding, self.dilation,
                                    self.deformable_groups, self.backward_dtype is not None)
        return _DCNv2.apply(input, offset, mask, weight, bias, self.stride, self.padding, self.dilation,
                            self.deformable_groups)

    forward = __call__


def _psroi_check(rois, offset, no_trans, part_size):
    if rois.dim() != 2 or rois.shape[1] != 5:
        raise RuntimeError("DCNv2PoolingFunction: rois must be [n, 5], got %s" % (tuple(rois.shape),))
    if not no_trans and (offset.dim() != 4 or offset.shape[0] < rois.shape[0] or
                         tuple(offset.shape[2:]) != (part_size, part_size)):
        raise RuntimeError("DCNv2PoolingFunction: offset must be [>=n, 2*classes, %d, %d], got %s"
                           % (part_size, part_size, tuple(offset.shape)))


def _psroi_forward_f64(ctx, data, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size,
                       part_size, sample_per_part, trans_std):
    """float64 (dcn_v2_psroi_pooling_cuda_double.cu); rois may be float32 or float64 (both hold box corners
    exactly in float64)."""
    no_trans = bool(no_trans)
    if rois.dtype not in (torch.float32, torch.float64):
        raise RuntimeError("DCNv2PoolingFunction: rois must be float32 or float64, got %s" % (rois.dtype,))
    data, = _f64c("DCNv2PoolingFunction", data)
    rois = rois.double().contiguous()
    if not no_trans:
        offset, = _f64c("DCNv2PoolingFunction", offset)
    _psroi_check(rois, offset, no_trans, part_size)
    n, (b, c, h, w) = int(rois.shape[0]), data.shape
    out = torch.empty((n, output_dim, pooled_size, pooled_size), dtype=torch.float64, device=data.device)
    cnt = torch.empty_like(out)
    ct = 2 if no_trans else int(offset.shape[1])
    C.psroi_pooling_forward_f64(ptr(data), ptr(rois), 0 if no_trans else ptr(offset), ptr(out), ptr(cnt), b, c, h, w,
                                n, ct, int(no_trans), float(spatial_scale), output_dim, group_size, pooled_size,
                                part_size, sample_per_part, float(trans_std), stream_ptr(data))
    ctx.save_for_backward(data, rois, offset if not no_trans else data.new_empty(0), cnt)
    ctx.cfg = (spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size, sample_per_part, trans_std, ct)
    return out


def _psroi_backward_f64(ctx, grad_output):
    data, rois, offset, cnt = ctx.saved_tensors
    spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size, sample_per_part, trans_std, ct = ctx.cfg
    go = grad_output.double().contiguous()
    grad_input = torch.zeros_like(data)
    grad_offset = None if no_trans else torch.zeros_like(offset)
    n, (b, c, h, w) = int(rois.shape[0]), data.shape
    ws = workspace(C.psroi_pooling_f64_workspace_bytes(b, c, h, w), data.device)
    C.psroi_pooling_backward_f64(ptr(go), ptr(data), ptr(rois), 0 if no_trans else ptr(offset), ptr(cnt),
                                 ptr(grad_input), 0 if no_trans else ptr(grad_offset), b, c, h, w, n, ct,
                                 int(no_trans), float(spatial_scale), output_dim, group_size, pooled_size, part_size,
                                 sample_per_part, float(trans_std), ptr(ws), ws.numel(), stream_ptr(data))
    return (grad_input, None, grad_offset) + (None,) * 8


class _PSROIPooling(Function):
    """dcn_v2_func.py:76-146 as a modern autograd.Function."""

    @staticmethod
    def forward(ctx, data, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size,
                sample_per_part, trans_std):
        if not data.is_cuda:
            raise NotImplementedError("DCNv2PoolingFunction: CUDA tensors only (dcn_v2_func.py:100-101)")
        ctx.f64 = data.dtype == torch.float64
        if ctx.f64:
            return _psroi_forward_f64(ctx, data, rois, offset, spatial_scale, pooled_size, output_dim, no_trans,
                                      group_size, part_size, sample_per_part, trans_std)
        data, rois = f32c(data), f32c(rois)
        no_trans = bool(no_trans)
        if not no_trans:
            offset = f32c(offset)
        _psroi_check(rois, offset, no_trans, part_size)
        n, (b, c, h, w) = int(rois.shape[0]), data.shape
        out = torch.empty((n, output_dim, pooled_size, pooled_size), dtype=torch.float32, device=data.device)
        cnt = torch.empty_like(out)
        ct = 2 if no_trans else int(offset.shape[1])
        C.psroi_pooling_forward(ptr(data), ptr(rois), 0 if no_trans else ptr(offset), ptr(out), ptr(cnt), b, c, h, w,
                                n, ct, int(no_trans), float(spatial_scale), output_dim, group_size, pooled_size,
                                part_size, sample_per_part, float(trans_std), stream_ptr(data))
        ctx.save_for_backward(data, rois, offset if not no_trans else data.new_empty(0), cnt)
        ctx.cfg = (spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size, sample_per_part, trans_std, ct)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        if not grad_output.is_cuda:
            raise NotImplementedError("DCNv2PoolingFunction: CUDA tensors only (dcn_v2_func.py:117-118)")
        if ctx.f64:     # bit-reproducible in every mode: no alert
            return _psroi_backward_f64(ctx, grad_output)
        if _deterministic():
            _alert_not_deterministic("DCNv2PoolingFunction backward (atomic scatter)")
        data, rois, offset, cnt = ctx.saved_tensors
        spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size, sample_per_part, trans_std, ct = ctx.cfg
        grad_output = f32c(grad_output)
        grad_input = torch.zeros_like(data)                                   # :119-120, accumulated into
        grad_offset = None if no_trans else torch.zeros_like(offset)
        n, (b, c, h, w) = int(rois.shape[0]), data.shape
        C.psroi_pooling_backward(ptr(grad_output), ptr(data), ptr(rois), 0 if no_trans else ptr(offset), ptr(cnt),
                                 ptr(grad_input), 0 if no_trans else ptr(grad_offset), b, c, h, w, n, ct, int(no_trans),
                                 float(spatial_scale), output_dim, group_size, pooled_size, part_size, sample_per_part,
                                 float(trans_std), stream_ptr(data))
        return (grad_input, None, grad_offset) + (None,) * 8


class DCNv2PoolingFunction(object):
    """Deformable PSROI pooling, callable as an instance like the reference's old-style Function
    (dcn_v2_func.py:76-146): `DCNv2PoolingFunction(spatial_scale, pooled_size, output_dim, no_trans,
    group_size=1, part_size=None, sample_per_part=4, trans_std=.0)(data, rois, offset)`."""

    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0):
        self.spatial_scale = spatial_scale
        self.pooled_size = pooled_size
        self.output_dim = output_dim
        self.no_trans = no_trans
        self.group_size = group_size
        self.part_size = pooled_size if part_size is None else part_size
        self.sample_per_part = sample_per_part
        self.trans_std = trans_std
        assert 0.0 <= self.trans_std <= 1.0                                    # :97

    def __call__(self, data, rois, offset):
        return _PSROIPooling.apply(data, rois, offset, self.spatial_scale, self.pooled_size, self.output_dim,
                                   self.no_trans, self.group_size, self.part_size, self.sample_per_part,
                                   self.trans_std)

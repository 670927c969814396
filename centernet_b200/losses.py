"""Mirror of src/lib/models/losses.py for the classes the trainers use
(trains/ctdet.py:19-25, trains/multi_pose.py:18-26, trains/exdet.py:19-23):
FocalLoss / _neg_loss, RegL1Loss, RegLoss, NormRegL1Loss, RegWeightedL1Loss, plus
FocalSplatLoss -- the same focal loss with the Gaussian target rebuilt on the fly from
per-image object lists (utils/image.py:126-141 + datasets/sample/ctdet.py:111-117), so the
dense target map is never built on the CPU nor copied to the device.

Each loss is a torch.autograd.Function whose forward runs ONE fused CUDA pass that also
produces the gradient (saved for backward), i.e. forward+backward read the prediction once.

A bf16 / fp16 prediction (the head of a bf16 backbone, or of one under autocast) is read in place: forward runs
the loss pass on the half tensor and saves it, backward runs the gradient pass, which reads the incoming gradient
on the device and writes the gradient in the input's dtype (FocalSplatLoss keeps its unscaled fp32 gradient
instead and backward scales and rounds it).  Loss and gradient are bit for bit those of the fp32 path on the
.float() upcast (the gradient rounded once, after the scale); no fp32 copy of the input is made.
"""
import torch
from torch import nn

from ._lib import C, dtype_code, f32c, floatc, ptr, require_cuda, stream_ptr, workspace

_HALF = (torch.bfloat16, torch.float16)


class _FocalFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt, logits):
        require_cuda(pred, gt, what="FocalLoss")
        ctx.half = pred.dtype in _HALF
        if ctx.half:
            p, g = floatc(pred), f32c(gt)
            out = torch.empty(2, dtype=torch.float32, device=p.device)
            ws = workspace(C.focal_workspace_bytes(p.numel()), p.device)
            C.focal_loss_ex(ptr(p), dtype_code(p), ptr(g), p.numel(), int(logits), ptr(out), ptr(ws), ws.numel(),
                            stream_ptr(p))
            if pred.requires_grad:
                ctx.save_for_backward(p, g, out)
                ctx.logits = int(logits)
            return out[0]
        p, g = f32c(pred), f32c(gt)
        out = torch.empty(2, dtype=torch.float32, device=p.device)
        need_grad = pred.requires_grad
        grad = torch.empty_like(p) if need_grad else None
        ws = workspace(C.focal_workspace_bytes(p.numel()), p.device)
        C.focal_loss(ptr(p), ptr(g), p.numel(), int(logits), 1.0, ptr(out), ptr(grad), ptr(ws), ws.numel(),
                     stream_ptr(p))
        ctx.save_for_backward(grad)
        return out[0]

    @staticmethod
    def backward(ctx, grad_out):
        if ctx.half:
            if not ctx.needs_input_grad[0]:
                return None, None, None
            p, g, out = ctx.saved_tensors
            grad, go = torch.empty_like(p), f32c(grad_out)
            C.focal_grad_ex(ptr(p), dtype_code(p), ptr(g), p.numel(), ctx.logits, ptr(out), ptr(go),
                            ptr(grad), stream_ptr(p))
            return grad, None, None
        (grad,) = ctx.saved_tensors
        return (grad * grad_out if grad is not None else None), None, None


def _neg_loss(pred, gt):
    """models/losses.py:42-67: penalty-reduced pixel-wise focal loss on an already
    sigmoided/clamped prediction (trains/ctdet.py:34 applies _sigmoid first)."""
    return _FocalFn.apply(pred, gt, False)


def _neg_loss_from_logits(logits, gt):
    """_sigmoid (models/utils.py:8-10) + _neg_loss fused: takes the raw head output."""
    return _FocalFn.apply(logits, gt, True)


class FocalLoss(nn.Module):
    """models/losses.py:114-121."""

    def __init__(self):
        super().__init__()
        self.neg_loss = _neg_loss

    def forward(self, out, target):
        return self.neg_loss(out, target)


class _FocalSplatFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, logits):
        require_cuda(pred, obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, what="FocalSplatLoss")
        ctx.half = pred.dtype in _HALF
        p = floatc(pred) if ctx.half else f32c(pred)
        b, c, h, w = [int(v) for v in p.shape]
        m = int(obj_cls.shape[1])
        i32 = lambda t: t.to(torch.int32).contiguous()
        cls, cx, cy, rad = i32(obj_cls), i32(obj_cx), i32(obj_cy), i32(obj_radius)
        val = obj_valid.to(torch.uint8).contiguous()
        out = torch.empty(2, dtype=torch.float32, device=p.device)
        ws = workspace(C.focal_workspace_bytes(p.numel()), p.device)
        if ctx.half:   # the unscaled fp32 gradient is kept: rebuilding the target in backward costs more (DESIGN 4.3.1)
            g32 = torch.empty(p.shape, dtype=torch.float32, device=p.device) if pred.requires_grad else None
            C.focal_splat_loss_ex(ptr(p), dtype_code(p), ptr(cls), ptr(cx), ptr(cy), ptr(rad), ptr(val), b, m, c, h, w,
                                  int(logits), ptr(out), ptr(g32), ptr(ws), ws.numel(), stream_ptr(p))
            ctx.save_for_backward(g32)
            ctx.dtype = p.dtype
            return out[0]
        grad = torch.empty_like(p) if pred.requires_grad else None
        C.focal_splat_loss(ptr(p), ptr(cls), ptr(cx), ptr(cy), ptr(rad), ptr(val), b, m, c, h, w, int(logits), 1.0,
                           ptr(out), ptr(grad), ptr(ws), ws.numel(), stream_ptr(p))
        ctx.save_for_backward(grad)
        return out[0]

    @staticmethod
    def backward(ctx, grad_out):
        if ctx.half:
            (g32,) = ctx.saved_tensors
            if g32 is None or not ctx.needs_input_grad[0]:
                return (None,) * 7
            grad, go = torch.empty(g32.shape, dtype=ctx.dtype, device=g32.device), f32c(grad_out)
            C.focal_splat_grad_ex(ptr(g32), g32.numel(), ptr(go), ptr(grad), dtype_code(grad), stream_ptr(g32))
            return (grad,) + (None,) * 6
        (grad,) = ctx.saved_tensors
        return (grad * grad_out if grad is not None else None), None, None, None, None, None, None


class FocalSplatLoss(nn.Module):
    """Focal loss against the Gaussian target of the listed objects, fused.

    forward(out [B,C,H,W], obj_cls, obj_cx, obj_cy, obj_radius, obj_valid  (all [B,M])):
    obj_cx/obj_cy are the integer centres ``ct_int`` and obj_radius the
    ``max(0, int(gaussian_radius(...)))`` of datasets/sample/ctdet.py:111-117.
    A centre outside the map paints the part of its window that overlaps the map, as
    draw_umich_gaussian does; objects with obj_valid = 0, a negative radius or a class
    outside [0, C) are skipped.

    num_pos is counted from the lists: one positive per distinct valid centre inside the
    map.  That is the reference's count of target pixels equal to 1 up to a radius of about
    12,000: beyond it the fp32 target next to the centre rounds to 1 as well, and the
    reference counts those pixels too.  gaussian_radius of any box on a 512x512 input
    stays far below that."""

    def __init__(self, from_logits=False):
        super().__init__()
        self.from_logits = from_logits

    def forward(self, out, obj_cls, obj_cx, obj_cy, obj_radius, obj_valid):
        return _FocalSplatFn.apply(out, obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, self.from_logits)


def splat_gaussian(obj_cls, obj_cx, obj_cy, obj_radius, obj_valid, num_classes, height, width):
    """Dense [B,C,H,W] target built on the device (draw_umich_gaussian, utils/image.py:126-141), bit for
    bit; centres outside the map paint the overlap of their window, as there."""
    require_cuda(obj_cls, what="splat_gaussian")
    i32 = lambda t: t.to(torch.int32).contiguous()
    cls, cx, cy, rad = i32(obj_cls), i32(obj_cx), i32(obj_cy), i32(obj_radius)
    val = obj_valid.to(torch.uint8).contiguous()
    b, m = [int(v) for v in cls.shape]
    hm = torch.empty((b, num_classes, height, width), dtype=torch.float32, device=cls.device)
    C.splat_gaussian(ptr(cls), ptr(cx), ptr(cy), ptr(rad), ptr(val), b, m, num_classes, height, width, ptr(hm),
                     stream_ptr(cls))
    return hm


class _RegFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, output, mask, ind, target, mode):
        require_cuda(output, mask, ind, target, what="RegLoss")
        ctx.half = output.dtype in _HALF
        o, t = (floatc(output) if ctx.half else f32c(output)), f32c(target)
        b, d = int(o.shape[0]), int(o.shape[1])
        hw = int(o.shape[2]) * int(o.shape[3])
        m = int(ind.shape[1])
        msk = f32c(mask)   # mask.float() as in the reference: bool, uint8 and fractional float weights alike
        ind = ind.long().contiguous()
        if ctx.half:
            out = torch.empty(2, dtype=torch.float32, device=o.device)   # loss, the gradient's denominator
            C.reg_loss_ex(ptr(o), dtype_code(o), ptr(msk), ptr(ind), ptr(t), b, d, hw, m, mode, ptr(out), stream_ptr(o))
            if output.requires_grad:
                ctx.save_for_backward(o, msk, ind, t, out)
                ctx.mode = mode
            return out[0]
        out = torch.empty(1, dtype=torch.float32, device=o.device)
        grad = torch.zeros_like(o) if output.requires_grad else None
        C.reg_loss(ptr(o), ptr(msk), ptr(ind), ptr(t), b, d, hw, m, mode, 1.0, ptr(out), ptr(grad), stream_ptr(o))
        ctx.save_for_backward(grad)
        return out[0]

    @staticmethod
    def backward(ctx, grad_out):
        if ctx.half:
            if not ctx.needs_input_grad[0]:
                return (None,) * 5
            o, msk, ind, t, out = ctx.saved_tensors
            grad, go = torch.empty_like(o), f32c(grad_out)   # the call fills all of grad
            C.reg_loss_grad_ex(ptr(o), dtype_code(o), ptr(msk), ptr(ind), ptr(t), int(o.shape[0]), int(o.shape[1]),
                               int(o.shape[2]) * int(o.shape[3]), int(ind.shape[1]), ctx.mode, ptr(out),
                               ptr(go), ptr(grad), stream_ptr(o))
            return (grad,) + (None,) * 4
        (grad,) = ctx.saved_tensors
        return (grad * grad_out if grad is not None else None), None, None, None, None


class RegL1Loss(nn.Module):
    """models/losses.py:139-149."""

    def forward(self, output, mask, ind, target):
        return _RegFn.apply(output, mask, ind, target, 0)


class RegLoss(nn.Module):
    """models/losses.py:123-137 (smooth-L1 / (num + 1e-4))."""

    def forward(self, output, mask, ind, target):
        return _RegFn.apply(output, mask, ind, target, 1)


class NormRegL1Loss(nn.Module):
    """models/losses.py:151-163."""

    def forward(self, output, mask, ind, target):
        return _RegFn.apply(output, mask, ind, target, 2)


class RegWeightedL1Loss(nn.Module):
    """models/losses.py:165-175 (mask is a float weight [B, M, D])."""

    def forward(self, output, mask, ind, target):
        return _RegFn.apply(output, mask, ind, target, 3)


# ------------------------------------------------------------------ ddd-only ride-alongs (trains/ddd.py:14)
# Not on the heat-map hot path (SURVEY 8a stops at A16): kept so that a full overlay of models/losses.py
# exports every class the trainers import.  The gather is the library's kernel (differentiable); the few
# hundred gathered values are reduced with stock tensor ops.
from .utils import _transpose_and_gather_feat  # noqa: E402
import torch.nn.functional as F  # noqa: E402


class L1Loss(nn.Module):
    """models/losses.py:177-185 (mean over all B*M*D elements of the masked L1)."""

    def forward(self, output, mask, ind, target):
        pred = _transpose_and_gather_feat(output, ind)
        m = mask.unsqueeze(2).expand_as(pred).float()
        return F.l1_loss(pred * m, target * m, reduction="mean")


def compute_rot_loss(output, target_bin, target_res, mask):
    """models/losses.py:205-237: two orientation bins, each a 2-way classification (cross entropy on the
    mask-zeroed logits, mean over all rows) plus smooth-L1 on sin/cos of the residual over the rows whose
    bin label is set (mean over those rows, skipped when there are none)."""
    output = output.reshape(-1, 8)
    target_bin = target_bin.reshape(-1, 2)
    target_res = target_res.reshape(-1, 2)
    m = mask.reshape(-1, 1).float()
    total = output.new_zeros(())
    for k in range(2):
        logits = output[:, 4 * k:4 * k + 2] * m
        total = total + F.cross_entropy(logits, target_bin[:, k].long(), reduction="mean")
        rows = target_bin[:, k].nonzero()[:, 0]
        if rows.numel() > 0:
            o = output.index_select(0, rows)
            r = target_res.index_select(0, rows)[:, k]
            total = total + F.smooth_l1_loss(o[:, 4 * k + 2], torch.sin(r), reduction="mean") \
                          + F.smooth_l1_loss(o[:, 4 * k + 3], torch.cos(r), reduction="mean")
    return total


class BinRotLoss(nn.Module):
    """models/losses.py:187-194."""

    def forward(self, output, mask, ind, rotbin, rotres):
        pred = _transpose_and_gather_feat(output, ind)
        return compute_rot_loss(pred, rotbin, rotres, mask)

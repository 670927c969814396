"""Mirror of src/lib/models/utils.py (reference lines cited per function)."""
import torch

from ._lib import C, dtype_code, f32c, floatc, ptr, require_cuda, stream_ptr


def _sigmoid(x):
    """models/utils.py:8-10 -- in-place sigmoid then clamp to [1e-4, 1-1e-4]."""
    return torch.clamp(x.sigmoid_(), min=1e-4, max=1 - 1e-4)


def _gather_feat(feat, ind, mask=None):
    """models/utils.py:12-20.  feat [B, N, D], ind [B, M] -> [B, M, D].
    Index plumbing only (not a hot kernel): plain tensor ops on the caller's device."""
    dim = feat.size(2)
    ind = ind.unsqueeze(2).expand(ind.size(0), ind.size(1), dim)
    feat = feat.gather(1, ind)
    if mask is not None:
        mask = mask.unsqueeze(2).expand_as(feat)
        feat = feat[mask].view(-1, dim)
    return feat


class _TransposeGather(torch.autograd.Function):
    """Differentiable like the reference's permute + gather: the losses of models/losses.py
    (RegL1Loss, RegLoss, NormRegL1Loss, RegWeightedL1Loss, L1Loss, BinRotLoss) back-propagate
    through `pred = _transpose_and_gather_feat(output, ind)`.  A bf16 / fp16 feat is read in place (the rows
    come out in fp32, as for any dtype) and its gradient is written in its dtype: the fp32 scatter of the upcast
    rounded once, with no fp32 map in between."""

    @staticmethod
    def forward(ctx, feat, ind):
        half = feat.dtype in (torch.bfloat16, torch.float16)
        f = floatc(feat) if half else f32c(feat)
        ind = ind.contiguous().long()
        B, Cc, H, W = f.shape
        M = ind.shape[1]
        out = torch.empty((B, M, Cc), dtype=torch.float32, device=f.device)
        if B * M * Cc and half:
            C.gather_feat_ex(ptr(f), dtype_code(f), ptr(ind), ptr(out), B, Cc, H * W, M, stream_ptr(f))
        elif B * M * Cc:
            C.gather_feat(ptr(f), ptr(ind), ptr(out), B, Cc, H * W, M, stream_ptr(f))
        ctx.save_for_backward(ind)
        ctx.shape = (B, Cc, H, W)
        ctx.in_dtype = feat.dtype
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (ind,) = ctx.saved_tensors
        B, Cc, H, W = ctx.shape
        g = f32c(grad_out)
        M = ind.shape[1]
        if ctx.in_dtype in (torch.bfloat16, torch.float16):
            if B * M * Cc == 0:
                return torch.zeros((B, Cc, H, W), dtype=ctx.in_dtype, device=g.device), None
            grad_feat = torch.empty((B, Cc, H, W), dtype=ctx.in_dtype, device=g.device)   # the call zero-fills it
            C.gather_feat_backward_ex(ptr(g), ptr(ind), ptr(grad_feat), dtype_code(grad_feat), B, Cc, H * W, M,
                                      stream_ptr(g))
            return grad_feat, None
        grad_feat = torch.zeros((B, Cc, H, W), dtype=torch.float32, device=g.device)
        if B * M * Cc:
            C.gather_feat_backward(ptr(g), ptr(ind), ptr(grad_feat), B, Cc, H * W, M, stream_ptr(g))
        return grad_feat.to(ctx.in_dtype), None


def _transpose_and_gather_feat(feat, ind):
    """models/utils.py:22-26, without the full NCHW->NHWC transpose copy: the kernel
    reads feat[b, :, ind[b, m]] directly.  feat [B, C, H, W], ind [B, M] -> [B, M, C].
    Differentiable w.r.t. feat (scatter-add adjoint, cnb_gather_feat_backward)."""
    require_cuda(feat, ind, what="_transpose_and_gather_feat")
    return _TransposeGather.apply(feat, ind)


def flip_tensor(x):
    """models/utils.py:28-29."""
    return torch.flip(x, [3])


def flip_lr(x, flip_idx):
    """models/utils.py:33-39 -- stays on the device (the reference round-trips via numpy)."""
    tmp = torch.flip(x, [3]).clone()
    for e in flip_idx:
        a = tmp[:, e[0]].clone()
        tmp[:, e[0]] = tmp[:, e[1]]
        tmp[:, e[1]] = a
    return tmp


def flip_lr_off(x, flip_idx):
    """models/utils.py:41-50."""
    shape = x.shape
    tmp = torch.flip(x, [3]).clone().view(shape[0], 17, 2, shape[2], shape[3])
    tmp[:, :, 0] *= -1
    for e in flip_idx:
        a = tmp[:, e[0]].clone()
        tmp[:, e[0]] = tmp[:, e[1]]
        tmp[:, e[1]] = a
    return tmp.view(shape)

"""Fused inference for the IDA up-sampling of DLASeg (cnb_ida_up_add).

Every step of pose_dla_dcn's ``IDAUp.forward`` projects ``layers[i]`` with a DeformConv, up-samples it with a
depthwise ``ConvTranspose2d(o, o, 2f, stride=f, padding=f // 2, groups=o, bias=False)``, adds ``layers[i - 1]`` and
runs the sum through a second DeformConv.  ``fuse_ida_up(model)`` replaces the up-sampling and the add of every such
step with one kernel, which reads the low-resolution map and the skip once and writes the sum once: the up-sampled
map never reaches HBM.  The sum is written in the skip's layout.  Numeric contract: that of include/centernet_b200.h (fp32 FMA chain over
the valid taps, + skip in fp32, one rounding to the output dtype).

Opt-in and inference only: with grad enabled on an input or the weight, on CPU tensors, for dtypes other than fp32 /
bf16, for inputs of two dtypes, under autocast (unless it is bf16 and both inputs are bf16 already) and for shapes the
step does not fit, a step runs the original up-sampling and add; so does an f = 2 step with fewer than 2^21 output
elements, where the original step is the faster one (DESIGN §4.14).  dlav0's IDAUp (same attribute names, a different
forward) is left alone.
"""
import inspect

import torch
from torch import nn

from ._lib import C, dtype_code, ptr, require_cuda, stream_ptr
from .dcn_v2 import DCN

__all__ = ["ida_up_add", "fuse_ida_up", "is_ida_up"]

_FACTORS = (2, 4, 8)
# f = 2 steps with fewer output elements than this run the original step: measured on an H100 (DESIGN §4.14), every
# such dla_34 step at B = 1 is bound by host time, where cuDNN's conv + the add cost less than this module's call
_F2_MIN_OUT = 1 << 21


def _cl(t):
    return t.is_contiguous(memory_format=torch.channels_last) and not t.is_contiguous()


def _operand(t, cl):
    """t in the layout the kernel reads (NCHW, or channels_last when cl), 16-byte aligned."""
    fmt = torch.channels_last if cl else torch.contiguous_format
    t = t.contiguous(memory_format=fmt)
    if t.data_ptr() % 16:   # a view at an odd offset: the kernel's vector accesses need 16-byte alignment
        t = t.clone(memory_format=fmt)
    return t


def ida_up_add(p, weight, f, skip, channels_last=None):
    """conv_transpose2d(p, weight, stride=f, padding=f // 2, groups=C) + skip in one kernel, under the contract
    above.  p [B, C, Hp, Wp] and skip [B, C, f*Hp, f*Wp] share one dtype (fp32 or bf16); each is NCHW or
    channels_last.  weight [C, 1, 2f, 2f] is widened exactly to fp32.  The result has skip's dtype, and is
    channels_last when `channels_last` is True, NCHW when it is False and in skip's layout when it is None."""
    require_cuda(p, weight, skip, what="ida_up_add")
    if p.dtype not in (torch.float32, torch.bfloat16) or skip.dtype != p.dtype:
        raise TypeError("ida_up_add: p and skip must both be float32 or both bfloat16, got %s and %s"
                        % (p.dtype, skip.dtype))
    f = int(f)
    if p.dim() != 4:
        raise ValueError("ida_up_add: p must be [B, C, Hp, Wp], got %s" % (tuple(p.shape),))
    b, c, hp, wp = [int(v) for v in p.shape]
    if tuple(skip.shape) != (b, c, f * hp, f * wp):
        raise ValueError("ida_up_add: skip must be %s for p %s and f = %d, got %s"
                         % ((b, c, f * hp, f * wp), tuple(p.shape), f, tuple(skip.shape)))
    if tuple(weight.shape) != (c, 1, 2 * f, 2 * f):
        raise ValueError("ida_up_add: weight must be %s, got %s" % ((c, 1, 2 * f, 2 * f), tuple(weight.shape)))
    p_cl, skip_cl = _cl(p), _cl(skip)
    out_cl = skip_cl if channels_last is None else bool(channels_last)
    p, skip = _operand(p, p_cl), _operand(skip, skip_cl)
    w = weight.detach().float().contiguous()
    out = torch.empty(tuple(skip.shape), dtype=skip.dtype, device=skip.device,
                      memory_format=torch.channels_last if out_cl else torch.contiguous_format)
    C.ida_up_add(ptr(p), dtype_code(p), int(p_cl), ptr(w), f, ptr(skip), int(skip_cl), ptr(out), int(out_cl),
                 b, c, hp, wp, stream_ptr(p))
    return out


def _up_factor(up, o):
    """f when `up` is the depthwise up-sampling of an IDAUp step over o channels, else None."""
    if type(up) is not nn.ConvTranspose2d or up.bias is not None:
        return None
    f = up.stride[0]
    if f not in _FACTORS or up.stride != (f, f) or up.kernel_size != (2 * f, 2 * f) or \
            up.padding != (f // 2, f // 2) or up.output_padding != (0, 0) or up.dilation != (1, 1) or \
            up.padding_mode != "zeros":
        return None
    return f if up.in_channels == up.out_channels == up.groups == o else None


def _deform_conv(m):
    """The DCN of a pose_dla_dcn DeformConv-shaped module, else None."""
    conv = getattr(m, "conv", None)
    return conv if isinstance(m, nn.Module) and isinstance(conv, DCN) else None


def _steps(m):
    """The number of steps of a pose_dla_dcn IDAUp (proj_i, up_i, node_i for i = 1..n, consecutive), else 0."""
    n = 0
    while all(hasattr(m, "%s_%d" % (k, n + 1)) for k in ("proj", "up", "node")):
        n += 1
    if n == 0 or any(hasattr(m, "%s_%d" % (k, n + 1)) for k in ("proj", "up", "node")) or \
            any(hasattr(m, "%s_0" % k) for k in ("proj", "up", "node")):
        return 0
    for i in range(1, n + 1):
        proj, node = _deform_conv(getattr(m, "proj_%d" % i)), _deform_conv(getattr(m, "node_%d" % i))
        if proj is None or node is None:
            return 0
        o = node.in_channels
        if proj.out_channels != o or _up_factor(getattr(m, "up_%d" % i), o) is None:
            return 0
    return n


def is_ida_up(m):
    """True for a pose_dla_dcn IDAUp: a forward taking (layers, startp, endp) and consecutive proj_i / up_i / node_i,
    the projections and nodes DeformConv-shaped (`conv` is a DCN), every up a plain depthwise ConvTranspose2d of
    kernel 2f, stride f, padding f // 2 and no bias, f in {2, 4, 8}."""
    try:
        params = list(inspect.signature(m.forward).parameters)
    except (TypeError, ValueError):
        return False
    return params == ["layers", "startp", "endp"] and _steps(m) > 0


def _weight(up, dtype):
    """The up weight widened to fp32 as [C, 1, 2f, 2f] (under bf16 autocast rounded to bf16 first, as autocast's
    conv would), cached per weight version."""
    wt = up.weight
    key = (dtype, wt.device)
    hit = up.__dict__.get("_cnb_ida_w")
    if hit is not None and hit[0] is wt and hit[1] == wt._version and hit[2] == key:
        return hit[3]
    w = wt.detach()
    if dtype != w.dtype:
        w = w.to(dtype)
    w = w.float().contiguous()
    up.__dict__["_cnb_ida_w"] = (wt, wt._version, key, w)
    return w


def _fused_step(up, x, skip):
    """up(x) + skip through the kernel, or None where the original step runs (see the module docstring)."""
    wt = up.weight
    if torch.is_grad_enabled() and (x.requires_grad or skip.requires_grad or wt.requires_grad):
        return None
    if not isinstance(x, torch.Tensor) or not isinstance(skip, torch.Tensor):
        return None
    if not (x.is_cuda and skip.is_cuda and wt.is_cuda) or not (x.device == skip.device == wt.device):
        return None
    if x.dtype not in (torch.float32, torch.bfloat16) or skip.dtype != x.dtype:
        return None
    if torch.is_autocast_enabled("cuda"):
        if torch.get_autocast_dtype("cuda") != torch.bfloat16 or x.dtype != torch.bfloat16:
            return None   # autocast would hand back its own dtype; only bf16 inputs already match it
        wdt = torch.bfloat16
    elif wt.dtype != x.dtype:
        return None       # the original conv raises its dtype error
    else:
        wdt = wt.dtype
    f = up.stride[0]
    if x.dim() != 4 or skip.dim() != 4 or x.numel() == 0:
        return None
    b, c, hp, wp = [int(v) for v in x.shape]
    if c != up.in_channels or tuple(skip.shape) != (b, c, f * hp, f * wp):
        return None       # the original step raises its own error
    if f == 2 and b * c * hp * wp * 4 < _F2_MIN_OUT:
        return None
    # skip's layout in both dtypes: writing bf16 channels_last for the node's block kernel made the dla_34 chain
    # slower at B = 1 and 16 (DESIGN §4.14)
    return ida_up_add(x, _weight(up, wdt).view(c, 1, 2 * f, 2 * f), f, skip)


def _fused_forward(m):
    def forward(layers, startp, endp):
        for i in range(startp + 1, endp):
            j = i - startp
            up = getattr(m, "up_%d" % j)
            x = getattr(m, "proj_%d" % j)(layers[i])
            y = _fused_step(up, x, layers[i - 1])
            if y is None:
                y = up(x) + layers[i - 1]
            layers[i] = getattr(m, "node_%d" % j)(y)

    return forward


def fuse_ida_up(model):
    """Rewires every pose_dla_dcn IDAUp of `model` (is_ida_up) so that each step's up-sampling and skip add run in one
    kernel (ida_up_add), and returns the number of up layers covered (8 for dla_34: 6 in DLAUp, 2 in DLASeg.ida_up).
    The projections and nodes are still called as modules, so this composes with fuse_dcn_bn_relu, fuse_offset_conv
    and set_compute_dtype in any order; `layers` is updated in place exactly as before.  Only an instance `forward`
    is added: children, parameters and state-dict keys stay.  Calling it again does not wrap twice."""
    n = 0
    for m in model.modules():
        steps = m.__dict__.get("_cnb_ida_steps")
        if steps is None:
            if not is_ida_up(m):
                continue
            steps = _steps(m)
            m.forward = _fused_forward(m)
            m._cnb_ida_steps = steps
        n += steps
    return n

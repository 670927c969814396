"""Fused bf16 inference for the output heads (cnb_head_forward_bf16).

Every DLASeg / PoseResNet head is ``nn.Sequential(Conv2d(cin, head_conv, 3, padding=1), ReLU, Conv2d(head_conv, C, 1))``
(pose_dla_dcn.py:448-459, resnet_dcn.py:157-165, msra_resnet.py:135-143).  ``fuse_heads(model)`` turns each such head
into a ``FusedHead``, which runs the three layers in one kernel on bf16 wgmma at inference: the head_conv-channel
intermediate never reaches HBM.  The numeric contract is that of include/centernet_b200.h: input, W1 and W2 rounded
once to bf16, fp32 sums, ReLU and one bf16 rounding of the intermediate, output in the input's dtype.

Opt-in and inference only: with grad enabled on the input or any parameter, on CPU tensors, for dtypes other than
fp32 / bf16 and for shapes the kernel does not cover (cin or head_conv not a multiple of 32, head_conv > 256, C > 256)
a ``FusedHead`` runs the original Sequential.  Hourglass heads (``convolution`` + Conv2d) and single-conv heads
(head_conv = 0) are left alone.
"""
import torch
from torch import nn

from ._lib import C, dtype_code, f32c, ptr, require_cuda, stream_ptr, workspace

__all__ = ["FusedHead", "fuse_heads", "head_forward_bf16", "is_fusable_head"]


def is_fusable_head(m):
    """True for exactly Sequential(Conv2d 3x3 pad 1, ReLU, Conv2d 1x1), both convs plain (stride 1, no dilation or
    groups, zero padding) with a bias."""
    if not isinstance(m, nn.Sequential) or len(m) != 3:
        return False
    c1, act, c2 = m[0], m[1], m[2]
    if type(c1) is not nn.Conv2d or type(act) is not nn.ReLU or type(c2) is not nn.Conv2d:
        return False

    def plain(c, k, pad):
        return (c.kernel_size == (k, k) and c.stride == (1, 1) and c.padding == (pad, pad) and
                c.dilation == (1, 1) and c.groups == 1 and c.padding_mode == "zeros" and c.bias is not None)

    return plain(c1, 3, 1) and plain(c2, 1, 0) and c2.in_channels == c1.out_channels


def _supported(cin, cmid, cout):
    return C.head_w1t_bytes(cin, cmid) > 0 and C.head_w2t_bytes(cmid, cout) > 0


def _make_tiles(w1, w2):
    """bf16 weight tiles (w1t, w2t) of cnb_head_prepare_weights_bf16, from the fp32 upcast of w1 / w2 (exact for
    bf16 or fp16 parameters)."""
    cmid, cin = int(w1.shape[0]), int(w1.shape[1])
    cout = int(w2.shape[0])
    n1, n2 = C.head_w1t_bytes(cin, cmid), C.head_w2t_bytes(cmid, cout)
    buf = workspace(n1 + n2, w1.device)
    t1, t2 = buf[:n1], buf[n1:]
    a, b = f32c(w1), f32c(w2.reshape(cout, cmid))
    C.head_prepare_weights_bf16(ptr(a), ptr(b), cin, cmid, cout, ptr(t1), n1, ptr(t2), n2, stream_ptr(a))
    return t1, t2


def _tiles(head, w1, w2):
    """The head's weight tiles, rebuilt only when a weight changes: torch bumps `_version` on every in-place update
    (optimizer step, load_state_dict).  The cache holds the tensors themselves, so a replaced parameter is never
    mistaken for its predecessor."""
    hit = head.__dict__.get("_cnb_tiles")
    if hit is not None and hit[0] is w1 and hit[1] == w1._version and hit[2] is w2 and hit[3] == w2._version and \
            hit[4].device == w1.device:
        return hit[4], hit[5]
    t1, t2 = _make_tiles(w1, w2)
    head.__dict__["_cnb_tiles"] = (w1, w1._version, w2, w2._version, t1, t2)
    return t1, t2


def head_forward_bf16(x, w1, b1, w2, b2, tiles=None):
    """conv1x1(relu(conv3x3(x, w1, b1, padding=1)), w2, b2) under the bf16 contract above, in x's dtype (fp32 or
    bf16) and memory format (NCHW, or channels_last).  `tiles` are (w1t, w2t) from a FusedHead's cache; without them
    the weights are tiled for this call."""
    require_cuda(x, w1, b1, w2, b2, what="head_forward_bf16")
    if x.dtype not in (torch.float32, torch.bfloat16):
        raise TypeError("head_forward_bf16: the input must be float32 or bfloat16, got %s" % x.dtype)
    n, cin, h, w = [int(v) for v in x.shape]
    cmid, cout = int(w1.shape[0]), int(w2.shape[0])
    cl = x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous()
    fmt = torch.channels_last if cl else torch.contiguous_format
    x = x if cl else x.contiguous()
    if x.data_ptr() % 16:   # a view at an odd offset: the kernel's loads need 16-byte alignment
        x = x.clone(memory_format=fmt)
    if tiles is None:
        tiles = _make_tiles(w1, w2)
    out = torch.empty((n, cout, h, w), dtype=x.dtype, device=x.device, memory_format=fmt)
    ws = workspace(C.head_workspace_bytes(n, cin, h, w, dtype_code(x), int(cl)), x.device)
    bb1, bb2 = f32c(b1), f32c(b2)
    C.head_forward_bf16(ptr(x), dtype_code(x), int(cl), ptr(tiles[0]), ptr(bb1), ptr(tiles[1]), ptr(bb2), ptr(out),
                        n, cin, h, w, cmid, cout, ptr(ws), ws.numel(), stream_ptr(x))
    return out


class FusedHead(nn.Sequential):
    """A head Sequential whose inference runs in one fused bf16 kernel.  Same children, so the same state-dict keys
    (``hm.0.weight``, ``hm.2.bias``, ...); anything the kernel does not cover runs the original three layers."""

    def _fused_ok(self, x):
        c1, c2 = self[0], self[2]
        params = (c1.weight, c1.bias, c2.weight, c2.bias)
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
            return False
        if not x.is_cuda or x.dim() != 4 or any(not p.is_cuda or p.device != x.device for p in params):
            return False
        if x.dtype not in (torch.float32, torch.bfloat16) or x.numel() == 0:
            return False
        if torch.is_autocast_enabled("cuda") and (torch.get_autocast_dtype("cuda") != torch.bfloat16 or
                                                  x.dtype != torch.bfloat16):
            return False   # autocast would hand back its own dtype; only a bf16 input already matches it
        return int(x.shape[1]) == c1.in_channels and _supported(c1.in_channels, c1.out_channels, c2.out_channels)

    def forward(self, x):
        if not self._fused_ok(x):
            return super().forward(x)
        c1, c2 = self[0], self[2]
        return head_forward_bf16(x, c1.weight, c1.bias, c2.weight, c2.bias, tiles=_tiles(self, c1.weight, c2.weight))


def fuse_heads(model):
    """Turns every output head of `model` into a FusedHead in place and returns how many.  The heads are the modules
    a network registers under the names of its `heads` dict (DLASeg, PoseResNet: `self.__setattr__(head, fc)`) that
    are plain Sequentials of the head pattern (is_fusable_head); a Sequential of the same shape elsewhere in the
    network is left alone.  Only the module's class changes: children, parameters, hooks and state-dict keys stay, so a
    model-zoo checkpoint loads before or after fusing.  Composes with fuse_dcn_bn_relu and set_compute_dtype in any
    order."""
    n = 0
    for m in model.modules():
        heads = getattr(m, "heads", None)
        if not isinstance(heads, dict):
            continue
        for name in heads:
            fc = getattr(m, name, None) if isinstance(name, str) else None
            if type(fc) is nn.Sequential and is_fusable_head(fc):
                fc.__class__ = FusedHead
                n += 1
    return n

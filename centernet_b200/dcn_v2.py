"""Mirror of src/lib/models/networks/DCNv2/dcn_v2.py: DCNv2, DCN (+ DCNv2Pooling / DCNPooling
surface).  Parameter names (`weight`, `bias`, `conv_offset_mask.*`) match the reference so its
checkpoints load unchanged (SURVEY.md section 5)."""
import math

import torch
from torch import nn
from torch.nn.modules.utils import _pair

from .dcn_v2_func import (DCNv2Function, DCNv2PoolingFunction, _check_backward_dtype, _check_compute_dtype,
                          dcn_block_inference, dcn_fused_inference)


class DCNv2(nn.Module):
    """dcn_v2.py:14-41.  compute_dtype=torch.bfloat16 opts this module into the bf16 forward, and with it
    backward_dtype=torch.bfloat16 into the bf16 backward (DCNv2Function)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1,
                 compute_dtype=None, backward_dtype=None):
        super().__init__()
        self.compute_dtype = _check_compute_dtype(compute_dtype)
        self.backward_dtype = _check_backward_dtype(compute_dtype, backward_dtype)
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride = stride
        self.padding = padding
        self.dilation = dilation
        self.deformable_groups = deformable_groups
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels, *self.kernel_size))
        self.bias = nn.Parameter(torch.Tensor(out_channels))
        self.reset_parameters()

    def reset_parameters(self):   # dcn_v2.py:31-37
        n = self.in_channels
        for k in self.kernel_size:
            n *= k
        stdv = 1. / math.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)
        self.bias.data.zero_()

    def forward(self, input, offset, mask):
        func = DCNv2Function(self.stride, self.padding, self.dilation, self.deformable_groups,
                             getattr(self, "compute_dtype", None), getattr(self, "backward_dtype", None))
        return func(input, offset, mask, self.weight, self.bias)


class DCN(DCNv2):
    """dcn_v2.py:44-70: DCNv2 + the zero-initialised offset/mask conv."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1,
                 compute_dtype=None, backward_dtype=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, deformable_groups,
                         compute_dtype, backward_dtype)
        self.conv_offset_mask = nn.Conv2d(self.in_channels,
                                          self.deformable_groups * 3 * self.kernel_size[0] * self.kernel_size[1],
                                          kernel_size=self.kernel_size, stride=(self.stride, self.stride),
                                          padding=(self.padding, self.padding), bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()

    def forward(self, input):
        y = _block_forward(self, input)
        if y is not None:
            return y
        out = self.conv_offset_mask(input)
        # inference in fp32 uses the fused kernel; float64 (no fused form) takes the path below
        if input.is_cuda and not torch.is_grad_enabled() and self.kernel_size[0] * self.kernel_size[1] <= 9 and \
                input.dtype != torch.float64:
            # inference: chunk / cat / sigmoid (the three lines below) run inside the DCN kernel's sampler
            return dcn_fused_inference(input, out, self.weight, self.bias, self.stride, self.padding, self.dilation,
                                       self.deformable_groups,
                                       compute_dtype=getattr(self, "compute_dtype", None))
        o1, o2, mask = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        mask = torch.sigmoid(mask)
        func = DCNv2Function(self.stride, self.padding, self.dilation, self.deformable_groups,
                             getattr(self, "compute_dtype", None), getattr(self, "backward_dtype", None))
        return func(input, offset, mask, self.weight, self.bias)


class DCNv2Pooling(nn.Module):
    """dcn_v2.py:73-106."""

    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0):
        super().__init__()
        self.spatial_scale, self.pooled_size, self.output_dim, self.no_trans = spatial_scale, pooled_size, output_dim, no_trans
        self.group_size = group_size
        self.part_size = pooled_size if part_size is None else part_size
        self.sample_per_part, self.trans_std = sample_per_part, trans_std
        self.func = DCNv2PoolingFunction(spatial_scale, pooled_size, output_dim, no_trans, group_size, self.part_size,
                                         sample_per_part, trans_std)

    def forward(self, data, rois, offset):
        if self.no_trans:
            offset = data.new()
        return self.func(data, rois, offset)


class DCNPooling(DCNv2Pooling):
    """dcn_v2.py:108-171: the offsets and the modulation mask are predicted from a first, undeformed pooling
    pass (`offset_fc`, `mask_fc`, last layers zero-initialised; same submodule names for state dicts)."""

    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0, deform_fc_dim=1024):
        super().__init__(spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size, sample_per_part,
                         trans_std)
        self.deform_fc_dim = deform_fc_dim
        if not no_trans:
            self.func_offset = DCNv2PoolingFunction(spatial_scale, pooled_size, output_dim, True, group_size,
                                                    self.part_size, sample_per_part, trans_std)
            feat = pooled_size * pooled_size * output_dim
            self.offset_fc = nn.Sequential(
                nn.Linear(feat, deform_fc_dim), nn.ReLU(inplace=True),
                nn.Linear(deform_fc_dim, deform_fc_dim), nn.ReLU(inplace=True),
                nn.Linear(deform_fc_dim, pooled_size * pooled_size * 2))
            self.offset_fc[4].weight.data.zero_()
            self.offset_fc[4].bias.data.zero_()
            self.mask_fc = nn.Sequential(
                nn.Linear(feat, deform_fc_dim), nn.ReLU(inplace=True),
                nn.Linear(deform_fc_dim, pooled_size * pooled_size * 1), nn.Sigmoid())
            self.mask_fc[2].weight.data.zero_()
            self.mask_fc[2].bias.data.zero_()

    def forward(self, data, rois):
        if self.no_trans:
            return self.func(data, rois, data.new())
        n = rois.shape[0]
        x = self.func_offset(data, rois, data.new())
        offset = self.offset_fc(x.view(n, -1)).view(n, 2, self.pooled_size, self.pooled_size)
        mask = self.mask_fc(x.view(n, -1)).view(n, 1, self.pooled_size, self.pooled_size)
        return self.func(data, rois, offset) * mask


def _block_forward(dcn, x, bn_scale=None, bn_shift=None, relu=False):
    """The DCN block kernel for a module flagged by fuse_offset_conv, or None where the module runs its usual path:
    not flagged, compute_dtype not bf16, training, grad mode, autocast, not a CUDA float32 / bfloat16 input, or outside
    the kernel's range (dcn_block_inference)."""
    if not getattr(dcn, "offset_conv_fused", False) or getattr(dcn, "compute_dtype", None) != torch.bfloat16 or \
            dcn.training or torch.is_grad_enabled() or not x.is_cuda or torch.is_autocast_enabled("cuda"):
        return None
    om = dcn.conv_offset_mask
    return dcn_block_inference(x, om.weight, om.bias, dcn.weight, dcn.bias, dcn.stride, dcn.padding, dcn.dilation,
                               dcn.deformable_groups, bn_scale, bn_shift, relu)


def fuse_offset_conv(model):
    """Flags every DCN of `model` to run its conv_offset_mask inside the bf16 DCN kernel (cnb_dcnv2_forward_block_bf16)
    and returns how many it flagged.  A flagged DCN whose compute_dtype is torch.bfloat16 takes the block kernel in
    eval mode under no_grad on CUDA, inside the kernel's range, in DCN.forward and in the forward fuse_dcn_bn_relu
    installs; everything else runs as before.  The flag is read at call time, so this composes with set_compute_dtype
    and fuse_dcn_bn_relu in any order; it is a plain attribute, so state-dict keys do not change."""
    n = 0
    for m in model.modules():
        if isinstance(m, DCN):
            m.offset_conv_fused = True
            n += 1
    return n


# ------------------------------------------------------------------ N3: DCN + BatchNorm + ReLU (pose_dla_dcn.py:345-357)
def fold_bn(bn):
    """Inference BatchNorm as y = scale * x + shift (float64 fold, fp32 result)."""
    var = bn.running_var.double()
    scale = (bn.weight.double() if bn.affine else torch.ones_like(var)) / torch.sqrt(var + bn.eps)
    shift = (bn.bias.double() if bn.affine else torch.zeros_like(var)) - bn.running_mean.double() * scale
    return scale.float().contiguous(), shift.float().contiguous()


def fuse_dcn_bn_relu(model):
    """Rewires every `DeformConv`-shaped module of `model` (attributes `conv`: DCN and `actf`:
    Sequential(BatchNorm2d, ReLU), pose_dla_dcn.py:345-357) so that in eval mode under no_grad the BatchNorm and
    the ReLU run in the DCN kernel's epilogue (no extra passes over the activation).  Training / grad mode keeps
    the original three-module path.  Returns the number of modules fused."""
    n = 0
    for m in model.modules():
        conv, actf = getattr(m, "conv", None), getattr(m, "actf", None)
        if not (isinstance(conv, DCN) and isinstance(actf, nn.Sequential) and len(actf) == 2 and
                isinstance(actf[0], nn.BatchNorm2d) and isinstance(actf[1], nn.ReLU)):
            continue
        orig = m.forward

        def fused(x, _m=m, _orig=orig):
            c, bn = _m.conv, _m.actf[0]
            if _m.training or torch.is_grad_enabled() or not x.is_cuda or not bn.track_running_stats or \
                    x.dtype == torch.float64:
                return _orig(x)
            scale, shift = fold_bn(bn)
            y = _block_forward(c, x, scale, shift, True)
            if y is not None:
                return y
            om = c.conv_offset_mask(x)
            return dcn_fused_inference(x, om, c.weight, c.bias, c.stride, c.padding, c.dilation, c.deformable_groups,
                                       bn_scale=scale, bn_shift=shift, relu=True,
                                       compute_dtype=getattr(c, "compute_dtype", None))

        m.forward = fused
        n += 1
    return n


def set_compute_dtype(model, dtype, backward_dtype=None):
    """Sets `compute_dtype` and `backward_dtype` on every DCNv2 / DCN module of `model` (None: the default
    fp32-accurate forward; torch.bfloat16: the bf16 forward, and with backward_dtype=torch.bfloat16 the bf16 backward)
    and returns how many it set.  The reference network code builds DCN(...) without keywords; this turns the bf16
    path on for such a model without touching its code.  Composes with fuse_dcn_bn_relu in either order (the fused
    forward reads the attribute at call time)."""
    _check_compute_dtype(dtype)
    _check_backward_dtype(dtype, backward_dtype)
    n = 0
    for m in model.modules():
        if isinstance(m, DCNv2):
            m.compute_dtype = dtype
            m.backward_dtype = backward_dtype
            n += 1
    return n

"""GPU parity for DCNv2 forward / backward (A10-A12) through the DCNv2Function / DCN mirrors.
Forward <= 1e-4 abs vs the fp64 oracle (fp32-accurate mode, SURVEY.md section 8d); backward
compared with autograd through the fp64 oracle at the gradcheck tolerances of DCNv2/test.py:90,115."""
import numpy as np
import pytest
import torch

from oracle.dcn_ref import dcn_v2_forward

pytestmark = pytest.mark.gpu


def make(B, Ci, H, W, Co, dg, stride=1, seed=0, off_scale=2.0):
    g = torch.Generator().manual_seed(seed)
    Ho = (H + 2 - 3) // stride + 1
    Wo = (W + 2 - 3) // stride + 1
    x = torch.randn(B, Ci, H, W, generator=g)
    off = torch.randn(B, 18 * dg, Ho, Wo, generator=g) * off_scale
    m = torch.sigmoid(torch.randn(B, 9 * dg, Ho, Wo, generator=g))
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (3.0 * Ci ** 0.5)
    b = torch.randn(Co, generator=g)
    return x, off, m, w, b


def test_zero_offset_identity_kat():
    """DCNv2/test.py:32-65 (check_zero_offset) on the CUDA op."""
    from centernet_b200.dcn_v2 import DCNv2
    N, C, H, W = 2, 2, 4, 4
    torch.manual_seed(0)
    conv_offset = torch.zeros(N, 18, H, W, device="cuda")
    conv_mask = torch.full((N, 9, H, W), 0.5, device="cuda")
    dcn = DCNv2(C, C, (3, 3), stride=1, padding=1, dilation=1, deformable_groups=1).cuda()
    dcn.weight.data.zero_()
    dcn.bias.data.zero_()
    for i in range(C):
        dcn.weight.data[i, i, 1, 1] = 1.0
    x = torch.randn(N, C, H, W, device="cuda")
    out = dcn(x, conv_offset, conv_mask) * 2
    assert (out - x).abs().max().item() < 1e-6


def test_empty_output_grid_raises():
    """A 2x2 image under a 3x3 kernel without padding has no output pixel: the workspace queries return 0 for it and
    the call is refused, so DCNv2Function raises RuntimeError."""
    from centernet_b200.dcn_v2_func import DCNv2Function
    x = torch.randn(2, 64, 2, 2, device="cuda")
    off = torch.zeros(2, 18, 0, 0, device="cuda")
    m = torch.zeros(2, 9, 0, 0, device="cuda")
    w = torch.randn(64, 64, 3, 3, device="cuda")
    with pytest.raises(RuntimeError):
        DCNv2Function(1, 0, 1, 1)(x, off, m, w, torch.zeros(64, device="cuda"))


SHAPES = [
    # B, Cin, H, W, Cout, dg, stride
    (2, 64, 32, 32, 64, 1, 1),     # dla_34 style 64->64
    (1, 128, 16, 16, 128, 1, 1),   # Cout > 64 -> two accumulator sets
    (2, 12, 9, 11, 5, 2, 1),       # odd sizes, 2 deformable groups, partial channel chunk
    (2, 6, 10, 14, 7, 1, 2),       # stride 2
    (1, 256, 8, 8, 64, 1, 1),      # deep reduction
]


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", SHAPES)
def test_forward_vs_oracle(B, Ci, H, W, Co, dg, stride):
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = make(B, Ci, H, W, Co, dg, stride)
    want = dcn_v2_forward(x, off, m, w, b, stride, 1, 1, dg)
    got = DCNv2Function(stride, 1, 1, dg)(x.cuda(), off.cuda(), m.cuda(), w.cuda(), b.cuda())
    assert got.shape == want.shape
    err = (got.double().cpu() - want).abs().max().item()
    assert err <= 1e-4, err


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", [(2, 16, 12, 12, 8, 1, 1), (1, 12, 9, 11, 5, 2, 1), (2, 6, 10, 14, 7, 1, 2),
                                                    (1, 64, 16, 16, 64, 1, 1)])
def test_backward_vs_oracle_autograd(B, Ci, H, W, Co, dg, stride):
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = make(B, Ci, H, W, Co, dg, stride, seed=3, off_scale=1.3)
    leaves = [t.clone().double().requires_grad_(True) for t in (x, off, m, w, b)]
    out = dcn_v2_forward(*leaves, stride, 1, 1, dg)
    go = torch.randn(out.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    (out * go).sum().backward()
    cl = [t.clone().cuda().requires_grad_(True) for t in (x, off, m, w, b)]
    got = DCNv2Function(stride, 1, 1, dg)(*cl)
    (got * go.float().cuda()).sum().backward()
    for name, a, r in zip(("input", "offset", "mask", "weight", "bias"), cl, leaves):
        ref = r.grad
        err = (a.grad.double().cpu() - ref).abs().max().item()
        scale = max(1.0, ref.abs().max().item())
        assert err <= 1e-3 * scale, (name, err, scale)      # fp32 gradcheck tolerance of test.py:115 (atol 1e-3)


def _raw_backward(x, off, m, w, go, stride, dg, tensor_cores, pad=1, dil=1):
    from centernet_b200._lib import C, ptr, stream_ptr, workspace
    B, Ci, H, W = x.shape
    Co, _, kh, kw = w.shape
    grads = [torch.zeros_like(x), torch.zeros_like(off), torch.zeros_like(m), torch.zeros_like(w),
             torch.zeros(Co, device=x.device)]
    ws, wsb, keep = 0, 0, None
    if tensor_cores:
        wsb = C.dcnv2_backward_workspace_bytes(B, Ci, Co, H, W, kh, kw, stride, pad, dil, dg)
        assert wsb > 0
        keep = workspace(wsb, x.device)
        ws = ptr(keep)
    C.dcnv2_backward(ptr(x), ptr(off), ptr(m), ptr(w), ptr(go), *[ptr(g) for g in grads], B, Ci, H, W, Co, kh, kw,
                     stride, stride, pad, pad, dil, dil, dg, ws, wsb, stream_ptr(x))
    torch.cuda.synchronize()
    return grads


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", [(2, 64, 40, 48, 64, 1, 1), (3, 96, 17, 23, 40, 1, 1), (2, 128, 16, 16, 272, 1, 1),
                                                    (2, 64, 16, 24, 64, 2, 1), (2, 40, 19, 21, 24, 1, 2)])
def test_backward_tensor_core_vs_fp32_path(B, Ci, H, W, Co, dg, stride):
    """cnb_dcnv2_backward with the workspace (wgmma, 3xTF32) against the same call without it (fp32 CUDA cores) on
    shapes the reference-pinned cases do not reach: ragged tiles, channel blocks with padding, Cout > 256 (dW falls
    back to fp32), two deformable groups, stride 2; and the deterministic part of the tensor-core path repeats."""
    x, off, m, w, _ = [t.cuda() for t in make(B, Ci, H, W, Co, dg, stride, seed=11, off_scale=1.5)]
    Ho = (H + 2 - 3) // stride + 1; Wo = (W + 2 - 3) // stride + 1
    go = torch.randn(B, Co, Ho, Wo, generator=torch.Generator().manual_seed(5)).cuda()
    a = _raw_backward(x, off, m, w, go, stride, dg, True)
    a2 = _raw_backward(x, off, m, w, go, stride, dg, True)
    r = _raw_backward(x, off, m, w, go, stride, dg, False)
    for name, u, v in zip(("input", "offset", "mask", "weight", "bias"), a, r):
        scale = max(1.0, v.abs().max().item())
        assert (u - v).abs().max().item() <= 2e-4 * scale, (name, (u - v).abs().max().item(), scale)
    for name, u, v in zip(("offset", "mask", "weight", "bias"), a[1:], a2[1:]):
        if name == "weight" and Co > 256:
            continue      # fp32 fallback: atomics
        assert torch.equal(u, v), name + " not bit-identical run to run"


@pytest.mark.parametrize("B,Ci,H,W,Co,dg", [(2, 64, 40, 48, 64, 1), (2, 96, 17, 23, 40, 1), (1, 64, 16, 24, 32, 2), (2, 160, 12, 12, 24, 1)])
def test_backward_deterministic_mode(B, Ci, H, W, Co, dg):
    """cnb_dcnv2_set_deterministic(1): grad_input through the fixed-order gather.  Offsets within +-1.9 pixels keep every
    sample in the gather window, so ALL five gradients repeat bit for bit; with free offsets the far samples take the
    atomic path and the result still matches the fp32 path."""
    from centernet_b200._lib import C
    x, off, m, w, _ = [t.cuda() for t in make(B, Ci, H, W, Co, dg, 1, seed=13, off_scale=1.5)]
    go = torch.randn(B, Co, H, W, generator=torch.Generator().manual_seed(6)).cuda()
    r = _raw_backward(x, off, m, w, go, 1, dg, False)
    try:
        C.dcnv2_set_deterministic(1)
        assert C.dcnv2_get_deterministic() == 1
        a = _raw_backward(x, off, m, w, go, 1, dg, True)
        offc = off.clamp(-1.9, 1.9)
        d1 = _raw_backward(x, offc, m, w, go, 1, dg, True)
        d2 = _raw_backward(x, offc, m, w, go, 1, dg, True)
    finally:
        C.dcnv2_set_deterministic(0)
    rc = _raw_backward(x, offc, m, w, go, 1, dg, False)
    for name, u, v in zip(("input", "offset", "mask", "weight", "bias"), a, r):
        scale = max(1.0, v.abs().max().item())
        assert (u - v).abs().max().item() <= 2e-4 * scale, (name, (u - v).abs().max().item(), scale)
    for name, u, v in zip(("input", "offset", "mask", "weight", "bias"), d1, rc):
        scale = max(1.0, v.abs().max().item())
        assert (u - v).abs().max().item() <= 2e-4 * scale, ("clamped", name, (u - v).abs().max().item(), scale)
    for name, u, v in zip(("input", "offset", "mask", "weight", "bias"), d1, d2):
        assert torch.equal(u, v), name + " not bit-identical run to run in deterministic mode"


@pytest.mark.parametrize("kh,kw,pad,dil,stride", [(1, 3, 1, 1, 1), (3, 3, 2, 2, 1), (1, 1, 0, 1, 1), (3, 2, 1, 1, 2)])
def test_backward_tensor_core_other_kernels(kh, kw, pad, dil, stride):
    """Fewer than 9 taps (zero weight tiles for the missing ones), dilation 2, 1x1: tensor-core backward vs the fp32 path."""
    B, Ci, H, W, Co, dg = 2, 64, 20, 26, 48, 1
    gen = torch.Generator().manual_seed(31)
    Ho = (H + 2 * pad - (dil * (kh - 1) + 1)) // stride + 1
    Wo = (W + 2 * pad - (dil * (kw - 1) + 1)) // stride + 1
    kt = kh * kw
    x = torch.randn(B, Ci, H, W, generator=gen).cuda()
    off = (torch.randn(B, 2 * kt * dg, Ho, Wo, generator=gen) * 1.5).cuda()
    m = torch.sigmoid(torch.randn(B, kt * dg, Ho, Wo, generator=gen)).cuda()
    w = (torch.randn(Co, Ci, kh, kw, generator=gen) / (Ci * kt) ** 0.5).cuda()
    go = torch.randn(B, Co, Ho, Wo, generator=gen).cuda()
    a = _raw_backward(x, off, m, w, go, stride, dg, True, pad, dil)
    r = _raw_backward(x, off, m, w, go, stride, dg, False, pad, dil)
    for name, u, v in zip(("input", "offset", "mask", "weight", "bias"), a, r):
        scale = max(1.0, v.abs().max().item())
        assert (u - v).abs().max().item() <= 2e-4 * scale, (name, (u - v).abs().max().item(), scale)


def test_backward_batch_chunks():
    """The column gradient is held to ~1.5 GiB: 33 images of 64@128x128 (42 MB of dcol each) run as two passes of 30 + 3
    images.  The chunked tensor-core backward must equal the fp32 path image by image (first, boundary and last ones)."""
    B, Ci, H, W, Co = 33, 64, 128, 128, 64
    g = torch.Generator(device="cuda").manual_seed(23)
    x = torch.randn(B, Ci, H, W, device="cuda", generator=g)
    off = torch.randn(B, 18, H, W, device="cuda", generator=g) * 1.5
    m = torch.sigmoid(torch.randn(B, 9, H, W, device="cuda", generator=g))
    w = torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) / (3.0 * Ci ** 0.5)
    go = torch.randn(B, Co, H, W, device="cuda", generator=g)
    a = _raw_backward(x, off, m, w, go, 1, 1, True)
    r = _raw_backward(x, off, m, w, go, 1, 1, False)
    for name, u, v in zip(("input", "offset", "mask"), a[:3], r[:3]):
        for img in (0, 29, 30, 32):
            scale = max(1.0, v[img].abs().max().item())
            assert (u[img] - v[img]).abs().max().item() <= 2e-4 * scale, (name, img)
    for name, u, v in zip(("weight", "bias"), a[3:], r[3:]):
        scale = max(1.0, v.abs().max().item())
        assert (u - v).abs().max().item() <= 5e-4 * scale, (name, (u - v).abs().max().item(), scale)


@pytest.mark.parametrize("B,Ci,H,W,Co", [(2, 64, 24, 40, 64), (2, 128, 17, 19, 96)])
def test_backward_channels_last(B, Ci, H, W, Co):
    """A channels_last activation goes through forward (sampled in place) and backward (cnb_dcnv2_backward_ex: input and
    grad_input channels-last, no layout passes); results equal the NCHW path, grad_input comes back channels_last."""
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = [t.cuda() for t in make(B, Ci, H, W, Co, 1, 1, seed=17, off_scale=1.5)]
    go = torch.randn(B, Co, H, W, generator=torch.Generator().manual_seed(8)).cuda()
    ref = [t.clone().requires_grad_(True) for t in (x, off, m, w, b)]
    out_ref = DCNv2Function(1, 1, 1, 1)(*ref)
    (out_ref * go).sum().backward()
    cl = [x.clone().contiguous(memory_format=torch.channels_last).requires_grad_(True)] + \
        [t.clone().requires_grad_(True) for t in (off, m, w, b)]
    out = DCNv2Function(1, 1, 1, 1)(*cl)
    (out * go).sum().backward()
    assert (out - out_ref).abs().max().item() <= 1e-5
    assert cl[0].grad.is_contiguous(memory_format=torch.channels_last)
    for name, u, v in zip(("input", "offset", "mask", "weight", "bias"), cl, ref):
        scale = max(1.0, v.grad.abs().max().item())
        assert (u.grad - v.grad).abs().max().item() <= 1e-4 * scale, (name, (u.grad - v.grad).abs().max().item())


def test_dcn_module_and_state_dict_names():
    from centernet_b200.dcn_v2 import DCN
    dcn = DCN(16, 8, kernel_size=(3, 3), stride=1, padding=1, deformable_groups=1).cuda()
    assert sorted(dcn.state_dict().keys()) == ["bias", "conv_offset_mask.bias", "conv_offset_mask.weight", "weight"]
    x = torch.randn(2, 16, 20, 20, device="cuda", requires_grad=True)
    y = dcn(x)
    # zero-initialised offset conv: offsets 0, mask 0.5 -> equals 0.5 * conv2d(x, weight) + bias
    ref = 0.5 * torch.nn.functional.conv2d(x, dcn.weight, None, 1, 1) + dcn.bias.view(1, -1, 1, 1)
    assert (y - ref).abs().max().item() < 1e-4
    y.sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()
    assert dcn.weight.grad is not None and dcn.conv_offset_mask.weight.grad is not None
    with pytest.raises(NotImplementedError):
        dcn.cpu()(torch.randn(1, 16, 8, 8))


def test_fused_inference_paths():
    """N3: conv_offset_mask glue (chunk / cat / sigmoid) fused into the sampler, BatchNorm + ReLU into the epilogue;
    channels_last activations sampled in place; cached weight tiles follow in-place weight updates."""
    from centernet_b200.dcn_v2 import DCN, fuse_dcn_bn_relu
    from torch import nn
    torch.manual_seed(0)

    class DeformConv(nn.Module):          # shape of pose_dla_dcn.py:345-357
        def __init__(self, chi, cho):
            super().__init__()
            self.actf = nn.Sequential(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))
            self.conv = DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)

        def forward(self, x):
            return self.actf(self.conv(x))

    # conv_offset_mask runs on cuDNN: keep it fp32 so that the NCHW and channels_last inputs get the same offsets
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        _fused_inference_cases(DeformConv, fuse_dcn_bn_relu)


def _fused_inference_cases(DeformConv, fuse_dcn_bn_relu):
    for chi, cho, hw in ((64, 64, 40), (128, 256, 16), (24, 40, 9)):
        m = DeformConv(chi, cho).cuda()
        m.conv.conv_offset_mask.weight.data.normal_(0, 0.02); m.conv.conv_offset_mask.bias.data.normal_(0, 0.5)
        m.actf[0].running_mean.normal_(0, 0.3); m.actf[0].running_var.uniform_(0.5, 2.0)
        m.actf[0].weight.data.uniform_(0.5, 1.5); m.actf[0].bias.data.normal_(0, 0.2)
        m.eval()
        x = torch.randn(2, chi, hw, hw, device="cuda")
        with torch.enable_grad():
            want_dcn = m.conv(x)                       # unfused three-op path (grad mode)
            want = m.actf(want_dcn.clone())
        with torch.no_grad():
            got_dcn = m.conv(x)                        # fused prologue
            assert (got_dcn - want_dcn).abs().max().item() <= 1e-4
            assert fuse_dcn_bn_relu(m) == 1
            got = m(x)
            assert (got - want).abs().max().item() <= 2e-4
            if chi % 32 == 0:
                xcl = x.contiguous(memory_format=torch.channels_last)
                assert (m(xcl) - want).abs().max().item() <= 2e-4
            # in-place weight update must invalidate the cached tiles
            m.conv.weight.data.mul_(0.5)
            with torch.enable_grad():
                want2 = m.actf(m.conv(x))
            assert (m(x) - want2).abs().max().item() <= 2e-4

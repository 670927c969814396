"""GPU: the opt-in bf16 DCNv2 forward (compute_dtype=torch.bfloat16).

1. On inputs where every step is exact (x on a 1/8 grid, half-integer offsets, mask in {1/4, 1/2, 1}, W on a 1/64
   grid, bias on a 2^-13 grid, Cin <= 256): every column value has at most 7 significant bits (exact in bf16), every
   product lies on a 2^-13 grid and every partial sum stays below 2^9 (exact in fp32).  So the fp32 output must
   EQUAL the fp64 oracle and the bf16 output its RN rounding.
2. Random data against a derived bound: |y - y64| <= 2^-7 S + 2^-8 |y64| + 1e-5, S = the oracle on |x_b|, |W_b|.
3. Layouts and dtypes: fp32 in == bf16 in, channels_last == NCHW, output dtype, bit-identical repeats.
4. Autograd: the fp32 backward at the upcast operands, bit for bit.
5. Modules: DCN, fuse_dcn_bn_relu + set_compute_dtype, weight-tile invalidation, the unchanged default."""
import pytest
import torch

from oracle.dcn_ref import dcn_v2_forward
from test_dcn_gpu import make

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _out_hw(H, W, kh, kw, stride, pad, dil):
    return (H + 2 * pad - (dil * (kh - 1) + 1)) // stride + 1, (W + 2 * pad - (dil * (kw - 1) + 1)) // stride + 1


def exact_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil, seed=0):
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = _out_hw(H, W, kh, kw, stride, pad, dil)
    kt = kh * kw
    x = torch.randint(-8, 9, (B, Ci, H, W), generator=g).float() / 8                # 1/8 grid in [-1, 1]
    off = torch.randint(-7, 8, (B, 2 * kt * dg, Ho, Wo), generator=g).float() / 2   # integer / half-integer, +-3.5 px
    m = torch.tensor([0.25, 0.5, 1.0])[torch.randint(0, 3, (B, kt * dg, Ho, Wo), generator=g)]
    w = torch.randint(-8, 9, (Co, Ci, kh, kw), generator=g).float() / 64            # 1/64 grid in [-1/8, 1/8]
    b = torch.randint(-1024, 1025, (Co,), generator=g).float() / 8192               # 2^-13 grid
    return x, off, m, w, b


EXACT = [
    # B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil
    (2, 64, 20, 24, 64, 1, 3, 3, 1, 1, 1),
    (2, 80, 17, 19, 40, 2, 3, 3, 1, 1, 1),      # 40 channels a group: ragged blocks (pad slots), two groups
    (2, 64, 21, 23, 72, 2, 3, 3, 2, 1, 1),      # stride 2, two groups of 32, one Cout tile of 128
    (1, 32, 18, 18, 32, 1, 3, 3, 1, 2, 2),      # dilation 2
    (2, 64, 16, 16, 48, 1, 1, 1, 1, 0, 1),      # 1x1
    (2, 64, 16, 20, 64, 1, 1, 3, 1, 1, 1),      # 1x3
    (1, 256, 8, 8, 272, 1, 3, 3, 1, 1, 1),      # small map: split-K partials; Cout 272 = three Cout tiles
]


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil", EXACT)
def test_exact_grid_bit_exact(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    from centernet_b200.dcn_v2_func import DCNv2Function, dcn_fused_inference
    x, off, m, w, b = exact_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil)
    want = dcn_v2_forward(x, off, m, w, b, stride, pad, dil, dg)
    want32 = want.float()
    assert torch.equal(want32.double(), want)          # the grid makes the fp64 answer exact in fp32
    xc, offc, mc, wc, bc = [t.cuda() for t in (x, off, m, w, b)]
    f = DCNv2Function(stride, pad, dil, dg, compute_dtype=BF)
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        y = f(xin, offc, mc, wc, bc)
        assert y.dtype == torch.float32 and y.is_contiguous()
        assert torch.equal(y.cpu(), want32)
        y16 = f(xin.to(BF), offc, mc, wc, bc)
        assert y16.dtype == BF
        assert torch.equal(y16.cpu(), want32.to(BF))

    # fused: raw conv_offset_mask output (mask logits 0 / 100 -> sigmoid exactly 1/2 / 1) + BN (scale in {1/2, 1, 2},
    # shift on the 2^-13 grid) + ReLU; every step stays exact
    g = torch.Generator().manual_seed(1)
    m2 = torch.where(m == 1.0, 1.0, 0.5)
    om = torch.cat([off, torch.where(m2 == 1.0, 100.0, 0.0)], dim=1)
    sc = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (Co,), generator=g)]
    sh = torch.randint(-1024, 1025, (Co,), generator=g).float() / 8192
    want_f = torch.relu(dcn_v2_forward(x, off, m2, w, b, stride, pad, dil, dg) * sc.double().view(1, -1, 1, 1) +
                        sh.double().view(1, -1, 1, 1))
    want_f32 = want_f.float()
    assert torch.equal(want_f32.double(), want_f)
    omc, scc, shc = om.cuda(), sc.cuda(), sh.cuda()
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        y = dcn_fused_inference(xin, omc, wc, bc, stride, pad, dil, dg, bn_scale=scc, bn_shift=shc, relu=True,
                                compute_dtype=BF)
        assert y.dtype == torch.float32
        assert torch.equal(y.cpu(), want_f32)
        y16 = dcn_fused_inference(xin.to(BF), omc, wc, bc, stride, pad, dil, dg, bn_scale=scc, bn_shift=shc,
                                  relu=True, compute_dtype=BF)
        assert y16.dtype == BF
        assert torch.equal(y16.cpu(), want_f32.to(BF))


DLA34 = [(512, 16, 256), (256, 32, 256), (256, 32, 128), (128, 64, 128), (128, 64, 64), (64, 128, 64), (256, 32, 64)]


@pytest.mark.parametrize("Ci,HW,Co", DLA34)
def test_random_within_bound(Ci, HW, Co):
    """Two bf16 roundings of <= 2^-9 each (column value, weight) and the fp32 accumulate, with a 2x margin; the bf16
    output adds one more rounding of <= 2^-9 |y|.  y64 is the fp64 oracle at the bf16 activation."""
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = make(2, Ci, HW, HW, Co, 1, seed=21)
    xb = x.to(BF).float()
    wb = w.to(BF).float()
    y64 = dcn_v2_forward(xb, off, m, w, b)
    S = dcn_v2_forward(xb.abs(), off, m, wb.abs(), None)
    bound = 2.0 ** -7 * S + 2.0 ** -8 * y64.abs() + 1e-5
    f = DCNv2Function(1, 1, 1, 1, compute_dtype=BF)
    offc, mc, wc, bc = off.cuda(), m.cuda(), w.cuda(), b.cuda()
    x16 = x.to(BF).cuda().contiguous(memory_format=torch.channels_last)
    for y in (f(x16, offc, mc, wc, bc), f(x.cuda(), offc, mc, wc, bc)):
        err = (y.double().cpu() - y64).abs()
        assert (err <= bound).all(), ((err - bound).max().item(), err.max().item())
    # and it is a bf16 result: the fp32-accurate default is far closer
    y32 = DCNv2Function(1, 1, 1, 1)(x.cuda(), offc, mc, wc, bc)
    assert (y32.double().cpu() - dcn_v2_forward(x, off, m, w, b)).abs().max().item() <= 1e-4


@pytest.mark.parametrize("B,Ci,H,W,Co,dg", [(2, 64, 40, 48, 64, 1), (2, 128, 16, 16, 272, 1), (3, 96, 17, 23, 40, 2),
                                             (1, 256, 8, 8, 64, 1)])
def test_layouts_dtypes_and_repeats(B, Ci, H, W, Co, dg):
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = [t.cuda() for t in make(B, Ci, H, W, Co, dg, seed=5)]
    f = DCNv2Function(1, 1, 1, dg, compute_dtype=BF)
    y32 = f(x, off, m, w, b)
    y16 = f(x.to(BF), off, m, w, b)
    assert y32.dtype == torch.float32 and y16.dtype == BF
    assert torch.equal(y32.to(BF), y16)                      # fp32 in == its bf16 rounding in
    cl = x.contiguous(memory_format=torch.channels_last)
    assert torch.equal(f(cl, off, m, w, b), y32)             # fp32 channels_last (rounded by the flat pass)
    assert torch.equal(f(cl.to(BF), off, m, w, b), y16)      # bf16 channels_last (sampled in place when whole blocks)
    assert torch.equal(f(x.to(BF), off, m, w, b), y16)       # repeats bit for bit
    assert torch.equal(f(x, off.to(BF).float(), m, w, b), f(x, off.to(BF), m, w, b))   # bf16 offsets are upcast
    assert torch.equal(f(x, off, m, w.to(BF), b.to(BF)), f(x, off, m, w.to(BF).float(), b.to(BF).float()))


def _grads(fn, leaves, go):
    leaves = [t.detach().clone().requires_grad_(True) for t in leaves]
    y = fn(*leaves)
    y.backward(go.to(y.dtype))
    return y, [t.grad for t in leaves]


@pytest.mark.parametrize("x_dtype,wb_dtype", [(BF, torch.float32), (torch.float32, torch.float32), (BF, BF)])
def test_autograd_matches_fp32_backward_at_upcast_operands(x_dtype, wb_dtype):
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = [t.cuda() for t in make(2, 64, 24, 20, 96, 1, seed=3, off_scale=1.3)]
    x, w, b = x.to(x_dtype), w.to(wb_dtype), b.to(wb_dtype)
    go = torch.randn(2, 96, 24, 20, generator=torch.Generator().manual_seed(9)).cuda()
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            y, g = _grads(DCNv2Function(1, 1, 1, 1, compute_dtype=BF), (x, off, m, w, b), go)
            # the default fp32 path at the operands the bf16 forward used: bf16 activation and weight, upcast
            _, r = _grads(DCNv2Function(1, 1, 1, 1), (x.to(BF).float(), off, m, w.to(BF).float(), b.float()),
                          go.to(y.dtype).float())
        finally:
            torch.use_deterministic_algorithms(False)
        assert y.dtype == x_dtype
        for name, a, ref, leaf in zip(("input", "offset", "mask", "weight", "bias"), g, r, (x, off, m, w, b)):
            assert a.dtype == leaf.dtype, name
            if name == "input" and not det:       # default mode scatters grad_input with float atomics
                assert (a.float() - ref).abs().max().item() <= 1e-2 * max(1.0, ref.abs().max().item()), name
            else:
                assert torch.equal(a, ref.to(leaf.dtype)), name


def _deform_conv(chi, cho):
    from torch import nn
    from centernet_b200.dcn_v2 import DCN

    class DeformConv(nn.Module):          # shape of pose_dla_dcn.py:345-357
        def __init__(self):
            super().__init__()
            self.actf = nn.Sequential(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))
            self.conv = DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)

        def forward(self, x):
            return self.actf(self.conv(x))

    m = DeformConv().cuda()
    m.conv.conv_offset_mask.weight.data.normal_(0, 0.02)
    m.conv.conv_offset_mask.bias.data.normal_(0, 0.5)
    m.actf[0].running_mean.normal_(0, 0.3)
    m.actf[0].running_var.uniform_(0.5, 2.0)
    m.actf[0].weight.data.uniform_(0.5, 1.5)
    m.actf[0].bias.data.normal_(0, 0.2)
    return m.eval()


def _close(a, b, rel=1e-2):
    return (a.float() - b.float()).abs().max().item() <= rel * max(1.0, b.float().abs().max().item())


def test_modules():
    from centernet_b200.dcn_v2 import DCN, DCNv2, fuse_dcn_bn_relu, set_compute_dtype
    from centernet_b200.dcn_v2_func import DCNv2Function
    torch.manual_seed(0)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        # DCN(compute_dtype=bf16): grad mode (DCNv2Function) and no_grad (fused kernel) agree
        dcn = DCN(64, 64, 3, 1, 1, compute_dtype=BF).cuda()
        dcn.conv_offset_mask.weight.data.normal_(0, 0.02)
        dcn.conv_offset_mask.bias.data.normal_(0, 0.5)
        x = torch.randn(2, 64, 24, 24, device="cuda")
        y_grad = dcn(x)
        with torch.no_grad():
            y_inf = dcn(x)
        assert y_grad.dtype == y_inf.dtype == torch.float32
        assert _close(y_inf, y_grad)
        y_grad.sum().backward()
        assert dcn.weight.grad is not None and dcn.conv_offset_mask.weight.grad is not None
        dcn16 = DCN(64, 64, 3, 1, 1, compute_dtype=BF).cuda().to(BF)       # a bf16 model
        dcn16.load_state_dict(dcn.state_dict())
        with torch.no_grad():
            y16 = dcn16(x.to(BF))
        assert y16.dtype == BF and _close(y16, y_inf, 3e-2)             # its offset conv runs in bf16 too

        # fuse_dcn_bn_relu + set_compute_dtype compose, in either order
        for fuse_first in (True, False):
            m = _deform_conv(64, 64)
            x = torch.randn(2, 64, 20, 20, device="cuda")
            with torch.no_grad():
                want32 = m(x)
            if fuse_first:
                assert fuse_dcn_bn_relu(m) == 1
            assert set_compute_dtype(m, BF) == 1
            if not fuse_first:
                assert fuse_dcn_bn_relu(m) == 1
            with torch.enable_grad():
                want = m.actf(m.conv(x))                               # unfused, bf16 forward
            with torch.no_grad():
                got = m(x)                                             # fused, bf16 forward
                got_cl = m(x.contiguous(memory_format=torch.channels_last))
            assert got.dtype == torch.float32
            assert _close(got, want, 2e-3) and _close(got, want32)
            assert not torch.equal(got, want32)                        # the flag took effect
            assert torch.equal(got_cl, got)

        # an in-place weight update invalidates the cached bf16 tiles (and leaves the TF32 tiles apart)
        x, off, mk, w, b = [t.cuda() for t in make(2, 64, 16, 16, 64, 1, seed=7)]
        f16, f32 = DCNv2Function(1, 1, compute_dtype=BF), DCNv2Function(1, 1)
        y16a, y32a = f16(x, off, mk, w, b), f32(x, off, mk, w, b)
        w.mul_(0.5)
        y16b, y32b = f16(x, off, mk, w, b), f32(x, off, mk, w, b)
        w2 = w.clone()                                                 # a new tensor: freshly built tiles
        assert torch.equal(y16b, f16(x, off, mk, w2, b)) and torch.equal(y32b, f32(x, off, mk, w2, b))
        assert not torch.equal(y16a, y16b) and not torch.equal(y32a, y32b)

        # a module without the flag still computes a bf16 input in fp32 and returns fp32
        plain = DCNv2(64, 64, 3, 1, 1).cuda()
        xb = x.to(BF)
        y = plain(xb, off, mk)
        assert y.dtype == torch.float32
        assert torch.equal(y, plain(xb.float(), off, mk))

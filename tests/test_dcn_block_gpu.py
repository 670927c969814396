"""The DCN block kernel (cnb_dcnv2_forward_block_bf16) on the GPU: conv_offset_mask, sigmoid, deformable sampling, bf16
contraction and the folded BN + ReLU in one kernel.

Exact grids: x on the 1/8 grid, W_om sparse with entries 4 (offset rows) and 800 (mask rows), b_om on the 1/2 grid,
so om = conv(x, W_om) + b_om is exact in fp32 in any summation order; the offsets are multiples of 1/2 that vary per
pixel (and reach over the image edge), and the mask logits are 0 or 100 (sigmoid exactly 1/2 or 1).  On them the block
equals dcn_fused_inference fed the exact om, and the fp64 oracle, bit for bit."""
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from oracle.dcn_ref import dcn_v2_forward
from test_bf16_gpu import exact_inputs

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def exact_om_weights(Ci, seed=0):
    """W_om [27][Ci][3][3]: every offset row holds one 4 at a random (channel, tap), every mask row one 800 at the
    centre tap of channel 0 (whose x is 0 or 1/8, so the logit is 0 or 100); b_om on the 1/2 grid in [-2, 2]."""
    g = torch.Generator().manual_seed(seed)
    w = torch.zeros(27, Ci, 3, 3)
    for c in range(18):
        ci, t = int(torch.randint(0, Ci, (1,), generator=g)), int(torch.randint(0, 9, (1,), generator=g))
        w[c, ci, t // 3, t % 3] = 4.0
    w[18:, 0, 1, 1] = 800.0
    b = torch.randint(-4, 5, (27,), generator=g).float() / 2
    b[18:] = 0.0
    return w, b


def exact_case(B, Ci, H, W, Co, seed=0):
    x, _, _, w, b = exact_inputs(B, Ci, H, W, Co, 1, 3, 3, 1, 1, 1, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    x[:, 0] = torch.randint(0, 2, (B, H, W), generator=g).float() / 8
    w_om, b_om = exact_om_weights(Ci, seed)
    om = F.conv2d(x.double(), w_om.double(), b_om.double(), padding=1)
    assert torch.equal(om.float().double(), om)
    return x, w_om, b_om, w, b, om.float()


def bn_case(Co, seed=0):
    g = torch.Generator().manual_seed(seed + 2)
    sc = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (Co,), generator=g)]
    sh = torch.randint(-1024, 1025, (Co,), generator=g).float() / 8192
    return sc, sh


def oracle(x, om, w, b, sc=None, sh=None):
    off, logit = om[:, :18].double(), om[:, 18:].double()
    y = dcn_v2_forward(x, off, torch.sigmoid(logit), w, b)
    if sc is not None:
        y = torch.relu(y * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    return y


EXACT = [
    # B, Ci, H, W, Co
    (1, 32, 128, 128, 64),
    (2, 64, 96, 320, 128),
    (3, 256, 16, 16, 256),       # small map: split-K
    (65, 64, 7, 13, 64),
    (4, 512, 17, 5, 72),         # narrow map (16 x 8 tiles), ragged Cout
    (5, 128, 1, 1, 256),
    (2, 256, 32, 48, 200),       # ragged Cout over two tiles
]


@pytest.mark.parametrize("B,Ci,H,W,Co", EXACT)
def test_exact_grid_bit_exact(B, Ci, H, W, Co):
    from centernet_b200.dcn_v2_func import dcn_block_inference, dcn_fused_inference
    x, w_om, b_om, w, b, om = exact_case(B, Ci, H, W, Co)
    sc, sh = bn_case(Co)
    xc, w_omc, b_omc, wc, bc, omc, scc, shc = [t.cuda() for t in (x, w_om, b_om, w, b, om, sc, sh)]
    small = B * H * W * Ci * Co <= 2 ** 27
    want = want_bn = None
    if small:     # the fp64 oracle is slow on the large maps; the two-launch path stands in for it there
        want, want_bn = oracle(x, om, w, b).float(), oracle(x, om, w, b, sc, sh).float()
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        for dt in (torch.float32, BF):
            xi = xin.to(dt)
            for bn in (False, True):
                kw = dict(bn_scale=scc, bn_shift=shc, relu=True) if bn else {}
                y = dcn_block_inference(xi, w_omc, b_omc, wc, bc, 1, 1, 1, 1, **kw)
                assert y is not None and y.dtype == dt and y.shape == (B, Co, H, W)
                ref = dcn_fused_inference(xi, omc, wc, bc, 1, 1, 1, 1, compute_dtype=BF, **kw)
                assert torch.equal(y, ref)
                if small:
                    assert torch.equal(y.cpu(), (want_bn if bn else want).to(dt))


DLA34 = [(512, 16, 256), (256, 32, 256), (256, 32, 128), (128, 64, 128), (128, 64, 64), (64, 128, 64), (256, 32, 64)]


def block_bound(xb, w_omb, b_om, wb, b):
    """fp64 oracle at the bf16 operands and the bound of |block - oracle|: the bf16 bound of test_bf16_gpu (two
    roundings of <= 2^-9 and the fp32 accumulate, 2x margin) plus the offset term.  om's fp32 error is at most
    e = 2^-23 (9 Ci + 1) sum |x_b w_om_b| (+ |b_om| rounding); bilinear interpolation is Lipschitz in the offset with a
    constant of 2 max|x| per axis, and the sigmoid's slope is at most 1/4, so a column value moves by at most
    max|x| (2 e_dy + 2 e_dx + e_logit / 4); the output by sum |w_b| times that (4x margin)."""
    om = F.conv2d(xb.double(), w_omb.double(), b_om.double(), padding=1)
    S_om = F.conv2d(xb.double().abs(), w_omb.double().abs(), b_om.double().abs(), padding=1)
    e = 2.0 ** -23 * (9 * xb.shape[1] + 2) * S_om
    off, m = om[:, :18], torch.sigmoid(om[:, 18:])
    y64 = dcn_v2_forward(xb, off, m, wb, b)
    S = dcn_v2_forward(xb.abs(), off, m, wb.abs(), None)
    xmax = xb.abs().amax(dim=(1, 2, 3)).double().view(-1, 1, 1, 1)
    col_err = xmax * (2 * e[:, 0:18:2] + 2 * e[:, 1:18:2] + e[:, 18:] / 4)          # per (image, tap, pixel)
    wsum = wb.double().abs().sum(dim=1)                                               # [Co][3][3]
    off_term = torch.einsum("btyx,ot->boyx", col_err, wsum.reshape(wb.shape[0], 9))
    bound = 2.0 ** -7 * S + 2.0 ** -8 * y64.abs() + 4 * off_term + 1e-5
    return y64, bound


@pytest.mark.parametrize("Ci,HW,Co", DLA34)
def test_random_within_bound(Ci, HW, Co):
    from centernet_b200.dcn_v2_func import dcn_block_inference
    g = torch.Generator().manual_seed(31)
    x = torch.randn(2, Ci, HW, HW, generator=g)
    w_om = torch.randn(27, Ci, 3, 3, generator=g) * (3.0 / (3.0 * Ci ** 0.5))   # offsets of a few px: many samples
    b_om = torch.randn(27, generator=g) * 2                                      # land outside the image
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (3.0 * Ci ** 0.5)
    b = torch.randn(Co, generator=g)
    xb, w_omb, wb = x.to(BF).float(), w_om.to(BF).float(), w.to(BF).float()
    y64, bound = block_bound(xb, w_omb, b_om, wb, b)
    for xin in (x.cuda(), x.to(BF).cuda().contiguous(memory_format=torch.channels_last)):
        y = dcn_block_inference(xin, w_om.cuda(), b_om.cuda(), w.cuda(), b.cuda(), 1, 1, 1, 1)
        err = (y.double().cpu() - y64).abs()
        lim = bound + (2.0 ** -8 * y64.abs() if y.dtype == BF else 0)
        assert (err <= lim).all(), ((err - lim).max().item(), err.max().item())


def test_nonfinite_inputs_match_the_two_launch_path():
    from centernet_b200.dcn_v2_func import dcn_block_inference, dcn_fused_inference
    g = torch.Generator().manual_seed(7)
    B, Ci, H, W, Co = 2, 64, 24, 40, 64
    x = torch.randn(B, Ci, H, W, generator=g)
    x[0, 3, 5, 7] = float("nan")
    x[1, 10, 0, 0] = float("inf")
    x[1, 20, 23, 39] = -float("inf")
    x[0, 0, 12, 20] = float("nan")
    w_om = torch.randn(27, Ci, 3, 3, generator=g) * 0.05
    b_om = torch.randn(27, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) * 0.05
    b = torch.randn(Co, generator=g)
    xc, w_omc, b_omc, wc, bc = [t.cuda() for t in (x, w_om, b_om, w, b)]
    for xin in (xc, xc.to(BF).contiguous(memory_format=torch.channels_last)):
        y = dcn_block_inference(xin, w_omc, b_omc, wc, bc, 1, 1, 1, 1)
        # the om the block computes: exact products of the bf16 operands, summed in fp32 (the order only moves
        # finite values, so non-finite positions are the same in any order)
        om = F.conv2d(xin.float().to(BF).double(), w_omc.to(BF).double(), b_omc.double(), padding=1).float()
        ref = dcn_fused_inference(xin, om, wc, bc, 1, 1, 1, 1, compute_dtype=BF)
        # and the fp64 oracle at the same om and the bf16 operands: NaN activations make the om of their 3x3
        # neighbourhood NaN, every sample there lies outside and stores 0 * NaN = NaN (DESIGN §4.4)
        want = oracle(xin.float().to(BF).cpu(), om.cpu(), w.to(BF).float(), b)
        for y_ in (y, ref):
            assert torch.equal(torch.isnan(y_).cpu(), torch.isnan(want))
            assert torch.equal(torch.isposinf(y_).cpu(), torch.isposinf(want))
            assert torch.equal(torch.isneginf(y_).cpu(), torch.isneginf(want))
        assert torch.isnan(y).any()


def test_repeats_are_bit_identical():
    from centernet_b200.dcn_v2_func import dcn_block_inference
    g = torch.Generator().manual_seed(3)
    x = torch.randn(16, 128, 64, 64, generator=g).cuda().to(BF).contiguous(memory_format=torch.channels_last)
    w_om = (torch.randn(27, 128, 3, 3, generator=g) * 0.1).cuda()
    b_om, w, b = torch.randn(27, generator=g).cuda(), (torch.randn(128, 128, 3, 3, generator=g) * 0.03).cuda(), \
        torch.randn(128, generator=g).cuda()
    y0 = dcn_block_inference(x, w_om, b_om, w, b, 1, 1, 1, 1)
    for _ in range(3):
        assert torch.equal(dcn_block_inference(x, w_om, b_om, w, b, 1, 1, 1, 1), y0)


class _DeformConv(nn.Module):
    """pose_dla_dcn.DeformConv: DCN, then Sequential(BatchNorm2d, ReLU)."""

    def __init__(self, chi, cho):
        super().__init__()
        from centernet_b200.dcn_v2 import DCN
        self.actf = nn.Sequential(nn.BatchNorm2d(cho, momentum=0.1), nn.ReLU(inplace=True))
        self.conv = DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)

    def forward(self, x):
        return self.actf(self.conv(x))


def _model(seed=0):
    torch.manual_seed(seed)
    m = nn.Sequential(_DeformConv(64, 64), _DeformConv(64, 128))
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            mod.running_mean.uniform_(-0.5, 0.5)
            mod.running_var.uniform_(0.5, 2.0)
            mod.weight.data.uniform_(0.5, 1.5)
            mod.bias.data.uniform_(-0.2, 0.2)
        if hasattr(mod, "conv_offset_mask"):
            mod.conv_offset_mask.weight.data.normal_(0, 0.05)
            mod.conv_offset_mask.bias.data.normal_(0, 0.5)
    return m.cuda().eval()


def test_modules_take_the_block_kernel_in_eval_and_the_old_path_in_grad_mode():
    from centernet_b200.dcn_v2 import fuse_dcn_bn_relu, fuse_offset_conv, set_compute_dtype
    from centernet_b200.dcn_v2_func import dcn_block_inference
    from centernet_b200.dcn_v2 import fold_bn
    x = torch.randn(2, 64, 40, 56, device="cuda")
    plain = _model()
    set_compute_dtype(plain, BF)
    fused = _model()
    assert fuse_offset_conv(fused) == 2 and set_compute_dtype(fused, BF) == 2 and fuse_dcn_bn_relu(fused) == 2
    with torch.no_grad():
        y = fused(x)
        h = x
        for blk in plain:   # the kernel, called directly on the same parameters
            c = blk.conv
            sc, sh = fold_bn(blk.actf[0])
            h = dcn_block_inference(h, c.conv_offset_mask.weight, c.conv_offset_mask.bias, c.weight, c.bias, 1, 1, 1,
                                    1, sc, sh, True)
        assert torch.equal(y, h)
        # DCN.forward on its own, without BN fusion
        d = fused[0].conv
        assert torch.equal(d(x), dcn_block_inference(x, d.conv_offset_mask.weight, d.conv_offset_mask.bias, d.weight,
                                                     d.bias, 1, 1, 1, 1))
    # grad mode: exactly the unflagged module
    ya, yb = fused(x), plain(x)
    assert torch.equal(ya, yb)


def test_tile_cache_follows_the_weights():
    from centernet_b200.dcn_v2 import fuse_offset_conv, set_compute_dtype
    m = _model(1)
    fuse_offset_conv(m)
    set_compute_dtype(m, BF)
    x = torch.randn(1, 64, 32, 32, device="cuda")
    other = _model(2)
    with torch.no_grad():
        y0 = m(x)
        m.load_state_dict(other.state_dict())
        set_compute_dtype(other, BF)
        fuse_offset_conv(other)
        y1 = m(x)
        assert torch.equal(y1, other(x)) and not torch.equal(y0, y1)
        m[0].conv.conv_offset_mask.weight.mul_(0.5)                    # in place: the version moves
        m[0].conv.weight.mul_(2.0)
        other[0].conv.conv_offset_mask.weight.mul_(0.5)
        other[0].conv.weight.mul_(2.0)
        y2 = m(x)
        assert torch.equal(y2, other(x)) and not torch.equal(y2, y1)

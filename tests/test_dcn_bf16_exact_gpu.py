"""GPU: the bf16 DCNv2 paths, bit for bit against the fp64 oracle on exact grids, at every geometry and sampling
boundary of test_dcn_fp32_exact_gpu.

Paths: the bf16 forward (DCNv2Function(compute_dtype=bf16), fp32 and bf16 input and output, NCHW and channels_last),
the bf16 fused inference form (plain, and BN + ReLU in the epilogue), the bf16 backward (autograd in default and
deterministic mode, and cnb_dcnv2_backward_bf16 at every dtype pairing of x and dY, NCHW and channels_last) with its
fallback above Cout 256, and the DCN block kernel at samples exactly on the image edge.

The grids are those of test_dcn_fp32_exact_gpu (x and dY in {0, +-1/2, +-1}, W in {0, +-1/16, +-1/8}, half-integer
offsets, mask in {1/4, 1/2, 1}): every operand is a bf16 value, every column value (<= 6 significant bits) is exact in
bf16, and every product and partial sum is exact in fp32 in any order (the budgets are in that file's docstring).  So
each fp32 result EQUALS the fp64 oracle and each bf16 result is its RN rounding.  Each test first asserts that the
fp64 answers are fp32 values.  The geometries reach the bf16 kernels' branches: 6 channels a group (less than one
8-channel k-chunk), Cout 1 and 5 (K of the column-gradient GEMM below one k16 step), Cout 65 and 272, stride 3,
dilation 3, pad 0, 2x2 / 3x1 / 3x2 kernels, Ho * Wo < 128 and the Wo < 12 tile shapes."""
import pytest
import torch
import torch.nn.functional as F

from oracle.dcn_ref import dcn_v2_forward
from test_bf16_bwd_gpu import NAMES, oracle_grads
from test_bf16_bwd_gpu import raw_backward as raw_backward_bf16
from test_dcn_block_gpu import bn_case, exact_om_weights, oracle as block_oracle
from test_dcn_fp32_exact_gpu import BOUNDARY, CASES, _det, _exact32, autograd, boundary_offsets, grid_inputs

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
GEOM = "B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil"


def check_forward(x, off, m, w, b, stride, pad, dil, dg):
    from centernet_b200.dcn_v2_func import DCNv2Function, dcn_fused_inference
    Co = w.shape[0]
    want = _exact32(dcn_v2_forward(x, off, m, w, b, stride, pad, dil, dg))
    xc, offc, mc, wc, bc = [t.cuda() for t in (x, off, m, w, b)]
    f = DCNv2Function(stride, pad, dil, dg, compute_dtype=BF)
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        for dt in (torch.float32, BF):
            y = f(xin.to(dt), offc, mc, wc, bc)
            assert y.dtype == dt and y.is_contiguous()
            assert torch.equal(y.cpu(), want.to(dt)), ("DCNv2Function", dt, xin.is_contiguous())
    assert torch.equal(f(xc, offc, mc, wc, None).cpu(),
                       _exact32(dcn_v2_forward(x, off, m, w, None, stride, pad, dil, dg))), "bias=None"

    g = torch.Generator().manual_seed(1)
    m2 = torch.where(m == 1.0, 1.0, 0.5)
    om = torch.cat([off, torch.where(m2 == 1.0, 100.0, 0.0)], dim=1).cuda()
    sc = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (Co,), generator=g)]
    sh = torch.randint(-8, 9, (Co,), generator=g).float() / 8
    y64 = dcn_v2_forward(x, off, m2, w, b, stride, pad, dil, dg)
    want_plain = _exact32(y64)
    want_bn = _exact32(torch.relu(y64 * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)))
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        for dt in (torch.float32, BF):
            y = dcn_fused_inference(xin.to(dt), om, wc, bc, stride, pad, dil, dg, bn_scale=sc.cuda(),
                                    bn_shift=sh.cuda(), relu=True, compute_dtype=BF)
            assert y.dtype == dt and torch.equal(y.cpu(), want_bn.to(dt)), ("fused BN + ReLU", dt, xin.is_contiguous())
            y = dcn_fused_inference(xin.to(dt), om, wc, bc, stride, pad, dil, dg, compute_dtype=BF)
            assert y.dtype == dt and torch.equal(y.cpu(), want_plain.to(dt)), ("fused", dt, xin.is_contiguous())


def check_backward(x, off, m, w, b, go, stride, pad, dil, dg):
    from centernet_b200._lib import C
    from centernet_b200.dcn_v2_func import DCNv2Function
    Ci, Co = x.shape[1], w.shape[0]
    want = [_exact32(t) for t in oracle_grads(x, off, m, w, b, go, stride, pad, dil, dg)]
    xc, offc, mc, wc, bc, goc = [t.cuda() for t in (x, off, m, w, b, go)]
    f = DCNv2Function(stride, pad, dil, dg, compute_dtype=BF, backward_dtype=BF)
    cl_ok = (Ci // dg) % 32 == 0
    fallback = C.dcnv2_backward_bf16_workspace_bytes(*x.shape[:2], Co, *x.shape[2:], *w.shape[2:], stride, pad, dil,
                                                     dg) == 0
    assert fallback == (Co > 256)
    try:
        for det in (False, True):
            _det(det)
            for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
                for xdt in (torch.float32, BF):           # grad_output takes the output's (= the input's) dtype
                    got = autograd(f, xin.to(xdt), offc, mc, wc, bc, goc)
                    assert got[0].dtype == xdt
                    for name, a, ref in zip(NAMES, got, want):
                        assert torch.equal(a.cpu(), ref.to(a.dtype)), (name, det, xdt, xin.is_contiguous())
            if fallback:
                continue
            for x_cl in ((False, True) if cl_ok else (False,)):
                for xdt, gdt in ((torch.float32, BF), (BF, torch.float32), (torch.float32, torch.float32), (BF, BF)):
                    got = raw_backward_bf16(xc.to(xdt), x_cl, offc, mc, wc, goc.to(gdt), stride, pad, dil, dg)
                    for name, a, ref in zip(NAMES, got, want):
                        assert torch.equal(a.cpu(), ref), (name, det, xdt, gdt, x_cl)
    finally:
        _det(False)
    assert C.dcnv2_get_deterministic() == 0


# the bf16 C ABI takes one stride / pad / dilation for both axes: every CASES and BOUNDARY geometry is isotropic
@pytest.mark.parametrize(GEOM, CASES)
def test_exact_grid_forward(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    x, off, m, w, b, _ = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil)
    check_forward(x, off, m, w, b, stride, pad, dil, dg)


@pytest.mark.parametrize(GEOM, CASES)
def test_exact_grid_backward(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    x, off, m, w, b, go = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil)
    check_backward(x, off, m, w, b, go, stride, pad, dil, dg)


@pytest.mark.parametrize(GEOM, BOUNDARY)
def test_sampling_boundaries(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    x, off, m, w, b, go = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil, seed=3)
    off = boundary_offsets(off, H, W, kh, kw, stride, pad, dil, dg)
    check_forward(x, off, m, w, b, stride, pad, dil, dg)
    check_backward(x, off, m, w, b, go, stride, pad, dil, dg)


# ---------------------------------------------------------------- the DCN block at the image edge
def edge_case(B, Ci, H, W, Co, seed=0):
    """3x3, stride 1, pad 1.  Channels 1..18 carry the offsets: offset row r of W_om reads carrier channel 1 + r at
    the centre tap with weight 1 (b_om 0), and the carriers have zero main weights.  Carrier values are chosen so
    that tap t of pixel p samples at (hs[(p + t) % 8], ws[(p // 8 + 3 t) % 8]) of the boundary sets, every one a
    half-integer below 128 (exact in bf16).  Channel 0 drives the mask logits through the mask rows of
    exact_om_weights (0 or 100: sigmoid 1/2 or 1)."""
    assert Ci >= 19
    from test_bf16_bwd_gpu import exact_bwd_inputs
    x, _, _, w, b, _ = exact_bwd_inputs(B, Ci, H, W, Co, 1, 3, 3, 1, 1, 1, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    x[:, 0] = torch.randint(0, 2, (B, H, W), generator=g).float() / 8
    w_om, b_om = exact_om_weights(Ci, seed)
    w_om[:18] = 0.0
    b_om[:18] = 0.0
    hs = (-1.5, -1.0, -0.5, 0.0, H - 1.0, H - 0.5, float(H), H + 0.5)
    ws = (-1.5, -1.0, -0.5, 0.0, W - 1.0, W - 0.5, float(W), W + 0.5)
    for t in range(9):
        i, j = t // 3, t % 3
        w_om[2 * t, 1 + 2 * t, 1, 1] = 1.0
        w_om[2 * t + 1, 2 + 2 * t, 1, 1] = 1.0
        for p in range(H * W):
            ho, wo = p // W, p % W
            x[:, 1 + 2 * t, ho, wo] = hs[(p + t) % 8] - (ho - 1 + i)
            x[:, 2 + 2 * t, ho, wo] = ws[(p // 8 + 3 * t) % 8] - (wo - 1 + j)
    w[:, 1:19] = 0.0
    assert (x.abs() < 128).all() and torch.equal(x.to(BF).float(), x)
    om = F.conv2d(x.double(), w_om.double(), b_om.double(), padding=1)
    assert torch.equal(om.float().double(), om)
    return x, w_om, b_om, w, b, om


@pytest.mark.parametrize("B,Ci,H,W,Co", [(2, 32, 12, 12, 16), (1, 64, 10, 21, 72), (1, 32, 24, 9, 32)])
def test_block_sampling_boundaries(B, Ci, H, W, Co):
    from centernet_b200.dcn_v2_func import dcn_block_inference
    x, w_om, b_om, w, b, om = edge_case(B, Ci, H, W, Co)
    # every boundary position is reached: at least one sample of each row / column of the two sets
    off = om[:, :18]
    base_h = (torch.arange(H).view(1, H, 1) - 1 + torch.arange(3).repeat_interleave(3).view(9, 1, 1)).double()
    hpos = off[:, 0::2] + base_h.view(1, 9, H, 1)
    assert all(bool((hpos == v).any()) for v in (-1.5, -1.0, -0.5, 0.0, H - 1.0, H - 0.5, float(H), H + 0.5))
    sc, sh = bn_case(Co)
    want = _exact32(block_oracle(x, om, w, b))
    want_bn = _exact32(block_oracle(x, om, w, b, sc, sh))
    xc, w_omc, b_omc, wc, bc, scc, shc = [t.cuda() for t in (x, w_om, b_om, w, b, sc, sh)]
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        for dt in (torch.float32, BF):
            for bn in (False, True):
                kw = dict(bn_scale=scc, bn_shift=shc, relu=True) if bn else {}
                y = dcn_block_inference(xin.to(dt), w_omc, b_omc, wc, bc, 1, 1, 1, 1, **kw)
                assert y.dtype == dt
                assert torch.equal(y.cpu(), (want_bn if bn else want).to(dt)), (dt, bn, xin.is_contiguous())

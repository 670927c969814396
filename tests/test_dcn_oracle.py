"""CPU: pins the DCNv2 oracle (oracle/dcn_ref.py) with the reference's own known-answer test
(DCNv2/test.py:32-65: zero offsets + identity centre tap + mask 0.5 => 2*DCN(x) == x) and a
cross-check against torchvision.ops.deform_conv2d (third party, same offset layout / bilinear rule), and at the
sampling boundaries with known answers worked out by hand from the reference's rule."""
import math

import pytest
import torch

from oracle.dcn_ref import dcn_v2_forward


def test_zero_offset_identity_kat():
    torch.manual_seed(0)
    N, C, H, W = 2, 2, 4, 4
    x = torch.randn(N, C, H, W)
    w = torch.zeros(C, C, 3, 3)
    for i in range(C):
        w[i, i, 1, 1] = 1.0
    out = dcn_v2_forward(x, torch.zeros(N, 18, H, W), torch.full((N, 9, H, W), 0.5), w, torch.zeros(C))
    assert (out * 2 - x.double()).abs().max().item() < 1e-10          # test.py:62 bound


@pytest.mark.parametrize("stride,dg", [(1, 1), (1, 2), (2, 2)])
def test_against_torchvision(stride, dg):
    tv = pytest.importorskip("torchvision")
    from torchvision.ops import deform_conv2d
    torch.manual_seed(1)
    B, Ci, H, W, Co = 2, 6, 9, 11, 5
    Ho = (H + 2 - 3) // stride + 1
    Wo = (W + 2 - 3) // stride + 1
    x = torch.randn(B, Ci, H, W)
    off = torch.randn(B, 18 * dg, Ho, Wo) * 2.5
    m = torch.rand(B, 9 * dg, Ho, Wo)
    w = torch.randn(Co, Ci, 3, 3)
    b = torch.randn(Co)
    a = dcn_v2_forward(x, off, m, w, b, stride, 1, 1, dg)
    t = deform_conv2d(x.double(), off.double(), w.double(), b.double(), stride=stride, padding=1, dilation=1,
                      mask=m.double())
    assert (a - t).abs().max().item() < 1e-10


# ---------------------------------------------------------------- sampling boundaries: known answers
# One channel, one 1x1 tap of weight 1, mask 1 and a stride larger than the map: a single output pixel whose sampling
# position is exactly (dy, dx).  The reference samples only when -1 < h < H and -1 < w < W (dcn_v2_im2col_cuda.cu:165),
# and then reads each of the four corners only when it lies in the map (:18-47).  Its dOffset is the coordinate weight
# of :75-116: zero outside the same open box, else the difference of the corner values across the cell, each corner
# counted only when it lies in the map.
BH, BW = 4, 5
XB = (torch.arange(BH * BW, dtype=torch.float64) + 1).view(BH, BW)     # x[h, w] = 1 + h * W + w: never 0


def _sample(h, w):
    """(value, d value / d dy, d value / d dx, d value / d x) of the oracle at position (h, w)."""
    x = XB.view(1, 1, BH, BW).clone().requires_grad_(True)
    off = torch.tensor([h, w], dtype=torch.float64).view(1, 2, 1, 1).requires_grad_(True)
    y = dcn_v2_forward(x, off, torch.ones(1, 1, 1, 1), torch.ones(1, 1, 1, 1), None, stride=BH + BW, padding=0)
    assert y.shape == (1, 1, 1, 1)
    y.sum().backward()
    return y.item(), off.grad[0, 0, 0, 0].item(), off.grad[0, 1, 0, 0].item(), x.grad[0, 0]


def _x(h, w):
    return XB[h, w].item() if 0 <= h < BH and 0 <= w < BW else 0.0


def _reference_rule(h, w):
    """dmcn_im2col_bilinear (:18-47) behind the check of :165, and dmcn_get_coordinate_weight (:75-116), written out
    scalar by scalar: (value, dy weight, dx weight)."""
    if not (-1 < h < BH and -1 < w < BW):
        return 0.0, 0.0, 0.0
    hl, wl = math.floor(h), math.floor(w)
    lh, lw = h - hl, w - wl
    v1, v2, v3, v4 = _x(hl, wl), _x(hl, wl + 1), _x(hl + 1, wl), _x(hl + 1, wl + 1)   # 0 when out of range
    val = (1 - lh) * (1 - lw) * v1 + (1 - lh) * lw * v2 + lh * (1 - lw) * v3 + lh * lw * v4
    dh = -(1 - lw) * v1 - lw * v2 + (1 - lw) * v3 + lw * v4
    dw = -(1 - lh) * v1 + (1 - lh) * v2 - lh * v3 + lh * v4
    return val, dh, dw


BOUNDARY_H = (-40.0, -1.5, -1.0, -0.75, -0.5, 0.0, 1.0, 1.5, BH - 1.0, BH - 0.5, BH - 0.25, float(BH), BH + 0.5, 40.0)
BOUNDARY_W = (-40.0, -1.5, -1.0, -0.5, 0.0, 2.0, 2.5, BW - 1.0, BW - 0.5, float(BW), BW + 0.5, 40.0)


def test_boundary_known_answers():
    w = 2.0                                   # an interior integer column: only the row is at the boundary
    for h in (-1.0, float(BH), -40.0, -1.5, BH + 0.5):
        assert _sample(h, w)[:3] == (0.0, 0.0, 0.0), h           # outside the open box: no value, no gradient
    assert _sample(-0.5, w)[0] == 0.5 * XB[0, 2].item()          # the row above the map counts 0
    assert _sample(BH - 0.5, w)[0] == 0.5 * XB[BH - 1, 2].item()  # the row below the map counts 0
    assert _sample(-0.75, w)[0] == 0.25 * XB[0, 2].item()
    # at an exact integer row, dOffset is the one-sided (floor) difference x[h + 1] - x[h]
    assert _sample(0.0, w)[1] == XB[1, 2].item() - XB[0, 2].item()
    assert _sample(1.0, w)[1] == XB[2, 2].item() - XB[1, 2].item()
    assert _sample(BH - 1.0, w)[1] == -XB[BH - 1, 2].item()      # x[H] is out of range: counted as 0
    assert _sample(-0.5, w)[1] == XB[0, 2].item()                 # x[-1] is out of range: counted as 0
    assert _sample(BH - 0.5, w)[1] == -XB[BH - 1, 2].item()
    # and the same along w, at an interior integer row
    assert _sample(1.0, -1.0)[:3] == (0.0, 0.0, 0.0) and _sample(1.0, float(BW))[:3] == (0.0, 0.0, 0.0)
    assert _sample(1.0, -0.5)[0] == 0.5 * XB[1, 0].item() and _sample(1.0, -0.5)[2] == XB[1, 0].item()
    assert _sample(1.0, BW - 1.0)[2] == -XB[1, BW - 1].item()
    assert _sample(1.0, 0.0)[2] == XB[1, 1].item() - XB[1, 0].item()
    # a corner of the map: one valid corner of the four
    val, dh, dw, gx = _sample(-0.5, -0.5)
    assert (val, dh, dw) == (0.25 * XB[0, 0].item(), 0.5 * XB[0, 0].item(), 0.5 * XB[0, 0].item())
    assert gx[0, 0].item() == 0.25 and gx.abs().sum().item() == 0.25     # dX: the corner weight, on that corner only


def test_boundary_grid_matches_reference_rule():
    """Every combination of the boundary rows and columns against the reference's rule written out scalar by scalar."""
    for h in BOUNDARY_H:
        for w in BOUNDARY_W:
            val, dh, dw, gx = _sample(h, w)
            assert (val, dh, dw) == _reference_rule(h, w), (h, w)
            if not (-1 < h < BH and -1 < w < BW):
                assert gx.abs().sum().item() == 0.0, (h, w)


def test_anisotropic_geometry():
    """(h, w) pairs of stride, padding and dilation: at zero offsets with mask 1 the oracle is a plain convolution."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 3, 11, 13, generator=g, dtype=torch.float64)
    w = torch.randn(4, 3, 3, 2, generator=g, dtype=torch.float64)
    b = torch.randn(4, generator=g, dtype=torch.float64)
    for stride, pad, dil in (((1, 2), (2, 0), (2, 1)), ((3, 1), (0, 1), (1, 3)), (2, 1, 2)):
        want = torch.nn.functional.conv2d(x, w, b, stride, pad, dil)
        _, _, Ho, Wo = want.shape
        got = dcn_v2_forward(x, torch.zeros(2, 12, Ho, Wo), torch.ones(2, 6, Ho, Wo), w, b, stride, pad, dil)
        assert got.shape == want.shape and (got - want).abs().max().item() < 1e-12


# ---------------------------------------------------------------- non-finite inputs: the reference's rule
# The reference never reads an out-of-range corner (v = 0, :31-41) and never samples outside the open box (val = 0,
# :160-168), but it multiplies every in-range corner by its weight, 0 included, and stores val * mask for every sample
# (:174).  One output pixel per sample: a 1x1 tap of weight 1, stride 1, pad 0, so y[p] = bias + mask[p] * val[p].
NH, NW = 4, 5
NPOS = (-1.5, -1.0, -0.5, 0.0, 0.5, 1.0, 2.0, NH - 1.0, NH - 0.5, float(NH))


def _one_tap(x, pos, m=None):
    """y[k] = the oracle's sample of x [NH, NW] at pos[k] = (h, w) times m[k]: a 1x1 tap of weight 1 at stride 1, pad 0,
    each sample on an output pixel of its own (the rest sample at -40, outside)."""
    n = len(pos)
    m = torch.ones(n, dtype=torch.float64) if m is None else m
    ys = []
    for k0 in range(0, n, NH * NW):
        chunk = pos[k0:k0 + NH * NW]
        off = torch.full((1, 2, NH, NW), -40.0, dtype=torch.float64)
        mk = torch.ones(1, 1, NH, NW, dtype=torch.float64)
        for k, (h, w) in enumerate(chunk):
            ho, wo = divmod(k, NW)
            off[0, 0, ho, wo], off[0, 1, ho, wo], mk[0, 0, ho, wo] = h - ho, w - wo, m[k0 + k]
        y = dcn_v2_forward(x.view(1, 1, NH, NW), off, mk, torch.ones(1, 1, 1, 1), None, stride=1, padding=0)
        ys.append(y.view(-1)[:len(chunk)])
    return torch.cat(ys)


def _touches_origin(h, w):
    """Whether the sample at (h, w) reads corner (0, 0) with a zero / non-zero weight: (reads, weight)."""
    if not (-1 < h < NH and -1 < w < NW):
        return False, 0.0
    hl, wl = math.floor(h), math.floor(w)
    if hl not in (-1, 0) or wl not in (-1, 0):
        return False, 0.0
    lh, lw = h - hl, w - wl
    return True, (lh if hl == -1 else 1 - lh) * (lw if wl == -1 else 1 - lw)


def test_nonfinite_at_the_origin_reaches_only_the_samples_that_read_it():
    pos = [(h, w) for h in NPOS for w in (-1.5, -1.0, -0.5, 0.0, 0.5, 1.0, 2.0, NW - 1.5)]
    for v in (float("nan"), float("inf"), -float("inf")):
        x = XB[:NH, :NW].clone()
        x[0, 0] = v
        y = _one_tap(x, pos)
        for k, (h, w) in enumerate(pos):
            reads, wt = _touches_origin(h, w)
            if not reads:
                assert math.isfinite(y[k].item()), (v, h, w)        # v * ok would give NaN here
            elif wt == 0.0 or math.isnan(v):
                assert math.isnan(y[k].item()), (v, h, w)           # in range with weight 0: 0 * Inf = NaN
            else:
                assert y[k].item() == v, (v, h, w)


def test_nonfinite_mask_and_offsets():
    x = XB[:NH, :NW].clone()
    pos = [(-40.0, 1.0), (float(NH), 1.0), (1.0, -1.0), (1.5, 1.5), (0.0, 0.0)]   # three outside, two inside
    y = _one_tap(x, pos, torch.full((len(pos),), float("nan"), dtype=torch.float64))
    assert torch.isnan(y).all()                       # val * NaN for the outside samples too (val = 0 there)
    # NaN / Inf offsets: never inside the open box, so val = 0 and the output is 0 * mask
    for bad in (float("nan"), float("inf"), -float("inf")):
        y = _one_tap(x, [(bad, 1.0), (1.0, bad), (bad, bad)], torch.full((3,), 0.5, dtype=torch.float64))
        assert torch.equal(y, torch.zeros(3, dtype=torch.float64)), bad
        y = _one_tap(x, [(bad, 1.0)], torch.full((1,), float("nan"), dtype=torch.float64))
        assert torch.isnan(y).all(), bad


def test_nonfinite_x_gradients():
    """An Inf at (0, 0) that a sample does not read leaves that sample's dOffset and dMask finite; dX never depends
    on x."""
    x = XB[:NH, :NW].clone()
    x[0, 0] = float("inf")
    x = x.view(1, 1, NH, NW).requires_grad_(True)
    off = torch.full((1, 2, NH, NW), -40.0, dtype=torch.float64)
    pos = [(2.0, 2.5), (-0.5, -0.5), (1.5, 3.0)]             # pixel 1 reads (0, 0), pixels 0 and 2 do not
    for k, (h, w) in enumerate(pos):
        off[0, 0, 0, k], off[0, 1, 0, k] = h, w - k
    off.requires_grad_(True)
    m = torch.full((1, 1, NH, NW), 0.5, dtype=torch.float64, requires_grad=True)
    dcn_v2_forward(x, off, m, torch.ones(1, 1, 1, 1), None, stride=1, padding=0).sum().backward()
    assert torch.isfinite(x.grad).all()
    assert x.grad[0, 0, 0, 0].item() == 0.125                 # the corner weight 1/4 times the mask
    assert torch.isfinite(off.grad[0, :, 0, 0]).all() and torch.isfinite(off.grad[0, :, 0, 2]).all()
    assert math.isfinite(m.grad[0, 0, 0, 0].item()) and math.isfinite(m.grad[0, 0, 0, 2].item())
    assert torch.isinf(off.grad[0, :, 0, 1]).all() and m.grad[0, 0, 0, 1].item() == float("inf")

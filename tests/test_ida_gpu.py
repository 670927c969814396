"""The IDA up-sampling step (cnb_ida_up_add) on the GPU: depthwise transposed conv + skip add in one pass.

Exact grids: p on the 1/4 grid with |p| <= 16, skip on the 1/4 grid with |skip| < 64, and the bilinear weights of
fill_up_weights (odd multiples of 1/16, 1/64 and 1/256 for f = 2, 4, 8) or random multiples of 1/16 in [-1, 1].  Every
product and every partial sum is then exact in fp32 and every input exact in bf16, so the fp32 output equals the fp64
oracle bit for bit and the bf16 output equals its RN rounding, whatever the summation order."""
import copy

import pytest
import torch
import torch.nn.functional as F

from test_ida_abi import Neck, bilinear_, neck_inputs

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
U32 = 2.0 ** -24          # unit roundoff of fp32
U16 = 2.0 ** -8           # unit roundoff of bf16 (RN)


def up_weight(C, f, kind, seed=0):
    if kind == "bilinear":
        return bilinear_(torch.nn.ConvTranspose2d(C, C, 2 * f, stride=f, padding=f // 2, groups=C,
                                                  bias=False)).weight.detach().clone()
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-16, 17, (C, 1, 2 * f, 2 * f), generator=g).float() / 16


def oracle(p, w, f, skip):
    return F.conv_transpose2d(p.double().cpu(), w.double().cpu(), stride=f, padding=f // 2,
                              groups=p.shape[1]) + skip.double().cpu()


def magnitude(p, w, f, skip):
    """sum |w p| over the taps of each output element + |skip|: the scale of every error bound here."""
    return F.conv_transpose2d(p.double().abs().cpu(), w.double().abs().cpu(), stride=f, padding=f // 2,
                              groups=p.shape[1]) + skip.double().abs().cpu()


def fused_bound(S, dtype):
    """Four FMAs and one add in fp32 (at most 5 roundings of a partial sum bounded by S), then the output rounding."""
    return S * (6 * U32 + (U16 if dtype == BF else 0.0))


def _layout(t, cl):
    return t.contiguous(memory_format=torch.channels_last) if cl else t.contiguous()


EXACT = [
    # B, C, hp, wp, f
    (1, 1, 1, 1, 2), (3, 3, 3, 5, 2), (1, 64, 16, 16, 2), (65, 3, 3, 5, 4), (3, 128, 16, 16, 4),
    (1, 256, 32, 32, 2), (65, 1, 1, 1, 8), (1, 64, 64, 64, 2), (3, 3, 32, 32, 8), (1, 256, 16, 16, 8),
    (65, 64, 3, 5, 2), (3, 1, 64, 64, 4), (1, 128, 1, 1, 4), (65, 256, 1, 1, 2), (3, 64, 32, 32, 4),
    (1, 3, 64, 64, 8), (65, 128, 3, 5, 8),
]


@pytest.mark.parametrize("B,C,hp,wp,f", EXACT)
@pytest.mark.parametrize("kind", ["bilinear", "random"])
def test_exact_grids_match_the_fp64_oracle(B, C, hp, wp, f, kind):
    from centernet_b200.ida import ida_up_add
    g = torch.Generator().manual_seed(B * 1000 + C + f)
    p = torch.randint(-64, 65, (B, C, hp, wp), generator=g).float() / 4
    skip = torch.randint(-255, 256, (B, C, f * hp, f * wp), generator=g).float() / 4
    w = up_weight(C, f, kind, seed=C + f)
    want = oracle(p, w, f, skip)
    assert torch.equal(want.float().double(), want)              # the grid is exact in fp32
    for dtype in (torch.float32, BF):
        pd, sd = p.to(dtype).cuda(), skip.to(dtype).cuda()
        assert torch.equal(pd.double().cpu(), p.double()) and torch.equal(sd.double().cpu(), skip.double())
        ref = want.float().to(dtype)
        wd = w.to(dtype).cuda()                                   # the weights are exact in bf16 too
        for p_cl in (False, True):
            for s_cl in (False, True):
                for o_cl in (False, True):
                    y = ida_up_add(_layout(pd, p_cl), wd, f, _layout(sd, s_cl), channels_last=o_cl)
                    assert y.dtype == dtype and y.shape == skip.shape
                    assert y.is_contiguous(memory_format=torch.channels_last if o_cl else torch.contiguous_format)
                    assert torch.equal(y.cpu(), ref), (dtype, p_cl, s_cl, o_cl)


def test_output_layout_defaults_to_skips():
    from centernet_b200.ida import ida_up_add
    p, skip, w = torch.randn(2, 8, 4, 4).cuda(), torch.randn(2, 8, 8, 8).cuda(), up_weight(8, 2, "random").cuda()
    assert ida_up_add(p, w, 2, skip).is_contiguous()
    y = ida_up_add(p, w, 2, skip.contiguous(memory_format=torch.channels_last))
    assert y.is_contiguous(memory_format=torch.channels_last) and not y.is_contiguous()
    # a view at an odd offset is copied to an aligned tensor first
    big = torch.randn(2 * 8 * 8 * 8 + 1, device="cuda")
    odd = big[1:].view(2, 8, 8, 8)
    assert torch.equal(ida_up_add(p, w, 2, odd), ida_up_add(p, w, 2, odd.clone()))


RANDOM = [(16, 256, 16, 16, 2), (16, 128, 32, 32, 2), (4, 64, 64, 64, 2), (4, 64, 32, 32, 4), (2, 24, 20, 12, 8),
          (3, 5, 7, 9, 2)]


@pytest.mark.parametrize("B,C,hp,wp,f", RANDOM)
@pytest.mark.parametrize("dtype", [torch.float32, BF])
def test_random_data_within_the_bound(B, C, hp, wp, f, dtype):
    from centernet_b200.ida import ida_up_add
    g = torch.Generator().manual_seed(C * f + hp)
    p = torch.randn(B, C, hp, wp, generator=g).to(dtype)
    skip = (torch.randn(B, C, f * hp, f * wp, generator=g) * 3).to(dtype)
    w = (torch.randn(C, 1, 2 * f, 2 * f, generator=g) / f).to(dtype)
    want, S = oracle(p, w, f, skip), magnitude(p, w, f, skip)
    bound = fused_bound(S, dtype)
    for p_cl, s_cl in ((False, False), (True, False), (False, True), (True, True)):
        y = ida_up_add(_layout(p.cuda(), p_cl), w.cuda(), f, _layout(skip.cuda(), s_cl))
        assert ((y.double().cpu() - want).abs() <= bound).all()
    # the unfused module on cuDNN, TF32 off: the same bound in fp32; in bf16 it rounds twice
    up = torch.nn.ConvTranspose2d(C, C, 2 * f, stride=f, padding=f // 2, groups=C, bias=False).to(dtype).cuda()
    with torch.no_grad():
        up.weight.copy_(w)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            z = (up(p.cuda()) + skip.cuda()).double().cpu()
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    unfused = bound if dtype == torch.float32 else S * (6 * U32 + 2 * U16 + U16 * U16)
    assert ((z - want).abs() <= unfused).all()


@pytest.mark.parametrize("dtype", [torch.float32, BF])
def test_non_finite_inputs_follow_the_unfused_module(dtype):
    from centernet_b200.ida import ida_up_add
    B, C, hp, wp, f = 2, 16, 9, 7, 2
    g = torch.Generator().manual_seed(5)
    p = torch.randn(B, C, hp, wp, generator=g)
    skip = torch.randn(B, C, f * hp, f * wp, generator=g)
    for t in (p, skip):
        flat = t.view(-1)
        idx = torch.randperm(flat.numel(), generator=g)[:3 * max(1, flat.numel() // 50)].view(3, -1)
        flat[idx[0]], flat[idx[1]], flat[idx[2]] = float("nan"), float("inf"), -float("inf")
    p[0, 0, 0, :] = float("inf")                  # along the image edges, where some taps are out of range
    p[1, 1, :, -1] = -float("inf")
    w = torch.rand(C, 1, 2 * f, 2 * f, generator=g) + 0.25
    p, skip, w = p.to(dtype).cuda(), skip.to(dtype).cuda(), w.to(dtype).cuda()
    y = ida_up_add(p, w, f, skip)
    with torch.no_grad():
        z = F.conv_transpose2d(p, w, stride=f, padding=f // 2, groups=C) + skip
    yc, zc = y.float().cpu(), z.float().cpu()
    assert torch.equal(yc.isnan(), zc.isnan())
    assert torch.equal(yc == float("inf"), zc == float("inf")) and torch.equal(yc == -float("inf"), zc == -float("inf"))
    assert yc.isnan().any() and (yc == float("inf")).any() and (yc == -float("inf")).any()
    bits = y.view(torch.int16 if dtype == BF else torch.int32)
    for _ in range(3):                            # bit-identical repeats, NaN payloads included
        assert torch.equal(ida_up_add(p, w, f, skip).view(bits.dtype), bits)


# ------------------------------------------------------------------ module level
def _neck(seed=0):
    torch.manual_seed(seed)
    m = Neck()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.uniform_(-0.2, 0.2)
            mod.running_var.uniform_(0.5, 2.0)
        if hasattr(mod, "conv_offset_mask"):
            mod.conv_offset_mask.weight.data.normal_(0, 0.01)
            mod.conv_offset_mask.bias.data.normal_(0, 0.3)
    return m.cuda().eval()


def _max_err(a, b):
    return (a.float() - b.float()).abs().max().item()


def test_module_fp32_matches_the_unfused_neck(monkeypatch):
    from centernet_b200 import ida as I
    monkeypatch.setattr(I, "_F2_MIN_OUT", 0)           # every step of the small test neck through the kernel
    plain = _neck()
    fused = copy.deepcopy(plain)
    assert I.fuse_ida_up(fused) == 8
    x = neck_inputs(2, 32, device="cuda")
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            a, b = fused(x), plain(x)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert a.dtype == torch.float32 and a.shape == (2, 64, 32, 32)
    assert _max_err(a, b) <= 1e-4 * b.abs().max().item()


class Spy:
    """Counts the calls of the C entry point that reach the GPU."""

    def __init__(self, c):
        self.c, self.n = c, 0

    def __getattr__(self, name):
        return getattr(self.c, name)

    def ida_up_add(self, *a):
        self.n += 1
        return self.c.ida_up_add(*a)


@pytest.mark.parametrize("order", ["ida_first", "ida_last"])
def test_module_bf16_with_the_dcn_block_fusions(monkeypatch, order):
    from centernet_b200 import ida as I
    from centernet_b200.dcn_v2 import fuse_dcn_bn_relu, fuse_offset_conv, set_compute_dtype
    monkeypatch.setattr(I, "_F2_MIN_OUT", 0)

    def block_fusions(m):
        assert set_compute_dtype(m, BF) == 16 and fuse_offset_conv(m) == 16 and fuse_dcn_bn_relu(m) == 16

    plain = _neck().to(BF)
    fused = copy.deepcopy(plain)
    block_fusions(plain)
    if order == "ida_first":
        assert I.fuse_ida_up(fused) == 8
        block_fusions(fused)
    else:
        block_fusions(fused)
        assert I.fuse_ida_up(fused) == 8
    seen = []
    for name, mod in fused.named_modules():
        if name.split(".")[-1].startswith("node_"):
            mod.register_forward_pre_hook(lambda m, a: seen.append(a[0]))
    spy = Spy(I.C)
    monkeypatch.setattr(I, "C", spy)
    x = neck_inputs(2, 32, dtype=BF, device="cuda")
    with torch.no_grad():
        a, b = fused(x), plain(x)
        ref = _neck()(neck_inputs(2, 32, device="cuda"))             # the fp32 neck on the same parameters
    assert spy.n == 8 and len(seen) == 8
    assert all(t.dtype == BF and t.is_contiguous() for t in seen)          # the skips' layout (NCHW) here
    # a channels_last neck stays channels_last: every node reads its input in place
    seen.clear()
    spy.n = 0
    with torch.no_grad():
        c = fused([t.contiguous(memory_format=torch.channels_last) for t in x])
    assert spy.n == 8 and all(t.is_contiguous(memory_format=torch.channels_last) and not t.is_contiguous()
                              for t in seen[:1])
    assert _max_err(c, a) <= 2 ** -5 * ref.abs().max().item()
    assert a.dtype == BF and a.shape == (2, 64, 32, 32)
    # the fused step rounds once where the unfused one rounds twice: both stay as close to the fp32 neck
    scale = ref.abs().max().item()
    e_fused, e_plain = _max_err(a, ref), _max_err(b, ref)
    assert _max_err(a, b) <= 2 ** -5 * scale
    assert e_fused <= max(2 * e_plain, 2 ** -6 * scale)


def test_module_grad_mode_runs_the_original_steps(monkeypatch):
    from centernet_b200 import ida as I
    plain = _neck()
    fused = copy.deepcopy(plain)
    I.fuse_ida_up(fused)
    spy = Spy(I.C)
    monkeypatch.setattr(I, "C", spy)
    monkeypatch.setattr(I, "_F2_MIN_OUT", 0)
    x = neck_inputs(1, 16, device="cuda")
    a, b = fused(x), plain(x)
    assert spy.n == 0 and torch.equal(a, b) and a.requires_grad


def test_small_f2_steps_take_the_original_step(monkeypatch):
    from centernet_b200 import ida as I
    fused = _neck()
    I.fuse_ida_up(fused)
    spy = Spy(I.C)
    monkeypatch.setattr(I, "C", spy)
    with torch.no_grad():
        fused(neck_inputs(1, 32, device="cuda"))
    assert spy.n == 1                                   # only ida_up.up_2 (f = 4)

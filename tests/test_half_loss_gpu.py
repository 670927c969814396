"""Training losses on bf16 / fp16 heads read in place (csrc/focal.cu, csrc/decode_api.cu): focal loss, the fused target
splat, the Reg*Loss family and the feature gather.  The oracle is the fp32 call on the .float() upcast: the loss has to
equal it bit for bit, and the gradient autograd receives has to be (g32 * w).to(dtype) bit for bit for any loss weight
w, at every size, alignment and layout the kernels branch on, at non-finite inputs, and with repeated indices."""
import numpy as np
import pytest
import torch

from helpers import golden

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
WEIGHTS = [1.0, 0.1, 2.5, -2.5, 0.0, 1024.0]


# ------------------------------------------------------------------ helpers
def L():
    from centernet_b200 import losses
    return losses


def same_bits(got, want, what):
    """Bit equality of two tensors of one dtype; NaNs have to sit at the same places."""
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    got, want = got.detach().contiguous(), want.detach().contiguous()
    nan_g, nan_w = torch.isnan(got), torch.isnan(want)
    assert torch.equal(nan_g, nan_w), "%s: NaN pattern differs at %d elements" % (what, int((nan_g != nan_w).sum()))
    ints = {2: torch.int16, 4: torch.int32}[got.element_size()]
    g = torch.where(nan_g, torch.zeros_like(got), got).view(ints)
    w = torch.where(nan_w, torch.zeros_like(want), want).view(ints)
    bad = g != w
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError("%s: %d of %d elements differ, first at %d: got %r, want %r" % (
            what, int(bad.sum()), bad.numel(), i, float(got.flatten()[i]), float(want.flatten()[i])))


def offset_view(t, offset):
    """t on the device as a contiguous view `offset` elements into its storage (odd offsets: not 8-byte aligned)."""
    buf = torch.zeros(t.numel() + 8, dtype=t.dtype, device="cuda")
    v = buf[offset:offset + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def check(fn, xh, weights=WEIGHTS, what="", through_graph=False):
    """fn(pred) -> loss.  Half pred against the fp32 call on its upcast: loss bits, and pred.grad for every weight.
    through_graph: the weight reaches the op inside a [B,M,C] gradient, not as a scalar on its output, so the wanted
    gradient is the one autograd returns through fn(pred.float()) (a map element no index selects is +0 there)."""
    x32 = xh.detach().float().requires_grad_(True)
    l32 = fn(x32)
    l32.backward()
    g32 = x32.grad
    for w in weights:
        x = xh.detach().requires_grad_(True)
        loss = fn(x)
        assert loss.dtype == torch.float32
        same_bits(loss.detach(), l32.detach(), "%s loss" % what)
        (w * loss).backward()
        assert x.grad.dtype == xh.dtype and x.grad.shape == xh.shape
        want = (g32 * w).to(xh.dtype)
        if through_graph:
            xu = xh.detach().requires_grad_(True)
            (w * fn(xu.float())).backward()
            want = xu.grad
        same_bits(x.grad, want, "%s grad, w=%g" % (what, w))
    return l32.detach(), g32


def focal_inputs(n, seed, logits, dtype):
    g = torch.Generator(device="cuda").manual_seed(seed)
    gt = torch.rand(n, device="cuda", generator=g) * 0.98
    gt[::7] = 1.0
    gt[3::11] = 0.0
    x = torch.randn(n, device="cuda", generator=g) * 2.0 - 1.0
    if not logits:
        x = torch.clamp(torch.sigmoid(x), 1e-4, 1 - 1e-4)
    return x.to(dtype), gt


def focal_fn(logits, gt):
    fn = L()._neg_loss_from_logits if logits else L()._neg_loss
    return lambda p: fn(p, gt)


def objects(B, M, C, H, W, seed, rmax=11):
    g = torch.Generator().manual_seed(seed)
    r = lambda hi, lo=0: torch.randint(lo, hi, (B, M), generator=g).cuda()
    return r(C), r(W), r(H), r(rmax + 1), (torch.rand(B, M, generator=g) < 0.8).cuda()


def splat_fn(logits, objs):
    mod = L().FocalSplatLoss(from_logits=logits)
    return lambda p: mod(p, *objs)


def heat(shape, seed, logits, dtype):
    x, _ = focal_inputs(int(np.prod(shape)), seed, logits, dtype)
    return x.view(shape)


# ------------------------------------------------------------------ dense focal loss
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 4099])
def test_focal_dense_sizes(n, logits, dtype):
    x, gt = focal_inputs(n, 11 + n % 97, logits, dtype)
    check(focal_fn(logits, gt), x, what="n=%d" % n)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("logits", [False, True])
def test_focal_dense_above_the_grid_cap(logits, dtype):
    """More float4 groups than 16384 CTAs x 256 threads: every CTA loops whatever the device's own cap, + a tail."""
    n = 16384 * 256 * 4 + 4099
    x, gt = focal_inputs(n, 5, logits, dtype)
    check(focal_fn(logits, gt), x, weights=[0.1], what="n=%d" % n)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("offsets", [(1, 0), (3, 0), (0, 2), (3, 3), (4, 0)])
def test_focal_dense_unaligned(offsets, logits, dtype):
    """pred 1 and 3 elements off (2-byte loads inside the groups of four), gt off 16 bytes (no groups of four, as the
    fp32 kernel then does), pred 8 but not 16 bytes off."""
    x, gt = focal_inputs(4099, 5, logits, dtype)
    xv, gv = offset_view(x, offsets[0]), offset_view(gt, offsets[1])
    check(focal_fn(logits, gv), xv, weights=[1.0, -2.5], what="offsets=%s" % (offsets,))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("layout", ["channels_last", "strided", "transposed"])
def test_focal_dense_layouts(layout, logits, dtype):
    x = heat((2, 6, 12, 20), 23, logits, dtype)
    gt = focal_inputs(x.numel(), 23, logits, dtype)[1].view(x.shape)
    if layout == "channels_last":
        xv = x.contiguous(memory_format=torch.channels_last)
    elif layout == "strided":
        xv = torch.repeat_interleave(x, 2, dim=3)[..., ::2]
    else:
        xv = x.transpose(2, 3).contiguous().transpose(2, 3)
    assert not xv.is_contiguous() and torch.equal(xv, x)
    check(focal_fn(logits, gt), xv, weights=[1.0, 0.1], what=layout)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("kind", ["no_positive", "all_positive", "half_gt"])
def test_focal_dense_targets(kind, logits, dtype):
    x, gt = focal_inputs(1031, 3, logits, dtype)
    if kind == "no_positive":       # num_pos == 0: the un-normalised branch, positives out of the gradient
        gt = gt.clamp(max=0.99)
    elif kind == "all_positive":
        gt = torch.ones_like(gt)
    else:                           # a half target keeps its upcast
        gt = gt.to(dtype)
    check(focal_fn(logits, gt), x, weights=[1.0, -2.5], what=kind)


def _golden_focal_names():
    return [str(n) for n in golden("loss_edges")["focal_names"]]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", _golden_focal_names())
def test_focal_golden_edges(name, dtype):
    """NaN / +-inf predictions, logits at +-inf and around both clamp points, p = 0 and 1, rounded to the dtype; and a
    weight that overflows fp16 (inf, as .to(float16) makes it)."""
    g = golden("loss_edges")
    x = torch.as_tensor(g["f_%s_x" % name]).cuda().to(dtype)
    gt = torch.as_tensor(g["f_%s_gt" % name]).cuda()
    logits = bool(g["f_%s_logits" % name])
    check(focal_fn(logits, gt), x, weights=[1.0, -2.5, 3e5], what=name)
    check(focal_fn(logits, offset_view(gt, 0)), offset_view(x, 1), weights=[1.0], what=name + " unaligned")


def test_fp16_gradient_overflows_to_inf():
    x, gt = focal_inputs(4099, 7, True, torch.float16)
    _, g32 = check(focal_fn(True, gt), x, weights=[1e8], what="overflow")
    x = x.detach().requires_grad_(True)
    (1e8 * focal_fn(True, gt)(x)).backward()
    assert torch.isinf(x.grad).any() and not torch.isinf(g32 * 1e8).any()


# ------------------------------------------------------------------ fused splat + focal loss
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("shape", [(3, 5, 30, 30), (2, 3, 96, 320), (1, 2, 8, 130), (2, 80, 128, 128)])
def test_splat_shapes(shape, logits, dtype):
    B, C, H, W = shape
    objs = objects(B, 128 if H == 128 else 17, C, H, W, 31 + W)
    check(splat_fn(logits, objs), heat(shape, 41, logits, dtype), weights=[1.0, 0.1, -2.5, 0.0, 1024.0],
          what="shape=%s" % (shape,))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ["offset1", "offset3", "offset4", "channels_last", "strided"])
def test_splat_alignment_and_layouts(case, dtype):
    shape = (2, 4, 12, 32)
    x = heat(shape, 43, True, dtype)
    if case.startswith("offset"):
        xv = offset_view(x, int(case[-1]))
    elif case == "channels_last":
        xv = x.contiguous(memory_format=torch.channels_last)
    else:
        xv = torch.repeat_interleave(x, 2, dim=3)[..., ::2]
    check(splat_fn(True, objects(2, 9, 4, 12, 32, 47, rmax=5)), xv, weights=[1.0, -2.5], what=case)


@pytest.mark.parametrize("dtype", DTYPES)
def test_splat_above_the_grid_cap(dtype):
    """B * C planes above the cap of 16384 CTAs: CTAs take several planes."""
    shape = (129, 128, 4, 8)
    objs = objects(129, 6, 128, 4, 8, 53, rmax=2)
    check(splat_fn(True, objs), heat(shape, 59, True, dtype), weights=[0.1], what="grid cap")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("case", ["radius0", "table_overflow", "outside", "duplicates", "none_valid"])
def test_splat_object_edges(case, logits, dtype):
    B, C, H, W = 2, 3, 64, 72
    i = lambda *v: torch.tensor(v, dtype=torch.int64).cuda().view(1, -1).repeat(B, 1)
    cls, valid = i(0, 1, 2, 0), i(1, 1, 1, 1).bool()
    if case == "radius0":
        objs = (cls, i(5, 0, 71, 30), i(5, 0, 63, 30), i(0, 0, 0, 0), valid)
    elif case == "table_overflow":     # 2 r^2 + 1 floats per table: 56, 60 and 70 overflow the 24 KB, 3 fits
        objs = (i(0, 0, 0, 1), i(20, 40, 60, 30), i(20, 30, 40, 30), i(56, 60, 3, 70), valid)
    elif case == "outside":            # centres off every edge: the overlap is painted, no positive is counted
        objs = (cls, i(-3, 75, 10, 200), i(10, -2, 66, 30), i(6, 6, 6, 6), valid)
    elif case == "duplicates":         # one positive per distinct centre
        objs = (i(1, 1, 1, 2), i(9, 9, 9, 9), i(7, 7, 7, 7), i(2, 5, 2, 3), valid)
    else:                              # num_pos == 0
        objs = (cls, i(5, 6, 7, 8), i(5, 6, 7, 8), i(2, 2, 2, 2), torch.zeros_like(valid))
    check(splat_fn(logits, objs), heat((B, C, H, W), 61, logits, dtype), weights=[1.0, -2.5], what=case)


# ------------------------------------------------------------------ Reg*Loss and the gather
def reg_mod(mode):
    return [L().RegL1Loss, L().RegLoss, L().NormRegL1Loss, L().RegWeightedL1Loss][mode]()


def reg_inputs(B, D, H, W, M, seed, mode, dtype, mask_kind="float"):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = (torch.randn(B, D, H, W, device="cuda", generator=g) * 3).to(dtype)
    ind = torch.randint(0, H * W, (B, M), device="cuda", generator=g)
    target = torch.randn(B, M, D, device="cuda", generator=g) * 3 + (2.0 if mode == 2 else 0.0)
    mshape = (B, M, D) if mode == 3 else (B, M)
    mask = torch.rand(mshape, device="cuda", generator=g)
    if mask_kind != "float":
        mask = (mask < 0.7).to({"uint8": torch.uint8, "bool": torch.bool}[mask_kind])
    return out, mask, ind, target


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("mask_kind", ["float", "uint8", "bool"])
def test_reg_modes_and_masks(mask_kind, mode, dtype):
    out, mask, ind, target = reg_inputs(3, 2, 16, 24, 32, 71 + mode, mode, dtype, mask_kind)
    check(lambda o: reg_mod(mode)(o, mask, ind, target), out, what="mode %d %s mask" % (mode, mask_kind))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_reg_repeated_and_out_of_range_indices(mode, dtype):
    """One index 2, 3 and 128 times in an image (their gradients add in fp32 in ascending m, then round once), and
    indices outside the map (skipped: the loss ignores them and nothing is written for them)."""
    B, D, H, W, M = 3, 34, 16, 16, 128
    out, mask, ind, target = reg_inputs(B, D, H, W, M, 83, mode, dtype)
    out = (out.float() * 0.05).to(dtype) if mode == 1 else out   # |diff| < 1 as well: smooth-L1's quadratic side
    ind[0, 5] = ind[0, 90] = 17
    ind[0, 7] = ind[0, 8] = ind[0, 127] = 255
    ind[1, :] = 0
    ind[2, 3], ind[2, 4], ind[2, 100] = -1, H * W, 2 ** 40
    buf = torch.zeros(out.numel() + 512, dtype=dtype, device="cuda")
    view = buf[256:256 + out.numel()].view(out.shape)
    view.copy_(out)
    check(lambda o: reg_mod(mode)(o, mask, ind, target), out, what="mode %d repeats" % mode)
    x = view.detach().requires_grad_(True)
    (2.5 * reg_mod(mode)(x, mask, ind, target)).backward()
    assert not buf[:256].any() and not buf[256 + out.numel():].any()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layout", ["channels_last", "offset1"])
def test_reg_layouts(layout, dtype):
    out, mask, ind, target = reg_inputs(2, 4, 8, 12, 16, 89, 0, dtype)
    ov = out.contiguous(memory_format=torch.channels_last) if layout == "channels_last" else offset_view(out, 1)
    check(lambda o: reg_mod(0)(o, mask, ind, target), ov, weights=[1.0, -2.5], what=layout)


@pytest.mark.parametrize("dtype", DTYPES)
def test_transpose_and_gather(dtype):
    """The gather's rows are fp32 and those of the upcast; its gradient for a [B,M,C] incoming gradient (no scalar
    scale) is the fp32 scatter rounded once, repeated and out-of-range indices included."""
    from centernet_b200.utils import _transpose_and_gather_feat
    out, _, ind, _ = reg_inputs(3, 8, 16, 16, 128, 97, 0, dtype)
    ind[0, 5] = ind[0, 90] = 17
    ind[0, 7] = ind[0, 8] = ind[0, 127] = 255
    ind[1, :] = 3
    ind[2, 3], ind[2, 4] = -1, 16 * 16
    gout = torch.randn(3, 128, 8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    x32 = out.float().requires_grad_(True)
    r32 = _transpose_and_gather_feat(x32, ind)
    r32.backward(gout)
    x = out.detach().requires_grad_(True)
    rows = _transpose_and_gather_feat(x, ind)
    assert rows.dtype == torch.float32
    same_bits(rows, r32, "gathered rows")
    rows.backward(gout)
    same_bits(x.grad, x32.grad.to(dtype), "gather grad")
    # no objects: an empty result and a zero gradient
    x = out.detach().requires_grad_(True)
    empty = _transpose_and_gather_feat(x, ind[:, :0])
    assert empty.shape == (3, 0, 8)
    empty.sum().backward()
    assert x.grad.dtype == dtype and not x.grad.any()


@pytest.mark.parametrize("dtype", DTYPES)
def test_l1_and_binrot_through_the_gather(dtype):
    g = torch.Generator(device="cuda").manual_seed(101)
    B, H, W, M = 2, 12, 20, 24
    ind = torch.randint(0, H * W, (B, M), device="cuda", generator=g)
    ind[0, 1] = ind[0, 2]
    mask = (torch.rand(B, M, device="cuda", generator=g) < 0.7)
    dep = torch.randn(B, 1, H, W, device="cuda", generator=g).to(dtype)
    tgt = torch.randn(B, M, 1, device="cuda", generator=g)
    check(lambda o: L().L1Loss()(o, mask, ind, tgt), dep, what="L1Loss", through_graph=True)
    rot = torch.randn(B, 8, H, W, device="cuda", generator=g).to(dtype)
    rotbin = torch.randint(0, 2, (B, M, 2), device="cuda", generator=g)
    rotres = torch.randn(B, M, 2, device="cuda", generator=g)
    check(lambda o: L().BinRotLoss()(o, mask, ind, rotbin, rotres), rot, what="BinRotLoss", through_graph=True)


# ------------------------------------------------------------------ autograd plumbing, memory, streams
@pytest.mark.parametrize("dtype", DTYPES)
def test_no_gradient_when_none_is_required(dtype):
    x, gt = focal_inputs(4099, 13, True, dtype)
    shape = (2, 3, 16, 20)
    hm = heat(shape, 13, True, dtype)
    objs = objects(2, 9, 3, 16, 20, 13, rmax=4)
    out, mask, ind, target = reg_inputs(2, 2, 16, 20, 9, 13, 0, dtype)
    for fn, t in ((focal_fn(True, gt), x), (splat_fn(True, objs), hm),
                  (lambda o: reg_mod(0)(o, mask, ind, target), out)):
        live = t.detach().requires_grad_(True)
        want = fn(live)
        got = fn(t.detach())
        assert not got.requires_grad and got.grad_fn is None
        same_bits(got, want.detach(), "loss without grad")


def _peak_above_live(step):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_no_fp32_copy_of_the_heat_map_is_made():
    """Forward + backward of a [16,80,128,128] bf16 head.  Dense target: the gradient is numel * 2 bytes and any fp32
    copy of the map (numel * 4) would break the bound.  FocalSplatLoss keeps one fp32 temporary, its unscaled
    gradient: numel * 6 with the half gradient, and a second fp32 map would break numel * 8."""
    shape = (16, 80, 128, 128)
    numel = int(np.prod(shape))
    objs = objects(16, 128, 80, 128, 128, 3)
    gt = L().splat_gaussian(*objs, 80, 128, 128)
    for logits in (False, True):
        for fn, bound in ((focal_fn(logits, gt), numel * 4), (splat_fn(logits, objs), numel * 8)):
            x = heat(shape, 17, logits, torch.bfloat16).requires_grad_(True)
            rise = _peak_above_live(lambda: (0.1 * fn(x)).backward())
            assert x.grad is not None and x.grad.dtype == torch.bfloat16
            assert rise < bound, "peak rose by %d bytes (bound %d)" % (rise, bound)
            del x


def test_no_fp32_copy_of_the_regression_map_is_made():
    shape = (16, 34, 128, 128)
    numel = int(np.prod(shape))
    out, mask, ind, target = reg_inputs(16, 34, 128, 128, 128, 19, 0, torch.bfloat16)
    from centernet_b200.utils import _transpose_and_gather_feat
    for fn in (lambda o: reg_mod(0)(o, mask, ind, target), lambda o: _transpose_and_gather_feat(o, ind).sum()):
        x = out.detach().requires_grad_(True)
        rise = _peak_above_live(lambda: (0.1 * fn(x)).backward())
        assert x.grad.dtype == torch.bfloat16
        assert rise < numel * 4, "peak rose by %d bytes (numel * 4 = %d)" % (rise, numel * 4)


@pytest.mark.parametrize("dtype", DTYPES)
def test_run_to_run_and_side_stream(dtype):
    shape = (4, 8, 64, 64)
    hm = heat(shape, 29, True, dtype)
    gt = focal_inputs(hm.numel(), 29, True, dtype)[1].view(shape)
    objs = objects(4, 32, 8, 64, 64, 29)
    out, mask, ind, target = reg_inputs(4, 8, 64, 64, 128, 29, 0, dtype)
    ind[0, :64] = 5

    def run():
        res = []
        for fn, t in ((focal_fn(True, gt), hm), (splat_fn(True, objs), hm),
                      (lambda o: reg_mod(0)(o, mask, ind, target), out)):
            x = t.detach().requires_grad_(True)
            loss = fn(x)
            (0.1 * loss).backward()
            res += [loss.detach(), x.grad]
        return res
    first, second = run(), run()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        third = run()
    side.synchronize()
    torch.cuda.current_stream().wait_stream(side)
    for a, b, c in zip(first, second, third):
        same_bits(b, a, "second run")
        same_bits(c, a, "side stream")


def test_autocast_head_matches_the_explicit_upcast():
    """A 1x1 conv head under autocast(bfloat16) into the focal loss on logits + RegL1Loss: the conv's weight gradient
    equals that of the same graph with an explicit .float() before each loss."""
    torch.manual_seed(7)
    conv = torch.nn.Conv2d(16, 6, 1).cuda()
    feat = torch.randn(2, 16, 32, 32, device="cuda")
    gt = focal_inputs(2 * 4 * 32 * 32, 37, True, torch.float32)[1].view(2, 4, 32, 32)
    _, mask, ind, target = reg_inputs(2, 2, 32, 32, 16, 37, 0, torch.float32)
    ind[0, 3] = ind[0, 9]
    grads = []
    for upcast in (False, True):
        conv.zero_grad(set_to_none=True)
        with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
            head = conv(feat)
            assert head.dtype == torch.bfloat16
            hm, wh = head[:, :4], head[:, 4:]
            if upcast:
                hm, wh = hm.float(), wh.float()
            loss = L()._neg_loss_from_logits(hm, gt) + 0.1 * L().RegL1Loss()(wh, mask, ind, target)
        loss.backward()
        grads.append((loss.detach(), conv.weight.grad.clone(), conv.bias.grad.clone()))
    for a, b, what in zip(grads[0], grads[1], ("loss", "weight grad", "bias grad")):
        same_bits(a, b, what)

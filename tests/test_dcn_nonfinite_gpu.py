"""GPU: every DCNv2 path against the fp64 oracle at NaN / +-Inf inputs (DESIGN §4.4, "Non-finite inputs").

The reference never reads an out-of-range corner and never samples outside the open box (-1, H) x (-1, W), but it
multiplies every in-range corner by its weight (0 included: 0 * Inf = NaN) and stores val * mask for every sample, so
a NaN mask gives NaN outside the image too.  oracle/dcn_ref.py applies that rule; tests/test_dcn_oracle.py pins it.

Inputs: the exact grids and sampling-boundary offsets of test_dcn_fp32_exact_gpu (every finite output and gradient is
an fp32 value, and bf16-exact where a bf16 path rounds), with NaN, +Inf or -Inf injected into x (at (0, 0), the other
corners, the edge rows and columns and the interior, in the first and last 32-channel block, in a ragged group), NaN
masks at samples inside and outside the image, NaN / +-Inf offsets, and for the fused forms NaN / +-Inf mask logits.
Every value is small, so nothing overflows: whether an element is NaN, +Inf or -Inf does not depend on the order of
any sum, and the kernels must give the oracle's pattern.

Forward: the fp32 CUDA-core, bf16, fused and block paths and the fp64 DCNv2Function give the oracle's NaN, +Inf and
-Inf positions and its finite values bit for bit.  The 3xTF32 paths split every column value v into hi + (v - hi),
which is NaN for v = +-Inf: they give the oracle's finite mask, NaN wherever it has NaN, and where it has +-Inf that
Inf or NaN.

Backward (non-finite x; finite dY, W and mask): dX does not depend on x, so it stays finite and bit-equal to the
oracle in default and deterministic mode; dOffset, dMask and dW have the oracle's NaN / +-Inf pattern (the 3xTF32 dW
its finite mask only), dBias is exact."""
import pytest
import torch
import torch.nn.functional as F

from oracle.dcn_ref import dcn_v2_forward
from test_bf16_bwd_gpu import NAMES, oracle_grads
from test_bf16_bwd_gpu import raw_backward as raw_backward_bf16
from test_dcn_block_gpu import bn_case, exact_case, oracle as block_oracle
from test_dcn_fp32_exact_gpu import _det, autograd, boundary_offsets, grid_inputs, raw_backward, raw_forward

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
NAN, INF = float("nan"), float("inf")


def pattern(got, want, what, inf_may_be_nan=False, finite_only=False):
    """got (any float dtype, any device) against the fp64 oracle want: the NaN / +Inf / -Inf positions (or, with
    finite_only, the finite mask alone; with inf_may_be_nan, an oracle +-Inf may come out as NaN), and the finite
    elements bit for bit at got's dtype."""
    g = got.detach().double().cpu()
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(g), fin), ("finite mask",) + tuple(what)
    if not finite_only:
        assert torch.equal(torch.isnan(g) & torch.isnan(want), torch.isnan(want)), ("NaN",) + tuple(what)
        for sel in (torch.isposinf, torch.isneginf):
            w = sel(want)
            if inf_may_be_nan:
                assert (sel(g) | torch.isnan(g))[w].all(), (sel.__name__,) + tuple(what)
            else:
                assert torch.equal(sel(g), w), (sel.__name__,) + tuple(what)
        if not inf_may_be_nan:
            assert torch.equal(torch.isnan(g), torch.isnan(want)), ("NaN",) + tuple(what)
    exp = want[fin].float()
    assert torch.equal(exp.double(), want[fin]), "the grid's finite fp64 answer is not an fp32 value"
    assert torch.equal(got.detach().cpu()[fin], exp.to(got.dtype)), ("finite values",) + tuple(what)


class Paths(list):
    """Runs pattern() on every path and keeps going, so that one failing test names every path that breaks."""

    def check(self, *args, **kw):
        try:
            pattern(*args, **kw)
        except AssertionError as e:
            self.append(str(e))

    def done(self):
        assert not self, "\n".join(self)


# ---------------------------------------------------------------- inputs
GEOMS = [
    # B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil
    (2, 64, 12, 12, 8, 1, 3, 3, 1, 1, 1),       # two 32-channel blocks
    (1, 80, 11, 13, 8, 2, 3, 3, 1, 1, 1),       # 40 channels a group: ragged blocks, two groups
    (1, 32, 24, 24, 4, 1, 3, 3, 2, 2, 2),       # stride 2, dilation 2
]


def x_sites(B, Ci, H, W, kind):
    """(b, c, h, w) of the injected x elements.  'origin': (0, 0) of one channel in the first and one in the last
    32-channel block (the element every kernel used to read for an out-of-range corner); 'edges': the other three
    corners, edge rows and columns and the interior, spread over channels and images."""
    last = Ci - 1
    if kind == "origin":
        return [(0, 3, 0, 0), (B - 1, last, 0, 0)]
    return [(0, 0, 0, W - 1), (B - 1, 5, H - 1, 0), (0, last, H - 1, W - 1), (B - 1, 33 % Ci, 0, W // 2),
            (0, Ci // 2, H // 2, 0), (B - 1, last - 1, H - 1, W // 3), (0, 7, H // 2, W - 1), (B - 1, 1, H // 2, W // 2)]


def case(geom, x_kind=None, v=NAN, mask_nan=False, off_bad=None, seed=3):
    B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil = geom
    x, off, m, w, b, go = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil, seed=seed)
    off = boundary_offsets(off, H, W, kh, kw, stride, pad, dil, dg)
    if x_kind:
        for s in x_sites(B, Ci, H, W, x_kind):
            x[s] = v
    Ho, Wo = off.shape[2:]
    if mask_nan:     # boundary pixels 0..99 (many samples outside the image) and a few interior ones
        m[0, :, 0, :] = NAN
        m[-1, 0, Ho // 2, :Wo // 2] = NAN
        m[0, -1, Ho - 1, Wo - 1] = NAN
    if off_bad is not None:
        off[0, 0, 0, 1] = off_bad                     # tap 0, dy
        off[-1, 3, Ho // 2, Wo // 2] = off_bad        # tap 1, dx
        off[0, -2, Ho - 1, Wo // 3] = off_bad         # last tap of the last group, dy
    return x, off, m, w, b, go


FW_CASES = ([("x", kind, v) for kind in ("origin", "edges") for v in (NAN, INF, -INF)] +
            [("mask", None, NAN)] + [("offset", None, v) for v in (NAN, INF, -INF)])


def _ids(c):
    return "%s-%s-%s" % c


# ---------------------------------------------------------------- forward
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: "x".join(map(str, g[:5])))
@pytest.mark.parametrize("what,kind,v", FW_CASES, ids=[_ids(c) for c in FW_CASES])
def test_forward(geom, what, kind, v):
    from centernet_b200.dcn_v2_func import DCNv2Function, dcn_fused_inference
    B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil = geom
    x, off, m, w, b, _ = case(geom, x_kind=kind, v=v, mask_nan=what == "mask",
                              off_bad=v if what == "offset" else None)
    want = dcn_v2_forward(x, off, m, w, b, stride, pad, dil, dg)
    # NaN / Inf offsets only move samples outside: the output is finite there (0 * mask)
    assert torch.isfinite(want).all() == (what == "offset")
    ck = Paths()
    xc, offc, mc, wc, bc = [t.cuda() for t in (x, off, m, w, b)]
    xcl = xc.contiguous(memory_format=torch.channels_last)
    ck.check(raw_forward(xc, offc, mc, wc, bc, stride, pad, dil, dg, False), want, ("ABI, CUDA cores",))
    ck.check(raw_forward(xc, offc, mc, wc, bc, stride, pad, dil, dg, True), want, ("ABI, 3xTF32",), inf_may_be_nan=True)
    f32, f16 = DCNv2Function(stride, pad, dil, dg), DCNv2Function(stride, pad, dil, dg, compute_dtype=BF)
    for xin in (xc, xcl):
        lay = ("NCHW" if xin is xc else "channels_last",)
        ck.check(f32(xin, offc, mc, wc, bc), want, ("DCNv2Function 3xTF32",) + lay, inf_may_be_nan=True)
        ck.check(f16(xin, offc, mc, wc, bc), want, ("DCNv2Function bf16, fp32 out",) + lay)
        ck.check(f16(xin.to(BF), offc, mc, wc, bc), want, ("DCNv2Function bf16, bf16 out",) + lay)
    f64 = DCNv2Function(stride, pad, dil, dg)
    y64 = f64(*[t.double().cuda() for t in (x, off, m, w, b)])
    ck.check(y64, want, ("fp64 DCNv2Function",))

    # the fused forms take the raw conv_offset_mask output: mask logits 100 / 0 (sigmoid 1 / 1/2), a NaN mask as a
    # NaN logit; and +-Inf logits (sigmoid exactly 1 / 0)
    m2 = torch.where(m == 1.0, 1.0, torch.where(torch.isnan(m), NAN, 0.5))
    logit = torch.where(m2 == 1.0, 100.0, torch.where(torch.isnan(m2), NAN, 0.0))
    if what == "offset":
        logit[0, 0, 0, 2] = INF
        logit[-1, -1, 1, 1] = -INF
    sig = torch.sigmoid(logit.double())
    om = torch.cat([off, logit], dim=1).cuda()
    gen = torch.Generator().manual_seed(1)
    sc = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (Co,), generator=gen)]
    sh = torch.randint(-8, 9, (Co,), generator=gen).float() / 8
    y64 = dcn_v2_forward(x, off, sig, w, b, stride, pad, dil, dg)
    want_bn = torch.relu(y64 * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    # torch.relu keeps NaN, as the kernels' epilogue does
    for xin in (xc, xcl):
        lay = ("NCHW" if xin is xc else "channels_last",)
        for dt, cdt, tf in ((torch.float32, None, True), (torch.float32, BF, False), (BF, BF, False)):
            kw_ = dict(compute_dtype=cdt) if cdt is not None else {}
            y = dcn_fused_inference(xin.to(dt), om, wc, bc, stride, pad, dil, dg, **kw_)
            ck.check(y, y64, ("fused", dt, cdt) + lay, inf_may_be_nan=tf)
            y = dcn_fused_inference(xin.to(dt), om, wc, bc, stride, pad, dil, dg, bn_scale=sc.cuda(),
                                    bn_shift=sh.cuda(), relu=True, **kw_)
            if tf:   # deviation (c): a +-Inf before the ReLU may come out NaN, and ReLU keeps that NaN (-Inf -> 0)
                pre = torch.isinf(y64)
                ck.check(y.cpu()[~pre], want_bn[~pre], ("fused BN + ReLU", dt, cdt) + lay)
                g = y.double().cpu()[pre]
                if not (torch.isnan(g) | (g == want_bn[pre])).all():
                    ck.append(str(("fused BN + ReLU at an Inf", dt, cdt) + lay))
            else:
                ck.check(y, want_bn, ("fused BN + ReLU", dt, cdt) + lay)
    ck.done()


# ---------------------------------------------------------------- the DCN block
BLOCK = [(2, 32, 12, 12, 16), (1, 64, 9, 20, 40)]


@pytest.mark.parametrize("B,Ci,H,W,Co", BLOCK)
@pytest.mark.parametrize("v", [NAN, INF, -INF], ids=["nan", "inf", "-inf"])
def test_block(B, Ci, H, W, Co, v):
    """NaN / Inf activations: the block's own offset conv turns them into NaN offsets and mask logits in their 3x3
    neighbourhood (every sample there is 'outside', and NaN * val = NaN), and the sampler meets them at corners."""
    from centernet_b200.dcn_v2_func import dcn_block_inference
    x, w_om, b_om, w, b, _ = exact_case(B, Ci, H, W, Co, seed=4)
    for s in [(0, 3, 0, 0), (B - 1, Ci - 1, 0, 0), (0, 5, H - 1, W - 1), (B - 1, 1, H // 2, W // 2),
              (0, 0, 0, W // 2)]:   # channel 0 drives the mask logits
        x[s] = v
    sc, sh = bn_case(Co)
    xc, w_omc, b_omc, wc, bc, scc, shc = [t.cuda() for t in (x, w_om, b_om, w, b, sc, sh)]
    # the oracle is fed the fp64 offset conv of the block's bf16 operands (x and W_om are bf16-exact here)
    om = F.conv2d(x.to(BF).double(), w_om.to(BF).double(), b_om.double(), padding=1)
    want, want_bn = block_oracle(x, om, w, b), block_oracle(x, om, w, b, sc, sh)
    assert not torch.isfinite(want).all()
    ck = Paths()
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        for dt in (torch.float32, BF):
            for bn in (False, True):
                kw = dict(bn_scale=scc, bn_shift=shc, relu=True) if bn else {}
                y = dcn_block_inference(xin.to(dt), w_omc, b_omc, wc, bc, 1, 1, 1, 1, **kw)
                ck.check(y, want_bn if bn else want, ("block", dt, "BN + ReLU" if bn else "plain",
                                                      "NCHW" if xin.is_contiguous() else "channels_last"))
    ck.done()


# ---------------------------------------------------------------- backward
BW_GEOMS = GEOMS[:2]


@pytest.mark.parametrize("geom", BW_GEOMS, ids=lambda g: "x".join(map(str, g[:5])))
@pytest.mark.parametrize("kind,v", [(k, v) for k in ("origin", "edges") for v in (NAN, INF, -INF)],
                         ids=["%s-%s" % (k, v) for k in ("origin", "edges") for v in ("nan", "inf", "-inf")])
def test_backward(geom, kind, v):
    from centernet_b200._lib import C
    from centernet_b200.dcn_v2_func import DCNv2Function
    B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil = geom
    x, off, m, w, b, go = case(geom, x_kind=kind, v=v)
    want = oracle_grads(x, off, m, w, b, go, stride, pad, dil, dg)
    assert torch.isfinite(want[0]).all() and torch.isfinite(want[4]).all()
    assert not torch.isfinite(want[1]).all() and not torch.isfinite(want[3]).all()
    xc, offc, mc, wc, bc, goc = [t.cuda() for t in (x, off, m, w, b, go)]
    xcl = xc.contiguous(memory_format=torch.channels_last)
    cl_ok = (Ci // dg) % 32 == 0

    ck = Paths()

    def check(got, what, tf32_dw, G=None):
        for k, (name, a, ref) in enumerate(zip(NAMES, got, want)):
            if a is None:
                continue
            exp = ref if G is None or G[k] is None else G[k].double() + ref
            ck.check(a, exp, (name,) + tuple(what), finite_only=(name == "weight" and tf32_dw))

    f32 = DCNv2Function(stride, pad, dil, dg)
    f16 = DCNv2Function(stride, pad, dil, dg, compute_dtype=BF, backward_dtype=BF)
    try:
        for det in (False, True):
            _det(det)
            for xin in ((xc, xcl) if cl_ok else (xc,)):
                lay = "NCHW" if xin is xc else "channels_last"
                check(autograd(f32, xin, offc, mc, wc, bc, goc), ("3xTF32 autograd", det, lay), True)
                for xdt in (torch.float32, BF):
                    got = autograd(f16, xin.to(xdt), offc, mc, wc, bc, goc)
                    check(got, ("bf16 autograd", det, lay, xdt), False)
            got, G = raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "tc")
            check(got, ("ABI, tensor cores", det), True, G)
            if cl_ok:
                got, G = raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "tc", x_cl=True)
                check(got, ("ABI _ex, channels_last", det), True, G)
            for x_cl in ((False, True) if cl_ok else (False,)):
                got = raw_backward_bf16(xc.to(BF), x_cl, offc, mc, wc, goc.to(BF), stride, pad, dil, dg)
                check(got, ("ABI bf16", det, x_cl), False)
        _det(False)
        got, G = raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "fp32")
        check(got, ("ABI, CUDA cores",), False, G)
    finally:
        _det(False)
    assert C.dcnv2_get_deterministic() == 0
    ck.done()

"""GPU: the opt-in bf16 DCNv2 backward (compute_dtype=backward_dtype=torch.bfloat16).

1. Exact grids: x and dY in {0, +-1/2, +-1}, W in {0, +-1/16, +-1/8}, half-integer offsets (fractions 0 or 1/2, so the
   corner weights are in {0, 1/4, 1/2, 1}), mask in {1/4, 1/2, 1}, Cin <= 256, Cout <= 272.  Then
     dcol = sum_o W dY        lies on a 2^-5 grid below 272/8 = 34        (11 bits)
     the column value          lies on a 2^-5 grid below 1                 (6 bits: exact in bf16)
     dW partial sums           lie on a 2^-6 grid below B*Ho*Wo <= 960     (16 bits)
     dMask partial sums        lie on a 2^-8 grid below 256 * 34           (22 bits)
     dOffset partial sums      lie on a 2^-9 grid below 256 * 34 * 2       (24 bits)
     dX partial sums           lie on a 2^-9 grid below 34 * 9 taps * 81   (24 bits: a sample with |offset| <= 3.5
                               reaches an input element from at most a 9 x 9 window of output pixels per tap)
     dBias                     lies on a 2^-1 grid
   so every product and every partial sum is exact in fp32 in any order, and all five gradients must EQUAL the fp64
   autograd of the oracle -- in default mode too (exact atomics commute).
2. Random data on the dla_34 layer shapes against bounds derived at the bf16 operands.
3. Run-to-run bit identity; batch-composition invariance of dX in deterministic mode.
4. The fallback above Cout 256: today's bf16 autograd, bit for bit in deterministic mode.
5. Modules: DCN training in fp32 and bf16, set_compute_dtype + fuse_dcn_bn_relu, reproducible SGD steps."""
import pytest
import torch

from oracle.dcn_ref import dcn_v2_forward
from test_bf16_gpu import EXACT, DLA34, _out_hw
from test_dcn_gpu import make

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
NAMES = ("input", "offset", "mask", "weight", "bias")


def exact_bwd_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil, seed=0):
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = _out_hw(H, W, kh, kw, stride, pad, dil)
    kt = kh * kw
    x = torch.randint(-2, 3, (B, Ci, H, W), generator=g).float() / 2
    off = torch.randint(-7, 8, (B, 2 * kt * dg, Ho, Wo), generator=g).float() / 2
    m = torch.tensor([0.25, 0.5, 1.0])[torch.randint(0, 3, (B, kt * dg, Ho, Wo), generator=g)]
    w = torch.randint(-2, 3, (Co, Ci, kh, kw), generator=g).float() / 16
    b = torch.randint(-8, 9, (Co,), generator=g).float() / 8
    go = torch.randint(-2, 3, (B, Co, Ho, Wo), generator=g).float() / 2
    return x, off, m, w, b, go


def oracle_grads(x, off, m, w, b, go, stride=1, pad=1, dil=1, dg=1):
    leaves = [None if t is None else t.detach().double().requires_grad_(True) for t in (x, off, m, w, b)]
    dcn_v2_forward(*leaves, stride, pad, dil, dg).backward(go.double())
    return [None if t is None else t.grad for t in leaves]


def autograd(f, x, off, m, w, b, go):
    leaves = [t.detach().clone().requires_grad_(True) for t in (x, off, m, w, b)]
    y = f(*leaves)
    y.backward(go.to(y.dtype))
    return [t.grad for t in leaves]


def raw_backward(x, x_cl, off, m, w, go, stride, pad, dil, dg):
    """One cnb_dcnv2_backward_bf16 call (x and go of either dtype): fp32 gradients, grad_input in x's layout."""
    from centernet_b200._lib import C, ptr, stream_ptr, workspace
    B, Ci, H, W = x.shape
    Co, _, kh, kw = w.shape
    xin = x.contiguous(memory_format=torch.channels_last) if x_cl else x.contiguous()
    gx = torch.zeros_like(xin, dtype=torch.float32)
    grads = [gx, torch.zeros_like(off), torch.zeros_like(m), torch.zeros_like(w), torch.zeros(Co, device=x.device)]
    dt = {torch.float32: C.DTYPE_F32, BF: C.DTYPE_BF16}
    go = go.contiguous()
    wsb = C.dcnv2_backward_bf16_workspace_bytes(B, Ci, Co, H, W, kh, kw, stride, pad, dil, dg)
    ws = workspace(wsb, x.device)
    C.dcnv2_backward_bf16(ptr(xin), dt[x.dtype], int(x_cl), ptr(off), ptr(m), ptr(w), ptr(go), dt[go.dtype],
                          ptr(gx), int(x_cl), *[ptr(t) for t in grads[1:]], B, Ci, H, W, Co, kh, kw, stride, pad, dil,
                          dg, ptr(ws), wsb, stream_ptr(x))
    return grads


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil", EXACT)
def test_exact_grid_equals_oracle(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b, go = exact_bwd_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil)
    want = oracle_grads(x, off, m, w, b, go, stride, pad, dil, dg)
    want32 = [t.float() for t in want]
    for a, a32 in zip(want, want32):
        assert torch.equal(a32.double(), a)          # the grid makes the fp64 gradients exact in fp32
    xc, offc, mc, wc, bc, goc = [t.cuda() for t in (x, off, m, w, b, go)]
    f = DCNv2Function(stride, pad, dil, dg, compute_dtype=BF, backward_dtype=BF)
    cl_ok = (Ci // dg) % 32 == 0
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
                for xdt in (torch.float32, BF):              # grad_output has the output's (= the input's) dtype
                    got = autograd(f, xin.to(xdt), offc, mc, wc, bc, goc)
                    assert got[0].dtype == xdt                   # a bf16 grad_input: the RN rounding of the exact one
                    for name, a, ref in zip(NAMES, got, want32):
                        assert torch.equal(a.cpu(), ref.to(a.dtype)), (name, det, xdt, xin.is_contiguous())
            if Co <= 256:
                # the C ABI with the other pairings: fp32 input with a bf16 grad_output and the reverse
                for x_cl in ((False, True) if cl_ok else (False,)):
                    for xdt, gdt in ((torch.float32, BF), (BF, torch.float32), (torch.float32, torch.float32)):
                        got = raw_backward(xc.to(xdt), x_cl, offc, mc, wc, goc.to(gdt), stride, pad, dil, dg)
                        for name, a, ref in zip(NAMES, got, want32):
                            assert torch.equal(a.cpu(), ref), (name, det, xdt, gdt, x_cl)
                        assert got[0].is_contiguous(memory_format=torch.channels_last if x_cl else
                                                    torch.contiguous_format)
        finally:
            torch.use_deterministic_algorithms(False)


def _abs_oracle(xb, off, m, wb, gob):
    """The oracle's gradients at |x_b|, |W_b|, |dY_b|: upper bounds of the sums behind dW, dMask and dX."""
    return oracle_grads(xb.abs(), off, m, wb.abs(), None, gob.abs())


@pytest.mark.parametrize("Ci,HW,Co", DLA34)
def test_random_within_bound(Ci, HW, Co):
    """Against the fp64 oracle at the bf16 operands (x_b, W_b, dY_b), with S the oracle's gradients at |x_b|, |W_b|,
    |dY_b| (upper bounds of the sums of magnitudes behind dX, dMask and dW):
      dW:          2^-8 S_w (the column value's one RN rounding, <= 2^-9 relative, with a 2x margin) + 2^-12 S_w for the
                   fp32 accumulation over the pixels;
      dMask, dX:   g S with g = (Cout + Cin + 9 * 81 + 16) 2^-24: the fp32 sums of the column gradient (Cout exact
                   products), of the channel reduction and of at most 9 x 81 scattered contributions;
      dOffset:     2^-12 of its largest magnitude (its corner differences have no absolute-value form in the oracle);
    a bf16 grad_input adds its own rounding, 2^-8 |dX|.  For a bf16 grad_output the same three must lie within twice
    those bounds of today's bf16 autograd (one bf16 ulp, 2^-7 |dX|, apart for grad_input) and dBias must equal it; for
    an fp32 one dBias sums the unrounded dY in a fixed tree (depth * 2^-24 * sum |dY|).
    The offsets lie on a 2^-16 grid, so every sampling position (below 256) is exact in fp32: the kernels and the
    oracle agree on the geometry, and the bounds cover the arithmetic alone.  (Elsewhere an fp32 position such as
    66.9999993 -> 67.0 can land in the next cell, where dOffset jumps; every fp32 path shares that.)"""
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = make(2, Ci, HW, HW, Co, 1, seed=21)
    off = torch.round(off * 2.0 ** 16) / 2.0 ** 16
    go = torch.randn(2, Co, HW, HW, generator=torch.Generator().manual_seed(22))
    xb, wb, gob = x.to(BF).float(), w.to(BF).float(), go.to(BF).float()
    ref = oracle_grads(xb, off, m, wb, b, gob)
    S = _abs_oracle(xb, off, m, wb, gob)
    g = (Co + Ci + 9 * 81 + 16) * 2.0 ** -24
    bounds = {"input": g * S[0] + 1e-6, "offset": 2.0 ** -12 * ref[1].abs().max().item() + 1e-6,
              "mask": g * S[2] + 1e-6, "weight": (2.0 ** -8 + 2.0 ** -12) * S[3] + 1e-6}
    xc, offc, mc, wc, bc, goc = [t.cuda() for t in (x, off, m, w, b, go)]
    new = DCNv2Function(1, 1, 1, 1, compute_dtype=BF, backward_dtype=BF)
    old = DCNv2Function(1, 1, 1, 1, compute_dtype=BF)
    for xdt in (torch.float32, BF):
        got = autograd(new, xc.to(xdt), offc, mc, wc, bc, goc)
        for name, a, r in zip(NAMES[:4], got, ref):
            err = (a.double().cpu() - r).abs()
            if xdt == BF and name == "input":
                err = err - 2.0 ** -8 * r.abs()
            assert (err <= bounds[name]).all(), (name, xdt, (err - bounds[name]).max().item())
        if xdt == BF:      # bf16 grad_output: against today's bf16 autograd (fp32 backward at the upcast operands)
            was = autograd(old, xc.to(xdt), offc, mc, wc, bc, goc)
            assert torch.equal(got[4], was[4])
            for name, a, r in zip(NAMES[:3], got[:3], was[:3]):
                err = (a.double() - r.double()).abs().cpu()
                if name == "input":                         # both rounded to bf16: up to one ulp apart
                    err = err - 2.0 ** -7 * r.double().abs().cpu()
                assert (err <= 2 * bounds[name]).all(), (name, (err - 2 * bounds[name]).max().item())
        else:              # fp32 grad_output: dBias sums it unrounded, in a fixed tree of depth <= 13 + slices / 256
            gb = go.double().sum((0, 2, 3))
            depth = 13 + (2 * (HW * HW + 31) // 32 + 255) // 256
            bound = depth * 2.0 ** -24 * go.double().abs().sum((0, 2, 3))
            assert ((got[4].double().cpu() - gb).abs() <= bound).all()


def test_run_to_run_and_batch_composition():
    from centernet_b200.dcn_v2_func import DCNv2Function
    f = DCNv2Function(1, 1, 1, 1, compute_dtype=BF, backward_dtype=BF)
    x, off, m, w, b = [t.cuda() for t in make(2, 128, 64, 64, 128, 1, seed=31, off_scale=4.0)]
    go = torch.randn(2, 128, 64, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    for xin in (x.to(BF), x.to(BF).contiguous(memory_format=torch.channels_last)):
        a = autograd(f, xin, off, m, w, b, go)
        c = autograd(f, xin, off, m, w, b, go)
        for name, u, v in zip(NAMES[1:], a[1:], c[1:]):
            assert torch.equal(u, v), name
        torch.use_deterministic_algorithms(True)
        try:
            a = autograd(f, xin, off, m, w, b, go)
            c = autograd(f, xin, off, m, w, b, go)
        finally:
            torch.use_deterministic_algorithms(False)
        for name, u, v in zip(NAMES, a, c):
            assert torch.equal(u, v), name

    # 37 images of 64@128^2 run as two batch chunks (36 + 1, plan_backward_bf16's ~1.5 GiB of column gradient);
    # images 0, 35 and 36 alone must give the same dX, dOffset and dMask bits
    B, Ci, H, W, Co = 37, 64, 128, 128, 64
    g = torch.Generator(device="cuda").manual_seed(29)
    x = torch.randn(B, Ci, H, W, device="cuda", generator=g).to(BF)
    off = torch.randn(B, 18, H, W, device="cuda", generator=g) * 4.0
    m = torch.sigmoid(torch.randn(B, 9, H, W, device="cuda", generator=g))
    w = torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) / (3.0 * Ci ** 0.5)
    go = torch.randn(B, Co, H, W, device="cuda", generator=g).to(BF)
    from centernet_b200._lib import C
    C.dcnv2_set_deterministic(1)
    try:
        full = raw_backward(x, False, off, m, w, go, 1, 1, 1, 1)
        for img in (0, 35, 36):
            sl = slice(img, img + 1)
            one = raw_backward(x[sl], False, off[sl].contiguous(), m[sl].contiguous(), w, go[sl], 1, 1, 1, 1)
            for name, u, v in zip(NAMES[:3], full[:3], one[:3]):
                assert torch.equal(u[sl], v), (name, img)
    finally:
        C.dcnv2_set_deterministic(0)


def test_fallback_above_cout_256():
    from centernet_b200._lib import C
    from centernet_b200.dcn_v2_func import DCNv2Function
    assert C.dcnv2_backward_bf16_workspace_bytes(2, 128, 272, 16, 16, 3, 3, 1, 1, 1, 1) == 0
    x, off, m, w, b = [t.cuda() for t in make(2, 128, 16, 16, 272, 1, seed=13)]
    go = torch.randn(2, 272, 16, 16, device="cuda")
    new = DCNv2Function(1, 1, 1, 1, compute_dtype=BF, backward_dtype=BF)
    old = DCNv2Function(1, 1, 1, 1, compute_dtype=BF)
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            a = autograd(new, x.to(BF), off, m, w, b, go)
            r = autograd(old, x.to(BF), off, m, w, b, go)
        finally:
            torch.use_deterministic_algorithms(False)
        for name, u, v in zip(NAMES, a, r):
            if name in ("input", "weight") and not det:   # default mode: float atomics (the fp32 dW kernel above 256)
                assert (u.float() - v.float()).abs().max().item() <= 1e-2 * max(1.0, v.float().abs().max().item())
            else:
                assert torch.equal(u, v), (name, det)


def _stack(cin, cout, n):
    from torch import nn
    from centernet_b200.dcn_v2 import DCN

    class DeformConv(nn.Module):          # shape of pose_dla_dcn.py:345-357
        def __init__(self, chi, cho):
            super().__init__()
            self.actf = nn.Sequential(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))
            self.conv = DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)

        def forward(self, x):
            return self.actf(self.conv(x))

    torch.manual_seed(5)
    layers = [DeformConv(cin if i == 0 else cout, cout) for i in range(n)]
    for l in layers:
        l.conv.conv_offset_mask.weight.data.normal_(0, 0.02)
        l.conv.conv_offset_mask.bias.data.normal_(0, 0.5)
    return nn.Sequential(*layers).cuda()


def test_modules_train():
    from centernet_b200.dcn_v2 import DCN, fuse_dcn_bn_relu, set_compute_dtype
    torch.manual_seed(0)
    # DCN with both flags, an fp32 and a bf16 model: every parameter gets a gradient of its own dtype
    for dt in (torch.float32, BF):
        dcn = DCN(64, 64, 3, 1, 1, compute_dtype=BF, backward_dtype=BF).cuda().to(dt)
        dcn.conv_offset_mask.weight.data.normal_(0, 0.02)
        dcn.conv_offset_mask.bias.data.normal_(0, 0.5)
        x = torch.randn(2, 64, 24, 24, device="cuda").to(dt).requires_grad_(True)
        y = dcn(x)
        assert y.dtype == dt
        y.float().square().sum().backward()
        for name, p in dcn.named_parameters():
            assert p.grad is not None and p.grad.dtype == dt and p.grad.abs().sum().item() > 0, name
        assert x.grad.dtype == dt

    # set_compute_dtype(..., backward_dtype) composes with fuse_dcn_bn_relu: training runs the unfused path with the
    # bf16 backward, inference the fused kernel; in deterministic mode both orders give the same gradient bits
    grads = []
    x = torch.randn(2, 64, 20, 20, device="cuda")
    for fuse_first in (True, False):
        model = _stack(64, 64, 1)
        if fuse_first:
            assert fuse_dcn_bn_relu(model) == 1
        assert set_compute_dtype(model, BF, backward_dtype=BF) == 1
        if not fuse_first:
            assert fuse_dcn_bn_relu(model) == 1
        model.train()
        torch.use_deterministic_algorithms(True)
        try:
            model(x).square().sum().backward()
        finally:
            torch.use_deterministic_algorithms(False)
        grads.append({n: p.grad.clone() for n, p in model.named_parameters()})
        model.eval()
        with torch.no_grad():
            assert model(x).dtype == torch.float32
    assert grads[0].keys() == grads[1].keys()
    for n in grads[0]:
        assert torch.equal(grads[0][n], grads[1][n]), n
    model = _stack(64, 64, 1)
    set_compute_dtype(model, BF)                      # today's backward: the weight gradient differs in its last bits
    torch.use_deterministic_algorithms(True)
    try:
        model(x).square().sum().backward()
    finally:
        torch.use_deterministic_algorithms(False)
    assert not torch.equal(model[0].conv.weight.grad, grads[0]["0.conv.weight"])

    # a few SGD steps of a small DeformConv stack are reproducible bit for bit under deterministic mode
    def train():
        model = _stack(32, 64, 2)
        set_compute_dtype(model, BF, backward_dtype=BF)
        opt = torch.optim.SGD(model.parameters(), lr=1e-2, momentum=0.9)
        g = torch.Generator(device="cuda").manual_seed(4)
        torch.use_deterministic_algorithms(True)
        try:
            for _ in range(3):
                xb = torch.randn(2, 32, 24, 24, device="cuda", generator=g)
                opt.zero_grad()
                model(xb).square().mean().backward()
                opt.step()
        finally:
            torch.use_deterministic_algorithms(False)
        return [p.detach().clone() for p in model.parameters()]
    for u, v in zip(train(), train()):
        assert torch.equal(u, v)

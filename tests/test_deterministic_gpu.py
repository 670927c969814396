"""GPU: deterministic training backward.  With cnb_dcnv2_set_deterministic(1) (Python: torch.use_deterministic_algorithms
or CNB_DCN_DETERMINISTIC=1) all five DCNv2 gradients repeat bit for bit for any offsets, stride, deformable groups,
Cout and layout, and do not depend on how the batch is split; the loss gradients repeat bit for bit unconditionally.
Every repeat runs a correct computation a fixed small number of times."""
import json
import os
import subprocess
import sys

import pytest
import torch

from oracle.dcn_ref import dcn_v2_forward

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("input", "offset", "mask", "weight", "bias")


def make(B, Ci, H, W, Co, dg, stride=1, seed=0, off_scale=5.0):
    g = torch.Generator().manual_seed(seed)
    Ho = (H + 2 - 3) // stride + 1
    Wo = (W + 2 - 3) // stride + 1
    x = torch.randn(B, Ci, H, W, generator=g)
    off = torch.randn(B, 18 * dg, Ho, Wo, generator=g) * off_scale
    m = torch.sigmoid(torch.randn(B, 9 * dg, Ho, Wo, generator=g))
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (3.0 * Ci ** 0.5)
    b = torch.randn(Co, generator=g)
    go = torch.randn(B, Co, Ho, Wo, generator=g)
    return x, off, m, w, b, go


def raw_backward(x, off, m, w, go, stride, dg, det):
    """cnb_dcnv2_backward on the tensor-core path (det=True: deterministic mode, workspace queried in that mode) or on
    the fp32 CUDA-core path (det=False, no workspace)."""
    from centernet_b200._lib import C, ptr, stream_ptr, workspace
    B, Ci, H, W = x.shape
    Co = w.shape[0]
    grads = [torch.zeros_like(x), torch.zeros_like(off), torch.zeros_like(m), torch.zeros_like(w),
             torch.zeros(Co, device=x.device)]
    C.dcnv2_set_deterministic(int(det))
    try:
        ws, wsb, keep = 0, 0, None
        if det:
            wsb = C.dcnv2_backward_workspace_bytes(B, Ci, Co, H, W, 3, 3, stride, 1, 1, dg)
            keep = workspace(wsb, x.device)
            ws = ptr(keep)
        C.dcnv2_backward(ptr(x), ptr(off), ptr(m), ptr(w), ptr(go), *[ptr(g) for g in grads], B, Ci, H, W, Co, 3, 3,
                         stride, stride, 1, 1, 1, 1, dg, ws, wsb, stream_ptr(x))
        torch.cuda.synchronize()
    finally:
        C.dcnv2_set_deterministic(0)
    return grads


def oracle_grads(x, off, m, w, b, go, stride, dg):
    leaves = [t.clone().double().requires_grad_(True) for t in (x, off, m, w, b)]
    (dcn_v2_forward(*leaves, stride, 1, 1, dg) * go.double()).sum().backward()
    return [t.grad for t in leaves]


def assert_close(got, want, tol, what):
    for name, u, v in zip(NAMES, got, want):
        v = v.to(u.device, u.dtype) if v.dtype != torch.float64 else v
        diff = (u.double().cpu() - v.double().cpu()).abs().max().item()
        scale = max(1.0, v.abs().max().item())
        assert diff <= tol * scale, (what, name, diff, scale)


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride,off_scale", [
    (2, 64, 24, 28, 64, 1, 1, 5.0),     # most samples land more than 2 px from their tap
    (2, 64, 21, 23, 48, 1, 2, 4.0),     # stride 2
    (2, 40, 15, 17, 24, 2, 1, 4.0),     # two deformable groups, 20 channels per group (padded channel block)
    (2, 64, 12, 12, 272, 1, 1, 6.0),    # Cout > 256: dW by the fp32 kernel, per-split partials
])
def test_free_offsets_bit_identical(B, Ci, H, W, Co, dg, stride, off_scale):
    x, off, m, w, b, go = make(B, Ci, H, W, Co, dg, stride, seed=41, off_scale=off_scale)
    xc, offc, mc, wc, goc = [t.cuda() for t in (x, off, m, w, go)]
    runs = [raw_backward(xc, offc, mc, wc, goc, stride, dg, True) for _ in range(3)]
    for r in runs[1:]:
        for name, u, v in zip(NAMES, runs[0], r):
            assert torch.equal(u, v), name + " not bit-identical run to run in deterministic mode"
    assert all(torch.isfinite(t).all() for t in runs[0])
    assert_close(runs[0], raw_backward(xc, offc, mc, wc, goc, stride, dg, False), 2e-4, "fp32 path")
    assert_close(runs[0], oracle_grads(x, off, m, w, b, go, stride, dg), 1e-3, "fp64 oracle")


def test_channels_last_keeps_layout_and_bits(monkeypatch):
    """Deterministic mode keeps a channels_last activation: the backward takes it in place (no NCHW copy is saved),
    grad_input comes back channels_last, and its values are the NCHW run's bit for bit."""
    import centernet_b200.dcn_v2_func as F
    monkeypatch.setattr(F, "_DETERMINISTIC", True)
    x, off, m, w, b, go = [t.cuda() for t in make(2, 64, 20, 24, 64, 1, 1, seed=43, off_scale=4.0)]

    def run(xin):
        leaves = [xin.clone().requires_grad_(True)] + [t.clone().requires_grad_(True) for t in (off, m, w, b)]
        out = F.DCNv2Function(1, 1, 1, 1)(*leaves)
        (out * go).sum().backward()
        return out, [t.grad for t in leaves]

    try:
        xcl = x.contiguous(memory_format=torch.channels_last)
        out_cl, g_cl = run(xcl)
        assert out_cl.grad_fn.x_cl, "the channels_last activation was not kept for the backward"
        assert g_cl[0].is_contiguous(memory_format=torch.channels_last) and not g_cl[0].is_contiguous()
        _, g_cl2 = run(xcl)
        _, g_nchw = run(x)
    finally:
        from centernet_b200._lib import C
        C.dcnv2_set_deterministic(0)
    for name, u, v, u2 in zip(NAMES, g_cl, g_nchw, g_cl2):
        assert torch.equal(u, u2), name + " (channels_last) not bit-identical run to run"
        assert torch.equal(u, v), name + ": channels_last and NCHW differ"


def test_batch_composition_invariance():
    """33 images of 64@128^2 run as two batch chunks (32 + 1); images 0, 29, 30 and 32 alone must give the same bits."""
    B, Ci, H, W, Co = 33, 64, 128, 128, 64
    g = torch.Generator(device="cuda").manual_seed(29)
    x = torch.randn(B, Ci, H, W, device="cuda", generator=g)
    off = torch.randn(B, 18, H, W, device="cuda", generator=g) * 4.0
    m = torch.sigmoid(torch.randn(B, 9, H, W, device="cuda", generator=g))
    w = torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) / (3.0 * Ci ** 0.5)
    go = torch.randn(B, Co, H, W, device="cuda", generator=g)
    full = raw_backward(x, off, m, w, go, 1, 1, True)
    for img in (0, 29, 30, 32):
        sl = slice(img, img + 1)
        one = raw_backward(x[sl].contiguous(), off[sl].contiguous(), m[sl].contiguous(), w, go[sl].contiguous(), 1, 1, True)
        for name, u, v in zip(NAMES[:3], full[:3], one[:3]):
            assert torch.equal(u[sl], v), (name, img)
    del full


def test_concentrated_samples():
    """Every sample of a 64@32^2 image lands on the same 2x2 input neighbourhood (9216 contributions per element)."""
    B, Ci, H, W, Co = 1, 64, 32, 32, 64
    x, _, m, w, b, go = make(B, Ci, H, W, Co, 1, 1, seed=47)
    ho = torch.arange(H, dtype=torch.float32).view(1, 1, H, 1)
    wo = torch.arange(W, dtype=torch.float32).view(1, 1, 1, W)
    ki = torch.arange(9).div(3, rounding_mode="floor").float().view(1, 9, 1, 1)
    kj = torch.arange(9).remainder(3).float().view(1, 9, 1, 1)
    dy = 16.3 - (ho - 1 + ki)
    dx = 16.6 - (wo - 1 + kj)
    off = torch.stack([dy.expand(1, 9, H, W), dx.expand(1, 9, H, W)], 2).reshape(1, 18, H, W).contiguous()
    xc, offc, mc, wc, goc = [t.cuda() for t in (x, off, m, w, go)]
    runs = [raw_backward(xc, offc, mc, wc, goc, 1, 1, True) for _ in range(2)]
    for name, u, v in zip(NAMES, runs[0], runs[1]):
        assert torch.equal(u, v), name
    gx = runs[0][0]
    assert torch.isfinite(gx).all()
    nz = gx.abs().sum(1)[0].nonzero().tolist()
    assert sorted(map(tuple, nz)) == [(16, 16), (16, 17), (17, 16), (17, 17)]
    assert_close(runs[0], oracle_grads(x, off, m, w, b, go, 1, 1), 1e-3, "fp64 oracle")


def test_non_finite_grad_output():
    """One inf in dY: grad_input is non-finite wherever the fp32 path's is; the other image stays finite and exact."""
    x, off, m, w, b, go = [t.cuda() for t in make(2, 64, 16, 16, 64, 1, 1, seed=53, off_scale=3.0)]
    clean = raw_backward(x, off, m, w, go, 1, 1, True)
    go[0, 5, 7, 9] = float("inf")
    det = raw_backward(x, off, m, w, go, 1, 1, True)
    ref = raw_backward(x, off, m, w, go, 1, 1, False)
    bad = ~torch.isfinite(ref[0])
    assert bad.any()
    assert (~torch.isfinite(det[0][bad])).all()
    assert torch.equal(det[0][1], clean[0][1])


def _repeat(fn, n=3):
    outs = [fn() for _ in range(n)]
    for o in outs[1:]:
        for u, v in zip(outs[0], o):
            assert torch.equal(u, v)
    return outs[0]


def test_losses_bit_identical():
    """FocalLoss, FocalSplatLoss, RegL1Loss / RegWeightedL1Loss and the _transpose_and_gather_feat adjoint repeat bit
    for bit, repeated `ind` entries included; the gather adjoint sums repeats exactly like index_add in fp64."""
    from centernet_b200 import losses as L
    from centernet_b200.utils import _transpose_and_gather_feat
    g = torch.Generator(device="cuda").manual_seed(61)
    B, C, H, W, M = 4, 6, 40, 48, 16
    logits = torch.randn(B, C, H, W, device="cuda", generator=g)
    pred = torch.sigmoid(logits).clamp(1e-4, 1 - 1e-4)
    cls = torch.randint(0, C, (B, M), device="cuda", generator=g)
    cx = torch.randint(0, W, (B, M), device="cuda", generator=g)
    cy = torch.randint(0, H, (B, M), device="cuda", generator=g)
    rad = torch.randint(0, 6, (B, M), device="cuda", generator=g)
    val = torch.ones(B, M, dtype=torch.uint8, device="cuda")
    gt = L.splat_gaussian(cls, cx, cy, rad, val, C, H, W)
    ind = (cy * W + cx).long()
    ind[:, 1] = ind[:, 0]                              # duplicates inside every image
    ind[:, 2] = ind[:, 0]
    reg = torch.randn(B, 2, H, W, device="cuda", generator=g)
    tgt = torch.randn(B, M, 2, device="cuda", generator=g)
    rmask = torch.ones(B, M, dtype=torch.uint8, device="cuda")
    wmask = torch.rand(B, M, 2, device="cuda", generator=g)

    def grad_of(fn, t):
        t = t.clone().requires_grad_(True)
        loss = fn(t)
        loss.backward()
        return loss.detach(), t.grad

    _repeat(lambda: grad_of(lambda p: L.FocalLoss()(p, gt), pred))
    _repeat(lambda: grad_of(lambda p: L.FocalSplatLoss(from_logits=True)(p, cls, cx, cy, rad, val), logits))
    _repeat(lambda: grad_of(lambda o: L.RegL1Loss()(o, rmask, ind, tgt), reg))
    _repeat(lambda: grad_of(lambda o: L.RegWeightedL1Loss()(o, wmask, ind, tgt), reg))
    go = torch.randn(B, M, 2, device="cuda", generator=g)
    _, gfeat = _repeat(lambda: grad_of(lambda f: (_transpose_and_gather_feat(f, ind) * go).sum(), reg))
    want = torch.zeros(B, 2, H * W, dtype=torch.float64, device="cuda")
    want.scatter_add_(2, ind.unsqueeze(1).expand(B, 2, M), go.double().permute(0, 2, 1))
    assert (gfeat.double().view(B, 2, -1) - want).abs().max().item() <= 1e-6


E2E = r"""
import json, sys, torch
from torch import nn
sys.path.insert(0, ROOT)
from centernet_b200.dcn_v2 import DCN
from centernet_b200 import losses as L
torch.use_deterministic_algorithms(True)

class Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.stem = nn.Conv2d(3, 32, 3, padding=1)
        self.dcn = DCN(32, 32, kernel_size=(3, 3), stride=1, padding=1, deformable_groups=1)
        self.dcn.conv_offset_mask.weight.data.normal_(0, 0.5)    # offsets well past 2 px
        self.dcn.conv_offset_mask.bias.data.normal_(0, 1.0)
        self.actf = nn.Sequential(nn.BatchNorm2d(32), nn.ReLU(inplace=True))
        self.hm = nn.Conv2d(32, 3, 1)
        self.wh = nn.Conv2d(32, 2, 1)
        self.reg = nn.Conv2d(32, 2, 1)
    def forward(self, x):
        y = self.actf(self.dcn(self.stem(x)))
        return self.hm(y), self.wh(y), self.reg(y)

def train(fmt):
    torch.manual_seed(7)
    net = Net().cuda().to(memory_format=fmt)
    opt = torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9)
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, W, M = 2, 32, 32, 8
    x = torch.randn(B, 3, H, W, device="cuda", generator=g).contiguous(memory_format=fmt)
    cls = torch.randint(0, 3, (B, M), device="cuda", generator=g)
    cx = torch.randint(0, W, (B, M), device="cuda", generator=g)
    cy = torch.randint(0, H, (B, M), device="cuda", generator=g)
    rad = torch.randint(0, 4, (B, M), device="cuda", generator=g)
    val = torch.ones(B, M, dtype=torch.uint8, device="cuda")
    ind = (cy * W + cx).long()
    msk = torch.ones(B, M, dtype=torch.uint8, device="cuda")
    wh_t = torch.rand(B, M, 2, device="cuda", generator=g) * 8
    reg_t = torch.rand(B, M, 2, device="cuda", generator=g)
    om = net.dcn.conv_offset_mask(net.stem(x))
    big = om[:, :18].abs().max().item()
    for _ in range(3):
        hm, wh, reg = net(x)
        loss = L.FocalSplatLoss(from_logits=True)(hm, cls, cx, cy, rad, val) + 0.1 * L.RegL1Loss()(wh, msk, ind, wh_t) \
            + L.RegL1Loss()(reg, msk, ind, reg_t)
        opt.zero_grad()
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    return [p.detach().clone() for p in net.parameters()], big

res = {}
for name, fmt in (("nchw", torch.contiguous_format), ("channels_last", torch.channels_last)):
    a, big = train(fmt)
    b, _ = train(fmt)
    res[name] = all(torch.equal(u, v) for u, v in zip(a, b))
    res[name + "_max_offset"] = big
    res[name + "_finite"] = all(bool(torch.isfinite(u).all()) for u in a)
print(json.dumps(res))
"""


def test_end_to_end_training_reproducible():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    env.pop("CNB_DCN_FP32", None)
    p = subprocess.run([sys.executable, "-c", "ROOT = %r\n" % ROOT + E2E], env=env, cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    for fmt in ("nchw", "channels_last"):
        assert res[fmt + "_max_offset"] > 2.0, res
        assert res[fmt + "_finite"], res
        assert res[fmt], (fmt, "parameters differ between two identical training runs")


def test_unsupported_configurations_raise_or_warn():
    """The fp32-only DCN backward (here: no workspace through the C ABI) and the PSROI backward have no deterministic
    implementation: RuntimeError under torch.use_deterministic_algorithms(True), a warning and a normal run under
    warn_only=True."""
    from centernet_b200._lib import C, ptr, stream_ptr
    from centernet_b200.dcn_v2_func import DCNv2PoolingFunction
    x, off, m, w, _, go = [t.cuda() for t in make(1, 16, 8, 8, 8, 1, 1, seed=67, off_scale=1.0)]
    grads = [torch.zeros_like(t) for t in (x, off, m, w)] + [torch.zeros(8, device="cuda")]
    C.dcnv2_set_deterministic(1)
    try:
        with pytest.raises(RuntimeError, match="deterministic"):
            C.dcnv2_backward(ptr(x), ptr(off), ptr(m), ptr(w), ptr(go), *[ptr(g) for g in grads], 1, 16, 8, 8, 8, 3, 3,
                             1, 1, 1, 1, 1, 1, 1, 0, 0, stream_ptr(x))
    finally:
        C.dcnv2_set_deterministic(0)

    data = torch.randn(1, 8, 12, 12, device="cuda")
    rois = torch.tensor([[0, 4.0, 4.0, 30.0, 30.0]], device="cuda")
    fn = DCNv2PoolingFunction(0.25, 2, 8, True, 1, 2, 2, 0.0)   # output_dim = channels (group size 1)

    def psroi_backward():
        d = data.clone().requires_grad_(True)
        fn(d, rois, d.new()).sum().backward()
        return d.grad

    try:
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="deterministic"):
            psroi_backward()
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.warns(UserWarning, match="deterministic"):
            gd = psroi_backward()
        assert torch.isfinite(gd).all() and gd.abs().sum() > 0
    finally:
        torch.use_deterministic_algorithms(False)


FP32_DCN = r"""
import sys, warnings, torch
sys.path.insert(0, ROOT)
from centernet_b200.dcn_v2_func import DCNv2Function
torch.use_deterministic_algorithms(True, warn_only=WARN_ONLY)
g = torch.Generator().manual_seed(1)
t = [torch.randn(1, 8, 10, 10, generator=g), torch.randn(1, 18, 10, 10, generator=g),
     torch.rand(1, 9, 10, 10, generator=g), torch.randn(4, 8, 3, 3, generator=g), torch.randn(4, generator=g)]
t = [v.cuda().requires_grad_(True) for v in t]
with warnings.catch_warnings(record=True) as rec:
    warnings.simplefilter("always")
    try:
        DCNv2Function(1, 1, 1, 1)(*t).sum().backward()
    except RuntimeError as e:
        print("RAISED", "deterministic" in str(e))
        sys.exit(0)
print("RAN", any("deterministic" in str(r.message) for r in rec), bool(torch.isfinite(t[0].grad).all()))
"""


@pytest.mark.parametrize("warn_only", [False, True])
def test_fp32_dcn_backward_under_deterministic_mode(warn_only):
    """CNB_DCN_FP32=1 selects the fp32 CUDA-core DCN, which has no deterministic backward."""
    env = dict(os.environ, CNB_DCN_FP32="1")
    p = subprocess.run([sys.executable, "-c", "ROOT = %r\nWARN_ONLY = %r\n" % (ROOT, warn_only) + FP32_DCN], env=env,
                       cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    assert p.stdout.split() == (["RAN", "True", "True"] if warn_only else ["RAISED", "True"]), p.stdout

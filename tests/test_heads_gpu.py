"""GPU: the fused bf16 output head (cnb_head_forward_bf16, centernet_b200.heads).

1. Exact grids: x in {-1, 0, 1}, at most 250 non-zero W1 entries (+-1) per head_conv channel and an integer b1, so every
   intermediate is an integer of magnitude <= 252 (exact in bf16); W2 in {-1, 0, 1}, b2 on a 1/4 grid, so every
   output has at most 18 significant bits (exact in fp32).  The fp32 output must EQUAL the fp64 oracle and the bf16
   output its RN rounding, for every head width, layout, input dtype and the border taps of odd map sizes.
2. Random data against a bound from sum |a * b| of the fp64 oracle at the bf16 operands (intermediate rounded as in
   the contract); the autocast module meets the same bound.
3. NaN / Inf inputs give the unfused module's NaN / Inf pattern; repeats are bit-identical.
4. fuse_heads on a model: the fused path, its fall-backs, the weight-tile cache and the ctdet decode on its bf16 hm."""
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from centernet_b200 import heads as H

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
DEV = "cuda"
WIDTHS = (1, 2, 3, 4, 5, 8, 17, 34, 80, 256)   # every ctdet / multi_pose / ddd / exdet head width, and the limit


def exact_case(B, cin, cmid, Hh, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-1, 2, (B, cin, Hh, W), generator=g).float()
    K = cin * 9
    w1 = torch.zeros(cmid, K)
    for o in range(cmid):
        idx = torch.randperm(K, generator=g)[:min(250, K)]
        w1[o, idx] = torch.randint(0, 2, (idx.numel(),), generator=g).float() * 2 - 1
    w1 = w1.view(cmid, cin, 3, 3)
    b1 = torch.randint(-2, 3, (cmid,), generator=g).float()
    return x, w1, b1, g


def oracle_mid(x, w1, b1):
    """fp64 3x3 conv + bias, ReLU, rounded to bf16 (through fp32)."""
    m = F.conv2d(x.double(), w1.double(), b1.double(), padding=1).clamp_min(0)
    return m.float().to(BF).double()


def oracle_out(mid, w2, b2):
    return F.conv2d(mid, w2.double()[:, :, None, None], b2.double())


def run(x, w1, b1, w2, b2, cl):
    x = x.contiguous(memory_format=torch.channels_last) if cl else x.contiguous()
    return H.head_forward_bf16(x, w1, b1, w2, b2)


EXACT = [   # (B, cin, head_conv, H, W)
    (1, 64, 256, 128, 128),
    (2, 64, 256, 96, 320),
    (64, 64, 256, 7, 13),
    (1, 256, 64, 128, 128),
    (64, 256, 64, 7, 13),
    (1, 64, 64, 96, 320),
    (1, 256, 256, 16, 24),
    (3, 32, 96, 9, 17),
    (2, 64, 160, 1, 1),
    (65, 64, 256, 17, 5),
]


@pytest.mark.parametrize("case", EXACT, ids=lambda c: "B%d_cin%d_hc%d_%dx%d" % c)
def test_exact_grid_bit_for_bit(case):
    B, cin, cmid, Hh, W = case
    x, w1, b1, g = exact_case(B, cin, cmid, Hh, W, seed=sum(case))
    xd, w1d, b1d = x.to(DEV), w1.to(DEV), b1.to(DEV)
    mid = oracle_mid(xd, w1d, b1d)
    for C in WIDTHS:
        w2 = torch.randint(-1, 2, (C, cmid), generator=g).float().to(DEV)
        b2 = (torch.randint(-8, 9, (C,), generator=g).float() / 4).to(DEV)
        want = oracle_out(mid, w2, b2)
        for dt in (torch.float32, BF):
            for cl in (False, True):
                y = run(xd.to(dt), w1d, b1d, w2.view(C, cmid, 1, 1), b2, cl)
                assert y.dtype == dt and y.shape == (B, C, Hh, W)
                if cl and Hh * W > 1:
                    assert y.is_contiguous(memory_format=torch.channels_last)
                else:
                    assert y.is_contiguous()
                ref = want.float() if dt == torch.float32 else want.float().to(BF)
                assert torch.equal(y, ref), (C, dt, cl, (y.double() - ref.double()).abs().max().item())


def _bound(xb, w1b, b1, w2b, b2, mid64, bf16_out):
    cin, cmid = w1b.shape[1], w1b.shape[0]
    s1 = F.conv2d(xb.abs(), w1b.abs(), b1.abs(), padding=1)
    e1 = 9 * cin * 2.0 ** -22 * s1                       # fp32 accumulation of GEMM 1
    dmid = e1 + 2.0 ** -7 * (mid64.clamp_min(0) + e1)   # plus one bf16 ulp where the rounding goes the other way
    midr = mid64.clamp_min(0).float().to(BF).double()
    w2a = w2b.abs()[:, :, None, None]
    s2 = F.conv2d(midr + dmid, w2a, b2.abs())
    out64 = F.conv2d(midr, w2b[:, :, None, None], b2)
    bound = F.conv2d(dmid, w2a) + cmid * 2.0 ** -22 * s2
    if bf16_out:
        bound = bound + 2.0 ** -8 * (out64.abs() + bound)
    return out64, bound + 1e-6


@pytest.mark.parametrize("case", [(2, 64, 256, 80, 128, 128), (3, 256, 64, 34, 96, 320), (8, 64, 256, 2, 7, 13)],
                         ids=lambda c: "B%d_cin%d_hc%d_C%d_%dx%d" % c)
def test_random_within_bound_and_autocast_too(case):
    B, cin, cmid, C, Hh, W = case
    g = torch.Generator().manual_seed(7 + C)
    x = torch.randn(B, cin, Hh, W, generator=g).to(DEV)
    head = nn.Sequential(nn.Conv2d(cin, cmid, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(cmid, C, 1)).to(DEV)
    xb, w1b = x.to(BF).double(), head[0].weight.to(BF).double()
    w2b = head[2].weight.to(BF).double().view(C, cmid)
    b1, b2 = head[0].bias.double(), head[2].bias.double()
    mid64 = F.conv2d(xb, w1b, b1, padding=1)
    with torch.no_grad():
        for dt in (torch.float32, BF):
            out64, bound = _bound(xb, w1b, b1, w2b, b2, mid64, dt == BF)
            for cl in (False, True):
                y = run(x.to(dt), head[0].weight, head[0].bias, head[2].weight, head[2].bias, cl)
                err = (y.double() - out64).abs()
                assert bool((err <= bound).all()), (dt, cl, (err - bound).max().item())
        out64, bound = _bound(xb, w1b, b1, w2b, b2, mid64, True)
        with torch.autocast("cuda", dtype=BF):
            ya = head(x)
        err = (ya.double() - out64).abs()
        assert bool((err <= bound).all()), (err - bound).max().item()


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_input_pattern(bad):
    g = torch.Generator().manual_seed(3)
    head = nn.Sequential(nn.Conv2d(64, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 80, 1))
    x = torch.randn(2, 64, 13, 19, generator=g)
    x[0, 5, 0, 0] = bad          # a corner: border taps
    x[1, 17, 6, 9] = bad
    x[1, 40, 12, 18] = bad
    with torch.no_grad():
        ref = nn.Sequential(*[m for m in head]).double()
        for p in ref.parameters():
            p.copy_(p.to(BF).double())
        want = ref(x.to(BF).double())
        for dt in (torch.float32, BF):
            for cl in (False, True):
                y = run(x.to(DEV, dt), head[0].weight.to(DEV), head[0].bias.to(DEV), head[2].weight.to(DEV),
                        head[2].bias.to(DEV), cl).cpu()
                assert torch.equal(torch.isnan(y), torch.isnan(want)), (dt, cl)
                assert torch.equal(torch.isposinf(y), torch.isposinf(want)), (dt, cl)
                assert torch.equal(torch.isneginf(y), torch.isneginf(want)), (dt, cl)
                assert bool(torch.isnan(want).any() or torch.isinf(want).any())


def test_repeat_is_bit_identical():
    g = torch.Generator().manual_seed(11)
    x = torch.randn(8, 64, 128, 128, generator=g).to(DEV, BF).contiguous(memory_format=torch.channels_last)
    head = nn.Sequential(nn.Conv2d(64, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 80, 1)).to(DEV)
    a = run(x, head[0].weight, head[0].bias, head[2].weight, head[2].bias, True)
    b = run(x, head[0].weight, head[0].bias, head[2].weight, head[2].bias, True)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


class _Net(nn.Module):
    def __init__(self, heads, head_conv=256, cin=64):
        super().__init__()
        self.heads = heads
        for name, c in heads.items():
            fc = nn.Sequential(nn.Conv2d(cin, head_conv, 3, padding=1, bias=True), nn.ReLU(inplace=True),
                               nn.Conv2d(head_conv, c, 1, stride=1, padding=0, bias=True))
            if "hm" in name:
                fc[-1].bias.data.fill_(-2.19)
            self.__setattr__(name, fc)

    def forward(self, y):
        return {h: self.__getattr__(h)(y) for h in self.heads}


def test_fuse_heads_model_paths_and_tile_cache():
    torch.manual_seed(0)
    net = _Net({"hm": 80, "wh": 2, "reg": 2}).to(DEV).eval()
    x = torch.randn(2, 64, 32, 48, device=DEV)
    with torch.no_grad():
        ref = {k: H.head_forward_bf16(x, m[0].weight, m[0].bias, m[2].weight, m[2].bias)
               for k, m in ((h, getattr(net, h)) for h in net.heads)}
        plain = net(x)
    assert H.fuse_heads(net) == 3
    with torch.no_grad():
        got = net(x)
        for k in ref:
            assert torch.equal(got[k], ref[k]), k
        # a weight update in place invalidates the cached tiles
        net.hm[0].weight.mul_(0.5)
        want = H.head_forward_bf16(x, net.hm[0].weight, net.hm[0].bias, net.hm[2].weight, net.hm[2].bias)
        assert torch.equal(net(x)["hm"], want)
        net.hm[0].weight.mul_(2.0)
    # grad enabled with parameters that require it: the original three layers, bit for bit
    got = net(x)
    for k in plain:
        assert torch.equal(got[k], plain[k]), k
        assert got[k].requires_grad
    # CPU tensors: the original path
    cpu = _Net({"hm": 4}).eval()
    xc = torch.randn(1, 64, 8, 8)
    with torch.no_grad():
        a = cpu(xc)["hm"]
        H.fuse_heads(cpu)
        assert torch.equal(cpu(xc)["hm"], a)


def test_ctdet_decode_on_fused_bf16_hm():
    from centernet_b200.decode import ctdet_decode_from_logits
    torch.manual_seed(1)
    net = _Net({"hm": 80, "wh": 2, "reg": 2}).to(DEV).eval()
    H.fuse_heads(net)
    x = (torch.randn(4, 64, 128, 128, device=DEV) * 2).to(BF).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        out = net(x)
    assert out["hm"].dtype == BF
    a = ctdet_decode_from_logits(out["hm"], out["wh"], out["reg"], K=100)
    b = ctdet_decode_from_logits(out["hm"].float(), out["wh"].float(), out["reg"].float(), K=100)
    assert torch.equal(a, b)

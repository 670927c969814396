"""GPU: float64 DCNv2 and deformable PSROI pooling (the reference's dcn_v2_double build).

The reference's own check (DCNv2/test.py:67-90, gradcheck in float64 with the default nondet_tol=0, i.e. the
backward must repeat bit for bit), its zero-offset known answer at its float64 bound, parity with the fp64
restatements (oracle/dcn_ref.py, and a float64 restatement of dcn_v2_psroi_pooling_cuda_double.cu below),
parity of both with stored outputs of the reference's own float64 kernels (tests/golden/ref_gpu_f64.npz),
reproducibility across runs and batch splits, and the dtype rules."""
import math
import os
import warnings

import numpy as np
import pytest
import torch
from torch.autograd import gradcheck

from oracle import dcn_ref

pytestmark = pytest.mark.gpu

D = torch.float64


def _dcn_inputs(N, inC, H, W, outC, kh, kw, dg, stride=1, pad=1, dil=1, seed=0, off_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    Ho = (H + 2 * pad - (dil * (kh - 1) + 1)) // stride + 1
    Wo = (W + 2 * pad - (dil * (kw - 1) + 1)) // stride + 1
    x = torch.randn(N, inC, H, W, generator=g, dtype=D)
    off = torch.randn(N, dg * 2 * kh * kw, Ho, Wo, generator=g, dtype=D) * off_scale
    m = torch.rand(N, dg * kh * kw, Ho, Wo, generator=g, dtype=D)
    w = torch.randn(outC, inC, kh, kw, generator=g, dtype=D)
    b = torch.rand(outC, generator=g, dtype=D)
    return x, off, m, w, b


# ------------------------------------------------------------------ 1. the reference's gradcheck
GRADCHECK = [
    # N, inC, H, W, outC, kh, kw, dg, stride, pad, dil
    (2, 2, 4, 4, 2, 3, 3, 1, 1, 1, 1),      # DCNv2/test.py:67-90 exactly
    (2, 4, 4, 4, 2, 3, 3, 2, 1, 1, 1),      # deformable_groups = 2
    (2, 2, 6, 6, 3, 3, 3, 1, 2, 1, 1),      # stride 2
    (2, 2, 6, 6, 2, 3, 3, 1, 1, 2, 2),      # dilation 2
    (1, 2, 5, 5, 2, 5, 5, 1, 1, 2, 1),      # 5x5 kernel
    (2, 2, 4, 7, 3, 3, 3, 1, 1, 1, 1),      # non-square image
]


@pytest.mark.parametrize("N,inC,H,W,outC,kh,kw,dg,stride,pad,dil", GRADCHECK)
def test_reference_gradcheck_double(N, inC, H, W, outC, kh, kw, dg, stride, pad, dil):
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = [t.cuda().requires_grad_(True) for t in _dcn_inputs(N, inC, H, W, outC, kh, kw, dg, stride, pad,
                                                                          dil, seed=1)]
    mask = torch.sigmoid(m)          # test.py:80
    func = DCNv2Function(stride=stride, padding=pad, dilation=dil, deformable_groups=dg)
    assert gradcheck(func, (x, off, mask, w, b), eps=1e-6, atol=1e-5, rtol=1e-3)


def _dpool_case(trans_std, seed):
    g = torch.Generator().manual_seed(seed)
    if trans_std == 0.0:    # DCNv2/test.py:148-166
        inp = torch.randn(2, 3, 5, 5, generator=g, dtype=D) * 0.01
        N = 4
        bi = torch.randint(2, (N, 1), generator=g).to(D)
        x = torch.rand((N, 1), generator=g, dtype=D) * 15
        y = torch.rand((N, 1), generator=g, dtype=D) * 15
        w = torch.rand((N, 1), generator=g, dtype=D) * 10
        h = torch.rand((N, 1), generator=g, dtype=D) * 10
    else:                   # boxes inside the map, so that no shifted sample is clamped to the border
        inp = torch.randn(2, 3, 12, 12, generator=g, dtype=D)
        N = 4
        bi = torch.randint(2, (N, 1), generator=g).to(D)
        x = 14 + torch.rand((N, 1), generator=g, dtype=D) * 4
        y = 14 + torch.rand((N, 1), generator=g, dtype=D) * 4
        w = 4 + torch.rand((N, 1), generator=g, dtype=D) * 8
        h = 4 + torch.rand((N, 1), generator=g, dtype=D) * 8
    rois = torch.cat((bi, x, y, x + w, y + h), dim=1)
    offset = torch.randn(N, 2, 3, 3, generator=g, dtype=D)
    return inp, rois, offset


@pytest.mark.parametrize("trans_std", [0.0, 0.1])
def test_reference_gradcheck_dpooling_double(trans_std):
    from centernet_b200.dcn_v2 import DCNv2Pooling
    inp, rois, offset = _dpool_case(trans_std, seed=5)
    inp, rois, offset = inp.cuda().requires_grad_(True), rois.cuda(), offset.cuda().requires_grad_(True)
    dpooling = DCNv2Pooling(spatial_scale=1.0 / 4, pooled_size=3, output_dim=3, no_trans=False, group_size=1,
                            trans_std=trans_std).cuda()
    assert gradcheck(dpooling, (inp, rois, offset), eps=1e-6, atol=1e-5, rtol=1e-3)


# ------------------------------------------------------------------ 2. zero-offset known answer
def kat_inputs():
    """DCNv2/test.py:32-65 in float64: identity weights (conv_identify, :21-30), zero offsets, mask sigmoid(0)."""
    N, inC, outC = 2, 2, 2
    x = torch.randn(N, inC, 4, 4, generator=torch.Generator().manual_seed(11), dtype=D)
    w = torch.zeros(outC, inC, 3, 3, dtype=D)
    for q in range(outC):
        w[q, q % inC, 1, 1] = 1.0
    return x, torch.zeros(N, 18, 4, 4, dtype=D), torch.full((N, 9, 4, 4), 0.5, dtype=D), w, torch.zeros(outC, dtype=D)


def test_zero_offset_known_answer_double():
    """DCNv2/test.py:32-65 in float64 through the DCNv2 module, held to its bound d < 1e-10."""
    from centernet_b200.dcn_v2 import DCNv2
    x, off, mask, w, b = [t.cuda() for t in kat_inputs()]
    dcn = DCNv2(2, 2, (3, 3), stride=1, padding=1, dilation=1, deformable_groups=1).cuda().double()
    with torch.no_grad():
        dcn.weight.copy_(w)
        dcn.bias.copy_(b)
    out = dcn(x, off, mask) * 2
    assert out.dtype == D
    assert (x - out).abs().max().item() < 1e-10


# ------------------------------------------------------------------ 3. parity with the fp64 oracle
LAYERS = [
    (2, 64, 128, 128, 64, 1, 1), (2, 128, 64, 64, 128, 1, 1), (2, 256, 32, 32, 256, 1, 1),
    (2, 512, 16, 16, 256, 1, 1), (2, 128, 64, 64, 64, 1, 1), (2, 256, 32, 32, 128, 1, 1),
    (2, 64, 32, 32, 64, 2, 1), (2, 12, 9, 11, 5, 2, 1), (2, 6, 10, 14, 7, 1, 2),
]
BWD_LAYERS = [(2, 64, 64, 64, 64, 1, 1), (2, 128, 32, 32, 128, 1, 1), (2, 256, 16, 16, 256, 1, 1),
              (1, 512, 16, 16, 256, 1, 1), (2, 64, 16, 16, 64, 2, 1), (1, 12, 9, 11, 5, 2, 1), (2, 6, 10, 14, 7, 1, 2)]


def _layer(B, Ci, H, W, Co, dg, stride, seed):
    x, off, m, w, b = _dcn_inputs(B, Ci, H, W, Co, 3, 3, dg, stride, seed=seed, off_scale=2.0)
    return x, off, torch.sigmoid(m), w / (3.0 * Ci ** 0.5), b


def _close(got, want, rel):
    scale = want.abs().max().item()
    err = (got.detach().cpu() - want.detach()).abs().max().item()
    assert err <= rel * max(scale, 1e-300), "max err %.3e vs %.1e * %.3e" % (err, rel, scale)


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", LAYERS)
def test_forward_vs_fp64_oracle(B, Ci, H, W, Co, dg, stride):
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = _layer(B, Ci, H, W, Co, dg, stride, seed=0)
    got = DCNv2Function(stride, 1, 1, dg)(*[t.cuda() for t in (x, off, m, w, b)])
    assert got.dtype == D
    _close(got, dcn_ref.dcn_v2_forward(x, off, m, w, b, stride, 1, 1, dg), 1e-11)


GRAD_NAMES = ("input", "offset", "mask", "weight", "bias")


def bwd_inputs(case):
    B, Ci, H, W, Co, dg, stride = case
    x, off, m, w, b = _layer(*case, seed=3)
    go = torch.randn(B, Co, (H - 1) // stride + 1, (W - 1) // stride + 1, generator=torch.Generator().manual_seed(9),
                     dtype=D)
    return x, off, m, w, b, go


def _our_grads(case, x, off, m, w, b, go):
    from centernet_b200.dcn_v2_func import DCNv2Function
    cu = [t.cuda().requires_grad_(True) for t in (x, off, m, w, b)]
    (DCNv2Function(case[-1], 1, 1, case[-2])(*cu) * go.cuda()).sum().backward()
    for t in cu:
        assert t.grad.dtype == D
    return [t.grad for t in cu]


def _oracle_grads(case, x, off, m, w, b, go):
    leaves = [t.clone().requires_grad_(True) for t in (x, off, m, w, b)]
    (dcn_ref.dcn_v2_forward(*leaves, case[-1], 1, 1, case[-2]) * go).sum().backward()
    return [t.grad for t in leaves]


@pytest.mark.parametrize("case", BWD_LAYERS)
def test_backward_vs_fp64_oracle(case):
    inputs = bwd_inputs(case)
    for name, a, r in zip(GRAD_NAMES, _our_grads(case, *inputs), _oracle_grads(case, *inputs)):
        _close(a, r, 1e-10)


# float64 restatement of dcn_v2_psroi_pooling_cuda_double.cu (forward :61-148, backward :150-270)
def _psroi64(data, rois, trans, no_trans, spatial_scale, output_dim, group_size, pooled_size, part_size,
             sample_per_part, trans_std, grad_out=None):
    B, C, H, W = data.shape
    N, P = rois.shape[0], pooled_size
    ncls = 1 if no_trans else trans.shape[1] // 2
    each = output_dim if no_trans else output_dim // ncls
    out = np.zeros((N, output_dim, P, P))
    cnt = np.zeros((N, output_dim, P, P))
    gd = np.zeros(data.shape)
    gt = None if no_trans else np.zeros(trans.shape)
    rnd = lambda v: math.floor(abs(v) + 0.5) * (1 if v >= 0 else -1)   # C round()
    for n in range(N):
        bi = int(rois[n, 0])
        sw = rnd(rois[n, 1]) * spatial_scale - 0.5
        sh = rnd(rois[n, 2]) * spatial_scale - 0.5
        ew = (rnd(rois[n, 3]) + 1.) * spatial_scale - 0.5
        eh = (rnd(rois[n, 4]) + 1.) * spatial_scale - 0.5
        rw, rh = max(ew - sw, 0.1), max(eh - sh, 0.1)
        bw, bh = rw / P, rh / P
        subw, subh = bw / sample_per_part, bh / sample_per_part
        for ctop in range(output_dim):
            cls = ctop // each
            for ph in range(P):
                for pw in range(P):
                    part_h = math.floor(ph / P * part_size)
                    part_w = math.floor(pw / P * part_size)
                    tx = 0.0 if no_trans else trans[n, cls * 2, part_h, part_w] * trans_std
                    ty = 0.0 if no_trans else trans[n, cls * 2 + 1, part_h, part_w] * trans_std
                    ws = pw * bw + sw + tx * rw
                    hs = ph * bh + sh + ty * rh
                    gw = min(max(math.floor(pw * group_size / P), 0), group_size - 1)
                    gh = min(max(math.floor(ph * group_size / P), 0), group_size - 1)
                    c = (ctop * group_size + gh) * group_size + gw
                    pl = data[bi, c]
                    samples = []
                    for ih in range(sample_per_part):
                        for iw in range(sample_per_part):
                            w = ws + iw * subw
                            h = hs + ih * subh
                            if w < -0.5 or w > W - 0.5 or h < -0.5 or h > H - 0.5:
                                continue
                            samples.append((min(max(w, 0.), W - 1.), min(max(h, 0.), H - 1.)))
                    s = 0.0
                    for w, h in samples:
                        x0, x1, y0, y1 = math.floor(w), math.ceil(w), math.floor(h), math.ceil(h)
                        dx, dy = w - x0, h - y0
                        s += (1 - dx) * (1 - dy) * pl[y0, x0] + (1 - dx) * dy * pl[y1, x0] + \
                            dx * (1 - dy) * pl[y0, x1] + dx * dy * pl[y1, x1]
                    k = len(samples)
                    out[n, ctop, ph, pw] = 0.0 if k == 0 else s / k
                    cnt[n, ctop, ph, pw] = k
                    if grad_out is None or k == 0:
                        continue
                    dv = grad_out[n, ctop, ph, pw] / k
                    for w, h in samples:
                        x0, x1, y0, y1 = math.floor(w), math.ceil(w), math.floor(h), math.ceil(h)
                        dx, dy = w - x0, h - y0
                        gd[bi, c, y0, x0] += (1 - dx) * (1 - dy) * dv
                        gd[bi, c, y1, x0] += (1 - dx) * dy * dv
                        gd[bi, c, y0, x1] += dx * (1 - dy) * dv
                        gd[bi, c, y1, x1] += dx * dy * dv
                        if no_trans:
                            continue
                        u00, u01, u10, u11 = pl[y0, x0], pl[y1, x0], pl[y0, x1], pl[y1, x1]
                        gt[n, cls * 2, part_h, part_w] += \
                            (u11 * dy + u10 * (1 - dy) - u01 * dy - u00 * (1 - dy)) * trans_std * dv * rw
                        gt[n, cls * 2 + 1, part_h, part_w] += \
                            (u11 * dx + u01 * (1 - dx) - u10 * dx - u00 * (1 - dx)) * trans_std * dv * rh
    return out, cnt, gd, gt


PS_CASES = [   # seed, B, C, H, W, N, output_dim, group, pooled, part, spp, classes, trans_std, no_trans
    (1, 2, 8, 9, 9, 5, 2, 2, 3, 3, 2, 2, 0.1, False),
    (2, 2, 18, 12, 10, 6, 2, 3, 4, 2, 3, 1, 0.3, False),
    (3, 1, 4, 7, 7, 4, 4, 1, 3, 3, 4, 2, 0.0, False),
    (4, 3, 16, 16, 16, 7, 16, 1, 7, 7, 4, 1, 0.1, True),
    (5, 2, 98, 20, 24, 12, 2, 7, 7, 7, 4, 1, 0.1, False),
]


def _ps_case(seed, B, C, H, W, N, output_dim, group, pooled, part, spp, classes, trans_std, no_trans):
    rng = np.random.default_rng(seed)
    data = rng.standard_normal((B, C, H, W))
    x = rng.uniform(-6, W * 4 - 8, N); y = rng.uniform(-6, H * 4 - 8, N)
    w = rng.uniform(1, W * 3, N); h = rng.uniform(1, H * 3, N)
    rois = np.stack([rng.integers(0, B, N).astype(np.float64), x, y, x + w, y + h], 1)
    trans = None if no_trans else rng.standard_normal((N, 2 * classes, part, part))
    cfg = dict(no_trans=no_trans, spatial_scale=0.25, output_dim=output_dim, group_size=group, pooled_size=pooled,
               part_size=part, sample_per_part=spp, trans_std=trans_std)
    return data, rois, trans, cfg


def ps_grad(shape):
    return np.random.default_rng(9).standard_normal(shape)


def _ps_fn(cfg):
    from centernet_b200.dcn_v2_func import DCNv2PoolingFunction
    return DCNv2PoolingFunction(cfg["spatial_scale"], cfg["pooled_size"], cfg["output_dim"], cfg["no_trans"],
                                cfg["group_size"], cfg["part_size"], cfg["sample_per_part"], cfg["trans_std"])


@pytest.mark.parametrize("case", PS_CASES)
def test_psroi_vs_fp64_restatement(case):
    data, rois, trans, cfg = _ps_case(*case)
    d = torch.from_numpy(data).cuda().requires_grad_(True)
    t = d.new() if trans is None else torch.from_numpy(trans).cuda().requires_grad_(True)
    out = _ps_fn(cfg)(d, torch.from_numpy(rois).cuda(), t)
    assert out.dtype == D
    go = ps_grad(tuple(out.shape))
    want, cnt, gd, gt = _psroi64(data, rois, trans, grad_out=go, **cfg)
    _close(out, torch.from_numpy(want), 1e-11)
    out.backward(torch.from_numpy(go).cuda())
    assert d.grad.dtype == D
    _close(d.grad, torch.from_numpy(gd), 1e-10)
    if trans is not None:
        _close(t.grad, torch.from_numpy(gt), 1e-10)


# ------------------------------------------------------------------ 4. parity with the reference's float64 kernels
# tests/golden/ref_gpu_f64.npz: outputs of the reference's own dcn_v2_double kernels (dcn_v2_im2col_cuda_double.cu,
# dcn_v2_psroi_pooling_cuda_double.cu compiled unmodified, oracle/build_ref_f64.py), made on an H100 by
# tests/golden/make_golden_ref_gpu_f64.py from the inputs rebuilt here (a seeded sample of 1024 positions per large
# tensor).  Our kernels and the fp64 restatements are each held to it.
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_gpu_f64.npz")
_G = None


def key(kind, case):
    return kind + "_" + "_".join(str(v) for v in case)


def ref(k):
    """(flat positions, reference values there, reference max |value|) of the stored tensor `k`."""
    global _G
    if _G is None:
        _G = np.load(GOLDEN)
    return _G[k + "/idx"], _G[k + "/val"], float(_G[k + "/absmax"])


def _pinned(t, k, rel):
    idx, val, amax = ref(k)
    got = (t.detach().cpu() if torch.is_tensor(t) else torch.from_numpy(np.asarray(t))).double().reshape(-1).numpy()[idx]
    err = np.abs(got - val).max() if idx.size else 0.0
    assert err <= rel * max(amax, 1e-300), "%s: max err %.3e vs %.1e * %.3e" % (k, err, rel, amax)


def test_reference_kat_pinned():
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, mask, w, b = [t.cuda() for t in kat_inputs()]
    _pinned(DCNv2Function(1, 1)(x, off, mask, w, b) * 2, "kat", 1e-11)
    _pinned(dcn_ref.dcn_v2_forward(*kat_inputs()) * 2, "kat", 1e-11)


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", LAYERS)
def test_forward_pinned_to_reference_f64(B, Ci, H, W, Co, dg, stride):
    from centernet_b200.dcn_v2_func import DCNv2Function
    case = (B, Ci, H, W, Co, dg, stride)
    x, off, m, w, b = _layer(*case, seed=0)
    _pinned(DCNv2Function(stride, 1, 1, dg)(*[t.cuda() for t in (x, off, m, w, b)]), key("fwd", case), 1e-11)
    _pinned(dcn_ref.dcn_v2_forward(x, off, m, w, b, stride, 1, 1, dg), key("fwd", case), 1e-11)


@pytest.mark.parametrize("case", BWD_LAYERS)
def test_backward_pinned_to_reference_f64(case):
    inputs = bwd_inputs(case)
    for name, a, r in zip(GRAD_NAMES, _our_grads(case, *inputs), _oracle_grads(case, *inputs)):
        _pinned(a, key("bwd_" + name, case), 1e-10)
        _pinned(r, key("bwd_" + name, case), 1e-10)


@pytest.mark.parametrize("case", PS_CASES)
def test_psroi_pinned_to_reference_f64(case):
    data, rois, trans, cfg = _ps_case(*case)
    d = torch.from_numpy(data).cuda().requires_grad_(True)
    t = d.new() if trans is None else torch.from_numpy(trans).cuda().requires_grad_(True)
    out = _ps_fn(cfg)(d, torch.from_numpy(rois).cuda(), t)
    go = ps_grad(tuple(out.shape))
    out.backward(torch.from_numpy(go).cuda())
    want, cnt, gd, gt = _psroi64(data, rois, trans, grad_out=go, **cfg)
    c = case[:1]
    assert ref(key("ps_cnt", c))[2] > 0      # the stored reference pass did sample
    _pinned(out, key("ps_out", c), 1e-11)
    _pinned(want, key("ps_out", c), 1e-11)
    _pinned(cnt, key("ps_cnt", c), 0.0)
    _pinned(d.grad, key("ps_gi", c), 1e-10)
    _pinned(gd, key("ps_gi", c), 1e-10)
    if trans is not None:
        _pinned(t.grad, key("ps_gt", c), 1e-10)
        _pinned(gt, key("ps_gt", c), 1e-10)


# ------------------------------------------------------------------ 5. reproducibility
def _grads(x, off, m, w, b):
    from centernet_b200.dcn_v2_func import DCNv2Function
    leaves = [t.clone().requires_grad_(True) for t in (x, off, m, w, b)]
    y = DCNv2Function(1, 1, 1, 1)(*leaves)
    go = torch.randn(y.shape, generator=torch.Generator().manual_seed(21), dtype=D).cuda()
    y.backward(go[: y.shape[0]])
    return [t.grad for t in leaves]


def test_backward_bit_reproducible_and_batch_invariant():
    x, off, m, w, b = [t.cuda() for t in _dcn_inputs(3, 64, 64, 64, 64, 3, 3, 1, seed=7, off_scale=2.0)]
    w = w / 24.0
    g1 = _grads(x, off, m, w, b)
    g2 = _grads(x, off, m, w, b)
    for a, c in zip(g1, g2):
        assert torch.equal(a, c)
    # each image alone gets the bits it gets inside the batch (grad_input, grad_offset, grad_mask)
    from centernet_b200.dcn_v2_func import DCNv2Function
    go = torch.randn(3, 64, 64, 64, generator=torch.Generator().manual_seed(21), dtype=D).cuda()
    full = [t.clone().requires_grad_(True) for t in (x, off, m)]
    DCNv2Function(1, 1, 1, 1)(*full, w, b).backward(go)
    for i in range(3):
        one = [t[i:i + 1].clone().requires_grad_(True) for t in (x, off, m)]
        DCNv2Function(1, 1, 1, 1)(*one, w, b).backward(go[i:i + 1])
        for a, c in zip(full, one):
            assert torch.equal(a.grad[i:i + 1], c.grad)


def test_psroi_backward_bit_reproducible():
    data, rois, trans, cfg = _ps_case(*PS_CASES[4])
    grads = []
    for _ in range(2):
        d = torch.from_numpy(data).cuda().requires_grad_(True)
        t = torch.from_numpy(trans).cuda().requires_grad_(True)
        out = _ps_fn(cfg)(d, torch.from_numpy(rois).cuda(), t)
        out.backward(torch.ones_like(out))
        grads.append((d.grad, t.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


def test_nonfinite_grad_output_gives_nan_grad_input_of_that_image_only():
    x, off, m, w, b = [t.cuda() for t in _dcn_inputs(2, 8, 9, 9, 4, 3, 3, 1, seed=2)]
    from centernet_b200.dcn_v2_func import DCNv2Function
    xi = x.clone().requires_grad_(True)
    y = DCNv2Function(1, 1, 1, 1)(xi, off, m, w, b)
    go = torch.ones_like(y)
    go[1, 0, 0, 0] = float("inf")
    y.backward(go)
    assert torch.isnan(xi.grad[1]).all() and torch.isfinite(xi.grad[0]).all()


# ------------------------------------------------------------------ 6. dtypes
def test_dtypes_modules_and_mixing():
    from centernet_b200.dcn_v2 import DCN, DCNv2, DCNv2Pooling
    from centernet_b200.dcn_v2_func import DCNv2Function, dcn_fused_inference
    torch.manual_seed(0)
    x = torch.randn(2, 8, 10, 10, dtype=D, device="cuda", requires_grad=True)
    dcn = DCN(8, 4, 3, 1, 1).cuda().double()
    with torch.no_grad():
        dcn.conv_offset_mask.weight.normal_(0, 0.1)
    y = dcn(x)
    assert y.dtype == D
    y.sum().backward()
    assert x.grad.dtype == D and dcn.weight.grad.dtype == D and dcn.conv_offset_mask.weight.grad.dtype == D
    with torch.no_grad():
        y2 = dcn(x)
    assert y2.dtype == D and torch.equal(y2, y.detach())
    v2 = DCNv2(8, 4, 3, 1, 1).cuda().double()
    off = torch.randn(2, 18, 10, 10, dtype=D, device="cuda")
    msk = torch.rand(2, 9, 10, 10, dtype=D, device="cuda")
    assert v2(x, off, msk).dtype == D
    with pytest.raises(RuntimeError, match="float64"):
        v2(x, off.float(), msk)
    with pytest.raises(RuntimeError, match="float64"):
        DCNv2Function(1, 1)(x, off, msk, v2.weight.float(), v2.bias)
    with pytest.raises(NotImplementedError):
        dcn_fused_inference(x, torch.zeros(2, 27, 10, 10, dtype=D, device="cuda"), v2.weight, v2.bias, 1, 1, 1, 1)
    pool = DCNv2Pooling(0.25, 3, 4, False, group_size=1, trans_std=0.1).cuda()
    rois = torch.tensor([[0, 4, 4, 30, 30], [1, 2, 6, 20, 36]], device="cuda")
    data = torch.randn(2, 4, 10, 10, dtype=D, device="cuda", requires_grad=True)
    pt = torch.zeros(2, 2, 3, 3, dtype=D, device="cuda", requires_grad=True)
    for r in (rois.float(), rois.double()):
        out = pool(data, r, pt)
        assert out.dtype == D
        out.sum().backward()
        assert data.grad.dtype == D and pt.grad.dtype == D
    with pytest.raises(RuntimeError, match="float64"):
        pool(data, rois.float(), pt.float())


def test_deterministic_algorithms_run_without_warnings():
    from centernet_b200.dcn_v2 import DCNv2Pooling
    from centernet_b200.dcn_v2_func import DCNv2Function
    x, off, m, w, b = [t.cuda().requires_grad_(True) for t in _dcn_inputs(2, 4, 6, 6, 3, 3, 3, 1, seed=4)]
    data, rois, trans, cfg = _ps_case(*PS_CASES[0])
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            DCNv2Function(1, 1, 1, 1)(x, off, m, w, b).sum().backward()
            d = torch.from_numpy(data).cuda().requires_grad_(True)
            t = torch.from_numpy(trans).cuda().requires_grad_(True)
            _ps_fn(cfg)(d, torch.from_numpy(rois).cuda(), t).sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert x.grad is not None and d.grad is not None and t.grad is not None

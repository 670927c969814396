"""GPU: everything DCNv2 / deformable-PSROI pinned to THE REFERENCE ITSELF -- tests/golden/ref_gpu.npz holds
outputs of the reference's own two .cu files, compiled unmodified for sm_90a (oracle/build_ref.py) under a cuBLAS
restatement of the THC host loop (oracle/ref_host.cu), run on an H100 by tests/golden/make_golden_ref_gpu.py
on the seeded inputs rebuilt here (large tensors: a fixed sample of 1024 positions).  Three-way: the fp64
restatement (oracle/dcn_ref.py), the numpy restatement (oracle/psroi_np.py) and our kernels are each held to it.
Tolerances: forward <= 1e-4 abs (north_star), backward at DCNv2/test.py:90,115 (atol 1e-3, scaled)."""
import os

import numpy as np
import pytest
import torch

from oracle import dcn_ref, psroi_np

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_gpu.npz")
GRAD_NAMES = ("input", "offset", "mask", "weight", "bias")


def make(B, Ci, H, W, Co, dg, stride=1, seed=0, off_scale=2.0):
    g = torch.Generator().manual_seed(seed)
    Ho = (H + 2 - 3) // stride + 1
    Wo = (W + 2 - 3) // stride + 1
    x = torch.randn(B, Ci, H, W, generator=g)
    off = torch.randn(B, 18 * dg, Ho, Wo, generator=g) * off_scale
    m = torch.sigmoid(torch.randn(B, 9 * dg, Ho, Wo, generator=g))
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (3.0 * Ci ** 0.5)
    b = torch.randn(Co, generator=g)
    return x, off, m, w, b


def make_bwd(B, Ci, H, W, Co, dg, stride):
    x, off, m, w, b = make(B, Ci, H, W, Co, dg, stride, seed=3, off_scale=1.3)
    Ho = (H + 2 - 3) // stride + 1; Wo = (W + 2 - 3) // stride + 1
    go = torch.randn(B, Co, Ho, Wo, generator=torch.Generator().manual_seed(9))
    return x, off, m, w, b, go


def kat_input():
    return torch.randn(2, 2, 4, 4, generator=torch.Generator().manual_seed(11))


def key(kind, case):
    return kind + "_" + "_".join(str(v) for v in case)


_G = None


def ref(k):
    """(flat positions, reference values there, reference max |value|) of the stored tensor `k`."""
    global _G
    if _G is None:
        _G = np.load(GOLDEN)
    return _G[k + "/idx"], _G[k + "/val"], float(_G[k + "/absmax"])


def at(t, idx):
    return t.detach().reshape(-1).cpu().numpy()[idx]


# BASELINE configs[1] (dla_34 512x512) DCN layer shapes (SURVEY 3.2) + odd / strided / grouped cases
LAYERS = [
    # B, Cin, H, W, Cout, dg, stride
    (2, 64, 128, 128, 64, 1, 1),
    (2, 128, 64, 64, 128, 1, 1),
    (2, 256, 32, 32, 256, 1, 1),
    (2, 512, 16, 16, 256, 1, 1),
    (2, 128, 64, 64, 64, 1, 1),
    (2, 256, 32, 32, 128, 1, 1),
    (2, 64, 32, 32, 64, 2, 1),
    (2, 12, 9, 11, 5, 2, 1),
    (2, 6, 10, 14, 7, 1, 2),
]
FP32_LAYERS = [(2, 64, 128, 128, 64, 1, 1), (2, 512, 16, 16, 256, 1, 1)]
BWD_LAYERS = [(2, 64, 64, 64, 64, 1, 1), (2, 128, 32, 32, 128, 1, 1), (2, 256, 16, 16, 256, 1, 1),
              (1, 512, 16, 16, 256, 1, 1), (2, 64, 16, 16, 64, 2, 1), (1, 12, 9, 11, 5, 2, 1), (2, 6, 10, 14, 7, 1, 2)]


def test_reference_zero_offset_kat_on_ref():
    """DCNv2/test.py:32-65: the reference's known answer (sanity of the stored host-loop restatement), and ours."""
    from centernet_b200.dcn_v2_func import DCNv2Function
    x = kat_input()
    idx, val, _ = ref("kat")
    assert np.abs(val - x.numpy().ravel()[idx]).max() < 1e-7
    C = x.shape[1]
    w = torch.zeros(C, C, 3, 3)
    for i in range(C):
        w[i, i, 1, 1] = 1.0
    out = DCNv2Function(1, 1, 1, 1)(x.cuda(), torch.zeros(2, 18, 4, 4, device="cuda"),
                                    torch.full((2, 9, 4, 4), 0.5, device="cuda"), w.cuda(), torch.zeros(C, device="cuda")) * 2
    assert (out.cpu() - x).abs().max().item() < 1e-6


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", LAYERS)
def test_forward_three_way(B, Ci, H, W, Co, dg, stride):
    from centernet_b200.dcn_v2_func import DCNv2Function
    case = (B, Ci, H, W, Co, dg, stride)
    x, off, m, w, b = make(*case)
    cu = [t.cuda() for t in (x, off, m, w, b)]
    idx, want, _ = ref(key("fwd", case))
    got = DCNv2Function(stride, 1, 1, dg)(*cu)          # tensor-core (wgmma, 3xTF32) path
    torch.cuda.synchronize()
    Ho = (H + 2 - 3) // stride + 1; Wo = (W + 2 - 3) // stride + 1
    assert tuple(got.shape) == (B, Co, Ho, Wo)
    err = np.abs(at(got, idx) - want).max()
    assert err <= 1e-4, ("kernel vs reference", err)
    orc = dcn_ref.dcn_v2_forward(x, off, m, w, b, stride, 1, 1, dg)
    err_o = np.abs(at(orc, idx) - want.astype(np.float64)).max()
    assert err_o <= 1e-4, ("fp64 oracle vs reference", err_o)
    # whole tensor: the kernel against the fp64 oracle, which the lines above pin to the reference
    err_f = (got.double().cpu() - orc).abs().max().item()
    assert err_f <= 1e-4, ("kernel vs fp64 oracle, whole tensor", err_f)


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", FP32_LAYERS)
def test_forward_fp32_path_vs_reference(B, Ci, H, W, Co, dg, stride):
    """cnb_dcnv2_forward without a workspace = the fp32 CUDA-core contraction."""
    from centernet_b200._lib import C, ptr, stream_ptr
    case = (B, Ci, H, W, Co, dg, stride)
    x, off, m, w, b = [t.cuda() for t in make(*case, seed=5)]
    idx, want, _ = ref(key("fp32", case))
    Ho = (H + 2 - 3) // stride + 1; Wo = (W + 2 - 3) // stride + 1
    out = torch.empty(B, Co, Ho, Wo, device="cuda")
    C.dcnv2_forward(ptr(x), ptr(off), ptr(m), ptr(w), ptr(b), ptr(out), B, Ci, H, W, Co, 3, 3, stride, stride, 1, 1, 1, 1,
                    dg, 0, 0, stream_ptr(x))
    assert np.abs(at(out, idx) - want).max() <= 1e-4
    orc = dcn_ref.dcn_v2_forward(*[t.cpu() for t in (x, off, m, w, b)], stride, 1, 1, dg)
    assert np.abs(at(orc, idx) - want.astype(np.float64)).max() <= 1e-4
    assert (out.double().cpu() - orc).abs().max().item() <= 1e-4     # whole tensor


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,stride", BWD_LAYERS)
def test_backward_three_way(B, Ci, H, W, Co, dg, stride):
    from centernet_b200.dcn_v2_func import DCNv2Function
    case = (B, Ci, H, W, Co, dg, stride)
    x, off, m, w, b, go = make_bwd(*case)
    cu = [t.cuda() for t in (x, off, m, w, b)]
    cl = [t.clone().requires_grad_(True) for t in cu]
    (DCNv2Function(stride, 1, 1, dg)(*cl) * go.cuda()).sum().backward()
    leaves = [t.clone().double().requires_grad_(True) for t in (x, off, m, w, b)]
    (dcn_ref.dcn_v2_forward(*leaves, stride, 1, 1, dg) * go.double()).sum().backward()
    for name, a, o in zip(GRAD_NAMES, cl, leaves):
        idx, r, absmax = ref(key("bwd_" + name, case))
        scale = max(1.0, absmax)
        err = np.abs(at(a.grad, idx) - r).max()
        assert err <= 1e-3 * scale, ("kernel vs reference", name, err, scale)
        err_o = np.abs(at(o.grad, idx) - r.astype(np.float64)).max()
        assert err_o <= 1e-3 * scale, ("fp64 oracle vs reference", name, err_o, scale)
        err_f = (a.grad.double().cpu() - o.grad).abs().max().item()
        assert err_f <= 1e-3 * scale, ("kernel vs fp64 oracle, whole tensor", name, err_f, scale)


# ---------------------------------------------------------------- deformable PSROI pooling (N4)
def _case(seed, B, C, H, W, N, output_dim, group, pooled, part, spp, classes, trans_std, no_trans):
    rng = np.random.default_rng(seed)
    data = rng.standard_normal((B, C, H, W)).astype(np.float32)
    x = rng.uniform(-6, W * 4 - 8, N); y = rng.uniform(-6, H * 4 - 8, N)
    w = rng.uniform(1, W * 3, N); h = rng.uniform(1, H * 3, N)
    rois = np.stack([rng.integers(0, B, N).astype(np.float64), x, y, x + w, y + h], 1).astype(np.float32)
    trans = None if no_trans else rng.standard_normal((N, 2 * classes, part, part)).astype(np.float32)
    cfg = dict(no_trans=no_trans, spatial_scale=0.25, output_dim=output_dim, group_size=group, pooled_size=pooled,
               part_size=part, sample_per_part=spp, trans_std=trans_std)
    return data, rois, trans, cfg


def ps_kwargs(cfg):
    return dict(spatial_scale=cfg["spatial_scale"], pooled_size=cfg["pooled_size"], output_dim=cfg["output_dim"],
                no_trans=cfg["no_trans"], group_size=cfg["group_size"], part_size=cfg["part_size"],
                sample_per_part=cfg["sample_per_part"], trans_std=cfg["trans_std"])


def ps_grad(shape):
    return np.random.default_rng(9).standard_normal(shape).astype(np.float32)


PS_CASES = [
    (1, 2, 8, 9, 9, 5, 2, 2, 3, 3, 2, 2, 0.1, False),
    (2, 2, 18, 12, 10, 6, 2, 3, 4, 2, 3, 1, 0.3, False),
    (3, 1, 4, 7, 7, 4, 4, 1, 3, 3, 4, 2, 0.0, False),
    (4, 3, 16, 16, 16, 7, 16, 1, 7, 7, 4, 1, 0.1, True),
    (5, 2, 98, 20, 24, 12, 2, 7, 7, 7, 4, 1, 0.1, False),    # DCNv2/test.py:148-166 style: group 7, 7x7 bins
]


@pytest.mark.parametrize("case", PS_CASES)
def test_psroi_three_way(case):
    from centernet_b200.dcn_v2_func import DCNv2PoolingFunction
    data, rois, trans, cfg = _case(*case)
    k = case[:1]
    o_idx, ref_out, _ = ref(key("ps_out", k))
    c_idx, ref_cnt, _ = ref(key("ps_cnt", k))
    gi_idx, ref_gi, _ = ref(key("ps_gi", k))
    gt_idx, ref_gt, _ = ref(key("ps_gt", k))
    d = torch.from_numpy(data).cuda(); r = torch.from_numpy(rois).cuda()
    t = torch.zeros(1, device="cuda") if trans is None else torch.from_numpy(trans).cuda()
    # numpy restatement vs the reference
    want, cnt = psroi_np.psroi_forward(data, rois, trans, **cfg)
    go_np = ps_grad(want.shape)
    go = torch.from_numpy(go_np).cuda()
    np.testing.assert_allclose(want.ravel()[o_idx], ref_out, rtol=0, atol=1e-5)
    np.testing.assert_array_equal(cnt.ravel()[c_idx], ref_cnt)
    gd, gt = psroi_np.psroi_backward(go_np, data, rois, trans, cnt, **cfg)
    np.testing.assert_allclose(gd.ravel()[gi_idx], ref_gi, rtol=1e-4, atol=1e-4)
    if trans is not None:
        np.testing.assert_allclose(gt.ravel()[gt_idx], ref_gt, rtol=1e-4, atol=1e-4)
    # our kernels vs the reference
    fn = DCNv2PoolingFunction(cfg["spatial_scale"], cfg["pooled_size"], cfg["output_dim"], cfg["no_trans"],
                              cfg["group_size"], cfg["part_size"], cfg["sample_per_part"], cfg["trans_std"])
    dd = d.clone().requires_grad_(True)
    tt = d.new() if trans is None else t.clone().requires_grad_(True)
    out = fn(dd, r, tt)
    # same expression order; nvcc contracts a few multiply-adds differently in the two builds: a handful of ulps
    assert np.abs(at(out, o_idx) - ref_out).max() <= 2e-5
    out.backward(go)
    np.testing.assert_allclose(at(dd.grad, gi_idx), ref_gi, rtol=1e-4, atol=1e-4)
    if trans is not None:
        np.testing.assert_allclose(at(tt.grad, gt_idx), ref_gt, rtol=1e-4, atol=1e-4)

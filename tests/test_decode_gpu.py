"""GPU parity: the CUDA decode family (through the pybind11 -> C ABI boundary) against
(a) the committed reference goldens and (b) the numpy oracle on seeded inputs.
Bar: scores / indices / class ids bit-exact (tie-aware where the reference's order is
open), box and offset floats within 1e-4 (BASELINE.json north_star)."""
import numpy as np
import pytest
import torch

from helpers import assert_dets_bits, assert_dets_equal, golden
from oracle import decode_np as O

pytestmark = pytest.mark.gpu
TOL = 1e-4


def dev(*arrs):
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


def noise(B, C, H, W, seed, bias=2.19):
    g = torch.Generator().manual_seed(seed)
    return torch.sigmoid(torch.randn(B, C, H, W, generator=g) - bias).numpy()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(*shape, generator=g) * scale).numpy()


# ------------------------------------------------------------------ goldens
def test_golden_raw_ops():
    from centernet_b200 import decode as D
    g = golden("raw_ops")
    K = int(g["K"])
    heat, = dev(g["heat"])
    nms = D._nms(heat)
    np.testing.assert_array_equal(nms.cpu().numpy(), g["nms"])
    s, inds, clses, ys, xs = D._topk(nms, K=K)
    assert inds.dtype == torch.int64 and clses.dtype == torch.int32
    for got, key in ((s, "topk_scores"), (inds, "topk_inds"), (clses, "topk_clses"), (ys, "topk_ys"), (xs, "topk_xs")):
        np.testing.assert_array_equal(got.cpu().numpy(), g[key])
    cs, ci, cy, cx = D._topk_channel(nms, K=K)
    for got, key in ((cs, "ch_scores"), (ci, "ch_inds"), (cy, "ch_ys"), (cx, "ch_xs")):
        np.testing.assert_array_equal(got.cpu().numpy(), g[key])


def test_golden_ctdet():
    from centernet_b200 import decode as D
    g = golden("ctdet_noise")
    K = int(g["K"])
    heat, wh, reg = dev(g["heat"], g["wh"], g["reg"])
    assert_dets_equal(g["dets"], D.ctdet_decode(heat, wh, reg=reg, K=K).cpu().numpy(), atol=TOL, what="ctdet")
    assert_dets_equal(g["dets_noreg"], D.ctdet_decode(heat, wh, K=K).cpu().numpy(), atol=TOL, what="ctdet_noreg")
    g = golden("ctdet_blobs_catspec")
    heat, wh, reg = dev(g["heat"], g["wh"], g["reg"])
    got = D.ctdet_decode(heat, wh, reg=reg, cat_spec_wh=True, K=int(g["K"])).cpu().numpy()
    assert_dets_equal(g["dets"], got, atol=TOL, what="ctdet_catspec")
    g = golden("ctdet_ties")
    heat, wh, reg = dev(g["heat"], g["wh"], g["reg"])
    got = D.ctdet_decode(heat, wh, reg=reg, K=int(g["K"])).cpu().numpy()
    assert_dets_equal(g["dets"], got, atol=TOL, positive_only=True, what="ctdet_ties")


def test_golden_ddd():
    from centernet_b200 import decode as D
    g = golden("ddd")
    K = int(g["K"])
    heat, rot, depth, dim, wh, reg = dev(g["heat"], g["rot"], g["depth"], g["dim"], g["wh"], g["reg"])
    assert_dets_bits(g["dets"], D.ddd_decode(heat, rot, depth, dim, wh=wh, reg=reg, K=K).cpu().numpy(),
                     score_col=2, what="ddd")
    assert_dets_bits(g["dets_min"], D.ddd_decode(heat, rot, depth, dim, K=K).cpu().numpy(), score_col=2,
                     what="ddd_min")


# ------------------------------------------------------------------ oracle sweeps
CTDET_SHAPES = [
    # B, C, H, W, K, cat_spec, reg
    (2, 80, 128, 128, 100, False, True),    # BASELINE configs[1] geometry (whole plane per stage, TMA)
    (1, 80, 128, 128, 100, False, False),   # configs[0]: single image
    (3, 3, 96, 320, 40, False, True),       # ddd geometry: strips + 3 column blocks
    (2, 5, 30, 30, 17, True, True),         # W % 4 != 0 -> generic loader
    (2, 4, 200, 152, 64, False, True),      # tall planes -> several strips with halo rows
    (1, 1, 4, 4, 5, False, False),          # tiny
    (5, 2, 16, 520, 33, True, False),       # 5 column blocks
    (150, 2, 16, 16, 8, False, True),       # more images than SMs: a CTA spans several images
]


@pytest.mark.parametrize("B,C,H,W,K,cat,use_reg", CTDET_SHAPES)
def test_ctdet_vs_oracle(B, C, H, W, K, cat, use_reg):
    from centernet_b200 import decode as D
    heat = noise(B, C, H, W, 317 + B + C)
    wh = rnd((B, 2 * C if cat else 2, H, W), 1, 32.0)
    reg = rnd((B, 2, H, W), 2) if use_reg else None
    want = O.ctdet_decode(heat, wh, reg, cat_spec_wh=cat, K=K)
    dh, dw, dr = dev(heat, wh, reg)
    got = D.ctdet_decode(dh, dw, reg=dr, cat_spec_wh=cat, K=K)
    assert got.shape == (B, K, 6) and got.dtype == torch.float32 and got.is_cuda
    # the oracle and the kernel share one tie rule, so even tie groups agree exactly
    np.testing.assert_array_equal(got[..., 4:].cpu().numpy(), want[..., 4:])
    np.testing.assert_allclose(got[..., :4].cpu().numpy(), want[..., :4], rtol=0, atol=TOL)
    # inputs are not mutated
    np.testing.assert_array_equal(dh.cpu().numpy(), heat)


def test_ctdet_edge_cases():
    from centernet_b200 import decode as D
    B, C, H, W, K = 2, 3, 12, 20, 9
    wh = rnd((B, 2, H, W), 1, 8.0); reg = rnd((B, 2, H, W), 2)
    cases = {
        "all_zero": np.zeros((B, C, H, W), np.float32),
        "constant_plateau": np.full((B, C, H, W), 0.25, np.float32),
        "saturated": np.ones((B, C, H, W), np.float32),
    }
    few = np.zeros((B, C, H, W), np.float32)
    few[0, 1, 3, 3] = 0.9; few[0, 2, 11, 19] = 0.9; few[1, 0, 0, 0] = 0.2
    cases["fewer_than_k_peaks"] = few
    neg = -noise(B, C, H, W, 5)                    # all negative: zeros (non-peaks) outrank negative peaks
    cases["all_negative"] = neg
    mixed = noise(B, C, H, W, 6) - 0.05
    cases["mixed_sign"] = mixed.astype(np.float32)
    ties = np.round(noise(B, C, H, W, 7, bias=0.0) * 8) / 8   # heavy quantisation: many equal peaks
    cases["quantised_ties"] = ties.astype(np.float32)
    for name, heat in cases.items():
        want = O.ctdet_decode(heat, wh, reg, K=K)
        got = D.ctdet_decode(*dev(heat, wh, reg), K=K).cpu().numpy()
        np.testing.assert_array_equal(got[..., 4:], want[..., 4:], err_msg=name)
        np.testing.assert_allclose(got[..., :4], want[..., :4], rtol=0, atol=TOL, err_msg=name)


def test_topk_without_nms_and_channel():
    from centernet_b200 import decode as D
    B, C, H, W, K = 3, 7, 40, 36, 25
    scores = (noise(B, C, H, W, 11) - 0.02).astype(np.float32)   # some negatives, no peak test
    want = O.topk(scores, K)
    got = D._topk(dev(scores)[0], K=K)
    for a, b in zip(want, got):
        np.testing.assert_array_equal(b.cpu().numpy(), a)
    want = O.topk_channel(scores, K)
    got = D._topk_channel(dev(scores)[0], K=K)
    for a, b in zip(want, got):
        np.testing.assert_array_equal(b.cpu().numpy(), a)


def test_large_k_and_overflow_path():
    from centernet_b200 import decode as D
    # K=1000 with dense peaks exercises the overflow-safe expansion and repeated pruning
    B, C, H, W, K = 1, 2, 128, 128, 1000
    heat = noise(B, C, H, W, 21, bias=0.0)
    wh = rnd((B, 2, H, W), 1, 8.0)
    want = O.ctdet_decode(heat, wh, None, K=K)
    got = D.ctdet_decode(*dev(heat, wh), K=K).cpu().numpy()
    np.testing.assert_array_equal(got[..., 4:], want[..., 4:])
    # plateau map: every pixel is a peak with the same score
    heat = np.full((1, 3, 128, 128), 0.5, np.float32)
    want = O.ctdet_decode(heat, wh, None, K=100)
    got = D.ctdet_decode(*dev(heat, wh), K=100).cpu().numpy()
    np.testing.assert_array_equal(got[..., 4:], want[..., 4:])


@pytest.mark.parametrize("B,C", [(4, 80), (64, 80), (3, 7)])
def test_hot_kernel_overflow_rescan(B, C):
    """Adversarial for the running threshold: every plane is brighter than all planes before it, so the
    threshold is always stale, the key buffer overflows between rendezvous points and the exact
    per-image rebuild (select.cu flush -> rescan) has to produce the answer."""
    from centernet_b200 import decode as D
    H = W = 128
    K = 100
    g = torch.Generator(device="cuda").manual_seed(99 + B)
    base = torch.rand(B, C, H, W, device="cuda", generator=g)
    ramp = torch.linspace(0.01, 0.99, C, device="cuda").view(1, C, 1, 1)
    heat = (base * 0.01 + ramp).contiguous()
    wh = torch.rand(B, 2, H, W, device="cuda", generator=g) * 8
    dets = D.ctdet_decode(heat, wh, K=K)
    hmax = torch.nn.functional.max_pool2d(heat, 3, stride=1, padding=1)
    ref_s, ref_i = torch.topk((heat * (hmax == heat).float()).view(B, -1), K)
    assert torch.equal(ref_s, dets[..., 4])
    assert torch.equal(ref_i // (H * W), dets[..., 5].long())


def test_full_size_properties():
    """BASELINE configs[1] size (B=64): oracle too slow for every run, so check size-independent
    properties: sorted scores, every detection is a 3x3 peak with score == heat at (cls, y, x),
    result equals torch.topk over the peak-masked map as a multiset of scores, batch-shard
    invariance (decode(B=64)[i] == decode(image i alone))."""
    from centernet_b200 import decode as D
    B, C, H, W, K = 64, 80, 128, 128, 100
    g = torch.Generator(device="cuda").manual_seed(317)
    heat = torch.sigmoid(torch.randn(B, C, H, W, device="cuda", generator=g) - 2.19)
    wh = torch.rand(B, 2, H, W, device="cuda", generator=g) * 32
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g)
    dets = D.ctdet_decode(heat, wh, reg=reg, K=K)
    sc = dets[..., 4]
    assert bool((sc[:, :-1] >= sc[:, 1:]).all())
    hmax = torch.nn.functional.max_pool2d(heat, 3, stride=1, padding=1)
    masked = heat * (hmax == heat).float()
    ref_s, ref_i = torch.topk(masked.view(B, -1), K)
    assert torch.equal(ref_s, sc)
    cls = dets[..., 5].long()
    # recover (y, x) from the box centre minus the regression offset
    cx = (dets[..., 0] + dets[..., 2]) / 2; cy = (dets[..., 1] + dets[..., 3]) / 2
    flat_ref = ref_i % (H * W)
    ys, xs = flat_ref // W, flat_ref % W
    assert torch.equal(cls, ref_i // (H * W))       # tie-free at this seed (SURVEY appendix A)
    bi = torch.arange(B, device="cuda")[:, None]
    assert torch.allclose(cx, xs.float() + reg[bi, 0, ys, xs], atol=1e-3)
    assert torch.allclose(cy, ys.float() + reg[bi, 1, ys, xs], atol=1e-3)
    for i in (0, 17, 63):
        single = D.ctdet_decode(heat[i:i + 1].contiguous(), wh[i:i + 1].contiguous(), reg=reg[i:i + 1].contiguous(), K=K)
        assert torch.equal(single[0], dets[i])
    # against the oracle on a 2-image slice of the same batch
    want = O.ctdet_decode(heat[:2].cpu().numpy(), wh[:2].cpu().numpy(), reg[:2].cpu().numpy(), K=K)
    np.testing.assert_array_equal(dets[:2, :, 4:].cpu().numpy(), want[..., 4:])
    np.testing.assert_allclose(dets[:2, :, :4].cpu().numpy(), want[..., :4], rtol=0, atol=TOL)


def test_error_behaviour():
    from centernet_b200 import decode as D
    heat = torch.rand(1, 2, 8, 8, device="cuda")
    with pytest.raises(RuntimeError):          # K > H*W: torch.topk raises in the reference too
        D.ctdet_decode(heat, torch.rand(1, 2, 8, 8, device="cuda"), K=65)
    with pytest.raises(RuntimeError):
        D.ctdet_decode(heat, torch.rand(1, 3, 8, 8, device="cuda"), K=4)


def test_golden_exct():
    from centernet_b200 import decode as D
    g = golden("exct")
    K, ND = int(g["K"]), int(g["num_dets"])
    maps = dev(g["t"], g["l"], g["b"], g["r"], g["ct"])
    regs = dev(g["t_regr"], g["l_regr"], g["b_regr"], g["r_regr"])
    got = D.exct_decode(*maps, *regs, K=K, num_dets=ND).cpu().numpy()
    assert_dets_equal(g["dets"], got, atol=TOL, positive_only=True, what="exct")
    got = D.exct_decode(*maps, K=K, num_dets=ND).cpu().numpy()
    assert_dets_equal(g["dets_noreg"], got, atol=TOL, positive_only=True, what="exct_noreg")
    got = D.exct_decode(*maps, *regs, K=K, num_dets=ND, aggr_weight=0.1).cpu().numpy()
    assert_dets_equal(g["dets_aggr"], got, atol=TOL, positive_only=True, what="exct_aggr")
    agn_maps = dev(g["t1"], g["l1"], g["b1"], g["r1"], g["ct"])
    got = D.agnex_ct_decode(*agn_maps, *regs, K=K, num_dets=ND).cpu().numpy()
    assert_dets_equal(g["dets_agn"], got, atol=TOL, positive_only=True, what="agnex")


def _extreme_maps(B, C, H, W, seed, n_obj=8):
    """Structured t/l/b/r/centre maps: boxes whose extreme points and centre carry peaks of one class."""
    rng = np.random.default_rng(seed)
    base = (0.03 * rng.random((5, B, C, H, W))).astype(np.float32)
    for b in range(B):
        for _ in range(n_obj):
            c = rng.integers(0, C)
            x0, x1 = sorted(rng.integers(2, W - 2, 2)); y0, y1 = sorted(rng.integers(2, H - 2, 2))
            if x1 - x0 < 4 or y1 - y0 < 4:
                continue
            tx, bx = rng.integers(x0, x1 + 1, 2); ly, ry = rng.integers(y0, y1 + 1, 2)
            sc = rng.uniform(0.3, 0.95, 5).astype(np.float32)
            base[0, b, c, y0, tx] = sc[0]; base[1, b, c, ly, x0] = sc[1]
            base[2, b, c, y1, bx] = sc[2]; base[3, b, c, ry, x1] = sc[3]
            base[4, b, c, (y0 + y1) // 2, (x0 + x1) // 2] = sc[4]
    return [base[i] for i in range(5)]


@pytest.mark.parametrize("B,C,H,W,K,ND,aggr", [(2, 6, 48, 64, 12, 300, 0.0), (1, 80, 128, 128, 20, 1000, 0.0),
                                               (2, 3, 32, 40, 9, 200, 0.1)])
def test_exct_vs_oracle(B, C, H, W, K, ND, aggr):
    """Exact agreement with the oracle on EVERY row (the oracle and the kernel share the tie rule:
    score desc, tuple index asc), including the non-positive filler rows."""
    from centernet_b200 import decode as D
    maps = _extreme_maps(B, C, H, W, 40 + K)
    regs = [rnd((B, 2, H, W), 50 + i) for i in range(4)]
    want = O.exct_decode(*maps, *regs, K=K, num_dets=ND, aggr_weight=aggr)
    got = D.exct_decode(*dev(*maps), *dev(*regs), K=K, num_dets=ND, aggr_weight=aggr).cpu().numpy()
    assert got.shape == (B, ND, 14)
    assert (want[..., 4] > 0).sum() > 0
    np.testing.assert_array_equal(got[..., 4], want[..., 4])
    np.testing.assert_array_equal(got[..., 13], want[..., 13])
    np.testing.assert_allclose(got, want, rtol=0, atol=TOL)
    # class-agnostic variant
    t1, l1, b1, r1 = [m.max(axis=1, keepdims=True) for m in maps[:4]]
    want = O.agnex_ct_decode(t1, l1, b1, r1, maps[4], *regs, K=K, num_dets=ND, aggr_weight=aggr)
    got = D.agnex_ct_decode(*dev(t1, l1, b1, r1, maps[4]), *dev(*regs), K=K, num_dets=ND, aggr_weight=aggr).cpu().numpy()
    np.testing.assert_array_equal(got[..., 4], want[..., 4])
    np.testing.assert_allclose(got, want, rtol=0, atol=TOL)


@pytest.mark.parametrize("scale_ct,thr_s,thr_c,neg", [(3.0, 0.1, 0.1, False), (1.0, 0.35, 0.5, False), (0.5, 0.1, 0.1, True)])
def test_exct_block_pruning_is_exact(scale_ct, thr_s, thr_c, neg):
    """k_exct_tuples skips whole (top, left) blocks against a bound built from the best bottom / right scores and the
    largest centre value.  Inputs that stress the bound: centre values above 1 (nothing clamps the centre map), high
    thresholds (most tuples carry the score penalty), extreme maps with negative values (non-positive candidates),
    num_dets small enough that the running threshold climbs early -- every row must still equal the oracle's."""
    from centernet_b200 import decode as D
    B, C, H, W, K, ND = 2, 5, 40, 48, 16, 150
    maps = _extreme_maps(B, C, H, W, 77, n_obj=10)
    maps[4] = (maps[4] * scale_ct).astype(np.float32)
    if neg:
        maps = [m - np.float32(0.02) for m in maps]
    regs = [rnd((B, 2, H, W), 60 + i) for i in range(4)]
    kw = dict(K=K, num_dets=ND, scores_thresh=thr_s, center_thresh=thr_c)
    want = O.exct_decode(*maps, *regs, **kw)
    got = D.exct_decode(*dev(*maps), *dev(*regs), **kw).cpu().numpy()
    np.testing.assert_array_equal(got[..., 4], want[..., 4])
    np.testing.assert_array_equal(got[..., 13], want[..., 13])
    np.testing.assert_allclose(got, want, rtol=0, atol=TOL)
    t1, l1, b1, r1 = [m.max(axis=1, keepdims=True) for m in maps[:4]]
    want = O.agnex_ct_decode(t1, l1, b1, r1, maps[4], *regs, **kw)
    got = D.agnex_ct_decode(*dev(t1, l1, b1, r1, maps[4]), *dev(*regs), **kw).cpu().numpy()
    np.testing.assert_array_equal(got[..., 4], want[..., 4])
    np.testing.assert_allclose(got, want, rtol=0, atol=TOL)


def test_topk_nonpositive_scores():
    from centernet_b200 import decode as D
    scores = -noise(2, 3, 12, 16, 31)                       # every score negative, no peak test
    scores[0, 1, 3, 3] = 0.0; scores[1, 2, 0, 0] = 0.25
    want = O.topk(scores.astype(np.float32), 7)
    got = D._topk(dev(scores.astype(np.float32))[0], K=7)
    for a, b in zip(want, got):
        np.testing.assert_array_equal(b.cpu().numpy(), a)

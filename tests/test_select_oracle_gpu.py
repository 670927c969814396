"""GPU: the fused peak-NMS + top-K selection (select.cu: k_select_hot, k_select_stage1, k_select_finalize) against
an independent reference, oracle/select_torch.py (max_pool2d + stable sort, pinned to the numpy oracle and to the
reference's goldens by tests/test_select_oracle.py), in every plan regime, at every K the hot kernel branches on,
on maps that drive each branch (ties, plateaus, zeros, negatives, subnormals, huge scores, buffer overflow), for
fp32 / fp16 / bf16 heads and logits, and on non-finite scores under the library's rule (DESIGN.md, "Non-finite
scores").

Bar: every row of the K, including the non-positive fillers, equals the reference's on all 6 columns
(np.array_equal: -0.0 == +0.0).  The plan query (cnb_select_plan_info) asserts which regime each case reaches on
the SM count of the device the suite runs on."""
import math

import numpy as np
import pytest
import torch

import big_inputs as BI
import select_maps as SM
from oracle import decode_np as O
from oracle import select_torch as ST

pytestmark = pytest.mark.gpu
HW = 128


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _plan(t, B, C, K, H=HW, W=HW):
    from centernet_b200 import _C
    return _C.select_plan_info(t.data_ptr(), B, C, H, W, K, 1, t.element_size())


def _heads(B, C, H, W, seed, cat=False, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(1000 + seed)
    wh = (torch.rand(B, 2 * C if cat else 2, H, W, device="cuda", generator=g) * 32).to(dtype)
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g).to(dtype)
    return wh, reg


def _same(got, want, what):
    got = got.detach().cpu().numpy(); want = want.detach().cpu().numpy()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if np.array_equal(got, want):
        return
    rows = np.argwhere(~(got == want).all(-1))
    b, k = rows[0]
    raise AssertionError("%s: %d rows differ, first image %d row %d: got %s, want %s"
                         % (what, len(rows), b, k, got[b, k].tolist(), want[b, k].tolist()))


def _ctdet(heat, K, reg=True, cat=False, nonfinite="reference", logits=False, what=""):
    """Runs the library's ctdet decode on heat (or logits) and compares with the reference on the .float() upcast."""
    from centernet_b200 import decode as D
    B, C, H, W = heat.shape
    wh, rg = _heads(B, C, H, W, K + C, cat=cat, dtype=heat.dtype)
    rg = rg if reg else None
    if logits:
        got = D.ctdet_decode_from_logits(heat, wh, reg=rg, cat_spec_wh=cat, K=K)
        ref_heat = torch.sigmoid(heat.float())
    else:
        got = D.ctdet_decode(heat, wh, reg=rg, cat_spec_wh=cat, K=K)
        ref_heat = heat.float()
    want = ST.ctdet_decode(ref_heat, wh, rg, cat_spec_wh=cat, K=K, nonfinite=nonfinite)
    _same(got, want, what or "ctdet")
    return got


# ------------------------------------------------------------------ plan regimes at 128x128 (hot kernel)
def _regime(name, n):
    """(B, C, predicate on the plan) of a named regime for a device with n SMs."""
    return {
        "one_cta": (1, 3, lambda p: p["n_cta"] == 1 and p["local_img"] == 1),
        "small_batch_shrink": (1, 80, lambda p: p["n_cta"] == 27 and p["max_slots"] > 8 and p["wb"] == 0),
        "equal_split": (math.ceil(4 * n / 80), 80, lambda p: p["n_cta"] == n and p["wb"] == 0 and p["max_slots"] > 1),
        "weighted_b64": (64, 80, lambda p: p["n_cta"] == n and p["wb"] == 4),
        "weighted_b150": (150, 80, lambda p: p["n_cta"] == n and p["wb"] == 4),
        "local_finalize": (4 * n, 3, lambda p: p["n_cta"] == n and p["local_img"] == 1),
        "c1_below_n": (n - 1, 1, lambda p: p["n_cta"] == n - 1 and p["local_img"] == 1 and p["max_slots"] == 1),
        "c1_at_n": (n, 1, lambda p: p["n_cta"] == n and p["local_img"] == 1 and p["max_slots"] == 1),
        "c1_above_n": (n + 1, 1, lambda p: p["n_cta"] == n and p["local_img"] == 1 and p["max_slots"] == 1),
    }[name]


REGIMES = ["one_cta", "small_batch_shrink", "equal_split", "weighted_b64", "weighted_b150", "local_finalize",
           "c1_below_n", "c1_at_n", "c1_above_n"]


@pytest.mark.parametrize("name", REGIMES)
def test_plan_regimes(name):
    n = _sms()
    B, C, pred = _regime(name, n)
    K = 100
    heat = SM.make_map("noise", B, C, HW, HW, seed=B * 7 + C, device="cuda")
    p = _plan(heat, B, C, K)
    print("plan %-18s SMs=%d B=%d C=%d: %s" % (name, n, B, C, p))
    assert p["hot"] == 1 and pred(p), p
    _ctdet(heat, K, what=name)
    if B * C <= 1600:          # a second map per regime: ties across classes and CTAs
        _ctdet(SM.make_map("ties", B, C, HW, HW, seed=3, device="cuda"), K, what=name + " ties")


# ------------------------------------------------------------------ K at the hot geometry
HOT_K = [1, 2, 31, 32, 33, 100, 127, 128, 129, 200, 255, 256]


@pytest.mark.parametrize("K", HOT_K)
@pytest.mark.parametrize("B", [2, 16])
@pytest.mark.parametrize("kind", ["noise", "ties"])
def test_hot_k(K, B, kind):
    heat = SM.make_map(kind, B, 80, HW, HW, seed=K, device="cuda")
    p = _plan(heat, B, 80, K)
    assert p["hot"] == 1 and p["seg_cap"] == (256 if K <= 128 else K) and p["max_slots"] > 1, p
    _ctdet(heat, K, what="K=%d B=%d %s" % (K, B, kind))


# ------------------------------------------------------------------ 128x128 beyond the hot kernel (K > 256)
@pytest.mark.parametrize("K", [257, 512, 1000, 1024])
@pytest.mark.parametrize("B", [1, 3])
def test_non_hot_large_k(K, B):
    C = 80
    heat = SM.make_map("noise", B, C, HW, HW, seed=K + B, device="cuda")
    p = _plan(heat, B, C, K)
    print("plan K=%d B=%d: %s" % (K, B, p))
    # the grid shrinks until max_slots*K fits the separate finalize, which runs because it exceeds the fused buffer
    assert p["hot"] == 0 and p["n_cta"] < min(_sms(), B * C) and p["max_slots"] * K <= 8192, p
    assert p["fused_finalize"] == 0 and p["max_slots"] * K > 2048, p
    _ctdet(heat, K, what="K=%d B=%d" % (K, B))
    _ctdet(SM.make_map("few", B, C, HW, HW, seed=K, device="cuda"), K, what="few K=%d B=%d" % (K, B))


def test_k_above_limit_raises():
    from centernet_b200 import decode as D
    heat = SM.make_map("noise", 1, 80, HW, HW, device="cuda")
    wh, reg = _heads(1, 80, HW, HW, 0)
    with pytest.raises((RuntimeError, NotImplementedError)):
        D.ctdet_decode(heat, wh, reg=reg, K=1025)


# ------------------------------------------------------------------ map distributions at hot regimes
@pytest.mark.parametrize("kind", SM.KINDS)
@pytest.mark.parametrize("B", [2, 16])
def test_hot_maps(kind, B):
    heat = SM.make_map(kind, B, 80, HW, HW, seed=11, device="cuda")
    assert _plan(heat, B, 80, 100)["hot"] == 1
    _ctdet(heat, 100, what="%s B=%d" % (kind, B))


@pytest.mark.parametrize("B", [4, 64])
def test_brightening_ramp_tie_order(B):
    """Every plane brighter than all before it: the threshold is always stale, the key buffer overflows and the
    flush rescans; the plateau-free ramp plus quantised noise also leaves ties that must come out by index."""
    heat = SM.make_map("ramp", B, 80, HW, HW, seed=B, device="cuda")
    heat = torch.round(heat * 64) / 64
    _ctdet(heat, 100, what="ramp B=%d" % B)


def test_constant_plateau_overflow_and_chunked_prune():
    """B=1, C=80, K=100 of one constant: every segment's buffer overflows (flush rescan), and more than SEL_CAP keys
    clear the union cut of the 27 segments (chunked sort-prune in the finalize)."""
    heat = torch.full((1, 80, HW, HW), 0.5, device="cuda")
    p = _plan(heat, 1, 80, 100)
    assert p["hot"] == 1 and p["max_slots"] > 8 and p["max_slots"] * 100 > 2048, p
    _ctdet(heat, 100, what="plateau")
    _ctdet(heat, 100, reg=False, cat=True, what="plateau cat")


def test_misaligned_view_takes_the_generic_path():
    """A contiguous view 4 bytes off alignment cannot be loaded by TMA: the generic stage-1 kernel runs, with a larger
    grid than the hot plan of the same shape, so the workspace query has to cover both plans."""
    B, C, K = 2, 80, 100
    buf = torch.empty(B * C * HW * HW + 1, device="cuda")
    heat = buf[1:].view(B, C, HW, HW)
    heat.copy_(SM.make_map("noise", B, C, HW, HW, seed=5, device="cuda"))
    p = _plan(heat, B, C, K)
    assert p["use_tma"] == 0 and p["hot"] == 0, p
    _ctdet(heat, K, what="misaligned")
    heat.copy_(SM.make_map("mixed", B, C, HW, HW, seed=6, device="cuda"))
    _ctdet(heat, K, what="misaligned mixed")


@pytest.mark.parametrize("K,kind", [(100, "noise"), (256, "noise"), (100, "few"), (1, "ties")])
@pytest.mark.parametrize("reg,cat", [(True, False), (False, False), (True, True)])
def test_epilogue(K, kind, reg, cat):
    """reg / no reg / cat_spec_wh on the rank-sort (K=100), bitonic (K=256) and fill (few peaks) paths, which gather
    the rows in different places."""
    heat = SM.make_map(kind, 2, 80, HW, HW, seed=21, device="cuda")
    _ctdet(heat, K, reg=reg, cat=cat, what="epilogue K=%d %s reg=%s cat=%s" % (K, kind, reg, cat))
    # the local finalize (whole images inside one CTA) gathers from shared memory
    heat = SM.make_map(kind, 4 * _sms(), 3, HW, HW, seed=22, device="cuda")
    _ctdet(heat, min(K, 100), reg=reg, cat=cat, what="local epilogue K=%d %s" % (K, kind))


# ------------------------------------------------------------------ logits and 16-bit heads
def _logits(kind, B, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    shape = (B, C, HW, HW)
    if kind == "noise":
        return torch.randn(shape, device="cuda", generator=g) - 2.19
    if kind == "saturated":    # x >= 17: sigmoid 1.0 plateaus next to ordinary peaks
        x = torch.randn(shape, device="cuda", generator=g) - 2.19
        sat = torch.rand(shape, device="cuda", generator=g) < 0.002
        return torch.where(sat, 17 + 10 * torch.rand(shape, device="cuda", generator=g), x)
    if kind == "ulp":          # collide_margin / logit_lower_bound: peaks by equal sigmoid, not by equal logit
        return SM.ulp_neighbours(B, C, HW, HW, [-3.0, 0.5, 3.0, 6.0, 9.0, 11.5, 14.0], seed=seed, device="cuda")
    if kind == "underflow":    # sigmoid 0 or subnormal
        return -80 - 40 * torch.rand(shape, device="cuda", generator=g)
    if kind == "inf":
        x = torch.randn(shape, device="cuda", generator=g) - 2.19
        sel = torch.rand(shape, device="cuda", generator=g)
        x = torch.where(sel < 0.001, torch.full_like(x, float("inf")), x)
        return torch.where(sel > 0.995, torch.full_like(x, float("-inf")), x)
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["noise", "saturated", "ulp", "underflow", "inf"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_logits(kind, dtype):
    lg = _logits(kind, 2, 80, 5).to(dtype)
    assert _plan(lg, 2, 80, 100)["hot"] == 1
    _ctdet(lg, 100, logits=True, what="logits %s %s" % (kind, dtype))
    _ctdet(lg, 256, logits=True, reg=False, what="logits K=256 %s %s" % (kind, dtype))


@pytest.mark.parametrize("kind", SM.KINDS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_heads(kind, dtype):
    heat = SM.make_map(kind, 2, 80, HW, HW, seed=31, device="cuda").to(dtype)
    assert _plan(heat, 2, 80, 100)["hot"] == 1
    _ctdet(heat, 100, what="%s %s" % (kind, dtype))


# ------------------------------------------------------------------ other decodes through the same selection
@pytest.mark.parametrize("K", [1, 200])
def test_multi_pose(K):
    from centernet_b200 import decode as D
    heat, wh, kps, reg, hm_hp, hp_off = BI.multi_pose_inputs(seed=400 + K, B=2)
    want = O.multi_pose_decode(heat, wh, kps, reg, hm_hp, hp_off, K=K)
    dev = [torch.from_numpy(a).cuda() for a in (heat, wh, kps, reg, hm_hp, hp_off)]
    got = D.multi_pose_decode(dev[0], dev[1], dev[2], reg=dev[3], hm_hp=dev[4], hp_offset=dev[5], K=K)
    _same(got, torch.from_numpy(want), "multi_pose K=%d" % K)
    # the joint selection: _topk_channel of the NMS'd joint maps, raw outputs
    hm = ST.nms(dev[4])
    for a, b, what in zip(D._topk_channel(hm, K=K), ST.topk_channel(hm, K), ("scores", "inds", "ys", "xs")):
        assert torch.equal(a, b), "topk_channel %s K=%d" % (what, K)


def test_exdet_clamps_extreme_maps():
    """Extreme-point maps with values above 1: the hot kernel ranks by min(score, 1) (decode.py:299-302)."""
    from centernet_b200 import decode as D
    maps, regs = BI.exct_inputs(seed=401, B=1, C=80)
    maps = [m * np.float32(1.6) if i < 4 else m for i, m in enumerate(maps)]
    assert max(float(m.max()) for m in maps[:4]) > 1
    K, ND = 40, 1000
    want = O.exct_decode(*maps, *regs, K=K, num_dets=ND)
    got = D.exct_decode(*[torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in maps + regs], K=K, num_dets=ND)
    assert (want[..., 4] > 0).sum() > 0
    assert np.array_equal(got.cpu().numpy(), want)


# ------------------------------------------------------------------ back to back on one stream
def test_back_to_back_plans():
    from centernet_b200 import decode as D
    cases = [("hot B=64", SM.make_map("noise", 64, 80, HW, HW, seed=1, device="cuda"), 100, False),
             ("B=1 K=256", SM.make_map("ties", 1, 80, HW, HW, seed=2, device="cuda"), 256, False),
             ("non-hot K=1000", SM.make_map("noise", 1, 80, HW, HW, seed=3, device="cuda"), 1000, False),
             ("bf16 logits", _logits("noise", 2, 80, 4).bfloat16(), 100, True)]
    heads = [_heads(h.shape[0], h.shape[1], HW, HW, i, dtype=h.dtype) for i, (_, h, _, _) in enumerate(cases)]
    fn = lambda lg: D.ctdet_decode_from_logits if lg else D.ctdet_decode
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        outs = [fn(lg)(h, wh, reg=rg, K=K) for (_, h, K, lg), (wh, rg) in zip(cases, heads)]
    s.synchronize()
    for (what, h, K, lg), (wh, rg), got in zip(cases, heads, outs):
        alone = fn(lg)(h, wh, reg=rg, K=K)
        torch.cuda.synchronize()
        assert torch.equal(got, alone), what
        want = ST.ctdet_decode(torch.sigmoid(h.float()) if lg else h, wh, rg, K=K)
        _same(got, want, what)


# ------------------------------------------------------------------ non-finite scores (the library's rule)
@pytest.mark.parametrize("kind,B,C", [("noise", 2, 80), ("few", 2, 80), ("few", 16, 80), ("mixed", 2, 80),
                                      ("neg_const", 2, 3), ("plateau", 1, 80), ("ramp", 4, 80)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_nonfinite_hot(kind, B, C, dtype):
    heat = SM.poison(SM.make_map(kind, B, C, HW, HW, seed=41, device="cuda").to(dtype), seed=B)
    assert _plan(heat, B, C, 100)["hot"] == 1
    _ctdet(heat, 100, nonfinite="library", what="nonfinite %s B=%d C=%d %s" % (kind, B, C, dtype))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_nonfinite_logits(dtype):
    lg = SM.poison(_logits("noise", 2, 80, 7).to(dtype), seed=3)
    _ctdet(lg, 100, logits=True, nonfinite="library", what="nonfinite logits %s" % dtype)
    lg = SM.poison(_logits("underflow", 2, 80, 8).to(dtype), seed=4)      # < K positive scores: the fill
    _ctdet(lg, 100, logits=True, nonfinite="library", what="nonfinite underflow logits %s" % dtype)


# (B, C, H, W, K, misaligned, the stage-1 path the plan must select)
GENERIC = [(1, 80, 128, 128, 1000, False, "mode 2 + separate finalize"),
           (2, 5, 64, 96, 50, False, "mode 1"),
           (2, 1, 8, 12, 96, False, "mode 1, every pixel ranked"),
           (2, 3, 40, 320, 40, False, "mode 0 (TMA)"),
           (2, 5, 30, 30, 17, False, "mode 0 (no TMA: w % 4)"),
           (2, 1, 9, 10, 90, False, "mode 0 (no TMA), every pixel ranked"),
           (2, 4, 64, 64, 64, True, "mode 0 (no TMA: misaligned)")]


@pytest.mark.parametrize("B,C,H,W,K,mis,path", GENERIC, ids=[g[-1] for g in GENERIC])
@pytest.mark.parametrize("kind", ["noise", "few", "neg_const", "mixed"])
def test_nonfinite_generic_paths(B, C, H, W, K, mis, path, kind):
    buf = torch.empty(B * C * H * W + 1, device="cuda")
    heat = (buf[1:] if mis else buf[:-1]).view(B, C, H, W)
    heat.copy_(SM.poison(SM.make_map(kind, B, C, H, W, seed=K, device="cuda"), seed=C))
    p = _plan(heat, B, C, K, H, W)
    assert p["hot"] == 0, p
    assert p["use_tma"] == (0 if "no TMA" in path else 1), p
    if "separate" in path:
        assert p["fused_finalize"] == 0, p
    _ctdet(heat, K, nonfinite="library", what="%s %s" % (path, kind))
    # raw _topk / _topk_channel outputs on the NMS'd map (no peak test inside the kernel)
    from centernet_b200 import decode as D
    nm = ST.nms(heat, nonfinite="library")
    for a, b in zip(D._topk(nm, K=K), ST.topk(nm, K)):
        assert np.array_equal(a.cpu().numpy(), b.cpu().numpy()), path
    kc = min(K, H * W)
    for a, b in zip(D._topk_channel(nm, K=kc), ST.topk_channel(nm, kc)):
        assert np.array_equal(a.cpu().numpy(), b.cpu().numpy()), path

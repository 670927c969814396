"""multi_pose_decode and ddd_decode from the heads' raw logits and from bf16 / fp16 heads.

Contract 1: multi_pose_decode_from_logits(hm, ..., hm_hp) == multi_pose_decode(torch.sigmoid(hm), ...,
torch.sigmoid(hm_hp)), and ddd_decode_from_logits(hm, rot, dep, ...) == ddd_decode(torch.sigmoid(hm), rot,
1. / (torch.sigmoid(dep) + 1e-6) - 1., ...), bit for bit, with torch's own CUDA ops on the right.
Contract 2: every one of the four functions returns for half heads (any mix of dtypes) what it returns for their
.float() upcast.  The fp32 decodes on the right are pinned bit for bit against the reference and the oracle elsewhere
(test_pose_ddd_edges_gpu.py, test_pose_aggr_loss_gpu.py, test_decode_gpu.py, test_big_golden.py)."""
import numpy as np
import pytest
import torch

import big_inputs as BI

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]


def _up(t):
    return None if t is None else t.float()


def _sig(t):
    return None if t is None else torch.sigmoid(t)


def _dep(t):
    return 1. / (torch.sigmoid(t) + 1e-6) - 1.   # detectors/ddd.py:62


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _pose_heads(B, H=128, W=128, J=17, seed=0):
    """Logits of hm and hm_hp (about half of the joints' peaks pass the 0.1 threshold) and the regression heads."""
    g = _gen(seed)
    hm = torch.randn(B, 1, H, W, device="cuda", generator=g) * 2 - 2.19
    wh = torch.rand(B, 2, H, W, device="cuda", generator=g) * 40
    hps = (torch.rand(B, 2 * J, H, W, device="cuda", generator=g) - 0.5) * 24
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g)
    hm_hp = torch.randn(B, J, H, W, device="cuda", generator=g) * 2 - 2.19
    off = torch.rand(B, 2, H, W, device="cuda", generator=g)
    return [hm, wh, hps, reg, hm_hp, off]


def _ddd_heads(B, H=96, W=320, C=3, seed=0):
    g = _gen(seed)
    hm = torch.randn(B, C, H, W, device="cuda", generator=g) * 2 - 2.19
    rot = torch.randn(B, 8, H, W, device="cuda", generator=g)
    dep = torch.rand(B, 1, H, W, device="cuda", generator=g) * 195 - 105
    dim = torch.rand(B, 3, H, W, device="cuda", generator=g) * 4
    wh = torch.rand(B, 2, H, W, device="cuda", generator=g) * 60
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g)
    return [hm, rot, dep, dim, wh, reg]


def _unchanged(ts, keep):
    for t, k in zip(ts, keep):
        assert t is None or torch.equal(t, k), "input modified"


def _clone(ts):
    return [None if t is None else t.clone() for t in ts]


def _pose_logits_check(heads, K):
    """Contract 1 for multi_pose."""
    from centernet_b200 import decode as D
    hm, wh, hps, reg, hm_hp, off = heads
    keep = _clone(heads)
    got = D.multi_pose_decode_from_logits(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=off, K=K)
    want = D.multi_pose_decode(_sig(hm), wh, hps, reg=reg, hm_hp=_sig(hm_hp), hp_offset=off, K=K)
    _unchanged(heads, keep)
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert torch.equal(got, want)
    return got


def _ddd_logits_check(heads, K):
    """Contract 1 for ddd."""
    from centernet_b200 import decode as D
    hm, rot, dep, dim, wh, reg = heads
    keep = _clone(heads)
    got = D.ddd_decode_from_logits(hm, rot, dep, dim, wh=wh, reg=reg, K=K)
    want = D.ddd_decode(torch.sigmoid(hm), rot, _dep(dep), dim, wh=wh, reg=reg, K=K)
    _unchanged(heads, keep)
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert torch.equal(got, want)
    return got


def _half_check(fn, heads, K):
    """Contract 2: fn(heads) == fn(heads.float())."""
    keep = _clone(heads)
    got = fn(*heads, K=K)
    want = fn(*[_up(t) for t in heads], K=K)
    _unchanged(heads, keep)
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert torch.equal(got, want)
    return got


POSE_VARIANTS = {"full": (1, 1, 1), "no_reg": (0, 1, 1), "no_offset": (1, 1, 0), "no_hm_hp": (1, 0, 0)}


def _variant(heads, name):
    r, hp, off = POSE_VARIANTS[name]
    return heads[:3] + [heads[3] if r else None, heads[4] if hp else None, heads[5] if off else None]


# ------------------------------------------------------------------ contract 1, multi_pose
@pytest.mark.parametrize("variant", list(POSE_VARIANTS))
@pytest.mark.parametrize("hw", [(128, 128), (64, 64), (96, 160), (72, 90)], ids=["hot", "64", "96x160", "w90"])
def test_pose_logits_geometry(hw, variant):
    heads = _variant(_pose_heads(2, *hw, seed=hw[1]), variant)
    dets = _pose_logits_check(heads, K=100)
    if variant != "no_hm_hp":   # the joint snapping happened at least sometimes
        assert not torch.equal(dets, _pose_logits_check(_variant(heads, "no_hm_hp"), K=100))


@pytest.mark.parametrize("B", [1, 2, 8, 64])
def test_pose_logits_batch(B):
    _pose_logits_check(_pose_heads(B, seed=B), K=100)


@pytest.mark.parametrize("K", [1, 20, 100, 256, 300])
@pytest.mark.parametrize("hw", [(128, 128), (96, 160)], ids=["hot", "96x160"])
def test_pose_logits_k(K, hw):
    _pose_logits_check(_pose_heads(3, *hw, seed=K), K=K)


# ------------------------------------------------------------------ contract 1, ddd
@pytest.mark.parametrize("with_wh_reg", [True, False], ids=["wh_reg", "min"])
@pytest.mark.parametrize("hw", [(96, 320), (128, 128)], ids=["kitti", "hot"])
@pytest.mark.parametrize("K", [40, 100])
def test_ddd_logits(hw, with_wh_reg, K):
    heads = _ddd_heads(2, *hw, seed=K + hw[1])
    if not with_wh_reg:
        heads[4] = heads[5] = None
    _ddd_logits_check(heads, K)


# dep values at which the transform is delicate: 0, tiny, around the sigmoid's saturation to 0 (exp(-x) overflows
# near x = -88.7, the sum s + 1e-6 is 1e-6 below about -13.8) and to 1 (above about 16.6), and the range ends
_DEP_SPECIAL = [0.0, -0.0, 1e-3, -1e-3, 1e-7, -1e-7, 1.0, -1.0, -13.8, -13.9, -16.0, -20.0, -30.0, -87.0, -88.0,
                -88.7, -89.0, -103.0, -104.9, -105.0, 9.0, 15.9, 16.6, 17.0, 17.4, 30.0, 88.0, 89.9, 90.0]


def _spread_dep(shape, seed):
    """dep logits over [-105, 90]: a linear sweep, random values and every special value, shuffled."""
    n = int(np.prod(shape))
    g = _gen(seed)
    sweep = torch.linspace(-105, 90, n // 2, device="cuda")
    rnd = torch.rand(n - n // 2 - len(_DEP_SPECIAL), device="cuda", generator=g) * 195 - 105
    v = torch.cat([sweep, rnd, torch.tensor(_DEP_SPECIAL, device="cuda")])
    return v[torch.randperm(n, device="cuda", generator=g)].view(shape)


def test_ddd_depth_every_pixel():
    """K = h*w: every position of every image is gathered, so all 65536 dep values pass through the epilogue."""
    B, H, W = 64, 32, 32
    heads = _ddd_heads(B, H, W, C=1, seed=11)
    heads[2] = _spread_dep((B, 1, H, W), 12)
    dets = _ddd_logits_check(heads, K=H * W)
    # the transform really saw the extremes: 1/(0 + 1e-6) - 1 and 1/(1 + 1e-6) - 1
    d = dets[..., 11]
    assert float(d.max()) > 9.9e5 and float(d.min()) < 0


@pytest.mark.parametrize("hw", [(96, 320), (128, 128)], ids=["kitti", "hot"])
def test_ddd_depth_k1000(hw):
    B = 24 if hw == (96, 320) else 16
    heads = _ddd_heads(B, *hw, seed=13)
    heads[2] = _spread_dep((B, 1) + hw, 14)
    _ddd_logits_check(heads, K=1000)


# ------------------------------------------------------------------ contract 2, all four functions
def _fns():
    from centernet_b200 import decode as D
    pose = lambda f: (lambda hm, wh, hps, reg, hm_hp, off, K: f(hm, wh, hps, reg=reg, hm_hp=hm_hp,  # noqa: E731
                                                                  hp_offset=off, K=K))
    ddd = lambda f: (lambda hm, rot, dep, dim, wh, reg, K: f(hm, rot, dep, dim, wh=wh, reg=reg, K=K))  # noqa: E731
    return {"multi_pose": pose(D.multi_pose_decode), "multi_pose_logits": pose(D.multi_pose_decode_from_logits),
            "ddd": ddd(D.ddd_decode), "ddd_logits": ddd(D.ddd_decode_from_logits)}


FNS = ["multi_pose", "multi_pose_logits", "ddd", "ddd_logits"]


def _heads_for(fn, B, hw=None, seed=0):
    if fn.startswith("multi_pose"):
        heads = _pose_heads(B, *(hw or (128, 128)), seed=seed)
    else:
        heads = _ddd_heads(B, *(hw or (96, 320)), seed=seed)
    if not fn.endswith("logits"):   # heat maps, not logits
        heads[0] = torch.sigmoid(heads[0])
        if fn == "multi_pose":
            heads[4] = torch.sigmoid(heads[4])
        else:
            heads[2] = _dep(heads[2])
    return heads


def _k(fn):
    return 100 if fn.startswith("multi_pose") else 40


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("hw", [None, (128, 128), (96, 160)], ids=["default", "hot", "96x160"])
def test_half_all_heads(fn, dt, hw):
    heads = [t.to(dt) for t in _heads_for(fn, 3, hw, seed=21)]
    _half_check(_fns()[fn], heads, _k(fn))


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("K", [1, 100, 256, 300])
def test_half_k(fn, K):
    heads = [t.to(torch.bfloat16) for t in _heads_for(fn, 2, (128, 128), seed=K)]
    _half_check(_fns()[fn], heads, K)


MIXED = {   # one dtype pattern per function (f = fp32, b = bf16, h = fp16), in argument order
    "multi_pose": "bfhbhf", "multi_pose_logits": "hbfhbb", "ddd": "fbhfbh", "ddd_logits": "bfbhhf"}
_DT = {"f": torch.float32, "b": torch.bfloat16, "h": torch.float16}


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("hw", [(128, 128), (96, 320)], ids=["hot", "kitti"])
def test_mixed_dtypes(fn, hw):
    heads = [t.to(_DT[c]) for t, c in zip(_heads_for(fn, 2, hw, seed=31), MIXED[fn])]
    _half_check(_fns()[fn], heads, _k(fn))


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("B", [1, 8, 64])
def test_half_pose_batch(B, dt):
    for fn in ("multi_pose", "multi_pose_logits"):
        heads = [t.to(dt) for t in _heads_for(fn, B, seed=40 + B)]
        _half_check(_fns()[fn], heads, 100)


def _big_pose(dt, logits):
    """tests/big_inputs.multi_pose_inputs() (2 x 128 x 128, 17 joints) with heat and hm_hp as maps or as logits,
    rounded to dt: the rounding puts many ties at the K-th score."""
    heat, wh, kps, reg, hm_hp, off = [torch.from_numpy(a).cuda() for a in BI.multi_pose_inputs()]
    if logits:
        heat, hm_hp = [torch.logit(m.double(), eps=1e-6).float() for m in (heat, hm_hp)]
    return [t.to(dt) for t in (heat, wh, kps, reg, hm_hp, off)]


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("fn", ["multi_pose", "multi_pose_logits"])
def test_half_big_inputs_with_ties(fn, dt):
    heads = _big_pose(dt, fn.endswith("logits"))
    dets = _half_check(_fns()[fn], heads, 100)
    s = dets[..., 4]
    assert any(int((s[b] == s[b, -1]).sum()) > 1 for b in range(s.shape[0])), "expected ties at the K-th score"


def _offset_view(t):
    """A contiguous copy of t whose base lies one element past a fresh allocation: not 16-byte aligned."""
    flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = flat[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("fn", FNS)
def test_misaligned_maps(fn, dt):
    """Hot geometry, but the maps' base is not 16-byte aligned: the widening path, same dets."""
    heads = [t.to(dt) for t in _heads_for(fn, 2, (128, 128), seed=51)]
    aligned = _fns()[fn](*heads, K=_k(fn))
    heads = [_offset_view(t) for t in heads]
    got = _half_check(_fns()[fn], heads, _k(fn))
    assert torch.equal(got, aligned)
    if fn.startswith("multi_pose"):   # only the joint map misaligned, and only the centre map
        for i in (0, 4):
            hs = list(heads)
            hs[i] = hs[i].contiguous().clone()
            assert torch.equal(_half_check(_fns()[fn], hs, _k(fn)), aligned)


@pytest.mark.parametrize("fn", FNS)
def test_non_default_stream(fn):
    heads = [t.to(torch.float16) for t in _heads_for(fn, 4, seed=61)]
    want = _fns()[fn](*[_up(t) for t in heads], K=_k(fn))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = _fns()[fn](*heads, K=_k(fn))
    s.synchronize()
    assert torch.equal(got, want)


# ------------------------------------------------------------------ the big multi_pose golden, fed as logits
def test_big_golden_multi_pose_as_logits():
    """test_big_golden's multi_pose inputs as logits: multi_pose_decode_from_logits equals multi_pose_decode on
    torch.sigmoid of those logits (not the golden itself: the sigmoid does not give the original maps back)."""
    heads = _big_pose(torch.float32, True)
    _pose_logits_check(heads, K=100)
    _pose_logits_check(_variant(heads, "no_reg"), K=100)
    _pose_logits_check(_variant(heads, "no_offset"), K=100)

"""GPU: multi_pose_decode and ddd_decode bit for bit, with no tolerance anywhere.

* Every case of tests/golden/pose_ddd_edges.npz (thresholds, box edges, the distance limit, distance ties,
  degenerate boxes, K, optional heads, NaN and inf in every regression head) on the fp32 entry points, on the
  dtype-generic `_ex` kernels with the same fp32 heads, and with every head that bf16 / fp16 represent exactly
  cast to that dtype.  Against the library-mode oracle always, and against the reference's golden wherever the
  library's non-finite rule does not change the answer.
* Seeded sweeps against the oracle at the hot 128x128 selection, KITTI-like 96x320, 40x56 and odd maps, K from 1
  to 1024, J = 1 and 17, and B = 64 (B*J > 1024 joint planes).
* The joint threshold in logit space: multi_pose_decode_from_logits at the logits whose CUDA sigmoid falls on
  either side of float32(0.1).
* The flip test: multi_pose_decode_flip_from_logits against the reference's composition in torch ops.
"""
import numpy as np
import pytest
import torch

from helpers import assert_dets_bits, golden
from oracle import decode_np as O
from test_pose_ddd_edges import DDD, LIBRARY_CHANGES, POSE, ddd_heads, pose_heads

pytestmark = pytest.mark.gpu
G = golden("pose_ddd_edges")


def dev(*arrs):
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


def exact_in(t, dt):
    """t cast to dt when that loses nothing (inf and NaN included), else t."""
    if t is None:
        return None
    c = t.to(dt)
    back = c.float()
    same = (back == t) | (torch.isnan(back) & torch.isnan(t))
    return c if bool(same.all()) else t


def cast_exact(heads, dt):
    out = [exact_in(t, dt) for t in heads]
    return out, any(t is not None and t.dtype == dt for t in out)


def pose(heads, K, fn=None):
    from centernet_b200 import decode as D
    heat, wh, kps, reg, hm_hp, off = heads
    return (fn or D.multi_pose_decode)(heat, wh, kps, reg=reg, hm_hp=hm_hp, hp_offset=off, K=K)


def ddd(heads, K, fn=None):
    from centernet_b200 import decode as D
    heat, rot, dep, dim, wh, reg = heads
    return (fn or D.ddd_decode)(heat, rot, dep, dim, wh=wh, reg=reg, K=K)


# ------------------------------------------------------------------ the golden edge cases
@pytest.mark.parametrize("name", POSE)
def test_multi_pose_edge_case(name):
    from centernet_b200 import decode as D
    ins, K = pose_heads(name), int(G[name + "__K"])
    want = O.multi_pose_decode(*ins, K=K, nonfinite="library")
    if name not in LIBRARY_CHANGES:
        assert_dets_bits(G[name + "__dets"], want, what=name + " oracle")
    heads = dev(*ins)
    assert_dets_bits(want, pose(heads, K).cpu().numpy(), what=name + " fp32")
    ex = D._multi_pose_ex(*heads, K, 0).cpu().numpy()                  # the dtype-generic kernel on fp32 heads
    assert_dets_bits(want, ex, what=name + " _ex fp32")
    for dt in (torch.bfloat16, torch.float16):
        half, any_half = cast_exact(heads, dt)
        if any_half:
            assert_dets_bits(want, pose(half, K).cpu().numpy(), what="%s %s" % (name, dt))


@pytest.mark.parametrize("name", DDD)
def test_ddd_edge_case(name):
    from centernet_b200 import decode as D
    ins, K = ddd_heads(name), int(G[name + "__K"])
    want = O.ddd_decode(*ins[:4], wh=ins[4], reg=ins[5], K=K)
    assert_dets_bits(G[name + "__dets"], want, score_col=2, what=name + " oracle")
    heads = dev(*ins)
    # the oracle shares the kernels' order of equal scores, so even the zero-score rows agree in place
    assert_dets_bits(want, ddd(heads, K).cpu().numpy(), score_col=2, what=name + " fp32")
    got = D._ddd_ex(*heads, K, 0).cpu().numpy()
    assert_dets_bits(want, got, score_col=2, what=name + " _ex fp32")
    for dt in (torch.bfloat16, torch.float16):
        half, any_half = cast_exact(heads, dt)
        if any_half:
            assert_dets_bits(want, ddd(half, K).cpu().numpy(), score_col=2, what="%s %s" % (name, dt))


# ------------------------------------------------------------------ seeded sweeps against the oracle
def _noise(rng, shape, bias):
    return (1 / (1 + np.exp(-(rng.standard_normal(shape) - bias)))).astype(np.float32)


def _pose_inputs(B, J, H, W, seed):
    rng = np.random.default_rng(seed)
    heat = _noise(rng, (B, 1, H, W), 2.19)
    wh = (rng.random((B, 2, H, W)) * 30).astype(np.float32)
    kps = (rng.standard_normal((B, 2 * J, H, W)) * 6).astype(np.float32)
    reg = rng.random((B, 2, H, W), dtype=np.float32)
    hm_hp = _noise(rng, (B, J, H, W), 1.0)
    off = rng.random((B, 2, H, W), dtype=np.float32)
    return [heat, wh, kps, reg, hm_hp, off]


POSE_SWEEP = [  # B, J, H, W, K
    (2, 17, 128, 128, 100), (3, 17, 128, 128, 256), (2, 1, 128, 128, 257), (2, 1, 128, 128, 1024),
    (1, 17, 128, 128, 1), (2, 17, 96, 320, 100), (3, 17, 40, 56, 31), (2, 1, 37, 61, 257), (2, 2, 5, 7, 35),
    (64, 17, 128, 128, 100), (8, 1, 33, 45, 1024)]


@pytest.mark.parametrize("B,J,H,W,K", POSE_SWEEP)
def test_multi_pose_sweep(B, J, H, W, K):
    ins = _pose_inputs(B, J, H, W, seed=B * 1000 + J * 10 + K)
    want = O.multi_pose_decode(*ins, K=K, nonfinite="library")
    got = pose(dev(*ins), K).cpu().numpy()
    assert_dets_bits(want, got, what="multi_pose B=%d J=%d %dx%d K=%d" % (B, J, H, W, K))
    if B * J > 1024 or K >= 256:   # variants without reg and without hp_offset through the same selections
        ins_nr = ins[:3] + [None, ins[4], None]
        want = O.multi_pose_decode(*ins_nr, K=K, nonfinite="library")
        assert_dets_bits(want, pose(dev(*ins_nr), K).cpu().numpy(), what="multi_pose no reg / offset")


DDD_SWEEP = [  # B, C, H, W, K
    (2, 3, 96, 320, 100), (2, 1, 128, 128, 1024), (3, 3, 40, 56, 257), (64, 3, 32, 32, 100), (2, 3, 7, 9, 31),
    (1, 1, 128, 128, 1)]


@pytest.mark.parametrize("B,C,H,W,K", DDD_SWEEP)
def test_ddd_sweep(B, C, H, W, K):
    rng = np.random.default_rng(B * 100 + C * 10 + K)
    heat = _noise(rng, (B, C, H, W), 2.19)
    heads = [(rng.standard_normal((B, ch, H, W)) * 8).astype(np.float32) for ch in (8, 1, 3, 2, 2)]
    for wh_reg in (True, False):
        ins = [heat] + heads[:3] + (heads[3:] if wh_reg else [None, None])
        want = O.ddd_decode(*ins[:4], wh=ins[4], reg=ins[5], K=K)
        got = ddd(dev(*ins), K).cpu().numpy()
        assert_dets_bits(want, got, score_col=2, what="ddd B=%d C=%d %dx%d K=%d" % (B, C, H, W, K))


# ------------------------------------------------------------------ the joint threshold in logit space
def _logits_around(target):
    """Logits whose torch CUDA sigmoid is the largest value below target, the smallest above it, and target
    itself if some logit gives exactly that."""
    x0 = float(np.log(target / (1 - target)))
    c = torch.tensor([x0], dtype=torch.float32).view(torch.int32)
    bits = torch.arange(int(c) - 4096, int(c) + 4096, dtype=torch.int32)
    xs = bits.view(torch.float32).cuda()
    s = torch.sigmoid(xs)
    t = torch.tensor(target, dtype=torch.float32, device="cuda")
    out = {"lt": float(xs[s < t].max()), "gt": float(xs[s > t].min())}
    if bool((s == t).any()):
        out["eq"] = float(xs[s == t][0])
    return out


def test_joint_threshold_in_logit_space():
    from centernet_b200 import decode as D
    xs = _logits_around(np.float32(0.1))
    B, H, W, J, K = len(xs), 128, 128, 2, 4
    hm = torch.full((B, 1, H, W), -20.0, device="cuda")
    hm_hp = torch.full((B, J, H, W), -20.0, device="cuda")
    wh = torch.full((B, 2, H, W), 6.0, device="cuda")
    kps = torch.zeros((B, 2 * J, H, W), device="cuda")
    reg = torch.full((B, 2, H, W), 0.25, device="cuda")
    off = torch.full((B, 2, H, W), 0.5, device="cuda")
    for i, (y, x) in enumerate(((40, 40), (10, 100), (100, 10), (90, 90))):
        hm[:, 0, y, x] = 3.0 - 0.5 * i
        kps[:, 0, y, x] = 0.75                      # joint 0 regressed to (x + 0.75, y + 0.5)
        kps[:, 1, y, x] = 0.5
    for b, x in enumerate(xs.values()):
        hm_hp[b, 0, 40, 40] = x                      # candidate (40.5, 40.5) next to the first detection's joint 0
    hm_hp[:, 1, 60, 60] = 1.0
    heads = [hm, wh, kps, reg, hm_hp, off]
    got = pose(heads, K, fn=D.multi_pose_decode_from_logits)
    want = pose([torch.sigmoid(hm), wh, kps, reg, torch.sigmoid(hm_hp), off], K)
    assert torch.equal(got, want)
    snapped = got[:, 0, 5].cpu().numpy() == np.float32(40.5)
    assert list(snapped) == [k == "gt" for k in xs], (list(xs), got[:, 0, 5:7])
    for dt in (torch.bfloat16, torch.float16):   # the other heads in half precision: the same dets
        half = [heads[0], wh.to(dt), kps.to(dt), reg.to(dt), hm_hp, off.to(dt)]
        assert torch.equal(pose(half, K, fn=D.multi_pose_decode_from_logits), got)


# ------------------------------------------------------------------ flip test (detectors/multi_pose.py:43-50)
FLIP_IDX = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]


def _flip_lr(x):
    tmp = torch.flip(x, [3]).clone()
    for a, b in FLIP_IDX:
        tmp[:, [a, b]] = tmp[:, [b, a]]
    return tmp


def _flip_lr_off(x):
    n, c, h, w = x.shape
    tmp = torch.flip(x, [3]).clone().view(n, 17, 2, h, w)
    tmp[:, :, 0] *= -1
    for a, b in FLIP_IDX:
        tmp[:, [a, b]] = tmp[:, [b, a]]
    return tmp.view(n, c, h, w)


@pytest.mark.parametrize("n,H,W,K", [(1, 128, 128, 100), (2, 96, 160, 64), (1, 40, 56, 31)])
@pytest.mark.parametrize("variant", ["full", "no_reg_off", "no_hm_hp"])
def test_flip_test(n, H, W, K, variant):
    from centernet_b200 import decode as D
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + K)
    r = lambda c, s=1.0, o=0.0: torch.randn(2 * n, c, H, W, device="cuda", generator=g) * s + o  # noqa: E731
    hm, wh, hps, reg, hm_hp, off = r(1, 2, -2.19), r(2, 10, 20), r(34, 6), r(2, 0.3, 0.5), r(17, 2, -2.19), r(2, 0.3, 0.5)
    if variant == "no_reg_off":
        reg = off = None
    if variant == "no_hm_hp":
        hm_hp = off = None
    got = D.multi_pose_decode_flip_from_logits(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=off, flip_idx=FLIP_IDX,
                                               K=K)
    h = torch.sigmoid(hm)
    heat = (h[:n] + torch.flip(h[n:], [3])) / 2
    whm = (wh[:n] + torch.flip(wh[n:], [3])) / 2
    hpsm = (hps[:n] + _flip_lr_off(hps[n:])) / 2
    hp = None
    if hm_hp is not None:
        s = torch.sigmoid(hm_hp)
        hp = (s[:n] + _flip_lr(s[n:])) / 2
    want = D.multi_pose_decode(heat, whm, hpsm, reg=None if reg is None else reg[:n], hm_hp=hp,
                               hp_offset=None if off is None else off[:n], K=K)
    assert torch.equal(got, want)
    # and the composition itself against the oracle
    ora = O.multi_pose_decode(*[None if t is None else t.cpu().numpy()
                                for t in (heat, whm, hpsm, None if reg is None else reg[:n], hp,
                                          None if off is None else off[:n])], K=K, nonfinite="library")
    assert_dets_bits(ora, want.cpu().numpy(), what="flip composition")

"""Generates tests/golden/loss_edges.npz: the reference's training losses and target splat at the inputs
where a fused kernel is most likely to part from them -- non-finite predictions and targets, the _sigmoid
clamp points, centres on and outside the map border, radius 0 and radii larger than the map, duplicate
centres, and the Reg*Loss family with float / bool / uint8 masks, repeated indices and the smooth-L1 branch
point.  Runs the UNMODIFIED reference functions (models/losses.py, models/utils.py, utils/image.py) on the
CPU in fp32 and stores their inputs, outputs and autograd gradients.

Run in the build container only:  python tests/golden/make_golden_loss_edges.py
The GPU box has no /root/reference; tests read the committed .npz file.  The output is deterministic:
re-running it reproduces the file value for value.
"""
import hashlib
import os
import sys
import warnings

import numpy as np
import torch

REF = "/root/reference/src/lib"
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))

from models import losses as L  # noqa: E402
from models import utils as U  # noqa: E402
from utils import image as I  # noqa: E402

F32 = np.float32
GAUSS_RMAX = 200    # gaussian2D digests for r = 0 .. GAUSS_RMAX


def ulps(x, k):
    """x moved by k fp32 ulps (k may be negative)."""
    x = F32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, F32(np.inf) if k > 0 else F32(-np.inf), dtype=F32)
    return F32(x)


def sigmoid_crossing(level, rising=True):
    """Smallest fp32 x with fp32 sigmoid(x) >= level (torch's CPU sigmoid, as _sigmoid runs it)."""
    lo, hi = F32(-30), F32(30)
    sig = lambda v: torch.sigmoid(torch.tensor([v], dtype=torch.float32)).item()
    while np.nextafter(lo, hi, dtype=F32) != hi:
        mid = F32((float(lo) + float(hi)) / 2)
        if mid in (lo, hi):
            break
        if sig(mid) >= level:
            hi = mid
        else:
            lo = mid
    return hi


# ------------------------------------------------------------------ focal loss
def focal_ref(x, gt, logits):
    """Reference loss and its autograd gradient w.r.t. x (pred, or the logit through _sigmoid)."""
    xt = torch.from_numpy(np.asarray(x, F32).copy()).requires_grad_(True)
    g = torch.from_numpy(np.asarray(gt, F32).copy())
    pred = U._sigmoid(xt.clone()) if logits else xt
    loss = L._neg_loss(pred, g)
    loss.backward()
    return F32(loss.item()), xt.grad.numpy().astype(F32)


def focal_cases(rng):
    n = 13
    base_gt = rng.uniform(0.0, 0.9, n).astype(F32)
    base_gt[[1, 8]] = 1.0                       # two positives
    base_p = rng.uniform(0.05, 0.95, n).astype(F32)
    base_l = rng.normal(0.0, 2.0, n).astype(F32)
    nan, inf = F32(np.nan), F32(np.inf)
    cases = {}

    def case(name, x, gt, logits):
        cases[name] = (np.asarray(x, F32), np.asarray(gt, F32), int(logits))

    def with_(arr, **kv):
        a = arr.copy()
        for k, v in kv.items():
            a[int(k[1:])] = v
        return a

    nopos = np.minimum(base_gt, F32(0.9))
    # pred given directly (_neg_loss)
    case("pred_nan", with_(base_p, i3=nan), base_gt, 0)
    case("gt_nan", base_p, with_(base_gt, i5=nan), 0)
    case("p1_pos", with_(base_p, i1=1.0), base_gt, 0)          # log(1 - 1) * 1 * 0 * 0 = NaN
    case("p0_neg", with_(base_p, i4=0.0), base_gt, 0)          # log(0) * 1 * 0 = NaN
    case("p1_neg", with_(base_p, i4=1.0), base_gt, 0)          # +inf
    case("p0_pos", with_(base_p, i8=0.0), base_gt, 0)          # +inf
    case("p0_neg_nopos", with_(base_p, i4=0.0), nopos, 0)      # num_pos == 0: the NaN positive term is dropped
    case("p1_neg_nopos", with_(base_p, i4=1.0), nopos, 0)
    case("p1_pos_p0_neg", with_(base_p, i1=1.0, i4=0.0), base_gt, 0)
    case("pred_out_of_range", with_(base_p, i2=1.5, i3=-0.25), base_gt, 0)
    case("gt_above1", base_p, with_(base_gt, i6=1.5, i7=np.nextafter(F32(1), F32(2), dtype=F32)), 0)
    case("gt_inf", base_p, with_(base_gt, i6=inf), 0)
    case("gt_neg", base_p, with_(base_gt, i6=-0.5, i7=-inf), 0)
    case("gt_below1", base_p, with_(base_gt, i6=np.nextafter(F32(1), F32(0), dtype=F32), i7=0.0), 0)
    case("pred_nan_nopos", with_(base_p, i3=nan), nopos, 0)
    # raw logits (_sigmoid + _neg_loss)
    case("logit_nan", with_(base_l, i3=nan), base_gt, 1)
    case("logit_nan_pos", with_(base_l, i1=nan), base_gt, 1)
    case("logit_gt_nan", base_l, with_(base_gt, i5=nan), 1)
    case("logit_clamped_gt_nan", with_(base_l, i5=20.0, i6=-20.0), with_(base_gt, i5=nan, i6=nan), 1)
    case("logit_gt_inf", with_(base_l, i5=20.0), with_(base_gt, i5=inf, i6=inf), 1)
    case("logit_gt_above1", base_l, with_(base_gt, i6=1.5), 1)
    # logits at +-inf, +-100 and around both clamp points, each at a positive and at a negative pixel
    lo_x, hi_x = sigmoid_crossing(F32(1e-4)), sigmoid_crossing(F32(1 - 1e-4))
    xs = [inf, -inf, F32(100), F32(-100), F32(0)]
    for c in (F32(-9.2103), F32(9.2103), lo_x, hi_x):
        xs += [ulps(c, k) for k in range(-4, 5)]
    xs = np.asarray(xs, F32)
    x2 = np.repeat(xs, 2)
    g2 = np.tile(np.asarray([1.0, 0.3], F32), len(xs))
    case("logit_extremes", x2, g2, 1)
    return cases, dict(sigmoid_lo_crossing=lo_x, sigmoid_hi_crossing=hi_x)


# ------------------------------------------------------------------ Reg*Loss family
REG_CLASSES = (L.RegL1Loss, L.RegLoss, L.NormRegL1Loss, L.RegWeightedL1Loss)


def reg_ref(mode, output, mask, ind, target):
    o = torch.from_numpy(output.copy()).requires_grad_(True)
    loss = REG_CLASSES[mode]()(o, torch.from_numpy(mask.copy()), torch.from_numpy(ind.copy()),
                               torch.from_numpy(target.copy()))
    loss.backward()
    return F32(loss.item()), o.grad.numpy().astype(F32)


def reg_cases(rng):
    B, M, D, H, W = 2, 6, 2, 4, 4
    HW = H * W
    cases = {}

    def base():
        output = rng.normal(0, 1.5, (B, D, H, W)).astype(F32)
        ind = rng.integers(0, HW, (B, M)).astype(np.int64)
        target = rng.normal(0, 1.5, (B, M, D)).astype(F32)
        return output, ind, target

    for mode in range(4):
        def add(name, output, mask, ind, target):
            tgt = np.abs(target) + F32(0.5) if mode == 2 else target
            cases["%s_m%d" % (name, mode)] = (mode, output, mask, ind, tgt.astype(F32))

        shp = (B, M, D) if mode == 3 else (B, M)
        o, i, t = base()
        add("frac", o, rng.choice(np.asarray([0, 0.25, 0.5, 1.0, 1.5], F32), shp), i, t)
        o, i, t = base()
        add("bool", o, rng.random(shp) > 0.4, i, t)
        o, i, t = base()
        add("u8_2", o, rng.choice(np.asarray([0, 1, 2], np.uint8), shp), i, t)
        o, i, t = base()
        add("zero", o, np.zeros(shp, F32 if mode == 3 else np.uint8), i, t)
        o, i, t = base()
        i[0, :] = i[0, 0]                       # one pixel gathered six times
        i[1, 3:] = i[1, 1]
        add("dup_ind", o, rng.choice(np.asarray([0.5, 1.0, 2.0], F32), shp), i, t)
        # |pred - target| at 1 exactly and at the fp32 neighbours of 1 (the smooth-L1 branch point)
        o = rng.normal(0, 1.5, (B, D, H, W)).astype(F32)
        i = np.stack([rng.permutation(HW)[:M] for _ in range(B)]).astype(np.int64)
        t = np.zeros((B, M, D), F32)
        deltas = np.asarray([1, -1, np.nextafter(F32(1), F32(0), dtype=F32), np.nextafter(F32(1), F32(2), dtype=F32),
                             -np.nextafter(F32(1), F32(0), dtype=F32), -np.nextafter(F32(1), F32(2), dtype=F32)], F32)
        for b in range(B):
            for m in range(M):
                for d in range(D):
                    if mode == 2:
                        t[b, m, d] = F32(1)             # pred / (1 + 1e-4) against 1
                    o[b, d, i[b, m] // W, i[b, m] % W] = deltas[(b * M + m + d) % len(deltas)] + t[b, m, d]
        cases["sl1_edge_m%d" % mode] = (mode, o, np.ones((B, M, D) if mode == 3 else (B, M), F32), i, t)
    return cases


# ------------------------------------------------------------------ target splat
def splat_cases():
    """name -> (B, C, H, W, [(b, cls, cx, cy, r, valid), ...])."""
    cases = {}
    # centres on every border and corner
    H, W, objs = 12, 16, []
    pts = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (W // 2, 0), (0, H // 2), (W - 1, H // 2), (W // 2, H - 1)]
    for k, (x, y) in enumerate(pts):
        objs.append((0, k, x, y, 2 + k % 3, 1))
    cases["borders"] = (1, len(pts), H, W, objs)
    # centres outside the map by 1 .. r+1 on each side and beyond each corner, one class plane each
    H, W, r, objs = 11, 13, 3, []
    k = 0
    for d in range(1, r + 2):
        for (x, y) in ((-d, H // 2), (W - 1 + d, H // 2), (W // 2, -d), (W // 2, H - 1 + d),
                       (-d, -d), (W - 1 + d, H - 1 + d), (-d, H - 1 + d), (W - 1 + d, -d)):
            objs.append((0, k, x, y, r, 1))
            k += 1
    cases["outside"] = (1, k, H, W, objs)
    # the 8x8, r=2 example: x=-1 paints 10 pixels, x=9 paints 5
    cases["outside_8x8"] = (1, 2, 8, 8, [(0, 0, -1, 3, 2, 1), (0, 1, 9, 4, 2, 1)])
    # radius 0 and radii larger than the map, inside and outside it
    cases["radius_extremes"] = (2, 3, 8, 8, [(0, 0, 3, 4, 0, 1), (0, 0, 7, 7, 0, 1), (0, 1, 2, 5, 30, 1),
                                             (0, 2, -5, 3, 30, 1), (1, 0, 0, 0, 11, 1), (1, 1, 9, -2, 20, 1),
                                             (1, 2, 4, 4, 0, 1), (1, 2, 5, 4, 9, 1)])
    # duplicate (cls, cx, cy) with different radii (one positive, the largest Gaussian wins)
    cases["duplicates"] = (2, 2, 10, 12, [(0, 0, 5, 5, 1, 1), (0, 0, 5, 5, 4, 1), (0, 0, 5, 5, 2, 1),
                                          (0, 1, 0, 9, 3, 1), (0, 1, 0, 9, 0, 1), (0, 1, 4, 2, 2, 0),
                                          (1, 1, 11, 0, 5, 1), (1, 1, 11, 0, 2, 1), (1, 0, -1, 4, 2, 1),
                                          (1, 0, -1, 4, 3, 1)])
    return cases


def splat_ref(B, C, H, W, objs):
    M = max(sum(1 for o in objs if o[0] == b) for b in range(B))
    cls = np.zeros((B, M), np.int32); cx = np.zeros((B, M), np.int32); cy = np.zeros((B, M), np.int32)
    rad = np.zeros((B, M), np.int32); val = np.zeros((B, M), np.uint8)
    fill = [0] * B
    hm = np.zeros((B, C, H, W), F32)
    for (b, c, x, y, r, v) in objs:
        m = fill[b]; fill[b] += 1
        cls[b, m], cx[b, m], cy[b, m], rad[b, m], val[b, m] = c, x, y, r, v
        if v:
            I.draw_umich_gaussian(hm[b, c], (x, y), r)
    return cls, cx, cy, rad, val, hm


def gauss_digest(r):
    d = 2 * r + 1
    return hashlib.sha256(I.gaussian2D((d, d), sigma=d / 6).astype(F32).tobytes()).digest()


def main():
    warnings.simplefilter("ignore")
    rng = np.random.default_rng(2024)
    out = {}

    fc, crossings = focal_cases(rng)
    out["focal_names"] = np.asarray(sorted(fc))
    for name in sorted(fc):
        x, gt, logits = fc[name]
        loss, grad = focal_ref(x, gt, logits)
        out.update({"f_%s_x" % name: x, "f_%s_gt" % name: gt, "f_%s_logits" % name: np.int32(logits),
                    "f_%s_loss" % name: loss, "f_%s_grad" % name: grad})
    out.update({k: np.float32(v) for k, v in crossings.items()})

    rc = reg_cases(rng)
    out["reg_names"] = np.asarray(sorted(rc))
    for name in sorted(rc):
        mode, o, mask, ind, t = rc[name]
        loss, grad = reg_ref(mode, o, mask, ind, t)
        out.update({"r_%s_mode" % name: np.int32(mode), "r_%s_output" % name: o, "r_%s_mask" % name: mask,
                    "r_%s_ind" % name: ind, "r_%s_target" % name: t, "r_%s_loss" % name: loss,
                    "r_%s_grad" % name: grad})

    sc = splat_cases()
    out["splat_names"] = np.asarray(sorted(sc))
    for name in sorted(sc):
        B, C, H, W, objs = sc[name]
        cls, cx, cy, rad, val, hm = splat_ref(B, C, H, W, objs)
        pred = np.clip(1 / (1 + np.exp(-rng.normal(-1.0, 2.0, (B, C, H, W)))), 1e-4, 1 - 1e-4).astype(F32)
        loss, grad = focal_ref(pred, hm, 0)
        out.update({"s_%s_cls" % name: cls, "s_%s_cx" % name: cx, "s_%s_cy" % name: cy, "s_%s_rad" % name: rad,
                    "s_%s_valid" % name: val, "s_%s_chw" % name: np.asarray([C, H, W], np.int32),
                    "s_%s_hm" % name: hm, "s_%s_pred" % name: pred, "s_%s_loss" % name: loss,
                    "s_%s_grad" % name: grad})

    # gaussian2D of every radius 0..GAUSS_RMAX, cast to fp32 (what draw_umich_gaussian stores): SHA-256 digests
    out["gauss_digest"] = np.frombuffer(b"".join(gauss_digest(r) for r in range(GAUSS_RMAX + 1)),
                                        np.uint8).reshape(GAUSS_RMAX + 1, 32).copy()

    path = os.path.join(HERE, "loss_edges.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()

"""Generates tests/golden/ddd_tail.npz: the UNMODIFIED reference's DddDetector.pre_process (detectors/ddd.py:30-55),
post_process + merge_outputs (:75-88) and utils.post_process.ddd_post_process, called as plain functions on a stub
`self` that carries `opt`, `num_classes`, `mean`, `std` and `calib`.  The metas of the tail cases are what
pre_process returns for KITTI-sized images (c = (w/2, h/2), s = int32 [w, h] or the input size with keep_res).
Build container only; tests read the .npz.  Layout: tests/ddd_tail_cases.py.

    python tests/golden/make_golden_ddd_tail.py
"""
import os
import sys
import types
import zlib

import numpy as np
import torch

REF = "/root/reference/src/lib"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(HERE))                       # tests/: ddd_tail_cases
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))      # the repository: oracle


def _stub(name, **attrs):
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    sys.modules[name] = mod
    return mod


# progress and matplotlib are not installed here; the detector methods use neither.  models.model pulls in the
# networks (and the compiled DCNv2 extension) for create_model / load_model, which they do not use either.
_stub("progress", bar=_stub("progress.bar", Bar=object))
_stub("matplotlib", pyplot=_stub("matplotlib.pyplot"))
_stub("models.model", create_model=None, load_model=None)

from detectors import ddd as DDD  # noqa: E402
from utils import post_process as PP  # noqa: E402
from utils.image import get_affine_transform  # noqa: E402

import ddd_tail_cases as CS  # noqa: E402

F32 = np.float32
NAN = F32(np.nan)


def opt(keep_res=False):
    ih, iw = CS.INPUT_HW
    return types.SimpleNamespace(input_h=ih, input_w=iw, keep_res=keep_res, down_ratio=4, output_h=ih // 4,
                                 output_w=iw // 4, num_classes=CS.NUM_CLASSES, peak_thresh=CS.PEAK_THRESH)


def detector(keep_res=False):
    calib = np.array([[707.0493, 0, 604.0814, 45.75831], [0, 707.0493, 180.5066, -0.3454157],
                      [0, 0, 1., 0.004981016]], dtype=np.float32)
    return types.SimpleNamespace(opt=opt(keep_res), num_classes=CS.NUM_CLASSES, calib=calib,
                                 mean=np.array(CS.MEAN, F32).reshape(1, 1, 3), std=np.array(CS.STD, F32).reshape(1, 1, 3))


def ref_meta(h, w, keep_res, calib=None, seed=0):
    this = detector(keep_res)
    _, meta = DDD.DddDetector.pre_process(this, CS.ddd_image(h, w, seed), 1, calib)
    return meta


def other_calib(rng):
    """A KITTI-like projection matrix of another camera."""
    P = np.array(detector().calib, np.float64)
    P[0, 0] = P[1, 1] = P[0, 0] * rng.uniform(0.95, 1.05)
    P[0, 2] += rng.uniform(-8, 8); P[1, 2] += rng.uniform(-4, 4)
    P[0, 3] = rng.uniform(-400, 50); P[1, 3] = rng.uniform(-2, 2); P[2, 3] = rng.uniform(-0.01, 0.01)
    return P.astype(F32)


def ddd_rows(rng, B, K, out_hw, classes=(0, 1, 2)):
    """[B, K, 18] ddd_decode-shaped rows: x, y = integer peak + float32 offset, score (descending), rot[8], depth
    through 1 / (sigmoid + 1e-6) - 1 in float32 (about 1e6 and about -1e-6 included), dim[3], w, h, class."""
    oh, ow = out_hw
    d = np.zeros((B, K, 18), F32)
    d[..., 0] = rng.integers(0, ow, (B, K)).astype(F32) + rng.random((B, K)).astype(F32)
    d[..., 1] = rng.integers(0, oh, (B, K)).astype(F32) + rng.random((B, K)).astype(F32)
    d[..., 2] = np.sort(rng.random((B, K)).astype(F32), axis=1)[:, ::-1]
    d[..., 3:11] = rng.normal(0, 1.5, (B, K, 8))
    raw = torch.from_numpy(rng.normal(0, 2, (B, K)).astype(F32))
    raw[:, 0], raw[:, 1] = -30.0, 30.0
    d[..., 11] = (1. / (raw.sigmoid() + 1e-6) - 1.).numpy()
    d[..., 12:15] = np.array([1.5, 1.6, 3.9], F32) + rng.normal(0, 0.3, (B, K, 3)).astype(F32)
    d[..., 15:17] = rng.uniform(1, 60, (B, K, 2))
    d[..., 17] = np.asarray(classes, F32)[rng.integers(0, len(classes), (B, K))]
    return d


def x_onto(t, target):
    """A float32 x whose back-projection (t0 x + t1 y) + t2, rounded to float32, is exactly `target` (t1 = 0)."""
    x = F32((float(target) - t[0, 2]) / t[0, 0])
    for _ in range(64):
        u = F32(t[0, 0] * np.float64(x) + t[0, 2])
        if u == target:
            return x
        x = np.nextafter(x, F32(np.inf) if u < target else F32(-np.inf))
    raise RuntimeError("no float32 x maps onto %r" % target)


def add_specials(d, meta, P):
    """Edge rows in image 0: scores at, just above, NaN and +inf at the cut; class ids -0.0, 3, NaN, 1.5; a bin tie;
    a NaN in the unselected bin (either way); alpha = float32(pi) with u = P[0, 2], so rot_y = float32(pi) exactly."""
    r = d[0]
    r[2, 2], r[3, 2], r[4, 2], r[5, 2] = F32(0.2), np.nextafter(F32(0.2), F32(1)), NAN, F32(np.inf)
    r[6:10, 2] = 0.9
    r[6, 17], r[7, 17], r[8, 17], r[9, 17] = F32(-0.0), F32(3), NAN, F32(1.5)
    r[10:14, 2] = 0.9
    r[10:14, 17] = 0
    r[10, 8] = r[10, 4]                              # rot[1] == rot[5]: bin 2
    r[11, 4], r[11, 8], r[11, 9] = 2.0, 0.0, NAN     # bin 1 selected, NaN sin in bin 2
    r[12, 4], r[12, 8], r[12, 5] = 0.0, 2.0, NAN     # bin 2 selected, NaN sin in bin 1
    r[13, 4], r[13, 8], r[13, 9], r[13, 10] = 0.0, 1.0, 1.0, 0.0     # bin 2, atan2(1, 0) + pi / 2 = float32(pi)
    t = get_affine_transform(meta["c"], meta["s"], 0, (CS.INPUT_HW[1] // 4, CS.INPUT_HW[0] // 4), inv=1)
    r[13, 0] = x_onto(t, P[0, 2])


def run_merge(dets, metas):
    """DddDetector.post_process + merge_outputs once per image, each with its own meta."""
    this = detector()
    res = []
    for i in range(dets.shape[0]):
        det = DDD.DddDetector.post_process(this, torch.from_numpy(dets[i:i + 1].copy()), metas[i])
        res.append(DDD.DddDetector.merge_outputs(this, [det]))
    return res


def run_dropin(dets, metas):
    return PP.ddd_post_process(dets.copy(), [m["c"] for m in metas], [m["s"] for m in metas],
                               [m["calib"] for m in metas], opt())


def tail_cases(rng):
    """(name, form, [(h, w, keep_res, calib)], K, specials, classes)."""
    kitti = [(375, 1242), (370, 1224), (374, 1238), (376, 1241), (370, 1226)]
    cal = [other_calib(rng) for _ in range(3)]
    three = [(375, 1242, False, cal[0]), (370, 1224, False, cal[1]), (376, 1241, False, cal[2])]
    return [("kitti_default", 0, [(375, 1242, False, None)], 100, True, (0, 1, 2)),
            ("keep_res", 0, [(375, 1242, True, None)], 100, True, (0, 1, 2)),
            ("kitti_sizes", 0, [(h, w, False, None) for h, w in kitti[1:]], 100, False, (0, 1, 2)),
            ("calib_b3", 0, three, 100, True, (0, 1, 2)),
            ("dropin_b3", 1, three, 100, True, (0, 1, 2)),
            ("empties", 0, [(375, 1242, False, None)], 100, False, (0, 2)),
            ("k1000", 0, [(375, 1242, False, None)], 1000, True, (0, 1, 2))]


def main():
    rng = np.random.default_rng(20261016)
    out = {}
    names = []
    for name, form, imgs, K, specials, classes in tail_cases(rng):
        metas = [ref_meta(h, w, kr, calib, seed=k) for k, (h, w, kr, calib) in enumerate(imgs)]
        dets = ddd_rows(rng, len(imgs), K, (CS.INPUT_HW[0] // 4, CS.INPUT_HW[1] // 4), classes)
        if name == "empties":
            dets[0, dets[0, :, 17] == 2, 2] *= F32(0.19)                  # class 2: every score below the cut
        if specials:
            add_specials(dets, metas[0], metas[0]["calib"])
        res = run_merge(dets, metas) if form == 0 else run_dropin(dets, metas)
        rows, lens = CS.flatten(res)
        out.update({name + "_dets": dets, name + "_c": np.stack([m["c"] for m in metas]),
                    name + "_s": np.stack([m["s"] for m in metas]).astype(np.int32),
                    name + "_calib": np.stack([m["calib"] for m in metas]).astype(F32),
                    name + "_hw": np.array([metas[0]["out_height"], metas[0]["out_width"]], np.int64),
                    name + "_form": np.int64(form), name + "_out": rows, name + "_len": lens})
        names.append(name)
    out["names"] = np.array(names)
    pre = []
    for name, (h, w, keep_res) in CS.PRE_CASES.items():
        img = CS.ddd_image(h, w)
        images, meta = DDD.DddDetector.pre_process(detector(keep_res), img, 1)
        images = np.ascontiguousarray(images.numpy())
        out.update({name + "_img_crc": np.uint32(zlib.crc32(img.view(np.uint8))),
                    name + "_crc": np.uint32(zlib.crc32(images.view(np.uint8))),
                    name + "_shape": np.array(images.shape, np.int64), name + "_sample": images[:, :, ::9, ::7].copy(),
                    name + "_c": meta["c"], name + "_s": meta["s"], name + "_calib": meta["calib"],
                    name + "_hw": np.array([meta["out_height"], meta["out_width"]], np.int64)})
        pre.append(name)
    out["pre_names"] = np.array(pre)
    path = os.path.join(HERE, "ddd_tail.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

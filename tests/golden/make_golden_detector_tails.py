"""Generates tests/golden/detector_tails.npz: the UNMODIFIED reference tails of MultiPoseDetector (detectors/
multi_pose.py:62-81) and ExdetDetector (detectors/exdet.py:85-122), `post_process` of every image and scale followed
by `merge_outputs`, called as plain functions on a stub `self` that carries `opt`, `num_classes` and
`max_per_image`.  The reference's compiled soft_nms / soft_nms_39 (oracle/build_ref.py) are set in the detector
modules; detectors/exdet.py uses `soft_nms` without importing it, so the name is injected there.  Build container
only; tests read the .npz.

    python tests/golden/make_golden_detector_tails.py

Layout: `mp_names` lists the multi_pose merges; case `m` has `m_dets` (float32 [S, B, K, 40] decode outputs),
`m_c` / `m_s` (float32 [S, B, 2]; `m_s_scalar` [B] marks images whose scale is the scalar m_s[..., 0]),
`m_scales` (float64 [S]), `m_hw` (int [S, 2] output height, width), `m_nms` (int) and `m_out` (float32 [B, N, 39],
merge_outputs' rows).  `ex_names` lists the exdet merges; case `e` has `e_dets` (float32 [S, P*B, N, 14]),
`e_c`, `e_s`, `e_s_scalar`, `e_scales`, `e_hw` as above, `e_cfg` (int: num_classes, max_per_image, flip) and
`e_out` (float32 [R, 7]: image, class id, x1, y1, x2, y2, score, in image / class order).
"""
import os
import sys
import types

import numpy as np
import torch

REF = "/root/reference/src/lib"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(REF))      # detectors/exdet.py imports _init_paths from src/
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def _stub(name, **attrs):
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    sys.modules[name] = mod
    return mod


# progress and matplotlib are not installed here; the tails use neither.  models.model pulls in the networks
# (and the compiled DCNv2 extension) for create_model / load_model, which the tails do not use either.
_stub("progress", bar=_stub("progress.bar", Bar=object))
_stub("matplotlib", pyplot=_stub("matplotlib.pyplot"))
_stub("models.model", create_model=None, load_model=None)

from detectors import exdet as EX  # noqa: E402
from detectors import multi_pose as MP  # noqa: E402
from oracle import build_ref  # noqa: E402
from utils.image import get_affine_transform  # noqa: E402
from centernet_b200.post_process import _inv_affine  # noqa: E402

nms = build_ref.load_nms()
assert nms is not None, "oracle/_ref nms module not built (python -m oracle.build_ref, where the reference exists)"
MP.soft_nms_39 = nms.soft_nms_39
EX.soft_nms = nms.soft_nms          # the name exdet.py uses at :109 but never imports

F32 = np.float32
NAN_NEG = np.array([0xffc00000], np.uint32).view(F32)[0]


def q(v, grid=0.125):
    """Values on a 1/8 lattice: exact differences and a compressible golden."""
    return (np.round(np.asarray(v) / grid) * grid).astype(F32)


def pose_like(rng, B, K, out_hw):
    """[B, K, 40] multi_pose_decode-shaped rows: box, score (descending), 17 keypoints, class 0."""
    oh, ow = out_hw
    d = np.zeros((B, K, 40), F32)
    x = rng.uniform(-2, ow, (B, K)); y = rng.uniform(-2, oh, (B, K))
    k = K // 3
    x[:, :2 * k] = np.repeat(x[:, :k], 2, axis=1) + rng.uniform(-1, 1, (B, 2 * k))
    y[:, :2 * k] = np.repeat(y[:, :k], 2, axis=1) + rng.uniform(-1, 1, (B, 2 * k))
    d[..., 0], d[..., 1] = q(x), q(y)
    d[..., 2] = q(x + rng.uniform(2, 30, (B, K))); d[..., 3] = q(y + rng.uniform(2, 30, (B, K)))
    d[..., 4] = q(np.sort(rng.uniform(0, 1, (B, K)), axis=1)[:, ::-1], 2.0 ** -12)
    d[..., 5:39] = np.round(rng.uniform(-4, max(oh, ow) + 4, (B, K, 34)))
    return d


def exct_like(rng, n_img, N, nc, out_hw, classes=None, levels=None, specials=False):
    """[n_img, N, 14] exct_decode-shaped rows: box (x1 < x2 on the output grid), score, the four extreme points
    (zero: post_process ignores them), class id."""
    oh, ow = out_hw
    d = np.zeros((n_img, N, 14), F32)
    x = rng.uniform(-2, ow, (n_img, N)); y = rng.uniform(-2, oh, (n_img, N))
    k = N // 3
    x[:, :2 * k] = np.repeat(x[:, :k], 2, axis=1) + rng.uniform(-1, 1, (n_img, 2 * k))
    y[:, :2 * k] = np.repeat(y[:, :k], 2, axis=1) + rng.uniform(-1, 1, (n_img, 2 * k))
    d[..., 0], d[..., 1] = q(x), q(y)
    d[..., 2] = q(x + rng.uniform(1, 24, (n_img, N))); d[..., 3] = q(y + rng.uniform(1, 24, (n_img, N)))
    s = rng.uniform(0.0, 1.0, (n_img, N)) if levels is None else rng.integers(1, levels + 1, (n_img, N)) / levels
    d[..., 4] = np.maximum(q(np.sort(s, axis=1)[:, ::-1], 2.0 ** -12), F32(2.0 ** -12))
    if specials:       # scores <= 0 (dropped), -0.0, NaN (dropped) and +inf (kept: inf > 0)
        vals = np.array([0.0, -0.0, -0.25, NAN_NEG, np.inf], F32)
        pick = rng.random((n_img, N)) < 0.12
        d[..., 4][pick] = vals[rng.integers(0, len(vals), int(pick.sum()))]
    pool = np.arange(nc) if classes is None else np.asarray(classes)
    d[..., 13] = pool[rng.integers(0, len(pool), (n_img, N))]
    return d


def metas_for(rng, B, scales, dyadic=False):
    """Per-image centres and scalar / vector scales whose inverse affine is the same from cv2.getAffineTransform
    (the reference) and from the float64 solve of the device tails' host side (post_process._inv_affine, shared with
    ctdet_merge_device): for about one meta in five the two differ in the last bit of a matrix entry, which moves a
    back-projected corner by one float32 ulp now and then; such metas are drawn again."""
    while True:
        c, s, s_scalar, hw = _draw_metas(rng, B, scales, dyadic)
        if all(np.array_equal(get_affine_transform(c[k, i], F32(s[k, i, 0]) if s_scalar[i] else s[k, i], 0,
                                                   (int(hw[k, 1]), int(hw[k, 0])), inv=1),
                              _inv_affine(c[k, i], F32(s[k, i, 0]) if s_scalar[i] else s[k, i],
                                          (int(hw[k, 1]), int(hw[k, 0]))))
               for k in range(len(scales)) for i in range(B)):
            return c, s, s_scalar, hw


def _draw_metas(rng, B, scales, dyadic):
    """`dyadic`: image scale = 4 x the output width and centres on a 1/2 grid, so the back-projection is exact and
    the (long) reference output compresses."""
    hw = np.array([[int(round(128 * sc)), int(round(128 * sc)) + 32] for sc in scales], np.int64)
    base_c = np.stack([rng.uniform(150, 400, B), rng.uniform(100, 300, B)], 1)
    base_s = np.stack([rng.uniform(480, 800, B), rng.uniform(360, 640, B)], 1)
    if dyadic:
        base_c = np.round(base_c * 2) / 2
        base_s[:, 0] = 4 * hw[0, 1] / scales[0]
    s_scalar = np.arange(B) % 2 == 0                 # scalar max(h, w) scales and --keep_res vector scales
    base_s[s_scalar, 1] = base_s[s_scalar, 0]
    c = np.stack([base_c * sc for sc in scales], 0).astype(F32)
    s = np.stack([base_s * sc for sc in scales], 0).astype(F32)
    return c, s, s_scalar, hw


def ref_meta(c, s, s_scalar, hw, k, i):
    return {"c": c[k, i], "s": F32(s[k, i, 0]) if s_scalar[i] else s[k, i].copy(),
            "out_height": int(hw[k, 0]), "out_width": int(hw[k, 1])}


def ref_multi_pose(dets, c, s, s_scalar, scales, hw, run_nms):
    S, B = dets.shape[0], dets.shape[1]
    this = types.SimpleNamespace(opt=types.SimpleNamespace(nms=bool(run_nms), test_scales=list(scales)),
                                 num_classes=1)
    out = []
    for i in range(B):
        detections = [MP.MultiPoseDetector.post_process(this, torch.from_numpy(dets[k, i:i + 1].copy()),
                                                        ref_meta(c, s, s_scalar, hw, k, i), float(scales[k]))
                      for k in range(S)]
        out.append(np.array(MP.MultiPoseDetector.merge_outputs(this, detections)[1], F32).reshape(-1, 39))
    return np.stack(out, 0)


def ref_exdet(dets, c, s, s_scalar, scales, hw, nc, mpi, flip):
    S, P = dets.shape[0], 2 if flip else 1
    B = dets.shape[1] // P
    this = types.SimpleNamespace(opt=types.SimpleNamespace(), num_classes=nc, max_per_image=mpi)
    flat = []
    for i in range(B):
        detections = [EX.ExdetDetector.post_process(this, torch.from_numpy(dets[k, P * i:P * i + P].copy()),
                                                    ref_meta(c, s, s_scalar, hw, k, i), float(scales[k]))
                      for k in range(S)]
        res = EX.ExdetDetector.merge_outputs(this, detections)
        for j in range(1, nc + 1):
            a = res[j]
            flat.append(np.concatenate([np.full((len(a), 1), i, F32), np.full((len(a), 1), j, F32), a], 1))
    return np.concatenate(flat, 0)


SCALES5 = (0.5, 0.75, 1.0, 1.25, 1.5)


def mp_cases():
    """(name, scales, B, K, nms)."""
    return [("mp_s1", (1.0,), 2, 100, 0), ("mp_s1_nms", (1.0,), 2, 100, 1), ("mp_s5", SCALES5, 2, 40, 0)]


def ex_cases():
    """(name, scales, B, N, num_classes, max_per_image, flip, extra exct_like arguments)."""
    return [("flip_s5", SCALES5, 2, 64, 80, 100, 1, dict(specials=True)),
            ("noflip_s1", (1.0,), 3, 100, 80, 100, 0, dict(specials=True)),
            ("noflip_s5_sparse", SCALES5, 2, 40, 80, 100, 0, dict(classes=(0, 3, 17, 79), specials=True)),
            ("mpi_above", (1.0, 1.25), 2, 50, 3, 1000, 1, dict(specials=True)),
            ("list4096", (1.0,), 1, 2048, 2, 100000, 1, dict(classes=(1,))),
            ("wide_ties", SCALES5, 1, 512, 80, 100, 1, dict(levels=16))]


def main():
    rng = np.random.default_rng(20261016)
    out = {}
    names = []
    for name, scales, B, K, run_nms in mp_cases():
        c, s, s_scalar, hw = metas_for(rng, B, scales, dyadic=K > 256)
        dets = np.stack([pose_like(rng, B, K, hw[k]) for k in range(len(scales))], 0)
        out.update({name + "_dets": dets, name + "_c": c, name + "_s": s, name + "_s_scalar": s_scalar,
                    name + "_scales": np.array(scales, np.float64), name + "_hw": hw, name + "_nms": np.int64(run_nms),
                    name + "_out": ref_multi_pose(dets, c, s, s_scalar, scales, hw, run_nms)})
        names.append(name)
    out["mp_names"] = np.array(names)
    names = []
    for name, scales, B, N, nc, mpi, flip, kw in ex_cases():
        c, s, s_scalar, hw = metas_for(rng, B, scales, dyadic=N > 1000)
        P = 2 if flip else 1
        dets = np.stack([exct_like(rng, P * B, N, nc, hw[k], **kw) for k in range(len(scales))], 0)
        out.update({name + "_dets": dets, name + "_c": c, name + "_s": s, name + "_s_scalar": s_scalar,
                    name + "_scales": np.array(scales, np.float64), name + "_hw": hw,
                    name + "_cfg": np.array([nc, mpi, flip], np.int64),
                    name + "_out": ref_exdet(dets, c, s, s_scalar, scales, hw, nc, mpi, flip)})
        names.append(name)
    out["ex_names"] = np.array(names)
    path = os.path.join(HERE, "detector_tails.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

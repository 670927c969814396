"""Device time per ctdet, multi_pose, ddd or exdet training batch (centernet_b200.train_input), the host->device
bytes per image against the reference loader's, and (ctdet) the numpy oracle's CPU time per image.

    python tools/train_input_time.py [--iters 50] [--sampler ctdet|multi_pose|ddd|exdet]

Synthetic COCO-sized sources (ragged 640x480 / 480x640 / 500x375 / 427x640), 512x512 input, 80 classes, 128
object slots, about 7 objects per image, colour augmentation on; B = 32, 64 and 114.  Per batch it times, with
CUDA events over --iters batches after a warm-up, build_ctdet_batch (H2D copy of the packed pinned buffer + image
kernels + targets) with and without the dense hm, and the same from a buffer already on the device (kernels
only).  The reference's loader is not part of the repository, so the host-side figure is the numpy oracle
(tests/train_np.py: warp, color_aug, normalisation, targets, hm splat) on one core: a stand-in for the per-pixel
work this moves off the host, not a measurement of cv2.

--sampler multi_pose: the same sources at 512x512 input, 17 joints, 32 slots, about 7 people per image with
random joint visibilities, colour augmentation on; B = 32 and 64, with aug_rot 0 and 1 (every image rotated, up to
+-60 degrees), each timed as build_multi_pose_batch with the H2D copy, from a buffer already on the device, and
per image; with dense hm / hm_hp and, for aug_rot 0, without (a rotated batch needs the dense hm).  Prints one
JSON line, with the card's name and power limit read in the same run.

--sampler ddd: synthetic KITTI-sized sources (ragged around 1242x375), 1280x384 input, 3 classes, 50 slots, about 8
positives, 4 ignore objects (DontCare and single-class) and a skipped one per image, aug_ddd 0.5; B = 32 and 64,
with point ignores and with rect_mask, each timed as build_ddd_batch with the H2D copy and from a buffer already
on the device (kernels only).  Prints one JSON line, with the card's name and power limit read in the same run.

--sampler exdet: the COCO-sized sources at 512x512 input, 80 classes, 128 slots, about 7 objects per image with
random extreme points on their box sides, flip 0.5 and colour augmentation on; B = 32 and 64, each timed as
build_exdet_batch with the H2D copy and from a buffer already on the device (kernels only), with the object lists
only and with the five dense maps.  Prints one JSON line, with the card's name, power limit and max SM clock read in
the same run."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from centernet_b200 import train_input as T  # noqa: E402
import ddd_train_cases as DC  # noqa: E402
import exdet_train_cases as EC  # noqa: E402
import multi_pose_train_cases as MC  # noqa: E402
import train_cases as TC  # noqa: E402

SIZES = [(480, 640), (640, 480), (375, 500), (640, 427), (427, 640), (333, 500)]


def make_samples(b, seed):
    opt = TC.make_opt(dict(TC.CASES["crop"]))
    rng = np.random.default_rng(seed)
    np.random.seed(seed); random.seed(seed)
    data_rng = np.random.RandomState(seed)
    out = []
    for i in range(b):
        h, w = SIZES[i % len(SIZES)]
        s = T.sample_params(h, w, opt, 'train', data_rng, TC.EIG_VAL, TC.EIG_VEC)
        n = int(rng.integers(1, 15))
        x0, y0 = rng.uniform(0, w, n), rng.uniform(0, h, n)
        boxes = np.stack([x0, y0, x0 + rng.uniform(4, 200, n), y0 + rng.uniform(4, 200, n)], 1).astype(np.float32)
        s.update(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), boxes=boxes,
                 cls=rng.integers(0, 80, n).astype(np.int32), max_objs=128, num_classes=80, mean=TC.MEAN,
                 std=TC.STD, cat_spec_wh=False, reg_offset=True)
        out.append(s)
    return out


def make_pose_samples(b, seed, aug_rot):
    case = dict(MC.CASES["mp_coco"], aug_rot=aug_rot, rotate=30.0)
    opt = MC.make_opt(case)
    rng = np.random.default_rng(seed)
    np.random.seed(seed); random.seed(seed)
    data_rng = np.random.RandomState(seed)
    out = []
    for i in range(b):
        h, w = SIZES[i % len(SIZES)]
        s = T.multi_pose_params(h, w, opt, 'train', data_rng, MC.EIG_VAL, MC.EIG_VEC)
        n = int(rng.integers(1, 15))
        x0, y0 = rng.uniform(0, w, n), rng.uniform(0, h, n)
        bw, bh = rng.uniform(4, 200, n), rng.uniform(4, 200, n)
        boxes = np.stack([x0, y0, x0 + bw, y0 + bh], 1).astype(np.float32)
        kps = [np.stack([x0[k] + rng.uniform(-0.2, 1.2, 17) * bw[k], y0[k] + rng.uniform(-0.2, 1.2, 17) * bh[k],
                         rng.choice([0., 1., 2.], 17)], 1).astype(np.float32).reshape(-1) for k in range(n)]
        s.update(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), boxes=boxes, cls=np.zeros(n, np.int64),
                 keypoints=kps, max_objs=32, num_classes=1, num_joints=17,
                 flip_idx=[tuple(e) for e in MC.COCO_FLIP_IDX], mean=MC.MEAN, std=MC.STD, reg_offset=True,
                 hm_hp=True, reg_hp_offset=True)
        out.append(s)
    return out


def make_ddd_samples(b, seed, rect_mask):
    case = dict(DC.CASES["kitti"], rect_mask=rect_mask)
    opt = DC.make_opt(case)
    rng = np.random.default_rng(seed)
    np.random.seed(seed); random.seed(seed)
    out = []
    for i in range(b):
        h, w = DC.KITTI_SIZES[i % len(DC.KITTI_SIZES)]
        s = T.ddd_params(h, w, opt, 'train')
        n = 13
        x0, y0 = rng.uniform(0, 0.9 * w, n), rng.uniform(0.3 * h, 0.8 * h, n)
        bw, bh = rng.uniform(15, 250, n), rng.uniform(15, 150, n)
        boxes = np.stack([x0, y0, x0 + bw, y0 + bh], 1).astype(np.float32)
        cls = np.array([0, 1, 1, 2, 1, 1, 0, 1, -1, -3, -2, -1, -99])[rng.permutation(n)]
        s.update(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), boxes=boxes, cls=cls,
                 alpha=rng.uniform(-np.pi, np.pi, n), depth=rng.uniform(3, 70, n),
                 dim=list(rng.uniform(0.5, 4, (n, 3))), max_objs=50, num_classes=3, mean=DC.MEAN, std=DC.STD,
                 rect_mask=rect_mask, reg_bbox=True, reg_offset=True)
        out.append(s)
    return out


def make_exdet_samples(b, seed):
    case = dict(EC.CASES["ex_coco"])
    opt = EC.make_opt(case)
    rng = np.random.default_rng(seed)
    np.random.seed(seed); random.seed(seed)
    data_rng = np.random.RandomState(seed)
    out = []
    for i in range(b):
        h, w = SIZES[i % len(SIZES)]
        s = T.exdet_params(h, w, opt, 'train', data_rng, EC.EIG_VAL, EC.EIG_VEC)
        n = int(rng.integers(1, 15))
        x0, y0 = rng.uniform(0, w, n), rng.uniform(0, h, n)
        bw, bh = rng.uniform(4, 200, n), rng.uniform(4, 200, n)
        u = rng.random((n, 4))
        pts = np.stack([x0 + u[:, 0] * bw, y0, x0, y0 + u[:, 1] * bh, x0 + u[:, 2] * bw, y0 + bh, x0 + bw,
                        y0 + u[:, 3] * bh], 1).astype(np.float32)
        s.update(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), points=list(pts),
                 cls=rng.integers(0, 80, n), max_objs=128, num_classes=80, mean=EC.MEAN, std=EC.STD,
                 agnostic_ex=False, reg_offset=True)
        out.append(s)
    return out


def time_batches(packed, iters, dense_hm, build=None):
    build = build or T.build_ctdet_batch
    kw = {} if dense_hm is None else dict(dense_hm=dense_hm)
    for _ in range(3):
        build(packed, **kw)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        build(packed, **kw)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def oracle_cpu_ms(samples, n):
    import train_np as TN
    from oracle import image_np
    t0 = time.perf_counter()
    for s in samples[:n]:
        TN.train_image(s['image'], T.affine_transform(s['c'], s['s'], [512, 512]), s['flip'], 512, 512, TC.MEAN,
                       TC.STD, s['order'], s['blend'], s['light'])
        t = TN.ctdet_targets(s['boxes'], s['cls'], s['flip'], s['image'].shape[1], s['trans_output'], 128, 80, 128,
                             128)
        lists = [t[k][None] for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid')]
        image_np.splat_objects(*lists, 80, 128, 128)
    return (time.perf_counter() - t0) * 1e3 / n


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main_multi_pose(iters):
    # the reference's per-image transfer: input, hm, hm_hp and the targets of multi_pose.py:161-177
    m, j, r = 32, 17, 128
    ref_bytes = 3 * 512 * 512 * 4 + (1 + j) * r * r * 4 + m * (1 + 8 + 2 * 4 + 2 * 4 + 2 * j * 4 + 2 * j) \
        + m * j * (2 * 4 + 8 + 8)
    res = {"gpu": gpu_info(), "sampler": "multi_pose", "batches": {}}
    build = T.build_multi_pose_batch
    for b in (32, 64):
        for aug_rot in (0.0, 1.0):
            packed = T.collate_multi_pose(make_pose_samples(b, b, aug_rot))
            on_device = dict(packed, buffer=packed['buffer'].cuda())
            rr = {"rotated_images": int(sum(packed['scalars']['rotated'])),
                  "ms_per_batch_dense": time_batches(packed, iters, True, build),
                  "ms_per_batch_dense_kernels_only": time_batches(on_device, iters, True, build),
                  "h2d_bytes_per_image": packed['buffer'].numel() / b, "reference_h2d_bytes_per_image": ref_bytes}
            rr["us_per_image_dense"] = rr["ms_per_batch_dense"] * 1e3 / b
            if aug_rot == 0:
                rr["ms_per_batch_lists"] = time_batches(packed, iters, False, build)
                rr["ms_per_batch_lists_kernels_only"] = time_batches(on_device, iters, False, build)
                rr["us_per_image_lists"] = rr["ms_per_batch_lists"] * 1e3 / b
            res["batches"]["B%d_aug_rot%g" % (b, aug_rot)] = rr
    print(json.dumps(res))


def main_ddd(iters):
    # the reference's per-image transfer: input, hm and the targets of ddd.py:143-149
    m, oh, ow = 50, 96, 320
    ref_bytes = 3 * 384 * 1280 * 4 + 3 * oh * ow * 4 + m * (4 + 3 * 4 + 8 + 2 * 8 + 2 * 4 + 1 + 1 + 2 * 4 + 2 * 4)
    res = {"gpu": gpu_info(), "sampler": "ddd", "batches": {}}
    for b in (32, 64):
        for rect in (False, True):
            packed = T.collate_ddd(make_ddd_samples(b, b, rect))
            on_device = dict(packed, buffer=packed['buffer'].cuda())
            rr = {"ms_per_batch": time_batches(packed, iters, None, T.build_ddd_batch),
                  "ms_per_batch_kernels_only": time_batches(on_device, iters, None, T.build_ddd_batch),
                  "h2d_bytes_per_image": packed['buffer'].numel() / b, "reference_h2d_bytes_per_image": ref_bytes}
            rr["us_per_image"] = rr["ms_per_batch"] * 1e3 / b
            rr["us_per_image_kernels_only"] = rr["ms_per_batch_kernels_only"] * 1e3 / b
            res["batches"]["B%d_%s" % (b, "rect_mask" if rect else "point_ignores")] = rr
    print(json.dumps(res))


def main_exdet(iters):
    # the reference's per-image transfer: input, the five maps and the targets of exdet.py:130-135
    m, c, r = 128, 80, 128
    ref_bytes = 3 * 512 * 512 * 4 + 5 * c * r * r * 4 + m * (1 + 4 * (2 * 4 + 8))
    res = {"gpu": gpu_info(), "sampler": "exdet", "batches": {}}
    for b in (32, 64):
        packed = T.collate_exdet(make_exdet_samples(b, b))
        on_device = dict(packed, buffer=packed['buffer'].cuda())
        rr = {"h2d_bytes_per_image": packed['buffer'].numel() / b, "reference_h2d_bytes_per_image": ref_bytes}
        for dense in (False, True):
            tag = "dense" if dense else "lists"
            rr["ms_per_batch_" + tag] = time_batches(packed, iters, dense, T.build_exdet_batch)
            rr["ms_per_batch_%s_kernels_only" % tag] = time_batches(on_device, iters, dense, T.build_exdet_batch)
            rr["us_per_image_" + tag] = rr["ms_per_batch_" + tag] * 1e3 / b
            rr["us_per_image_%s_kernels_only" % tag] = rr["ms_per_batch_%s_kernels_only" % tag] * 1e3 / b
        res["batches"]["B%d" % b] = rr
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--oracle-images", type=int, default=4)
    ap.add_argument("--sampler", choices=("ctdet", "multi_pose", "ddd", "exdet"), default="ctdet")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_input_time: needs a CUDA device (no CPU timing is reported)")
    if args.sampler == "multi_pose":
        return main_multi_pose(args.iters)
    if args.sampler == "ddd":
        return main_ddd(args.iters)
    if args.sampler == "exdet":
        return main_exdet(args.iters)
    res = {"gpu": gpu_info(), "batches": {}}
    ref_bytes = 3 * 512 * 512 * 4 + 80 * 128 * 128 * 4 + 128 * (2 * 4 + 2 * 4 + 8 + 1)
    for b in (32, 64, 114):
        samples = make_samples(b, b)
        packed = T.collate_ctdet(samples)
        on_device = dict(packed, buffer=packed['buffer'].cuda())   # the same batch without the H2D copy
        r = {"ms_per_batch": time_batches(packed, args.iters, False),
             "ms_per_batch_kernels_only": time_batches(on_device, args.iters, False),
             "ms_per_batch_dense_hm": time_batches(packed, args.iters, True),
             "h2d_bytes_per_image": packed['buffer'].numel() / b,
             "reference_h2d_bytes_per_image": ref_bytes}
        r["us_per_image"] = r["ms_per_batch"] * 1e3 / b
        res["batches"][b] = r
    res["oracle_cpu_ms_per_image_stand_in"] = oracle_cpu_ms(make_samples(args.oracle_images, 7), args.oracle_images)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

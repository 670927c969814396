"""Seeded inputs of tests/golden/train_multi_pose.npz (tests/golden/make_golden_train_multi_pose.py): per case the
options of the multi_pose sampler, ragged image sizes, seeded uint8 images and COCO-keypoint-style annotations,
rebuilt identically on every machine from numpy's PCG64 stream, so only what the reference returned for them is
stored.  Images, normalisation and colour constants are those of tests/train_cases.py."""
import types

import numpy as np

from train_cases import EIG_VAL, EIG_VEC, MEAN, ORDERS, STD  # noqa: F401  (re-exported for the tests)

COCO_FLIP_IDX = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]

_BASE = dict(split='train', not_rand_crop=False, flip=0.5, no_color_aug=False, input_res=512, down_ratio=4,
             scale=0.4, shift=0.1, aug_rot=0.0, rotate=0.0, reg_offset=True, hm_hp=True, reg_hp_offset=True,
             num_classes=1, num_joints=17, flip_idx=COCO_FLIP_IDX, max_objs=32, n_objs=(1, 20), empty=(),
             hm_samples=1)
CASES = {
    # COCO-hp defaults: random crop, flip 0.5, colour, no rotation; sources from a few pixels (below the 128
    # border) to 640 x 480, one image without annotations
    "mp_coco": dict(_BASE, seed=21, sizes=[(480, 640), (640, 480), (333, 500), (90, 100), (7, 5), (427, 640)],
                    empty=(4,)),
    # every image flipped: the joint swaps
    "mp_flip": dict(_BASE, seed=22, sizes=[(427, 640), (375, 500), (200, 150), (640, 427)], flip=1.0),
    # every image rotated (aug_rot 1): constant hm, zero reg_mask / hps_mask, zero-size boxes get targets
    "mp_rot": dict(_BASE, seed=23, sizes=[(480, 640), (300, 260), (512, 512), (123, 321)], aug_rot=1.0,
                   rotate=30.0),
    # the three randn of not_rand_crop, then rotation for about half the images; fewer slots than objects
    "mp_shift": dict(_BASE, seed=24, sizes=[(480, 640), (300, 260), (640, 360), (123, 321), (200, 200)],
                     not_rand_crop=True, aug_rot=0.5, rotate=40.0, max_objs=6, n_objs=(4, 20), hm_samples=2),
    # no colour, no hm_hp (hence no reg_hp_offset), no reg_offset, 256 input
    "mp_plain": dict(_BASE, seed=25, sizes=[(256, 256), (180, 320), (320, 180)], no_color_aug=True, hm_hp=False,
                     reg_hp_offset=False, reg_offset=False, input_res=256),
    # five joints whose flip pairs share joints (the swaps compose in order), two classes
    "mp_small": dict(_BASE, seed=26, sizes=[(300, 400), (250, 250), (400, 300), (90, 120)], num_joints=5,
                     flip_idx=[[1, 2], [2, 3], [0, 4], [3, 1]], flip=0.7, num_classes=2),
}


def make_opt(case):
    opt = types.SimpleNamespace(**{k: case[k] for k in ('not_rand_crop', 'flip', 'no_color_aug', 'input_res',
                                                        'down_ratio', 'scale', 'shift', 'aug_rot', 'rotate',
                                                        'reg_offset', 'hm_hp', 'reg_hp_offset')})
    opt.output_res = case['input_res'] // case['down_ratio']
    opt.mse_loss = False
    opt.dense_hp = False
    opt.debug = 1          # the sampler then also returns meta (c, s)
    opt.hm_gauss = 0
    return opt


def _rng(name, i, what):
    return np.random.default_rng([sum(map(ord, name)), i, what])


def case_image(name, i):
    """uint8 BGR source: noise over a diagonal ramp."""
    h, w = CASES[name]['sizes'][i]
    r = _rng(name, i, 0)
    ramp = (np.arange(h)[:, None, None] * 3 + np.arange(w)[None, :, None] * 2 + np.array([0, 85, 170])) % 256
    return ((ramp + r.integers(0, 96, (h, w, 3))) % 256).astype(np.uint8)


def case_anns(name, i):
    """COCO person annotations: boxes partly outside the image, some of zero width or height; per joint
    visibility 0, 1 or 2 (objects without a visible joint among them), joints spread past the box and the image,
    invisible joints sometimes with coordinates (the sampler must ignore them)."""
    case = CASES[name]
    h, w = case['sizes'][i]
    nj = case['num_joints']
    r = _rng(name, i, 1)
    lo, hi = case['n_objs']
    n = 0 if i in case['empty'] else int(r.integers(lo, hi + 1))
    anns = []
    for _ in range(n):
        x, y = round(float(r.uniform(-0.2, 1.05) * w), 2), round(float(r.uniform(-0.2, 1.05) * h), 2)
        bw, bh = round(float(r.uniform(0, 0.6) * w), 2), round(float(r.uniform(0, 0.6) * h), 2)
        u = r.random()
        if u < 0.1:
            bw = 0.0
        elif u < 0.15:
            bh = 0.0
        vis = r.choice([0, 1, 2], size=nj, p=[0.35, 0.2, 0.45])
        if r.random() < 0.15:
            vis[:] = 0
        px = np.round(x + r.uniform(-0.4, 1.4, nj) * max(bw, 8.0), 1)
        py = np.round(y + r.uniform(-0.4, 1.4, nj) * max(bh, 8.0), 1)
        hidden = (vis == 0) & (r.random(nj) < 0.7)
        px[hidden], py[hidden] = 0.0, 0.0
        kps = np.stack([px, py, vis.astype(np.float64)], 1).reshape(-1)
        anns.append({'bbox': [x, y, bw, bh], 'category_id': int(r.integers(0, case['num_classes'])) + 1,
                     'keypoints': [float(v) for v in kps]})
    return anns


def case_objects(name, i):
    """What MultiPoseTrainInput reads from the first max_objs annotations: float32 box corners [n, 4], classes
    int(category_id) - 1 and the float32 keypoint lists."""
    anns = case_anns(name, i)[:CASES[name]['max_objs']]
    boxes = np.array([[a['bbox'][0], a['bbox'][1], a['bbox'][0] + a['bbox'][2], a['bbox'][1] + a['bbox'][3]]
                      for a in anns], np.float32).reshape(-1, 4)
    cls = np.array([int(a['category_id']) - 1 for a in anns], np.int64)
    return boxes, cls, [np.array(a['keypoints'], np.float32) for a in anns]


def case_dataset(name, coco, img_dir, data_rng):
    """The attributes MultiPoseDataset.__getitem__ reads (COCOHP's, with the case's joints and slots)."""
    case = CASES[name]
    return dict(opt=make_opt(case), coco=coco, images=list(range(len(case['sizes']))), img_dir=img_dir,
                max_objs=case['max_objs'], num_classes=case['num_classes'], num_joints=case['num_joints'],
                flip_idx=case['flip_idx'], mean=MEAN.reshape(1, 1, 3), std=STD.reshape(1, 1, 3),
                _data_rng=data_rng, _eig_val=EIG_VAL, _eig_vec=EIG_VEC, split=case['split'])

"""Seeded inputs of tests/golden/train.npz (tests/golden/make_golden_train.py): per case the options of the
ctdet sampler, ragged image sizes, seeded uint8 images and COCO-style annotations, rebuilt identically on every
machine from numpy's PCG64 stream, so only what the reference returned for them is stored."""
import types

import numpy as np

MEAN = np.array([0.40789654, 0.44719302, 0.47026115], np.float32)
STD = np.array([0.28863828, 0.27408164, 0.27809835], np.float32)
EIG_VAL = np.array([0.2141788, 0.01817699, 0.00341571], np.float32)
EIG_VEC = np.array([[-0.58752847, -0.69563484, 0.41340352],
                    [-0.5832747, 0.00994535, -0.81221408],
                    [-0.56089297, 0.71832671, 0.41158938]], np.float32)
ORDERS = ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))

_BASE = dict(split='train', keep_res=False, not_rand_crop=False, flip=0.5, no_color_aug=False, input_h=512,
             input_w=512, pad=31, down_ratio=4, scale=0.4, shift=0.1, cat_spec_wh=False, reg_offset=True,
             num_classes=80, max_objs=128, n_objs=(0, 24), hm_samples=1)
CASES = {
    # COCO defaults: random crop, flip, colour; sources from a few pixels (below the 128 border) to 1280 x 960
    "crop": dict(_BASE, seed=11, sizes=[(480, 640), (640, 480), (333, 500), (90, 100), (7, 5), (960, 1280)]),
    "crop2": dict(_BASE, seed=12, sizes=[(427, 640), (375, 500), (512, 512), (200, 150), (640, 427), (31, 40)],
                  flip=1.0),
    # the three randn draws of not_rand_crop; fewer slots than objects (max_objs 6 < up to 30 objects)
    "shift": dict(_BASE, seed=13, sizes=[(480, 640), (300, 260), (640, 360), (123, 321)], not_rand_crop=True,
                  max_objs=6, n_objs=(4, 30), input_h=384, input_w=384),
    # keep_res with equal source sizes (one batch), cat_spec_wh
    "keep": dict(_BASE, seed=14, sizes=[(200, 300), (200, 300), (200, 300)], keep_res=True, cat_spec_wh=True,
                 num_classes=7),
    # no colour augmentation, no offset regression, small maps, several hm samples
    "plain": dict(_BASE, seed=15, sizes=[(256, 256), (180, 320), (320, 180)], no_color_aug=True, reg_offset=False,
                  input_h=256, input_w=256, num_classes=5, hm_samples=3),
    # get_affine_transform(rot != 0) + cv2.warpAffine + color_aug, outside the sampler
    "rot": dict(_BASE, seed=16, sizes=[(300, 400)], rot=23.0, scale=1.1, out=192),
    "rot2": dict(_BASE, seed=17, sizes=[(257, 190)], rot=-71.5, scale=0.8, out=128),
}


def make_opt(case):
    opt = types.SimpleNamespace(**{k: case[k] for k in ('keep_res', 'not_rand_crop', 'flip', 'no_color_aug',
                                                        'input_h', 'input_w', 'pad', 'down_ratio', 'scale',
                                                        'shift', 'cat_spec_wh', 'reg_offset')})
    opt.mse_loss = False
    opt.dense_wh = False
    opt.debug = 1          # the sampler then also returns meta (c, s)
    opt.hm_gauss = 0
    return opt


def cat_ids(case):
    """COCO-style category ids (sparse, from 1) -> class index."""
    return {3 * k + 1: k for k in range(case['num_classes'])}


def _rng(name, i, what):
    return np.random.default_rng([sum(map(ord, name)), i, what])


def case_image(name, i):
    """uint8 BGR source: noise over a diagonal ramp (not constant, so every blend and the mean matter)."""
    h, w = CASES[name]['sizes'][i]
    r = _rng(name, i, 0)
    ramp = (np.arange(h)[:, None, None] * 3 + np.arange(w)[None, :, None] * 2 + np.array([0, 85, 170])) % 256
    return ((ramp + r.integers(0, 96, (h, w, 3))) % 256).astype(np.uint8)


def case_anns(name, i):
    """COCO annotations: boxes partly outside the image, some of zero width or height (they collapse)."""
    case = CASES[name]
    h, w = case['sizes'][i]
    r = _rng(name, i, 1)
    lo, hi = case['n_objs']
    n = 0 if i == 0 and lo == 0 else int(r.integers(lo, hi + 1))
    anns = []
    for _ in range(n):
        x, y = round(float(r.uniform(-0.2, 1.05) * w), 2), round(float(r.uniform(-0.2, 1.05) * h), 2)
        bw, bh = round(float(r.uniform(0, 0.6) * w), 2), round(float(r.uniform(0, 0.6) * h), 2)
        if r.random() < 0.1:
            bw = 0.0
        anns.append({'bbox': [x, y, bw, bh], 'category_id': 3 * int(r.integers(0, case['num_classes'])) + 1})
    return anns

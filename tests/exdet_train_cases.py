"""Seeded inputs of tests/golden/train_exdet.npz (tests/golden/make_golden_train_exdet.py): per case the options of the
exdet sampler, ragged image sizes, seeded uint8 images and COCO-extreme-style annotations, rebuilt identically on
every machine from numpy's PCG64 stream, so only what the reference returned for them is stored.  Each case's first
image also carries crafted objects: two of one class overlapping and sharing their top point, one whose top and
left points coincide, a few source pixels wide (radius 0) and one reaching past every border.  Images, normalisation
and colour constants are those of tests/train_cases.py."""
import types

import numpy as np

from train_cases import EIG_VAL, EIG_VEC, MEAN, ORDERS, STD  # noqa: F401  (re-exported for the tests)

_BASE = dict(split='train', not_rand_crop=False, flip=0.5, no_color_aug=False, input_res=256, down_ratio=4,
             scale=0.4, shift=0.1, agnostic_ex=False, reg_offset=True, num_classes=5, max_objs=32, n_objs=(1, 16),
             empty=(), hm_samples=99, crafted=True)
CASES = {
    # COCO defaults: 512 input, 80 classes, 128 slots, random crop, flip 0.5, colour; sources from below the 128
    # border to 640 x 480, one image without annotations; the 80-class maps of the first sample only
    "ex_coco": dict(_BASE, seed=51, sizes=[(480, 640), (640, 480), (333, 500), (90, 100), (427, 640), (7, 5)],
                    input_res=512, num_classes=80, max_objs=128, n_objs=(4, 30), empty=(5,), hm_samples=1),
    # one heat map for all classes of the extreme points
    "ex_agn": dict(_BASE, seed=52, sizes=[(300, 400), (250, 250), (400, 300), (120, 90)], agnostic_ex=True),
    # every image flipped: mirrored points, l <-> r
    "ex_flip": dict(_BASE, seed=53, sizes=[(427, 640), (375, 500), (200, 150), (640, 427)], flip=1.0),
    # the three randn of not_rand_crop: a float64 centre off the integers
    "ex_shift": dict(_BASE, seed=54, sizes=[(480, 640), (300, 260), (640, 360), (123, 321), (200, 200)],
                     not_rand_crop=True),
    # no colour, no reg_offset, fewer slots than annotations
    "ex_plain": dict(_BASE, seed=55, sizes=[(256, 256), (180, 320), (320, 180)], no_color_aug=True,
                     reg_offset=False, max_objs=6, n_objs=(8, 20)),
    # the val split draws nothing
    "ex_val": dict(_BASE, seed=56, sizes=[(300, 400), (500, 375), (256, 256)], split='val', num_classes=3),
}


def make_opt(case):
    opt = types.SimpleNamespace(**{k: case[k] for k in ('not_rand_crop', 'flip', 'no_color_aug', 'input_res',
                                                        'scale', 'shift', 'agnostic_ex', 'reg_offset',
                                                        'num_classes')})
    opt.output_res = case['input_res'] // case['down_ratio']
    opt.mse_loss = False
    return opt


def cat_ids(case):
    """COCO-style category ids (1-based, with gaps) to classes 0 .. C - 1."""
    return {3 * c + 1: c for c in range(case['num_classes'])}


def _rng(name, i, what):
    return np.random.default_rng([sum(map(ord, name)) + 2000, i, what])


def case_image(name, i):
    """uint8 BGR source: noise over a diagonal ramp."""
    h, w = CASES[name]['sizes'][i]
    r = _rng(name, i, 0)
    ramp = (np.arange(h)[:, None, None] * 3 + np.arange(w)[None, :, None] * 2 + np.array([0, 85, 170])) % 256
    return ((ramp + r.integers(0, 96, (h, w, 3))) % 256).astype(np.uint8)


def _ann(cat, x0, y0, x1, y1, u):
    """Extreme points t, l, b, r of the box [x0, x1] x [y0, y1], each at fraction u[j] along its side."""
    pts = [[x0 + u[0] * (x1 - x0), y0], [x0, y0 + u[1] * (y1 - y0)], [x0 + u[2] * (x1 - x0), y1],
           [x1, y0 + u[3] * (y1 - y0)]]
    return {'extreme_points': [[round(float(x), 1), round(float(y), 1)] for x, y in pts], 'category_id': int(cat)}


def case_anns(name, i):
    """COCO extreme-point annotations: boxes partly or wholly outside the image, some of zero width or height,
    some with the top below the bottom or the left right of the right (h or w <= 0), small ones of radius 0."""
    case = CASES[name]
    h, w = case['sizes'][i]
    ids = sorted(cat_ids(case))
    r = _rng(name, i, 1)
    anns = []
    if i in case['empty']:
        return anns
    if case['crafted'] and i == 0:
        c = ids[1]
        x0, y0 = 0.45 * w, 0.45 * h
        anns.append(_ann(c, x0, y0, x0 + 0.2 * w, y0 + 0.25 * h, [0.5, 0.4, 0.6, 0.5]))
        # same class, overlapping, the same top point
        anns.append(_ann(c, x0 - 0.05 * w, y0, x0 + 0.25 * w, y0 + 0.15 * h, [0.5, 0.3, 0.5, 0.7]))
        # top and left coincide at the corner
        anns.append(_ann(ids[0], 0.4 * w, 0.4 * h, 0.55 * w, 0.6 * h, [0.0, 0.0, 0.5, 0.5]))
        # a few source pixels: radius 0
        anns.append(_ann(ids[2], 0.5 * w, 0.52 * h, 0.5 * w + 5, 0.52 * h + 4, [0.5, 0.5, 0.5, 0.5]))
        # past every border: clipped at both ends of both axes
        anns.append(_ann(ids[0], -0.6 * w, -0.6 * h, 1.6 * w, 1.6 * h, [0.3, 0.6, 0.7, 0.2]))
    lo, hi = case['n_objs']
    for _ in range(int(r.integers(lo, hi + 1))):
        x0, y0 = float(r.uniform(-0.2, 1.05) * w), float(r.uniform(-0.2, 1.05) * h)
        bw, bh = float(r.uniform(0, 0.6) * w), float(r.uniform(0, 0.6) * h)
        kind = r.random()
        if kind < 0.08:
            bw = 0.0
        elif kind < 0.14:
            bh = 0.0
        elif kind < 0.24:
            bw, bh = float(r.uniform(1, 8)), float(r.uniform(1, 8))
        x1, y1 = x0 + bw, y0 + bh
        if 0.24 <= kind < 0.28:
            y0, y1 = y1, y0       # top below bottom: h < 0
        elif 0.28 <= kind < 0.32:
            x0, x1 = x1, x0       # left right of right: w < 0
        anns.append(_ann(ids[int(r.integers(0, len(ids)))], x0, y0, x1, y1, r.random(4)))
    return anns


def case_objects(name, i):
    """What ExdetTrainInput reads from the first max_objs annotations: the float32 extreme points [n, 4, 2] and the
    classes cat_ids[category_id]."""
    case = CASES[name]
    anns = case_anns(name, i)[:case['max_objs']]
    pts = np.array([a['extreme_points'] for a in anns], np.float32).reshape(-1, 4, 2)
    ids = cat_ids(case)
    cls = np.array([ids[a['category_id']] for a in anns], np.int64)
    return pts, cls


def case_dataset(name, coco, img_dir, data_rng):
    """The attributes EXDetDataset.__getitem__ reads (COCO's, with the case's options)."""
    case = CASES[name]
    return dict(opt=make_opt(case), coco=coco, images=list(range(len(case['sizes']))), img_dir=img_dir,
                max_objs=case['max_objs'], cat_ids=cat_ids(case), mean=MEAN.reshape(1, 1, 3),
                std=STD.reshape(1, 1, 3), _data_rng=data_rng, _eig_val=EIG_VAL, _eig_vec=EIG_VEC,
                split=case['split'])


def input_sample(x):
    """The strided sample of an input [3, H, W] the golden stores (the whole input is pinned by its CRC)."""
    return x[:, ::17, ::13]

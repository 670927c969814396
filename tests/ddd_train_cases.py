"""Seeded inputs of tests/golden/train_ddd.npz (tests/golden/make_golden_train_ddd.py): per case the options of the
ddd sampler, ragged KITTI-sized images and KITTI-style annotations (the full class map: Van / Truck and
Person_sitting ignore one class, DontCare all of them, Tram / Misc are skipped), rebuilt identically on every
machine from numpy's PCG64 stream, so only what the reference returned for them is stored.  Each case's first
image also carries crafted objects: a positive drawn before an ignore region that covers it, one drawn after it,
and an ignore object on a positive's peak.  Also the float32 (h, w) pairs of the radius table."""
import math
import types

import numpy as np

# KITTI (datasets/dataset/kitti.py)
MEAN = np.array([0.485, 0.456, 0.406], np.float32)
STD = np.array([0.229, 0.224, 0.225], np.float32)
CAT_IDS = {1: 0, 2: 1, 3: 2, 4: -3, 5: -3, 6: -2, 7: -99, 8: -99, 9: -1}
CALIB = np.array([[707.0493, 0, 604.0814, 45.75831], [0, 707.0493, 180.5066, -0.3454157], [0, 0, 1., 0.004981016]],
                 np.float32)
KITTI_SIZES = [(375, 1242), (370, 1224), (374, 1238), (376, 1241), (375, 1242), (370, 1226)]

_BASE = dict(split='train', keep_res=False, input_h=384, input_w=1280, down_ratio=4, aug_ddd=0.5, scale=0.4,
             shift=0.1, rect_mask=False, reg_bbox=True, reg_offset=True, alpha_in_degree=False, num_classes=3,
             max_objs=50, n_objs=(6, 24), crafted=True)
CASES = {
    # KITTI defaults: aug_ddd 0.5, point ignores, 50 slots
    "kitti": dict(_BASE, seed=41, sizes=KITTI_SIZES),
    # rect_mask: ignore rectangles overwrite hm
    "rect": dict(_BASE, seed=42, sizes=KITTI_SIZES[:5], rect_mask=True),
    # every image augmented (reg_mask stays 0)
    "aug": dict(_BASE, seed=43, sizes=KITTI_SIZES[1:6], aug_ddd=1.0),
    # keep_res, no wh / reg heads, alpha in degrees, a small input, fewer slots than annotations
    "keep": dict(_BASE, seed=44, sizes=[(120, 400), (128, 380), (100, 390), (125, 410)], keep_res=True,
                 input_h=128, input_w=384, reg_bbox=False, reg_offset=False, alpha_in_degree=True, max_objs=6,
                 n_objs=(8, 20), crafted=False),
    # the val split draws nothing
    "val": dict(_BASE, seed=45, sizes=KITTI_SIZES[:3], split='val', rect_mask=True),
}


def make_opt(case):
    opt = types.SimpleNamespace(**{k: case[k] for k in ('keep_res', 'input_h', 'input_w', 'aug_ddd', 'scale',
                                                        'shift', 'rect_mask', 'reg_bbox', 'reg_offset',
                                                        'num_classes')})
    opt.output_h, opt.output_w = case['input_h'] // case['down_ratio'], case['input_w'] // case['down_ratio']
    opt.mse_loss = False
    opt.debug = 1          # the sampler then also returns meta (c, s)
    return opt


def _rng(name, i, what):
    return np.random.default_rng([sum(map(ord, name)) + 1000, i, what])


def case_image(name, i):
    """uint8 BGR source: noise over a diagonal ramp."""
    h, w = CASES[name]['sizes'][i]
    r = _rng(name, i, 0)
    ramp = (np.arange(h)[:, None, None] * 3 + np.arange(w)[None, :, None] * 2 + np.array([0, 85, 170])) % 256
    return ((ramp + r.integers(0, 96, (h, w, 3))) % 256).astype(np.uint8)


def _ann(r, cat, x, y, bw, bh, deg):
    alpha = float(r.uniform(-180, 180)) if deg else float(r.uniform(-math.pi, math.pi))
    if r.random() < 0.1:   # the bin boundaries
        alpha = float(r.choice([math.pi / 6, 5 * math.pi / 6, -math.pi / 6, -5 * math.pi / 6, math.pi, -math.pi]))
        alpha = math.degrees(alpha) - 45 if deg else alpha
    return {'bbox': [round(x, 2), round(y, 2), round(bw, 2), round(bh, 2)], 'category_id': int(cat), 'alpha': alpha,
            'depth': round(float(r.uniform(2, 80)), 2),
            'dim': [round(float(v), 2) for v in r.uniform([1.2, 0.4, 0.5], [4.0, 2.8, 12.0])]}


def case_anns(name, i):
    """KITTI annotations: boxes partly or wholly outside the image (wholly above or below: clipped to h <= 0),
    categories 1-9 with Car most frequent, alpha in radians (degrees with alpha_in_degree) including the bin
    boundaries, depth and dim."""
    case = CASES[name]
    h, w = case['sizes'][i]
    deg = case['alpha_in_degree']
    r = _rng(name, i, 1)
    anns = []
    if case['crafted'] and i == 0:
        x, y = 0.45 * w, 0.5 * h
        anns.append(_ann(r, 2, x, y, 60, 40, deg))                  # positive, then an ignore region over it
        anns.append(_ann(r, 9, x - 30, y - 20, 120, 80, deg))       # DontCare (all classes)
        anns.append(_ann(r, 2, x + 10, y + 5, 30, 20, deg))         # positive inside it, after it
        anns.append(_ann(r, 1, 0.2 * w, 0.3 * h, 40, 90, deg))      # positive ...
        anns.append(_ann(r, 6, 0.2 * w, 0.3 * h, 40, 90, deg))      # ... and an ignore on its peak (class 0)
        anns.append(_ann(r, 4, 0.7 * w, 0.4 * h, 80, 50, deg))      # Van: ignores class 1
        anns.append(_ann(r, 2, 0.7 * w + 20, 0.4 * h + 10, 50, 30, deg))
    lo, hi = case['n_objs']
    for _ in range(int(r.integers(lo, hi + 1))):
        cat = int(r.choice(np.arange(1, 10), p=[0.12, 0.45, 0.06, 0.08, 0.03, 0.03, 0.04, 0.04, 0.15]))
        x, y = float(r.uniform(-0.15, 1.05) * w), float(r.uniform(-0.1, 1.05) * h)
        bw, bh = float(r.uniform(2, 0.35 * w)), float(r.uniform(2, 0.6 * h))
        u = r.random()
        if u < 0.06:
            y = -bh - float(r.uniform(1, 40))       # wholly above the image
        elif u < 0.1:
            y = h + float(r.uniform(1, 40))         # wholly below
        elif u < 0.14:
            bw = 0.0
        anns.append(_ann(r, cat, x, y, bw, bh, deg))
    return anns


def case_objects(name, i):
    """What DddTrainInput reads from the first max_objs annotations: float32 corners [n, 4], classes, alpha
    (float64, after _convert_alpha), depth (float64) and dim ([n, 3] float64)."""
    case = CASES[name]
    anns = case_anns(name, i)[:case['max_objs']]
    boxes = np.array([[a['bbox'][0], a['bbox'][1], a['bbox'][0] + a['bbox'][2], a['bbox'][1] + a['bbox'][3]]
                      for a in anns], np.float32).reshape(-1, 4)
    cls = np.array([CAT_IDS[a['category_id']] for a in anns], np.int64)
    conv = (lambda a: math.radians(a + 45)) if case['alpha_in_degree'] else (lambda a: a)
    alpha = np.array([conv(a['alpha']) for a in anns], np.float64)
    depth = np.array([a['depth'] for a in anns], np.float64)
    dim = np.array([a['dim'] for a in anns], np.float64).reshape(-1, 3)
    return boxes, cls, alpha, depth, dim


def case_dataset(name, coco, img_dir, data_rng):
    """The attributes DddDataset.__getitem__ reads (KITTI's, with the case's options)."""
    case = CASES[name]
    return dict(opt=make_opt(case), coco=coco, images=list(range(len(case['sizes']))), img_dir=img_dir,
                max_objs=case['max_objs'], cat_ids=dict(CAT_IDS), alpha_in_degree=case['alpha_in_degree'],
                mean=MEAN.reshape(1, 1, 3), std=STD.reshape(1, 1, 3), split=case['split'], calib=CALIB,
                _data_rng=data_rng, _eig_val=np.zeros(3, np.float32), _eig_vec=np.eye(3, dtype=np.float32))


def input_sample(x):
    """The strided sample of an input [3, H, W] the golden stores (the whole input is pinned by its CRC)."""
    return x[:, ::37, ::29]


RADIUS_PAIRS = 1 << 20
NEAR_ULPS = 4


def radius_pairs():
    """The random float32 (h, w) pairs of the radius table: KITTI-sized output boxes, a quarter of them small."""
    r = np.random.default_rng(4711)
    h = r.uniform(0, 96, RADIUS_PAIRS).astype(np.float32)
    w = r.uniform(0, 320, RADIUS_PAIRS).astype(np.float32)
    small = r.random(RADIUS_PAIRS) < 0.25
    h[small] = (h[small] / 24).astype(np.float32)
    w[small] = (w[small] / 40).astype(np.float32)
    ok = (h > 0) & (w > 0)
    return h[ok], w[ok]


def near_pairs(h0, w0):
    """The near-integer pairs of the radius table from its base pairs: per base pair (h0, w0) the widths w0 - 4 ulp
    .. w0 + 4 ulp in order, at the same h0.  Returns float32 h, w of 9 entries per base pair."""
    h0, w0 = np.asarray(h0, np.float32), np.asarray(w0, np.float32)
    lo, hi = [w0], [w0]
    for _ in range(NEAR_ULPS):
        lo.insert(0, np.nextafter(lo[0], np.float32(0)))
        hi.append(np.nextafter(hi[-1], np.float32(np.inf)))
    w = np.stack(lo + hi[1:], 1).reshape(-1)
    return np.repeat(h0, 2 * NEAR_ULPS + 1), w

"""numpy restatement of the ddd training sampler's targets and hm given its drawn parameters
(datasets/sample/ddd.py:86-140), written from the numeric contract of DESIGN.md section 4.11 and pinned by
tests/golden/train_ddd.npz (the unmodified DddDataset.__getitem__ on seeded images).  The float32 affine map and the
image are those of tests/train_np.py; hm is painted in object order as the reference paints it."""
import numpy as np

from oracle import image_np
from train_np import affine_f32

F32 = np.float32


def _sq(b):
    """b ** 2 of float32 scalars as numpy evaluates it (float32 scalar power: the C library's powf)."""
    return np.array([F32(v) ** 2 for v in np.asarray(b, F32).reshape(-1)], F32).reshape(np.shape(b))


def gaussian_radius_f32(h, w, square=_sq):
    """gaussian_radius((h, w)) (utils/image.py:95-115) on float32 h, w: every operation float32, the Python
    constants rounded to float32 at each use, numpy's left-to-right order, min(r1, r2, r3) the first smallest;
    b ** 2 is `square` (numpy's scalar power by default)."""
    h, w = np.asarray(h, F32), np.asarray(w, F32)
    b1 = (h + w).astype(F32)
    c1 = (((w * h).astype(F32) * F32(0.3)).astype(F32) / F32(1.7)).astype(F32)
    r1 = ((b1 + np.sqrt((square(b1) - (F32(4) * c1).astype(F32)).astype(F32))).astype(F32) / F32(2)).astype(F32)
    b2 = (F32(2) * (h + w).astype(F32)).astype(F32)
    c2 = ((F32(0.3) * w).astype(F32) * h).astype(F32)
    r2 = ((b2 + np.sqrt((square(b2) - (F32(16) * c2).astype(F32)).astype(F32))).astype(F32) / F32(2)).astype(F32)
    b3 = (F32(-1.4) * (h + w).astype(F32)).astype(F32)
    c3 = ((F32(-0.3) * w).astype(F32) * h).astype(F32)
    r3 = ((b3 + np.sqrt((square(b3) - (F32(4 * 2.8) * c3).astype(F32)).astype(F32))).astype(F32) / F32(2)).astype(F32)
    m = np.where(r2 < r1, r2, r1)
    return np.where(r3 < m, r3, m).astype(F32)


def ddd_targets(boxes, cls, alpha, depth, dim, aug, trans_output, max_objs, num_classes, out_h, out_w, rect_mask):
    """ddd.py:86-140 for one image: float32 corners boxes [n, 4], classes, alpha (float64, converted), depth and dim
    -> dict of the targets (hm, dep, dim, ind, rotbin, rotres, reg_mask, rot_mask, wh, reg) with the reference's
    shapes and dtypes."""
    m, C = max_objs, num_classes
    r = {'hm': np.zeros((C, out_h, out_w), F32), 'wh': np.zeros((m, 2), F32), 'reg': np.zeros((m, 2), F32),
         'dep': np.zeros((m, 1), F32), 'rotbin': np.zeros((m, 2), np.int64), 'rotres': np.zeros((m, 2), F32),
         'dim': np.zeros((m, 3), F32), 'ind': np.zeros(m, np.int64), 'reg_mask': np.zeros(m, np.uint8),
         'rot_mask': np.zeros(m, np.uint8)}
    hm = r['hm']
    for k in range(min(len(boxes), m)):
        c = int(cls[k])
        if c <= -99:
            continue
        x0, y0 = affine_f32(trans_output, boxes[k][0], boxes[k][1])
        x1, y1 = affine_f32(trans_output, boxes[k][2], boxes[k][3])
        x0, x1 = [F32(min(max(v, F32(0)), F32(out_w - 1))) for v in (x0, x1)]
        y0, y1 = [F32(min(max(v, F32(0)), F32(out_h - 1))) for v in (y0, y1)]
        h, w = F32(y1 - y0), F32(x1 - x0)
        if not (h > 0 and w > 0):
            continue
        rad = max(0, int(gaussian_radius_f32(h, w)))
        ct = np.array([(x0 + x1) / F32(2), (y0 + y1) / F32(2)], F32)
        ci = ct.astype(np.int32)
        if c < 0:
            ignore = list(range(C)) if c == -1 else [-c - 2]
            if rect_mask:
                hm[ignore, int(y0):int(y1) + 1, int(x0):int(x1) + 1] = F32(0.9999)
            else:
                for cc in ignore:
                    image_np.draw_umich_gaussian(hm[cc], ct, rad)
                hm[ignore, ci[1], ci[0]] = F32(0.9999)
            continue
        image_np.draw_umich_gaussian(hm[c], ct, rad)
        r['wh'][k] = w, h
        a = float(alpha[k])
        if a < np.pi / 6. or a > 5 * np.pi / 6.:
            r['rotbin'][k, 0] = 1
            r['rotres'][k, 0] = a - (-0.5 * np.pi)
        if a > -np.pi / 6. or a < -5 * np.pi / 6.:
            r['rotbin'][k, 1] = 1
            r['rotres'][k, 1] = a - (0.5 * np.pi)
        r['dep'][k] = depth[k]
        r['dim'][k] = dim[k]
        r['ind'][k] = int(ci[1]) * out_w + int(ci[0])
        r['reg'][k] = ct - ci
        r['reg_mask'][k] = 0 if aug else 1
        r['rot_mask'][k] = 1
    return r

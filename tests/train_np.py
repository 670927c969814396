"""numpy restatement of the ctdet training sampler given its drawn parameters (datasets/sample/ctdet.py:69-127 and
color_aug, utils/image.py:198-230), written from the numeric contract of DESIGN.md section 4.9 and pinned by
tests/golden/train.npz (the unmodified CTDetDataset.__getitem__ on seeded images):
  warp          oracle.pre_np.warp_affine_linear of the source, mirrored first (img[:, ::-1]) when flipped;
  grey          cv2.cvtColor(float32 BGR -> GRAY) = fma(r, 0.299f, fma(b, 0.114f, g * 0.587f)), each fma one
                rounding of the exact value (emulated in long double, where a * b + c is exact at these scales);
  gs.mean()     numpy's pairwise float32 sum (the fixed tree of pairwise_sum_f32) / n in float32;
  blends        float32 x * a, + f32(gs_mean * b) (contrast), + f32(gs * b) (saturation);
  lighting      f32(f64(x) + d[c]);
  targets       float64 t0 x + t1 y + t2 rounded to float32, the rest as ctdet.py in float32 / float64."""
import numpy as np

from oracle import image_np, pre_np

F32 = np.float32
ORDERS = ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))


def fma_f32(a, b, c):
    """float32 fused multiply-add (one rounding).  a * b is exact in float64; the sum is exact in x86 long double
    for the [0, 1] operands of the grey conversion."""
    ld = np.longdouble
    return (np.asarray(a, F32).astype(np.float64).astype(ld) * np.asarray(b, F32).astype(ld)
            + np.asarray(c, F32).astype(ld)).astype(F32)


def grey(x):
    """cv2.cvtColor(x, COLOR_BGR2GRAY) of a float32 [H, W, 3] image."""
    b, g, r = x[..., 0], x[..., 1], x[..., 2]
    return fma_f32(r, F32(0.299), fma_f32(b, F32(0.114), (g * F32(0.587)).astype(F32)))


def _leaves(n, start=0, out=None):
    out = [] if out is None else out
    if n <= 128:
        out.append((start, n))
        return out
    h = n // 2
    h -= h % 8
    _leaves(h, start, out)
    _leaves(n - h, start + h, out)
    return out


def _leaf_sums(a, leaves):
    sums = {}
    for length in sorted({n for _, n in leaves}):
        starts = np.array([s for s, n in leaves if n == length], np.int64)
        v = a[starts[:, None] + np.arange(length)[None, :]]
        if length < 8:
            res = np.zeros(len(starts), F32)
            for i in range(length):
                res = (res + v[:, i]).astype(F32)
        else:
            r = v[:, :8].copy()
            i = 8
            while i < length - length % 8:
                r = (r + v[:, i:i + 8]).astype(F32)
                i += 8
            res = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
            for j in range(i, length):
                res = (res + v[:, j]).astype(F32)
        sums.update(zip(starts.tolist(), res.astype(F32)))
    return sums


def pairwise_sum_f32(a):
    """numpy's pairwise summation of a float32 vector: n < 8 in order; n <= 128 eight strided accumulators
    combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) plus the n % 8 tail; else the two halves split at
    n/2 - (n/2) % 8."""
    a = np.ascontiguousarray(a, F32).reshape(-1)
    sums = _leaf_sums(a, _leaves(a.size))

    def rec(n, start):
        if n <= 128:
            return sums[start]
        h = n // 2
        h -= h % 8
        return F32(rec(h, start) + rec(n - h, start + h))

    return F32(rec(a.size, 0))


def grey_mean(gs):
    """gs.mean() of a float32 grey image."""
    return F32(pairwise_sum_f32(gs) / F32(gs.size))


def color_aug(x, order, blend, light):
    """color_aug on the float32 [H, W, 3] image x / 255, given the drawn order code, blend (a, b) pairs of
    brightness, contrast, saturation, and the lighting offsets."""
    gs = grey(x)
    gs_mean = grey_mean(gs)
    x = x.copy()
    for kind in ORDERS[order]:
        a, b = F32(blend[2 * kind]), F32(blend[2 * kind + 1])
        x = (x * a).astype(F32)
        if kind == 1:
            x = (x + F32(gs_mean * b)).astype(F32)
        elif kind == 2:
            x = (x + (gs * b).astype(F32)[..., None]).astype(F32)
    return (x.astype(np.float64) + np.asarray(light, np.float64).reshape(1, 1, 3)).astype(F32)


def train_image(img, matrix, flip, out_w, out_h, mean, std, order=-1, blend=None, light=None):
    """One training input [3, out_h, out_w] float32: warp (forward matrix), /255, color_aug when order >= 0,
    (x - mean) / std, CHW."""
    src = img[:, ::-1, :] if flip else img
    x = pre_np.warp_affine_linear(np.ascontiguousarray(src), matrix, (out_w, out_h)).astype(F32) / F32(255)
    if order >= 0:
        x = color_aug(x, order, blend, light)
    x = ((x - np.asarray(mean, F32).reshape(1, 1, 3)) / np.asarray(std, F32).reshape(1, 1, 3)).astype(F32)
    return x.transpose(2, 0, 1)


def affine_f32(t, x, y):
    """affine_transform of one float32 point, float64 t0 x + t1 y + t2 in that order, rounded to float32."""
    t = np.asarray(t, np.float64).reshape(2, 3)
    x, y = np.float64(F32(x)), np.float64(F32(y))
    return F32(t[0, 0] * x + t[0, 1] * y + t[0, 2]), F32(t[1, 0] * x + t[1, 1] * y + t[1, 2])


def ctdet_targets(boxes, cls, flip, width, trans_output, max_objs, num_classes, out_h, out_w):
    """ctdet.py:99-127 for one image: boxes [n, 4] float32 corners, cls [n] -> dict of wh, ind, reg, reg_mask,
    cat_spec_wh, cat_spec_mask and the FocalSplatLoss lists (obj_cls, obj_cx, obj_cy, obj_radius, obj_valid)."""
    m = max_objs
    r = {'wh': np.zeros((m, 2), F32), 'reg': np.zeros((m, 2), F32), 'ind': np.zeros(m, np.int64),
         'reg_mask': np.zeros(m, np.uint8), 'cat_spec_wh': np.zeros((m, 2 * num_classes), F32),
         'cat_spec_mask': np.zeros((m, 2 * num_classes), np.uint8)}
    for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius'):
        r[k] = np.zeros(m, np.int32)
    r['obj_valid'] = np.zeros(m, np.uint8)
    for k in range(min(len(boxes), m)):
        x0, y0, x1, y1 = [F32(v) for v in boxes[k]]
        if flip:
            x0, x1 = F32(F32(F32(width) - x1) - F32(1)), F32(F32(F32(width) - x0) - F32(1))
        x0, y0 = affine_f32(trans_output, x0, y0)
        x1, y1 = affine_f32(trans_output, x1, y1)
        x0, x1 = [F32(min(max(v, F32(0)), F32(out_w - 1))) for v in (x0, x1)]
        y0, y1 = [F32(min(max(v, F32(0)), F32(out_h - 1))) for v in (y0, y1)]
        h, w = F32(y1 - y0), F32(x1 - x0)
        if h > 0 and w > 0:
            rad = max(0, int(image_np.gaussian_radius((int(np.ceil(h)), int(np.ceil(w))))))
            ct = np.array([(x0 + x1) / F32(2), (y0 + y1) / F32(2)], F32)
            ci = ct.astype(np.int32)
            c = int(cls[k])
            r['wh'][k] = w, h
            r['ind'][k] = int(ci[1]) * out_w + int(ci[0])
            r['reg'][k] = ct - ci.astype(F32)
            r['reg_mask'][k] = 1
            r['cat_spec_wh'][k, 2 * c:2 * c + 2] = w, h
            r['cat_spec_mask'][k, 2 * c:2 * c + 2] = 1
            r['obj_cls'][k], r['obj_cx'][k], r['obj_cy'][k], r['obj_radius'][k] = c, ci[0], ci[1], rad
            r['obj_valid'][k] = 1
    return r


def gaussian_radius_ops(height, width):
    """gaussian_radius((height, width)) for integer sides as the device evaluates it: each float64 operation of
    utils/image.py:95-115 in source order, b3 ** 2 as b3 * b3."""
    mo1 = 0.30000000000000004
    b1 = height + width
    c1 = float(width * height) * mo1 / 1.7
    r1 = (b1 + np.sqrt(float(b1 * b1) - 4.0 * c1)) / 2.0
    b2 = 2 * (height + width)
    c2 = mo1 * width * height
    r2 = (b2 + np.sqrt(float(b2 * b2) - 16.0 * c2)) / 2.0
    b3 = -1.4 * (height + width)
    c3 = -mo1 * width * height
    r3 = (b3 + np.sqrt(b3 * b3 - (4.0 * 2.8) * c3)) / 2.0
    return min(r1, r2, r3)

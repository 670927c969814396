"""CPU restatement of the ddd detector's tail (TEST INFRASTRUCTURE), row by row as the reference computes it, so that
it is also the host baseline tools/detector_tail_time.py times:

  utils/post_process.py:13-47     get_alpha, ddd_post_process_2d (back-projection, alpha, per-class columns)
  utils/post_process.py:49-80     ddd_post_process_3d (box, location, rot_y per row; calibs[0] for every image)
  utils/ddd_utils.py:66-111       unproject_2d_to_3d, alpha2rot_y, ddd2locrot
  detectors/ddd.py:75-88          post_process + merge_outputs (score > peak_thresh)

Pinned by tests/golden/ddd_tail.npz (tests/golden/make_golden_ddd_tail.py runs the unmodified reference)."""
import numpy as np

from centernet_b200.post_process import cv_inv_affine
from oracle.post_np import F32

HALF_PI, PI, TWO_PI = F32(0.5 * np.pi), F32(np.pi), F32(2 * np.pi)


def affine_points(coords, center, scale, output_size):
    """transform_preds (utils/image.py:19-24) point by point: (t0 x + t1 y) + t2 in float64 with the point in float32,
    on cv2.getAffineTransform's own matrix (restated bit for bit by cv_inv_affine: at the KITTI metas the plain
    float64 solve misses it by one ulp).  coords [N, 2] -> float64 [N, 2]."""
    t = cv_inv_affine(center, scale, output_size)
    x = np.asarray(coords, F32)[:, 0].astype(np.float64)
    y = np.asarray(coords, F32)[:, 1].astype(np.float64)
    return np.stack([(t[0, 0] * x + t[0, 1] * y) + t[0, 2], (t[1, 0] * x + t[1, 1] * y) + t[1, 2]], 1)


def get_alpha(rot):
    """rot [n, 8] float32 -> float64 [n]: bin 1 when rot[1] > rot[5] (NaN and ties pick bin 2), each bin's
    atan2(sin, cos) -+ float32(pi / 2) in float32.  The reference blends the bins as alpha1 * idx + alpha2 * (1 - idx),
    in float64 (1 - bool is int64), so a NaN in either bin makes alpha NaN."""
    a1 = np.arctan2(rot[:, 2], rot[:, 3]) - HALF_PI
    a2 = np.arctan2(rot[:, 6], rot[:, 7]) + HALF_PI
    out = np.where(rot[:, 1] > rot[:, 5], a1, a2).astype(np.float64)
    out[np.isnan(a1) | np.isnan(a2)] = np.nan
    return out


def _class_rows(d, j):
    """Rows whose class (last column) equals j: -0.0 is class 0; NaN, non-integer and out-of-range ids match none."""
    return d[d[:, -1] == j]


def post_process_2d(dets, c, s, out_w, out_h, num_classes):
    """-> list (per image) of {class id: float32 [n, 10] = x, y, score, alpha, depth, dim[3], w, h} (image frame)."""
    if dets.shape[2] <= 16:
        raise ValueError("ddd dets without wh (16 columns) cannot be post-processed")
    ret = []
    for i in range(dets.shape[0]):
        d = np.array(dets[i], F32, copy=True)
        d[:, 0:2] = affine_points(d[:, 0:2], c[i], s[i], (out_w, out_h))
        per = {}
        for j in range(num_classes):
            r = _class_rows(d, j)
            per[j + 1] = np.concatenate([r[:, 0:3], get_alpha(r[:, 3:11])[:, None].astype(F32), r[:, 11:15],
                                         affine_points(r[:, 15:17], c[i], s[i], (out_w, out_h)).astype(F32)], axis=1)
        ret.append(per)
    return ret


def locrot(center, alpha, dim, depth, P):
    """unproject_2d_to_3d + Y += dim0 / 2 and alpha2rot_y for one row, float32 scalar steps left to right; the
    wrap compares with float32(pi) (a float32 scalar against a Python float compares in float32 under numpy 2)."""
    z = depth - P[2, 3]
    x = (center[0] * depth - P[0, 3] - P[0, 2] * z) / P[0, 0]
    y = (center[1] * depth - P[1, 3] - P[1, 2] * z) / P[1, 1]
    y = y + dim[0] / F32(2)
    rot_y = alpha + np.arctan2(center[0] - P[0, 2], P[0, 0])
    if rot_y > PI:
        rot_y = rot_y - TWO_PI
    if rot_y < -PI:
        rot_y = rot_y + TWO_PI
    return (x, y, z), rot_y


def post_process_3d(dets2d, calibs):
    """dets2d from post_process_2d -> {class id: float32 [n, 13] = alpha, x1, y1, x2, y2, dim[3], X, Y, Z, rot_y,
    score}, np.array([], float32) for a class without rows.  calibs[0] serves every image, as in the reference."""
    P = np.asarray(calibs[0], F32)
    ret = []
    for per in dets2d:
        out = {}
        for cls, rows in per.items():
            preds = []
            for r in rows:
                cx, cy, score, alpha, depth = r[0], r[1], r[2], r[3], r[4]
                dim, w, h = r[5:8], r[8], r[9]
                loc, rot_y = locrot(r[0:2], alpha, dim, depth, P)
                preds.append([alpha, cx - w / F32(2), cy - h / F32(2), cx + w / F32(2), cy + h / F32(2),
                              dim[0], dim[1], dim[2], loc[0], loc[1], loc[2], rot_y, score])
            out[cls] = np.array(preds, dtype=F32)
        ret.append(out)
    return ret


def ddd_post_process(dets, c, s, calibs, out_w, out_h, num_classes):
    """utils/post_process.py:75-80; dets [B, K, 18] float32 (left unmodified)."""
    return post_process_3d(post_process_2d(np.asarray(dets, F32), c, s, out_w, out_h, num_classes), calibs)


def merge_outputs(results, num_classes, peak_thresh):
    """detectors/ddd.py:82-88: a non-empty class keeps its rows with score > peak_thresh (compared in float32: NaN
    dropped, +inf kept); an empty class keeps its shape (0,)."""
    out = dict(results)
    for j in range(1, num_classes + 1):
        if len(out[j]):
            out[j] = out[j][out[j][:, -1] > F32(peak_thresh)]
    return out


def detector_tail(dets, meta, num_classes, peak_thresh=0.2):
    """DddDetector.post_process + merge_outputs run once per image, each with its own calibration: dets [B, K, 18],
    meta with per-image 'c', 's', 'calib' and 'out_height', 'out_width'."""
    res = []
    for i in range(dets.shape[0]):
        r = ddd_post_process(dets[i:i + 1], [meta["c"][i]], [meta["s"][i]], [meta["calib"][i]], meta["out_width"],
                             meta["out_height"], num_classes)[0]
        res.append(merge_outputs(r, num_classes, peak_thresh))
    return res

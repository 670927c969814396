"""CPU restatement of the reference's detection post-processing (TEST INFRASTRUCTURE, SURVEY 8f N2):

  utils/image.py:19-24,27-60,63-71  transform_preds / get_affine_transform / affine_transform
  utils/post_process.py:83-114      ctdet_post_process, multi_pose_post_process
  external/nms.pyx:77-169,171-275   soft_nms, soft_nms_39 (in-place, swap-with-last discard)
  detectors/ctdet.py:76-92          merge_outputs (concat over scales, soft-NMS, top max_per_image)

Pinned by tests/golden/post.npz (tests/golden/make_golden_post.py runs the unmodified reference functions
and the reference's Cython soft-NMS compiled by oracle/build_ref.py)."""
import numpy as np

F32 = np.float32


def get_affine_transform_inv(center, scale, output_size):
    """utils/image.py:27-60 with rot = 0, shift = 0, inv = 1: the 2x3 float64 matrix mapping output-grid
    coordinates back to image coordinates.  Point construction in float32 as the reference; the 3-point solve
    (cv2.getAffineTransform there) in float64."""
    if not isinstance(scale, (np.ndarray, list, tuple)):
        scale = np.array([scale, scale], dtype=F32)
    scale = np.asarray(scale, dtype=F32)
    center = np.asarray(center, dtype=F32)
    src_w = scale[0]
    dst_w, dst_h = output_size[0], output_size[1]
    src_dir = np.array([0.0, src_w * F32(-0.5)], F32)      # get_dir([0, src_w * -0.5], 0), :74-81
    dst_dir = np.array([0, dst_w * -0.5], F32)
    src = np.zeros((3, 2), F32); dst = np.zeros((3, 2), F32)
    src[0] = center
    src[1] = center + src_dir
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5], F32) + dst_dir
    third = lambda a, b: b + np.array([-(a - b)[1], (a - b)[0]], F32)   # get_3rd_point, :69-71
    src[2] = third(src[0], src[1]); dst[2] = third(dst[0], dst[1])
    A = np.concatenate([dst.astype(np.float64), np.ones((3, 1))], axis=1)      # [x y 1] . m = x'
    return np.linalg.solve(A, src.astype(np.float64)).T                         # 2 x 3


def transform_preds(coords, center, scale, output_size):
    """utils/image.py:19-24: float64 result of t . [x, y, 1] with the point in float32."""
    t = get_affine_transform_inv(center, scale, output_size)
    coords = np.asarray(coords)
    out = np.zeros(coords.shape)
    pts = np.concatenate([coords[:, 0:2].astype(F32), np.ones((coords.shape[0], 1), F32)], axis=1)
    out[:, 0:2] = pts.astype(np.float64) @ t.T
    return out


def ctdet_post_process(dets, c, s, h, w, num_classes):
    """utils/post_process.py:83-99 -> list (per image) of {class id (1-based): [[x1,y1,x2,y2,score], ...]}."""
    dets = np.array(dets, dtype=F32, copy=True)
    ret = []
    for i in range(dets.shape[0]):
        dets[i, :, :2] = transform_preds(dets[i, :, 0:2], c[i], s[i], (w, h))
        dets[i, :, 2:4] = transform_preds(dets[i, :, 2:4], c[i], s[i], (w, h))
        classes = dets[i, :, -1]
        ret.append({j + 1: dets[i, classes == j, :5].astype(F32) for j in range(num_classes)})
    return ret


def multi_pose_post_process(dets, c, s, h, w):
    """utils/post_process.py:102-114 -> list of {1: [N, 39]} (bbox 4, score, 17 keypoints)."""
    dets = np.asarray(dets, dtype=F32)
    ret = []
    for i in range(dets.shape[0]):
        bbox = transform_preds(dets[i, :, :4].reshape(-1, 2), c[i], s[i], (w, h))
        pts = transform_preds(dets[i, :, 5:39].reshape(-1, 2), c[i], s[i], (w, h))
        ret.append({1: np.concatenate([bbox.reshape(-1, 4), dets[i, :, 4:5], pts.reshape(-1, 34)], axis=1).astype(F32)})
    return ret


def _min(a, b):
    """nms.pyx:21-22 (`a if a <= b else b`): a NaN `b` is returned, a NaN `a` is not -- unlike Python's min."""
    return a if a <= b else b


def _max(a, b):
    """nms.pyx:18-19 (`a if a >= b else b`)."""
    return a if a >= b else b


def _pivot(scores, i):
    """nms.pyx:87-102: `maxscore = boxes[i, 4]`, then `if maxscore < boxes[pos, 4]` over the later rows.  A NaN at
    row i is never replaced; otherwise the first maximum wins and NaN rows are never picked (np.argmax would take
    the first NaN)."""
    s = scores[i:]
    if np.isnan(s[0]):
        return i
    return i + int(np.argmax(np.where(np.isnan(s), -np.inf, s)))


def soft_nms(boxes, sigma=0.5, Nt=0.3, threshold=0.001, method=0, ncols_swap=0):
    """external/nms.pyx:77-169 (ncols_swap = 0) and :171-275 (soft_nms_39: ncols_swap = 34 extra columns that are
    SWAPPED where the five box columns are COPIED).  In place on the float32 array; returns the final N.
    Float32 storage, with the double-precision intermediates the generated C has (integer literals become 1.0)."""
    N = boxes.shape[0]
    sigma, Nt, threshold = F32(sigma), F32(Nt), F32(threshold)
    one = F32(1)
    i = 0
    while i < N:
        maxpos = _pivot(boxes[:N, 4], i)
        t = boxes[i, :5].copy()
        boxes[i, :5] = boxes[maxpos, :5]
        boxes[maxpos, :5] = t
        if ncols_swap:
            k = boxes[i, 5:5 + ncols_swap].copy()
            boxes[i, 5:5 + ncols_swap] = boxes[maxpos, 5:5 + ncols_swap]
            boxes[maxpos, 5:5 + ncols_swap] = k
        tx1, ty1, tx2, ty2 = boxes[i, 0], boxes[i, 1], boxes[i, 2], boxes[i, 3]
        pos = i + 1
        while pos < N:
            x1, y1, x2, y2 = boxes[pos, 0], boxes[pos, 1], boxes[pos, 2], boxes[pos, 3]
            # Cython turns the literal 1 into the C double 1.0: float differences, then double arithmetic, one
            # rounding on assignment to the `cdef float` (see the generated C of nms.pyx:133-139)
            D = np.float64
            area = F32((D(F32(x2 - x1)) + 1.0) * (D(F32(y2 - y1)) + 1.0))
            iw = F32(D(F32(_min(tx2, x2) - _max(tx1, x1))) + 1.0)
            if iw > 0:
                ih = F32(D(F32(_min(ty2, y2) - _max(ty1, y1))) + 1.0)
                if ih > 0:
                    ua = F32(((D(F32(tx2 - tx1)) + 1.0) * (D(F32(ty2 - ty1)) + 1.0) + D(area)) - D(F32(iw * ih)))
                    ov = F32(F32(iw * ih) / ua)
                    if method == 1:
                        weight = F32(1.0 - D(ov)) if ov > Nt else one
                    elif method == 2:
                        weight = F32(np.exp(float(F32(F32(-F32(ov * ov)) / sigma))))
                    else:
                        weight = F32(0) if ov > Nt else one
                    boxes[pos, 4] = F32(weight * boxes[pos, 4])
                    if boxes[pos, 4] < threshold:
                        boxes[pos, :5] = boxes[N - 1, :5]
                        if ncols_swap:
                            k = boxes[pos, 5:5 + ncols_swap].copy()
                            boxes[pos, 5:5 + ncols_swap] = boxes[N - 1, 5:5 + ncols_swap]
                            boxes[N - 1, 5:5 + ncols_swap] = k
                        N -= 1
                        pos -= 1
            pos += 1
        i += 1
    return N


def merge_outputs(detections, num_classes, max_per_image=100, run_nms=True):
    """detectors/ctdet.py:76-92.  detections: list (per scale) of {class: [n, 5]}.  soft_nms's keep list is
    ignored by the reference, so every row -- stale duplicates beyond N included -- stays in the result."""
    results = {}
    for j in range(1, num_classes + 1):
        results[j] = np.concatenate([d[j] for d in detections], axis=0).astype(F32)
        if run_nms:
            soft_nms(results[j], Nt=0.5, method=2)
    scores = np.hstack([results[j][:, 4] for j in range(1, num_classes + 1)])
    if len(scores) > max_per_image:
        kth = len(scores) - max_per_image
        thresh = np.partition(scores, kth)[kth]
        for j in range(1, num_classes + 1):
            results[j] = results[j][results[j][:, 4] >= thresh]
    return results

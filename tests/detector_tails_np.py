"""CPU restatement of the multi_pose and exdet detector tails (TEST INFRASTRUCTURE), on the numpy soft-NMS of
oracle/post_np.py:

  utils/image.py:19-24,63-66        transform_preds / affine_transform, point by point
  detectors/multi_pose.py:75-81     merge_outputs (concat over scales, soft_nms_39)
  detectors/exdet.py:85-95          post_process (un-mirroring of the second half, back-projection, scale)
  detectors/exdet.py:97-122         merge_outputs (score > 0, per-class soft-NMS, top max_per_image)

Pinned by tests/golden/detector_tails.npz (tests/golden/make_golden_detector_tails.py runs the unmodified
reference detectors with the reference's compiled soft-NMS).  `soft_nms` is looked up in this module, so a caller
may set it to the compiled routine (tools/detector_tail_time.py does)."""
import numpy as np

from oracle.post_np import F32, get_affine_transform_inv, soft_nms  # noqa: F401  (soft_nms: replaceable)


def affine_points(coords, center, scale, output_size):
    """transform_preds (utils/image.py:19-24) as affine_transform (:63-66) computes it point by point:
    np.dot(t, [x, y, 1.]) = (t0 x + t1 y) + t2 in float64 with the point in float32, elementwise so that no fused
    multiply-add or BLAS summation order enters.  coords [N, 2] -> float64 [N, 2]."""
    t = get_affine_transform_inv(center, scale, output_size)
    x = np.asarray(coords, F32)[:, 0].astype(np.float64)
    y = np.asarray(coords, F32)[:, 1].astype(np.float64)
    return np.stack([(t[0, 0] * x + t[0, 1] * y) + t[0, 2], (t[1, 0] * x + t[1, 1] * y) + t[1, 2]], 1)


def multi_pose_merge_outputs(detections, run_nms):
    """detectors/multi_pose.py:75-81.  detections: list (per scale) of {1: [n, 39]} (post_process of each scale,
    the division by the scale included).  Returns {1: [N, 39] float32}; every row stays, as the reference keeps
    them (it returns `.tolist()` of this array)."""
    res = np.concatenate([d[1] for d in detections], axis=0).astype(F32)
    if run_nms:
        soft_nms(res, Nt=0.5, method=2, ncols_swap=34)
    return {1: res}


def exdet_post_process(dets, meta, scale=1):
    """detectors/exdet.py:85-95 for one image: dets [P, N, 14] (P = 2 with flip: the image and its mirror) ->
    [P*N, 14] float32.  The rows are split into two equal halves as reshape(2, -1, 14) splits them (without flip
    too: the reference then mirrors the second half of the image's own rows), x1 / x2 of the second half become
    out_width - x2 / out_width - x1, both corners are back-projected, then divided by the scale."""
    out_width, out_height = meta["out_width"], meta["out_height"]
    dets = np.array(dets, dtype=F32, copy=True).reshape(2, -1, 14)
    x1, x2 = dets[1, :, 0].copy(), dets[1, :, 2].copy()
    dets[1, :, 0] = F32(out_width) - x2
    dets[1, :, 2] = F32(out_width) - x1
    dets = dets.reshape(-1, 14)
    dets[:, 0:2] = affine_points(dets[:, 0:2], meta["c"], meta["s"], (out_width, out_height))
    dets[:, 2:4] = affine_points(dets[:, 2:4], meta["c"], meta["s"], (out_width, out_height))
    dets[:, 0:4] /= F32(scale)
    return dets


def exdet_merge_outputs(detections, num_classes, max_per_image=100):
    """detectors/exdet.py:97-122 with the compiled soft_nms in scope.  detections: list (per scale) of [n, 14].
    Rows with score > 0 (NaN dropped), grouped by the class in the last column, Gaussian soft-NMS (Nt 0.5) on
    every class list (all rows kept), then the max_per_image cut.  Returns {class id: [n, 5] float32}."""
    det = np.concatenate(list(detections), axis=0).astype(F32)
    det = det[det[:, 4] > 0]
    classes = det[:, -1]
    results = {}
    for j in range(num_classes):
        results[j + 1] = det[classes == j][:, 0:5].astype(F32)
        soft_nms(results[j + 1], Nt=0.5, method=2)
    scores = np.hstack([results[j][:, -1] for j in range(1, num_classes + 1)])
    if len(scores) > max_per_image:
        kth = len(scores) - max_per_image
        thresh = np.partition(scores, kth)[kth]
        for j in range(1, num_classes + 1):
            results[j] = results[j][results[j][:, -1] >= thresh]
    return results

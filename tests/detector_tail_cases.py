"""Inputs of tests/golden/detector_tails.npz (tests/golden/make_golden_detector_tails.py) and the numpy oracle of
the multi_pose / exdet tails (tests/detector_tails_np.py) run on them, shared by the CPU and GPU tests."""
import numpy as np

import detector_tails_np as O


def _metas(g, name):
    c, s, scalar = g[name + "_c"], g[name + "_s"], g[name + "_s_scalar"]
    scales, hw = g[name + "_scales"], g[name + "_hw"]
    return [{"c": [c[k, i] for i in range(c.shape[1])],
             "s": [np.float32(s[k, i, 0]) if scalar[i] else s[k, i] for i in range(c.shape[1])],
             "out_height": int(hw[k, 0]), "out_width": int(hw[k, 1]), "scale": float(scales[k])}
            for k in range(len(scales))]


def multi_pose_case(g, name):
    """Per-scale [B, K, 40] detections, the metas of multi_pose_merge_device and the nms flag."""
    dets = g[name + "_dets"]
    return [dets[k] for k in range(dets.shape[0])], _metas(g, name), bool(int(g[name + "_nms"]))


def exdet_case(g, name):
    """Per-scale [P*B, N, 14] detections, the metas of exdet_merge_device, num_classes, max_per_image, flip."""
    dets = g[name + "_dets"]
    nc, mpi, flip = (int(v) for v in g[name + "_cfg"])
    return [dets[k] for k in range(dets.shape[0])], _metas(g, name), nc, mpi, bool(flip)


def _image_meta(m, i):
    return {"c": m["c"][i], "s": m["s"][i], "out_height": m["out_height"], "out_width": m["out_width"]}


def oracle_multi_pose(dets, metas, nms):
    """MultiPoseDetector.post_process of every image and scale + merge_outputs -> [B, N, 39]."""
    out = []
    for i in range(dets[0].shape[0]):
        per_scale = []
        for d, m in zip(dets, metas):      # utils/post_process.py:102-114, then the division by the scale
            size = (m["out_width"], m["out_height"])
            bbox = O.affine_points(d[i, :, :4].reshape(-1, 2), m["c"][i], m["s"][i], size).reshape(-1, 4)
            pts = O.affine_points(d[i, :, 5:39].reshape(-1, 2), m["c"][i], m["s"][i], size).reshape(-1, 34)
            r = np.concatenate([bbox, d[i, :, 4:5], pts], axis=1).astype(np.float32)
            r[:, :4] /= np.float32(m["scale"])
            r[:, 5:] /= np.float32(m["scale"])
            per_scale.append({1: r})
        out.append(O.multi_pose_merge_outputs(per_scale, nms or len(dets) > 1)[1])
    return np.stack(out, 0)


def oracle_exdet(dets, metas, nc, mpi, flip):
    """ExdetDetector.post_process of every image and scale + merge_outputs -> list of {class id: [n, 5]}."""
    p = 2 if flip else 1
    res = []
    for i in range(dets[0].shape[0] // p):
        per_scale = [O.exdet_post_process(d[p * i:p * i + p], _image_meta(m, i), m["scale"]) for d, m in zip(dets, metas)]
        res.append(O.exdet_merge_outputs(per_scale, nc, mpi))
    return res

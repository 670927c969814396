"""Mirror of src/lib/utils/post_process.py (ctdet_post_process, multi_pose_post_process), of
src/lib/external/nms.pyx (soft_nms, soft_nms_39) and of CtdetDetector.merge_outputs
(detectors/ctdet.py:76-92), computed on the device (SURVEY 8f N2).

Two ways in:
  * the drop-in functions keep the reference's signatures and return types (numpy in, python lists /
    in-place arrays out) so `detectors/*.py` work unchanged -- but they also accept the CUDA tensor that
    `ctdet_decode` returned, which removes the `dets.detach().cpu().numpy()` of detectors/ctdet.py:48;
  * `ctdet_merge_device` is the whole tail of a detector run (back-projection of every scale, per-class
    concat, soft-NMS, top max_per_image) in four launches with ONE device->host copy at the end;
    `multi_pose_merge_device` and `exdet_merge_device` are the same for MultiPoseDetector and ExdetDetector.
"""
import numpy as np
import torch

from ._lib import C, ptr, same_device, stream_ptr

# Longest soft-NMS list and most detections per image of a merge (k_soft_nms holds a list in shared memory,
# k_topk_keep sorts an image's scores there; csrc/post.cu).
MAX_ROWS = 4096


# ------------------------------------------------------------------ utils/image.py:27-60 (host, float64, B matrices)
def _affine_points(center, scale, output_size):
    """The three float32 point pairs (src in the image, dst on the output grid) of get_affine_transform(center,
    scale, 0, output_size)."""
    f32 = np.float32
    if not isinstance(scale, (np.ndarray, list, tuple)):
        scale = np.array([scale, scale], dtype=f32)
    scale = np.asarray(scale, dtype=f32).reshape(-1)
    center = np.asarray(center, dtype=f32).reshape(2)
    src_w = scale[0]
    dst_w, dst_h = output_size
    src = np.zeros((3, 2), f32); dst = np.zeros((3, 2), f32)
    src[0] = center
    src[1] = center + np.array([0.0, src_w * f32(-0.5)], f32)
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5], f32) + np.array([0, dst_w * -0.5], f32)
    for p in (src, dst):
        d = p[0] - p[1]
        p[2] = p[1] + np.array([-d[1], d[0]], f32)
    return src, dst


def _inv_affine(center, scale, output_size):
    """2x3 float64 matrix of get_affine_transform(center, scale, 0, output_size, inv=1): output-grid -> image.
    rot = 0, so the three point pairs of the reference define a uniform scale + translation; it is solved
    from the same float32 points in float64 (cv2.getAffineTransform there)."""
    src, dst = _affine_points(center, scale, output_size)
    a = np.concatenate([dst.astype(np.float64), np.ones((3, 1))], axis=1)
    return np.linalg.solve(a, src.astype(np.float64)).T


def cv_affine_transform(src, dst):
    """cv2.getAffineTransform(src, dst) to the bit, without OpenCV: the 6x6 system of imgwarp.cpp (rows
    [x, y, 1, 0, 0, 0] / [0, 0, 0, x, y, 1] per point, right-hand side the dst coordinates) solved as cv::solve's
    DECOMP_LU solves it (hal LUImpl: partial pivoting on the largest |a|, elimination by multiples of -1 / pivot,
    back substitution dividing by the pivot), every step a rounded float64 operation.  Returns 2x3 float64."""
    src = np.asarray(src, np.float32).reshape(3, 2).astype(np.float64).tolist()
    dst = np.asarray(dst, np.float32).reshape(3, 2).astype(np.float64).tolist()
    a, b = [], []
    for (x, y), (u, v) in zip(src, dst):
        a += [[x, y, 1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, x, y, 1.0]]
        b += [u, v]
    m = 6
    for i in range(m):
        k = i
        for j in range(i + 1, m):
            if abs(a[j][i]) > abs(a[k][i]):
                k = j
        if a[k][i] == 0.0:
            raise ValueError("cv_affine_transform: the three points are collinear")
        if k != i:
            a[i], a[k] = a[k], a[i]
            b[i], b[k] = b[k], b[i]
        d = -1.0 / a[i][i]
        for j in range(i + 1, m):
            alpha = a[j][i] * d
            for c in range(i + 1, m):
                a[j][c] += alpha * a[i][c]
            b[j] += alpha * b[i]
    for i in range(m - 1, -1, -1):
        s = b[i]
        for c in range(i + 1, m):
            s -= a[i][c] * b[c]
        b[i] = s / a[i][i]
    return np.array(b, np.float64).reshape(2, 3)


def cv_inv_affine(center, scale, output_size):
    """get_affine_transform(center, scale, 0, output_size, inv=1) as the reference computes it (cv2 included), for
    the ddd tail: at the KITTI metas (int32 image-size scales) the float64 solve of _inv_affine misses cv2 by one
    ulp in some entries, which moves a back-projected coordinate by one float32 ulp now and then."""
    src, dst = _affine_points(center, scale, output_size)
    return cv_affine_transform(dst, src)


def _trans_tensor(c, s, w, h, device):
    mats = np.stack([_inv_affine(c[i], s[i], (w, h)) for i in range(len(c))], 0).reshape(len(c), 6)
    return torch.from_numpy(np.ascontiguousarray(mats)).to(device)


def _as_cuda(dets):
    if isinstance(dets, torch.Tensor):
        if not dets.is_cuda:
            raise NotImplementedError("post_process: CUDA tensors or numpy arrays only (no CPU path)")
        return dets.detach().float().contiguous()
    return torch.from_numpy(np.ascontiguousarray(dets, dtype=np.float32)).cuda()


def transform_dets(dets, c, s, h, w, pairs):
    """Back-projects the (x, y) column pairs `pairs` = ((col0, n), (col0, n)) of dets [B, N, D]; returns a new
    CUDA tensor (the decode output is left untouched)."""
    d = _as_cuda(dets)
    b, n, dim = [int(v) for v in d.shape]
    out = torch.empty_like(d)
    t = _trans_tensor(c, s, w, h, d.device)
    (a0, na), (b0, nb) = pairs
    C.post_transform(ptr(d), ptr(out), ptr(t), b, n, dim, a0, na, b0, nb, stream_ptr(d))
    return out


# ------------------------------------------------------------------ utils/post_process.py:83-99
def ctdet_post_process(dets, c, s, h, w, num_classes):
    """dets: [B, K, 6] numpy array or CUDA tensor -> list (per image) of {1-based class id: [[x1,y1,x2,y2,score]]}
    exactly as the reference (python lists of float32 rows)."""
    out = transform_dets(dets, c, s, h, w, ((0, 2), (0, 0)))
    b, n, _ = [int(v) for v in out.shape]
    rows = torch.empty((b, n, 5), dtype=torch.float32, device=out.device)
    offs = torch.empty((b, num_classes + 1), dtype=torch.int32, device=out.device)
    C.group_by_class(ptr(out), b, n, num_classes, ptr(rows), ptr(offs), stream_ptr(out))
    rows_h, offs_h = rows.cpu().numpy(), offs.cpu().numpy()
    ret = []
    for i in range(b):
        ret.append({j + 1: rows_h[i, offs_h[i, j]:offs_h[i, j + 1]].tolist() for j in range(num_classes)})
    return ret


# ------------------------------------------------------------------ utils/post_process.py:102-114
def multi_pose_post_process(dets, c, s, h, w):
    """dets: [B, K, 40] -> list of {1: [[bbox(4), score, 17 x (x, y)] ...]} in image coordinates."""
    out = transform_dets(dets, c, s, h, w, ((0, 2), (5, 17)))
    host = out[:, :, :39].cpu().numpy()
    return [{np.ones(1, dtype=np.int32)[0]: host[i].tolist()} for i in range(host.shape[0])]


# ------------------------------------------------------------------ external/nms.pyx:77-275
def _soft_nms(boxes, sigma, Nt, threshold, method, d):
    if not (isinstance(boxes, np.ndarray) and boxes.dtype == np.float32 and boxes.ndim == 2 and boxes.shape[1] >= d):
        raise TypeError("soft_nms: boxes must be a float32 [N, >=%d] numpy array (modified in place)" % d)
    n = int(boxes.shape[0])
    if n == 0:
        return []
    if n > MAX_ROWS:
        raise NotImplementedError("soft_nms: lists longer than %d boxes are not implemented" % MAX_ROWS)
    dev = torch.device("cuda", torch.cuda.current_device())
    src = torch.from_numpy(np.ascontiguousarray(boxes[:, :d])).to(dev)
    dst = torch.empty_like(src)
    offs = torch.tensor([0, n], dtype=torch.int32, device=dev)
    fin = torch.empty(1, dtype=torch.int32, device=dev)
    C.soft_nms(ptr(src), ptr(dst), ptr(offs), 1, 1, n, d, float(sigma), float(Nt), float(threshold), int(method),
               ptr(fin), stream_ptr(src))
    keep = int(fin.item())
    if keep < 0:
        raise RuntimeError("soft_nms: the list of %d boxes was not processed" % n)
    boxes[:, :d] = dst.cpu().numpy()
    return list(range(keep))


def soft_nms(boxes, sigma=0.5, Nt=0.3, threshold=0.001, method=0):
    """Drop-in for external.nms.soft_nms: `boxes` [N, 5] float32 is modified IN PLACE exactly as the reference
    leaves it (rows beyond the returned length included); returns the keep list."""
    return _soft_nms(boxes, sigma, Nt, threshold, method, 5)


def soft_nms_39(boxes, sigma=0.5, Nt=0.3, threshold=0.001, method=0):
    """Drop-in for external.nms.soft_nms_39 ([N, 39]: box, score, 17 keypoints)."""
    return _soft_nms(boxes, sigma, Nt, threshold, method, 39)


# ------------------------------------------------------------------ detectors/ctdet.py:47-92, on the device
def ctdet_merge_device(dets_per_scale, metas, num_classes, max_per_image=100, nms=False):
    """The tail of CtdetDetector.run for one image batch: for every test scale `ctdet_post_process` (+ the
    division by the scale, detectors/ctdet.py:47-58), then `merge_outputs` (:76-92): per-class concatenation
    over the scales, soft-NMS (Nt 0.5, Gaussian) when there are several scales or `nms` is set, and the cut to
    the max_per_image best scores.
      dets_per_scale: list of [B, K, 6] CUDA tensors (ctdet_decode outputs), one per test scale;
      metas: one dict per scale with the keys of base_detector.pre_process's `meta` (:58-62): 'c' and 's' as
             per-image sequences, 'out_height', 'out_width', plus 'scale' (the test scale, default 1).
    Returns a list (per image) of {class id: float32 [n, 5] array} -- one device->host copy in total."""
    S = len(dets_per_scale)
    assert len(metas) == S
    parts = []
    for k in range(S):
        m = metas[k]
        t = transform_dets(dets_per_scale[k], m["c"], m["s"], m["out_height"], m["out_width"], ((0, 2), (0, 0)))
        sc = float(m.get("scale", 1.0))
        if sc != 1.0:   # a tensor divisor: torch turns division by a Python scalar into a multiplication by 1/scale
            t[:, :, :4] /= torch.tensor(sc, dtype=torch.float32, device=t.device)
        parts.append(t)
    allp = torch.cat(parts, dim=1).contiguous()          # scale-major, like np.concatenate over `detections`
    b, n, _ = [int(v) for v in allp.shape]
    if n > MAX_ROWS:
        raise NotImplementedError("ctdet_merge_device: at most %d detections per image" % MAX_ROWS)
    rows = torch.empty((b, n, 5), dtype=torch.float32, device=allp.device)
    offs = torch.empty((b, num_classes + 1), dtype=torch.int32, device=allp.device)
    C.group_by_class(ptr(allp), b, n, num_classes, ptr(rows), ptr(offs), stream_ptr(allp))
    fin = None
    if S > 1 or nms:
        fin = torch.empty((b, num_classes), dtype=torch.int32, device=allp.device)
        C.soft_nms(ptr(rows), ptr(rows), ptr(offs), b, num_classes, n, 5, 0.5, 0.5, 0.001, 2, ptr(fin), stream_ptr(rows))
    keep = torch.empty((b, n), dtype=torch.uint8, device=allp.device)
    C.topk_keep(ptr(rows), b, n, 5, ptr(offs), num_classes, int(max_per_image), ptr(keep), 0, stream_ptr(rows))
    cols = [rows.view(b, -1), keep.float(), offs.float()]
    if fin is not None:
        cols.append(fin.float())        # list lengths after soft-NMS (<= 4096: exact in float32)
    packed = torch.cat(cols, dim=1).cpu().numpy()   # one D2H
    rows_h = packed[:, :n * 5].reshape(b, n, 5)
    keep_h = packed[:, n * 5:n * 6] > 0
    offs_h = packed[:, n * 6:n * 6 + num_classes + 1].astype(np.int64)
    if fin is not None and (packed[:, n * 6 + num_classes + 1:] < 0).any():
        raise RuntimeError("ctdet_merge_device: soft-NMS left a class list unprocessed")
    ret = []
    for i in range(b):
        res = {}
        for j in range(num_classes):
            a, e = offs_h[i, j], offs_h[i, j + 1]
            res[j + 1] = rows_h[i, a:e][keep_h[i, a:e]].astype(np.float32)
        ret.append(res)
    return ret


# ------------------------------------------------------------------ detectors/multi_pose.py and exdet.py tails
# Most rows per image of the exdet merge (k_soft_nms_strided and k_topk_keep_wide, csrc/post.cu).
MAX_IMAGE_ROWS = 32768


def _check_tail_inputs(what, dets_per_scale, metas, width):
    """Shapes, devices and metas of a device tail, checked before anything is launched.  Returns B (rows of the
    first dimension) and the device."""
    if len(dets_per_scale) == 0 or len(metas) != len(dets_per_scale):
        raise ValueError("%s: one meta per scale and at least one scale (got %d detections, %d metas)"
                         % (what, len(dets_per_scale), len(metas)))
    for d in dets_per_scale:
        if not isinstance(d, torch.Tensor) or not d.is_cuda:
            raise NotImplementedError("%s: CUDA tensors only (no CPU path)" % what)
    dev = same_device(*dets_per_scale)
    b = int(dets_per_scale[0].shape[0]) if dets_per_scale[0].dim() == 3 else -1
    for d in dets_per_scale:
        if d.dim() != 3 or int(d.shape[2]) != width or int(d.shape[0]) != b or int(d.shape[1]) < 1 or b < 1:
            raise ValueError("%s: every scale must be [B, N, %d] with one B, got %s"
                             % (what, width, [tuple(t.shape) for t in dets_per_scale]))
    return b, dev


def _tail_transforms(what, metas, n_img, device):
    """[S, n_img, 6] float64 inverse affines of every scale and image, in ONE copy from pinned memory (no host
    synchronisation)."""
    mats = []
    for m in metas:
        if len(m["c"]) != n_img or len(m["s"]) != n_img:
            raise ValueError("%s: metas need one 'c' and one 's' per image (%d)" % (what, n_img))
        mats.append([_inv_affine(m["c"][i], m["s"][i], (m["out_width"], m["out_height"])).reshape(6)
                     for i in range(n_img)])
    host = torch.from_numpy(np.ascontiguousarray(np.array(mats, np.float64))).pin_memory()
    return host.to(device, non_blocking=True)


def _divide_by_scale(t, cols, scale):
    """`dets[..., cols] /= scale` in float32, as numpy divides a float32 array by a Python float (a tensor
    divisor: torch turns division by a Python scalar into a multiplication by 1/scale)."""
    if scale != 1.0:
        div = torch.full((), scale, dtype=torch.float32, device=t.device)
        for a, e in cols:
            t[:, :, a:e] /= div


def multi_pose_merge_device(dets_per_scale, metas, nms=False):
    """The tail of MultiPoseDetector.run for one image batch: for every test scale `post_process`
    (detectors/multi_pose.py:62-73: multi_pose_post_process, then the box and the keypoints divided by the scale),
    then `merge_outputs` (:75-81): concatenation over the scales and, when `nms` is set or there are several
    scales, soft_nms_39 (Nt 0.5, Gaussian) on the whole list.  Every row is kept, as the reference keeps it.
      dets_per_scale: list of [B, K, 40] CUDA tensors (multi_pose_decode outputs), one per test scale;
      metas: one dict per scale, the keys of ctdet_merge_device ('c', 's' per image, 'out_height', 'out_width',
             'scale').
    Returns a list (per image) of {1: list of 39-float rows} -- one device->host copy in total.  The inputs are
    left unmodified."""
    what = "multi_pose_merge_device"
    b, dev = _check_tail_inputs(what, dets_per_scale, metas, 40)
    n = sum(int(d.shape[1]) for d in dets_per_scale)
    run_nms = bool(nms) or len(dets_per_scale) > 1
    if run_nms and n > MAX_ROWS:
        raise NotImplementedError("%s: soft-NMS takes at most %d rows per image (got %d)" % (what, MAX_ROWS, n))
    trans = _tail_transforms(what, metas, b, dev)
    parts = []
    for k, (d, m) in enumerate(zip(dets_per_scale, metas)):
        d = d.detach().float().contiguous()
        t = torch.empty_like(d)
        C.post_transform(ptr(d), ptr(t), ptr(trans[k]), b, int(d.shape[1]), 40, 0, 2, 5, 17, stream_ptr(d))
        t = t[:, :, :39]
        _divide_by_scale(t, ((0, 4), (5, 39)), float(m.get("scale", 1.0)))
        parts.append(t)
    allp = torch.cat(parts, dim=1).contiguous()          # scale-major, like np.concatenate over `detections`
    if run_nms:
        offs = torch.zeros((b, 2), dtype=torch.int32, device=dev)
        offs[:, 1] = n
        out = torch.empty_like(allp)
        C.soft_nms(ptr(allp), ptr(out), ptr(offs), b, 1, n, 39, 0.5, 0.5, 0.001, 2, 0, stream_ptr(allp))
        allp = out
    host = allp.cpu().numpy()                             # one D2H
    return [{1: host[i].tolist()} for i in range(b)]


def exdet_merge_device(dets_per_scale, metas, num_classes, max_per_image=100, flip=False):
    """The tail of ExdetDetector.run for one image batch: for every test scale `post_process`
    (detectors/exdet.py:85-95), then `merge_outputs` (:97-122) with the reference's compiled soft_nms.
      dets_per_scale: list of [P*B, N, 14] CUDA tensors (exct_decode / agnex_ct_decode outputs), one per test
             scale.  With `flip` P = 2 and image i is the pair of rows (2i, 2i+1) that base_detector.pre_process
             builds: the image, then its mirror;
      metas: one dict per scale, the keys of ctdet_merge_device.
    Per scale an image's P*N rows are split into two equal halves (as `reshape(2, -1, 14)` splits them), the
    second half is un-mirrored, both corners are back-projected and divided by the scale.  The merge keeps the
    rows with score > 0, groups them by the class in column 13, runs Gaussian soft-NMS (Nt 0.5) on every class
    list and cuts to the max_per_image best scores.  Like the reference, an image without `flip` has its N rows
    split in two and the second half mirrored, so N must be even.
    Returns a list (per image) of {class id: float32 [n, 5] array}, every row soft-NMS leaves included -- one
    device->host copy in total.  The inputs are left unmodified."""
    what = "exdet_merge_device"
    pb, dev = _check_tail_inputs(what, dets_per_scale, metas, 14)
    p = 2 if flip else 1
    if pb % p:
        raise ValueError("%s: with flip the batch holds image / mirror pairs (got %d rows)" % (what, pb))
    b = pb // p
    per_img = [p * int(d.shape[1]) for d in dets_per_scale]
    if any(r % 2 for r in per_img):
        raise ValueError("%s: an image's rows are split into two equal halves (detectors/exdet.py:87), so N must "
                         "be even without flip (got %s)" % (what, [int(d.shape[1]) for d in dets_per_scale]))
    n = sum(per_img)
    if n > MAX_IMAGE_ROWS:
        raise NotImplementedError("%s: at most %d rows per image (got %d)" % (what, MAX_IMAGE_ROWS, n))
    if not 0 < int(num_classes) <= 8192 or int(max_per_image) < 1:
        raise ValueError("%s: num_classes must be in [1, 8192] and max_per_image >= 1" % what)
    num_classes, max_per_image = int(num_classes), int(max_per_image)
    trans = _tail_transforms(what, metas, b, dev)
    parts = []
    for k, (d, m) in enumerate(zip(dets_per_scale, metas)):
        d = d.detach().float().contiguous()
        t = torch.empty((b, per_img[k], 14), dtype=torch.float32, device=dev)
        C.exdet_transform(ptr(d), ptr(t), ptr(trans[k]), b, per_img[k], 14, float(m["out_width"]), stream_ptr(d))
        _divide_by_scale(t, ((0, 4),), float(m.get("scale", 1.0)))
        parts.append(t)
    allp = torch.cat(parts, dim=1).contiguous() if len(parts) > 1 else parts[0]
    rows = torch.empty((b, n, 5), dtype=torch.float32, device=dev)
    offs = torch.empty((b, num_classes + 1), dtype=torch.int32, device=dev)
    C.group_positive_by_class(ptr(allp), b, n, 14, 13, num_classes, ptr(rows), ptr(offs), stream_ptr(allp))
    fin = torch.empty((b, num_classes), dtype=torch.int32, device=dev)
    C.soft_nms_strided(ptr(rows), ptr(rows), ptr(offs), b, num_classes, n, min(n, MAX_ROWS), 5, 0.5, 0.5, 0.001, 2,
                       ptr(fin), stream_ptr(rows))
    keep = torch.empty((b, n), dtype=torch.uint8, device=dev)
    C.topk_keep_wide(ptr(rows), b, n, 5, ptr(offs), num_classes, max_per_image, ptr(keep), 0, stream_ptr(rows))
    packed = torch.cat([rows.view(b, -1), keep.float(), offs.float(), fin.float()], dim=1).cpu().numpy()   # one D2H
    rows_h = packed[:, :n * 5].reshape(b, n, 5)
    keep_h = packed[:, n * 5:n * 6] > 0
    offs_h = packed[:, n * 6:n * 6 + num_classes + 1].astype(np.int64)      # <= 32768: exact in float32
    fin_h = packed[:, n * 6 + num_classes + 1:]
    if (fin_h < 0).any():
        raise RuntimeError("%s: a class list of more than %d rows was not processed by soft-NMS" % (what, MAX_ROWS))
    ret = []
    for i in range(b):
        res = {}
        for j in range(num_classes):
            a, e = offs_h[i, j], offs_h[i, j + 1]
            res[j + 1] = rows_h[i, a:e][keep_h[i, a:e]].astype(np.float32)
        ret.append(res)
    return ret


# ------------------------------------------------------------------ utils/post_process.py:13-80, detectors/ddd.py:75-88
DDD_COLS = 13        # alpha, x1, y1, x2, y2, dim[3], X, Y, Z, rot_y, score


def _ddd_tail(what, dets, c, s, calibs, out_w, out_h, num_classes, thresh):
    """cnb_ddd_tail on dets [B, N, 18] (numpy or CUDA), one inverse affine and one calibration per image, and ONE
    device->host copy.  thresh None: every row (ddd_post_process); else merge_outputs' score > float32(thresh).
    Returns a list (per image) of {class id: float32 [n, 13]}, a class without rows being np.array([], float32) as
    the reference builds it, and with a cut a class the cut emptied [0, 13]."""
    if isinstance(dets, torch.Tensor) and not dets.is_cuda:
        raise NotImplementedError("%s: CUDA tensors or numpy arrays only (no CPU path)" % what)
    shape = tuple(dets.shape)
    if len(shape) == 3 and shape[2] == 16:
        raise ValueError("%s: dets has 16 columns (ddd_decode without wh, --not_reg_bbox); the reference's "
                         "ddd_post_process_3d reads the box size from columns 8:10 of every row and raises IndexError "
                         "without it" % what)
    if len(shape) != 3 or shape[2] != 18 or shape[0] < 1 or shape[1] < 1:
        raise ValueError("%s: dets must be [B, N, 18] (ddd_decode with wh), got %s" % (what, shape))
    num_classes = int(num_classes)
    if not 0 < num_classes <= 8192:
        raise ValueError("%s: num_classes must be in [1, 8192]" % what)
    b, n = shape[0], shape[1]
    if n >= 1 << 24:
        raise NotImplementedError("%s: at most %d rows per image" % (what, (1 << 24) - 1))
    if len(c) != b or len(s) != b or len(calibs) != b:
        raise ValueError("%s: one 'c', 's' and calib per image (%d)" % (what, b))
    d = _as_cuda(dets)
    dev = d.device
    mats = np.stack([cv_inv_affine(c[i], s[i], (out_w, out_h)).reshape(6) for i in range(b)], 0)
    cal = np.stack([np.asarray(k, np.float32).reshape(12) for k in calibs], 0)
    # the matrices and the calibrations in ONE copy from pinned memory (no host synchronisation)
    host = np.concatenate([mats.astype(np.float64).view(np.uint8).reshape(-1), cal.view(np.uint8).reshape(-1)])
    params = torch.from_numpy(host).pin_memory().to(dev, non_blocking=True)
    trans, calib = params[:b * 48].view(torch.float64), params[b * 48:].view(torch.float32)
    rows = torch.empty((b, n * DDD_COLS), dtype=torch.float32, device=dev)
    offs = torch.empty((b, num_classes + 1), dtype=torch.int32, device=dev)
    seen = torch.empty((b, num_classes), dtype=torch.uint8, device=dev)
    C.ddd_tail(ptr(d), b, n, 18, ptr(trans), ptr(calib), num_classes, int(thresh is not None),
               float(np.float32(0.0 if thresh is None else thresh)), ptr(rows), ptr(offs), ptr(seen), stream_ptr(d))
    packed = torch.cat([rows, offs.float(), seen.float()], dim=1).cpu().numpy()   # one D2H
    rows_h = packed[:, :n * DDD_COLS].reshape(b, n, DDD_COLS)
    offs_h = packed[:, n * DDD_COLS:n * DDD_COLS + num_classes + 1].astype(np.int64)     # < 2^24: exact in float32
    seen_h = packed[:, n * DDD_COLS + num_classes + 1:] > 0
    ret = []
    for i in range(b):
        res = {}
        for j in range(num_classes):
            a, e = offs_h[i, j], offs_h[i, j + 1]
            res[j + 1] = rows_h[i, a:e].copy() if seen_h[i, j] else np.array([], np.float32)
        ret.append(res)
    return ret


def ddd_post_process(dets, c, s, calibs, opt):
    """Drop-in for utils/post_process.py:75-80 (ddd_post_process_2d then _3d) on the device.
      dets: [B, K, 18] ddd_decode output, numpy array or CUDA tensor (left unmodified; the reference writes the
            back-projected centres into it);
      c, s: per-image centres and scales; calibs: per-image 3x4 calibrations, of which -- as the reference does --
            calibs[0] is used for EVERY image (taken as float32, the dtype DddDetector and the dataset give it);
      opt: reads output_w, output_h and num_classes.
    Returns a list (per image) of {class id: float32 [n, 13] array of alpha, x1, y1, x2, y2, dim[3], X, Y, Z, rot_y,
    score}, a class without rows being np.array([], float32) of shape (0,).  Every value that does not go through an
    arctan2 equals the reference's bit for bit; alpha and rot_y are the float32 closest to the angle, numpy's float32
    arctan2 is within a few ulp of it.  16-column dets (no wh) raise ValueError: the reference cannot process them."""
    b = int(dets.shape[0])
    return _ddd_tail("ddd_post_process", dets, c, s, [calibs[0]] * b, int(opt.output_w), int(opt.output_h),
                     int(opt.num_classes), None)


def ddd_merge_device(dets, meta, num_classes, peak_thresh=0.2):
    """The tail of DddDetector.run for one image batch: `post_process` (detectors/ddd.py:75-80) of every image with
    its OWN calibration, then `merge_outputs` (:82-88), the cut to score > float32(peak_thresh) (NaN dropped, +inf
    kept).  Equals running the reference detector once per image.
      dets: [B, K, 18] CUDA tensor (or numpy array) from ddd_decode / ddd_decode_from_logits; one tensor, not a
            list of scales: DddDetector.pre_process ignores the test scale and merge_outputs reads detections[0] only;
      meta: 'c', 's' and 'calib' ([3, 4] float32) as per-image sequences, 'out_height', 'out_width' (ddd_pre_process
            returns them for one image).
    Returns a list (per image) of {class id: float32 [n, 13]}: a class without rows is np.array([], float32) of shape
    (0,), a class the cut emptied has shape (0, 13), as merge_outputs leaves them -- one device->host copy."""
    return _ddd_tail("ddd_merge_device", dets, meta["c"], meta["s"], meta["calib"], int(meta["out_width"]),
                     int(meta["out_height"]), num_classes, float(peak_thresh))

"""Mirror of BaseDetector.pre_process (src/lib/detectors/base_detector.py:37-65) on the device (SURVEY 8f N4):
the uint8 image crosses PCIe once (3 B/pixel instead of the 12-24 B/pixel of the normalised fp32 CHW batch the
reference uploads), and the affine warp, the normalisation, the layout change and the flip-test copy are one
kernel.  At test scales != 1 the reference first runs cv2.resize (INTER_LINEAR); its fixed-point filter is a second
small kernel (`cnb_resize_image`).  Bit-identical to the reference at every scale (tests/test_pre.py)."""
import numpy as np
import torch

from ._lib import C, ptr, stream_ptr
from .post_process import _affine_points, cv_affine_transform


def _forward_affine(center, scale, output_size):
    """get_affine_transform(c, s, 0, output_size) (utils/image.py:27-60, rot = 0, inv = 0) as a 2x3 float64."""
    f32 = np.float32
    if not isinstance(scale, (np.ndarray, list, tuple)):
        scale = np.array([scale, scale], dtype=f32)
    scale = np.asarray(scale, dtype=f32).reshape(-1)
    center = np.asarray(center, dtype=f32).reshape(2)
    dst_w, dst_h = output_size
    src = np.zeros((3, 2), f32); dst = np.zeros((3, 2), f32)
    src[0] = center
    src[1] = center + np.array([0.0, scale[0] * f32(-0.5)], f32)
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5], f32) + np.array([0, dst_w * -0.5], f32)
    for p in (src, dst):
        d = p[0] - p[1]
        p[2] = p[1] + np.array([-d[1], d[0]], f32)
    try:                                   # the reference's own solver when OpenCV is installed
        import cv2
        return np.asarray(cv2.getAffineTransform(np.float32(src), np.float32(dst)), np.float64)
    except ImportError:
        a = np.concatenate([src.astype(np.float64), np.ones((3, 1))], axis=1)
        return np.linalg.solve(a, dst.astype(np.float64)).T


def _invert(m):
    """What cv::warpAffine does to its forward matrix before sampling (imgwarp.cpp)."""
    m = [float(v) for v in np.asarray(m, np.float64).reshape(6)]
    d = m[0] * m[4] - m[1] * m[3]
    d = 1.0 / d if d != 0 else 0.0
    a11, a22 = m[4] * d, m[0] * d
    m[0] = a11; m[1] *= -d; m[3] *= -d; m[4] = a22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2] = b1; m[5] = b2
    return m


def pre_process(image, scale, mean, std, fix_res=True, input_h=512, input_w=512, pad=31, down_ratio=4,
                flip_test=False, device=None):
    """image: uint8 [H, W, 3] numpy array (BGR, as cv2.imread) or CUDA uint8 tensor.  Returns (images, meta) like
    the reference: images fp32 CUDA tensor [1 or 2, 3, inp_h, inp_w]; meta = {'c', 's', 'out_height', 'out_width'}."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if isinstance(image, torch.Tensor):
        if not image.is_cuda or image.dtype != torch.uint8:
            raise NotImplementedError("pre_process: uint8 CUDA tensor or numpy array")
        img = image.contiguous()
        dev = img.device
    else:
        img = torch.from_numpy(np.ascontiguousarray(image, dtype=np.uint8)).to(dev, non_blocking=True)
    height, width = int(img.shape[0]), int(img.shape[1])
    new_height, new_width = int(height * scale), int(width * scale)
    if (new_height, new_width) != (height, width):         # cv2.resize(image, (new_width, new_height)), :55
        resized = torch.empty((new_height, new_width, 3), dtype=torch.uint8, device=dev)
        C.resize_image(ptr(img), height, width, ptr(resized), new_height, new_width, stream_ptr(resized))
        img = resized
    if fix_res:
        inp_height, inp_width = input_h, input_w
        c = np.array([new_width / 2., new_height / 2.], dtype=np.float32)
        s = max(height, width) * 1.0
    else:
        inp_height = (new_height | pad) + 1
        inp_width = (new_width | pad) + 1
        c = np.array([new_width // 2, new_height // 2], dtype=np.float32)
        s = np.array([inp_width, inp_height], dtype=np.float32)
    minv = torch.tensor(_invert(_forward_affine(c, s, [inp_width, inp_height])), dtype=torch.float64, device=dev)
    mean_t = torch.tensor(np.asarray(mean, np.float32).reshape(3), device=dev)
    std_t = torch.tensor(np.asarray(std, np.float32).reshape(3), device=dev)
    out = torch.empty((2 if flip_test else 1, 3, inp_height, inp_width), dtype=torch.float32, device=dev)
    C.preprocess_image(ptr(img), new_height, new_width, ptr(minv), ptr(mean_t), ptr(std_t), ptr(out), inp_height, inp_width,
                       int(bool(flip_test)), stream_ptr(out))
    meta = {'c': c, 's': s, 'out_height': inp_height // down_ratio, 'out_width': inp_width // down_ratio}
    return out, meta


# DddDetector.__init__'s calibration (detectors/ddd.py:25-27), the default of ddd_pre_process.
KITTI_CALIB = np.array([[707.0493, 0, 604.0814, 45.75831],
                        [0, 707.0493, 180.5066, -0.3454157],
                        [0, 0, 1., 0.004981016]], dtype=np.float32)


def ddd_pre_process(image, input_h, input_w, mean, std, keep_res=False, calib=None, down_ratio=4, device=None):
    """DddDetector.pre_process (detectors/ddd.py:30-55) on the device, bit-identical to the reference: no resize (the
    detector ignores the test scale), c = (w / 2, h / 2), s = int32 [input_w, input_h] with keep_res else int32
    [w, h], the same warp as pre_process, and the detector's float32 normalisation (x / 255 then (x - mean) / std in
    float32, where BaseDetector normalises in float64).
      image: uint8 [H, W, 3] numpy array (BGR) or CUDA uint8 tensor; mean, std: 3 values each;
      calib: the image's 3x4 projection matrix (float32), default the detector's KITTI matrix.
    Returns (images [1, 3, input_h, input_w] fp32 CUDA tensor, meta {'c', 's', 'out_height', 'out_width', 'calib'});
    the uint8 image and the warp parameters are the only host->device copies."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if isinstance(image, torch.Tensor):
        if not image.is_cuda or image.dtype != torch.uint8:
            raise NotImplementedError("ddd_pre_process: uint8 CUDA tensor or numpy array")
        img = image.contiguous()
        dev = img.device
    else:
        img = torch.from_numpy(np.ascontiguousarray(image, dtype=np.uint8)).to(dev, non_blocking=True)
    if img.dim() != 3 or int(img.shape[2]) != 3:
        raise ValueError("ddd_pre_process: image must be [H, W, 3], got %s" % (tuple(img.shape),))
    height, width = int(img.shape[0]), int(img.shape[1])
    c = np.array([width / 2, height / 2], dtype=np.float32)
    s = np.array([input_w, input_h] if keep_res else [width, height], dtype=np.int32)
    # cv2.getAffineTransform's own matrix, OpenCV or not (the float64 solve misses it by one ulp at KITTI sizes)
    minv = np.array(_invert(cv_affine_transform(*_affine_points(c, s, [input_w, input_h]))), np.float64)
    norm = np.concatenate([np.asarray(mean, np.float32).reshape(3), np.asarray(std, np.float32).reshape(3)])
    params = torch.from_numpy(np.concatenate([minv.view(np.uint8), norm.view(np.uint8)])).to(dev, non_blocking=True)
    out = torch.empty((1, 3, input_h, input_w), dtype=torch.float32, device=dev)
    C.preprocess_image_f32(ptr(img), height, width, ptr(params[:48]), ptr(params[48:60]), ptr(params[60:72]),
                           ptr(out), input_h, input_w, 0, stream_ptr(out))
    calib = np.array(calib, dtype=np.float32) if calib is not None else KITTI_CALIB.copy()
    meta = {'c': c, 's': s, 'out_height': input_h // down_ratio, 'out_width': input_w // down_ratio, 'calib': calib}
    return out, meta

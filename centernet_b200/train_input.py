"""Training input of the ctdet sampler on the device (datasets/sample/ctdet.py:29-145 and color_aug,
utils/image.py:198-230).

The reference's loader warps, colour-augments, normalises and transposes every image on the host CPU, paints an
80 x 128 x 128 heat map in Python and copies the float batch across PCIe.  Here the host keeps what it must do --
cv2.imread, the COCO annotations and the random draws, from the same generators in the same order -- and the
device does the per-pixel arithmetic and the target geometry:

    loader = DataLoader(CTDetTrainInput(dataset), batch_size=..., collate_fn=collate_ctdet, pin_memory=True, ...)
    for packed in loader:
        batch = build_ctdet_batch(packed)      # one H2D copy of the uint8 images + parameters, 2-3 launches

`batch` holds what the reference's collated batch holds, on the device and bit for bit for the same RNG states
('input', 'reg_mask', 'ind', 'wh' or 'cat_spec_wh' / 'cat_spec_mask', 'reg' with opt.reg_offset; 'hm' with
dense_hm=True), plus the object lists FocalSplatLoss takes ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius',
'obj_valid').  `augment_images` is the image half alone, for explicit matrices, flips and colour parameters.
The numeric contract is DESIGN.md section 4.9.

The multi_pose sampler (datasets/sample/multi_pose.py:29-183) works the same way: MultiPoseTrainInput,
collate_multi_pose and build_multi_pose_batch, with the rotated crop, the keypoint targets, hm / hm_hp and the
joint lists of FocalSplatLoss (DESIGN.md section 4.10).

The ddd sampler (datasets/sample/ddd.py:27-157) too: DddTrainInput, collate_ddd and build_ddd_batch, with the
KITTI ignore regions painted into a dense hm on the device (DESIGN.md section 4.11).

The exdet sampler (datasets/sample/exdet.py:30-137) too: ExdetTrainInput, collate_exdet and build_exdet_batch, with
the extreme-point and centre targets and the object lists of the five heat maps, which FocalSplatLoss reads without
the maps ever existing (DESIGN.md section 4.12)."""
import itertools
import math
import os
import random

import numpy as np
import torch

from ._lib import C, _DTYPE_CODES, ptr, stream_ptr, workspace
from .losses import splat_gaussian
from .post_process import _affine_points, cv_affine_transform
from .pre_process import _invert

F32 = np.float32

# color_aug's functions list [brightness_, contrast_, saturation_] as kinds 0, 1, 2; an order code is the index
# of the shuffled list among the six permutations in lexicographic order (include/centernet_b200.h).
ORDERS = tuple(itertools.permutations(range(3)))
# Largest source side: the warp clamps source coordinates to [-32768, 32767].
MAX_SIDE = 32767


def _get_border(border, size):
    """CTDetDataset._get_border (ctdet.py:22-26)."""
    i = 1
    while size - border // i <= border // i:
        i *= 2
    return border // i


def affine_transform(center, scale, output_size, rot=0):
    """get_affine_transform(center, scale, rot, output_size) (utils/image.py:27-60) as a 2x3 float64, to the bit.
    A scale that is not an array becomes a float32 pair as there; an array scale (keep_res with a random crop, or
    ddd's int32 / float64 pair) keeps its float64 half-width, which the reference adds to the centre in float64.
    get_dir turns (0, -src_w / 2) by np.pi * rot / 180 in float64 (np.sin / np.cos, as there) and src[1] is the
    float64 sum rounded to float32; rot = 0 gives the unrotated point exactly.  The centre enters that sum as given:
    ctdet's and multi_pose's float32 centre exactly, ddd's float64 centre without a float32 rounding first."""
    if not isinstance(scale, np.ndarray):
        scale = np.array([scale, scale], dtype=F32)
    src, dst = _affine_points(center, scale.astype(F32), output_size)
    rot_rad = np.pi * rot / 180
    sn, cs = np.sin(rot_rad), np.cos(rot_rad)
    half = np.float64(scale[0]) * -0.5                  # src_point = [0, src_w * -0.5]
    src[1, 0] = F32(np.float64(center[0]) + (0 * cs - half * sn))
    src[1, 1] = F32(np.float64(center[1]) + (0 * sn + half * cs))
    d = src[0] - src[1]
    src[2] = src[1] + np.array([-d[1], d[0]], F32)
    return cv_affine_transform(src, dst)


def crop_draws(height, width, c, s, opt):
    """The crop draws of the train split (ctdet.py:44-57, multi_pose.py:45-57): np.random.choice and two
    randint, or the three randn of not_rand_crop.  Updates the centre c in place (float32 for ctdet and multi_pose;
    exdet's float64 one takes the random crop only); returns the scale."""
    if not opt.not_rand_crop:
        s = s * np.random.choice(np.arange(0.6, 1.4, 0.1))
        w_border = _get_border(128, width)
        h_border = _get_border(128, height)
        c[0] = np.random.randint(low=w_border, high=width - w_border)
        c[1] = np.random.randint(low=h_border, high=height - h_border)
    else:
        sf, cf = opt.scale, opt.shift
        c[0] += s * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
        c[1] += s * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
        s = s * np.clip(np.random.randn() * sf + 1, 1 - sf, 1 + sf)
    return s


def scale_shift_draws(height, width, c, s, opt):
    """ddd's aug_ddd draws (ddd.py:47-51) and exdet's not_rand_crop draws (exdet.py:49-53): three randn in the order
    scale, x shift, y shift, the shifts scaled by the image's width and height (not by s, as crop_draws scales
    them).  Updates the float64 centre c in place; returns the scale."""
    sf, cf = opt.scale, opt.shift
    s = s * np.clip(np.random.randn() * sf + 1, 1 - sf, 1 + sf)
    c[0] += width * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
    c[1] += height * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
    return s


def color_draws(split, opt, data_rng, eig_val, eig_vec):
    """color_aug's draws (utils/image.py:221-230) in the train split without opt.no_color_aug: random.shuffle of its
    three functions, one data_rng.uniform per blend in the order they run, then the lighting normal.  Returns
    (order code, blend [6] float32 (alpha, 1 - alpha) of brightness, contrast, saturation, light [3] float64);
    otherwise draws nothing and returns (-1, zeros, zeros), no colour augmentation."""
    if split != 'train' or opt.no_color_aug:
        return -1, np.zeros(6, F32), np.zeros(3, np.float64)
    blend = np.zeros(6, F32)
    kinds = [0, 1, 2]
    random.shuffle(kinds)
    for k in kinds:
        alpha = 1. + data_rng.uniform(low=-0.4, high=0.4)
        blend[2 * k], blend[2 * k + 1] = F32(alpha), F32(1 - alpha)
    light = np.dot(eig_vec, eig_val * data_rng.normal(scale=0.1, size=(3,)))
    return ORDERS.index(tuple(kinds)), blend, np.asarray(light, np.float64)


def sample_params(height, width, opt, split, data_rng, eig_val, eig_vec):
    """The random draws of CTDetDataset.__getitem__ (ctdet.py:41-67) and color_aug for one height x width image,
    from np.random, random and data_rng in the reference's order, and the matrices they give.  After the call
    the three generators are where the reference leaves them."""
    c = np.array([width / 2., height / 2.], dtype=np.float32)
    if opt.keep_res:
        input_h = (height | opt.pad) + 1
        input_w = (width | opt.pad) + 1
        s = np.array([input_w, input_h], dtype=np.float32)
    else:
        s = max(height, width) * 1.0
        input_h, input_w = opt.input_h, opt.input_w
    flipped = False
    if split == 'train':
        s = crop_draws(height, width, c, s, opt)
        if np.random.random() < opt.flip:
            flipped = True
            c[0] = width - c[0] - 1
    order, blend, light = color_draws(split, opt, data_rng, eig_val, eig_vec)
    output_h, output_w = input_h // opt.down_ratio, input_w // opt.down_ratio
    return {'c': c, 's': s, 'flip': flipped, 'input_h': input_h, 'input_w': input_w,
            'output_h': output_h, 'output_w': output_w,
            'minv': np.array(_invert(affine_transform(c, s, [input_w, input_h])), np.float64),
            'trans_output': affine_transform(c, s, [output_w, output_h]).reshape(6),
            'order': order, 'blend': blend, 'light': light}


class _TrainInput(torch.utils.data.Dataset):
    """Wraps a reference dataset instance, duck-typed on opt, coco, images, img_dir, max_objs, mean, std and split
    plus what the sampler's own fields read.  __getitem__ reads the image and its first max_objs annotations (no
    random draws), then makes the sampler's draws as the reference does and returns them with the uint8 image and
    the sampler's annotation fields; it does no pixel work (the sampler's collate_* + build_*_batch do).  The
    constructor rejects opt.mse_loss and the opt flags in `unsupported`, whose targets are not implemented."""
    unsupported = ()

    def __init__(self, dataset):
        opt, name = dataset.opt, type(self).__name__
        if opt.mse_loss:
            raise NotImplementedError("%s: opt.mse_loss (draw_msra_gaussian targets) is not implemented" % name)
        for flag in self.unsupported:
            if getattr(opt, flag):
                raise NotImplementedError("%s: opt.%s targets are not implemented" % (name, flag))
        self.dataset = dataset

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, index):
        import cv2
        ds = self.dataset
        img_id = ds.images[index]
        file_name = ds.coco.loadImgs(ids=[img_id])[0]['file_name']
        anns = ds.coco.loadAnns(ids=ds.coco.getAnnIds(imgIds=[img_id]))[:ds.max_objs]
        img = cv2.imread(os.path.join(ds.img_dir, file_name))
        sample = self._params(ds, img.shape[0], img.shape[1])
        sample.update(self._fields(ds, anns), image=img, max_objs=ds.max_objs, mean=np.asarray(ds.mean, F32).reshape(3),
                      std=np.asarray(ds.std, F32).reshape(3), reg_offset=bool(ds.opt.reg_offset))
        return sample


def _boxes(anns):
    """_coco_box_to_bbox of each annotation's bbox: [n, 4] float32 corners."""
    boxes = np.zeros((len(anns), 4), F32)
    for k, a in enumerate(anns):
        b = a['bbox']
        boxes[k] = np.array([b[0], b[1], b[0] + b[2], b[1] + b[3]], dtype=np.float32)
    return boxes


class CTDetTrainInput(_TrainInput):
    """Wraps a reference CTDetDataset instance (also duck-typed on cat_ids, num_classes, _data_rng, _eig_val and
    _eig_vec): sample_params' draws, the float32 box corners and the class cat_ids[category_id]; the batch is
    collate_ctdet + build_ctdet_batch's.  opt.dense_wh is rejected."""
    unsupported = ('dense_wh',)

    def _params(self, ds, height, width):
        return sample_params(height, width, ds.opt, ds.split, ds._data_rng, ds._eig_val, ds._eig_vec)

    def _fields(self, ds, anns):
        return {'boxes': _boxes(anns), 'cls': np.array([int(ds.cat_ids[a['category_id']]) for a in anns], np.int32),
                'num_classes': ds.num_classes, 'cat_spec_wh': bool(ds.opt.cat_spec_wh)}


class _Packer(object):
    """Arrays laid end to end in one byte buffer, each at a 16-byte aligned offset."""

    def __init__(self):
        self.parts, self.layout, self.size = [], {}, 0

    def add(self, name, a):
        a = np.ascontiguousarray(a)
        self.layout[name] = (self.size, a.dtype.str, a.shape)
        self.parts.append((self.size, a.reshape(-1).view(np.uint8)))
        self.size += (a.nbytes + 15) // 16 * 16

    def tensor(self, pin):
        buf = torch.empty(max(self.size, 16), dtype=torch.uint8, pin_memory=pin)
        host = buf.numpy()
        for off, a in self.parts:
            host[off:off + a.size] = a
        return buf

    def collated(self, scalars):
        """A collate_* result: the buffer (pinned in the main process), its layout and the scalars."""
        return {'buffer': self.tensor(_pin()), 'layout': self.layout, 'scalars': scalars}


def _pin():
    # pinned here when collating in the main process; a DataLoader worker leaves that to pin_memory=True
    return torch.utils.data.get_worker_info() is None and torch.cuda.is_available()


def _check_images(images):
    for img in images:
        if img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8:
            raise ValueError("train_input: images must be uint8 [H, W, 3], got %s %s" % (img.dtype, img.shape))
        if not (1 <= img.shape[0] <= MAX_SIDE and 1 <= img.shape[1] <= MAX_SIDE):
            raise NotImplementedError("train_input: source sides up to %d (got %s)" % (MAX_SIDE, img.shape[:2]))


def _pack_images(pk, images, minv, flip, order, blend, light, mean, std):
    b = len(images)
    sizes = [img.nbytes for img in images]
    pk.add('src', np.concatenate([np.ascontiguousarray(img).reshape(-1) for img in images]))
    pk.add('src_off', np.concatenate([[0], np.cumsum(sizes[:-1])]).astype(np.int64))
    pk.add('src_hw', np.array([img.shape[:2] for img in images], np.int32).reshape(b, 2))
    pk.add('minv', np.asarray(minv, np.float64).reshape(b, 6))
    pk.add('flip', np.asarray(flip, np.uint8).reshape(b))
    order = np.asarray(order, np.int64).reshape(b)
    if ((order < -1) | (order > 5)).any():
        raise ValueError("train_input: blend order codes are -1 (off) or 0..5")
    pk.add('order', order.astype(np.int32))
    pk.add('blend', np.asarray(blend, F32).reshape(b, 6))
    pk.add('light', np.asarray(light, np.float64).reshape(b, 3))
    pk.add('norm', np.concatenate([np.asarray(mean, F32).reshape(3), np.asarray(std, F32).reshape(3)]))


def _collate(samples, what, keys, same=None, slots=True, color=True):
    """What every collate_* (named `what` in the messages) does before it packs its slot arrays.  Raises ValueError
    when the samples differ in `same` (default: keys), for an image that is not uint8 [H, W, 3] and, with `slots`,
    for max_objs outside [1, 128] (FocalSplatLoss / splat_gaussian, the ddd heat map).  Packs the images -- with
    `color` the samples' flips and colour parameters, else neither -- and trans_output.  Returns the packer and the
    scalars: `keys` of the first sample, batch and color (any colour augmentation)."""
    s0 = samples[0]
    for s in samples:
        if any(s[k] != s0[k] for k in (keys if same is None else same)):
            raise ValueError("%s: samples with different settings cannot be batched" % what)
    images = [s['image'] for s in samples]
    _check_images(images)
    b, m = len(samples), int(s0['max_objs'])
    if slots and not 1 <= m <= 128:
        raise ValueError("%s: 1 to 128 object slots, got %d" % (what, m))
    if color:
        flip, order, blend, light = ([s[k] for s in samples] for k in ('flip', 'order', 'blend', 'light'))
    else:
        flip, order, blend, light = np.zeros(b, np.uint8), np.full(b, -1), np.zeros((b, 6), F32), np.zeros((b, 3))
    pk = _Packer()
    _pack_images(pk, images, [s['minv'] for s in samples], flip, order, blend, light, s0['mean'], s0['std'])
    pk.add('trans_output', np.array([s['trans_output'] for s in samples], np.float64).reshape(b, 6))
    scalars = {k: s0[k] for k in keys}
    scalars.update(batch=b, color=any(o >= 0 for o in order))
    return pk, scalars


def _views(buf, layout):
    out = {}
    for name, (off, dt, shape) in layout.items():
        dt = np.dtype(dt)
        n = int(np.prod(shape, dtype=np.int64)) * dt.itemsize
        out[name] = buf[off:off + n].view(getattr(torch, dt.name)).reshape(shape)
    return out


def _launch_images(v, b, out_h, out_w, color, dtype, memory_format, dev):
    if dtype not in _DTYPE_CODES:
        raise ValueError("train_input: dtype must be float32, bfloat16 or float16, got %s" % (dtype,))
    if memory_format not in (torch.contiguous_format, torch.channels_last):
        raise ValueError("train_input: memory_format must be contiguous_format or channels_last")
    if out_h * out_w > C.TRAIN_MAX_PIXELS:
        raise NotImplementedError("train_input: at most %d output pixels per image" % C.TRAIN_MAX_PIXELS)
    out = torch.empty((b, 3, out_h, out_w), dtype=dtype, device=dev, memory_format=memory_format)
    wsb = C.train_images_workspace_bytes(b, out_h, out_w) if color else 0
    ws = workspace(wsb, dev) if color else None
    C.train_images(ptr(v['src']), ptr(v['src_off']), ptr(v['src_hw']), ptr(v['minv']), ptr(v['flip']),
                   ptr(v['order']) if color else 0, ptr(v['blend']), ptr(v['light']), ptr(v['norm'][:3]),
                   ptr(v['norm'][3:]), b, out_h, out_w, ptr(out), _DTYPE_CODES[dtype],
                   int(memory_format == torch.channels_last), ptr(ws), wsb, stream_ptr(out))
    return out


def _device(device):
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


def _upload(packed, device, out_h, out_w, dtype, memory_format):
    """A collate_* result's one non-blocking H2D copy on the current stream and the image pass at out_h x out_w:
    returns the views of the device buffer and 'input'."""
    dev = _device(device)
    sc = packed['scalars']
    v = _views(packed['buffer'].to(dev, non_blocking=True), packed['layout'])
    return v, _launch_images(v, sc['batch'], out_h, out_w, sc['color'], dtype, memory_format, dev)


# The FocalSplatLoss object lists, returned as obj_*, hp_* (no class) and ex_*.
_LIST_KEYS = ('cls', 'cx', 'cy', 'radius', 'valid')


def _lists(shape, dev, n=5):
    """The last n of the _LIST_KEYS lists, of `shape`: int32, and uint8 for valid."""
    return [torch.empty(shape, dtype=torch.int32, device=dev) for _ in range(n - 1)] + \
        [torch.empty(shape, dtype=torch.uint8, device=dev)]


def augment_images(images, matrices, out_h, out_w, mean, std, flips=None, orders=None, blends=None, lights=None,
                   device=None, dtype=torch.float32, memory_format=torch.contiguous_format):
    """The image half of the training samplers for explicit parameters: per image cv2.warpAffine(img, M,
    (out_w, out_h), INTER_LINEAR) of the uint8 BGR source (mirrored first, img[:, ::-1], where flips says so),
    x / 255, color_aug when orders[b] >= 0, (x - mean) / std, as [B, 3, out_h, out_w] of dtype in memory_format.
      images: list of uint8 [H, W, 3] numpy arrays (any sizes); matrices: the FORWARD 2x3 matrices, as passed to
      cv2.warpAffine (rotated ones included); orders: blend order codes (ORDERS index, -1 = no colour
      augmentation), blends [B, 6] the float32 (alpha, 1 - alpha) of brightness, contrast and saturation,
      lights [B, 3] the float64 lighting offsets (see sample_params).
    One host->device copy and one launch (two with colour augmentation)."""
    dev = _device(device)
    images = [np.asarray(img) for img in images]
    _check_images(images)
    b = len(images)
    if b == 0:
        raise ValueError("augment_images: no images")
    minv = np.array([_invert(m) for m in np.asarray(matrices, np.float64).reshape(b, 2, 3)], np.float64)
    flips = np.zeros(b, np.uint8) if flips is None else np.asarray(flips, np.uint8)
    orders = np.full(b, -1) if orders is None else np.asarray(orders)
    pk = _Packer()
    _pack_images(pk, images, minv, flips, orders, np.zeros((b, 6), F32) if blends is None else blends,
                 np.zeros((b, 3)) if lights is None else lights, mean, std)
    buf = pk.tensor(_pin() and dev.type == "cuda").to(dev, non_blocking=True)
    return _launch_images(_views(buf, pk.layout), b, int(out_h), int(out_w), bool((orders >= 0).any()), dtype,
                          memory_format, dev)


def collate_ctdet(samples):
    """Packs CTDetTrainInput samples into one uint8 buffer (images, then the small per-image arrays) and the
    scalars build_ctdet_batch needs.  Raises ValueError when the samples have different input sizes (keep_res
    with images of different sizes), where the reference's default_collate fails too."""
    s0 = samples[0]
    for s in samples:
        if (s['input_h'], s['input_w']) != (s0['input_h'], s0['input_w']):
            raise ValueError("collate_ctdet: samples of different input sizes (%dx%d and %dx%d) cannot be batched"
                             % (s0['input_h'], s0['input_w'], s['input_h'], s['input_w']))
    pk, scalars = _collate(samples, 'collate_ctdet', ('input_h', 'input_w', 'output_h', 'output_w', 'max_objs',
                                                      'num_classes', 'cat_spec_wh', 'reg_offset'), same=(), slots=False)
    b, m = len(samples), int(s0['max_objs'])
    boxes = np.zeros((b, m, 4), F32)
    cls = np.zeros((b, m), np.int32)
    nobj = np.zeros(b, np.int32)
    for i, s in enumerate(samples):
        n = min(len(s['boxes']), m)
        boxes[i, :n], cls[i, :n], nobj[i] = s['boxes'][:n], s['cls'][:n], n
        if n and (cls[i, :n].min() < 0 or cls[i, :n].max() >= s0['num_classes']):
            raise ValueError("collate_ctdet: class id outside [0, %d)" % s0['num_classes'])
    pk.add('nobj', nobj)
    pk.add('boxes', boxes)
    pk.add('cls', cls)
    return pk.collated(scalars)


def build_ctdet_batch(packed, device=None, dtype=torch.float32, memory_format=torch.contiguous_format,
                      dense_hm=False):
    """The reference's collated ctdet batch, on the device, from a collate_ctdet result: one non-blocking H2D
    copy on the current stream, the image pass (one launch, two with colour augmentation) and the target kernel,
    plus splat_gaussian with dense_hm.  Keys, shapes and dtypes as ctdet.py:128-140 returns them; 'hm' only with
    dense_hm; always the FocalSplatLoss lists obj_cls, obj_cx, obj_cy, obj_radius (int32) and obj_valid (uint8).
    The packed host buffer is not modified."""
    sc = packed['scalars']
    b, m, nc, oh, ow = sc['batch'], sc['max_objs'], sc['num_classes'], sc['output_h'], sc['output_w']
    v, inp = _upload(packed, device, sc['input_h'], sc['input_w'], dtype, memory_format)
    dev = inp.device
    f32 = dict(dtype=torch.float32, device=dev)
    u8 = dict(dtype=torch.uint8, device=dev)
    wh, reg = torch.empty((b, m, 2), **f32), torch.empty((b, m, 2), **f32)
    ind, reg_mask = torch.empty((b, m), dtype=torch.int64, device=dev), torch.empty((b, m), **u8)
    csw = torch.empty((b, m, 2 * nc), **f32) if sc['cat_spec_wh'] else None
    csm = torch.empty((b, m, 2 * nc), **u8) if sc['cat_spec_wh'] else None
    lists = _lists((b, m), dev)
    C.ctdet_targets(ptr(v['boxes']), ptr(v['cls']), ptr(v['nobj']), ptr(v['flip']), ptr(v['src_hw']),
                    ptr(v['trans_output']), b, m, nc, oh, ow, ptr(wh), ptr(ind), ptr(reg), ptr(reg_mask), ptr(csw),
                    ptr(csm), *[ptr(t) for t in lists], stream_ptr(wh))
    ret = {'input': inp, 'reg_mask': reg_mask, 'ind': ind}
    if dense_hm:
        ret['hm'] = splat_gaussian(*lists, nc, oh, ow)
    if sc['cat_spec_wh']:
        ret.update(cat_spec_wh=csw, cat_spec_mask=csm)
    else:
        ret['wh'] = wh
    if sc['reg_offset']:
        ret['reg'] = reg
    ret.update(('obj_' + k, t) for k, t in zip(_LIST_KEYS, lists))
    return ret


# ---------------------------------------------------------------- multi_pose (datasets/sample/multi_pose.py)
def multi_pose_params(height, width, opt, split, data_rng, eig_val, eig_vec):
    """The random draws of MultiPoseDataset.__getitem__ (multi_pose.py:39-75) for one height x width image, in the
    reference's order -- crop draws, then ALWAYS one np.random.random() < aug_rot in the train split (a second
    randn for the angle when it succeeds), the flip draw, color_aug -- and the three matrices they give:
    trans_input (rotated; inverted for the warp), trans_output_rot (rotated, for the keypoints) and trans_output
    (rot 0, for the boxes).  The input is input_res square (there is no keep_res branch)."""
    c = np.array([width / 2., height / 2.], dtype=np.float32)
    s = max(height, width) * 1.0
    rot = 0
    flipped = False
    if split == 'train':
        s = crop_draws(height, width, c, s, opt)
        if np.random.random() < opt.aug_rot:
            rf = opt.rotate
            rot = np.clip(np.random.randn() * rf, -rf * 2, rf * 2)
        if np.random.random() < opt.flip:
            flipped = True
            c[0] = width - c[0] - 1
    order, blend, light = color_draws(split, opt, data_rng, eig_val, eig_vec)
    res, out_res = int(opt.input_res), int(opt.output_res)
    return {'c': c, 's': s, 'rot': rot, 'flip': flipped, 'input_res': res, 'output_res': out_res,
            'minv': np.array(_invert(affine_transform(c, s, [res, res], rot)), np.float64),
            'trans_output_rot': affine_transform(c, s, [out_res, out_res], rot).reshape(6),
            'trans_output': affine_transform(c, s, [out_res, out_res]).reshape(6),
            'order': order, 'blend': blend, 'light': light}


class MultiPoseTrainInput(_TrainInput):
    """Wraps a reference MultiPoseDataset instance (also duck-typed on num_classes, num_joints, flip_idx, _data_rng,
    _eig_val and _eig_vec): multi_pose_params' draws, the float32 box corners, the keypoints and the class
    int(category_id) - 1, as there; the batch is collate_multi_pose + build_multi_pose_batch's.  opt.dense_hp is
    rejected."""
    unsupported = ('dense_hp',)

    def _params(self, ds, height, width):
        return multi_pose_params(height, width, ds.opt, ds.split, ds._data_rng, ds._eig_val, ds._eig_vec)

    def _fields(self, ds, anns):
        opt = ds.opt
        return {'boxes': _boxes(anns), 'cls': np.array([int(a['category_id']) - 1 for a in anns], np.int64),
                'keypoints': [np.array(a['keypoints'], np.float32).reshape(-1) for a in anns],
                'num_classes': ds.num_classes, 'num_joints': ds.num_joints,
                'flip_idx': [tuple(e) for e in ds.flip_idx], 'hm_hp': bool(opt.hm_hp),
                'reg_hp_offset': bool(opt.reg_hp_offset)}


def flip_permutation(num_joints, flip_idx):
    """The joint order after multi_pose.py:112-113's swaps: new joint j is old joint perm[j].  The swaps are
    applied to arange(J) in order, so pairs that share a joint compose as they do there."""
    perm = list(range(num_joints))
    for a, b in flip_idx:
        perm[a], perm[b] = perm[b], perm[a]
    return np.array(perm, np.int32)


def collate_multi_pose(samples):
    """Packs MultiPoseTrainInput samples into one uint8 buffer: what collate_ctdet packs plus the keypoints
    [B, M, J, 3] float32, both output matrices, a per-image rotated byte and the joint permutation of the flip.
    Raises ValueError for input the target kernel cannot match or the reference cannot run: a keypoint list whose
    length is not 3 J, a visibility that is negative or not finite, a class outside [0, num_classes), more than
    128 slots, a rotated sample with a box of negative width or height, or samples of different settings."""
    s0 = samples[0]
    keys = ('input_res', 'output_res', 'max_objs', 'num_classes', 'num_joints', 'reg_offset', 'hm_hp', 'reg_hp_offset')
    pk, scalars = _collate(samples, 'collate_multi_pose', keys, same=keys + ('flip_idx',))
    b, m, nj, nc = len(samples), int(s0['max_objs']), int(s0['num_joints']), int(s0['num_classes'])
    if nj < 1:
        raise ValueError("collate_multi_pose: no joints")
    perm = flip_permutation(nj, s0['flip_idx'])
    boxes = np.zeros((b, m, 4), F32)
    cls = np.zeros((b, m), np.int32)
    kps = np.zeros((b, m, nj, 3), F32)
    nobj = np.zeros(b, np.int32)
    rotated = np.zeros(b, np.uint8)
    for i, s in enumerate(samples):
        n = min(len(s['boxes']), m)
        nobj[i], rotated[i] = n, s['rot'] != 0
        c = np.asarray(s['cls'][:n], np.int64)
        if n and (c.min() < 0 or c.max() >= nc):
            raise ValueError("collate_multi_pose: class id outside [0, %d)" % nc)
        for k in range(n):
            p = np.asarray(s['keypoints'][k], F32).reshape(-1)
            if p.size != 3 * nj:
                raise ValueError("collate_multi_pose: %d keypoint values, expected 3 x %d joints" % (p.size, nj))
            kps[i, k] = p.reshape(nj, 3)
        vis = kps[i, :n, :, 2]
        if not (np.isfinite(vis).all() and (vis >= 0).all()):
            raise ValueError("collate_multi_pose: keypoint visibilities must be finite and >= 0")
        bx = np.asarray(s['boxes'][:n], F32).reshape(n, 4)
        if rotated[i] and ((bx[:, 2] < bx[:, 0]) | (bx[:, 3] < bx[:, 1])).any():
            raise ValueError("collate_multi_pose: a box with negative width or height in a rotated sample "
                             "(gaussian_radius of it is NaN in the reference)")
        boxes[i, :n], cls[i, :n] = bx, c
    pk.add('trans_output_rot', np.array([s['trans_output_rot'] for s in samples], np.float64).reshape(b, 6))
    pk.add('nobj', nobj)
    pk.add('boxes', boxes)
    pk.add('cls', cls)
    pk.add('kps', kps)
    pk.add('rotated', rotated)
    pk.add('perm', perm)
    scalars['rotated'] = rotated.astype(bool).tolist()
    return pk.collated(scalars)


def build_multi_pose_batch(packed, device=None, dtype=torch.float32, memory_format=torch.contiguous_format,
                           dense_hm=False):
    """The reference's collated multi_pose batch, on the device, from a collate_multi_pose result: one
    non-blocking H2D copy on the current stream, the image pass at input_res x input_res and the target kernel,
    plus splat_gaussian with dense_hm.  Keys, shapes and dtypes as multi_pose.py:161-177 returns them: input,
    reg_mask u8, ind i64, wh, hps f32 [B,M,2J], hps_mask u8; reg with reg_offset; hp_offset f32 [B,M*J,2], hp_ind
    i64, hp_mask i64 with reg_hp_offset; hm [B,C,R,R] and, with hm_hp, hm_hp [B,J,R,R] only with dense_hm.  Always
    the FocalSplatLoss lists of the centres, obj_cls / obj_cx / obj_cy / obj_radius (int32) and obj_valid (uint8)
    [B,M], and with hm_hp those of the joints, hp_cx / hp_cy / hp_radius (int32) and hp_valid (uint8) [B,J,M]: as
    [B*J, M] views with class 0 they give hm_hp as [B*J, 1, R, R].  The reference fills hm of a rotated image
    with 0.9999, which no list expresses: dense_hm=False with a rotated sample raises ValueError.  The packed host
    buffer is not modified."""
    sc = packed['scalars']
    if not dense_hm and any(sc['rotated']):
        raise ValueError("build_multi_pose_batch: a rotated sample's hm is the constant 0.9999, which the object "
                         "lists cannot express; use dense_hm=True")
    b, m, nj, nc, r = sc['batch'], sc['max_objs'], sc['num_joints'], sc['num_classes'], sc['output_res']
    v, inp = _upload(packed, device, sc['input_res'], sc['input_res'], dtype, memory_format)
    dev = inp.device
    f32 = dict(dtype=torch.float32, device=dev)
    u8 = dict(dtype=torch.uint8, device=dev)
    i64 = dict(dtype=torch.int64, device=dev)
    wh, reg = torch.empty((b, m, 2), **f32), torch.empty((b, m, 2), **f32)
    ind, reg_mask = torch.empty((b, m), **i64), torch.empty((b, m), **u8)
    hps, hps_mask = torch.empty((b, m, 2 * nj), **f32), torch.empty((b, m, 2 * nj), **u8)
    hp_offset, hp_ind, hp_mask = torch.empty((b, m * nj, 2), **f32), torch.empty((b, m * nj), **i64), \
        torch.empty((b, m * nj), **i64)
    lists, hp_lists = _lists((b, m), dev), _lists((b, nj, m), dev, 4)
    C.multi_pose_targets(ptr(v['boxes']), ptr(v['cls']), ptr(v['nobj']), ptr(v['kps']), ptr(v['flip']),
                         ptr(v['rotated']), ptr(v['src_hw']), ptr(v['trans_output']), ptr(v['trans_output_rot']),
                         ptr(v['perm']), b, m, nj, r, ptr(wh), ptr(ind), ptr(reg), ptr(reg_mask), ptr(hps),
                         ptr(hps_mask), ptr(hp_offset), ptr(hp_ind), ptr(hp_mask), *[ptr(t) for t in lists],
                         *[ptr(t) for t in hp_lists], stream_ptr(wh))
    ret = {'input': inp}
    if dense_hm:
        hm = splat_gaussian(*lists, nc, r, r)
        if any(sc['rotated']):   # hm * 0 + 0.9999 (multi_pose.py:157-158), from the device copy of the flags
            hm.masked_fill_(v['rotated'].view(b, 1, 1, 1).bool(), F32(0.9999).item())
        ret['hm'] = hm
    ret.update(reg_mask=reg_mask, ind=ind, wh=wh, hps=hps, hps_mask=hps_mask)
    if sc['reg_offset']:
        ret['reg'] = reg
    if dense_hm and sc['hm_hp']:
        flat = [t.view(b * nj, m) for t in hp_lists]
        ret['hm_hp'] = splat_gaussian(torch.zeros_like(flat[0]), *flat, 1, r, r).view(b, nj, r, r)
    if sc['reg_hp_offset']:
        ret.update(hp_offset=hp_offset, hp_ind=hp_ind, hp_mask=hp_mask)
    ret.update(('obj_' + k, t) for k, t in zip(_LIST_KEYS, lists))
    if sc['hm_hp']:
        ret.update(('hp_' + k, t) for k, t in zip(_LIST_KEYS[1:], hp_lists))
    return ret


# ---------------------------------------------------------------- ddd (datasets/sample/ddd.py)
def ddd_params(height, width, opt, split):
    """The random draws of DddDataset.__getitem__ (ddd.py:37-66) for one height x width image and the matrices they
    give.  Only np.random draws: in the train split one np.random.random() < aug_ddd (none in val: the `and`
    short-circuits) and, when it succeeds, scale_shift_draws.  There is no flip and no colour augmentation.  The
    centre is float64 and the scale an int32 pair ([input_w, input_h] under keep_res, else [width, height]), float64
    once augmented."""
    c = np.array([width / 2., height / 2.])
    if opt.keep_res:
        s = np.array([opt.input_w, opt.input_h], dtype=np.int32)
    else:
        s = np.array([width, height], dtype=np.int32)
    aug = False
    if split == 'train' and np.random.random() < opt.aug_ddd:
        aug = True
        s = scale_shift_draws(height, width, c, s, opt)
    input_h, input_w = int(opt.input_h), int(opt.input_w)
    output_h, output_w = int(opt.output_h), int(opt.output_w)
    return {'c': c, 's': s, 'aug': aug, 'input_h': input_h, 'input_w': input_w, 'output_h': output_h,
            'output_w': output_w,
            'minv': np.array(_invert(affine_transform(c, s, [input_w, input_h])), np.float64),
            'trans_output': affine_transform(c, s, [output_w, output_h]).reshape(6)}


_DDD_IGNORED = {'alpha': 0., 'depth': 0., 'dim': [0., 0., 0.]}


class DddTrainInput(_TrainInput):
    """Wraps a reference DddDataset instance (also duck-typed on cat_ids and alpha_in_degree): ddd_params' draws and
    per annotation the float32 box corners, the class cat_ids[category_id], _convert_alpha(alpha) as float64, depth
    and dim; the batch is collate_ddd + build_ddd_batch's.  The number of classes is opt.num_classes, as there."""

    def _params(self, ds, height, width):
        return ddd_params(height, width, ds.opt, ds.split)

    def _fields(self, ds, anns):
        opt = ds.opt
        cls = np.array([int(ds.cat_ids[a['category_id']]) for a in anns], np.int64)
        # only positive classes read these in the reference; an ignore object may lack them
        vals = [a if c >= 0 else dict(_DDD_IGNORED, **a) for a, c in zip(anns, cls)]
        alpha = [math.radians(v['alpha'] + 45) if ds.alpha_in_degree else v['alpha'] for v in vals]
        return {'boxes': _boxes(anns), 'cls': cls, 'alpha': np.array(alpha, np.float64),
                'depth': np.array([v['depth'] for v in vals], np.float64),
                'dim': [np.asarray(v['dim'], np.float64).reshape(-1) for v in vals],
                'num_classes': int(opt.num_classes), 'rect_mask': bool(opt.rect_mask), 'reg_bbox': bool(opt.reg_bbox)}


def collate_ddd(samples):
    """Packs DddTrainInput samples into one uint8 buffer: the images (no flip, no colour augmentation), the output
    matrices, the per-image augmented byte and per slot the box, class, alpha (float64), depth and dim (float32).
    Raises ValueError for samples of different settings, max_objs outside [1, 128], a class the reference cannot
    index (anything but <= -99, -1, [-C - 1, -2] or [0, C)) and a dim that is not 3 values."""
    s0 = samples[0]
    keys = ('input_h', 'input_w', 'output_h', 'output_w', 'max_objs', 'num_classes', 'rect_mask', 'reg_bbox',
            'reg_offset')
    pk, scalars = _collate(samples, 'collate_ddd', keys, color=False)
    b, m, nc = len(samples), int(s0['max_objs']), int(s0['num_classes'])
    boxes = np.zeros((b, m, 4), F32)
    cls = np.zeros((b, m), np.int32)
    alpha = np.zeros((b, m), np.float64)
    depth = np.zeros((b, m), F32)
    dim = np.zeros((b, m, 3), F32)
    nobj = np.zeros(b, np.int32)
    for i, s in enumerate(samples):
        n = min(len(s['boxes']), m)
        c = np.asarray(s['cls'][:n], np.int64)
        ok = (c <= -99) | (c == -1) | ((c >= -nc - 1) & (c <= -2)) | ((c >= 0) & (c < nc))
        if not ok.all():
            raise ValueError("collate_ddd: class id %d is none of <= -99, -1, [%d, -2] or [0, %d)"
                             % (c[~ok][0], -nc - 1, nc))
        for k in range(n):
            d = np.asarray(s['dim'][k], np.float64).reshape(-1)
            if d.size != 3:
                raise ValueError("collate_ddd: dim has %d values, expected 3" % d.size)
            dim[i, k] = d
        nobj[i] = n
        boxes[i, :n] = np.asarray(s['boxes'][:n], F32).reshape(n, 4)
        cls[i, :n] = np.maximum(c, -99)
        alpha[i, :n] = np.asarray(s['alpha'][:n], np.float64)
        depth[i, :n] = np.asarray(s['depth'][:n], np.float64)
    pk.add('aug', np.array([bool(s['aug']) for s in samples], np.uint8))
    pk.add('nobj', nobj)
    pk.add('boxes', boxes)
    pk.add('cls', cls)
    pk.add('alpha', alpha)
    pk.add('depth', depth)
    pk.add('dim', dim)
    return pk.collated(scalars)


def build_ddd_batch(packed, device=None, dtype=torch.float32, memory_format=torch.contiguous_format):
    """The reference's collated ddd batch, on the device, from a collate_ddd result: one non-blocking H2D copy on
    the current stream, the image pass at input_h x input_w and cnb_ddd_targets (targets, then hm).  Keys, shapes and
    dtypes as ddd.py:143-149 returns them: input, hm [B,C,oh,ow] f32, dep [B,M,1] f32, dim [B,M,3] f32, ind i64,
    rotbin [B,M,2] i64, rotres [B,M,2] f32, reg_mask u8, rot_mask u8; wh with reg_bbox, reg with reg_offset.  hm is
    always dense: the ignore regions overwrite it in object order, which no object list expresses.  The packed host
    buffer is not modified."""
    sc = packed['scalars']
    b, m, nc, oh, ow = sc['batch'], sc['max_objs'], sc['num_classes'], sc['output_h'], sc['output_w']
    v, inp = _upload(packed, device, sc['input_h'], sc['input_w'], dtype, memory_format)
    dev = inp.device
    f32 = dict(dtype=torch.float32, device=dev)
    u8 = dict(dtype=torch.uint8, device=dev)
    i64 = dict(dtype=torch.int64, device=dev)
    hm = torch.empty((b, nc, oh, ow), **f32)
    dep, dim = torch.empty((b, m, 1), **f32), torch.empty((b, m, 3), **f32)
    ind, rotbin, rotres = torch.empty((b, m), **i64), torch.empty((b, m, 2), **i64), torch.empty((b, m, 2), **f32)
    reg_mask, rot_mask = torch.empty((b, m), **u8), torch.empty((b, m), **u8)
    wh, reg = torch.empty((b, m, 2), **f32), torch.empty((b, m, 2), **f32)
    C.ddd_targets(ptr(v['boxes']), ptr(v['cls']), ptr(v['nobj']), ptr(v['alpha']), ptr(v['depth']), ptr(v['dim']),
                  ptr(v['aug']), ptr(v['trans_output']), b, m, nc, oh, ow, int(sc['rect_mask']), ptr(hm), ptr(dep),
                  ptr(dim), ptr(ind), ptr(rotbin), ptr(rotres), ptr(reg_mask), ptr(rot_mask), ptr(wh), ptr(reg),
                  stream_ptr(hm))
    ret = {'input': inp, 'hm': hm, 'dep': dep, 'dim': dim, 'ind': ind, 'rotbin': rotbin, 'rotres': rotres,
           'reg_mask': reg_mask, 'rot_mask': rot_mask}
    if sc['reg_bbox']:
        ret['wh'] = wh
    if sc['reg_offset']:
        ret['reg'] = reg
    return ret


# ---------------------------------------------------------------- exdet (datasets/sample/exdet.py)
def exdet_params(height, width, opt, split, data_rng, eig_val, eig_vec):
    """The random draws of EXDetDataset.__getitem__ (exdet.py:36-65) for one height x width image, in the reference's
    order, and the matrices they give.  The centre is float64.  In the train split: the random crop's choice and two
    randint (ctdet's crop_draws), or under not_rand_crop scale_shift_draws; then the flip draw.  The flip mirrors the
    image but leaves the centre, so trans_input / trans_output are the unflipped get_affine_transform(c, s, 0,
    [res, res]) applied to the mirrored source.  color_aug's draws follow as in ctdet.  The input is input_res square
    (there is no keep_res branch)."""
    c = np.array([width / 2., height / 2.])
    s = max(height, width) * 1.0
    flipped = False
    if split == 'train':
        if not opt.not_rand_crop:
            s = crop_draws(height, width, c, s, opt)
        else:
            s = scale_shift_draws(height, width, c, s, opt)
        if np.random.random() < opt.flip:
            flipped = True
    order, blend, light = color_draws(split, opt, data_rng, eig_val, eig_vec)
    res, out_res = int(opt.input_res), int(opt.output_res)
    return {'c': c, 's': s, 'flip': flipped, 'input_res': res, 'output_res': out_res,
            'minv': np.array(_invert(affine_transform(c, s, [res, res])), np.float64),
            'trans_output': affine_transform(c, s, [out_res, out_res]).reshape(6),
            'order': order, 'blend': blend, 'light': light}


class ExdetTrainInput(_TrainInput):
    """Wraps a reference EXDetDataset instance (also duck-typed on cat_ids, _data_rng, _eig_val and _eig_vec):
    exdet_params' draws, the extreme_points as float32 (t, l, b, r) and the class cat_ids[category_id]; the batch is
    collate_exdet + build_exdet_batch's.  The number of classes is opt.num_classes, as there."""

    def _params(self, ds, height, width):
        return exdet_params(height, width, ds.opt, ds.split, ds._data_rng, ds._eig_val, ds._eig_vec)

    def _fields(self, ds, anns):
        return {'points': [np.array(a['extreme_points'], dtype=np.float32).reshape(-1) for a in anns],
                'cls': np.array([int(ds.cat_ids[a['category_id']]) for a in anns], np.int64),
                'num_classes': int(ds.opt.num_classes), 'agnostic_ex': bool(ds.opt.agnostic_ex)}


def collate_exdet(samples):
    """Packs ExdetTrainInput samples into one uint8 buffer: what collate_ctdet packs for the images (flip bytes and
    colour parameters included), trans_output, and per slot the extreme points [B, M, 4, 2] float32 (t, l, b, r) and
    the class.  Raises ValueError for samples of different settings, max_objs outside [1, 128], an extreme_points
    entry that is not 8 values, a class outside [0, num_classes) (the reference would index hm_c from the end) and a
    coordinate that is not finite (the reference's pts.astype(np.int32) of it is undefined)."""
    s0 = samples[0]
    keys = ('input_res', 'output_res', 'max_objs', 'num_classes', 'agnostic_ex', 'reg_offset')
    pk, scalars = _collate(samples, 'collate_exdet', keys)
    b, m, nc = len(samples), int(s0['max_objs']), int(s0['num_classes'])
    pts = np.zeros((b, m, 4, 2), F32)
    cls = np.zeros((b, m), np.int32)
    nobj = np.zeros(b, np.int32)
    for i, s in enumerate(samples):
        n = min(len(s['points']), m)
        c = np.asarray(s['cls'][:n], np.int64)
        if n and (c.min() < 0 or c.max() >= nc):
            raise ValueError("collate_exdet: class id outside [0, %d)" % nc)
        for k in range(n):
            p = np.asarray(s['points'][k], F32).reshape(-1)
            if p.size != 8:
                raise ValueError("collate_exdet: extreme_points has %d values, expected 4 x 2" % p.size)
            if not np.isfinite(p).all():
                raise ValueError("collate_exdet: extreme_points must be finite")
            pts[i, k] = p.reshape(4, 2)
        nobj[i], cls[i, :n] = n, c
    pk.add('nobj', nobj)
    pk.add('pts', pts)
    pk.add('cls', cls)
    return pk.collated(scalars)


EXDET_PARTS = ('t', 'l', 'b', 'r')


def build_exdet_batch(packed, device=None, dtype=torch.float32, memory_format=torch.contiguous_format,
                      dense_hm=False):
    """The reference's collated exdet batch, on the device, from a collate_exdet result: one non-blocking H2D copy on
    the current stream, the image pass at input_res x input_res (the mirrored source under the unflipped matrix) and
    cnb_exdet_targets, plus splat_gaussian with dense_hm.  Keys, shapes and dtypes as exdet.py:130-135 returns them:
    input; with reg_offset reg_mask u8 [B,M], reg_t / reg_l / reg_b / reg_r f32 [B,M,2] and ind_t / ind_l / ind_b /
    ind_r i64 [B,M]; with dense_hm hm_t / hm_l / hm_b / hm_r f32 [B,num_hm,R,R] (num_hm 1 under agnostic_ex, else C)
    and hm_c f32 [B,C,R,R].  Always the FocalSplatLoss lists: the centres obj_cls / obj_cx / obj_cy / obj_radius
    (int32) and obj_valid (uint8) [B,M], and the extreme points ex_cls / ex_cx / ex_cy / ex_radius (int32) and
    ex_valid (uint8) [4,B,M] in the order t, l, b, r -- ex_*[p] is part p's [B,M] list set, and the [4B, M] view
    of all four gives the four extreme maps in one splat.  The packed host buffer is not modified."""
    sc = packed['scalars']
    b, m, nc, r = sc['batch'], sc['max_objs'], sc['num_classes'], sc['output_res']
    num_hm = 1 if sc['agnostic_ex'] else nc
    v, inp = _upload(packed, device, sc['input_res'], sc['input_res'], dtype, memory_format)
    dev = inp.device
    reg = torch.empty((4, b, m, 2), dtype=torch.float32, device=dev)
    ind = torch.empty((4, b, m), dtype=torch.int64, device=dev)
    reg_mask = torch.empty((b, m), dtype=torch.uint8, device=dev)
    lists, ex_lists = _lists((b, m), dev), _lists((4, b, m), dev)
    C.exdet_targets(ptr(v['pts']), ptr(v['cls']), ptr(v['nobj']), ptr(v['flip']), ptr(v['src_hw']),
                    ptr(v['trans_output']), b, m, r, int(sc['agnostic_ex']), ptr(reg), ptr(ind), ptr(reg_mask),
                    *[ptr(t) for t in lists], *[ptr(t) for t in ex_lists], stream_ptr(reg))
    ret = {'input': inp}
    if dense_hm:
        hm = splat_gaussian(*[t.view(4 * b, m) for t in ex_lists], num_hm, r, r).view(4, b, num_hm, r, r)
        ret.update(('hm_' + p, hm[j]) for j, p in enumerate(EXDET_PARTS))
        ret['hm_c'] = splat_gaussian(*lists, nc, r, r)
    if sc['reg_offset']:
        ret['reg_mask'] = reg_mask
        ret.update(('reg_' + p, reg[j]) for j, p in enumerate(EXDET_PARTS))
        ret.update(('ind_' + p, ind[j]) for j, p in enumerate(EXDET_PARTS))
    ret.update(('obj_' + k, t) for k, t in zip(_LIST_KEYS, lists))
    ret.update(('ex_' + k, t) for k, t in zip(_LIST_KEYS, ex_lists))
    return ret

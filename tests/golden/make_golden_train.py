"""Generates tests/golden/train.npz with the UNMODIFIED CTDetDataset.__getitem__ of the reference
(datasets/sample/ctdet.py:29-145, color_aug of utils/image.py; cv2 from this image) -- build container only.

Each case is a dataset over seeded images (tests/train_cases.py) written as lossless PNGs to a temporary
directory, with a stub `coco`; np.random, random and the dataset's _data_rng are seeded per case.  Stored per
sample: the draws (c and s from meta -- opt.debug = 1 --, flip and the shuffle order replayed from the saved
generator states, the uniform / normal draws recorded by a proxy of _data_rng), CRCs of the three generator
states after the sample, the CRC and a strided sample of `input`, the full targets and, for the first samples of
each case, `hm`.  Rotation cases run get_affine_transform(rot != 0) + cv2.warpAffine + color_aug directly."""
import os
import random
import sys
import tempfile
import zlib

import numpy as np

REF = "/root/reference/src/lib"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(HERE))
import cv2  # noqa: E402
import importlib.util  # noqa: E402
# by path: the reference's datasets/ is a namespace package that an installed `datasets` would shadow
_spec = importlib.util.spec_from_file_location("ref_ctdet", os.path.join(REF, "datasets", "sample", "ctdet.py"))
_ctdet = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_ctdet)
CTDetDataset = _ctdet.CTDetDataset
from utils.image import color_aug, get_affine_transform  # noqa: E402

import train_cases as TC  # noqa: E402


class StubCOCO(object):
    def __init__(self, files, anns):
        self.files, self.anns = files, anns

    def loadImgs(self, ids):
        return [{'file_name': self.files[ids[0]]}]

    def getAnnIds(self, imgIds):
        return [(imgIds[0], k) for k in range(len(self.anns[imgIds[0]]))]

    def loadAnns(self, ids):
        return [self.anns[i][k] for i, k in ids]


class RecordingRng(object):
    """Delegates to a RandomState and records what uniform / normal returned."""

    def __init__(self, rng):
        self.rng, self.log = rng, []

    def uniform(self, *a, **k):
        v = self.rng.uniform(*a, **k); self.log.append(('u', v)); return v

    def normal(self, *a, **k):
        v = self.rng.normal(*a, **k); self.log.append(('n', v)); return v


def state_crcs(data_rng):
    k, pos = np.random.get_state()[1:3]
    c_np = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    c_py = zlib.crc32(np.asarray(random.getstate()[1], np.uint64).tobytes())
    k, pos = data_rng.get_state()[1:3]
    c_dr = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    return np.array([c_np, c_py, c_dr], np.uint32)


def replay_flip(ds, np_state, opt, height, width):
    """The flip draw of the sample that started from np_state (np.random is restored afterwards)."""
    saved = np.random.get_state()
    np.random.set_state(np_state)
    if not opt.not_rand_crop:
        wb, hb = ds._get_border(128, width), ds._get_border(128, height)
        np.random.choice(np.arange(0.6, 1.4, 0.1))
        np.random.randint(low=wb, high=width - wb); np.random.randint(low=hb, high=height - hb)
    else:
        np.random.randn(); np.random.randn(); np.random.randn()
    flip = np.random.random() < opt.flip
    np.random.set_state(saved)
    return flip


def replay_order(py_state):
    saved = random.getstate()
    random.setstate(py_state)
    kinds = [0, 1, 2]
    random.shuffle(kinds)
    random.setstate(saved)
    return TC.ORDERS.index(tuple(kinds))


def run_case(name, case, tmp, out):
    opt = TC.make_opt(case)
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        img = TC.case_image(name, i)
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(tmp, files[i]), img)
        anns[i] = TC.case_anns(name, i)
    ds = CTDetDataset.__new__(CTDetDataset)
    ds.opt, ds.coco, ds.images, ds.img_dir = opt, StubCOCO(files, anns), list(range(len(files))), tmp
    ds.max_objs, ds.num_classes, ds.cat_ids = case['max_objs'], case['num_classes'], TC.cat_ids(case)
    ds.mean, ds.std = TC.MEAN.reshape(1, 1, 3), TC.STD.reshape(1, 1, 3)
    ds._eig_val, ds._eig_vec, ds.split = TC.EIG_VAL, TC.EIG_VEC, case['split']
    rec = RecordingRng(np.random.RandomState(case['seed']))
    ds._data_rng = rec
    np.random.seed(case['seed']); random.seed(case['seed'])
    for i in range(len(files)):
        p = "%s_%d_" % (name, i)
        np_state, py_state = np.random.get_state(), random.getstate()
        rec.log = []
        h, w = case['sizes'][i]
        ret = ds.__getitem__(i)
        out[p + "states"] = state_crcs(rec.rng)
        out[p + "c"] = np.asarray(ret['meta']['c'], np.float32)
        s = ret['meta']['s']
        out[p + "s"] = np.asarray(s if isinstance(s, np.ndarray) else [s, s], np.float64)
        out[p + "s_is_array"] = np.bool_(isinstance(s, np.ndarray))
        out[p + "flip"] = np.bool_(case['split'] == 'train' and replay_flip(ds, np_state, opt, h, w))
        color = case['split'] == 'train' and not opt.no_color_aug
        out[p + "order"] = np.int32(replay_order(py_state) if color else -1)
        blend, light = np.zeros(6, np.float32), np.zeros(3, np.float64)
        if color:
            order = TC.ORDERS[int(out[p + "order"])]
            for kind, (_, alpha) in zip(order, rec.log[:3]):
                alpha = 1. + alpha
                blend[2 * kind], blend[2 * kind + 1] = np.float32(alpha), np.float32(1 - alpha)
            light = np.dot(TC.EIG_VEC, TC.EIG_VAL * rec.log[3][1])
        out[p + "blend"], out[p + "light"] = blend, light
        inp = np.ascontiguousarray(ret['input'], np.float32)
        out[p + "input_crc"] = np.uint32(zlib.crc32(inp.view(np.uint8)))
        out[p + "input_shape"] = np.array(inp.shape, np.int64)
        out[p + "input_sample"] = inp[:, ::17, ::13].copy()
        for k in ('reg_mask', 'ind', 'wh', 'reg', 'cat_spec_wh', 'cat_spec_mask'):
            if k in ret:
                out[p + k] = ret[k]
        if i < case.get('hm_samples', 1):
            out[p + "hm"] = ret['hm']


def run_rotation(name, case, out):
    rng = np.random.RandomState(case['seed'])
    random.seed(case['seed'])
    img = TC.case_image(name, 0)
    h, w = case['sizes'][0]
    c = np.array([w / 2., h / 2.], np.float32)
    m = get_affine_transform(c, max(h, w) * case['scale'], case['rot'], [case['out'], case['out']])
    py_state = random.getstate()
    inp = cv2.warpAffine(img, m, (case['out'], case['out']), flags=cv2.INTER_LINEAR).astype(np.float32) / 255.
    rec = RecordingRng(rng)
    color_aug(rec, inp, TC.EIG_VAL, TC.EIG_VEC)
    inp = ((inp - TC.MEAN.reshape(1, 1, 3)) / TC.STD.reshape(1, 1, 3)).transpose(2, 0, 1)
    order = replay_order(py_state)
    blend = np.zeros(6, np.float32)
    for kind, (_, alpha) in zip(TC.ORDERS[order], rec.log[:3]):
        alpha = 1. + alpha
        blend[2 * kind], blend[2 * kind + 1] = np.float32(alpha), np.float32(1 - alpha)
    p = name + "_0_"
    out[p + "matrix"] = np.asarray(m, np.float64)
    out[p + "order"], out[p + "blend"] = np.int32(order), blend
    out[p + "light"] = np.dot(TC.EIG_VEC, TC.EIG_VAL * rec.log[3][1])
    inp = np.ascontiguousarray(inp, np.float32)
    out[p + "input_crc"] = np.uint32(zlib.crc32(inp.view(np.uint8)))
    out[p + "input_shape"] = np.array(inp.shape, np.int64)
    out[p + "input_sample"] = inp[:, ::17, ::13].copy()


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, case in TC.CASES.items():
            if 'rot' in case:
                run_rotation(name, case, out)
            else:
                run_case(name, case, tmp, out)
    np.savez_compressed(os.path.join(HERE, "train.npz"), **out)
    orders = sorted({int(v) for k, v in out.items() if k.endswith("_order")})
    print("wrote train.npz: %d arrays, blend orders %s, %d bytes"
          % (len(out), orders, os.path.getsize(os.path.join(HERE, "train.npz"))))


if __name__ == "__main__":
    main()

"""Generates tests/golden/train_multi_pose.npz with the UNMODIFIED MultiPoseDataset.__getitem__ of the reference
(datasets/sample/multi_pose.py:29-183, color_aug and get_affine_transform of utils/image.py; cv2 from this image)
-- build container only.

Each case of tests/multi_pose_train_cases.py is a dataset over seeded images written as lossless PNGs to a
temporary directory, with make_golden_train.py's stub `coco`; np.random, random and the dataset's _data_rng are
seeded per case.  Stored per sample: c and s from meta (opt.debug = 1); rot and flip replayed from the saved
np.random state; the three matrices (trans_input, trans_output_rot, trans_output) recomputed with the reference's
get_affine_transform from those draws; the shuffle order, blend and lighting draws; CRCs of the three generator
states after the sample; the CRC and a strided sample of `input`; every target; and `hm` / `hm_hp` for the first
samples of each case."""
import os
import random
import sys
import tempfile
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_train as MG  # noqa: E402  (puts the reference and tests/ on sys.path)
import cv2  # noqa: E402
import importlib.util  # noqa: E402
_spec = importlib.util.spec_from_file_location("ref_multi_pose",
                                               os.path.join(MG.REF, "datasets", "sample", "multi_pose.py"))
_mp = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_mp)
MultiPoseDataset = _mp.MultiPoseDataset
from utils.image import get_affine_transform  # noqa: E402

import multi_pose_train_cases as MC  # noqa: E402

TARGETS = ('reg_mask', 'ind', 'wh', 'hps', 'hps_mask', 'reg', 'hp_offset', 'hp_ind', 'hp_mask')


def replay_rot_flip(ds, np_state, opt, height, width):
    """The rotation and flip draws of the sample that started from np_state (np.random is restored after)."""
    saved = np.random.get_state()
    np.random.set_state(np_state)
    if not opt.not_rand_crop:
        wb, hb = ds._get_border(128, width), ds._get_border(128, height)
        np.random.choice(np.arange(0.6, 1.4, 0.1))
        np.random.randint(low=wb, high=width - wb); np.random.randint(low=hb, high=height - hb)
    else:
        np.random.randn(); np.random.randn(); np.random.randn()
    rot = 0
    if np.random.random() < opt.aug_rot:
        rf = opt.rotate
        rot = np.clip(np.random.randn() * rf, -rf * 2, rf * 2)
    flip = np.random.random() < opt.flip
    np.random.set_state(saved)
    return rot, flip


def run_case(name, case, tmp, out):
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(tmp, files[i]), MC.case_image(name, i))
        anns[i] = MC.case_anns(name, i)
    rec = MG.RecordingRng(np.random.RandomState(case['seed']))
    ds = MultiPoseDataset.__new__(MultiPoseDataset)
    for k, v in MC.case_dataset(name, MG.StubCOCO(files, anns), tmp, rec).items():
        setattr(ds, k, v)
    opt = ds.opt
    np.random.seed(case['seed']); random.seed(case['seed'])
    res, out_res = opt.input_res, opt.output_res
    for i in range(len(files)):
        p = "%s_%d_" % (name, i)
        np_state, py_state = np.random.get_state(), random.getstate()
        rec.log = []
        h, w = case['sizes'][i]
        ret = ds.__getitem__(i)
        out[p + "states"] = MG.state_crcs(rec.rng)
        c = np.asarray(ret['meta']['c'], np.float32)
        s = ret['meta']['s']
        assert not isinstance(s, np.ndarray)
        out[p + "c"], out[p + "s"] = c, np.float64(s)
        rot, flip = replay_rot_flip(ds, np_state, opt, h, w)
        out[p + "rot"], out[p + "flip"] = np.float64(rot), np.bool_(flip)
        out[p + "trans_input"] = get_affine_transform(c, s, rot, [res, res])
        out[p + "trans_output_rot"] = get_affine_transform(c, s, rot, [out_res, out_res])
        out[p + "trans_output"] = get_affine_transform(c, s, 0, [out_res, out_res])
        color = not opt.no_color_aug
        out[p + "order"] = np.int32(MG.replay_order(py_state) if color else -1)
        blend, light = np.zeros(6, np.float32), np.zeros(3, np.float64)
        if color:
            for kind, (_, alpha) in zip(MC.ORDERS[int(out[p + "order"])], rec.log[:3]):
                alpha = 1. + alpha
                blend[2 * kind], blend[2 * kind + 1] = np.float32(alpha), np.float32(1 - alpha)
            light = np.dot(MC.EIG_VEC, MC.EIG_VAL * rec.log[3][1])
        out[p + "blend"], out[p + "light"] = blend, light
        inp = np.ascontiguousarray(ret['input'], np.float32)
        out[p + "input_crc"] = np.uint32(zlib.crc32(inp.view(np.uint8)))
        out[p + "input_shape"] = np.array(inp.shape, np.int64)
        out[p + "input_sample"] = inp[:, ::17, ::13].copy()
        for k in TARGETS:
            if k in ret:
                out[p + k] = ret[k]
        if i < case['hm_samples']:
            out[p + "hm"] = ret['hm']
            if 'hm_hp' in ret:
                out[p + "hm_hp"] = ret['hm_hp']


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, case in MC.CASES.items():
            run_case(name, case, tmp, out)
    path = os.path.join(HERE, "train_multi_pose.npz")
    np.savez_compressed(path, **out)
    rots = {n: [bool(out["%s_%d_rot" % (n, i)] != 0) for i in range(len(c['sizes']))] for n, c in MC.CASES.items()}
    print("wrote train_multi_pose.npz: %d arrays, %d bytes; rotated %s" % (len(out), os.path.getsize(path), rots))


if __name__ == "__main__":
    main()

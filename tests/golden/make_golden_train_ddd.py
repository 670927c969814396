"""Generates tests/golden/train_ddd.npz with the UNMODIFIED DddDataset.__getitem__ of the reference
(datasets/sample/ddd.py:27-157, get_affine_transform and gaussian_radius of utils/image.py; cv2 from this image) --
build container only.

Each case of tests/ddd_train_cases.py is a dataset over seeded images written as lossless PNGs to a temporary
directory, with make_golden_train.py's stub `coco` and ds.calib set; np.random, random and the dataset's _data_rng
are seeded per case.  Stored per sample: c and s from meta (opt.debug = 1); the augmentation draw replayed from the
saved np.random state; trans_input and trans_output recomputed with the reference's get_affine_transform; CRCs of
the three generator states after the sample; the CRC and a strided sample of `input`; every target and `hm`.
Also the radius table: the reference's gaussian_radius((h, w)) on the float32 pairs of ddd_train_cases.radius_pairs
(the CRCs of the float32 radii and of the int(radius) values, which the tests recompute from the pairs) and on
pairs found by search whose radius lies within a few ulp of an integer (each base pair and the float32 radii of it
and its neighbours, ddd_train_cases.near_pairs).  The script asserts that the cases reach the edges the
sampler branches on."""
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
import types  # noqa: E402
try:
    import pycocotools.coco  # noqa: E402,F401
except ImportError:   # the sampler imports it but reads annotations only through ds.coco (the stub here)
    sys.modules['pycocotools'] = types.ModuleType('pycocotools')
    sys.modules['pycocotools.coco'] = sys.modules['pycocotools'].coco = types.ModuleType('pycocotools.coco')
_spec = importlib.util.spec_from_file_location("ref_ddd", os.path.join(MG.REF, "datasets", "sample", "ddd.py"))
_ddd = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_ddd)
DddDataset = _ddd.DddDataset
from utils.image import gaussian_radius, get_affine_transform  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))   # the repository, for oracle/
import ddd_train_cases as DC  # noqa: E402

TARGETS = ('hm', 'dep', 'dim', 'ind', 'rotbin', 'rotres', 'reg_mask', 'rot_mask', 'wh', 'reg')
F32 = np.float32


def replay_aug(np_state, opt, split):
    saved = np.random.get_state()
    np.random.set_state(np_state)
    aug = split == 'train' and np.random.random() < opt.aug_ddd
    np.random.set_state(saved)
    return aug


def src1_f32_centre(c, s):
    """src[1] of get_affine_transform with the centre rounded to float32 before the float64 addition."""
    return F32(np.float64(F32(c[1])) + np.float64(s[0]) * -0.5)


def run_case(name, case, tmp, out, cover):
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(tmp, files[i]), DC.case_image(name, i))
        anns[i] = DC.case_anns(name, i)
    rec = MG.RecordingRng(np.random.RandomState(case['seed']))
    ds = DddDataset.__new__(DddDataset)
    for k, v in DC.case_dataset(name, MG.StubCOCO(files, anns), tmp, rec).items():
        setattr(ds, k, v)
    opt = ds.opt
    np.random.seed(case['seed']); random.seed(case['seed'])
    for i in range(len(files)):
        p = "%s_%d_" % (name, i)
        np_state = np.random.get_state()
        ret = ds.__getitem__(i)
        out[p + "states"] = MG.state_crcs(rec.rng)
        c, s = ret['meta']['c'], ret['meta']['s']
        assert c.dtype == np.float64
        out[p + "c"], out[p + "s"] = c, s
        aug = replay_aug(np_state, opt, case['split'])
        out[p + "aug"] = np.bool_(aug)
        out[p + "trans_input"] = get_affine_transform(c, s, 0, [opt.input_w, opt.input_h])
        out[p + "trans_output"] = get_affine_transform(c, s, 0, [opt.output_w, opt.output_h])
        if aug:
            cover['aug'] += 1
            cover['src1_differs'] += src1_f32_centre(c, s) != F32(c[1] + np.float64(s[0]) * -0.5)
        inp = np.ascontiguousarray(ret['input'], np.float32)
        out[p + "input_crc"] = np.uint32(zlib.crc32(inp.view(np.uint8)))
        out[p + "input_shape"] = np.array(inp.shape, np.int64)
        out[p + "input_sample"] = DC.input_sample(inp).copy()
        for k in TARGETS:
            if k in ret:
                out[p + k] = ret[k]
        cover_sample(name, i, out, p, cover)


def cover_sample(name, i, out, p, cover):
    """Counts the edges this sample reaches, from its objects and the reference's own trans_output."""
    import train_ddd_np as DN
    import train_np as TN
    case = DC.CASES[name]
    opt = DC.make_opt(case)
    boxes, cls, _, _, _ = DC.case_objects(name, i)
    t = out[p + "trans_output"]
    peaks, rects = [], []
    for k in range(len(boxes)):
        c = int(cls[k])
        if c <= -99:
            cover['skip99'] += 1
            continue
        x0, y0 = TN.affine_f32(t, boxes[k][0], boxes[k][1])
        x1, y1 = TN.affine_f32(t, boxes[k][2], boxes[k][3])
        x0, x1 = [F32(min(max(v, F32(0)), F32(opt.output_w - 1))) for v in (x0, x1)]
        y0, y1 = [F32(min(max(v, F32(0)), F32(opt.output_h - 1))) for v in (y0, y1)]
        h, w = F32(y1 - y0), F32(x1 - x0)
        if not h > 0:
            cover['h_le_0'] += 1
        if not (h > 0 and w > 0):
            continue
        ci = np.array([(x0 + x1) / F32(2), (y0 + y1) / F32(2)], F32).astype(np.int32)
        rad = max(0, int(DN.gaussian_radius_f32(h, w)))
        cl = set(range(case['num_classes'])) if c == -1 else {-c - 2} if c < 0 else {c}
        if c < 0:
            cover['ignore_all' if c == -1 else 'ignore_one'] += 1
            if case['rect_mask']:
                box = (int(x0), int(y0), int(x1), int(y1))
                for (px, py, pr, pc) in peaks:   # a positive drawn before, inside the rectangle's reach
                    if pc in cl and box[0] - pr <= px <= box[2] + pr and box[1] - pr <= py <= box[3] + pr:
                        cover['pos_before_rect'] += 1
                rects.append((box, cl))
            else:
                cover['ignore_on_peak'] += any(pc in cl and (px, py) == tuple(ci) for px, py, _, pc in peaks)
            continue
        for box, rc in rects:
            if c in rc and box[0] <= ci[0] <= box[2] and box[1] <= ci[1] <= box[3]:
                cover['pos_after_rect'] += 1
        peaks.append((int(ci[0]), int(ci[1]), rad, c))


def radius_table(out):
    h, w = DC.radius_pairs()
    ref = np.array([gaussian_radius((a, b)) for a, b in zip(h, w)], F32)
    out["radius_crc"] = np.uint32(zlib.crc32(ref.tobytes()))
    out["radius_int_crc"] = np.uint32(zlib.crc32(np.maximum(ref.astype(np.int64), 0).astype(np.int16).tobytes()))
    # pairs whose radius lies within a few ulp of an integer: bisect w for radius == k; the table keeps the base
    # pair and the radii of its neighbours (ddd_train_cases.near_pairs)
    r = np.random.default_rng(815)
    h0, w0 = [], []
    for _ in range(6000):
        hh = F32(r.choice([r.uniform(0.05, 4), r.uniform(1, 96)]))
        top = int(gaussian_radius((hh, F32(4000))))   # the radius grows with w up to about this
        if top < 1:
            continue
        k = float(r.integers(1, top + 1))
        lo, hi = 0.0, 4000.0
        for _ in range(60):
            mid = (lo + hi) / 2
            if float(gaussian_radius((hh, F32(mid)))) < k:
                lo = mid
            else:
                hi = mid
        x = F32(hi)
        if abs(float(gaussian_radius((hh, x))) - k) > 1e-4:   # k out of reach for this h
            continue
        h0.append(hh); w0.append(x)
    h0, w0 = np.array(h0, F32), np.array(w0, F32)
    hs, ws = DC.near_pairs(h0, w0)
    assert (ws > 0).all()
    rs = np.array([gaussian_radius((a, b)) for a, b in zip(hs, ws)], F32)
    near = np.abs(rs - np.round(rs)) < 1e-4
    print("near-integer search: %d pairs, %d within 1e-4 of an integer" % (len(rs), near.sum()))
    assert len(rs) > 10000 and near.mean() > 0.95
    out["radius_near_h0"], out["radius_near_w0"], out["radius_near"] = h0, w0, rs
    return len(h), len(rs)


def main():
    out = {}
    cover = dict.fromkeys(('aug', 'src1_differs', 'skip99', 'h_le_0', 'ignore_all', 'ignore_one', 'pos_before_rect',
                           'pos_after_rect', 'ignore_on_peak'), 0)
    with tempfile.TemporaryDirectory() as tmp:
        for name, case in DC.CASES.items():
            run_case(name, case, tmp, out, cover)
    n_rand, n_near = radius_table(out)
    print("coverage", cover)
    for k, v in cover.items():
        assert v > 0, "the cases do not reach %s" % k
    path = os.path.join(HERE, "train_ddd.npz")
    np.savez_compressed(path, **out)
    print("wrote train_ddd.npz: %d arrays, %d bytes; radius table %d random + %d near-integer pairs"
          % (len(out), os.path.getsize(path), n_rand, n_near))


if __name__ == "__main__":
    main()

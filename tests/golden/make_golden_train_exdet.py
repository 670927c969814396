"""Generates tests/golden/train_exdet.npz with the UNMODIFIED EXDetDataset.__getitem__ of the reference
(datasets/sample/exdet.py:30-137, color_aug, get_affine_transform and draw_umich_gaussian of utils/image.py; cv2 from
this image) -- build container only.

Each case of tests/exdet_train_cases.py is a dataset over seeded images written as lossless PNGs to a temporary
directory, with make_golden_train.py's stub `coco`; np.random, random and the dataset's _data_rng are seeded per
case.  exdet returns no meta, so c, s and the flip are replayed from the saved np.random state (the sampler's own
lines) and the shuffle order from the saved random state; trans_input and trans_output are recomputed from them with
the reference's get_affine_transform.  Stored per sample: those draws, the blend and lighting draws, CRCs of the
three generator states after the sample, the CRC and a strided sample of `input`, every target and, for the first
samples of each case, the five heat maps.  The script asserts that the cases reach the edges the sampler branches
on."""
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
_spec = importlib.util.spec_from_file_location("ref_exdet", os.path.join(MG.REF, "datasets", "sample", "exdet.py"))
_ex = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_ex)
EXDetDataset = _ex.EXDetDataset
from utils.image import gaussian_radius, get_affine_transform  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))   # the repository, for oracle/
import exdet_train_cases as EC  # noqa: E402
import train_exdet_np as EN  # noqa: E402

PARTS = ('t', 'l', 'b', 'r')
TARGETS = ('reg_mask',) + tuple('reg_' + p for p in PARTS) + tuple('ind_' + p for p in PARTS)
MAPS = tuple('hm_' + p for p in PARTS + ('c',))
F32 = np.float32


def replay_draws(ds, np_state, opt, split, height, width):
    """c, s and the flip of the sample that started from np_state: exdet.py:37-56 (np.random restored after)."""
    saved = np.random.get_state()
    np.random.set_state(np_state)
    c = np.array([width / 2., height / 2.])
    s = max(height, width) * 1.0
    flipped = False
    if split == 'train':
        if not opt.not_rand_crop:
            s = s * np.random.choice(np.arange(0.6, 1.4, 0.1))
            w_border, h_border = ds._get_border(128, width), ds._get_border(128, height)
            c[0] = np.random.randint(low=w_border, high=width - w_border)
            c[1] = np.random.randint(low=h_border, high=height - h_border)
        else:
            sf, cf = opt.scale, opt.shift
            s = s * np.clip(np.random.randn() * sf + 1, 1 - sf, 1 + sf)
            c[0] += width * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
            c[1] += height * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
        flipped = np.random.random() < opt.flip
    np.random.set_state(saved)
    return c, s, flipped


def src1_f32_centre(c, s):
    """src[1] of get_affine_transform with the centre rounded to float32 before the float64 addition."""
    return F32(np.float64(F32(c[1])) + np.float64(F32(s)) * -0.5)


def run_case(name, case, tmp, out, cover):
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(tmp, files[i]), EC.case_image(name, i))
        anns[i] = EC.case_anns(name, i)
    rec = MG.RecordingRng(np.random.RandomState(case['seed']))
    ds = EXDetDataset.__new__(EXDetDataset)
    for k, v in EC.case_dataset(name, MG.StubCOCO(files, anns), tmp, rec).items():
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
        c, s, flip = replay_draws(ds, np_state, opt, case['split'], h, w)
        assert c.dtype == np.float64
        out[p + "c"], out[p + "s"], out[p + "flip"] = c, np.float64(s), np.bool_(flip)
        out[p + "trans_input"] = get_affine_transform(c, s, 0, [res, res])
        out[p + "trans_output"] = get_affine_transform(c, s, 0, [out_res, out_res])
        color = case['split'] == 'train' and not opt.no_color_aug
        out[p + "order"] = np.int32(MG.replay_order(py_state) if color else -1)
        blend, light = np.zeros(6, F32), np.zeros(3, np.float64)
        if color:
            for kind, (_, alpha) in zip(EC.ORDERS[int(out[p + "order"])], rec.log[:3]):
                alpha = 1. + alpha
                blend[2 * kind], blend[2 * kind + 1] = F32(alpha), F32(1 - alpha)
            light = np.dot(EC.EIG_VEC, EC.EIG_VAL * rec.log[3][1])
        out[p + "blend"], out[p + "light"] = blend, light
        if case['not_rand_crop'] and case['split'] == 'train':
            cover['src1_differs'] += src1_f32_centre(c, s) != F32(c[1] + np.float64(F32(s)) * -0.5)
        inp = np.ascontiguousarray(ret['input'], F32)
        out[p + "input_crc"] = np.uint32(zlib.crc32(inp.view(np.uint8)))
        out[p + "input_shape"] = np.array(inp.shape, np.int64)
        out[p + "input_sample"] = EC.input_sample(inp).copy()
        for k in TARGETS:
            if k in ret:
                out[p + k] = ret[k]
        if i < case['hm_samples']:
            for k in MAPS:
                out[p + k] = ret[k]
        cover_sample(name, i, out, p, flip, cover)


def cover_sample(name, i, out, p, flip, cover):
    """Counts the edges this sample reaches, from its objects and the reference's own trans_output and maps."""
    case = EC.CASES[name]
    R = case['input_res'] // case['down_ratio']
    pts, cls = EC.case_objects(name, i)
    width = case['sizes'][i][1]
    seen, centres = {}, []
    for k in range(len(pts)):
        raw, q = EN.exdet_points(pts[k], flip, width, out[p + "trans_output"], R)
        hh, ww = F32(q[2, 1] - q[0, 1]), F32(q[3, 0] - q[1, 0])
        cover['h_le_0'] += not hh > 0
        cover['w_le_0'] += not ww > 0
        if not (hh > 0 and ww > 0):
            continue
        cover['clip_lo'] += bool((raw < 0).any())
        cover['clip_hi'] += bool((raw > R - 1).any())
        rad = max(0, int(gaussian_radius((int(np.ceil(hh)), int(np.ceil(ww))))))
        cover['radius_0'] += rad == 0
        qi = [tuple(v) for v in q.astype(np.int32)]
        cover['coincident_in_object'] += len(set(qi)) < 4
        for j in range(4):
            key = (j, 0 if case['agnostic_ex'] else int(cls[k]), qi[j])
            cover['coincident_across_objects'] += key in seen
            seen[key] = k
        ct = (int(F32(q[3, 0] + q[1, 0]) / F32(2)), int(F32(q[0, 1] + q[2, 1]) / F32(2)))
        for (cx, cy, cr, cc) in centres:
            if cc == int(cls[k]) and abs(cx - ct[0]) <= cr + rad and abs(cy - ct[1]) <= cr + rad:
                cover['overlap_same_class'] += 1
        centres.append((ct[0], ct[1], rad, int(cls[k])))
        if flip and pts[k][1, 0] != pts[k][3, 0]:
            cover['flip_swap'] += 1


def main():
    out = {}
    cover = dict.fromkeys(('src1_differs', 'h_le_0', 'w_le_0', 'clip_lo', 'clip_hi', 'radius_0',
                           'coincident_in_object', 'coincident_across_objects', 'overlap_same_class', 'flip_swap'),
                          0)
    with tempfile.TemporaryDirectory() as tmp:
        for name, case in EC.CASES.items():
            run_case(name, case, tmp, out, cover)
    print("coverage", cover)
    for k, v in cover.items():
        assert v > 0, "the cases do not reach %s" % k
    path = os.path.join(HERE, "train_exdet.npz")
    np.savez_compressed(path, **out)
    print("wrote train_exdet.npz: %d arrays, %d bytes" % (len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()

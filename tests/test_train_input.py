"""Training input of the ctdet sampler (centernet_b200.train_input), CPU side.  tests/golden/train.npz holds what
the UNMODIFIED CTDetDataset.__getitem__ returned for the seeded cases of tests/train_cases.py: the numpy
restatement (tests/train_np.py) must reproduce it bit for bit from the recorded draws, and the wrapper's draws
must equal the recorded ones and leave np.random, random and _data_rng in the recorded states."""
import os
import random
import zlib

import numpy as np
import pytest
import torch

import train_cases as TC
import train_np as TN
from helpers import golden
from oracle import image_np

from centernet_b200 import train_input as T
from centernet_b200._lib import C

SAMPLES = [(n, i) for n, c in TC.CASES.items() if 'rot' not in c for i in range(len(c['sizes']))]


def _input_size(case, h, w):
    if case['keep_res']:
        return (h | case['pad']) + 1, (w | case['pad']) + 1
    return case['input_h'], case['input_w']


def _scale(g, p):
    s = g[p + "s"]
    return s.astype(np.float64) if g[p + "s_is_array"] else np.float64(s[0])


def _boxes(name, i, case):
    anns = TC.case_anns(name, i)[:case['max_objs']]
    ids = TC.cat_ids(case)
    boxes = np.array([[a['bbox'][0], a['bbox'][1], a['bbox'][0] + a['bbox'][2], a['bbox'][1] + a['bbox'][3]]
                      for a in anns], np.float32).reshape(-1, 4)
    return boxes, np.array([ids[a['category_id']] for a in anns], np.int32)


def _check_input(x, g, p):
    x = np.ascontiguousarray(x, np.float32)
    assert tuple(x.shape) == tuple(g[p + "input_shape"])
    np.testing.assert_array_equal(x[:, ::17, ::13], g[p + "input_sample"])
    assert np.uint32(zlib.crc32(x.view(np.uint8))) == g[p + "input_crc"]


def oracle_sample(name, i, g):
    """The oracle's input and targets for golden sample (name, i) from its recorded draws."""
    case = TC.CASES[name]
    p = "%s_%d_" % (name, i)
    h, w = case['sizes'][i]
    ih, iw = _input_size(case, h, w)
    oh, ow = ih // case['down_ratio'], iw // case['down_ratio']
    c, s = g[p + "c"], _scale(g, p)
    x = TN.train_image(TC.case_image(name, i), T.affine_transform(c, s, [iw, ih]), bool(g[p + "flip"]), iw, ih,
                       TC.MEAN, TC.STD, int(g[p + "order"]), g[p + "blend"], g[p + "light"])
    boxes, cls = _boxes(name, i, case)
    t = TN.ctdet_targets(boxes, cls, bool(g[p + "flip"]), w, T.affine_transform(c, s, [ow, oh]), case['max_objs'],
                         case['num_classes'], oh, ow)
    return x, t, (oh, ow)


@pytest.mark.parametrize("name,i", SAMPLES)
def test_oracle_matches_golden(name, i):
    g = golden("train")
    case = TC.CASES[name]
    p = "%s_%d_" % (name, i)
    x, t, (oh, ow) = oracle_sample(name, i, g)
    _check_input(x, g, p)
    keys = ['reg_mask', 'ind'] + (['cat_spec_wh', 'cat_spec_mask'] if case['cat_spec_wh'] else ['wh'])
    for k in keys + (['reg'] if case['reg_offset'] else []):
        np.testing.assert_array_equal(t[k], g[p + k], err_msg=k)
    if p + "hm" in g:
        lists = [t[k][None] for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid')]
        np.testing.assert_array_equal(image_np.splat_objects(*lists, case['num_classes'], oh, ow)[0], g[p + "hm"])


@pytest.mark.parametrize("name", [n for n, c in TC.CASES.items() if 'rot' in c])
def test_oracle_rotated_warp_matches_golden(name):
    g = golden("train")
    case = TC.CASES[name]
    p = name + "_0_"
    x = TN.train_image(TC.case_image(name, 0), g[p + "matrix"], False, case['out'], case['out'], TC.MEAN, TC.STD,
                       int(g[p + "order"]), g[p + "blend"], g[p + "light"])
    _check_input(x, g, p)


def _state_crcs(data_rng):
    k, pos = np.random.get_state()[1:3]
    c_np = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    c_py = zlib.crc32(np.asarray(random.getstate()[1], np.uint64).tobytes())
    k, pos = data_rng.get_state()[1:3]
    c_dr = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    return np.array([c_np, c_py, c_dr], np.uint32)


@pytest.mark.parametrize("name", [n for n, c in TC.CASES.items() if 'rot' not in c])
def test_wrapper_draws_match_reference(name):
    g = golden("train")
    case = TC.CASES[name]
    opt = TC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(case['seed']); random.seed(case['seed'])
        data_rng = np.random.RandomState(case['seed'])
        for i, (h, w) in enumerate(case['sizes']):
            p = "%s_%d_" % (name, i)
            d = T.sample_params(h, w, opt, case['split'], data_rng, TC.EIG_VAL, TC.EIG_VEC)
            np.testing.assert_array_equal(_state_crcs(data_rng), g[p + "states"])
            np.testing.assert_array_equal(d['c'], g[p + "c"])
            s = d['s'] if isinstance(d['s'], np.ndarray) else [d['s'], d['s']]
            np.testing.assert_array_equal(np.asarray(s, np.float64), g[p + "s"])
            assert isinstance(d['s'], np.ndarray) == bool(g[p + "s_is_array"])
            assert d['flip'] == bool(g[p + "flip"]) and d['order'] == int(g[p + "order"])
            np.testing.assert_array_equal(d['blend'], g[p + "blend"])
            np.testing.assert_array_equal(d['light'], g[p + "light"])
            assert (d['input_h'], d['input_w']) == _input_size(case, h, w)
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


class _StubCOCO(object):
    def __init__(self, files, anns):
        self.files, self.anns = files, anns

    def loadImgs(self, ids):
        return [{'file_name': self.files[ids[0]]}]

    def getAnnIds(self, imgIds):
        return [(imgIds[0], k) for k in range(len(self.anns[imgIds[0]]))]

    def loadAnns(self, ids):
        return [self.anns[i][k] for i, k in ids]


def make_dataset(name, tmpdir):
    """A duck-typed CTDetDataset over the case's images written as PNGs (needs cv2)."""
    import cv2
    import types
    case = TC.CASES[name]
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(str(tmpdir), files[i]), TC.case_image(name, i))
        anns[i] = TC.case_anns(name, i)
    return types.SimpleNamespace(
        opt=TC.make_opt(case), coco=_StubCOCO(files, anns), images=list(range(len(files))), img_dir=str(tmpdir),
        max_objs=case['max_objs'], cat_ids=TC.cat_ids(case), num_classes=case['num_classes'],
        mean=TC.MEAN.reshape(1, 1, 3), std=TC.STD.reshape(1, 1, 3), _data_rng=np.random.RandomState(case['seed']),
        _eig_val=TC.EIG_VAL, _eig_vec=TC.EIG_VEC, split=case["split"])


def test_dataset_wrapper_reads_and_draws_like_reference(tmp_path):
    pytest.importorskip("cv2")
    g = golden("train")
    name = "crop"
    ds = make_dataset(name, tmp_path)
    w = T.CTDetTrainInput(ds)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(TC.CASES[name]['seed']); random.seed(TC.CASES[name]['seed'])
        for i in range(len(TC.CASES[name]['sizes'])):
            p = "%s_%d_" % (name, i)
            s = w[i]
            np.testing.assert_array_equal(s['image'], TC.case_image(name, i))
            np.testing.assert_array_equal(_state_crcs(ds._data_rng), g[p + "states"])
            np.testing.assert_array_equal(s['c'], g[p + "c"])
            boxes, cls = _boxes(name, i, TC.CASES[name])
            np.testing.assert_array_equal(s['boxes'], boxes)
            np.testing.assert_array_equal(s['cls'], cls)
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


def test_pairwise_mean_and_grey_restatements():
    rng = np.random.default_rng(5)
    for shape in ((512, 512), (384, 511), (97, 130), (128, 128), (1, 1), (3, 2), (7, 9), (1, 129), (131, 3)):
        a = rng.random(shape, dtype=np.float32)
        assert TN.grey_mean(a) == a.mean(), shape
    cv2 = pytest.importorskip("cv2")
    x = rng.integers(0, 256, (200, 333, 3)).astype(np.float32) / np.float32(255)
    np.testing.assert_array_equal(TN.grey(x), cv2.cvtColor(x, cv2.COLOR_BGR2GRAY))


def test_radius_in_device_order_matches_reference_radius():
    for h in range(1, 260):
        for w in range(1, 260):
            assert TN.gaussian_radius_ops(h, w) == image_np.gaussian_radius((h, w)), (h, w)


def test_train_images_abi_validation():
    p = 16

    def call(src=p, order=p, blend=p, light=p, mean=p, b=2, oh=64, ow=64, dt=0, cl=0, ws=p, wsb=1 << 20):
        return C.train_images(src, p, p, p, p, order, blend, light, mean, p, b, oh, ow, p, dt, cl, ws, wsb, 0)

    for kw, code in ((dict(src=0), 1), (dict(mean=0), 1), (dict(blend=0), 1), (dict(b=0), 1), (dict(oh=0), 1),
                     (dict(ow=-3), 1), (dict(dt=3), 1), (dict(cl=2), 1), (dict(ws=0), 1), (dict(wsb=4), 4)):
        with pytest.raises(RuntimeError, match="status %d" % code):
            call(**kw)
    with pytest.raises(NotImplementedError):
        call(oh=4096, ow=1025)
    assert C.train_images_workspace_bytes(0, 64, 64) == 0
    assert C.train_images_workspace_bytes(3, 512, 512) == 3 * 8 * 4   # 2048 leaves, 8 subtrees of 256 per image


def test_ctdet_targets_abi_validation():
    p = 16

    def call(boxes=p, csw=0, csm=0, b=2, m=8, nc=80, oh=128, ow=128, valid=p):
        return C.ctdet_targets(boxes, p, p, p, p, p, b, m, nc, oh, ow, p, p, p, p, csw, csm, p, p, p, p, valid, 0)

    for kw in (dict(boxes=0), dict(valid=0), dict(csw=p), dict(csm=p), dict(b=0), dict(m=0), dict(nc=0),
               dict(oh=0)):
        with pytest.raises(RuntimeError, match="status 1"):
            call(**kw)


def test_python_validation_before_any_copy(tmp_path):
    img = np.zeros((8, 8, 3), np.uint8)
    eye = np.array([[1., 0, 0], [0, 1., 0]])
    cuda = torch.device("cuda", 0)
    with pytest.raises(ValueError):
        T.augment_images([img], [eye], 8, 8, TC.MEAN, TC.STD, orders=[6], device=cuda)
    with pytest.raises(ValueError):
        T.augment_images([img[..., :2]], [eye], 8, 8, TC.MEAN, TC.STD, device=cuda)
    with pytest.raises(NotImplementedError):
        T.augment_images([np.zeros((32768, 1, 3), np.uint8)], [eye], 8, 8, TC.MEAN, TC.STD, device=cuda)
    a = dict(image=img, input_h=64, input_w=64)
    with pytest.raises(ValueError, match="different input sizes"):
        T.collate_ctdet([a, dict(a, input_w=96)])
    import types
    for flag in ("mse_loss", "dense_wh"):
        opt = TC.make_opt(TC.CASES["crop"])
        setattr(opt, flag, True)
        with pytest.raises(NotImplementedError):
            T.CTDetTrainInput(types.SimpleNamespace(opt=opt))

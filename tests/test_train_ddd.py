"""Training input of the ddd sampler (centernet_b200.train_input), CPU side.
tests/golden/train_ddd.npz holds what the UNMODIFIED DddDataset.__getitem__ returned for the seeded cases of
tests/ddd_train_cases.py: the wrapper's draws and matrices must equal the recorded ones and leave np.random, random
and _data_rng in the recorded states, and the numpy restatement (tests/train_ddd_np.py for the targets and hm,
tests/train_np.py for the image) must reproduce every target, hm and input bit for bit."""
import os
import random
import types
import zlib

import numpy as np
import pytest

import ddd_train_cases as DC
import train_ddd_np as DN
import train_np as TN
from helpers import assert_bits, golden, state_crcs, StubCOCO

from centernet_b200 import train_input as T
from centernet_b200._lib import C

SAMPLES = [(n, i) for n, c in DC.CASES.items() for i in range(len(c['sizes']))]
TARGETS = ('hm', 'dep', 'dim', 'ind', 'rotbin', 'rotres', 'reg_mask', 'rot_mask', 'wh', 'reg')


@pytest.mark.parametrize("name", list(DC.CASES))
def test_wrapper_draws_and_matrices_match_reference(name):
    g = golden("train_ddd")
    case = DC.CASES[name]
    opt = DC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(case['seed']); random.seed(case['seed'])
        data_rng = np.random.RandomState(case['seed'])
        for i, (h, w) in enumerate(case['sizes']):
            p = "%s_%d_" % (name, i)
            d = T.ddd_params(h, w, opt, case['split'])
            np.testing.assert_array_equal(state_crcs(data_rng), g[p + "states"], err_msg=p)
            assert_bits(d['c'], g[p + "c"], p + "c")
            assert_bits(d['s'], g[p + "s"], p + "s")
            assert d['aug'] == bool(g[p + "aug"]), p
            assert_bits(d['trans_output'].reshape(2, 3), g[p + "trans_output"], p + "trans_output")
            assert_bits(T.affine_transform(d['c'], d['s'], [d['input_w'], d['input_h']]), g[p + "trans_input"],
                  p + "trans_input")
            assert_bits(d['minv'], np.array(T._invert(g[p + "trans_input"]), np.float64), p + "minv")
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


@pytest.mark.parametrize("name,i", SAMPLES)
def test_oracle_matches_golden(name, i):
    g = golden("train_ddd")
    case = DC.CASES[name]
    opt = DC.make_opt(case)
    p = "%s_%d_" % (name, i)
    x = TN.train_image(DC.case_image(name, i), g[p + "trans_input"], False, opt.input_w, opt.input_h, DC.MEAN,
                       DC.STD)
    assert tuple(x.shape) == tuple(g[p + "input_shape"])
    np.testing.assert_array_equal(DC.input_sample(x), g[p + "input_sample"])
    assert np.uint32(zlib.crc32(np.ascontiguousarray(x, np.float32).view(np.uint8))) == g[p + "input_crc"]
    boxes, cls, alpha, depth, dim = DC.case_objects(name, i)
    t = DN.ddd_targets(boxes, cls, alpha, depth, dim, bool(g[p + "aug"]), g[p + "trans_output"], case['max_objs'],
                       case['num_classes'], opt.output_h, opt.output_w, case['rect_mask'])
    keys = [k for k in TARGETS if p + k in g]
    assert set(keys) == set(TARGETS) - ({'wh'} if not case['reg_bbox'] else set()) \
        - ({'reg'} if not case['reg_offset'] else set())
    for k in keys:
        assert_bits(t[k], g[p + k], p + k)


def test_radius_restatement_matches_reference_table():
    """The float32 restatement of gaussian_radius((h, w)) against the reference's values: the CRCs of the float32
    radii and of int(radius) over every random pair, and every near-integer pair to the bit."""
    g = golden("train_ddd")
    h, w = DC.radius_pairs()
    r = DN.gaussian_radius_f32(h, w)
    assert np.uint32(zlib.crc32(r.tobytes())) == g["radius_crc"]
    assert np.uint32(zlib.crc32(np.maximum(r.astype(np.int64), 0).astype(np.int16).tobytes())) == g["radius_int_crc"]
    assert_bits(DN.gaussian_radius_f32(*DC.near_pairs(g["radius_near_h0"], g["radius_near_w0"])), g["radius_near"],
          "near-integer radii")


def test_radius_square_is_the_c_library_power():
    """b ** 2 of a float32 scalar is not always the rounded b * b, and the table holds pairs whose int(radius)
    depends on it: a restatement squaring with b * b fails there."""
    g = golden("train_ddd")
    b = np.random.default_rng(5).uniform(0, 400, 20000).astype(np.float32)
    assert any(np.float32(v) ** 2 != np.float32(np.float64(v) * np.float64(v)) for v in b)
    h, w = DC.near_pairs(g["radius_near_h0"], g["radius_near_w0"])
    exact = DN.gaussian_radius_f32(h, w, square=lambda v: (v.astype(np.float64) ** 2).astype(np.float32))
    assert (exact.astype(np.int64) != g["radius_near"].astype(np.int64)).any()


def test_centre_enters_src1_as_given():
    """ctdet / multi_pose matrices (float32 centres, scalar or float32 / float64 scales) are the bits of the
    float32-centre formula; ddd's float64 centre is added without a float32 rounding first."""
    from centernet_b200.post_process import _affine_points, cv_affine_transform

    def f32_centre(center, scale, size):
        if not isinstance(scale, np.ndarray):
            scale = np.array([scale, scale], dtype=np.float32)
        src, dst = _affine_points(center, scale.astype(np.float32), size)
        src[1, 1] = np.float32(np.float64(np.float32(center[1])) + np.float64(scale[0]) * -0.5)
        d = src[0] - src[1]
        src[2] = src[1] + np.array([-d[1], d[0]], np.float32)
        return cv_affine_transform(src, dst)

    rng = np.random.default_rng(3)
    for _ in range(300):
        c = rng.uniform(-50, 1500, 2).astype(np.float32)
        s = np.float64(rng.uniform(5, 2000))
        if rng.random() < 0.3:
            s = np.array([rng.integers(32, 1300), rng.integers(32, 1300)], np.float32) * rng.choice(
                np.arange(0.6, 1.4, 0.1))
        size = [int(rng.integers(16, 1025)), int(rng.integers(16, 1025))]
        assert_bits(T.affine_transform(c, s, size), f32_centre(c, s, size), "float32 centre")
    g = golden("train_ddd")
    differs = 0
    for name, i in SAMPLES:
        p = "%s_%d_" % (name, i)
        opt = DC.make_opt(DC.CASES[name])
        c, s, size = g[p + "c"], g[p + "s"], [opt.output_w, opt.output_h]
        assert_bits(T.affine_transform(c, s, size), g[p + "trans_output"], p + "trans_output")
        differs += not np.array_equal(f32_centre(c, s, size), g[p + "trans_output"])
    assert differs > 0


@pytest.mark.parametrize("name", ["kitti", "keep"])
def test_dataset_wrapper_reads_and_draws_like_reference(tmp_path, name):
    cv2 = pytest.importorskip("cv2")
    g = golden("train_ddd")
    case = DC.CASES[name]
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(str(tmp_path), files[i]), DC.case_image(name, i))
        anns[i] = DC.case_anns(name, i)
    ds = types.SimpleNamespace(**DC.case_dataset(name, StubCOCO(files, anns), str(tmp_path),
                                                 np.random.RandomState(case['seed'])))
    w = T.DddTrainInput(ds)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(case['seed']); random.seed(case['seed'])
        for i in range(len(case['sizes'])):
            p = "%s_%d_" % (name, i)
            s = w[i]
            np.testing.assert_array_equal(s['image'], DC.case_image(name, i))
            np.testing.assert_array_equal(state_crcs(ds._data_rng), g[p + "states"])
            assert_bits(s['c'], g[p + "c"], p + "c")
            assert s['aug'] == bool(g[p + "aug"])
            boxes, cls, alpha, depth, dim = DC.case_objects(name, i)
            assert_bits(s['boxes'], boxes, p + "boxes")
            assert_bits(s['cls'], cls, p + "cls")
            assert_bits(s['alpha'], alpha, p + "alpha")
            assert_bits(s['depth'], depth, p + "depth")
            assert_bits(np.array(s['dim']).reshape(-1, 3), dim, p + "dim")
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


def test_ddd_targets_abi_validation():
    p = 16

    def call(boxes=p, alpha=p, aug=p, hm=p, reg=p, b=2, m=8, nc=3, oh=96, ow=320, rect=0):
        return C.ddd_targets(boxes, p, p, alpha, p, p, aug, p, b, m, nc, oh, ow, rect, hm, p, p, p, p, p, p, p, p, reg,
                             0)

    for kw in (dict(boxes=0), dict(alpha=0), dict(aug=0), dict(hm=0), dict(reg=0), dict(b=0), dict(m=0), dict(nc=0),
               dict(oh=0), dict(ow=-4), dict(rect=2), dict(b=1 << 16)):
        with pytest.raises(RuntimeError, match="status 1"):
            call(**kw)
    with pytest.raises(NotImplementedError, match="status 2"):
        call(m=129)
    for kw in (dict(h=0), dict(n=0)):
        a = dict(h=p, n=4)
        a.update(kw)
        with pytest.raises(RuntimeError, match="status 1"):
            C.ddd_gaussian_radius(a['h'], p, a['n'], p, 0)


def _sample(**kw):
    s = dict(image=np.zeros((40, 90, 3), np.uint8), boxes=np.array([[2, 3, 12, 20]], np.float32),
             cls=np.array([0]), alpha=np.array([0.3]), depth=np.array([12.5]), dim=[np.array([1.5, 1.6, 3.9])],
             aug=False, input_h=32, input_w=96, output_h=8, output_w=24, max_objs=50, num_classes=3,
             rect_mask=False, reg_bbox=True, reg_offset=True,
             minv=np.array(T._invert(np.array([[1., 0, 0], [0, 1., 0]]))), trans_output=np.zeros(6),
             mean=DC.MEAN, std=DC.STD)
    s.update(kw)
    return s


def test_collate_rejects_what_the_reference_cannot_run():
    T.collate_ddd([_sample(), _sample(aug=True)])   # accepted as is
    for c in (-1000, -99, -1, -2, -4, 0, 2):          # skipped, all classes, class 0 / 2 ignores, positives
        T.collate_ddd([_sample(cls=np.array([c]))])
    for c in (3, -5, -98):
        with pytest.raises(ValueError, match="class id"):
            T.collate_ddd([_sample(), _sample(cls=np.array([c]))])
    for d in ([np.array([1.5, 1.6])], [np.zeros(4)]):
        with pytest.raises(ValueError, match="dim"):
            T.collate_ddd([_sample(dim=d)])
    for m in (0, 129):
        with pytest.raises(ValueError, match="object slots"):
            T.collate_ddd([_sample(max_objs=m)])
    with pytest.raises(ValueError, match="different settings"):
        T.collate_ddd([_sample(), _sample(rect_mask=True)])
    # only the slots the reference reads are checked
    T.collate_ddd([_sample(max_objs=1, boxes=np.zeros((2, 4), np.float32), cls=np.array([0, 7]),
                           alpha=np.zeros(2), depth=np.zeros(2), dim=[np.zeros(3), np.zeros(2)])])


def test_mse_loss_is_rejected():
    opt = DC.make_opt(DC.CASES["kitti"])
    opt.mse_loss = True
    with pytest.raises(NotImplementedError):
        T.DddTrainInput(types.SimpleNamespace(opt=opt))

"""Training input of the exdet sampler (centernet_b200.train_input), CPU side.
tests/golden/train_exdet.npz holds what the UNMODIFIED EXDetDataset.__getitem__ returned for the seeded cases of
tests/exdet_train_cases.py: the wrapper's draws and matrices must equal the recorded ones and leave np.random, random
and _data_rng in the recorded states, and the numpy restatement (tests/train_exdet_np.py for the targets and maps,
tests/train_np.py for the image) must reproduce every target, heat map and input bit for bit."""
import os
import random
import types
import zlib

import numpy as np
import pytest

import exdet_train_cases as EC
import train_exdet_np as EN
import train_np as TN
from helpers import golden

from centernet_b200 import train_input as T
from centernet_b200._lib import C

SAMPLES = [(n, i) for n, c in EC.CASES.items() for i in range(len(c['sizes']))]
PARTS = ('t', 'l', 'b', 'r')
TARGETS = ('reg_mask',) + tuple('reg_' + p for p in PARTS) + tuple('ind_' + p for p in PARTS)
MAPS = tuple('hm_' + p for p in PARTS + ('c',))


def _state_crcs(data_rng):
    k, pos = np.random.get_state()[1:3]
    c_np = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    c_py = zlib.crc32(np.asarray(random.getstate()[1], np.uint64).tobytes())
    k, pos = data_rng.get_state()[1:3]
    c_dr = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    return np.array([c_np, c_py, c_dr], np.uint32)


def _bits(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, a.shape, b.dtype, b.shape)
    assert a.tobytes() == b.tobytes(), what


@pytest.mark.parametrize("name", list(EC.CASES))
def test_wrapper_draws_and_matrices_match_reference(name):
    g = golden("train_exdet")
    case = EC.CASES[name]
    opt = EC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(case['seed']); random.seed(case['seed'])
        data_rng = np.random.RandomState(case['seed'])
        for i, (h, w) in enumerate(case['sizes']):
            p = "%s_%d_" % (name, i)
            d = T.exdet_params(h, w, opt, case['split'], data_rng, EC.EIG_VAL, EC.EIG_VEC)
            np.testing.assert_array_equal(_state_crcs(data_rng), g[p + "states"], err_msg=p)
            _bits(d['c'], g[p + "c"], p + "c")
            _bits(np.float64(d['s']), g[p + "s"], p + "s")
            assert d['flip'] == bool(g[p + "flip"]) and d['order'] == int(g[p + "order"]), p
            _bits(d['blend'], g[p + "blend"], p + "blend")
            _bits(d['light'], g[p + "light"], p + "light")
            _bits(d['trans_output'].reshape(2, 3), g[p + "trans_output"], p + "trans_output")
            _bits(T.affine_transform(d['c'], d['s'], [d['input_res']] * 2), g[p + "trans_input"], p + "trans_input")
            _bits(d['minv'], np.array(T._invert(g[p + "trans_input"]), np.float64), p + "minv")
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


def test_float64_centre_reaches_src1_unrounded():
    """Under not_rand_crop the centre is off the integers; rounding it to float32 before get_affine_transform's
    float64 sum would change src[1] of some sample, and the matrices still match the golden."""
    g = golden("train_exdet")
    differs = 0
    for i in range(len(EC.CASES["ex_shift"]['sizes'])):
        p = "ex_shift_%d_" % i
        c, s = g[p + "c"], g[p + "s"][()]
        assert c.dtype == np.float64
        r = EC.make_opt(EC.CASES["ex_shift"]).output_res
        _bits(T.affine_transform(c, s, [r, r]), g[p + "trans_output"], p)
        differs += not np.array_equal(T.affine_transform(c.astype(np.float32), s, [r, r]), g[p + "trans_output"])
    assert differs > 0


@pytest.mark.parametrize("name,i", SAMPLES)
def test_oracle_matches_golden(name, i):
    g = golden("train_exdet")
    case = EC.CASES[name]
    p = "%s_%d_" % (name, i)
    res, r = case['input_res'], case['input_res'] // case['down_ratio']
    x = TN.train_image(EC.case_image(name, i), g[p + "trans_input"], bool(g[p + "flip"]), res, res, EC.MEAN, EC.STD,
                       int(g[p + "order"]), g[p + "blend"], g[p + "light"])
    assert tuple(x.shape) == tuple(g[p + "input_shape"])
    np.testing.assert_array_equal(EC.input_sample(x), g[p + "input_sample"])
    assert np.uint32(zlib.crc32(np.ascontiguousarray(x, np.float32).view(np.uint8))) == g[p + "input_crc"]
    pts, cls = EC.case_objects(name, i)
    t = EN.exdet_targets(pts, cls, bool(g[p + "flip"]), case['sizes'][i][1], g[p + "trans_output"],
                         case['max_objs'], r, case['agnostic_ex'])
    keys = [k for k in TARGETS if p + k in g]
    assert set(keys) == (set(TARGETS) if case['reg_offset'] else set())
    for k in keys:
        _bits(t[k], g[p + k], p + k)
    if i < case['hm_samples']:
        maps = EN.exdet_maps(t, case['num_classes'], r, case['agnostic_ex'])
        for k in MAPS:
            _bits(maps[k], g[p + k], p + k)
        assert g[p + "hm_t"].shape[0] == (1 if case['agnostic_ex'] else case['num_classes'])


class _StubCOCO(object):
    def __init__(self, files, anns):
        self.files, self.anns = files, anns

    def loadImgs(self, ids):
        return [{'file_name': self.files[ids[0]]}]

    def getAnnIds(self, imgIds):
        return [(imgIds[0], k) for k in range(len(self.anns[imgIds[0]]))]

    def loadAnns(self, ids):
        return [self.anns[i][k] for i, k in ids]


@pytest.mark.parametrize("name", ["ex_flip", "ex_plain"])
def test_dataset_wrapper_reads_and_draws_like_reference(tmp_path, name):
    cv2 = pytest.importorskip("cv2")
    g = golden("train_exdet")
    case = EC.CASES[name]
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(str(tmp_path), files[i]), EC.case_image(name, i))
        anns[i] = EC.case_anns(name, i)
    ds = types.SimpleNamespace(**EC.case_dataset(name, _StubCOCO(files, anns), str(tmp_path),
                                                 np.random.RandomState(case['seed'])))
    w = T.ExdetTrainInput(ds)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(case['seed']); random.seed(case['seed'])
        for i in range(len(case['sizes'])):
            p = "%s_%d_" % (name, i)
            s = w[i]
            np.testing.assert_array_equal(s['image'], EC.case_image(name, i))
            np.testing.assert_array_equal(_state_crcs(ds._data_rng), g[p + "states"])
            _bits(s['c'], g[p + "c"], p + "c")
            assert s['flip'] == bool(g[p + "flip"])
            pts, cls = EC.case_objects(name, i)
            _bits(np.array(s['points']).reshape(-1, 4, 2), pts, p + "points")
            _bits(s['cls'], cls, p + "cls")
            assert (s['num_classes'], s['agnostic_ex'], s['reg_offset']) == \
                (case['num_classes'], case['agnostic_ex'], case['reg_offset'])
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


def test_exdet_targets_abi_validation():
    p = 16

    def call(pts=p, flip=p, reg=p, ind=p, oval=p, ecls=p, eval_=p, b=2, m=8, res=128, agn=0):
        return C.exdet_targets(pts, p, p, flip, p, p, b, m, res, agn, reg, ind, p, p, p, p, p, oval, ecls, p, p, p,
                               eval_, 0)

    for kw in (dict(pts=0), dict(flip=0), dict(reg=0), dict(ind=0), dict(oval=0), dict(ecls=0), dict(eval_=0),
               dict(b=0), dict(m=0), dict(res=0), dict(res=-4), dict(res=1 << 16), dict(agn=2)):
        with pytest.raises(RuntimeError, match="status 1"):
            call(**kw)
    with pytest.raises(NotImplementedError, match="status 2"):
        call(m=129)


def _sample(**kw):
    s = dict(image=np.zeros((40, 30, 3), np.uint8),
             points=[np.array([6, 3, 2, 10, 7, 20, 12, 9], np.float32)], cls=np.array([0]), flip=False,
             input_res=64, output_res=16, max_objs=32, num_classes=2, agnostic_ex=False, reg_offset=True,
             minv=np.array(T._invert(np.array([[1., 0, 0], [0, 1., 0]]))), trans_output=np.zeros(6), order=-1,
             blend=np.zeros(6, np.float32), light=np.zeros(3), mean=EC.MEAN, std=EC.STD)
    s.update(kw)
    return s


def test_collate_rejects_what_the_kernel_cannot_match():
    T.collate_exdet([_sample(), _sample(flip=True, cls=np.array([1]))])   # accepted as is
    good = np.array([6, 3, 2, 10, 7, 20, 12, 9], np.float32)
    bad = [
        ("extreme_points has 6", dict(points=[good[:6]])),
        ("extreme_points has 10", dict(points=[np.zeros(10, np.float32)])),
        ("class id", dict(cls=np.array([2]))),
        ("class id", dict(cls=np.array([-1]))),
        ("finite", dict(points=[np.where(np.arange(8) == 0, np.nan, good).astype(np.float32)])),
        ("finite", dict(points=[np.where(np.arange(8) == 5, np.inf, good).astype(np.float32)])),
        ("finite", dict(points=[np.where(np.arange(8) == 2, -np.inf, good).astype(np.float32)])),
    ]
    for what, kw in bad:
        with pytest.raises(ValueError, match=what):
            T.collate_exdet([_sample(), _sample(**kw)])
    for m in (0, 129):
        with pytest.raises(ValueError, match="object slots"):
            T.collate_exdet([_sample(max_objs=m)])
    for k, v in (('input_res', 128), ('output_res', 32), ('max_objs', 8), ('num_classes', 3), ('agnostic_ex', True),
                 ('reg_offset', False)):
        with pytest.raises(ValueError, match="different settings"):
            T.collate_exdet([_sample(), _sample(**{k: v})])
    # only the slots the reference reads are checked
    T.collate_exdet([_sample(max_objs=1, points=[good, np.full(3, np.nan, np.float32)], cls=np.array([0, 9]))])


def test_collate_packs_points_classes_and_flips():
    good = np.array([6, 3, 2, 10, 7, 20, 12, 9], np.float32)
    packed = T.collate_exdet([_sample(), _sample(flip=True, points=[good, good + 1], cls=np.array([1, 0]))])
    v = T._views(packed['buffer'], packed['layout'])
    assert v['pts'].shape == (2, 32, 4, 2) and v['cls'].shape == (2, 32)
    np.testing.assert_array_equal(v['pts'][1, :2].numpy(), np.stack([good, good + 1]).reshape(2, 4, 2))
    np.testing.assert_array_equal(v['nobj'].numpy(), [1, 2])
    np.testing.assert_array_equal(v['flip'].numpy(), [0, 1])
    assert packed['scalars']['batch'] == 2 and not packed['scalars']['color']


def test_mse_loss_is_rejected():
    opt = EC.make_opt(EC.CASES["ex_coco"])
    opt.mse_loss = True
    with pytest.raises(NotImplementedError):
        T.ExdetTrainInput(types.SimpleNamespace(opt=opt))

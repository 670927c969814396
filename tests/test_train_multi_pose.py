"""Training input of the multi_pose sampler (centernet_b200.train_input), CPU side.
tests/golden/train_multi_pose.npz holds what the UNMODIFIED MultiPoseDataset.__getitem__ returned for the seeded
cases of tests/multi_pose_train_cases.py: the wrapper's draws and matrices must equal the recorded ones and leave
np.random, random and _data_rng in the recorded states, and the numpy restatement (tests/train_multi_pose_np.py for
the targets, tests/train_np.py for the image) must reproduce every target, hm, hm_hp and input bit for bit."""
import os
import random
import types
import zlib

import numpy as np
import pytest

import multi_pose_train_cases as MC
import train_multi_pose_np as MN
import train_np as TN
from helpers import golden

from centernet_b200 import train_input as T
from centernet_b200._lib import C

SAMPLES = [(n, i) for n, c in MC.CASES.items() for i in range(len(c['sizes']))]
TARGETS = ('reg_mask', 'ind', 'wh', 'hps', 'hps_mask', 'reg', 'hp_offset', 'hp_ind', 'hp_mask')


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


@pytest.mark.parametrize("name", list(MC.CASES))
def test_wrapper_draws_and_matrices_match_reference(name):
    g = golden("train_multi_pose")
    case = MC.CASES[name]
    opt = MC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(case['seed']); random.seed(case['seed'])
        data_rng = np.random.RandomState(case['seed'])
        for i, (h, w) in enumerate(case['sizes']):
            p = "%s_%d_" % (name, i)
            d = T.multi_pose_params(h, w, opt, case['split'], data_rng, MC.EIG_VAL, MC.EIG_VEC)
            np.testing.assert_array_equal(_state_crcs(data_rng), g[p + "states"], err_msg=p)
            _bits(d['c'], g[p + "c"], p + "c")
            _bits(np.float64(d['s']), g[p + "s"], p + "s")
            _bits(np.float64(d['rot']), g[p + "rot"], p + "rot")
            assert d['flip'] == bool(g[p + "flip"]) and d['order'] == int(g[p + "order"]), p
            _bits(d['blend'], g[p + "blend"], p + "blend")
            _bits(d['light'], g[p + "light"], p + "light")
            _bits(d['trans_output_rot'].reshape(2, 3), g[p + "trans_output_rot"], p + "trans_output_rot")
            _bits(d['trans_output'].reshape(2, 3), g[p + "trans_output"], p + "trans_output")
            _bits(d['minv'], np.array(T._invert(g[p + "trans_input"]), np.float64), p + "minv")
            _bits(T.affine_transform(d['c'], d['s'], [d['input_res']] * 2, d['rot']), g[p + "trans_input"],
                  p + "trans_input")
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


def test_cases_cover_the_edges():
    """The golden cases reach what the issue's semantics branch on."""
    g = golden("train_multi_pose")
    rot = [g["%s_%d_rot" % s] != 0 for s in SAMPLES]
    assert any(rot) and not all(rot)
    vis = np.concatenate([k.reshape(-1, 3)[:, 2] for n, i in SAMPLES for k in MC.case_objects(n, i)[2]])
    assert set(np.unique(vis).tolist()) == {0.0, 1.0, 2.0}
    no_kpt = small_neg = zero_rot = 0
    for name, i in SAMPLES:
        p = "%s_%d_" % (name, i)
        case = MC.CASES[name]
        boxes, cls, kps = MC.case_objects(name, i)
        r = case['input_res'] // case['down_ratio']
        for k in range(len(boxes)):
            pts = kps[k].reshape(-1, 3)
            if not (pts[:, 2] != 0).any() and g[p + "ind"][k] != 0:
                no_kpt += 1
            if g[p + "rot"] != 0 and (boxes[k, 2] == boxes[k, 0] or boxes[k, 3] == boxes[k, 1]):
                zero_rot += g[p + "ind"][k] != 0
            if g[p + "flip"]:
                continue
            for x, y, v in pts:
                if v > 0:
                    px, py = TN.affine_f32(g[p + "trans_output_rot"], x, y)
                    small_neg += (-1 < px < 0 and 0 <= py < r) or (-1 < py < 0 and 0 <= px < r)
    assert no_kpt > 0 and small_neg > 0 and zero_rot > 0, (no_kpt, small_neg, zero_rot)


def test_rotated_matrices_match_train_golden_and_unrotated_are_unchanged():
    """get_affine_transform(rot != 0) against the rotated cases of tests/golden/train.npz; rot = 0 against the
    unrotated formula the ctdet sampler used before rotation was supported."""
    import train_cases as TC
    g = golden("train")
    for name in ("rot", "rot2"):
        case = TC.CASES[name]
        h, w = case['sizes'][0]
        c = np.array([w / 2., h / 2.], np.float32)
        _bits(T.affine_transform(c, max(h, w) * case['scale'], [case['out']] * 2, case['rot']),
              g[name + "_0_matrix"], name)
    from centernet_b200.post_process import _affine_points, cv_affine_transform

    def unrotated(center, scale, size):
        if not isinstance(scale, np.ndarray):
            scale = np.array([scale, scale], dtype=np.float32)
        src, dst = _affine_points(center, scale.astype(np.float32), size)
        src[1, 1] = np.float32(np.float64(np.float32(center[1])) + np.float64(scale[0]) * -0.5)
        d = src[0] - src[1]
        src[2] = src[1] + np.array([-d[1], d[0]], np.float32)
        return cv_affine_transform(src, dst)

    rng = np.random.default_rng(3)
    for _ in range(300):
        c = (rng.uniform(-50, 1500, 2)).astype(np.float32)
        s = np.float64(rng.uniform(5, 2000))
        if rng.random() < 0.3:
            s = np.array([rng.integers(32, 1300), rng.integers(32, 1300)], np.float32) * rng.choice(
                np.arange(0.6, 1.4, 0.1))
        size = [int(rng.integers(16, 1025)), int(rng.integers(16, 1025))]
        _bits(T.affine_transform(c, s, size), unrotated(c, s, size), "rot 0")


@pytest.mark.parametrize("name,i", SAMPLES)
def test_oracle_matches_golden(name, i):
    g = golden("train_multi_pose")
    case = MC.CASES[name]
    p = "%s_%d_" % (name, i)
    res, r = case['input_res'], case['input_res'] // case['down_ratio']
    x = TN.train_image(MC.case_image(name, i), g[p + "trans_input"], bool(g[p + "flip"]), res, res, MC.MEAN,
                       MC.STD, int(g[p + "order"]), g[p + "blend"], g[p + "light"])
    assert tuple(x.shape) == tuple(g[p + "input_shape"])
    np.testing.assert_array_equal(x[:, ::17, ::13], g[p + "input_sample"])
    assert np.uint32(zlib.crc32(np.ascontiguousarray(x, np.float32).view(np.uint8))) == g[p + "input_crc"]
    boxes, cls, kps = MC.case_objects(name, i)
    nj = case['num_joints']
    rotated = bool(g[p + "rot"] != 0)
    t = MN.multi_pose_targets(boxes, cls, [k.reshape(nj, 3) for k in kps], bool(g[p + "flip"]),
                              case['sizes'][i][1], T.flip_permutation(nj, case['flip_idx']), rotated,
                              g[p + "trans_output"], g[p + "trans_output_rot"], case['max_objs'], r)
    keys = [k for k in TARGETS if p + k in g]
    assert set(keys) == set(TARGETS) - ({'reg'} if not case['reg_offset'] else set()) \
        - ({'hp_offset', 'hp_ind', 'hp_mask'} if not case['reg_hp_offset'] else set())
    for k in keys:
        _bits(t[k], g[p + k], p + k)
    if p + "hm" in g:
        hm, hm_hp = MN.multi_pose_maps(t, case['num_classes'], r, rotated)
        _bits(hm, g[p + "hm"], p + "hm")
        if p + "hm_hp" in g:
            _bits(hm_hp, g[p + "hm_hp"], p + "hm_hp")


class _StubCOCO(object):
    def __init__(self, files, anns):
        self.files, self.anns = files, anns

    def loadImgs(self, ids):
        return [{'file_name': self.files[ids[0]]}]

    def getAnnIds(self, imgIds):
        return [(imgIds[0], k) for k in range(len(self.anns[imgIds[0]]))]

    def loadAnns(self, ids):
        return [self.anns[i][k] for i, k in ids]


def test_dataset_wrapper_reads_and_draws_like_reference(tmp_path):
    cv2 = pytest.importorskip("cv2")
    g = golden("train_multi_pose")
    name = "mp_small"
    case = MC.CASES[name]
    files, anns = {}, {}
    for i in range(len(case['sizes'])):
        files[i] = "%s_%d.png" % (name, i)
        cv2.imwrite(os.path.join(str(tmp_path), files[i]), MC.case_image(name, i))
        anns[i] = MC.case_anns(name, i)
    ds = types.SimpleNamespace(**MC.case_dataset(name, _StubCOCO(files, anns), str(tmp_path),
                                                 np.random.RandomState(case['seed'])))
    w = T.MultiPoseTrainInput(ds)
    saved = np.random.get_state(), random.getstate()
    try:
        np.random.seed(case['seed']); random.seed(case['seed'])
        for i in range(len(case['sizes'])):
            p = "%s_%d_" % (name, i)
            s = w[i]
            np.testing.assert_array_equal(s['image'], MC.case_image(name, i))
            np.testing.assert_array_equal(_state_crcs(ds._data_rng), g[p + "states"])
            _bits(s['c'], g[p + "c"], p + "c")
            boxes, cls, kps = MC.case_objects(name, i)
            _bits(s['boxes'], boxes, p + "boxes")
            _bits(s['cls'], cls, p + "cls")
            for a, b in zip(s['keypoints'], kps):
                _bits(a, b, p + "keypoints")
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])


def test_flip_permutation_composes_swaps_in_order():
    np.testing.assert_array_equal(T.flip_permutation(5, [[1, 2], [2, 3], [0, 4], [3, 1]]), [4, 1, 3, 2, 0])
    pts = np.arange(5)
    for a, b in [[1, 2], [2, 3], [0, 4], [3, 1]]:
        pts[a], pts[b] = pts[b].copy(), pts[a].copy()
    np.testing.assert_array_equal(T.flip_permutation(5, [[1, 2], [2, 3], [0, 4], [3, 1]]), pts)
    np.testing.assert_array_equal(T.flip_permutation(17, MC.COCO_FLIP_IDX),
                                  [0, 2, 1, 4, 3, 6, 5, 8, 7, 10, 9, 12, 11, 14, 13, 16, 15])


def test_multi_pose_targets_abi_validation():
    p = 16

    def call(boxes=p, kps=p, rotated=p, perm=p, hp_mask=p, hval=p, b=2, m=8, nj=17, res=128):
        return C.multi_pose_targets(boxes, p, p, kps, p, rotated, p, p, p, perm, b, m, nj, res, p, p, p, p, p, p, p,
                                    p, hp_mask, p, p, p, p, p, p, p, p, hval, 0)

    for kw in (dict(boxes=0), dict(kps=0), dict(rotated=0), dict(perm=0), dict(hp_mask=0), dict(hval=0),
               dict(b=0), dict(m=0), dict(nj=0), dict(res=0), dict(res=-4), dict(b=1 << 16, m=128, nj=1024)):
        with pytest.raises(RuntimeError, match="status 1"):
            call(**kw)


def _sample(**kw):
    s = dict(image=np.zeros((40, 30, 3), np.uint8), boxes=np.array([[2, 3, 12, 20]], np.float32),
             cls=np.array([0]), keypoints=[np.tile(np.array([5, 6, 2], np.float32), 17)], rot=0, flip=False,
             input_res=64, output_res=16, max_objs=32, num_classes=1, num_joints=17,
             flip_idx=[tuple(e) for e in MC.COCO_FLIP_IDX], reg_offset=True, hm_hp=True, reg_hp_offset=True,
             minv=np.array(T._invert(np.array([[1., 0, 0], [0, 1., 0]]))), trans_output=np.zeros(6),
             trans_output_rot=np.zeros(6), order=-1, blend=np.zeros(6, np.float32), light=np.zeros(3),
             mean=MC.MEAN, std=MC.STD)
    s.update(kw)
    return s


def test_collate_rejects_what_the_kernel_cannot_match():
    T.collate_multi_pose([_sample(), _sample(rot=12.5)])   # accepted as is
    k = np.tile(np.array([5, 6, 2], np.float32), 17)
    bad = [
        ("keypoint values", dict(keypoints=[k[:-3]])),
        ("visibilities", dict(keypoints=[np.where(np.arange(51) == 2, -1, k).astype(np.float32)])),
        ("visibilities", dict(keypoints=[np.where(np.arange(51) == 5, np.nan, k).astype(np.float32)])),
        ("visibilities", dict(keypoints=[np.where(np.arange(51) == 8, np.inf, k).astype(np.float32)])),
        ("class id", dict(cls=np.array([1]))),
        ("class id", dict(cls=np.array([-1]))),
        ("negative width", dict(rot=-3.0, boxes=np.array([[12, 3, 2, 20]], np.float32))),
        ("negative width", dict(rot=7.0, boxes=np.array([[2, 30, 12, 20]], np.float32))),
    ]
    for what, kw in bad:
        with pytest.raises(ValueError, match=what):
            T.collate_multi_pose([_sample(), _sample(**kw)])
    with pytest.raises(ValueError, match="object slots"):
        T.collate_multi_pose([_sample(max_objs=129)])
    # only the slots the reference reads are checked; an unrotated negative side is the reference's empty box
    T.collate_multi_pose([_sample(max_objs=1, boxes=np.zeros((2, 4), np.float32), cls=np.array([0, 5]),
                                  keypoints=[k, k[:3]])])
    T.collate_multi_pose([_sample(boxes=np.array([[12, 3, 2, 20]], np.float32))])
    with pytest.raises(ValueError, match="different settings"):
        T.collate_multi_pose([_sample(), _sample(num_joints=5)])


def test_rotated_sample_needs_dense_hm_and_options_are_checked():
    packed = T.collate_multi_pose([_sample(), _sample(rot=3.0)])
    with pytest.raises(ValueError, match="dense_hm=True"):
        T.build_multi_pose_batch(packed)
    for flag in ("mse_loss", "dense_hp"):
        opt = MC.make_opt(MC.CASES["mp_coco"])
        setattr(opt, flag, True)
        with pytest.raises(NotImplementedError):
            T.MultiPoseTrainInput(types.SimpleNamespace(opt=opt))

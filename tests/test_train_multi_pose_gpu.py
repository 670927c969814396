"""Training input of the multi_pose sampler on the H100 (centernet_b200.train_input): the device batch against
tests/golden/train_multi_pose.npz and the numpy restatements (tests/train_np.py, tests/train_multi_pose_np.py) bit
for bit -- input in fp32 and bf16 / fp16 (the fp32 value rounded once), NCHW and channels_last, every target with
the reference's dtype, dense hm / hm_hp including the rotated 0.9999 maps -- and the trainer's losses on it."""
import functools
import random

import numpy as np
import pytest
import torch

import multi_pose_train_cases as MC
import train_multi_pose_np as MN
import train_np as TN
from helpers import assert_bits, golden

pytestmark = pytest.mark.gpu

DTYPES = (torch.float32, torch.bfloat16, torch.float16)
FORMATS = (torch.contiguous_format, torch.channels_last)
TARGETS = ('reg_mask', 'ind', 'wh', 'hps', 'hps_mask', 'reg', 'hp_offset', 'hp_ind', 'hp_mask')
LISTS = ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid')
HP_LISTS = ('hp_cx', 'hp_cy', 'hp_radius', 'hp_valid')


def case_samples(name):
    """The case's samples as MultiPoseTrainInput returns them, drawn from the golden seeds (no image files)."""
    from centernet_b200 import train_input as T
    case = MC.CASES[name]
    opt = MC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    np.random.seed(case['seed']); random.seed(case['seed'])
    data_rng = np.random.RandomState(case['seed'])
    out = []
    try:
        for i, (h, w) in enumerate(case['sizes']):
            s = T.multi_pose_params(h, w, opt, case['split'], data_rng, MC.EIG_VAL, MC.EIG_VEC)
            boxes, cls, kps = MC.case_objects(name, i)
            s.update(image=MC.case_image(name, i), boxes=boxes, cls=cls, keypoints=kps, max_objs=case['max_objs'],
                     num_classes=case['num_classes'], num_joints=case['num_joints'],
                     flip_idx=[tuple(e) for e in case['flip_idx']], mean=MC.MEAN, std=MC.STD,
                     reg_offset=case['reg_offset'], hm_hp=case['hm_hp'], reg_hp_offset=case['reg_hp_offset'])
            out.append(s)
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])
    return out


def restated(s):
    """tests/train_multi_pose_np.py's targets and maps for one sample."""
    from centernet_b200 import train_input as T
    nj, r = s['num_joints'], s['output_res']
    t = MN.multi_pose_targets(s['boxes'], s['cls'], [k.reshape(nj, 3) for k in s['keypoints']], s['flip'],
                              s['image'].shape[1], T.flip_permutation(nj, s['flip_idx']), s['rot'] != 0,
                              s['trans_output'], s['trans_output_rot'], s['max_objs'], r)
    t['hm'], t['hm_hp'] = MN.multi_pose_maps(t, s['num_classes'], r, s['rot'] != 0)
    return t


@functools.lru_cache(maxsize=None)
def oracle_inputs(name):
    from centernet_b200 import train_input as T
    out = []
    for s in case_samples(name):
        m = T.affine_transform(s['c'], s['s'], [s['input_res']] * 2, s['rot'])
        out.append(TN.train_image(s['image'], m, s['flip'], s['input_res'], s['input_res'], MC.MEAN, MC.STD,
                                  s['order'], s['blend'], s['light']))
    return np.stack(out)


def _expected_keys(case):
    keys = {'input', 'hm', 'reg_mask', 'ind', 'wh', 'hps', 'hps_mask'} | set(LISTS)
    keys |= {'reg'} if case['reg_offset'] else set()
    keys |= ({'hm_hp'} | set(HP_LISTS)) if case['hm_hp'] else set()
    keys |= {'hp_offset', 'hp_ind', 'hp_mask'} if case['reg_hp_offset'] else set()
    return keys


@pytest.mark.parametrize("name", list(MC.CASES))
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_multi_pose_batch_matches_reference(name, dtype, fmt):
    from centernet_b200 import train_input as T
    g = golden("train_multi_pose")
    case = MC.CASES[name]
    samples = case_samples(name)
    packed = T.collate_multi_pose(samples)
    host = packed['buffer'].clone()
    batch = T.build_multi_pose_batch(packed, dtype=dtype, memory_format=fmt, dense_hm=True)
    torch.cuda.synchronize()
    assert torch.equal(packed['buffer'], host), "the packed host buffer was modified"
    assert set(batch) == _expected_keys(case)
    inp = batch['input']
    assert inp.dtype == dtype and inp.is_contiguous(memory_format=fmt)
    got = inp.float().cpu().numpy()
    want = torch.from_numpy(oracle_inputs(name)).to(dtype).float().numpy()
    assert_bits(got, want, "%s input %s" % (name, dtype))
    r = case['input_res'] // case['down_ratio']
    for i, s in enumerate(samples):
        p = "%s_%d_" % (name, i)
        if dtype == torch.float32:
            np.testing.assert_array_equal(got[i][:, ::17, ::13], g[p + "input_sample"])
        for k in TARGETS:
            if k in batch:
                assert_bits(batch[k][i].cpu().numpy(), g[p + k], p + k)
        t = restated(s)
        for k in LISTS + (HP_LISTS if case['hm_hp'] else ()):
            assert_bits(batch[k][i].cpu().numpy(), t[k], p + k)
        assert_bits(batch['hm'][i].cpu().numpy(), t['hm'], p + "hm")
        assert tuple(batch['hm'].shape[1:]) == (case['num_classes'], r, r)
        if case['hm_hp']:
            assert_bits(batch['hm_hp'][i].cpu().numpy(), t['hm_hp'], p + "hm_hp")
        if p + "hm" in g:
            assert_bits(batch['hm'][i].cpu().numpy(), g[p + "hm"], p + "hm golden")
        if p + "hm_hp" in g:
            assert_bits(batch['hm_hp'][i].cpu().numpy(), g[p + "hm_hp"], p + "hm_hp golden")
        if s['rot'] != 0:
            assert (batch['hm'][i] == np.float32(0.9999).item()).all()


def test_multi_pose_batch_bit_identical_run_to_run():
    from centernet_b200 import train_input as T
    packed = T.collate_multi_pose(case_samples("mp_shift"))
    a = T.build_multi_pose_batch(packed, dense_hm=True)
    b = T.build_multi_pose_batch(packed, dense_hm=True)
    torch.cuda.synchronize()
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _golden_hm_samples(g, name):
    """Indices of the case's unrotated samples whose hm (and hm_hp) the golden holds."""
    return [i for i in range(len(MC.CASES[name]['sizes']))
            if "%s_%d_hm" % (name, i) in g and g["%s_%d_rot" % (name, i)] == 0]


def test_focal_splat_loss_on_both_list_sets():
    """FocalSplatLoss on the centre lists equals FocalLoss on the reference's hm; on the [B*J, 1, R, R] view of
    the joint lists it equals FocalLoss on hm_hp."""
    from centernet_b200 import losses as L
    from centernet_b200 import train_input as T
    g = golden("train_multi_pose")
    rng = np.random.default_rng(1)
    checked = 0
    for name in MC.CASES:
        case = MC.CASES[name]
        batch = T.build_multi_pose_batch(T.collate_multi_pose(case_samples(name)), dense_hm=True)
        for i in _golden_hm_samples(g, name):
            p = "%s_%d_" % (name, i)
            hm = torch.from_numpy(g[p + "hm"][None]).cuda()
            pred = torch.from_numpy(np.clip(rng.random(hm.shape, dtype=np.float32), 1e-4, 1 - 1e-4)).cuda()
            lf = L.FocalSplatLoss()(pred, *[batch[k][i:i + 1] for k in LISTS])
            np.testing.assert_allclose(lf.item(), L.FocalLoss()(pred, hm).item(), rtol=1e-6, err_msg=p + "hm")
            checked += 1
            if not case['hm_hp']:
                continue
            nj, m = case['num_joints'], case['max_objs']
            hp = torch.from_numpy(g[p + "hm_hp"]).cuda().view(nj, 1, *g[p + "hm_hp"].shape[1:])
            pred = torch.from_numpy(np.clip(rng.random(hp.shape, dtype=np.float32), 1e-4, 1 - 1e-4)).cuda()
            lists = [batch[k][i].reshape(nj, m) for k in HP_LISTS]
            lf = L.FocalSplatLoss()(pred, torch.zeros_like(lists[0]), *lists)
            np.testing.assert_allclose(lf.item(), L.FocalLoss()(pred, hp).item(), rtol=1e-6, err_msg=p + "hm_hp")
    assert checked >= 5


def _trainer_losses(out, batch, opt):
    """trains/multi_pose.py:57-80's composition (hm_weight, wh_weight 0.1, off_weight, hp_weight, hm_hp_weight)."""
    from centernet_b200 import losses as L
    ls = {'hm': L.FocalLoss()(out['hm'], batch['hm']),
          'hp': L.RegWeightedL1Loss()(out['hps'], batch['hps_mask'], batch['ind'], batch['hps']),
          'wh': L.RegL1Loss()(out['wh'], batch['reg_mask'], batch['ind'], batch['wh'])}
    if opt['reg_offset']:
        ls['off'] = L.RegL1Loss()(out['reg'], batch['reg_mask'], batch['ind'], batch['reg'])
    if opt['reg_hp_offset']:
        ls['hp_offset'] = L.RegL1Loss()(out['hp_offset'], batch['hp_mask'], batch['hp_ind'], batch['hp_offset'])
    if opt['hm_hp']:
        ls['hm_hp'] = L.FocalLoss()(out['hm_hp'], batch['hm_hp'])
    ls['loss'] = ls['hm'] + 0.1 * ls['wh'] + ls.get('off', 0) + ls['hp'] + ls.get('hm_hp', 0) \
        + ls.get('hp_offset', 0)
    return ls


@pytest.mark.parametrize("name", ["mp_coco", "mp_flip", "mp_small", "mp_plain"])
def test_trainer_losses_on_device_batch_equal_golden_batch(name):
    """The trainer's losses on the device batch equal them on the golden batch uploaded (the samples whose hm /
    hm_hp the golden holds)."""
    from centernet_b200 import train_input as T
    g = golden("train_multi_pose")
    case = MC.CASES[name]
    batch = T.build_multi_pose_batch(T.collate_multi_pose(case_samples(name)), dense_hm=True)
    idx = _golden_hm_samples(g, name)
    dev = {k: batch[k][idx] for k in batch if k not in LISTS + HP_LISTS + ('input',)}
    ref = {k: torch.from_numpy(np.stack([g["%s_%d_%s" % (name, i, k)] for i in idx])).cuda() for k in dev}
    for k in dev:
        assert dev[k].dtype == ref[k].dtype and dev[k].shape == ref[k].shape, k
    nj, r, b = case['num_joints'], case['input_res'] // case['down_ratio'], len(idx)
    gen = torch.Generator(device="cuda").manual_seed(7)
    rnd = lambda c, lo=0.0, hi=1.0: torch.rand((b, c, r, r), device="cuda", generator=gen) * (hi - lo) + lo
    out = {'hm': rnd(case['num_classes']).clamp(1e-4, 1 - 1e-4), 'hm_hp': rnd(nj).clamp(1e-4, 1 - 1e-4),
           'hps': rnd(2 * nj, -8, 8), 'wh': rnd(2, 0, 30), 'reg': rnd(2), 'hp_offset': rnd(2)}
    a, w = _trainer_losses(out, dev, case), _trainer_losses(out, ref, case)
    assert set(a) == set(w)
    for k in a:
        assert torch.equal(a[k], w[k]), (k, a[k].item(), w[k].item())
    assert a['loss'].item() > 0


def test_targets_edge_cases_against_restatement():
    """Random crops, flips and rotations on a batch of 7: zero objects, more objects than slots, joints just
    outside the map, no visible joint, zero-size boxes on rotated images, 128 slots."""
    from centernet_b200 import train_input as T
    rng = np.random.default_rng(9)
    nj, flip_idx = 17, [tuple(e) for e in MC.COCO_FLIP_IDX]
    samples = []
    for i in range(7):
        h, w = int(rng.integers(5, 700)), int(rng.integers(5, 700))
        n = (0, 3, 40, 130, 17, 1, 64)[i]
        x0, y0 = rng.uniform(-0.5, 1.2, n) * w, rng.uniform(-0.5, 1.2, n) * h
        bw, bh = rng.uniform(0, 0.7, n) * w, rng.uniform(0, 0.7, n) * h
        bw[rng.random(n) < 0.1] = 0
        boxes = np.stack([x0, y0, x0 + bw, y0 + bh], 1).astype(np.float32).reshape(-1, 4)
        kps = []
        for k in range(n):
            p = np.stack([x0[k] + rng.uniform(-0.5, 1.5, nj) * max(bw[k], 4), y0[k] + rng.uniform(-0.5, 1.5, nj)
                          * max(bh[k], 4), rng.choice([0., 1., 2.], nj)], 1).astype(np.float32)
            if rng.random() < 0.2:
                p[:, 2] = 0
            kps.append(p.reshape(-1))
        c = np.array([w / 2., h / 2.], np.float32)
        s = np.float64(max(h, w) * rng.uniform(0.6, 1.4))
        rot = 0 if i % 3 == 0 else np.float64(rng.uniform(-60, 60))
        flip = bool(i % 2)
        if flip:
            c[0] = w - c[0] - 1
        samples.append(dict(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), boxes=boxes,
                            cls=np.zeros(n, np.int64), keypoints=kps, c=c, s=s, rot=rot, flip=flip,
                            input_res=512, output_res=128, max_objs=128, num_classes=1, num_joints=nj,
                            flip_idx=flip_idx, mean=MC.MEAN, std=MC.STD, reg_offset=True, hm_hp=True,
                            reg_hp_offset=True, order=-1, blend=np.zeros(6, np.float32), light=np.zeros(3),
                            minv=np.array(T._invert(T.affine_transform(c, s, [512, 512], rot))),
                            trans_output_rot=T.affine_transform(c, s, [128, 128], rot).reshape(6),
                            trans_output=T.affine_transform(c, s, [128, 128]).reshape(6)))
    batch = T.build_multi_pose_batch(T.collate_multi_pose(samples), dense_hm=True)
    for i, s in enumerate(samples):
        t = restated(s)
        for k in TARGETS + LISTS + HP_LISTS + ('hm', 'hm_hp'):
            assert_bits(batch[k][i].cpu().numpy(), t[k], "%d %s" % (i, k))
    assert int(batch['obj_valid'][0].sum()) == 0 and int(batch['hp_mask'].sum()) > 0

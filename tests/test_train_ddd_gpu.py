"""Training input of the ddd sampler on the H100 (centernet_b200.train_input): the device batch against
tests/golden/train_ddd.npz and the numpy restatements (tests/train_np.py, tests/train_ddd_np.py) bit for bit --
input in fp32 and bf16 / fp16 (the fp32 value rounded once), NCHW and channels_last, every target with the
reference's dtype, hm with its ignore regions -- the device radius against the reference's radius table, and the
trainer's losses on the batch."""
import functools
import random
import zlib

import numpy as np
import pytest
import torch

import ddd_train_cases as DC
import train_ddd_np as DN
import train_np as TN
from helpers import golden

pytestmark = pytest.mark.gpu

DTYPES = (torch.float32, torch.bfloat16, torch.float16)
FORMATS = (torch.contiguous_format, torch.channels_last)
TARGETS = ('hm', 'dep', 'dim', 'ind', 'rotbin', 'rotres', 'reg_mask', 'rot_mask', 'wh', 'reg')


def _assert_bits(got, want, what):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, got.shape, want.dtype, want.shape)
    u = np.dtype("u%d" % got.itemsize)
    bad = got.view(u) != want.view(u)
    assert not bad.any(), "%s: %d of %d values differ, first at %s" % (what, bad.sum(), bad.size,
                                                                         np.argwhere(bad)[0])


def case_samples(name):
    """The case's samples as DddTrainInput returns them, drawn from the golden seeds (no image files)."""
    from centernet_b200 import train_input as T
    case = DC.CASES[name]
    opt = DC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    np.random.seed(case['seed']); random.seed(case['seed'])
    out = []
    try:
        for i, (h, w) in enumerate(case['sizes']):
            s = T.ddd_params(h, w, opt, case['split'])
            boxes, cls, alpha, depth, dim = DC.case_objects(name, i)
            s.update(image=DC.case_image(name, i), boxes=boxes, cls=cls, alpha=alpha, depth=depth, dim=list(dim),
                     max_objs=case['max_objs'], num_classes=case['num_classes'], mean=DC.MEAN, std=DC.STD,
                     rect_mask=case['rect_mask'], reg_bbox=case['reg_bbox'], reg_offset=case['reg_offset'])
            out.append(s)
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])
    return out


def restated(s):
    return DN.ddd_targets(s['boxes'], s['cls'], s['alpha'], s['depth'], s['dim'], s['aug'], s['trans_output'],
                          s['max_objs'], s['num_classes'], s['output_h'], s['output_w'], s['rect_mask'])


@functools.lru_cache(maxsize=None)
def oracle_inputs(name):
    from centernet_b200 import train_input as T
    out = []
    for s in case_samples(name):
        m = T.affine_transform(s['c'], s['s'], [s['input_w'], s['input_h']])
        out.append(TN.train_image(s['image'], m, False, s['input_w'], s['input_h'], DC.MEAN, DC.STD))
    return np.stack(out)


def _expected_keys(case):
    keys = {'input', 'hm', 'dep', 'dim', 'ind', 'rotbin', 'rotres', 'reg_mask', 'rot_mask'}
    keys |= {'wh'} if case['reg_bbox'] else set()
    keys |= {'reg'} if case['reg_offset'] else set()
    return keys


@pytest.mark.parametrize("name", list(DC.CASES))
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_ddd_batch_matches_reference(name, dtype, fmt):
    from centernet_b200 import train_input as T
    g = golden("train_ddd")
    case = DC.CASES[name]
    samples = case_samples(name)
    packed = T.collate_ddd(samples)
    host = packed['buffer'].clone()
    batch = T.build_ddd_batch(packed, dtype=dtype, memory_format=fmt)
    torch.cuda.synchronize()
    assert torch.equal(packed['buffer'], host), "the packed host buffer was modified"
    assert set(batch) == _expected_keys(case)
    inp = batch['input']
    assert inp.dtype == dtype and inp.is_contiguous(memory_format=fmt)
    got = inp.float().cpu().numpy()
    want = torch.from_numpy(oracle_inputs(name)).to(dtype).float().numpy()
    _assert_bits(got, want, "%s input %s" % (name, dtype))
    for i, s in enumerate(samples):
        p = "%s_%d_" % (name, i)
        if dtype == torch.float32:
            np.testing.assert_array_equal(DC.input_sample(got[i]), g[p + "input_sample"])
        t = restated(s)
        for k in TARGETS:
            if k in batch:
                _assert_bits(batch[k][i].cpu().numpy(), g[p + k], p + k)
                _assert_bits(batch[k][i].cpu().numpy(), t[k], p + k + " restated")


def test_ddd_batch_bit_identical_run_to_run():
    from centernet_b200 import train_input as T
    packed = T.collate_ddd(case_samples("rect"))
    a = T.build_ddd_batch(packed)
    b = T.build_ddd_batch(packed)
    torch.cuda.synchronize()
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_device_radius_matches_reference_table():
    """int(gaussian_radius((h, w))) of the device (the C library's powf square restated) on every pair of the
    reference's radius table: the random pairs against the numpy restatement value by value and the golden CRC,
    the near-integer pairs against the golden radii."""
    from centernet_b200._lib import C, ptr
    g = golden("train_ddd")
    h, w = DC.radius_pairs()
    r = np.maximum(DN.gaussian_radius_f32(h, w).astype(np.int64), 0).astype(np.int32)
    assert np.uint32(zlib.crc32(r.astype(np.int16).tobytes())) == g["radius_int_crc"]
    nh, nw = DC.near_pairs(g["radius_near_h0"], g["radius_near_w0"])
    for hh, ww, want in ((h, w, r), (nh, nw, np.maximum(g["radius_near"].astype(np.int64), 0).astype(np.int32))):
        th, tw = torch.from_numpy(hh).cuda(), torch.from_numpy(ww).cuda()
        out = torch.empty(len(hh), dtype=torch.int32, device="cuda")
        C.ddd_gaussian_radius(ptr(th), ptr(tw), len(hh), ptr(out), torch.cuda.current_stream().cuda_stream)
        _assert_bits(out.cpu().numpy(), want, "radius")


def test_targets_edge_cases_against_restatement():
    """Random KITTI-like batches of 5 with every class code, rect_mask on and off, 128 slots, zero objects, more
    objects than slots and boxes that collapse when clipped."""
    from centernet_b200 import train_input as T
    rng = np.random.default_rng(17)
    for rect in (False, True):
        samples = []
        for i in range(5):
            h, w = int(rng.integers(300, 400)), int(rng.integers(1100, 1300))
            n = (0, 9, 60, 140, 128)[i]
            x0, y0 = rng.uniform(-0.2, 1.1, n) * w, rng.uniform(-0.2, 1.1, n) * h
            bw, bh = rng.uniform(0, 0.3, n) * w, rng.uniform(0, 0.5, n) * h
            boxes = np.stack([x0, y0, x0 + bw, y0 + bh], 1).astype(np.float32).reshape(-1, 4)
            cls = rng.choice([0, 1, 2, -1, -2, -3, -4, -99, -500], n)
            c = np.array([w / 2., h / 2.])
            s = np.array([w, h], np.int32)
            aug = bool(i % 2)
            if aug:
                s = s * np.float64(rng.uniform(0.6, 1.4))
                c[0] += w * rng.uniform(-0.2, 0.2)
                c[1] += h * rng.uniform(-0.2, 0.2)
            samples.append(dict(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), boxes=boxes, cls=cls,
                                alpha=rng.uniform(-4, 4, n), depth=rng.uniform(1, 90, n),
                                dim=list(rng.uniform(0.5, 10, (n, 3))), c=c, s=s, aug=aug, input_h=384,
                                input_w=1280, output_h=96, output_w=320, max_objs=128, num_classes=3,
                                mean=DC.MEAN, std=DC.STD, rect_mask=rect, reg_bbox=True, reg_offset=True,
                                minv=np.array(T._invert(T.affine_transform(c, s, [1280, 384]))),
                                trans_output=T.affine_transform(c, s, [320, 96]).reshape(6)))
        batch = T.build_ddd_batch(T.collate_ddd(samples))
        for i, s in enumerate(samples):
            t = restated(s)
            for k in TARGETS:
                _assert_bits(batch[k][i].cpu().numpy(), t[k], "%s %d %s" % (rect, i, k))
        assert float(batch['hm'][0].abs().sum()) == 0 and int(batch['rot_mask'].sum()) > 0


def _trainer_losses(out, batch, opt):
    """trains/ddd.py:22-58's composition (hm_weight 1, dep_weight 1, dim_weight 1, rot_weight 1, wh_weight 0.1,
    off_weight 1; eval_oracle_dep off)."""
    from centernet_b200 import losses as L
    ls = {'hm': L.FocalLoss()(out['hm'], batch['hm']),
          'dep': L.L1Loss()(out['dep'], batch['reg_mask'], batch['ind'], batch['dep']),
          'dim': L.L1Loss()(out['dim'], batch['reg_mask'], batch['ind'], batch['dim']),
          'rot': L.BinRotLoss()(out['rot'], batch['rot_mask'], batch['ind'], batch['rotbin'], batch['rotres'])}
    if opt['reg_bbox']:
        ls['wh'] = L.L1Loss()(out['wh'], batch['rot_mask'], batch['ind'], batch['wh'])
    if opt['reg_offset']:
        ls['off'] = L.L1Loss()(out['reg'], batch['rot_mask'], batch['ind'], batch['reg'])
    ls['loss'] = ls['hm'] + ls['dep'] + ls['dim'] + ls['rot'] + 0.1 * ls.get('wh', 0) + ls.get('off', 0)
    return ls


@pytest.mark.parametrize("name", ["kitti", "rect", "aug", "keep"])
def test_trainer_losses_on_device_batch_equal_golden_batch(name):
    from centernet_b200 import train_input as T
    g = golden("train_ddd")
    case = DC.CASES[name]
    batch = T.build_ddd_batch(T.collate_ddd(case_samples(name)))
    n = len(case['sizes'])
    dev = {k: batch[k] for k in batch if k != 'input'}
    ref = {k: torch.from_numpy(np.stack([g["%s_%d_%s" % (name, i, k)] for i in range(n)])).cuda() for k in dev}
    for k in dev:
        assert dev[k].dtype == ref[k].dtype and dev[k].shape == ref[k].shape, k
    opt = DC.make_opt(case)
    oh, ow = opt.output_h, opt.output_w
    gen = torch.Generator(device="cuda").manual_seed(7)
    rnd = lambda c, lo=0.0, hi=1.0: torch.rand((n, c, oh, ow), device="cuda", generator=gen) * (hi - lo) + lo
    out = {'hm': rnd(case['num_classes']).clamp(1e-4, 1 - 1e-4), 'dep': rnd(1, 1, 80), 'dim': rnd(3, 0.5, 5),
           'rot': rnd(8, -2, 2), 'wh': rnd(2, 0, 60), 'reg': rnd(2)}
    a, w = _trainer_losses(out, dev, case), _trainer_losses(out, ref, case)
    assert set(a) == set(w)
    for k in a:
        assert torch.equal(a[k], w[k]), (k, a[k].item(), w[k].item())
    assert a['loss'].item() > 0

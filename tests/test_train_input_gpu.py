"""Training input of the ctdet sampler on the H100 (centernet_b200.train_input): the device batch against the
numpy restatement (tests/train_np.py) bit for bit in fp32, against the fp32 oracle rounded once in bf16 / fp16,
in NCHW and channels_last; targets, dense hm and the FocalSplatLoss lists against tests/golden/train.npz."""
import random

import numpy as np
import pytest
import torch

import train_cases as TC
import train_np as TN
from helpers import golden

pytestmark = pytest.mark.gpu

DTYPES = (torch.float32, torch.bfloat16, torch.float16)
FORMATS = (torch.contiguous_format, torch.channels_last)


def _want(x, dtype):
    """The fp32 oracle rounded once to dtype, as fp32 numbers."""
    return torch.from_numpy(np.ascontiguousarray(x)).to(dtype).float().numpy()


def _got(t):
    assert t.is_contiguous(memory_format=torch.channels_last) or t.is_contiguous()
    return t.float().cpu().numpy()


def _assert_bits(got, want, what):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), "%s: %d of %d values differ, first at %s" % (what, bad.sum(), bad.size,
                                                                         np.argwhere(bad)[0])


def case_samples(name):
    """The case's samples as CTDetTrainInput returns them, drawn from the golden seeds (no image files)."""
    from centernet_b200 import train_input as T
    case = TC.CASES[name]
    opt = TC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    np.random.seed(case['seed']); random.seed(case['seed'])
    data_rng = np.random.RandomState(case['seed'])
    out = []
    try:
        for i, (h, w) in enumerate(case['sizes']):
            s = T.sample_params(h, w, opt, case['split'], data_rng, TC.EIG_VAL, TC.EIG_VEC)
            anns = TC.case_anns(name, i)[:case['max_objs']]
            ids = TC.cat_ids(case)
            s.update(image=TC.case_image(name, i), max_objs=case['max_objs'], num_classes=case['num_classes'],
                     mean=TC.MEAN, std=TC.STD, cat_spec_wh=case['cat_spec_wh'], reg_offset=case['reg_offset'],
                     boxes=np.array([[a['bbox'][0], a['bbox'][1], a['bbox'][0] + a['bbox'][2],
                                      a['bbox'][1] + a['bbox'][3]] for a in anns], np.float32).reshape(-1, 4),
                     cls=np.array([ids[a['category_id']] for a in anns], np.int32))
            out.append(s)
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])
    return out


GOLDEN_CASES = [n for n, c in TC.CASES.items() if 'rot' not in c]


@pytest.mark.parametrize("name", GOLDEN_CASES)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_ctdet_batch_matches_reference(name, dtype, fmt):
    from centernet_b200 import train_input as T
    g = golden("train")
    case = TC.CASES[name]
    samples = case_samples(name)
    packed = T.collate_ctdet(samples)
    host = packed['buffer'].clone()
    batch = T.build_ctdet_batch(packed, dtype=dtype, memory_format=fmt, dense_hm=True)
    torch.cuda.synchronize()
    assert torch.equal(packed['buffer'], host), "the packed host buffer was modified"
    keys = {'input', 'reg_mask', 'ind', 'hm', 'obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid'}
    keys |= {'cat_spec_wh', 'cat_spec_mask'} if case['cat_spec_wh'] else {'wh'}
    keys |= {'reg'} if case['reg_offset'] else set()
    assert set(batch) == keys
    inp = batch['input']
    assert inp.dtype == dtype and inp.is_contiguous(memory_format=fmt)
    got = _got(inp)
    for i, s in enumerate(samples):
        p = "%s_%d_" % (name, i)
        x = TN.train_image(s['image'], T.affine_transform(s['c'], s['s'], [s['input_w'], s['input_h']]),
                           s['flip'], s['input_w'], s['input_h'], TC.MEAN, TC.STD, s['order'], s['blend'],
                           s['light'])
        _assert_bits(got[i], _want(x, dtype), p + "input")
        if dtype == torch.float32:
            np.testing.assert_array_equal(got[i][:, ::17, ::13], g[p + "input_sample"])
        for k in ('reg_mask', 'ind', 'wh', 'reg', 'cat_spec_wh', 'cat_spec_mask'):
            if k in batch:
                assert batch[k].dtype == torch.from_numpy(g[p + k]).dtype, k
                np.testing.assert_array_equal(batch[k][i].cpu().numpy(), g[p + k], err_msg=p + k)
        if p + "hm" in g:
            _assert_bits(batch['hm'][i].cpu().numpy(), g[p + "hm"], p + "hm")
        np.testing.assert_array_equal(batch['obj_valid'][i].cpu().numpy(), g[p + "reg_mask"])
        ind = g[p + "ind"]
        valid = g[p + "reg_mask"] == 1
        ow = s['output_w']
        np.testing.assert_array_equal(batch['obj_cy'][i].cpu().numpy()[valid], ind[valid] // ow)
        np.testing.assert_array_equal(batch['obj_cx'][i].cpu().numpy()[valid], ind[valid] % ow)


def test_ctdet_batch_bit_identical_run_to_run():
    from centernet_b200 import train_input as T
    packed = T.collate_ctdet(case_samples("crop"))
    a = T.build_ctdet_batch(packed, dense_hm=True)
    b = T.build_ctdet_batch(packed, dense_hm=True)
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_focal_splat_loss_on_emitted_lists():
    """FocalSplatLoss on the emitted object lists equals FocalLoss on the reference's dense hm (the golden)."""
    from centernet_b200 import losses as L
    from centernet_b200 import train_input as T
    g = golden("train")
    for name in ("crop2", "shift", "plain"):
        samples = case_samples(name)
        batch = T.build_ctdet_batch(T.collate_ctdet(samples))
        n = len([k for k in g if k.startswith(name + "_") and k.endswith("_hm")])
        hm = torch.from_numpy(np.stack([g["%s_%d_hm" % (name, i)] for i in range(n)])).cuda()
        rng = np.random.default_rng(1)
        pred = torch.from_numpy(np.clip(rng.random(hm.shape, dtype=np.float32), 1e-4, 1 - 1e-4)).cuda()
        lists = [batch[k][:n] for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid')]
        lf = L.FocalSplatLoss()(pred, *lists)
        ld = L.FocalLoss()(pred, hm)
        np.testing.assert_allclose(lf.item(), ld.item(), rtol=1e-6, err_msg=name)


def _random_case(rng, b, max_side, out_h, out_w, colour, rot=False, small=False):
    imgs, mats, flips, orders, blends, lights = [], [], [], [], [], []
    for i in range(b):
        if small and i % 3 == 0:
            h, w = int(rng.integers(1, 9)), int(rng.integers(1, 9))
        else:
            h, w = int(rng.integers(16, max_side[0] + 1)), int(rng.integers(16, max_side[1] + 1))
        if i == 0:
            h, w = max_side
        imgs.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        cx, cy, sc = w * rng.uniform(0.2, 0.8), h * rng.uniform(0.2, 0.8), max(h, w) * rng.uniform(0.6, 1.4)
        ang = np.deg2rad(rng.uniform(-45, 45)) if rot else 0.0
        k = out_w / sc
        mats.append(np.array([[k * np.cos(ang), -k * np.sin(ang), 0], [k * np.sin(ang), k * np.cos(ang), 0]]))
        mats[-1][:, 2] = np.array([out_w / 2, out_h / 2]) - mats[-1][:, :2] @ np.array([cx, cy])
        flips.append(int(rng.random() < 0.5))
        orders.append(i % 6 if colour else -1)
        alpha = 1 + np.array([0.4, -0.4, rng.uniform(-0.4, 0.4)])[rng.permutation(3)]
        bl = np.zeros(6, np.float32)
        bl[0::2], bl[1::2] = alpha.astype(np.float32), (1 - alpha).astype(np.float32)
        blends.append(bl)
        lights.append(np.dot(TC.EIG_VEC, TC.EIG_VAL * rng.normal(scale=0.1, size=3)))
    return imgs, mats, flips, orders, blends, lights


@pytest.mark.parametrize("b,max_side,out,colour,rot,small", [
    (1, (960, 1280), (512, 512), True, False, False),
    (7, (960, 1280), (512, 512), True, False, True),
    (7, (600, 800), (384, 512), False, False, True),
    (7, (480, 640), (256, 192), True, True, False),
    (64, (480, 640), (96, 128), True, False, True),
])
def test_augment_images_against_oracle(b, max_side, out, colour, rot, small):
    from centernet_b200 import train_input as T
    rng = np.random.default_rng(b * 1000 + out[0])
    imgs, mats, flips, orders, blends, lights = _random_case(rng, b, max_side, out[0], out[1], colour, rot, small)
    want = np.stack([TN.train_image(im, m, f, out[1], out[0], TC.MEAN, TC.STD, o, bl, li)
                     for im, m, f, o, bl, li in zip(imgs, mats, flips, orders, blends, lights)])
    first = None
    for dtype in DTYPES:
        for fmt in FORMATS:
            got = T.augment_images(imgs, mats, out[0], out[1], TC.MEAN, TC.STD, flips=flips, orders=orders,
                                   blends=blends, lights=lights, dtype=dtype, memory_format=fmt)
            assert got.dtype == dtype and got.is_contiguous(memory_format=fmt)
            _assert_bits(_got(got), _want(want, dtype), "B=%d %s %s" % (b, dtype, fmt))
            if dtype == torch.float32 and fmt == torch.contiguous_format:
                first = got
    again = T.augment_images(imgs, mats, out[0], out[1], TC.MEAN, TC.STD, flips=flips, orders=orders,
                             blends=blends, lights=lights)
    assert torch.equal(first, again)


@pytest.mark.parametrize("name", [n for n, c in TC.CASES.items() if 'rot' in c])
def test_rotated_warp_matches_reference(name):
    from centernet_b200 import train_input as T
    g = golden("train")
    case = TC.CASES[name]
    p = name + "_0_"
    got = T.augment_images([TC.case_image(name, 0)], [g[p + "matrix"]], case['out'], case['out'], TC.MEAN, TC.STD,
                           orders=[int(g[p + "order"])], blends=[g[p + "blend"]], lights=[g[p + "light"]])
    x = got[0].cpu().numpy()
    np.testing.assert_array_equal(x[:, ::17, ::13], g[p + "input_sample"])
    import zlib
    assert np.uint32(zlib.crc32(np.ascontiguousarray(x).view(np.uint8))) == g[p + "input_crc"]


def test_targets_edge_cases_against_oracle():
    """Zero objects, more objects than slots, boxes leaving the crop or collapsing on the clip, flipped boxes,
    cat_spec_wh, on a batch of 7 images with random crops."""
    from centernet_b200 import train_input as T
    rng = np.random.default_rng(9)
    samples = []
    for i in range(7):
        h, w = int(rng.integers(5, 700)), int(rng.integers(5, 700))
        n = (0, 3, 40, 130, 17, 1, 64)[i]
        x0 = rng.uniform(-0.5, 1.2, n) * w
        y0 = rng.uniform(-0.5, 1.2, n) * h
        bw, bh = rng.uniform(0, 0.7, n) * w, rng.uniform(0, 0.7, n) * h
        bw[rng.random(n) < 0.1] = 0
        boxes = np.stack([x0, y0, x0 + bw, y0 + bh], 1).astype(np.float32).reshape(-1, 4)
        c = np.array([w / 2., h / 2.], np.float32)
        s = np.float64(max(h, w) * rng.uniform(0.6, 1.4))
        flip = bool(i % 2)
        if flip:
            c[0] = w - c[0] - 1
        samples.append(dict(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), boxes=boxes,
                            cls=rng.integers(0, 80, n).astype(np.int32), c=c, s=s, flip=flip, input_h=512,
                            input_w=512, output_h=128, output_w=128, max_objs=128, num_classes=80, mean=TC.MEAN,
                            std=TC.STD, cat_spec_wh=True, reg_offset=True, order=-1, blend=np.zeros(6, np.float32),
                            light=np.zeros(3),
                            minv=np.array(T._invert(T.affine_transform(c, s, [512, 512]))),
                            trans_output=T.affine_transform(c, s, [128, 128]).reshape(6)))
    batch = T.build_ctdet_batch(T.collate_ctdet(samples), dense_hm=True)
    for i, s in enumerate(samples):
        t = TN.ctdet_targets(s['boxes'], s['cls'], s['flip'], s['image'].shape[1], s['trans_output'], 128, 80, 128,
                             128)
        for k in ('reg_mask', 'ind', 'reg', 'cat_spec_wh', 'cat_spec_mask', 'obj_cls', 'obj_cx', 'obj_cy',
                  'obj_radius', 'obj_valid'):
            np.testing.assert_array_equal(batch[k][i].cpu().numpy(), t[k], err_msg="%d %s" % (i, k))
    assert int(batch['reg_mask'][0].sum()) == 0

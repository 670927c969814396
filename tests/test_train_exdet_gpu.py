"""Training input of the exdet sampler on the H100 (centernet_b200.train_input): the device batch against
tests/golden/train_exdet.npz and the numpy restatements (tests/train_np.py, tests/train_exdet_np.py) bit for bit --
input in fp32 and bf16 / fp16 (the fp32 value rounded once), NCHW and channels_last, every target with the
reference's dtype, the five dense heat maps and their object lists -- and the trainer's losses on it."""
import functools
import random

import numpy as np
import pytest
import torch

import exdet_train_cases as EC
import train_exdet_np as EN
import train_np as TN
from helpers import assert_bits, golden

pytestmark = pytest.mark.gpu

DTYPES = (torch.float32, torch.bfloat16, torch.float16)
FORMATS = (torch.contiguous_format, torch.channels_last)
PARTS = ('t', 'l', 'b', 'r')
TARGETS = ('reg_mask',) + tuple('reg_' + p for p in PARTS) + tuple('ind_' + p for p in PARTS)
MAPS = tuple('hm_' + p for p in PARTS + ('c',))
LISTS = ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid')
EX_LISTS = ('ex_cls', 'ex_cx', 'ex_cy', 'ex_radius', 'ex_valid')


def case_samples(name):
    """The case's samples as ExdetTrainInput returns them, drawn from the golden seeds (no image files)."""
    from centernet_b200 import train_input as T
    case = EC.CASES[name]
    opt = EC.make_opt(case)
    saved = np.random.get_state(), random.getstate()
    np.random.seed(case['seed']); random.seed(case['seed'])
    data_rng = np.random.RandomState(case['seed'])
    out = []
    try:
        for i, (h, w) in enumerate(case['sizes']):
            s = T.exdet_params(h, w, opt, case['split'], data_rng, EC.EIG_VAL, EC.EIG_VEC)
            pts, cls = EC.case_objects(name, i)
            s.update(image=EC.case_image(name, i), points=list(pts.reshape(-1, 8)), cls=cls,
                     max_objs=case['max_objs'], num_classes=case['num_classes'], mean=EC.MEAN, std=EC.STD,
                     agnostic_ex=case['agnostic_ex'], reg_offset=case['reg_offset'])
            out.append(s)
    finally:
        np.random.set_state(saved[0]); random.setstate(saved[1])
    return out


def restated(s):
    """tests/train_exdet_np.py's targets and maps for one sample."""
    r = s['output_res']
    t = EN.exdet_targets(np.asarray(s['points'], np.float32).reshape(-1, 4, 2), s['cls'], s['flip'],
                         s['image'].shape[1], s['trans_output'], s['max_objs'], r, s['agnostic_ex'])
    t.update(EN.exdet_maps(t, s['num_classes'], r, s['agnostic_ex']))
    return t


@functools.lru_cache(maxsize=None)
def oracle_inputs(name):
    from centernet_b200 import train_input as T
    out = []
    for s in case_samples(name):
        m = T.affine_transform(s['c'], s['s'], [s['input_res']] * 2)
        out.append(TN.train_image(s['image'], m, s['flip'], s['input_res'], s['input_res'], EC.MEAN, EC.STD,
                                  s['order'], s['blend'], s['light']))
    return np.stack(out)


def _expected_keys(case, dense_hm):
    keys = {'input'} | set(LISTS) | set(EX_LISTS)
    keys |= set(TARGETS) if case['reg_offset'] else set()
    keys |= set(MAPS) if dense_hm else set()
    return keys


def _check_batch(name, samples, batch, dense_hm):
    g = golden("train_exdet")
    case = EC.CASES[name]
    assert set(batch) == _expected_keys(case, dense_hm)
    b, m, r = len(samples), case['max_objs'], case['input_res'] // case['down_ratio']
    num_hm = 1 if case['agnostic_ex'] else case['num_classes']
    for k in EX_LISTS:
        assert tuple(batch[k].shape) == (4, b, m) and batch[k].is_contiguous(), k
    for i, s in enumerate(samples):
        p = "%s_%d_" % (name, i)
        for k in TARGETS:
            if k in batch:
                assert_bits(batch[k][i].cpu().numpy(), g[p + k], p + k)
        t = restated(s)
        for k in LISTS:
            assert_bits(batch[k][i].cpu().numpy(), t[k], p + k)
        for k in EX_LISTS:
            assert_bits(batch[k][:, i].cpu().numpy(), t[k], p + k)
        if dense_hm:
            for k in MAPS:
                assert tuple(batch[k].shape) == (b, case['num_classes'] if k == 'hm_c' else num_hm, r, r), k
                assert_bits(batch[k][i].cpu().numpy(), t[k], p + k)
                if p + k in g:
                    assert_bits(batch[k][i].cpu().numpy(), g[p + k], p + k + " golden")


@pytest.mark.parametrize("name", list(EC.CASES))
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_exdet_batch_matches_reference(name, dtype, fmt):
    from centernet_b200 import train_input as T
    g = golden("train_exdet")
    samples = case_samples(name)
    packed = T.collate_exdet(samples)
    host = packed['buffer'].clone()
    batch = T.build_exdet_batch(packed, dtype=dtype, memory_format=fmt, dense_hm=True)
    torch.cuda.synchronize()
    assert torch.equal(packed['buffer'], host), "the packed host buffer was modified"
    inp = batch['input']
    assert inp.dtype == dtype and inp.is_contiguous(memory_format=fmt)
    got = inp.float().cpu().numpy()
    want = torch.from_numpy(oracle_inputs(name)).to(dtype).float().numpy()
    assert_bits(got, want, "%s input %s" % (name, dtype))
    if dtype == torch.float32:
        for i in range(len(samples)):
            np.testing.assert_array_equal(EC.input_sample(got[i]), g["%s_%d_input_sample" % (name, i)])
    _check_batch(name, samples, batch, True)


@pytest.mark.parametrize("name", list(EC.CASES))
def test_exdet_batch_without_dense_maps(name):
    """dense_hm=False: no heat map is built, and every other key is what the dense run returns."""
    from centernet_b200 import train_input as T
    samples = case_samples(name)
    packed = T.collate_exdet(samples)
    batch = T.build_exdet_batch(packed)
    dense = T.build_exdet_batch(packed, dense_hm=True)
    torch.cuda.synchronize()
    _check_batch(name, samples, batch, False)
    for k in batch:
        assert torch.equal(batch[k], dense[k]), k


def test_exdet_batch_bit_identical_run_to_run():
    from centernet_b200 import train_input as T
    packed = T.collate_exdet(case_samples("ex_coco"))
    a = T.build_exdet_batch(packed, dense_hm=True)
    b = T.build_exdet_batch(packed, dense_hm=True)
    torch.cuda.synchronize()
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _golden_hm_samples(g, name):
    return [i for i in range(len(EC.CASES[name]['sizes'])) if "%s_%d_hm_c" % (name, i) in g]


def test_focal_splat_loss_on_all_five_list_sets():
    """FocalSplatLoss on the centre lists equals FocalLoss on the reference's hm_c, and on ex_*[p] it equals
    FocalLoss on hm_t / hm_l / hm_b / hm_r."""
    from centernet_b200 import losses as L
    from centernet_b200 import train_input as T
    g = golden("train_exdet")
    rng = np.random.default_rng(1)
    checked = 0
    for name in EC.CASES:
        batch = T.build_exdet_batch(T.collate_exdet(case_samples(name)))
        for i in _golden_hm_samples(g, name):
            p = "%s_%d_" % (name, i)
            for j, part in enumerate(PARTS + ('c',)):
                hm = torch.from_numpy(g[p + "hm_" + part][None]).cuda()
                pred = torch.from_numpy(np.clip(rng.random(hm.shape, dtype=np.float32), 1e-4, 1 - 1e-4)).cuda()
                if part == 'c':
                    lists = [batch[k][i:i + 1] for k in LISTS]
                else:
                    lists = [batch[k][j, i:i + 1] for k in EX_LISTS]
                lf = L.FocalSplatLoss()(pred, *lists)
                np.testing.assert_allclose(lf.item(), L.FocalLoss()(pred, hm).item(), rtol=1e-6,
                                           err_msg=p + "hm_" + part)
                checked += 1
    assert checked >= 5 * 15


def _exdet_losses(out, batch, reg_offset):
    """trains/exdet.py:25-41's ExdetLoss for one stack, hm_weight 1, off_weight 1, with dense maps."""
    from centernet_b200 import losses as L
    hm_loss, reg_loss = 0, 0
    for p in PARTS + ('c',):
        hm_loss = hm_loss + L.FocalLoss()(out['hm_' + p], batch['hm_' + p])
        if p != 'c' and reg_offset:
            reg_loss = reg_loss + L.RegL1Loss()(out['reg_' + p], batch['reg_mask'], batch['ind_' + p],
                                                batch['reg_' + p])
    return {'hm_loss': hm_loss, 'off_loss': reg_loss, 'loss': hm_loss + reg_loss}


@pytest.mark.parametrize("name", ["ex_coco", "ex_agn", "ex_flip", "ex_plain"])
def test_trainer_losses_on_device_batch_equal_golden_batch(name):
    """ExdetLoss on the device batch equals it on the golden batch uploaded (the samples whose maps the golden
    holds)."""
    from centernet_b200 import train_input as T
    g = golden("train_exdet")
    case = EC.CASES[name]
    batch = T.build_exdet_batch(T.collate_exdet(case_samples(name)), dense_hm=True)
    idx = _golden_hm_samples(g, name)
    dev = {k: batch[k][idx] for k in batch if k not in LISTS + EX_LISTS + ('input',)}
    ref = {k: torch.from_numpy(np.stack([g["%s_%d_%s" % (name, i, k)] for i in idx])).cuda() for k in dev}
    for k in dev:
        assert dev[k].dtype == ref[k].dtype and dev[k].shape == ref[k].shape, k
    r, b = case['input_res'] // case['down_ratio'], len(idx)
    num_hm = 1 if case['agnostic_ex'] else case['num_classes']
    gen = torch.Generator(device="cuda").manual_seed(7)
    rnd = lambda c: torch.rand((b, c, r, r), device="cuda", generator=gen)
    out = {'hm_' + p: rnd(num_hm).clamp(1e-4, 1 - 1e-4) for p in PARTS}
    out['hm_c'] = rnd(case['num_classes']).clamp(1e-4, 1 - 1e-4)
    out.update(('reg_' + p, rnd(2)) for p in PARTS)
    a, w = _exdet_losses(out, dev, case['reg_offset']), _exdet_losses(out, ref, case['reg_offset'])
    for k in a:
        assert torch.equal(torch.as_tensor(a[k]), torch.as_tensor(w[k])), (k, float(a[k]), float(w[k]))
    assert float(a['loss']) > 0


@pytest.mark.parametrize("agnostic_ex", [False, True])
def test_targets_edge_cases_against_restatement(agnostic_ex):
    """Random crops and flips on a batch of 7 against the restatement: points outside the crop, coincident points
    (degenerate boxes and objects sharing a point), zero radius, the l <-> r swap of the flip, zero objects, more
    objects than slots, 128 slots."""
    from centernet_b200 import train_input as T
    rng = np.random.default_rng(11 + agnostic_ex)
    nc, res, out_res, m = 7, 512, 128, 128
    samples = []
    for i in range(7):
        h, w = int(rng.integers(5, 700)), int(rng.integers(5, 700))
        n = (0, 3, 40, 130, 17, 1, 64)[i]
        x0, y0 = rng.uniform(-0.5, 1.2, n) * w, rng.uniform(-0.5, 1.2, n) * h
        bw, bh = rng.uniform(-0.1, 0.7, n) * w, rng.uniform(-0.1, 0.7, n) * h
        small = rng.random(n) < 0.2
        bw[small], bh[small] = rng.uniform(0.5, 6, small.sum()), rng.uniform(0.5, 6, small.sum())
        u = rng.random((n, 4))
        u[rng.random(n) < 0.2, :2] = 0                                   # t and l at the corner
        pts = np.stack([x0 + u[:, 0] * bw, y0, x0, y0 + u[:, 1] * bh, x0 + u[:, 2] * bw, y0 + bh, x0 + bw,
                        y0 + u[:, 3] * bh], 1).astype(np.float32)
        if n > 2:
            pts[1] = pts[0]                                              # two objects at the same points
        c = np.array([w / 2., h / 2.])
        s = np.float64(max(h, w) * rng.uniform(0.6, 1.4))
        flip = bool(i % 2)
        samples.append(dict(image=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), points=list(pts),
                            cls=rng.integers(0, 3, n), c=c, s=s, flip=flip, input_res=res, output_res=out_res,
                            max_objs=m, num_classes=nc, agnostic_ex=agnostic_ex, reg_offset=True, mean=EC.MEAN,
                            std=EC.STD, order=-1, blend=np.zeros(6, np.float32), light=np.zeros(3),
                            minv=np.array(T._invert(T.affine_transform(c, s, [res, res]))),
                            trans_output=T.affine_transform(c, s, [out_res, out_res]).reshape(6)))
    batch = T.build_exdet_batch(T.collate_exdet(samples), dense_hm=True)
    zero_radius = 0
    for i, s in enumerate(samples):
        t = restated(s)
        for k in TARGETS + LISTS + MAPS:
            assert_bits(batch[k][i].cpu().numpy(), t[k], "%d %s" % (i, k))
        for k in EX_LISTS:
            assert_bits(batch[k][:, i].cpu().numpy(), t[k], "%d %s" % (i, k))
        zero_radius += int(((t['obj_radius'] == 0) & (t['obj_valid'] == 1)).sum())
    assert int(batch['obj_valid'][0].sum()) == 0 and int(batch['reg_mask'].sum()) > 0 and zero_radius > 0

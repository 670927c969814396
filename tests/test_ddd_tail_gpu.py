"""ddd_merge_device / ddd_post_process / ddd_pre_process on the device: against the reference's own results stored in
tests/golden/ddd_tail.npz and against the numpy restatement (tests/ddd_tail_np.py) -- class membership, order,
lengths, empty-class shapes, NaN positions and every column bit for bit but alpha and rot_y (within 2.5e-6 rad,
wrapped).  Also decode -> tail from ddd_decode_from_logits, a non-default stream, untouched inputs, and the copies
of a whole detector run (one image upload, one result download)."""
import types
import zlib

import numpy as np
import pytest
import torch

from ddd_tail_cases import (INPUT_HW, MEAN, NUM_CLASSES, PEAK_THRESH, PRE_CASES, STD, assert_ddd_equal, ddd_image,
                            flatten, oracle, tail_case)
from helpers import golden

pytestmark = pytest.mark.gpu

G = golden("ddd_tail")
NAMES = [str(n) for n in G["names"]]
F32 = np.float32


@pytest.fixture(scope="module")
def P():
    from centernet_b200 import post_process
    return post_process


def _opt(meta):
    return types.SimpleNamespace(output_w=meta["out_width"], output_h=meta["out_height"], num_classes=NUM_CLASSES)


def _run(P, dets, meta, form):
    if form == 0:
        return P.ddd_merge_device(dets, meta, NUM_CLASSES, PEAK_THRESH)
    return P.ddd_post_process(dets, meta["c"], meta["s"], meta["calib"], _opt(meta))


@pytest.mark.parametrize("name", NAMES)
def test_tail_golden(P, name):
    dets, meta, form = tail_case(G, name)
    want = (G[name + "_out"], G[name + "_len"])
    host = dets.copy()
    dev = torch.from_numpy(dets).cuda()
    for src in (host, dev):                         # numpy and CUDA input
        got = flatten(_run(P, src, meta, form))
        assert_ddd_equal(got, want, name + " vs reference")
        assert_ddd_equal(got, flatten(oracle(dets, meta, form)), name + " vs oracle")
    assert np.array_equal(host.view(np.uint32), dets.view(np.uint32))
    assert torch.equal(dev.cpu().view(torch.int32), torch.from_numpy(dets).view(torch.int32))


def test_rot_y_exactly_pi(P):
    """alpha = atan2(1, 0) + float32(pi / 2) = float32(pi) at u = P[0, 2]: rot_y stays float32(pi) (the wrap compares in
    float32), and the device gives those exact bits as the reference does."""
    dets, meta, form = tail_case(G, "kitti_default")
    rows, _ = flatten(P.ddd_merge_device(torch.from_numpy(dets).cuda(), meta, NUM_CLASSES, PEAK_THRESH))
    want = G["kitti_default_out"]
    at = want[:, 13] == F32(np.pi)
    assert at.any()
    np.testing.assert_array_equal(rows[at][:, [2, 13]], want[at][:, [2, 13]])


def _kitti_meta(B, seed):
    rng = np.random.default_rng(seed)
    sizes = [(375, 1242), (370, 1224), (374, 1238), (376, 1241), (370, 1226)]
    base = np.array([[707.0493, 0, 604.0814, 45.75831], [0, 707.0493, 180.5066, -0.3454157],
                     [0, 0, 1., 0.004981016]], np.float32)
    cal = []
    for i in range(B):
        k = base.copy()
        k[0, 2] += F32(rng.uniform(-5, 5)); k[0, 3] = F32(rng.uniform(-400, 50))
        cal.append(k)
    hw = [sizes[i % len(sizes)] for i in range(B)]
    return {"c": [np.array([w / 2, h / 2], F32) for h, w in hw], "s": [np.array([w, h], np.int32) for h, w in hw],
            "calib": cal, "out_height": INPUT_HW[0] // 4, "out_width": INPUT_HW[1] // 4}


def _heads(B, seed):
    g = torch.Generator().manual_seed(seed)
    H, W = INPUT_HW[0] // 4, INPUT_HW[1] // 4
    hm = torch.randn(B, NUM_CLASSES, H, W, generator=g) * 2 - 2
    rot = torch.randn(B, 8, H, W, generator=g) * 2
    dep = torch.randn(B, 1, H, W, generator=g) * 3
    dim = torch.randn(B, 3, H, W, generator=g) * 0.3 + 1.5
    wh = torch.rand(B, 2, H, W, generator=g) * 60
    reg = torch.rand(B, 2, H, W, generator=g)
    return [t.cuda() for t in (hm, rot, dep, dim, wh, reg)]


@pytest.mark.parametrize("B", [1, 32])
def test_decode_then_tail(P, B):
    """ddd_decode_from_logits on seeded 96 x 320 heads followed by the device tail == the decode's .cpu() followed by
    the restatement, for both forms."""
    from centernet_b200 import decode as D
    dets = D.ddd_decode_from_logits(*_heads(B, 40 + B), K=100)
    meta = _kitti_meta(B, B)
    host = dets.cpu().numpy()
    assert_ddd_equal(flatten(P.ddd_merge_device(dets, meta, NUM_CLASSES, PEAK_THRESH)),
                     flatten(oracle(host, meta, 0)), "merge B=%d" % B)
    assert_ddd_equal(flatten(P.ddd_post_process(dets, meta["c"], meta["s"], meta["calib"], _opt(meta))),
                     flatten(oracle(host, meta, 1)), "post_process B=%d" % B)


def test_stream_and_inputs_untouched(P):
    dets, meta, form = tail_case(G, "calib_b3")
    src = torch.from_numpy(dets).cuda()
    before = src.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = P.ddd_merge_device(src, meta, NUM_CLASSES, PEAK_THRESH)
    assert_ddd_equal(flatten(got), (G["calib_b3_out"], G["calib_b3_len"]), "side stream")
    assert torch.equal(src.view(torch.int32), before.view(torch.int32))


@pytest.mark.parametrize("name", sorted(PRE_CASES))
def test_pre_process_golden(name):
    from centernet_b200 import pre_process as PP
    h, w, keep_res = PRE_CASES[name]
    img = ddd_image(h, w)
    assert np.uint32(zlib.crc32(img.view(np.uint8))) == G[name + "_img_crc"]
    for src in (img, torch.from_numpy(img).cuda()):
        images, meta = PP.ddd_pre_process(src, INPUT_HW[0], INPUT_HW[1], MEAN, STD, keep_res=keep_res)
        images = np.ascontiguousarray(images.cpu().numpy())
        assert tuple(images.shape) == tuple(int(v) for v in G[name + "_shape"])
        np.testing.assert_array_equal(images[:, :, ::9, ::7], G[name + "_sample"])
        assert np.uint32(zlib.crc32(images.view(np.uint8))) == G[name + "_crc"]
        assert meta["s"].dtype == np.int32 and meta["c"].dtype == np.float32 and meta["calib"].dtype == np.float32
        np.testing.assert_array_equal(meta["c"], G[name + "_c"])
        np.testing.assert_array_equal(meta["s"], G[name + "_s"])
        np.testing.assert_array_equal(meta["calib"], G[name + "_calib"])
        assert [meta["out_height"], meta["out_width"]] == [int(v) for v in G[name + "_hw"]]


def test_detector_run_copies(P):
    """ddd_pre_process -> ddd_decode_from_logits -> ddd_merge_device: the uint8 image is the only image-sized upload
    (the other two host->device copies are the warp parameters, 72 B, and the tail's matrix + calibration, 96 B),
    and the results come back in ONE device->host copy.  The network's heads are made on the device beforehand."""
    from torch.profiler import ProfilerActivity, profile
    from centernet_b200 import decode as D
    from centernet_b200 import pre_process as PP
    img = ddd_image(375, 1242)
    heads = _heads(1, 7)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        images, meta = PP.ddd_pre_process(img, INPUT_HW[0], INPUT_HW[1], MEAN, STD)
        dets = D.ddd_decode_from_logits(*heads, K=100)
        res = P.ddd_merge_device(dets, {k: [meta[k]] for k in ("c", "s", "calib")} |
                                 {"out_height": meta["out_height"], "out_width": meta["out_width"]}, NUM_CLASSES)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "Memcpy" in e.name]
    h2d = [n for n in names if "HtoD" in n]
    d2h = [n for n in names if "DtoH" in n]
    assert len(d2h) == 1, names
    assert len(h2d) == 3, names
    assert len(res) == 1 and sorted(res[0]) == [1, 2, 3]

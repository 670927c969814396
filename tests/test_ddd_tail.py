"""The ddd tail without a GPU: the numpy restatement (tests/ddd_tail_np.py) against the reference's own
DddDetector.post_process + merge_outputs and utils.post_process.ddd_post_process stored in tests/golden/ddd_tail.npz,
what that golden covers, and the argument checks of the device tail and its C ABI, which refuse before anything
reaches the device."""
import types

import numpy as np
import pytest
import torch

from ddd_tail_cases import NUM_CLASSES, PEAK_THRESH, assert_ddd_equal, flatten, oracle, tail_case
from helpers import golden

G = golden("ddd_tail")
NAMES = [str(n) for n in G["names"]]
F32 = np.float32


@pytest.mark.parametrize("name", NAMES)
def test_oracle_vs_golden(name):
    dets, meta, form = tail_case(G, name)
    before = dets.copy()
    assert_ddd_equal(flatten(oracle(dets, meta, form)), (G[name + "_out"], G[name + "_len"]), name)
    assert np.array_equal(dets.view(np.uint32), before.view(np.uint32))


def test_golden_covers_the_edges():
    """The cases the GPU tests rely on: KITTI metas (int32 scales, several image sizes, keep_res), one calib per
    image and the drop-in's calibs[0], K = 1000, scores at the cut, class ids -0.0 / 3 / NaN / 1.5, bin ties, a NaN in
    the unselected bin, rot_y beyond +-pi and exactly float32(pi), and both kinds of empty class."""
    forms = {int(G[n + "_form"]) for n in NAMES}
    assert forms == {0, 1}
    sizes = {tuple(int(v) for v in s) for n in NAMES for s in G[n + "_s"]}
    assert {(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1226, 370), (1280, 384)} <= sizes
    assert all(G[n + "_s"].dtype == np.int32 for n in NAMES)
    assert max(G[n + "_dets"].shape[1] for n in NAMES) == 1000
    cal = G["calib_b3_calib"]
    assert len({c.tobytes() for c in cal}) == 3
    dets = np.concatenate([G[n + "_dets"].reshape(-1, 18) for n in NAMES])
    s, cls = dets[:, 2], dets[:, 17]
    assert (s == F32(PEAK_THRESH)).any() and (s == np.nextafter(F32(PEAK_THRESH), F32(1))).any()
    assert np.isnan(s).any() and np.isposinf(s).any()
    assert ((cls == 0) & np.signbit(cls)).any() and (cls == 3).any() and np.isnan(cls).any() and (cls == 1.5).any()
    assert (dets[:, 4] == dets[:, 8]).any()
    sel1 = dets[:, 4] > dets[:, 8]
    assert (sel1 & np.isnan(dets[:, 9])).any() and (~sel1 & np.isnan(dets[:, 5])).any()
    assert dets[:, 11].max() > 9e5 and (dets[:, 11] < 0).any()
    out = np.concatenate([G[n + "_out"] for n in NAMES])
    ry = out[:, 13]
    assert (ry == F32(np.pi)).any()                                   # not wrapped: compared in float32
    assert (np.abs(out[:, 2]) > np.pi).any()                          # alpha itself is never wrapped
    assert (ry > 3.1).any() and (ry < -3.1).any()                     # rot_y wrapped from beyond +pi and -pi
    lens = np.concatenate([G[n + "_len"] for n in NAMES])
    assert (lens == -1).any() and (lens == 0).any()                   # shape (0,) and a list the cut emptied
    assert np.isnan(out[:, 2]).any()


def test_cv_affine_matches_cv2():
    """cv_inv_affine / cv_affine_transform against live cv2.getAffineTransform on random metas: int32 image-size
    scales (the ddd detector's), scalar and vector float32 scales, any centre and output size."""
    cv2 = pytest.importorskip("cv2")
    from centernet_b200 import post_process as P
    rng = np.random.default_rng(2026)
    for t in range(1500):
        w, h = int(rng.integers(200, 2000)), int(rng.integers(100, 1200))
        s = [np.array([w, h], np.int32), F32(rng.uniform(100, 2000)), rng.uniform(100, 2000, 2).astype(F32)][t % 3]
        c = np.array([w / 2, h / 2], F32) if t % 2 else rng.uniform(0, 1000, 2).astype(F32)
        size = (int(rng.integers(16, 400)), int(rng.integers(16, 400)))
        src, dst = P._affine_points(c, s, size)
        np.testing.assert_array_equal(P.cv_inv_affine(c, s, size), cv2.getAffineTransform(dst, src))
        np.testing.assert_array_equal(P.cv_affine_transform(src, dst), cv2.getAffineTransform(src, dst))


@pytest.mark.parametrize("name", [str(n) for n in G["pre_names"]])
def test_oracle_pre_process(name):
    """DddDetector.pre_process restated (OpenCV's fixed-point warp of oracle/pre_np.py on cv2's matrix, then the
    detector's float32 normalisation) against the golden, bit for bit."""
    import zlib
    from centernet_b200 import post_process as P
    from ddd_tail_cases import INPUT_HW, MEAN, PRE_CASES, STD, ddd_image
    from oracle import pre_np
    h, w, keep_res = PRE_CASES[name]
    img = ddd_image(h, w)
    assert np.uint32(zlib.crc32(img.view(np.uint8))) == G[name + "_img_crc"]
    ih, iw = INPUT_HW
    s = np.array([iw, ih] if keep_res else [w, h], np.int32)
    m = P.cv_affine_transform(*P._affine_points(np.array([w / 2, h / 2], F32), s, (iw, ih)))
    x = pre_np.warp_affine_linear(img, m, (iw, ih)).astype(F32) / F32(255)
    x = (x - np.array(MEAN, F32)) / np.array(STD, F32)
    images = np.ascontiguousarray(x.transpose(2, 0, 1)[None])
    assert images.dtype == np.float32
    np.testing.assert_array_equal(images[:, :, ::9, ::7], G[name + "_sample"])
    assert np.uint32(zlib.crc32(images.view(np.uint8))) == G[name + "_crc"]
    np.testing.assert_array_equal(G[name + "_s"], s)


def _opt(nc=NUM_CLASSES):
    return types.SimpleNamespace(output_w=320, output_h=96, num_classes=nc)


def _meta(b):
    return {"c": [np.zeros(2, F32)] * b, "s": [np.array([1242, 375], np.int32)] * b,
            "calib": [np.eye(3, 4, dtype=F32)] * b, "out_height": 96, "out_width": 320}


def test_sixteen_columns_raise():
    """ddd_decode without wh (--not_reg_bbox): the reference's ddd_post_process_3d raises IndexError on every row."""
    from centernet_b200 import post_process as P
    d = np.zeros((1, 4, 16), F32)
    with pytest.raises(ValueError, match="16 columns"):
        P.ddd_post_process(d, [np.zeros(2, F32)], [np.array([1242, 375], np.int32)], [np.eye(3, 4)], _opt())
    with pytest.raises(ValueError, match="16 columns"):
        P.ddd_merge_device(d, _meta(1), NUM_CLASSES)
    with pytest.raises(ValueError, match="16 columns"):
        import ddd_tail_np as O
        O.ddd_post_process(d, [np.zeros(2, F32)], [np.array([1242, 375], np.int32)], [np.eye(3, 4)], 320, 96, 3)


def test_cpu_tensors_and_bad_shapes_raise():
    from centernet_b200 import post_process as P
    with pytest.raises(NotImplementedError, match="CUDA"):
        P.ddd_merge_device(torch.zeros(1, 4, 18), _meta(1), NUM_CLASSES)
    with pytest.raises(NotImplementedError, match="CUDA"):
        P.ddd_post_process(torch.zeros(1, 4, 18), [np.zeros(2, F32)], [np.array([1242, 375], np.int32)],
                           [np.eye(3, 4)], _opt())
    with pytest.raises(ValueError, match="18"):
        P.ddd_merge_device(np.zeros((1, 4, 17), F32), _meta(1), NUM_CLASSES)
    with pytest.raises(ValueError, match="num_classes"):
        P.ddd_merge_device(np.zeros((1, 4, 18), F32), _meta(1), 0)
    with pytest.raises(ValueError, match="per image"):
        P.ddd_merge_device(np.zeros((2, 4, 18), F32), _meta(1), NUM_CLASSES)


def test_abi_rejections():
    """Every argument is checked before a launch (fake pointers never reach the device)."""
    from centernet_b200 import _C
    # dets, b, n, d, trans, calib, nc, cut, thresh, rows, offsets, seen, stream; dets [1, 8, 18] at 1 << 20
    ok = [1 << 20, 1, 8, 18, 2 << 20, 3 << 20, 3, 1, 0.2, 4 << 20, 5 << 20, 6 << 20, 0]
    bad = [(0, 0), (4, 0), (5, 0), (9, 0), (10, 0),             # null pointers (seen may be null)
           (3, 16), (3, 17), (3, 19),                            # not the 18 columns of ddd_decode with wh
           (1, 0), (2, 0), (6, 0), (6, 8193),                    # no image, no row, classes out of range
           (9, (1 << 20) + 64),                                  # rows overlap dets
           (10, (2 << 20) + 8),                                  # offsets overlap trans
           (11, (3 << 20) + 4),                                  # seen overlaps calib
           (10, (4 << 20) + 100)]                                # offsets overlap rows
    for i, v in bad:
        args = list(ok)
        args[i] = v
        with pytest.raises(RuntimeError, match="cnb_ddd_tail"):
            _C.ddd_tail(*args)
    args = list(ok)
    args[11] = (5 << 20) + 8                                     # seen overlaps offsets
    with pytest.raises(RuntimeError, match="cnb_ddd_tail"):
        _C.ddd_tail(*args)

"""Inputs of tests/golden/ddd_tail.npz (tests/golden/make_golden_ddd_tail.py), the reference's results it stores,
and the comparison of ddd tail results, shared by the CPU and GPU tests, the golden generator and the timing tool.

Golden layout.  `names` lists the tail cases; case `n` has `n_dets` (float32 [B, K, 18] ddd_decode-like rows),
`n_c` (float32 [B, 2]), `n_s` (int32 [B, 2]), `n_calib` (float32 [B, 3, 4]), `n_hw` (output height, width),
`n_form` (0: DddDetector.post_process + merge_outputs once per image, each image with its own calib; 1:
utils.post_process.ddd_post_process on the whole batch, calibs[0] for every image), `n_out` (float32 [R, 15]:
image, class id, then the 13 result columns, in image / class order) and `n_len` (int [B, num_classes]: rows of
each class, -1 for the reference's shape-(0,) empty array).  `pre_names` lists the pre_process cases; case `p` has
`p_img_crc` (CRC32 of the input image, rebuilt by ddd_image), `p_crc` / `p_shape` / `p_sample` (CRC32, shape and a
strided sample of the images tensor), `p_c`, `p_s`, `p_hw` and `p_calib` of the meta."""
import numpy as np

import ddd_tail_np as O

F32 = np.float32
NUM_CLASSES = 3
PEAK_THRESH = 0.2
INPUT_HW = (384, 1280)           # KITTI default resolution (opts.py), output 96 x 320 at down_ratio 4
MEAN = [0.485, 0.456, 0.406]     # datasets/dataset/kitti.py
STD = [0.229, 0.224, 0.225]
ANGLE_TOL = 2.5e-6               # rad, wrapped: numpy's float32 arctan2 is not correctly rounded

# name: (height, width, keep_res)
PRE_CASES = {"p1242": (375, 1242, False), "p1242_keep": (375, 1242, True), "p1241": (376, 1241, False),
             "p1241_keep": (376, 1241, True)}


def ddd_image(h, w, seed=0):
    """Seeded uint8 BGR image (ramps + noise, integer arithmetic only)."""
    rng = np.random.default_rng(5000 + seed + h * 7 + w)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 5 + yy) % 256, (xx + yy * 3) % 256, (xx * yy // 11) % 256], 2)
    return ((base * 3) // 5 + rng.integers(0, 100, (h, w, 3))).astype(np.uint8)


def tail_case(g, name):
    """(dets [B, K, 18], meta of ddd_merge_device, form)."""
    B = g[name + "_dets"].shape[0]
    hw = g[name + "_hw"]
    meta = {"c": [g[name + "_c"][i] for i in range(B)], "s": [g[name + "_s"][i] for i in range(B)],
            "calib": [g[name + "_calib"][i] for i in range(B)], "out_height": int(hw[0]), "out_width": int(hw[1])}
    return g[name + "_dets"], meta, int(g[name + "_form"])


def oracle(dets, meta, form):
    """The numpy restatement on a golden case's inputs."""
    if form == 0:
        return O.detector_tail(dets, meta, NUM_CLASSES, PEAK_THRESH)
    return O.ddd_post_process(dets, meta["c"], meta["s"], meta["calib"], meta["out_width"], meta["out_height"],
                              NUM_CLASSES)


def flatten(res, num_classes=NUM_CLASSES):
    """Per-image {class id: array} -> ([R, 15] rows of image, class id, 13 columns; [B, num_classes] lengths with
    -1 for a shape-(0,) array).  Refuses any other shape and any dtype but float32."""
    rows, lens = [], np.zeros((len(res), num_classes), np.int64)
    for i, r in enumerate(res):
        assert sorted(r.keys()) == list(range(1, num_classes + 1)), sorted(r.keys())
        for j in range(1, num_classes + 1):
            a = r[j]
            assert isinstance(a, np.ndarray) and a.dtype == np.float32, (i, j, type(a), getattr(a, "dtype", None))
            if a.shape == (0,):
                lens[i, j - 1] = -1
                continue
            assert a.ndim == 2 and a.shape[1] == 13, (i, j, a.shape)
            lens[i, j - 1] = len(a)
            rows.append(np.concatenate([np.full((len(a), 1), i, F32), np.full((len(a), 1), j, F32), a], 1))
    return (np.concatenate(rows, 0) if rows else np.zeros((0, 15), F32)), lens


def wrapped_diff(a, b):
    """|a - b| folded into [0, pi] (float64): a +-pi wrap that flips between the two counts as close."""
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) % (2 * np.pi)
    return np.minimum(d, 2 * np.pi - d)


def assert_ddd_equal(got, want, what=""):
    """Flattened results (flatten's pair): same classes, order, lengths and NaN positions; every column bit for bit
    except alpha (column 0) and rot_y (11), which must be within ANGLE_TOL rad of wrapped angular difference."""
    (gr, gl), (wr, wl) = got, want
    np.testing.assert_array_equal(gl, wl, err_msg="%s: class lengths" % what)
    assert gr.shape == wr.shape, (what, gr.shape, wr.shape)
    exact = [0, 1] + [2 + k for k in range(13) if k not in (0, 11)]
    a, b = gr[:, exact], wr[:, exact]
    an, bn = np.isnan(a), np.isnan(b)
    bad = (an != bn) | (~an & ~bn & (a.view(np.uint32) != b.view(np.uint32)))
    if bad.any():
        i, k = np.argwhere(bad)[0]
        raise AssertionError("%s: %d values differ, first row %d column %d: got %r, want %r"
                             % (what, int(bad.sum()), i, exact[k], a[i, k], b[i, k]))
    for col, label in ((2, "alpha"), (13, "rot_y")):
        x, y = gr[:, col], wr[:, col]
        np.testing.assert_array_equal(np.isnan(x), np.isnan(y), err_msg="%s: %s NaN positions" % (what, label))
        ok = ~np.isnan(x)
        if ok.any():
            err = wrapped_diff(x[ok], y[ok]).max()
            assert err <= ANGLE_TOL, "%s: %s off by %.3g rad" % (what, label, err)

"""The multi_pose / exdet tails without a GPU: the numpy oracle (tests/detector_tails_np.py) against the
reference's own MultiPoseDetector / ExdetDetector post_process + merge_outputs stored in
tests/golden/detector_tails.npz, and the argument checks of the device tails and their C ABI, which refuse before anything reaches the device."""
import numpy as np
import pytest
import torch

from detector_tail_cases import exdet_case, multi_pose_case, oracle_exdet, oracle_multi_pose
from helpers import assert_same_bits, flat_results, golden

TAILS = golden("detector_tails")
MP_NAMES = [str(n) for n in TAILS["mp_names"]]
EX_NAMES = [str(n) for n in TAILS["ex_names"]]
LIVE_ROWS = 1000      # the oracle's soft-NMS is plain Python, O(N^2): longer lists are checked on the GPU only


def test_golden_covers_the_cases():
    """The golden keeps the cases the GPU tests rely on."""
    flips, scales, rows = set(), set(), []
    for n in EX_NAMES:
        dets, metas, nc, mpi, flip = exdet_case(TAILS, n)
        flips.add(flip); scales.add(len(dets))
        p = 2 if flip else 1
        rows.append(sum(p * d.shape[1] for d in dets))
        s = np.concatenate([d[..., 4].ravel() for d in dets])
        if n == "list4096":
            out = TAILS[n + "_out"]
            assert (out[:, 1] == 2).sum() == 4096 and mpi > rows[-1]        # one class list of exactly 4096 rows
    assert flips == {False, True} and scales == {1, 2, 5}
    assert max(rows) > 4096                                                # the wide cut
    allsc = np.concatenate([d[..., 4].ravel() for n in EX_NAMES for d in exdet_case(TAILS, n)[0]])
    assert np.isnan(allsc).any() and np.isposinf(allsc).any() and (allsc < 0).any()
    assert (np.signbit(allsc) & (allsc == 0)).any()                       # -0.0
    assert {bool(int(TAILS[n + "_nms"])) for n in MP_NAMES} == {False, True}


def _longest_list(dets, nc, flip):
    p = 2 if flip else 1
    longest = 0
    for i in range(dets[0].shape[0] // p):
        rows = np.concatenate([d[p * i:p * i + p].reshape(-1, 14) for d in dets])
        rows = rows[rows[:, 4] > 0]
        longest = max([longest] + [int((rows[:, 13] == j).sum()) for j in range(nc)])
    return longest


@pytest.mark.parametrize("name", EX_NAMES)
def test_oracle_exdet_tail(name):
    """post_process (un-mirroring of the second half, back-projection, division by the scale) and merge_outputs
    (score > 0, per-class soft-NMS, cut), every row of every class list, bit for bit."""
    dets, metas, nc, mpi, flip = exdet_case(TAILS, name)
    if _longest_list(dets, nc, flip) > LIVE_ROWS:
        pytest.skip("class lists longer than %d rows: checked against the stored reference on the GPU" % LIVE_ROWS)
    got = oracle_exdet(dets, metas, nc, mpi, flip)
    assert_same_bits(flat_results(got, nc), TAILS[name + "_out"], name)


@pytest.mark.parametrize("name", MP_NAMES)
def test_oracle_multi_pose_tail(name):
    dets, metas, nms = multi_pose_case(TAILS, name)
    assert_same_bits(oracle_multi_pose(dets, metas, nms), TAILS[name + "_out"], name)


def test_oracle_exdet_odd_rows_raise():
    """Without flip the reference splits an image's N rows in two (reshape(2, -1, 14)): an odd N raises."""
    import detector_tails_np as O
    with pytest.raises(ValueError):
        O.exdet_post_process(np.zeros((1, 7, 14), np.float32), {"c": [1, 1], "s": 4.0, "out_width": 8,
                                                                "out_height": 8})


def _meta(b):
    return {"c": [np.zeros(2, np.float32)] * b, "s": [64.0] * b, "out_height": 16, "out_width": 16}


def test_cpu_tensors_raise():
    from centernet_b200 import post_process as P
    with pytest.raises(NotImplementedError, match="CUDA"):
        P.exdet_merge_device([torch.zeros(2, 8, 14)], [_meta(1)], 80, flip=True)
    with pytest.raises(NotImplementedError, match="CUDA"):
        P.multi_pose_merge_device([torch.zeros(1, 8, 40)], [_meta(1)])
    with pytest.raises(NotImplementedError, match="CUDA"):
        P.exdet_merge_device([np.zeros((2, 8, 14), np.float32)], [_meta(1)], 80)


def test_abi_rejections():
    """Every argument is checked before a launch (fake pointers never reach the device)."""
    from centernet_b200 import _C
    bad_transform = [(0, 32, 48, 1, 4, 14, 8.0, 0),         # null pointer
                     (16, 16, 48, 1, 4, 14, 8.0, 0),        # out aliases rows
                     (16, 32, 48, 0, 4, 14, 8.0, 0),        # no image
                     (16, 32, 48, 1, 4, 3, 8.0, 0),         # fewer than 4 columns
                     (16, 32, 48, 1, 7, 14, 8.0, 0)]        # odd rows: no two equal halves
    for args in bad_transform:
        with pytest.raises(RuntimeError, match="cnb_exdet_transform"):
            _C.exdet_transform(*args)
    for args in [(16, 1, 8, 14, 14, 80, 32, 48, 0), (16, 1, 8, 4, 3, 80, 32, 48, 0), (16, 1, 8, 14, 13, 0, 32, 48, 0),
                 (16, 1, 8, 14, 13, 8193, 32, 48, 0), (0, 1, 8, 14, 13, 80, 32, 48, 0)]:
        with pytest.raises(RuntimeError, match="cnb_group_positive_by_class"):
            _C.group_positive_by_class(*args)
    nms_ok = [16, 16, 32, 1, 80, 8192, 4096, 5, 0.5, 0.5, 0.001, 2, 0, 0]
    for i, v in [(0, 0), (5, 0), (6, 0), (7, 4), (11, 3), (1, 16)]:   # null, stride, list cap, width, method, alias
        args = list(nms_ok); args[i] = v
        if i == 1:
            args[7] = 39
        with pytest.raises(RuntimeError, match="cnb_soft_nms_strided"):
            _C.soft_nms_strided(*args)
    for args in [(16, 0, 32, 5, 48, 80, 100, 64, 0, 0), (16, 1, 32, 4, 48, 80, 100, 64, 0, 0),
                 (16, 1, 32, 5, 48, 80, 0, 64, 0, 0), (0, 1, 32, 5, 48, 80, 100, 64, 0, 0)]:
        with pytest.raises(RuntimeError, match="cnb_topk_keep_wide"):
            _C.topk_keep_wide(*args)


def test_capacity_refusals():
    """More than 32768 rows per image or 4096 rows per soft-NMS list: NotImplementedError (CNB_EUNSUPPORTED)."""
    from centernet_b200 import _C
    with pytest.raises(NotImplementedError, match="32768"):
        _C.soft_nms_strided(16, 16, 32, 1, 80, 32769, 4096, 5, 0.5, 0.5, 0.001, 2, 0, 0)
    with pytest.raises(NotImplementedError, match="4096"):
        _C.soft_nms_strided(16, 16, 32, 1, 80, 32768, 4097, 5, 0.5, 0.5, 0.001, 2, 0, 0)
    with pytest.raises(NotImplementedError, match="32768"):
        _C.topk_keep_wide(16, 1, 32769, 5, 48, 80, 100, 64, 0, 0)

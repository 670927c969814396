"""CPU: pins the torch selection reference (oracle/select_torch.py), which the GPU selection tests compare the
kernels with, to the numpy oracle on every map distribution of tests/select_maps.py and to the unmodified
reference's own outputs (tests/golden/big_ctdet_*.npz), and pins the library's rule for non-finite scores on
hand-checked maps."""
import numpy as np
import pytest
import torch

import big_inputs as BI
import select_maps as SM
from helpers import golden
from oracle import decode_np as O
from oracle import select_torch as ST

FINITE = SM.KINDS      # every distribution is finite


@pytest.mark.parametrize("kind", FINITE)
@pytest.mark.parametrize("B,C,H,W,K", [(2, 3, 12, 20, 9), (1, 4, 9, 13, 40), (2, 2, 8, 12, 96)])
def test_reference_equals_numpy_oracle(kind, B, C, H, W, K):
    heat = SM.make_map(kind, B, C, H, W, seed=7 + K)
    g = torch.Generator().manual_seed(3)
    wh = torch.rand(B, 2 * C, H, W, generator=g) * 16
    reg = torch.rand(B, 2, H, W, generator=g)
    for r, cat in ((reg, False), (None, False), (reg, True)):
        w = wh if cat else wh[:, :2].contiguous()
        want = O.ctdet_decode(heat.numpy(), w.numpy(), None if r is None else r.numpy(), cat_spec_wh=cat, K=K)
        got = ST.ctdet_decode(heat, w, r, cat_spec_wh=cat, K=K).numpy()
        assert np.array_equal(got, want), (kind, cat, r is None)
        # the library's non-finite rule changes nothing on a finite map
        assert np.array_equal(ST.ctdet_decode(heat, w, r, cat, K, nonfinite="library").numpy(), want)
    s, i, c, y, x = ST.topk(ST.nms(heat), K)
    for a, b in zip((s, i, c, y, x), O.topk(O.nms(heat.numpy()), K)):
        assert np.array_equal(a.numpy(), b)
    s, i, y, x = ST.topk_channel(ST.nms(heat), min(K, H * W))
    for a, b in zip((s, i, y, x), O.topk_channel(O.nms(heat.numpy()), min(K, H * W))):
        assert np.array_equal(a.numpy(), b)


@pytest.mark.parametrize("kind", ["noise", "blobs"])
def test_reference_reproduces_big_goldens(kind):
    g = golden("big_ctdet_" + kind)
    heat, wh, reg = BI.ctdet_inputs(kind)
    assert BI.checksum(heat, wh, reg) == g["crc"]
    h, w, r = (torch.from_numpy(a) for a in (heat, wh, reg))
    got = ST.ctdet_decode(h, w, r, K=100).numpy()
    # the goldens come from torch.topk, which leaves the order of equal scores open: per tie group as a multiset
    from helpers import assert_dets_equal
    assert_dets_equal(g["dets"], got, what="big " + kind)
    assert_dets_equal(g["dets_noreg"], ST.ctdet_decode(h, w, None, K=100).numpy(), what="big noreg " + kind)
    # ... and in our tie order exactly what the numpy oracle returns
    assert np.array_equal(got, O.ctdet_decode(heat, wh, reg, K=100))


def test_signed_zero_fillers_in_index_order():
    """heat * keep leaves -0.0 at negative non-peaks and +0.0 at zero ones; both are the value 0 and rank by index."""
    heat = torch.tensor([[[[-0.5, 0.0, -0.5, -0.25, -0.5, 0.0]]]])
    v = ST.nms(heat)
    assert torch.signbit(v).tolist() == [[[[True, False, True, True, True, False]]]]
    s, i, c, y, x = ST.topk(v, 6)
    assert s.tolist() == [[0.0, 0.0, 0.0, 0.0, 0.0, -0.25]]
    assert i.tolist() == [[0, 1, 2, 4, 5, 3]]


def test_library_nonfinite_rule():
    nan, inf = float("nan"), float("inf")
    heat = torch.full((1, 1, 5, 6), -0.25)
    heat[0, 0, 0, 0] = nan          # NaN: scores 0 and is left out of its neighbours' 3x3 maximum
    heat[0, 0, 0, 1] = -0.5         # non-peak (the NaN beside it does not make it one): 0
    heat[0, 0, 4, 5] = inf          # +inf peak
    heat[0, 0, 2, 2] = -inf         # non-peak -inf: scores 0
    heat[0, 0, 3:5, 0:2] = -inf     # 2x2 -inf block at the border: (4, 0) sees only -inf around it
    heat[0, 0, 3, 2] = nan
    v = ST.nms(heat, nonfinite="library")[0, 0]
    assert v[0, 0] == 0 and v[3, 2] == 0                            # NaN
    assert v[2, 2] == 0                                             # -inf next to -0.25
    assert v[4, 5] == inf
    assert v[4, 0] == -inf and v[4, 1] == 0 and v[3, 0] == 0        # only (4, 0) has no finite neighbour
    assert v[0, 1] == 0 and v[1, 0] == -0.25                        # -0.25 beside the NaN is still a peak
    assert not torch.isnan(v).any()
    s, i, c, y, x = ST.topk(ST.nms(heat, nonfinite="library"), 30)
    assert s[0, 0] == inf and i[0, 0] == 29
    zeros = i[0][s[0] == 0].tolist()
    assert zeros == sorted(zeros) and set(zeros) == {0, 1, 14, 18, 19, 20, 22, 23, 25, 28}
    assert s[0, -1] == -inf and i[0, -1] == 24
    assert (s[0, 11:-1] == -0.25).all() and i[0, 11:-1].tolist() == sorted(i[0, 11:-1].tolist())
    # +inf plateau: every +inf pixel is a peak, ties by index
    heat = torch.zeros(1, 2, 4, 4)
    heat[0, 1, 1:3, 1:3] = inf
    s, i, c, y, x = ST.topk(ST.nms(heat, nonfinite="library"), 4)
    assert s.tolist() == [[inf] * 4] and (c * 16 + i).tolist() == [[21, 22, 25, 26]]

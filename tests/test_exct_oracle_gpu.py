"""GPU: exct_decode / agnex_ct_decode (exct.cu: k_exct_tuples, k_exct_merge, the centre-map passes) against an
independent reference, oracle/exct_torch.py (pinned to the numpy oracle and to the reference's golden by
tests/test_exct_oracle.py), in every group and candidate-buffer regime, at num_dets up to 2048, on ties, plateaus,
pruning-hostile maps, map edges and non-finite values.

Bar: every row of the output, filler rows included, equals the reference's on all 14 columns, bit for bit (the sign
of zero included; a NaN matches a NaN).  Every case runs through both exct_decode and agnex_ct_decode on the same
inputs.  The group count of each case is asserted through cnb_exct_groups on the SM count of the device the suite
runs on."""
import numpy as np
import pytest
import torch

from helpers import assert_same_bits
from oracle import exct_torch as E

pytestmark = pytest.mark.gpu
NEG_NAN = np.array([0xffc00000], np.uint32).view(np.float32)[0]   # x86's default NaN (inf - inf): sign bit set


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _groups(B, K, nd):
    from centernet_b200 import _C
    return _C.exct_groups(B, K, nd)


def _expected_groups(B, K, nd):
    return max(1, min(16, -(-2 * _sms() // B), K, 16384 // nd))


def _rand(shape, seed, lo=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(shape, generator=g) * (hi - lo) + lo


def _regs(B, H, W, seed):
    return [_rand((B, 2, H, W), seed + q, -0.5, 0.5) for q in range(4)]


def _run(maps, ct, regs, K, nd, agnostic, logits=False, **kw):
    """The library's decode (on CUDA, in the inputs' dtype) and the reference's (on the .float() upcast, after
    torch's CUDA sigmoid with logits), as numpy arrays."""
    from centernet_b200 import decode as D
    dev = [m.cuda() for m in maps], ct.cuda(), [None if r is None else r.cuda() for r in regs]
    name = ("agnex_ct_decode" if agnostic else "exct_decode") + ("_from_logits" if logits else "")
    got = getattr(D, name)(*dev[0], dev[1], *dev[2], K=K, num_dets=nd, **kw)
    fm = [m.float() for m in dev[0]] + [dev[1].float()]
    if logits:
        fm = [torch.sigmoid(m) for m in fm]
    ref = E.agnex_ct_decode if agnostic else E.exct_decode
    want = ref(*fm, *[None if r is None else r.float() for r in dev[2]], K=K, num_dets=nd, **kw)
    return got.cpu().numpy(), want.cpu().numpy()


def _check(maps, ct, regs, K, nd, what, groups=None, **kw):
    """Both decodes against the reference; returns the reference's (per class, agnostic) dets."""
    B = maps[0].shape[0]
    out = []
    for agnostic in (False, True):
        got, want = _run(maps, ct, regs, K, nd, agnostic, **kw)
        assert got.shape == (B, nd, 14)
        assert_same_bits(got, want, "%s (%s)" % (what, "agnostic" if agnostic else "per class"))
        out.append(want)
    if groups is not None:
        assert _groups(B, K, nd) == groups, (what, _groups(B, K, nd), groups)
    return out


def _boxes(B, C, H, W, seed, n_obj=12, base=0.03):
    """t/l/b/r/centre maps with boxes whose extreme points and centre carry peaks of one class, on low noise."""
    rng = np.random.default_rng(seed)
    m = (base * rng.random((5, B, C, H, W))).astype(np.float32)
    for b in range(B):
        for _ in range(n_obj):
            c = rng.integers(0, C)
            x0, x1 = sorted(rng.integers(0, W, 2)); y0, y1 = sorted(rng.integers(0, H, 2))
            tx, bx = rng.integers(x0, x1 + 1, 2); ly, ry = rng.integers(y0, y1 + 1, 2)
            sc = rng.uniform(0.3, 0.95, 5).astype(np.float32)
            m[0, b, c, y0, tx] = sc[0]; m[1, b, c, ly, x0] = sc[1]
            m[2, b, c, y1, bx] = sc[2]; m[3, b, c, ry, x1] = sc[3]
            m[4, b, c, (y0 + y1) // 2, (x0 + x1) // 2] = sc[4]
    t = [torch.from_numpy(np.ascontiguousarray(m[i])) for i in range(5)]
    return t[:4], t[4]


def _uniform(B, C, H, W, seed):
    maps = [_rand((B, C, H, W), seed + q) for q in range(5)]
    return maps[:4], maps[4]


# ------------------------------------------------------------------ group regimes
def test_default_group_count_unchanged():
    """The default num_dets = 1000 keeps 16 groups at small batch."""
    assert _groups(1, 40, 1000) == 16
    assert _groups(2, 100, 1000) == 16


def test_one_group_large_batch():
    """B >= 2 * SMs: one CTA per image."""
    B = 2 * _sms()
    maps, ct = _uniform(B, 2, 8, 8, 11)
    _check(maps, ct, _regs(B, 8, 8, 20), 5, 100, "one group, B=%d" % B, groups=1)


def test_one_group_k1():
    maps, ct = _boxes(1, 3, 12, 12, 3)
    _check(maps, ct, _regs(1, 12, 12, 30), 1, 1, "K=1", groups=1)


@pytest.mark.parametrize("K", [2, 7, 13])
def test_k_groups(K):
    """K < 16: one group per top index."""
    maps, ct = _uniform(1, 3, 16, 20, K)
    _check(maps, ct, _regs(1, 16, 20, 40), K, min(500, K ** 4), "K groups", groups=K, scores_thresh=0.05,
           center_thresh=0.05)


def test_intermediate_group_count():
    """B such that ceil(2 * SMs / B) = 5."""
    B = (2 * _sms() + 4) // 5
    maps, ct = _boxes(B, 2, 16, 16, 8, n_obj=4)
    _check(maps, ct, _regs(B, 16, 16, 50), 20, 200, "intermediate groups, B=%d" % B, groups=5)


# ------------------------------------------------------------------ num_dets and the candidate buffer
@pytest.mark.parametrize("nd", [1, 5, 1024, 1025, 2048])
def test_num_dets_16_groups(nd):
    """B = 1, K = 20: 1 (one key per group), 5 (the shared threshold rises at once), 1024 (16 x 1024 keys in the
    merge), 1025 and 2048 (more than 16384 keys over 16 groups: the group count must shrink)."""
    maps, ct = _uniform(1, 3, 24, 24, 100 + nd)
    _check(maps, ct, _regs(1, 24, 24, 60), 20, nd, "num_dets=%d" % nd, groups=_expected_groups(1, 20, nd),
           scores_thresh=0.05, center_thresh=0.05)


def test_num_dets_k4_every_tuple():
    """num_dets = K^4 = 1296: every tuple comes back, in (score desc, index asc) order."""
    maps, ct = _boxes(1, 2, 14, 14, 9, n_obj=3)
    _check(maps, ct, _regs(1, 14, 14, 70), 6, 6 ** 4, "num_dets=K^4", groups=6)


@pytest.mark.parametrize("B,nd", [(1, 2048), (32, 2048), (8, 1500)])
def test_num_dets_above_1024_at_small_batch(B, nd):
    maps, ct = _uniform(B, 2, 16, 16, B + nd)
    _check(maps, ct, _regs(B, 16, 16, 80), 16, nd, "B=%d num_dets=%d" % (B, nd),
           groups=_expected_groups(B, 16, nd), scores_thresh=0.0, center_thresh=0.0)


@pytest.mark.parametrize("K", [45, 46, 64])
def test_step_geometry(K):
    """K^2 below one 2048-tuple step (45), one full step and a 68-tuple remainder (46), two exact steps (64); with
    num_dets = 2048 the first two steps of a group fill the 4096-key buffer exactly."""
    maps, ct = _uniform(1, 2, 24, 24, K)
    _check(maps, ct, _regs(1, 24, 24, 90), K, 2048, "K=%d" % K, groups=_expected_groups(1, K, 2048),
           scores_thresh=0.05, center_thresh=0.05)


def test_many_cut_rounds_constant_maps():
    """Every valid tuple ties: the order is the tuple index across groups, cut rounds and the pruning test (which
    may not skip a block whose bound equals the threshold)."""
    B, C, H, W, K = 1, 1, 12, 12, 40
    maps = [torch.full((B, C, H, W), 0.5) for _ in range(4)]
    _check(maps, torch.full((B, C, H, W), 0.5), _regs(B, H, W, 95), K, 300, "constant", groups=16)


@pytest.mark.parametrize("nd", [100, 2048])
def test_constant_centre_on_structured_maps(nd):
    maps, _ = _boxes(2, 3, 20, 24, 12, n_obj=10)
    _check(maps, torch.full((2, 3, 20, 24), 0.4), _regs(2, 20, 24, 96), 30, nd, "constant centre")


# ------------------------------------------------------------------ ties, plateaus, thresholds, signed zeros
def test_aggregated_plateaus():
    """Aggregation pushes ridges above 1; the clamp turns them into plateaus of 1."""
    maps, ct = _uniform(2, 2, 16, 16, 7)
    maps = [(m * 0.3 + 0.75).contiguous() for m in maps]
    _check(maps, ct, _regs(2, 16, 16, 97), 12, 400, "aggregated plateaus", aggr_weight=0.5)


def test_inf_peaks_clamp_to_one():
    maps, ct = _boxes(1, 2, 16, 16, 13)
    for q, m in enumerate(maps):
        m[0, q % 2, 3 + q, 2:14:3] = float("inf")
    _check(maps, ct, _regs(1, 16, 16, 98), 10, 300, "+inf peaks")


def test_scores_on_the_thresholds():
    """Map values exactly at scores_thresh and centre values exactly at center_thresh are not penalised (the
    comparison is strict), values one ulp below are."""
    q = torch.tensor([0.25, 0.5, np.nextafter(np.float32(0.25), np.float32(0)), 0.75])
    maps = [q[torch.randint(0, 4, (1, 2, 12, 12), generator=torch.Generator().manual_seed(s))] for s in range(4)]
    ct = q[torch.randint(0, 4, (1, 2, 12, 12), generator=torch.Generator().manual_seed(9))]
    _check(maps, ct, _regs(1, 12, 12, 99), 15, 500, "thresholds", scores_thresh=0.25, center_thresh=0.25)


@pytest.mark.parametrize("ct_kind", ["zero", "neg_zero", "neg_subnormal"])
def test_signed_zero_scores(ct_kind):
    """All -0 extreme maps.  With a centre of -0 or of a negative subnormal (whose sum / 6 rounds to -0), tuples
    score -0 or +0; the rule treats both as one value ordered by tuple index."""
    B, C, H, W, K = 1, 2, 8, 10, 12
    maps = [torch.full((B, C, H, W), -0.0) for _ in range(4)]
    ct = torch.zeros(B, C, H, W)
    if ct_kind == "neg_zero":
        ct[..., ::2] = -0.0
    elif ct_kind == "neg_subnormal":
        ct[..., 1::3] = -1e-45
    outs = _check(maps, ct, _regs(B, H, W, 100), K, 600, "signed zeros " + ct_kind, scores_thresh=0.0,
                  center_thresh=-1.0)
    assert (outs[0][..., 4] == 0).sum() > 100


def test_quantised_maps_many_ties_at_the_cut():
    """Four score levels: thousands of tuples share the num_dets-th score, so the cut, the shared threshold and the
    pruning bound all meet ties."""
    lv = torch.tensor([0.2, 0.4, 0.6, 0.8])
    g = torch.Generator().manual_seed(5)
    maps = [lv[torch.randint(0, 4, (2, 3, 20, 20), generator=g)] for _ in range(4)]
    ct = lv[torch.randint(0, 4, (2, 3, 20, 20), generator=g)]
    _check(maps, ct, _regs(2, 20, 20, 101), 25, 50, "quantised")


def test_pruning_centre_outlier_and_negative_maps():
    """One centre value far above the rest keeps the pruning bound loose; negative extreme maps give non-positive
    candidates."""
    maps, ct = _boxes(2, 4, 24, 28, 14, n_obj=10)
    maps = [(m - 0.02).contiguous() for m in maps]
    ct[0, 1, 5, 5] = 1000.0
    ct[1, 3, 20, 2] = 50.0
    _check(maps, ct, _regs(2, 24, 28, 102), 30, 64, "centre outlier")


# ------------------------------------------------------------------ geometry
@pytest.mark.parametrize("B,C,H,W,K,nd", [(1, 1, 3, 3, 9, 2048), (2, 1, 2, 7, 5, 300), (1, 80, 32, 24, 20, 1000),
                                          (3, 1, 17, 5, 11, 700)])
def test_shapes(B, C, H, W, K, nd):
    maps, ct = _uniform(B, C, H, W, K + C)
    _check(maps, ct, _regs(B, H, W, 103), K, nd, "shape %s" % ((B, C, H, W, K),), scores_thresh=0.02,
           center_thresh=0.02)


def test_peaks_on_the_last_row_and_column():
    """Peaks on the map's last row and column, and odd l_x + r_x / t_y + b_y sums (the centre rounds down)."""
    B, C, H, W = 1, 2, 9, 13
    maps = [torch.zeros(B, C, H, W) for _ in range(4)]
    ct = _rand((B, C, H, W), 3, 0.2, 0.9)
    for q, m in enumerate(maps):
        m[0, :, H - 1, ::2] = 0.5 + 0.05 * q
        m[0, :, ::3, W - 1] = 0.6 + 0.05 * q
        m[0, :, 0, 1::4] = 0.7
    _check(maps, ct, _regs(B, H, W, 104), 16, 500, "last row / column", scores_thresh=0.0)


# ------------------------------------------------------------------ non-finite values
@pytest.mark.parametrize("val", ["nan", "neg_nan", "inf", "-inf"])
@pytest.mark.parametrize("cls", [0, 2])
def test_nonfinite_centre(val, cls):
    """A patch of the centre map of class cls set to val.  A NaN of either sign makes its tuples NaN, which rank
    first whatever their penalties; k_exct_tuples' block bound must not prune them.  In the agnostic decode the
    maximum over classes propagates the NaN (torch.max)."""
    B, C, H, W, K = 2, 3, 24, 24, 30
    maps, ct = _boxes(B, C, H, W, 15, n_obj=14)
    v = {"nan": float("nan"), "neg_nan": float(NEG_NAN), "inf": float("inf"), "-inf": float("-inf")}[val]
    ct[:, cls, 12:20, 10:22] = v
    if val == "neg_nan":
        assert (ct.view(torch.int32) == -4194304).any()          # the sign bit survived
    outs = _check(maps, ct, _regs(B, H, W, 105), K, 10, "centre %s class %d" % (val, cls))
    if "nan" in val:
        assert np.isnan(outs[1][..., 4]).any()                   # agnostic: every class's NaN reaches the max


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("val", ["nan", "neg_nan"])
def test_nan_centre_behind_pruned_blocks(val, dtype):
    """A NaN column on the centre map's right edge is reached only by tuples whose left and right points both lie
    on that column.  The one left peak there ranks low and sits right of every top point, so its (top, left) blocks
    carry the left penalty and come up when the threshold has long risen above their finite bound.  Their NaN tuples
    still rank first, so that bound must count a NaN of either sign as above every number.  fp32 takes k_ct_max;
    fp16 and bf16 take k_ct_scores (bf16 widens by a shift, which keeps the sign bit of a NaN)."""
    B, C, H, W, K = 1, 2, 24, 24, 30
    maps, ct = _boxes(B, C, H, W, 19, n_obj=12)
    for m in maps:
        m[..., W - 2:] = 0.0                                       # no other peak near the edge
    maps[1][0, 0, 5, W - 1] = 0.2                                   # left point on the last column
    maps[3][0, 1, 9, W - 1] = 0.6                                   # right point on the last column
    ct = ct.to(dtype)
    bits = ct.view(torch.int32 if dtype == torch.float32 else torch.int16)
    if val == "neg_nan":   # 0xffc00000 / 0xfe00 / 0xffc0
        bits[..., W - 1] = {torch.float32: -4194304, torch.float16: -512, torch.bfloat16: -64}[dtype]
    else:
        ct[..., W - 1] = float("nan")
    # scores_thresh above that left point's score: a second penalty on those blocks
    outs = _check(maps, ct, _regs(B, H, W, 112), K, 10, "NaN column %s %s" % (val, dtype), scores_thresh=0.25)
    for want in outs:
        assert np.isnan(want[..., 4]).all()


def test_inf_minus_inf_behind_pruned_blocks():
    """A NaN tuple made by arithmetic: a -inf right score (a -inf peak of a map that is -inf almost everywhere) plus
    a +inf centre value.  Top and left maps are finite, so the block bound of such a tuple is +inf, not NaN.
    Top point 1 reaches a +inf band of the centre map through every left point, so group 1 publishes NaN-level
    thresholds after a few blocks; top point 0 reaches the +inf right column only through the last-ranked left point
    (on the right edge).  Those later blocks of group 0 hold the NaN tuples of lowest index, the first rows of the
    result, and must not be pruned against group 1's threshold."""
    B, C, H, W, K, nd = 1, 1, 24, 16, 30, 10
    t = torch.zeros(B, C, H, W)
    t[0, 0, 2, 5] = 0.9                                             # top point 0: row 2
    t[0, 0, H - 1, 8] = 0.8                                         # top point 1: the last row
    for q in range(12):                                             # the other top points: rows 4..9, lower scores
        t[0, 0, 4 + q // 3 * 2, 1 + q % 3 * 4] = 0.5 - 0.01 * q
    l = torch.zeros(B, C, H, W)
    for q in range(20):                                             # 20 left points left of column 13
        l[0, 0, 1 + q // 4 * 4, 1 + q % 4 * 3] = 0.9 - 0.02 * q
    l[0, 0, 5, W - 1] = 0.2                                         # ranked after them: on the last column
    b = torch.zeros(B, C, H, W)
    for q in range(8):                                              # bottom points on rows 17..23
        b[0, 0, 17 + q % 7, 1 + q * 2] = 0.7 - 0.02 * q
    r = torch.full((B, C, H, W), float("-inf"))
    r[0, 0, 20, 8] = 0.6                                            # one finite right peak, far from row 0
    ct = torch.full((B, C, H, W), 0.5)
    ct[0, 0, 20:, :] = float("inf")                                 # reached only from top point 1
    ct[0, 0, :, W - 1] = float("inf")                               # reached only with l_x = r_x = W - 1
    outs = _check([t, l, b, r], ct, _regs(B, H, W, 113), K, nd, "inf - inf", groups=16, scores_thresh=-10.0,
                  center_thresh=-10.0)
    for want in outs:   # every row NaN, every one from top point 0 (t_y = 2 plus a regression in [-0.5, 0.5])
        assert np.isnan(want[..., 4]).all() and (np.abs(want[..., 6] - 2) <= 0.5).all()


@pytest.mark.parametrize("val", ["nan", "inf", "-inf"])
def test_nonfinite_extreme_maps(val):
    """NaN / inf in the four extreme maps follow the selection's rule: NaN scores 0, +inf clamps to 1, a -inf peak
    scores -inf."""
    B, C, H, W, K = 1, 2, 16, 16, 12
    maps, ct = _boxes(B, C, H, W, 16)
    v = float(val)
    maps[0][0, 0, 2:6, 2:6] = v
    maps[1][0, 1, :, 4] = v
    maps[2][0, :, 10, 8:] = v
    maps[3][0, 0, 7, 15] = v
    _check(maps, ct, _regs(B, H, W, 106), K, 400, "extreme maps %s" % val, scores_thresh=-10.0)
    if val == "-inf":   # every pixel a -inf peak: -inf + -inf ... and a centre of +inf make NaN tuples
        allneg = [torch.full((B, C, 5, 5), v) for _ in range(4)]
        ctp = torch.full((B, C, 5, 5), float("inf"))
        _check(allneg, ctp, [None] * 4, 4, 256, "all -inf, centre +inf", scores_thresh=-10.0)


def test_nonfinite_regression():
    """NaN / inf in the regression heads reach the coordinate columns only."""
    B, C, H, W, K = 1, 2, 16, 16, 14
    maps, ct = _boxes(B, C, H, W, 17)
    regs = _regs(B, H, W, 107)
    regs[0][0, 0, :8] = float("nan")
    regs[1][0, 1, :, :5] = float("inf")
    regs[2][0, 0, 8:, :] = float("-inf")
    regs[3][0, :, 3:9, 3:9] = float("nan")
    _check(maps, ct, regs, K, 300, "regression non-finite")


# ------------------------------------------------------------------ dtypes and logits (same host body)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_inputs_nonfinite_centre(dtype):
    """A half centre map is widened exactly, its NaNs keep their sign."""
    B, C, H, W, K = 1, 3, 20, 20, 20
    maps, ct = _boxes(B, C, H, W, 18, n_obj=12)
    ct[0, 2, 0:4, :] = float("inf")
    ct = ct.to(dtype)
    ct.view(torch.int16)[0, 1, 8:16, 6:18] = -64 if dtype == torch.bfloat16 else -512   # 0xffc0 / 0xfe00: -NaN
    assert torch.isnan(ct).sum() == 96
    maps = [m.to(dtype) for m in maps]
    regs = [r.to(dtype) for r in _regs(B, H, W, 108)]
    _check(maps, ct, regs, K, 12, "%s" % dtype)


@pytest.mark.parametrize("nd", [40, 2048])
def test_logits(nd):
    B, C, H, W, K = 2, 2, 16, 16, 18
    maps = [_rand((B, C, H, W), 200 + q, -6.0, 3.0) for q in range(4)]
    ct = _rand((B, C, H, W), 210, -6.0, 3.0)
    _check(maps, ct, _regs(B, H, W, 109), K, nd, "logits", logits=True)
    _check(maps, ct, _regs(B, H, W, 109), K, nd, "logits, aggregated", logits=True, aggr_weight=0.1)


# ------------------------------------------------------------------ sizes
def test_num_dets_zero_raises():
    """num_dets = 0 is rejected by the call (the fp32 workspace query, which runs first, sizes it harmlessly)."""
    from centernet_b200 import decode as D
    maps, ct = _uniform(1, 2, 16, 16, 1)
    for fn in (D.exct_decode, D.agnex_ct_decode):
        with pytest.raises(RuntimeError, match="non-positive"):
            fn(*[m.cuda() for m in maps], ct.cuda(), K=8, num_dets=0)


@pytest.mark.parametrize("K", [40, 100])
def test_large_k(K):
    maps, ct = _boxes(2, 4, 64, 64, K, n_obj=30)
    _check(maps, ct, _regs(2, 64, 64, 110), K, 1000, "K=%d" % K, groups=16)


def test_k255_one_image():
    """K = 255, the largest the ABI accepts: 4.2e9 tuples."""
    maps, ct = _boxes(1, 2, 32, 32, 255, n_obj=40)
    _check(maps, ct, _regs(1, 32, 32, 111), 255, 1000, "K=255", groups=16)

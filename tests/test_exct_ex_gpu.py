"""exct_decode / agnex_ct_decode from the maps' raw logits and from bf16 / fp16 inputs, and the edge aggregation of
half maps.

Contract 1: exct_decode_from_logits(t, l, b, r, ct, <regs>, ...) == exct_decode(torch.sigmoid(t), ..., torch.sigmoid(ct),
<regs>, ...) bit for bit, filler rows included, with torch's own CUDA sigmoid on the right; the same for
agnex_ct_decode_from_logits.  Contract 2: the four functions return for half inputs (any mix of dtypes, aligned or
not) what they return for their .float() upcast.  Contract 3: the aggregation helpers return for a half map the fp32
result of its .float() upcast.  The fp32 decodes on the right are pinned against the reference elsewhere
(test_pose_aggr_loss_gpu.py, test_big_golden.py)."""
import pytest
import torch

import big_inputs as BI

pytestmark = pytest.mark.gpu

HALF = [torch.bfloat16, torch.float16]
HIDS = ["bf16", "fp16"]
# (B, C, H, W): hot 128x128, two non-hot geometries, and 72x90 (rows not a whole number of 16-byte pieces in any
# dtype: the fallback aggregation kernels)
SHAPES = [(1, 80, 128, 128), (2, 4, 96, 160), (2, 3, 64, 64), (1, 5, 72, 90)]
SIDS = ["128x128", "96x160", "64x64", "72x90"]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _sig(t):
    return None if t is None else torch.sigmoid(t)


def _up(t):
    return None if t is None else t.float()


def _logit_inputs(B, C, H, W, seed, agnostic=False):
    """Gaussian logits of the five maps (a few percent of the peaks pass 0.1) and the four regression maps."""
    g = _gen(seed)
    cm = 1 if agnostic else C
    maps = [torch.randn(B, cm, H, W, device="cuda", generator=g) * 1.5 - 3.0 for _ in range(4)]
    maps.append(torch.randn(B, C, H, W, device="cuda", generator=g) * 1.5 - 3.0)
    regs = [torch.rand(B, 2, H, W, device="cuda", generator=g) for _ in range(4)]
    return maps, regs


def _golden_logits(B=1, C=80, seed=319):
    """tests/big_inputs.exct_inputs (boxes whose extreme points and centre carry peaks) turned into logits."""
    maps, regs = BI.exct_inputs(seed=seed, B=B, C=C)
    maps = [torch.logit(torch.from_numpy(m).cuda()) for m in maps]
    return maps, [torch.from_numpy(r).cuda() for r in regs]


def _fns(agnostic):
    from centernet_b200 import decode as D
    if agnostic:
        return D.agnex_ct_decode, D.agnex_ct_decode_from_logits
    return D.exct_decode, D.exct_decode_from_logits


def _check(maps, regs, agnostic, K, aggr, dtypes=None, st=0.1, ct_th=0.1, nd=1000, offset=False):
    """Both contracts on one input set: logits in the given per-tensor dtypes (default fp32)."""
    dec, dec_logits = _fns(agnostic)
    ins = list(maps) + list(regs if regs is not None else [None] * 4)
    if dtypes is not None:
        ins = [None if t is None else t.to(dt) for t, dt in zip(ins, dtypes)]
    if offset:  # a storage offset of one element: no base is 16-byte aligned (no TMA, no in-place hot selection)
        def shift(t):
            if t is None:
                return None
            buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
            v = buf[1:].view(t.shape)
            v.copy_(t)
            return v
        ins = [shift(t) for t in ins]
    keep = [None if t is None else t.clone() for t in ins]
    kw = dict(K=K, scores_thresh=st, center_thresh=ct_th, aggr_weight=aggr, num_dets=nd)
    up = [_up(t) for t in ins]
    # contract 1 on the upcast (fp32) logits: torch's sigmoid of the five maps, then the fp32 decode
    want = dec(*[_sig(t) for t in up[:5]], *up[5:], **kw)
    got = dec_logits(*ins, **kw)
    assert torch.equal(got, want)
    if dtypes is not None and any(dt != torch.float32 for dt in dtypes):
        assert torch.equal(dec_logits(*up, **kw), want)          # contract 2, logits form
        heat = [_sig(t).to(t.dtype) if t is not None else None for t in ins[:5]]   # half heat maps
        assert torch.equal(dec(*heat, *ins[5:], **kw), dec(*[_up(t) for t in heat], *up[5:], **kw))   # contract 2
    for t, k in zip(ins, keep):
        assert t is None or torch.equal(t, k)
    return want


@pytest.mark.parametrize("shape", SHAPES, ids=SIDS)
@pytest.mark.parametrize("agnostic", [False, True], ids=["exct", "agnex"])
@pytest.mark.parametrize("aggr", [0.0, 0.1])
@pytest.mark.parametrize("dt", [torch.float32] + HALF, ids=["fp32"] + HIDS)
def test_gaussian_logits(shape, agnostic, aggr, dt):
    B, C, H, W = shape
    maps, regs = _logit_inputs(B, C, H, W, seed=11 + B * C, agnostic=agnostic)
    want = _check(maps, regs, agnostic, 40, aggr, dtypes=[dt] * 9)
    assert (want[..., 4] > -1).any()   # real detections, not only fillers
    _check(maps, None, agnostic, 40, aggr, dtypes=[dt] * 9, nd=100)


@pytest.mark.parametrize("K", [40, 100])
@pytest.mark.parametrize("agnostic", [False, True], ids=["exct", "agnex"])
@pytest.mark.parametrize("aggr", [0.0, 0.1])
def test_golden_inputs_as_logits(K, agnostic, aggr):
    maps, regs = _golden_logits()
    if agnostic:   # class-agnostic extreme maps: the max over classes
        maps = [m.amax(1, keepdim=True) for m in maps[:4]] + [maps[4]]
    want = _check(maps, regs, agnostic, K, aggr)
    assert (want[..., 4] > 0).sum() > 10
    for dt in HALF:
        _check(maps, regs, agnostic, K, aggr, dtypes=[dt] * 9)


@pytest.mark.parametrize("shape", [(2, 80, 128, 128), (2, 4, 96, 160)], ids=["128x128", "96x160"])
@pytest.mark.parametrize("agnostic", [False, True], ids=["exct", "agnex"])
@pytest.mark.parametrize("aggr", [0.0, 0.1])
def test_mixed_dtypes_and_offsets(shape, agnostic, aggr):
    B, C, H, W = shape
    maps, regs = _logit_inputs(B, C, H, W, seed=5, agnostic=agnostic)
    dts = [torch.bfloat16, torch.float16, torch.float32, torch.bfloat16, torch.float16, torch.float32, torch.bfloat16,
           torch.float16, torch.bfloat16]
    _check(maps, regs, agnostic, 40, aggr, dtypes=dts)
    _check(maps, regs, agnostic, 40, aggr, dtypes=dts[::-1])
    for dt in HALF + [torch.float32]:
        _check(maps, regs, agnostic, 40, aggr, dtypes=[dt] * 9, offset=True)
    _check(maps, regs, agnostic, 40, aggr, dtypes=dts, offset=True)


@pytest.mark.parametrize("dt", [torch.float32] + HALF, ids=["fp32"] + HIDS)
@pytest.mark.parametrize("aggr", [0.0, 0.1])
def test_saturated_centre_tie_agnostic(dt, aggr):
    """Centre logits of different classes that all saturate to sigmoid 1.0: the agnostic class is the first of them
    (torch.max on the sigmoided map), not the argmax of the logits."""
    maps, regs = _golden_logits(C=8, seed=321)
    maps = [m.amax(1, keepdim=True) for m in maps[:4]] + [maps[4]]
    ct = maps[4]
    hot = ct.amax(1, keepdim=True) > 0.0      # the objects' centres (sigmoid > 0.5)
    ramp = torch.arange(ct.shape[1], device="cuda", dtype=torch.float32).view(1, -1, 1, 1)
    sat = 20.0 + 2.0 * ramp                   # 20, 22, ..., 34 (exact in every dtype): each sigmoid is exactly 1.0
    assert torch.equal(torch.sigmoid(sat), torch.ones_like(sat))
    maps[4] = torch.where(hot, sat, ct)
    want = _check(maps, regs, True, 40, aggr, dtypes=[dt] * 9)
    rows = want[0][want[0, :, 4] > 0]
    assert rows.shape[0] > 0
    assert (rows[:, 13] == 0.0).any()         # the first saturated class, not the largest logit's


@pytest.mark.parametrize("dt", [torch.float32] + HALF, ids=["fp32"] + HIDS)
@pytest.mark.parametrize("agnostic", [False, True], ids=["exct", "agnex"])
def test_scores_on_thresholds(dt, agnostic):
    """scores_thresh and center_thresh set exactly to sigmoid values that peaks of the maps take."""
    maps, regs = _golden_logits(B=1, C=6, seed=323)
    if agnostic:
        maps = [m.amax(1, keepdim=True) for m in maps[:4]] + [maps[4]]
    maps = [m.to(dt) for m in maps]
    t_sig = torch.sigmoid(maps[0].float())
    c_sig = torch.sigmoid(maps[4].float())
    peaks = t_sig.flatten()[t_sig.flatten() > 0.3].sort().values       # the boxes' top points
    st = float(peaks[peaks.numel() // 2].item())                        # exactly the score of one of them
    cpk = c_sig.flatten()[c_sig.flatten() > 0.3].sort().values
    ct_th = float(cpk[cpk.numel() // 3].item())
    for s, c in ((st, 0.1), (0.1, ct_th), (st, ct_th)):
        _check(maps, regs, agnostic, 40, 0.0, dtypes=[dt] * 9, st=s, ct_th=c)


# ------------------------------------------------------------------ contract 3: edge aggregation of half maps
@pytest.mark.parametrize("shape", SHAPES + [(1, 3, 40, 520), (1, 2, 520, 24)],
                         ids=SIDS + ["long-rows", "long-cols"])
@pytest.mark.parametrize("dt", HALF, ids=HIDS)
@pytest.mark.parametrize("offset", [False, True], ids=["aligned", "offset"])
def test_aggregate_half(shape, dt, offset):
    from centernet_b200 import decode as D
    g = _gen(17)
    x = (torch.round(torch.rand(*shape, device="cuda", generator=g) * 8) / 8).to(dt)   # many equal neighbours
    if offset:
        buf = torch.empty(x.numel() + 1, dtype=dt, device="cuda")
        v = buf[1:].view(x.shape)
        v.copy_(x)
        x = v
    keep = x.clone()
    for fn in (D._left_aggregate, D._right_aggregate, D._top_aggregate, D._bottom_aggregate):
        got = fn(x)
        assert got.dtype == torch.float32
        assert torch.equal(got, fn(x.float()))
    for fn in (D._h_aggregate, D._v_aggregate):
        for wgt in (0.1, 0.37):
            assert torch.equal(fn(x, wgt), fn(x.float(), wgt))
    assert torch.equal(x, keep)


def test_non_default_stream():
    from centernet_b200 import decode as D
    maps, regs = _logit_inputs(2, 80, 128, 128, seed=3)
    maps = [m.to(torch.bfloat16) for m in maps]
    want = D.exct_decode_from_logits(*maps, *regs, aggr_weight=0.1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = D.exct_decode_from_logits(*maps, *regs, aggr_weight=0.1)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(got, want)

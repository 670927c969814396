"""CPU: workspace query and argument checks (before any CUDA call) of the fp16 / bf16 / logits entry points of
exct_decode / agnex_ct_decode and of the edge aggregation, and how their Python functions refuse CPU tensors.  No
kernel runs here."""
import pytest
import torch

ALIGNED, MISALIGNED = 1 << 20, (1 << 20) + 2      # fake device addresses: only their alignment is looked at
F32, BF16, F16 = 0, 1, 2
HOT = (1, 80, 80, 128, 128, 40)                   # b, c, cc, h, w, k: hot geometry
SHAPES = [HOT, (2, 80, 80, 128, 128, 100), (8, 80, 80, 128, 128, 40), (2, 3, 3, 96, 160, 40), (3, 2, 2, 64, 64, 40),
          (1, 2, 2, 72, 90, 40)]
ND = 1000


def _q(ptrs=(ALIGNED,) * 4, dts=(F32,) * 9, logits=0, shape=HOT, aggr=0.0, nd=ND, agnostic=0):
    from centernet_b200 import _C
    return _C.exct_decode_ex_workspace_bytes(*ptrs, *dts, logits, *shape, aggr, nd, agnostic)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("aggr", [0.0, 0.1])
@pytest.mark.parametrize("agnostic", [0, 1])
def test_query_matches_fp32_workspace(shape, aggr, agnostic):
    from centernet_b200 import _C
    b, c, cc, h, w, k = shape
    if agnostic:
        shape = (b, c, 1, h, w, k)
    old = _C.exct_workspace_bytes(*shape, ND)
    # all fp32 heat maps: exactly the fp32 call's workspace
    assert _q(shape=shape, aggr=aggr, agnostic=agnostic) == old
    assert _q(ptrs=(MISALIGNED,) * 4, shape=shape, aggr=aggr, agnostic=agnostic) == old
    # half maps or logits, hot or widened, aligned or not: the fp32 copy of a widened map (and the fp32 scores of the
    # centre map) live in an aggregated-map region, so no byte is added
    for dt in (F32, BF16, F16):
        for logits in (0, 1):
            for ptrs in ((ALIGNED,) * 4, (MISALIGNED,) * 4, (ALIGNED, MISALIGNED, ALIGNED, MISALIGNED)):
                assert _q(ptrs=ptrs, dts=(dt,) * 9, logits=logits, shape=shape, aggr=aggr, agnostic=agnostic) == old
    mixed = (BF16, F16, F32, BF16, F16, F32, BF16, F16, F32)
    assert _q(dts=mixed, logits=1, shape=shape, aggr=aggr, agnostic=agnostic) == old


def test_query_misaligned_fp32_map_read_in_place():
    # a misaligned fp32 map next to a half one is read in place by the non-hot selection, whose scratch may be larger
    from centernet_b200 import _C
    old = _C.exct_workspace_bytes(*HOT, ND)
    got = _q(ptrs=(MISALIGNED, ALIGNED, ALIGNED, ALIGNED), dts=(F32, BF16, F32, F32, F32, F32, F32, F32, F32))
    assert got >= old
    # with aggregation every selection reads an aligned fp32 aggregated map
    assert _q(ptrs=(MISALIGNED, ALIGNED, ALIGNED, ALIGNED), dts=(F32, BF16, F32, F32, F32, F32, F32, F32, F32),
              aggr=0.1) == old


def test_query_returns_zero_for_rejected_arguments():
    for dt in (F32, BF16):
        for logits in (0, 1):
            dts = (dt,) * 9
            for shape in ((0, 80, 80, 128, 128, 40), (1, 0, 80, 128, 128, 40), (1, 80, 0, 128, 128, 40),
                          (1, 80, 80, -1, 128, 40), (1, 80, 80, 128, 0, 40), (1, 80, 80, 128, 128, 0),
                          (1, 80, 3, 128, 128, 40), (1, 80, 80, 128, 128, 256), (1, 2, 2, 4, 4, 17)):
                assert _q(dts=dts, logits=logits, shape=shape) == 0, shape
            assert _q(dts=dts, logits=logits, nd=0) == 0
            assert _q(dts=dts, logits=logits, nd=2049) == 0
            assert _q(dts=dts, logits=logits, shape=(1, 1, 1, 128, 128, 4), nd=257) == 0   # > k^4
            for i in range(4):
                ptrs = [ALIGNED] * 4
                ptrs[i] = 0
                assert _q(ptrs=ptrs, dts=dts, logits=logits) == 0
    for bad in (-1, 3, 7):
        for i in range(9):
            dts = [F32] * 9
            dts[i] = bad
            assert _q(dts=dts) == 0
            assert _q(dts=dts, logits=1) == 0


def _call(maps=(ALIGNED,) * 4, map_dts=(BF16,) * 4, ct=ALIGNED, ct_dt=BF16, regs=(ALIGNED,) * 4, reg_dts=(BF16,) * 4,
          logits=1, shape=HOT, nd=ND, agnostic=0, aggr=0.0, dets=ALIGNED, ws=ALIGNED, nbytes=None):
    from centernet_b200 import _C
    if nbytes is None:
        nbytes = _C.exct_workspace_bytes(*HOT, ND)
    ins = list(zip(maps, map_dts)) + [(ct, ct_dt)] + list(zip(regs, reg_dts))
    _C.exct_decode_ex(*[a for p_dt in ins for a in p_dt], logits, *shape, 0.1, 0.1, aggr, nd, agnostic, dets, ws,
                      nbytes, 0)


def test_exct_ex_rejects_bad_arguments():
    for bad in (-1, 3):
        for i in range(4):
            dts = [BF16] * 4
            dts[i] = bad
            with pytest.raises(RuntimeError, match="unknown dtype code"):
                _call(map_dts=dts)
            with pytest.raises(RuntimeError, match="unknown dtype code"):
                _call(reg_dts=dts)
        with pytest.raises(RuntimeError, match="unknown dtype code"):
            _call(ct_dt=bad)
    with pytest.raises(RuntimeError, match="unknown dtype code"):   # a null regression map's code is checked too
        _call(regs=(0, 0, 0, 0), reg_dts=(F32, F32, 9, F32))
    for i in range(4):
        maps = [ALIGNED] * 4
        maps[i] = 0
        with pytest.raises(RuntimeError, match="null pointer"):
            _call(maps=maps)
    for kw in ({"ct": 0}, {"dets": 0}, {"ws": 0}):
        with pytest.raises(RuntimeError, match="null pointer"):
            _call(**kw)
    with pytest.raises(RuntimeError, match="non-positive"):
        _call(shape=(0, 80, 80, 128, 128, 40))
    with pytest.raises(RuntimeError, match="non-positive"):
        _call(nd=0)
    with pytest.raises(RuntimeError, match="centre map has 3 classes"):
        _call(shape=(1, 80, 3, 128, 128, 40))
    with pytest.raises(NotImplementedError, match="k=256"):
        _call(shape=(1, 80, 80, 128, 128, 256))
    with pytest.raises(RuntimeError, match="exceeds k"):
        _call(shape=(1, 1, 1, 128, 128, 4), nd=257)
    with pytest.raises(NotImplementedError, match="num_dets=2049"):
        _call(nd=2049)
    with pytest.raises(RuntimeError, match="exceeds h"):       # the selection plan: k > h*w
        _call(shape=(1, 2, 2, 4, 4, 17), nd=10)
    from centernet_b200 import _C
    need = _C.exct_workspace_bytes(*HOT, ND)
    with pytest.raises(RuntimeError, match="workspace"):
        _call(nbytes=need - 1)
    for agnostic, aggr in ((0, 0.1), (1, 0.0)):
        with pytest.raises(RuntimeError, match="workspace"):
            _call(nbytes=need - 1, agnostic=agnostic, aggr=aggr, shape=HOT[:2] + (1,) + HOT[3:] if agnostic else HOT)
    # fp32 maps take the fp32 call's checks, under the _ex name
    with pytest.raises(RuntimeError, match="cnb_exct_decode_ex: workspace"):
        _call(map_dts=(F32,) * 4, ct_dt=F32, reg_dts=(F32,) * 4, logits=0, nbytes=need - 1)
    with pytest.raises(RuntimeError, match="cnb_exct_decode_ex: null pointer"):
        _call(map_dts=(F32,) * 4, ct_dt=F32, reg_dts=(F32,) * 4, logits=0, ct=0)


def test_edge_aggregate_ex_rejects_bad_arguments():
    from centernet_b200 import _C
    ok = dict(heat=ALIGNED, dt=BF16, sig=0, out=ALIGNED + 4096, n=1, c=2, h=8, w=8, wt=0.1, horizontal=1)

    def run(**kw):
        a = dict(ok, **kw)
        _C.edge_aggregate_ex(a["heat"], a["dt"], a["sig"], a["out"], a["n"], a["c"], a["h"], a["w"], a["wt"],
                             a["horizontal"], 0)
    for bad in (-1, 3):
        with pytest.raises(RuntimeError, match="unknown dtype code"):
            run(dt=bad)
    for kw in ({"heat": 0}, {"out": 0}):
        with pytest.raises(RuntimeError, match="null pointer"):
            run(**kw)
    with pytest.raises(RuntimeError, match="in-place"):
        run(out=ALIGNED)
    with pytest.raises(RuntimeError, match="non-positive"):
        run(h=0)
    for bad in (-1, 6):
        with pytest.raises(RuntimeError, match="bad direction code"):
            run(horizontal=bad)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16])
def test_python_functions_refuse_cpu_tensors(dt):
    from centernet_b200 import decode as D
    m = lambda: torch.zeros(1, 2, 8, 8, dtype=dt)  # noqa: E731
    r = lambda: torch.zeros(1, 2, 8, 8, dtype=dt)  # noqa: E731
    for fn in (D.exct_decode, D.agnex_ct_decode, D.exct_decode_from_logits, D.agnex_ct_decode_from_logits):
        with pytest.raises(NotImplementedError, match="only implemented for CUDA"):
            fn(m(), m(), m(), m(), m(), r(), r(), r(), r(), K=4, num_dets=10)
        with pytest.raises(NotImplementedError, match=fn.__name__):
            fn(m(), m(), m(), m(), m(), K=4, num_dets=10)
    for fn in (D._h_aggregate, D._v_aggregate, D._left_aggregate, D._right_aggregate, D._top_aggregate,
               D._bottom_aggregate):
        with pytest.raises(NotImplementedError, match="only implemented for CUDA"):
            fn(m())


def test_shape_queries_survive_rejected_num_dets_and_batch():
    """The fp32 workspace query and the group query take num_dets and b before any argument check: a zero must not
    reach a division (the call itself then rejects it)."""
    from centernet_b200 import _C
    b, c, cc, h, w, k = HOT
    for nd in (0, -3):
        assert isinstance(_C.exct_workspace_bytes(b, c, cc, h, w, k, nd), int)
        assert _C.exct_groups(1, 40, nd) == 0
    assert isinstance(_C.exct_workspace_bytes(0, c, cc, h, w, k, ND), int)
    assert _C.exct_groups(0, 40, ND) == 0
    assert _C.exct_groups(1, 0, ND) == 0

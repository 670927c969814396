"""CPU: workspace queries and argument checks (before any CUDA call) of the fp16 / bf16 / logits entry points of
multi_pose_decode and ddd_decode, and how their Python functions refuse CPU tensors.  No kernel runs here."""
import pytest
import torch

ALIGNED, MISALIGNED = 1 << 20, (1 << 20) + 2      # fake device addresses: only their alignment is looked at
F32, BF16, F16 = 0, 1, 2
POSE = (2, 1, 17, 128, 128, 100)                  # b, c, j, h, w, k: hot geometry
DDD = (2, 3, 96, 320, 100)                        # b, c, h, w, k: KITTI-sized maps are never hot


def _align(x, a=256):
    return (x + a - 1) // a * a


def _raw(n):  # raw top-K of n rows: int64 indices + four fp32 / int32 columns
    return _align(n * 8) + 4 * _align(n * 4)


@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("logits", [0, 1])
def test_pose_query_hot(dt, logits):
    from centernet_b200 import _C
    q = _C.multi_pose_decode_ex_workspace_bytes
    b, c, j, h, w, k = POSE
    old = _C.multi_pose_workspace_bytes(*POSE)
    # both maps read in place: exactly the fp32 call's workspace, no map copy
    assert q(ALIGNED, dt, ALIGNED, dt, logits, *POSE) == old
    assert q(ALIGNED, F32, ALIGNED, F32, logits, *POSE) == old
    assert q(ALIGNED, F32, ALIGNED, dt, logits, *POSE) == old
    # no hm_hp: one selection, the joint rows are still carved
    assert q(ALIGNED, dt, 0, F32, logits, *POSE) == _C.topk_workspace_bytes(b, c, h, w, k) + _raw(b * j * k)
    # a misaligned map is widened into one fp32 copy (shared by both selections: the larger one)
    assert q(MISALIGNED, dt, ALIGNED, dt, logits, *POSE) == old + _align(b * c * h * w * 4)
    assert q(ALIGNED, dt, MISALIGNED, dt, logits, *POSE) == old + _align(b * j * h * w * 4)
    assert q(MISALIGNED, dt, MISALIGNED, dt, logits, *POSE) == old + _align(b * j * h * w * 4)
    # K > 256 leaves the hot kernel: widen
    big = (b, c, j, h, w, 300)
    assert q(ALIGNED, dt, ALIGNED, dt, logits, *big) == (_C.multi_pose_workspace_bytes(*big)
                                                        + _align(b * j * h * w * 4))


@pytest.mark.parametrize("shape", [(2, 1, 17, 96, 160, 100), (3, 1, 5, 64, 64, 20), (1, 1, 17, 30, 30, 40)])
def test_pose_query_not_hot(shape):
    from centernet_b200 import _C
    q = _C.multi_pose_decode_ex_workspace_bytes
    b, c, j, h, w, k = shape
    old = _C.multi_pose_workspace_bytes(*shape)
    copy = _align(b * max(c, j) * h * w * 4)
    assert q(ALIGNED, F32, ALIGNED, F32, 0, *shape) == old          # fp32 heat maps: read in place
    assert q(ALIGNED, F32, ALIGNED, F32, 1, *shape) == old + copy   # fp32 logits: the sigmoid pass
    for dt in (BF16, F16):
        for logits in (0, 1):
            assert q(ALIGNED, dt, ALIGNED, dt, logits, *shape) == old + copy
            assert q(ALIGNED, dt, ALIGNED, F32, 0, *shape) == old + _align(b * c * h * w * 4)


@pytest.mark.parametrize("shape", [DDD, (2, 3, 128, 128, 100), (1, 3, 128, 128, 1000), (4, 1, 64, 64, 40)])
def test_ddd_query(shape):
    from centernet_b200 import _C
    q = _C.ddd_decode_ex_workspace_bytes
    b, c, h, w, k = shape
    f32 = _C.topk_workspace_bytes(*shape)
    copy = _align(b * c * h * w * 4)
    hot = h == 128 and w == 128 and k <= 256
    assert q(ALIGNED, F32, 0, *shape) == f32
    assert q(ALIGNED, F32, 1, *shape) == (f32 if hot else f32 + copy)
    for dt in (BF16, F16):
        for logits in (0, 1):
            assert q(ALIGNED, dt, logits, *shape) == (f32 if hot else f32 + copy)
            assert q(MISALIGNED, dt, logits, *shape) == f32 + copy


def test_queries_return_zero_for_rejected_arguments():
    from centernet_b200 import _C
    qp, qd = _C.multi_pose_decode_ex_workspace_bytes, _C.ddd_decode_ex_workspace_bytes
    for dt in (F32, BF16, F16):
        for logits in (0, 1):
            for b, c, j, h, w, k in ((0, 1, 17, 128, 128, 100), (2, 0, 17, 128, 128, 100), (2, 1, 0, 128, 128, 100),
                                     (2, 1, 17, -1, 128, 100), (2, 1, 17, 128, 128, 0), (2, 1, 17, 4, 4, 17),
                                     (2, 1, 17, 128, 128, 1025)):
                assert qp(ALIGNED, dt, ALIGNED, dt, logits, b, c, j, h, w, k) == 0, (b, c, j, h, w, k)
            for b, c, h, w, k in ((0, 3, 96, 320, 100), (2, 0, 96, 320, 100), (2, 3, 96, 0, 100),
                                  (2, 3, 96, 320, -5), (2, 3, 4, 4, 17), (2, 3, 96, 320, 1025)):
                assert qd(ALIGNED, dt, logits, b, c, h, w, k) == 0, (b, c, h, w, k)
    for bad in (-1, 3, 7):
        for logits in (0, 1):
            assert qp(ALIGNED, bad, ALIGNED, F32, logits, *POSE) == 0
            assert qp(ALIGNED, F32, ALIGNED, bad, logits, *POSE) == 0
            assert qp(ALIGNED, F32, 0, bad, logits, *POSE) == 0
            assert qd(ALIGNED, bad, logits, *DDD) == 0


def _pose_call(heat=ALIGNED, heat_dt=BF16, logits=0, wh=ALIGNED, wh_dt=BF16, kps=ALIGNED, kps_dt=BF16, reg=ALIGNED,
               reg_dt=BF16, hm_hp=ALIGNED, hm_hp_dt=BF16, off=ALIGNED, off_dt=BF16, shape=POSE, dets=ALIGNED,
               ws=ALIGNED, nbytes=None):
    from centernet_b200 import _C
    if nbytes is None:
        nbytes = _C.multi_pose_decode_ex_workspace_bytes(ALIGNED, BF16, ALIGNED, BF16, logits, *POSE)
    _C.multi_pose_decode_ex(heat, heat_dt, logits, wh, wh_dt, kps, kps_dt, reg, reg_dt, hm_hp, hm_hp_dt, off, off_dt,
                            *shape, dets, ws, nbytes, 0)


def test_multi_pose_ex_rejects_bad_arguments():
    for name in ("heat_dt", "wh_dt", "kps_dt", "reg_dt", "hm_hp_dt", "off_dt"):
        for bad in (-1, 3):
            with pytest.raises(RuntimeError, match="unknown dtype code"):
                _pose_call(**{name: bad})
    with pytest.raises(RuntimeError, match="unknown dtype code"):   # a null head's code is checked too
        _pose_call(reg=0, reg_dt=5)
    for name in ("heat", "wh", "kps", "dets", "ws"):
        with pytest.raises(RuntimeError, match="null pointer"):
            _pose_call(**{name: 0})
    with pytest.raises(RuntimeError, match="j=0"):
        _pose_call(shape=(2, 1, 0, 128, 128, 100))
    with pytest.raises(RuntimeError, match="hp_offset without hm_hp"):
        _pose_call(hm_hp=0)
    with pytest.raises(RuntimeError, match="non-positive"):
        _pose_call(shape=(0, 1, 17, 128, 128, 100))
    with pytest.raises(RuntimeError, match="exceeds"):
        _pose_call(logits=1, shape=(2, 1, 17, 4, 4, 17))
    with pytest.raises(NotImplementedError):
        _pose_call(shape=(2, 1, 17, 128, 128, 1025))
    from centernet_b200 import _C
    need = _C.multi_pose_decode_ex_workspace_bytes(ALIGNED, BF16, ALIGNED, BF16, 0, *POSE)
    with pytest.raises(RuntimeError, match="workspace"):
        _pose_call(nbytes=need - 1)
    with pytest.raises(RuntimeError, match="workspace"):
        _pose_call(heat=MISALIGNED, nbytes=need)     # a misaligned map needs its fp32 copy
    with pytest.raises(RuntimeError, match="workspace"):
        _pose_call(hm_hp=MISALIGNED, nbytes=need)


def _ddd_call(heat=ALIGNED, heat_dt=F16, logits=1, rot=ALIGNED, rot_dt=F16, dep=ALIGNED, dep_dt=F16, dim=ALIGNED,
              dim_dt=F16, wh=ALIGNED, wh_dt=F16, reg=ALIGNED, reg_dt=F16, shape=DDD, dets=ALIGNED, ws=ALIGNED,
              nbytes=None):
    from centernet_b200 import _C
    if nbytes is None:
        nbytes = _C.ddd_decode_ex_workspace_bytes(ALIGNED, F16, logits, *DDD)
    _C.ddd_decode_ex(heat, heat_dt, logits, rot, rot_dt, dep, dep_dt, dim, dim_dt, wh, wh_dt, reg, reg_dt, *shape,
                     dets, ws, nbytes, 0)


def test_ddd_ex_rejects_bad_arguments():
    for name in ("heat_dt", "rot_dt", "dep_dt", "dim_dt", "wh_dt", "reg_dt"):
        for bad in (-1, 3):
            with pytest.raises(RuntimeError, match="unknown dtype code"):
                _ddd_call(**{name: bad})
    with pytest.raises(RuntimeError, match="unknown dtype code"):
        _ddd_call(wh=0, wh_dt=9)
    for name in ("heat", "rot", "dep", "dim", "dets", "ws"):
        with pytest.raises(RuntimeError, match="null pointer"):
            _ddd_call(**{name: 0})
    with pytest.raises(RuntimeError, match="non-positive"):
        _ddd_call(shape=(2, 3, 96, 320, 0))
    with pytest.raises(RuntimeError, match="exceeds"):
        _ddd_call(shape=(2, 3, 4, 4, 17))
    with pytest.raises(NotImplementedError):
        _ddd_call(shape=(2, 3, 96, 320, 1025))
    from centernet_b200 import _C
    need = _C.ddd_decode_ex_workspace_bytes(ALIGNED, F16, 1, *DDD)
    with pytest.raises(RuntimeError, match="workspace"):
        _ddd_call(nbytes=need - 1)
    hot = (2, 3, 128, 128, 100)
    need = _C.ddd_decode_ex_workspace_bytes(ALIGNED, F16, 1, *hot)
    with pytest.raises(RuntimeError, match="workspace"):
        _ddd_call(heat=MISALIGNED, shape=hot, nbytes=need)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16])
def test_python_functions_refuse_cpu_tensors(dt):
    from centernet_b200 import decode as D
    B, J, H, W = 1, 2, 8, 8
    t = lambda c: torch.zeros(B, c, H, W, dtype=dt)  # noqa: E731
    for fn in (D.multi_pose_decode, D.multi_pose_decode_from_logits):
        with pytest.raises(NotImplementedError, match="only implemented for CUDA"):
            fn(t(1), t(2), t(2 * J), reg=t(2), hm_hp=t(J), hp_offset=t(2), K=4)
    for fn in (D.ddd_decode, D.ddd_decode_from_logits):
        with pytest.raises(NotImplementedError, match="only implemented for CUDA"):
            fn(t(3), t(8), t(1), t(3), wh=t(2), reg=t(2), K=4)
    with pytest.raises(NotImplementedError, match="multi_pose_decode_from_logits"):
        D.multi_pose_decode_from_logits(t(1), t(2), t(2 * J), K=4)
    with pytest.raises(NotImplementedError, match="ddd_decode_from_logits"):
        D.ddd_decode_from_logits(t(3), t(8), t(1), t(3), K=4)

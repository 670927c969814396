"""CPU: the bf16 DCNv2 backward's workspace query and argument checks (before any CUDA call), and the Python switches
of backward_dtype.  No kernel runs here."""
import pytest
import torch

BF = torch.bfloat16


def _align(n, a=256):
    return (n + a - 1) // a * a


def _plan_bytes(B, Ci, H, W, Co, det, splits=None):
    """The regions of plan_backward_bf16 for a 3x3, stride 1, pad 1, one-group shape (Cout <= 256)."""
    Ho, Wo = H, W
    nb = (Ci + 31) // 32
    tw = 16 if Wo >= 12 else 8
    th = 128 // tw
    tiles = ((Wo + tw - 1) // tw) * ((Ho + th - 1) // th)
    KS = (Co + 31) // 32
    Q = nb * 9
    RG = (Q + 3) // 4
    Qp = RG * 4
    xt = _align(B * H * W * nb * 32 * 4)
    gyt_img = tiles * KS * 128 * 32 * 2                       # one bf16 tile per (tile, 32-wide slice of Cout)
    dcol_img = _align(Ho * Wo * Qp * 32 * 4)                  # the column gradient stays fp32
    bc = min(B, max(1, (1536 << 20) // (dcol_img + gyt_img)))
    gyt = 2 * xt + _align(RG * KS * 128 * 32 * 2)             # [xt][dxt][bf16 weight tiles]
    data_end = gyt + _align(bc * gyt_img) + bc * dcol_img
    co_r = 64 if Co <= 64 else (Co + 127) // 128 * 128
    spi = (Ho * Wo + 31) // 32
    weight_end = gyt + _align(B * spi * co_r * 32 * 2) + _align(splits * RG * 128 * co_r * 4) + \
        _align(B * spi * co_r * 4)
    end = max(data_end, weight_end)
    if not det:
        return end, weight_end < data_end
    return end + _align((KS + 2 * B) * 4) + _align(bc * H * W * nb * 32 * 8), weight_end < data_end


def test_bf16_backward_workspace_from_plan():
    from centernet_b200 import _C
    q = _C.dcnv2_backward_bf16_workspace_bytes
    # dla_34 64@128x128 -> 64, B = 16: the data pass's regions decide the size (the weight pass's, which depend on
    # the SM count through the split count, are smaller for any split count up to 132)
    for det in (False, True):
        _C.dcnv2_set_deterministic(int(det))
        try:
            got = q(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1)
            fp32 = _C.dcnv2_backward_workspace_bytes(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1)
        finally:
            _C.dcnv2_set_deterministic(0)
        want, data_bound = _plan_bytes(16, 64, 128, 128, 64, det, splits=132 // 5)
        assert data_bound
        assert got == want
        assert 0 < got < fp32                                  # bf16 tiles: half of a TF32 hi/lo pair
    assert q(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1) == _plan_bytes(16, 64, 128, 128, 64, False, 26)[0]
    _C.dcnv2_set_deterministic(1)
    try:
        more = q(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1)
    finally:
        _C.dcnv2_set_deterministic(0)
    assert more > q(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1)   # the fixed-point dX of one batch chunk


def test_bf16_backward_query_returns_zero_for_rejected_shapes():
    from centernet_b200 import _C
    q = _C.dcnv2_backward_bf16_workspace_bytes
    assert q(2, 64, 64, 32, 32, 3, 3, 1, 1, 1, 1) > 0
    assert q(2, 64, 256, 32, 32, 3, 3, 1, 1, 1, 1) > 0          # Cout 256: the largest the weight pass covers
    assert q(2, 64, 272, 32, 32, 3, 3, 1, 1, 1, 1) == 0          # Cout > 256: the caller falls back
    assert q(2, 64, 64, 32, 32, 5, 5, 1, 2, 1, 1) == 0           # 25 taps
    assert q(2, 64, 64, 32, 32, 3, 3, 1, 1, 1, 3) == 0           # groups must divide cin
    assert q(2, 64, 64, 2, 2, 7, 7, 1, 0, 1, 1) == 0             # empty output grid
    assert q(0, 64, 64, 32, 32, 3, 3, 1, 1, 1, 1) == 0


def test_bf16_backward_rejects_bad_arguments():
    from centernet_b200 import _C
    F32, BF16 = _C.DTYPE_F32, _C.DTYPE_BF16
    shape = (2, 64, 16, 16, 64, 3, 3, 1, 1, 1, 1)   # b, cin, h, w, cout, kh, kw, stride, pad, dil, dg
    need =_C.dcnv2_backward_bf16_workspace_bytes(2, 64, 64, 16, 16, 3, 3, 1, 1, 1, 1)
    assert need > 0
    f = _C.dcnv2_backward_bf16

    def call(inp=16, in_dt=BF16, in_cl=0, off=16, msk=16, w=16, go=16, go_dt=BF16, gin=16, gin_cl=0, shp=shape,
             ws=256, wsb=need):
        # input, dtype, cl, offset, mask, weight, grad_output, dtype, grad_input, cl, grad_offset, grad_mask,
        # grad_weight, grad_bias, shape..., workspace, bytes, stream
        return f(inp, in_dt, in_cl, off, msk, w, go, go_dt, gin, gin_cl, 16, 16, 16, 16, *shp, ws, wsb, 0)

    for kw in ({"inp": 0}, {"off": 0}, {"msk": 0}, {"w": 0}, {"go": 0}, {"ws": 0}):
        with pytest.raises(RuntimeError, match="null pointer"):
            call(**kw)
    with pytest.raises(RuntimeError, match="dtype"):
        call(in_dt=2)                                            # fp16 is not an input of this call
    with pytest.raises(RuntimeError, match="dtype"):
        call(go_dt=-1)
    with pytest.raises(RuntimeError, match="deformable groups"):
        call(shp=(2, 64, 16, 16, 64, 3, 3, 1, 1, 1, 3))
    with pytest.raises(NotImplementedError, match="taps"):
        call(shp=(2, 64, 16, 16, 64, 5, 5, 1, 2, 1, 1))
    with pytest.raises(NotImplementedError, match="cout <= 256"):
        call(shp=(2, 64, 16, 16, 272, 3, 3, 1, 1, 1, 1))
    with pytest.raises(NotImplementedError, match="multiple of 32"):
        call(in_cl=1, shp=(2, 80, 16, 16, 64, 3, 3, 1, 1, 1, 2))   # 40 channels a group
    with pytest.raises(NotImplementedError, match="multiple of 32"):
        call(gin_cl=1, shp=(2, 80, 16, 16, 64, 3, 3, 1, 1, 1, 2))
    with pytest.raises(RuntimeError, match="workspace"):
        call(wsb=need - 1)
    _C.dcnv2_set_deterministic(1)
    try:
        with pytest.raises(RuntimeError, match="workspace"):
            call(go_dt=F32)                                      # the default-mode size is too small in this mode
    finally:
        _C.dcnv2_set_deterministic(0)
    with pytest.raises(RuntimeError, match="aligned"):
        call(inp=24, in_dt=F32)
    with pytest.raises(RuntimeError, match="aligned"):
        call(ws=264)
    with pytest.raises(RuntimeError, match="aligned"):
        call(in_cl=1, gin=24, gin_cl=1)


def test_backward_dtype_values():
    from centernet_b200.dcn_v2 import DCN, DCNv2
    from centernet_b200.dcn_v2_func import DCNv2Function
    assert DCNv2Function(1, 1).backward_dtype is None
    assert DCNv2Function(1, 1, compute_dtype=BF).backward_dtype is None
    assert DCNv2Function(1, 1, compute_dtype=BF, backward_dtype=BF).backward_dtype is BF
    assert DCN(4, 4, 3, 1, 1, compute_dtype=BF, backward_dtype=BF).backward_dtype is BF
    assert DCNv2(4, 4, 3, 1, 1).backward_dtype is None
    for cd, bd in ((None, BF), (BF, torch.float32), (BF, torch.float16), (BF, "bf16"), (None, torch.float32)):
        with pytest.raises(ValueError):
            DCNv2Function(1, 1, compute_dtype=cd, backward_dtype=bd)
        with pytest.raises(ValueError):
            DCN(4, 4, 3, 1, 1, compute_dtype=cd, backward_dtype=bd)
        with pytest.raises(ValueError):
            DCNv2(4, 4, 3, 1, 1, compute_dtype=cd, backward_dtype=bd)
    # CPU tensors: no fallback, as on the default path
    with pytest.raises(NotImplementedError):
        DCNv2Function(1, 1, compute_dtype=BF, backward_dtype=BF)(
            torch.zeros(1, 4, 4, 4), torch.zeros(1, 18, 4, 4), torch.zeros(1, 9, 4, 4), torch.zeros(4, 4, 3, 3),
            torch.zeros(4))


def test_set_compute_dtype_sets_backward_dtype():
    from torch import nn
    from centernet_b200.dcn_v2 import DCN, DCNv2, set_compute_dtype
    model = nn.Sequential(DCN(8, 8, 3, 1, 1), nn.Conv2d(8, 8, 3), nn.Sequential(DCNv2(8, 16, 3, 1, 1), nn.ReLU()),
                          DCN(16, 8, (3, 3), stride=2, padding=1))
    dcns = [m for m in model.modules() if isinstance(m, DCNv2)]
    assert all(m.backward_dtype is None for m in dcns)
    assert set_compute_dtype(model, BF, backward_dtype=BF) == 3
    assert all(m.compute_dtype is BF and m.backward_dtype is BF for m in dcns)
    assert set_compute_dtype(model, BF) == 3                     # backward_dtype back to the fp32 backward
    assert all(m.compute_dtype is BF and m.backward_dtype is None for m in dcns)
    assert set_compute_dtype(model, BF, BF) == 3
    assert set_compute_dtype(model, None) == 3
    assert all(m.compute_dtype is None and m.backward_dtype is None for m in dcns)
    for cd, bd in ((None, BF), (BF, torch.float16)):
        with pytest.raises(ValueError):
            set_compute_dtype(model, cd, backward_dtype=bd)
    assert all(m.compute_dtype is None and m.backward_dtype is None for m in dcns)   # a rejected call sets nothing
    assert set_compute_dtype(nn.Conv2d(2, 2, 1), BF, backward_dtype=BF) == 0

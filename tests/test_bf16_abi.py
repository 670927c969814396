"""CPU: the bf16 DCNv2 forward's workspace / tile queries and argument checks (before any CUDA call), and the Python
switches of compute_dtype.  No kernel runs here."""
import pytest
import torch


def test_bf16_workspace_and_tile_bytes():
    from centernet_b200 import _C
    q = _C.dcnv2_bf16_workspace_bytes
    # dla_34 64@128x128 -> 64, B=16: bf16 channels-last copy [16][128*128][2 blocks][32] and no split-K partials
    # (2048 items fill any GPU)
    assert q(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1) == 16 * 128 * 128 * 64 * 2
    # 512@16x16 -> 256, B=1: 4 items, split 8 ways: the bf16 copy and 8 fp32 partial outputs
    assert q(1, 512, 256, 16, 16, 3, 3, 1, 1, 1, 1) == 16 * 16 * 512 * 2 + 8 * 256 * 16 * 16 * 4
    # one bf16 tile [co_t][32] per (Cout tile, 32-channel block, tap): half of a TF32 hi or lo tile
    t = _C.dcnv2_wtiles_bf16_bytes
    assert t(64, 64, 3, 3, 1) == 1 * 2 * 9 * 64 * 32 * 2
    assert t(256, 256, 3, 3, 1) == 2 * 8 * 9 * 128 * 32 * 2
    assert 4 * t(64, 64, 3, 3, 1) == _C.dcnv2_wtiles_bytes(64, 64, 3, 3, 1)
    assert t(40, 24, 3, 3, 2) == 1 * 2 * 9 * 64 * 32 * 2          # ragged: 20 channels a group -> one padded block each


def test_bf16_queries_return_zero_for_rejected_shapes():
    from centernet_b200 import _C
    q = _C.dcnv2_bf16_workspace_bytes
    assert q(2, 64, 64, 32, 32, 5, 5, 1, 2, 1, 1) == 0           # 25 taps
    assert q(2, 64, 64, 32, 32, 3, 3, 1, 1, 1, 3) == 0           # groups must divide cin
    assert q(2, 64, 64, 2, 2, 7, 7, 1, 0, 1, 1) == 0             # empty output grid
    assert q(0, 64, 64, 32, 32, 3, 3, 1, 1, 1, 1) == 0
    assert _C.dcnv2_wtiles_bf16_bytes(64, 64, 5, 5, 1) == 0
    assert _C.dcnv2_wtiles_bf16_bytes(64, 64, 3, 3, 3) == 0


def test_bf16_forward_rejects_bad_arguments():
    from centernet_b200 import _C
    F32, BF16 = _C.DTYPE_F32, _C.DTYPE_BF16
    assert (F32, BF16) == (0, 1)
    shape = (2, 64, 16, 16, 64, 3, 3, 1, 1, 1, 1)   # b, cin, h, w, cout, kh, kw, stride, pad, dil, dg
    need = _C.dcnv2_bf16_workspace_bytes(2, 64, 64, 16, 16, 3, 3, 1, 1, 1, 1)
    assert need > 0
    f = _C.dcnv2_forward_bf16
    # input, dtype, cl, offset, mask, wtiles, bias, output, dtype, shape..., workspace, bytes, stream
    with pytest.raises(RuntimeError, match="null pointer"):
        f(0, BF16, 0, 16, 16, 16, 0, 16, BF16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="null pointer"):
        f(16, BF16, 0, 16, 0, 16, 0, 16, BF16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="null pointer"):
        f(16, BF16, 0, 16, 16, 16, 0, 16, BF16, *shape, 0, need, 0)
    with pytest.raises(RuntimeError, match="dtype"):
        f(16, 2, 0, 16, 16, 16, 0, 16, BF16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="dtype"):
        f(16, F32, 0, 16, 16, 16, 0, 16, -1, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="workspace"):
        f(16, F32, 0, 16, 16, 16, 0, 16, F32, *shape, 256, need - 1, 0)
    with pytest.raises(RuntimeError, match="aligned"):
        f(24, BF16, 0, 16, 16, 16, 0, 16, BF16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="deformable groups"):
        f(16, BF16, 0, 16, 16, 16, 0, 16, BF16, 2, 64, 16, 16, 64, 3, 3, 1, 1, 1, 3, 256, need, 0)
    with pytest.raises(NotImplementedError, match="taps"):
        f(16, BF16, 0, 16, 16, 16, 0, 16, BF16, 2, 64, 16, 16, 64, 5, 5, 1, 2, 1, 1, 256, need, 0)
    g = _C.dcnv2_forward_fused_bf16
    # input, dtype, cl, offset_mask, wtiles, bias, bn_scale, bn_shift, relu, output, dtype, shape..., ws, bytes, stream
    with pytest.raises(RuntimeError, match="null pointer"):
        g(16, BF16, 0, 0, 16, 0, 0, 0, 1, 16, BF16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="go together"):
        g(16, BF16, 0, 16, 16, 0, 16, 0, 1, 16, BF16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="dtype"):
        g(16, 7, 0, 16, 16, 0, 0, 0, 1, 16, BF16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="workspace"):
        g(16, BF16, 0, 16, 16, 0, 0, 0, 1, 16, BF16, *shape, 256, 16, 0)
    wtb = _C.dcnv2_wtiles_bf16_bytes(64, 64, 3, 3, 1)
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.dcnv2_prepare_weights_bf16(0, 64, 64, 3, 3, 1, 256, wtb, 0)
    with pytest.raises(RuntimeError, match="buffer"):
        _C.dcnv2_prepare_weights_bf16(16, 64, 64, 3, 3, 1, 256, wtb - 1, 0)
    with pytest.raises(NotImplementedError, match="taps"):
        _C.dcnv2_prepare_weights_bf16(16, 64, 64, 5, 5, 1, 256, wtb, 0)


def test_compute_dtype_values():
    from centernet_b200.dcn_v2 import DCN, DCNv2
    from centernet_b200.dcn_v2_func import DCNv2Function, dcn_fused_inference
    assert DCNv2Function(1, 1).compute_dtype is None
    assert DCNv2Function(1, 1, compute_dtype=torch.bfloat16).compute_dtype is torch.bfloat16
    for bad in (torch.float16, torch.float32, "bf16"):
        with pytest.raises(ValueError):
            DCNv2Function(1, 1, compute_dtype=bad)
        with pytest.raises(ValueError):
            DCN(4, 4, 3, 1, 1, compute_dtype=bad)
        with pytest.raises(ValueError):
            DCNv2(4, 4, 3, 1, 1, compute_dtype=bad)
        with pytest.raises(ValueError):
            dcn_fused_inference(torch.zeros(1, 4, 4, 4), torch.zeros(1, 27, 4, 4), torch.zeros(4, 4, 3, 3), None,
                                1, 1, 1, 1, compute_dtype=bad)
    # CPU tensors: no fallback, as on the default path
    x = torch.zeros(1, 4, 4, 4)
    with pytest.raises(NotImplementedError):
        DCNv2Function(1, 1, compute_dtype=torch.bfloat16)(x, torch.zeros(1, 18, 4, 4), torch.zeros(1, 9, 4, 4),
                                                          torch.zeros(4, 4, 3, 3), torch.zeros(4))
    with pytest.raises(NotImplementedError):
        dcn_fused_inference(x, torch.zeros(1, 27, 4, 4), torch.zeros(4, 4, 3, 3), None, 1, 1, 1, 1,
                            compute_dtype=torch.bfloat16)


def test_set_compute_dtype_counts_modules():
    from torch import nn
    from centernet_b200.dcn_v2 import DCN, DCNv2, set_compute_dtype
    model = nn.Sequential(DCN(8, 8, 3, 1, 1), nn.Conv2d(8, 8, 3), nn.Sequential(DCNv2(8, 16, 3, 1, 1), nn.ReLU()),
                          DCN(16, 8, (3, 3), stride=2, padding=1))
    assert all(m.compute_dtype is None for m in model.modules() if isinstance(m, DCNv2))
    assert set_compute_dtype(model, torch.bfloat16) == 3
    assert all(m.compute_dtype is torch.bfloat16 for m in model.modules() if isinstance(m, DCNv2))
    assert set_compute_dtype(model, None) == 3
    assert all(m.compute_dtype is None for m in model.modules() if isinstance(m, DCNv2))
    assert set_compute_dtype(nn.Conv2d(2, 2, 1), torch.bfloat16) == 0
    with pytest.raises(ValueError):
        set_compute_dtype(model, torch.float16)

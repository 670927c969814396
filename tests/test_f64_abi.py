"""CPU: the float64 DCNv2 / PSROI entry points validate their arguments before any CUDA call (CNB_EINVAL ->
RuntimeError), and their workspace queries are sane.  No kernel runs here."""
import pytest


def test_dcnv2_f64_workspace_query():
    from centernet_b200 import _C
    q = _C.dcnv2_f64_workspace_bytes
    base = q(2, 64, 64, 64, 64, 3, 3, 1, 1, 1, 1)
    assert base > 0 and base % 256 == 0
    # at least the two 64-bit limbs of the dX accumulator and the column gradient of both images
    assert base >= 2 * 2 * 64 * 64 * 64 * 8 + 2 * 64 * 9 * 64 * 64 * 8
    assert q(4, 64, 64, 64, 64, 3, 3, 1, 1, 1, 1) > base
    assert q(2, 64, 64, 32, 32, 5, 5, 1, 2, 1, 1) > 0           # 25 taps: covered
    assert q(2, 12, 5, 9, 11, 3, 3, 2, 1, 2, 2) > 0             # strided, dilated, grouped
    assert q(2, 64, 64, 32, 32, 3, 3, 1, 1, 1, 3) == 0          # groups must divide cin
    assert q(2, 64, 64, 2, 2, 7, 7, 1, 0, 1, 1) == 0            # empty output grid
    # the column gradient is held to ~1.5 GiB however large the batch
    assert q(64, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1) < q(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1) * 3


def test_dcnv2_f64_rejects_bad_arguments():
    from centernet_b200 import _C
    args = (2, 2, 4, 4, 2, 3, 3, 1, 1, 1, 1, 1, 1, 1)   # b, cin, h, w, cout, kh, kw, sh, sw, ph, pw, dh, dw, dg
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.dcnv2_forward_f64(0, 16, 16, 16, 16, 16, *args, 0)
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.dcnv2_forward_f64(16, 16, 16, 16, 16, 0, *args, 0)
    with pytest.raises(RuntimeError, match="deformable_groups"):
        _C.dcnv2_forward_f64(16, 16, 16, 16, 16, 16, 2, 3, 4, 4, 2, 3, 3, 1, 1, 1, 1, 1, 1, 2, 0)
    with pytest.raises(RuntimeError, match="bad shape"):
        _C.dcnv2_forward_f64(16, 16, 16, 16, 16, 16, 0, 2, 4, 4, 2, 3, 3, 1, 1, 1, 1, 1, 1, 1, 0)
    with pytest.raises(RuntimeError, match="stride"):
        _C.dcnv2_forward_f64(16, 16, 16, 16, 16, 16, 2, 2, 4, 4, 2, 3, 3, 0, 1, 1, 1, 1, 1, 1, 0)
    with pytest.raises(RuntimeError, match="empty output"):
        _C.dcnv2_forward_f64(16, 16, 16, 16, 16, 16, 2, 2, 2, 2, 2, 7, 7, 1, 1, 0, 0, 1, 1, 1, 0)
    need = _C.dcnv2_f64_workspace_bytes(2, 2, 2, 4, 4, 3, 3, 1, 1, 1, 1)
    ptrs = (16,) * 10
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.dcnv2_backward_f64(16, 16, 16, 16, 16, 0, 16, 16, 16, 16, *args, 256, need, 0)
    with pytest.raises(RuntimeError, match="workspace"):
        _C.dcnv2_backward_f64(*ptrs, *args, 256, need - 1, 0)
    with pytest.raises(RuntimeError, match="workspace"):
        _C.dcnv2_backward_f64(*ptrs, *args, 0, need, 0)
    with pytest.raises(RuntimeError, match="aligned"):
        _C.dcnv2_backward_f64(*ptrs, *args, 264, need, 0)
    assert "aligned" in _C.last_error()


def test_psroi_f64_rejects_bad_arguments():
    from centernet_b200 import _C
    assert _C.psroi_pooling_f64_workspace_bytes(2, 8, 9, 9) >= 2 * 2 * 8 * 9 * 9 * 8
    assert _C.psroi_pooling_f64_workspace_bytes(0, 8, 9, 9) == 0
    with pytest.raises(RuntimeError, match="channels"):
        _C.psroi_pooling_forward_f64(16, 16, 0, 16, 16, 1, 8, 9, 9, 2, 2, 1, 0.25, 4, 2, 3, 3, 2, 0.0, 0)
    with pytest.raises(RuntimeError, match="offsets"):
        _C.psroi_pooling_forward_f64(16, 16, 0, 16, 16, 1, 8, 9, 9, 2, 3, 0, 0.25, 2, 2, 3, 3, 2, 0.0, 0)
    with pytest.raises(RuntimeError, match="multiple"):
        _C.psroi_pooling_forward_f64(16, 16, 16, 16, 16, 1, 8, 9, 9, 2, 4, 0, 0.25, 3, 1, 3, 3, 2, 0.1, 0)
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.psroi_pooling_forward_f64(0, 16, 0, 16, 16, 1, 8, 9, 9, 2, 2, 1, 0.25, 2, 2, 3, 3, 2, 0.0, 0)
    need = _C.psroi_pooling_f64_workspace_bytes(1, 8, 9, 9)
    cfg = (1, 8, 9, 9, 2, 2, 1, 0.25, 2, 2, 3, 3, 2, 0.0)
    with pytest.raises(RuntimeError, match="workspace"):
        _C.psroi_pooling_backward_f64(16, 16, 16, 0, 16, 16, 0, *cfg, 256, need - 1, 0)
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.psroi_pooling_backward_f64(16, 16, 16, 0, 16, 0, 0, *cfg, 256, need, 0)


def test_f64_without_cuda_is_not_implemented():
    import torch
    from centernet_b200.dcn_v2_func import DCNv2Function, DCNv2PoolingFunction, dcn_fused_inference
    x = torch.zeros(1, 2, 4, 4, dtype=torch.float64)
    with pytest.raises(NotImplementedError):
        DCNv2Function(1, 1)(x, torch.zeros(1, 18, 4, 4, dtype=torch.float64), torch.zeros(1, 9, 4, 4, dtype=torch.float64),
                            torch.zeros(2, 2, 3, 3, dtype=torch.float64), torch.zeros(2, dtype=torch.float64))
    with pytest.raises(NotImplementedError):
        DCNv2PoolingFunction(0.25, 3, 2, True)(x, torch.zeros(1, 5), x.new())
    with pytest.raises(NotImplementedError):
        dcn_fused_inference(x, torch.zeros(1, 27, 4, 4, dtype=torch.float64), torch.zeros(2, 2, 3, 3, dtype=torch.float64),
                            None, 1, 1, 1, 1)

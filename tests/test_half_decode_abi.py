"""CPU: the fp16 / bf16 ctdet decode entry points' workspace queries and argument checks (before any CUDA call), and
the reference op sequence on half heads against its run on their fp32 upcast.  No kernel runs here."""
import numpy as np
import pytest
import torch

from helpers import assert_dets_equal

SHAPES = [(1, 80, 128, 128, 100), (64, 80, 128, 128, 100), (2, 80, 128, 128, 256), (3, 7, 128, 128, 1),
          (8, 80, 96, 320, 100), (2, 5, 30, 30, 40), (4, 80, 200, 152, 100), (2, 80, 128, 128, 1000),
          (150, 80, 128, 128, 100), (1, 1, 128, 128, 16)]
ALIGNED, MISALIGNED = 1 << 20, (1 << 20) + 2      # fake device addresses: only their alignment is looked at


def _align(x, a=256):
    return (x + a - 1) // a * a


def _hot(h, w, k):
    return h == 128 and w == 128 and k <= 256


def test_dtype_codes():
    from centernet_b200 import _C
    assert (_C.DTYPE_F32, _C.DTYPE_BF16, _C.DTYPE_F16) == (0, 1, 2)


@pytest.mark.parametrize("shape", SHAPES)
def test_f32_queries_equal_the_old_queries(shape):
    from centernet_b200 import _C
    b, c, h, w, k = shape
    q = _C.ctdet_decode_ex_workspace_bytes
    for p in (ALIGNED, MISALIGNED, 0):
        assert q(p, _C.DTYPE_F32, 0, b, c, h, w, k) == _C.topk_workspace_bytes(b, c, h, w, k)
        assert q(p, _C.DTYPE_F32, 1, b, c, h, w, k) == _C.ctdet_logits_workspace_bytes(p, b, c, h, w, k)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dt", [1, 2])
def test_half_queries(shape, dt):
    from centernet_b200 import _C
    b, c, h, w, k = shape
    q = _C.ctdet_decode_ex_workspace_bytes
    f32 = _C.topk_workspace_bytes(b, c, h, w, k)
    heat32 = _align(b * c * h * w * 4)
    if _hot(h, w, k):
        # read in place: no conversion buffer, no more scratch than fp32
        assert q(ALIGNED, dt, 0, b, c, h, w, k) == f32
        assert q(ALIGNED, dt, 1, b, c, h, w, k) == q(ALIGNED, _C.DTYPE_F32, 1, b, c, h, w, k)
        assert q(ALIGNED, dt, 1, b, c, h, w, k) <= f32
    else:
        assert q(ALIGNED, dt, 0, b, c, h, w, k) == f32 + heat32
        # logits: the fp32 form already materialises the sigmoid map; the 16-bit one reads the logits directly
        assert q(ALIGNED, dt, 1, b, c, h, w, k) == q(ALIGNED, _C.DTYPE_F32, 1, b, c, h, w, k)
    # misaligned base pointer: always the widening pass
    assert q(MISALIGNED, dt, 0, b, c, h, w, k) == f32 + heat32
    assert q(MISALIGNED, dt, 1, b, c, h, w, k) == q(MISALIGNED, _C.DTYPE_F32, 1, b, c, h, w, k)
    assert q(MISALIGNED, dt, 1, b, c, h, w, k) >= heat32


def test_queries_return_zero_for_rejected_shapes():
    from centernet_b200 import _C
    q = _C.ctdet_decode_ex_workspace_bytes
    for dt in (0, 1, 2):
        for logits in (0, 1):
            assert q(ALIGNED, dt, logits, 0, 80, 128, 128, 100) == 0
            assert q(ALIGNED, dt, logits, 2, 0, 128, 128, 100) == 0
            assert q(ALIGNED, dt, logits, 2, 80, -1, 128, 100) == 0
            assert q(ALIGNED, dt, logits, 2, 80, 128, 128, 0) == 0
            assert q(ALIGNED, dt, logits, 2, 80, 4, 4, 17) == 0        # k > h*w
            assert q(ALIGNED, dt, logits, 2, 80, 128, 128, 1025) == 0  # k beyond the selection envelope
    for bad in (-1, 3, 7):
        assert q(ALIGNED, bad, 0, 2, 80, 128, 128, 100) == 0
        assert q(ALIGNED, bad, 1, 2, 80, 128, 128, 100) == 0


def test_decode_ex_rejects_bad_arguments():
    from centernet_b200 import _C
    F32, BF16, F16 = _C.DTYPE_F32, _C.DTYPE_BF16, _C.DTYPE_F16
    f = _C.ctdet_decode_ex
    shape = (2, 80, 128, 128, 100)
    need = _C.ctdet_decode_ex_workspace_bytes(ALIGNED, BF16, 0, *shape)
    # heat, dt, logits, wh, dt, reg, dt, cat, b, c, h, w, k, dets, ws, bytes, stream
    with pytest.raises(RuntimeError, match="dtype"):
        f(ALIGNED, 3, 0, ALIGNED, F32, 0, F32, 0, *shape, ALIGNED, ALIGNED, need, 0)
    with pytest.raises(RuntimeError, match="dtype"):
        f(ALIGNED, BF16, 0, ALIGNED, -1, 0, F32, 0, *shape, ALIGNED, ALIGNED, need, 0)
    with pytest.raises(RuntimeError, match="dtype"):
        f(ALIGNED, F16, 1, ALIGNED, F16, ALIGNED, 9, 0, *shape, ALIGNED, ALIGNED, need, 0)
    for heat, wh, dets, ws in ((0, ALIGNED, ALIGNED, ALIGNED), (ALIGNED, 0, ALIGNED, ALIGNED),
                               (ALIGNED, ALIGNED, 0, ALIGNED), (ALIGNED, ALIGNED, ALIGNED, 0)):
        with pytest.raises(RuntimeError, match="null pointer"):
            f(heat, BF16, 0, wh, BF16, 0, F32, 0, *shape, dets, ws, need, 0)
    with pytest.raises(RuntimeError, match="non-positive"):
        f(ALIGNED, BF16, 0, ALIGNED, BF16, 0, F32, 0, 0, 80, 128, 128, 100, ALIGNED, ALIGNED, need, 0)
    with pytest.raises(RuntimeError, match="exceeds"):
        f(ALIGNED, F16, 1, ALIGNED, F16, 0, F32, 0, 2, 80, 4, 4, 17, ALIGNED, ALIGNED, need, 0)
    with pytest.raises(NotImplementedError):
        f(ALIGNED, F16, 0, ALIGNED, F16, 0, F32, 0, 2, 80, 128, 128, 1025, ALIGNED, ALIGNED, need, 0)
    with pytest.raises(RuntimeError, match="workspace"):
        f(ALIGNED, BF16, 0, ALIGNED, BF16, 0, F32, 0, *shape, ALIGNED, ALIGNED, need - 1, 0)
    with pytest.raises(RuntimeError, match="workspace"):
        f(MISALIGNED, BF16, 0, ALIGNED, BF16, 0, F32, 0, *shape, ALIGNED, ALIGNED, need, 0)   # needs the map


def test_flip_merge_ex_rejects_bad_arguments():
    from centernet_b200 import _C
    g = _C.flip_merge_ex
    # src, dt, dst, n, c, h, w, sigmoid, perm, sign, stream
    for bad in (-1, 3):
        with pytest.raises(RuntimeError, match="dtype"):
            g(ALIGNED, bad, ALIGNED, 1, 80, 128, 128, 1, 0, 0, 0)
    for dt in (0, 1, 2):
        with pytest.raises(RuntimeError, match="null pointer"):
            g(0, dt, ALIGNED, 1, 80, 128, 128, 1, 0, 0, 0)
        with pytest.raises(RuntimeError, match="null pointer"):
            g(ALIGNED, dt, 0, 1, 80, 128, 128, 0, 0, 0, 0)
        with pytest.raises(RuntimeError, match="non-positive"):
            g(ALIGNED, dt, ALIGNED, 0, 80, 128, 128, 0, 0, 0, 0)


def _bench_heads(B, seed=317, C=80, H=128, W=128):
    g = torch.Generator().manual_seed(seed)
    heat = torch.sigmoid(torch.randn(B, C, H, W, generator=g) - 2.19)
    wh = torch.rand(B, 2, H, W, generator=g) * 32
    reg = torch.rand(B, 2, H, W, generator=g)
    return heat, wh, reg


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_reference_ops_on_half_heads_equal_their_upcast(dt):
    """The reference's op sequence promotes half heads to fp32 (xs + reg, heat * keep.float(), the final cat), so
    on half tensors it returns the dets of the upcast, up to the order of tied scores."""
    from oracle import torch_port as TP
    heat, wh, reg = [t.to(dt) for t in _bench_heads(2)]
    got = TP.ctdet_decode(heat, wh, reg=reg, K=100)
    want = TP.ctdet_decode(heat.float(), wh.float(), reg=reg.float(), K=100)
    assert got.dtype == torch.float32
    assert_dets_equal(want.numpy(), got.numpy(), what="torch_port %s" % dt)
    # half inputs make ties at the K-th score routine: the defined order matters here
    s = got[:, :, 4].numpy()
    assert any(int(np.sum(s[b] == s[b, -1])) > 1 for b in range(s.shape[0]))

"""CPU: the fused head's size queries and argument checks (before any CUDA call), and fuse_heads on toy models shaped
like DLASeg, PoseResNet and the hourglass network: which heads it replaces, the unchanged state dict and the fall-back
to the original layers.  No kernel runs here."""
import io

import pytest
import torch
from torch import nn

from centernet_b200 import heads as H


def test_tile_and_workspace_bytes():
    from centernet_b200 import _C
    # W1: one bf16 tile [128 or head_conv][32] per (pass, 32-channel block, tap); W2: one [N2][32] per 32 channels
    assert _C.head_w1t_bytes(64, 256) == 2 * 2 * 9 * 128 * 32 * 2
    assert _C.head_w1t_bytes(256, 64) == 8 * 9 * 64 * 32 * 2
    assert _C.head_w1t_bytes(64, 96) == 2 * 9 * 128 * 32 * 2       # head_conv padded to 128
    assert _C.head_w2t_bytes(256, 80) == 8 * 128 * 32 * 2          # C padded to the next power of two >= 8
    assert _C.head_w2t_bytes(64, 1) == 2 * 8 * 32 * 2
    assert _C.head_w2t_bytes(256, 256) == 8 * 256 * 32 * 2
    F32, BF16 = _C.DTYPE_F32, _C.DTYPE_BF16
    q = _C.head_workspace_bytes
    assert q(8, 64, 128, 128, BF16, 1) == 0                          # read in place
    assert q(8, 64, 128, 128, BF16, 0) == 8 * 128 * 128 * 64 * 2     # bf16 channels-last copy
    assert q(8, 64, 128, 128, F32, 1) == 8 * 128 * 128 * 64 * 2


def test_queries_return_zero_outside_the_range():
    from centernet_b200 import _C
    assert _C.head_w1t_bytes(48, 256) == 0      # cin not a multiple of 32
    assert _C.head_w1t_bytes(64, 288) == 0      # head_conv > 256
    assert _C.head_w1t_bytes(64, 100) == 0      # head_conv not a multiple of 32
    assert _C.head_w2t_bytes(256, 257) == 0     # C > 256
    assert _C.head_w2t_bytes(256, 0) == 0
    assert _C.head_workspace_bytes(0, 64, 8, 8, 0, 0) == 0
    assert _C.head_workspace_bytes(1 << 16, 64, 256, 256, 0, 0) == 0   # beyond 32-bit indexing


def test_forward_and_prepare_reject_bad_arguments():
    from centernet_b200 import _C
    F32, BF16 = _C.DTYPE_F32, _C.DTYPE_BF16
    f = _C.head_forward_bf16
    shape = (2, 64, 16, 16, 256, 80)   # b, cin, h, w, head_conv, C
    need = _C.head_workspace_bytes(2, 64, 16, 16, F32, 0)
    # input, dtype, cl, w1t, b1, w2t, b2, out, shape..., ws, bytes, stream
    with pytest.raises(RuntimeError, match="null pointer"):
        f(0, F32, 0, 16, 16, 16, 16, 16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="null pointer"):
        f(16, F32, 0, 16, 0, 16, 16, 16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="dtype"):
        f(16, _C.DTYPE_F16, 0, 16, 16, 16, 16, 16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="bad shape"):
        f(16, F32, 0, 16, 16, 16, 16, 16, 2, 64, 0, 16, 256, 80, 256, need, 0)
    with pytest.raises(NotImplementedError, match="multiples of 32"):
        f(16, F32, 0, 16, 16, 16, 16, 16, 2, 48, 16, 16, 256, 80, 256, need, 0)
    with pytest.raises(NotImplementedError, match="multiples of 32"):
        f(16, F32, 0, 16, 16, 16, 16, 16, 2, 64, 16, 16, 256, 300, 256, need, 0)
    with pytest.raises(NotImplementedError, match="32-bit"):
        f(16, F32, 0, 16, 16, 16, 16, 16, 1 << 16, 64, 256, 256, 256, 80, 256, 1 << 40, 0)
    with pytest.raises(RuntimeError, match="null workspace"):
        f(16, F32, 0, 16, 16, 16, 16, 16, *shape, 0, need, 0)
    with pytest.raises(RuntimeError, match="workspace"):
        f(16, F32, 0, 16, 16, 16, 16, 16, *shape, 256, need - 1, 0)
    with pytest.raises(RuntimeError, match="aligned"):
        f(24, F32, 0, 16, 16, 16, 16, 16, *shape, 256, need, 0)
    with pytest.raises(RuntimeError, match="aligned"):
        f(16, BF16, 1, 16, 16, 40, 16, 16, *shape, 0, 0, 0)
    p = _C.head_prepare_weights_bf16
    n1, n2 = _C.head_w1t_bytes(64, 256), _C.head_w2t_bytes(256, 80)
    with pytest.raises(RuntimeError, match="null pointer"):
        p(0, 16, 64, 256, 80, 256, n1, 512, n2, 0)
    with pytest.raises(RuntimeError, match="too small"):
        p(16, 16, 64, 256, 80, 256, n1 - 1, 512, n2, 0)
    with pytest.raises(RuntimeError, match="aligned"):
        p(16, 16, 64, 256, 80, 264, n1, 512, n2, 0)
    with pytest.raises(NotImplementedError, match="multiples of 32"):
        p(16, 16, 64, 256, 257, 256, n1, 512, n2, 0)


def _head(cin, head_conv, c, final_kernel=1):
    return nn.Sequential(nn.Conv2d(cin, head_conv, kernel_size=3, padding=1, bias=True), nn.ReLU(inplace=True),
                         nn.Conv2d(head_conv, c, kernel_size=final_kernel, stride=1, padding=final_kernel // 2,
                                   bias=True))


class DLASegLike(nn.Module):
    """The head block of pose_dla_dcn.DLASeg, with a stand-in backbone that holds Sequentials of its own (`base` has
    the head pattern itself, but is not a head)."""

    def __init__(self, heads, head_conv, final_kernel=1):
        super().__init__()
        self.base = nn.Sequential(nn.Conv2d(3, 64, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(64, 64, 1))
        self.ida = nn.Sequential(nn.Conv2d(64, 64, 3, padding=1, bias=False), nn.BatchNorm2d(64), nn.ReLU())
        self.heads = heads
        for h, c in heads.items():
            fc = _head(64, head_conv, c, final_kernel) if head_conv > 0 else \
                nn.Conv2d(64, c, kernel_size=final_kernel, padding=final_kernel // 2, bias=True)
            self.__setattr__(h, fc)

    def forward(self, x):
        y = self.ida(self.base(x))
        return {h: self.__getattr__(h)(y) for h in self.heads}


class Convolution(nn.Module):
    """large_hourglass.convolution: conv + optional BN + ReLU."""

    def __init__(self, k, inp, out, with_bn=True):
        super().__init__()
        self.conv = nn.Conv2d(inp, out, (k, k), padding=(k // 2, k // 2), bias=not with_bn)
        self.bn = nn.BatchNorm2d(out) if with_bn else nn.Sequential()
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        return self.relu(self.bn(self.conv(x)))


class HourglassLike(nn.Module):
    """large_hourglass.exkp: a ModuleList of `convolution` + Conv2d per head and stack."""

    def __init__(self, heads):
        super().__init__()
        self.heads = heads
        for h, c in heads.items():
            self.__setattr__(h, nn.ModuleList([nn.Sequential(Convolution(3, 256, 256, with_bn=False),
                                                             nn.Conv2d(256, c, (1, 1))) for _ in range(2)]))


def test_fuse_heads_replaces_exactly_the_head_sequentials():
    ctdet = {"hm": 80, "wh": 2, "reg": 2}
    m = DLASegLike(ctdet, 256)
    assert H.fuse_heads(m) == 3
    assert all(type(getattr(m, h)) is H.FusedHead for h in ctdet)
    assert type(m.base) is nn.Sequential and type(m.ida) is nn.Sequential
    assert H.fuse_heads(m) == 0                      # already fused
    pose = {"hm": 1, "wh": 2, "hps": 34, "reg": 2, "hm_hp": 17, "hp_offset": 2}
    assert H.fuse_heads(DLASegLike(pose, 64)) == 6   # PoseResNet-style head_conv = 64
    ddd = {"hm": 3, "dep": 1, "rot": 8, "dim": 3, "wh": 2, "reg": 2}
    assert H.fuse_heads(DLASegLike(ddd, 256)) == 6
    exdet = dict([("hm_" + s, 80) for s in ("t", "l", "b", "r", "ct")] + [("reg_" + s, 2) for s in "tlbr"])
    assert H.fuse_heads(DLASegLike(exdet, 256)) == 9
    assert H.fuse_heads(DLASegLike(ctdet, 0)) == 0                  # head_conv = 0: single conv heads
    assert H.fuse_heads(DLASegLike(ctdet, 256, final_kernel=3)) == 0
    assert H.fuse_heads(HourglassLike(ctdet)) == 0
    # a head the kernel does not cover is still fused: it runs the original layers at call time
    assert H.fuse_heads(DLASegLike({"hm": 300}, 256)) == 1


def test_is_fusable_head_needs_the_exact_pattern():
    assert H.is_fusable_head(_head(64, 256, 80))
    assert not H.is_fusable_head(nn.Sequential(nn.Conv2d(64, 256, 3, padding=1, bias=False), nn.ReLU(),
                                               nn.Conv2d(256, 80, 1)))
    assert not H.is_fusable_head(nn.Sequential(nn.Conv2d(64, 256, 3, padding=1), nn.ReLU6(), nn.Conv2d(256, 80, 1)))
    assert not H.is_fusable_head(nn.Sequential(nn.Conv2d(64, 256, 3, padding=2, dilation=2), nn.ReLU(),
                                               nn.Conv2d(256, 80, 1)))
    assert not H.is_fusable_head(nn.Sequential(nn.Conv2d(64, 256, 3, padding=1, stride=2), nn.ReLU(),
                                               nn.Conv2d(256, 80, 1)))
    assert not H.is_fusable_head(nn.Sequential(nn.Conv2d(64, 256, 3, padding=1, groups=2), nn.ReLU(),
                                               nn.Conv2d(256, 80, 1)))
    assert not H.is_fusable_head(nn.Sequential(nn.Conv2d(64, 256, 3, padding=1), nn.ReLU(), nn.Conv2d(256, 80, 1),
                                               nn.Sigmoid()))


def _state_bytes(model):
    buf = io.BytesIO()
    torch.save(model.state_dict(), buf)
    return {k: v.numpy().tobytes() for k, v in model.state_dict().items()}, buf.getvalue()


def test_state_dict_round_trip_byte_for_byte():
    torch.manual_seed(0)
    ref = DLASegLike({"hm": 80, "wh": 2, "reg": 2}, 256)
    before, _ = _state_bytes(ref)
    fused = DLASegLike({"hm": 80, "wh": 2, "reg": 2}, 256)
    H.fuse_heads(fused)
    assert list(fused.state_dict().keys()) == list(ref.state_dict().keys())
    assert "hm.0.weight" in fused.state_dict() and "hm.2.bias" in fused.state_dict()
    fused.load_state_dict(ref.state_dict())          # a checkpoint saved before fusing loads after
    after, _ = _state_bytes(fused)
    assert after == before
    back = DLASegLike({"hm": 80, "wh": 2, "reg": 2}, 256)
    back.load_state_dict(fused.state_dict())         # and one saved after fusing loads into the plain model
    assert _state_bytes(back)[0] == before


def test_fall_back_runs_the_original_layers():
    torch.manual_seed(1)
    m = DLASegLike({"hm": 4, "wh": 2}, 64)
    x = torch.randn(2, 3, 12, 10)
    with torch.no_grad():
        want = m(x)
    H.fuse_heads(m)
    with torch.no_grad():                            # CPU tensors
        got = m(x)
    for k in want:
        assert torch.equal(got[k], want[k])
    got = m(x)                                       # grad enabled: autograd through the original layers
    assert got["hm"].requires_grad
    got["hm"].sum().backward()
    assert m.hm[0].weight.grad is not None
    head = m.hm
    with torch.no_grad():
        assert not head._fused_ok(torch.randn(1, 64, 8, 8))                       # CPU
        assert not head._fused_ok(torch.randn(1, 64, 8, 8, dtype=torch.float64))

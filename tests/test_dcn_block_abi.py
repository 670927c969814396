"""DCN block (cnb_dcnv2_forward_block_bf16) without a GPU: size queries, validation codes, fuse_offset_conv and which
path a module takes.  The path checks run on a tensor that reports itself as CUDA, with every forward entry point of
the C module replaced by a stub that records its name, so nothing is launched."""
import pytest
import torch
from torch import nn

from centernet_b200 import _C
from centernet_b200 import dcn_v2 as D
from centernet_b200 import dcn_v2_func as DF

BF = torch.bfloat16


def test_om_tile_and_workspace_bytes():
    for cin in (32, 64, 256, 512):
        assert _C.dcnv2_om_tiles_bytes(cin, 3, 3, 1) == (cin // 32) * 9 * 32 * 32 * 2
    need = _C.dcnv2_block_workspace_bytes(2, 64, 128, 40, 56, 3, 3, 1, 1, 1, 1)
    assert need == _C.dcnv2_bf16_workspace_bytes(2, 64, 128, 40, 56, 3, 3, 1, 1, 1, 1) > 0
    assert _C.dcnv2_block_workspace_bytes(65, 512, 72, 17, 5, 3, 3, 1, 1, 1, 1) > 0


@pytest.mark.parametrize("cin,kh,kw,stride,pad,dil,dg", [
    (48, 3, 3, 1, 1, 1, 1), (64, 1, 1, 1, 0, 1, 1), (64, 3, 3, 2, 1, 1, 1), (64, 3, 3, 1, 0, 1, 1),
    (64, 3, 3, 1, 2, 2, 1), (64, 3, 3, 1, 1, 1, 2), (64, 5, 5, 1, 2, 1, 1), (0, 3, 3, 1, 1, 1, 1)])
def test_queries_return_zero_outside_the_range(cin, kh, kw, stride, pad, dil, dg):
    assert _C.dcnv2_block_workspace_bytes(2, cin, 64, 32, 32, kh, kw, stride, pad, dil, dg) == 0
    if stride == 1 and pad == 1 and dil == 1:
        assert _C.dcnv2_om_tiles_bytes(cin, kh, kw, dg) == 0


def test_forward_and_prepare_reject_bad_arguments():
    F32, BF16 = _C.DTYPE_F32, _C.DTYPE_BF16
    f = _C.dcnv2_forward_block_bf16
    shape = (2, 64, 16, 16, 128, 3, 3, 1, 1, 1, 1)   # b, cin, h, w, cout, kh, kw, stride, pad, dil, dg
    need = _C.dcnv2_block_workspace_bytes(2, 64, 128, 16, 16, 3, 3, 1, 1, 1, 1)

    def call(x=16, dt=F32, cl=0, omt=16, bom=16, wt=16, b=16, sc=0, sh=0, out=16, shp=shape, ws=256, nbytes=need):
        f(x, dt, cl, omt, bom, wt, b, sc, sh, 1, out, *shp, ws, nbytes, 0)

    for kw in ({"x": 0}, {"omt": 0}, {"wt": 0}, {"out": 0}, {"ws": 0}):
        with pytest.raises(RuntimeError, match="null pointer"):
            call(**kw)
    with pytest.raises(RuntimeError, match="go together"):
        call(sc=16)
    with pytest.raises(RuntimeError, match="dtype"):
        call(dt=_C.DTYPE_F16)
    with pytest.raises(RuntimeError, match="non-positive"):
        call(shp=(2, 64, 0, 16, 128, 3, 3, 1, 1, 1, 1))
    for shp in ((2, 48, 16, 16, 128, 3, 3, 1, 1, 1, 1), (2, 64, 16, 16, 128, 3, 3, 2, 1, 1, 1),
                (2, 64, 16, 16, 128, 1, 1, 1, 0, 1, 1), (2, 64, 16, 16, 128, 3, 3, 1, 1, 1, 2)):
        with pytest.raises(NotImplementedError, match="3x3 kernel"):
            call(shp=shp)
    with pytest.raises(RuntimeError, match="workspace too small"):
        call(nbytes=need - 1)
    for kw in ({"x": 24}, {"omt": 40}, {"wt": 8}, {"ws": 264}):
        with pytest.raises(RuntimeError, match="aligned"):
            call(**kw)
    p = _C.dcnv2_prepare_om_weights_bf16
    n = _C.dcnv2_om_tiles_bytes(64, 3, 3, 1)
    with pytest.raises(RuntimeError, match="null pointer"):
        p(0, 64, 3, 3, 1, 256, n, 0)
    with pytest.raises(RuntimeError, match="bad shape"):
        p(16, 0, 3, 3, 1, 256, n, 0)
    with pytest.raises(NotImplementedError, match="3x3 kernel"):
        p(16, 64, 3, 3, 2, 256, n, 0)
    with pytest.raises(RuntimeError, match="buffer"):
        p(16, 64, 3, 3, 1, 256, n - 1, 0)
    with pytest.raises(RuntimeError, match="aligned"):
        p(16, 64, 3, 3, 1, 264, n, 0)


# ------------------------------------------------------------------ modules
class DeformConv(nn.Module):
    """pose_dla_dcn.DeformConv"""

    def __init__(self, chi, cho, **kw):
        super().__init__()
        self.actf = nn.Sequential(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))
        self.conv = D.DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1, **kw)

    def forward(self, x):
        return self.actf(self.conv(x))


class DLAUpLike(nn.Module):
    """The IDAUp of DLASeg: proj_i / node_i DeformConvs and ConvTranspose2d ups (pose_dla_dcn.py:360-390)."""

    def __init__(self, chs=(64, 128, 256)):
        super().__init__()
        for i, c in enumerate(chs[1:], 1):
            setattr(self, "proj_%d" % i, DeformConv(c, chs[0]))
            setattr(self, "up_%d" % i, nn.ConvTranspose2d(chs[0], chs[0], 4, stride=2, padding=1, groups=chs[0]))
            setattr(self, "node_%d" % i, DeformConv(chs[0], chs[0]))
        self.base = nn.Conv2d(3, chs[0], 3, padding=1)


class PoseResNetLike(nn.Module):
    """resnet_dcn's deconv layers: DCN, BN, ReLU, ConvTranspose2d, BN, ReLU per stage (resnet_dcn.py:216-250)."""

    def __init__(self, chs=(512, 256, 128, 64)):
        super().__init__()
        layers = []
        for a, b in zip(chs[:-1], chs[1:]):
            layers += [D.DCN(a, b, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1),
                       nn.BatchNorm2d(b), nn.ReLU(inplace=True), nn.ConvTranspose2d(b, b, 4, stride=2, padding=1),
                       nn.BatchNorm2d(b), nn.ReLU(inplace=True)]
        self.deconv_layers = nn.Sequential(*layers)


def test_fuse_offset_conv_counts_and_keeps_the_state_dict():
    for model, n in ((DLAUpLike(), 4), (PoseResNetLike(), 3), (nn.Sequential(nn.Conv2d(3, 8, 3)), 0)):
        keys = list(model.state_dict().keys())
        assert D.fuse_offset_conv(model) == n
        assert list(model.state_dict().keys()) == keys
        assert D.fuse_offset_conv(model) == n                      # idempotent
        assert sum(getattr(m, "offset_conv_fused", False) for m in model.modules()) == n
    plain = D.DCNv2(64, 64, 3, 1, 1)                               # no conv_offset_mask: not a DCN block
    assert D.fuse_offset_conv(nn.Sequential(plain)) == 0


class FakeCuda(torch.Tensor):
    """A CPU tensor that reports itself as CUDA, so the module takes its GPU branches into the stubbed C module."""

    @property
    def is_cuda(self):
        return True


class StubC:
    """The C module with every forward entry point and weight preparation recorded instead of run."""

    def __init__(self, block_ws=None):
        self.calls = []
        self.block_ws = block_ws

    def __getattr__(self, name):
        if name.startswith("dcnv2_forward") or name.startswith("dcnv2_prepare_"):
            return lambda *a: self.calls.append((name, a))
        return getattr(_C, name)

    def dcnv2_block_workspace_bytes(self, *a):
        return _C.dcnv2_block_workspace_bytes(*a) if self.block_ws is None else self.block_ws

    def forwards(self):
        return [c[0] for c in self.calls if c[0].startswith("dcnv2_forward")]


@pytest.fixture
def stub(monkeypatch):
    s = StubC()
    monkeypatch.setattr(DF, "C", s)
    monkeypatch.setattr(DF, "stream_ptr", lambda t: 0)
    return s


def _fake(x):
    return torch.Tensor._make_subclass(FakeCuda, x)


def _block(chi=64, cho=64, **kw):
    torch.manual_seed(0)
    m = DeformConv(chi, cho, **kw).eval()
    m.actf[0].running_var.fill_(2.0)
    return m


def _run(m, x, grad=False):
    with torch.set_grad_enabled(grad):
        return m(x)


@pytest.mark.parametrize("order", ["flag_first", "dtype_first", "bn_first"])
def test_composes_with_set_compute_dtype_and_fuse_dcn_bn_relu_in_any_order(stub, order):
    m = _block()
    steps = {"flag_first": (D.fuse_offset_conv, lambda m: D.set_compute_dtype(m, BF), D.fuse_dcn_bn_relu),
             "dtype_first": (lambda m: D.set_compute_dtype(m, BF), D.fuse_dcn_bn_relu, D.fuse_offset_conv),
             "bn_first": (D.fuse_dcn_bn_relu, D.fuse_offset_conv, lambda m: D.set_compute_dtype(m, BF))}[order]
    for step in steps:
        step(m)
    x = _fake(torch.randn(2, 64, 12, 20))
    y = _run(m, x)
    assert stub.forwards() == ["dcnv2_forward_block_bf16"]
    a = stub.calls[-1][1]
    assert a[1] == _C.DTYPE_F32 and a[2] == 0 and a[7] != 0 and a[8] != 0 and a[9] == 1   # BN folded, relu
    assert a[11:22] == (2, 64, 12, 20, 64, 3, 3, 1, 1, 1, 1)
    assert y.shape == (2, 64, 12, 20) and y.dtype == torch.float32
    # the DCN on its own: no BN, no relu
    stub.calls.clear()
    _run(m.conv, x)
    a = stub.calls[-1][1]
    assert stub.forwards() == ["dcnv2_forward_block_bf16"] and a[7] == 0 and a[8] == 0 and a[9] == 0
    # bf16 channels_last input: read in place, output bf16
    stub.calls.clear()
    xb = _fake(torch.randn(2, 64, 12, 20).to(BF).contiguous(memory_format=torch.channels_last))
    assert _run(m.conv, xb).dtype == BF
    a = stub.calls[-1][1]
    assert a[1] == _C.DTYPE_BF16 and a[2] == 1 and a[0] == xb.data_ptr()


def _fall_back_cases():
    def grad(m, x):
        return _run(m, x, grad=True)

    def training(m, x):
        m.train()
        return _run(m, x)

    def no_dtype(m, x):
        D.set_compute_dtype(m, None)
        return _run(m, x)

    def unflagged(m, x):
        for mod in m.modules():
            mod.offset_conv_fused = False
        return _run(m, x)

    return {"grad": grad, "training": training, "compute_dtype_none": no_dtype, "unflagged": unflagged}


@pytest.mark.parametrize("case", sorted(_fall_back_cases()))
@pytest.mark.parametrize("with_bn", [False, True])
def test_every_fall_back_takes_the_old_path(stub, case, with_bn):
    fn = _fall_back_cases()[case]
    want, got = [], []
    for flagged, rec in ((False, want), (True, got)):
        m = _block()
        D.set_compute_dtype(m, BF)
        if with_bn:
            D.fuse_dcn_bn_relu(m)
        if flagged:
            D.fuse_offset_conv(m)
        stub.calls.clear()
        fn(m if with_bn else m.conv, _fake(torch.randn(2, 64, 12, 20)))
        rec += stub.forwards()
    assert got == want and "dcnv2_forward_block_bf16" not in got and got


@pytest.mark.parametrize("kw,chi", [({"stride": 2}, 64), ({"padding": 0}, 64),
                                    ({"deformable_groups": 2}, 64), ({"kernel_size": 1, "padding": 0}, 64),
                                    ({}, 48)])
def test_out_of_range_modules_take_the_old_path(stub, kw, chi):
    args = dict(in_channels=chi, out_channels=64, kernel_size=3, stride=1, padding=1, dilation=1, deformable_groups=1)
    args.update(kw)
    torch.manual_seed(0)
    for flagged, rec in ((False, []), (True, [])):
        m = D.DCN(**args).eval()
        D.set_compute_dtype(m, BF)
        if flagged:
            D.fuse_offset_conv(m)
        stub.calls.clear()
        _run(m, _fake(torch.randn(2, chi, 12, 20)))
        rec += stub.forwards()
        if flagged:
            assert rec == want and rec == ["dcnv2_forward_fused_bf16"]
        else:
            want = rec


def test_zero_workspace_query_and_other_inputs_take_the_old_path(stub, monkeypatch):
    m = _block()
    D.set_compute_dtype(m, BF)
    D.fuse_offset_conv(m)
    stub.block_ws = 0                                   # the kernel declines the shape
    _run(m.conv, _fake(torch.randn(2, 64, 12, 20)))
    assert stub.forwards() == ["dcnv2_forward_fused_bf16"]
    stub.block_ws = None
    with pytest.raises(NotImplementedError):           # CPU tensors: today's error
        _run(m.conv, torch.randn(2, 64, 12, 20))
    stub.calls.clear()
    m64 = _block().double()
    D.set_compute_dtype(m64, BF)
    D.fuse_offset_conv(m64)
    with pytest.raises(RuntimeError, match="float32 or bfloat16"):   # float64: today's bf16-path error
        _run(m64.conv, _fake(torch.randn(2, 64, 12, 20, dtype=torch.float64)))
    assert "dcnv2_forward_block_bf16" not in stub.forwards()
    assert DF.dcn_block_inference(torch.randn(1, 64, 8, 8), m.conv.conv_offset_mask.weight,
                                  m.conv.conv_offset_mask.bias, m.conv.weight, m.conv.bias, 1, 1, 1, 1) is None

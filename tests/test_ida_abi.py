"""IDA up-sampling step (cnb_ida_up_add) without a GPU: the validation codes of the entry point, which modules
fuse_ida_up rewires, the state dict, idempotence and which path each step takes.  The path checks run on tensors that
report themselves as CUDA, with the entry point replaced by a stub that records its arguments, so nothing is
launched."""
import io
import math

import pytest
import torch
from torch import nn

from centernet_b200 import _C
from centernet_b200 import dcn_v2 as D
from centernet_b200 import ida as I

BF = torch.bfloat16


# ------------------------------------------------------------------ toy networks (behaviour of pose_dla_dcn / dlav0)
def bilinear_(up):
    """The bilinear up-sampling kernel pose_dla_dcn's fill_up_weights puts in every channel of a ConvTranspose2d."""
    k = up.weight.shape[2]
    f = math.ceil(k / 2)
    centre = (2 * f - 1 - f % 2) / (2.0 * f)
    row = torch.tensor([1 - abs(i / f - centre) for i in range(k)])
    with torch.no_grad():
        up.weight.copy_((row[:, None] * row[None, :]).expand_as(up.weight))
    return up


class DeformConv(nn.Module):
    """DCN 3x3, then BatchNorm2d + ReLU."""

    def __init__(self, chi, cho):
        super().__init__()
        self.actf = nn.Sequential(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))
        self.conv = D.DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)

    def forward(self, x):
        return self.actf(self.conv(x))


class IDAUp(nn.Module):
    """An IDA step per input after the first: project it to o channels, up-sample it by its factor, add the previous
    map and aggregate with a node; `layers` is updated in place."""

    def __init__(self, o, chs, up_f):
        super().__init__()
        for i in range(1, len(chs)):
            f = int(up_f[i])
            setattr(self, "proj_%d" % i, DeformConv(chs[i], o))
            setattr(self, "up_%d" % i, bilinear_(nn.ConvTranspose2d(o, o, 2 * f, stride=f, padding=f // 2,
                                                                    groups=o, bias=False)))
            setattr(self, "node_%d" % i, DeformConv(o, o))

    def forward(self, layers, startp, endp):
        for i in range(startp + 1, endp):
            k = i - startp
            layers[i] = getattr(self, "up_%d" % k)(getattr(self, "proj_%d" % k)(layers[i]))
            layers[i] = getattr(self, "node_%d" % k)(layers[i] + layers[i - 1])


class Neck(nn.Module):
    """DLASeg's dla_up and ida_up for dla_34 at down_ratio 4: inputs of 64, 128, 256 and 512 channels at strides 4,
    8, 16 and 32.  Its 8 up layers are those of the dla_34 table in DESIGN §4.14."""

    def __init__(self, chs=(64, 128, 256, 512)):
        super().__init__()
        self.dla_up = nn.Module()
        n = len(chs)
        for i in range(n - 1):            # ida_i merges the i + 2 coarsest maps into channels chs[n - 2 - i]
            o = chs[n - 2 - i]
            ins = [o] + [chs[n - 1 - i]] * (i + 1)
            setattr(self.dla_up, "ida_%d" % i, IDAUp(o, ins, [1] + [2] * (i + 1)))
        self.ida_up = IDAUp(chs[0], list(chs[:3]), [1, 2, 4])

    def forward(self, layers):
        layers = list(layers)
        out = [layers[-1]]
        for i in range(len(layers) - 1):
            getattr(self.dla_up, "ida_%d" % i)(layers, len(layers) - i - 2, len(layers))
            out.insert(0, layers[-1])
        y = [out[i].clone() for i in range(3)]
        self.ida_up(y, 0, len(y))
        return y[-1]


def neck_inputs(B, top, dtype=torch.float32, device="cpu", seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, c, top >> i, top >> i, generator=g).to(device=device, dtype=dtype)
            for i, c in enumerate((64, 128, 256, 512))]


class Dlav0IDAUp(nn.Module):
    """dlav0's IDAUp: the same attribute names, a 1x1-conv projection per input, a node on the concatenation."""

    def __init__(self, o=16, chs=(16, 32), up_f=(1, 2)):
        super().__init__()
        for i, c in enumerate(chs):
            f = up_f[i]
            setattr(self, "proj_%d" % i, nn.Identity() if c == o else nn.Conv2d(c, o, 1, bias=False))
            setattr(self, "up_%d" % i, nn.Identity() if f == 1 else
                    nn.ConvTranspose2d(o, o, 2 * f, stride=f, padding=f // 2, groups=o, bias=False))
        for i in range(1, len(chs)):
            setattr(self, "node_%d" % i, nn.Conv2d(2 * o, o, 3, padding=1, bias=False))

    def forward(self, layers):
        layers = [getattr(self, "up_%d" % i)(getattr(self, "proj_%d" % i)(x)) for i, x in enumerate(layers)]
        x = layers[0]
        for i in range(1, len(layers)):
            x = getattr(self, "node_%d" % i)(torch.cat([x, layers[i]], 1))
        return x


class ConvIDAUp(IDAUp):
    """The pose_dla_dcn forward over plain Conv2d projections and nodes: not DeformConv-shaped."""

    def __init__(self):
        nn.Module.__init__(self)
        self.proj_1 = nn.Conv2d(32, 16, 3, padding=1)
        self.up_1 = nn.ConvTranspose2d(16, 16, 4, stride=2, padding=1, groups=16, bias=False)
        self.node_1 = nn.Conv2d(16, 16, 3, padding=1)


def test_neck_has_the_dla34_up_shapes():
    shapes = sorted((m.in_channels, m.stride[0]) for m in Neck().modules() if isinstance(m, nn.ConvTranspose2d))
    assert shapes == sorted([(256, 2), (128, 2), (128, 2), (64, 2), (64, 2), (64, 2), (64, 2), (64, 4)])


# ------------------------------------------------------------------ C entry point: validation codes
def test_entry_rejects_bad_arguments():
    F32, BF16 = _C.DTYPE_F32, _C.DTYPE_BF16
    f = _C.ida_up_add

    def call(p=16, dt=F32, pcl=0, w=16, fac=2, skip=16, scl=0, out=32, ocl=0, shp=(2, 64, 8, 8)):
        f(p, dt, pcl, w, fac, skip, scl, out, ocl, *shp, 0)

    for kw in ({"p": 0}, {"w": 0}, {"skip": 0}, {"out": 0}):
        with pytest.raises(RuntimeError, match="null pointer"):
            call(**kw)
    for dt in (_C.DTYPE_F16, 7, -1):
        with pytest.raises(RuntimeError, match="dtype"):
            call(dt=dt)
    for kw in ({"pcl": 2}, {"scl": -1}, {"ocl": 3}):
        with pytest.raises(RuntimeError, match="0 or 1"):
            call(**kw)
    for shp in ((0, 64, 8, 8), (2, 0, 8, 8), (2, 64, 0, 8), (2, 64, 8, -1)):
        with pytest.raises(RuntimeError, match="bad shape"):
            call(shp=shp)
    for kw in ({"skip": 24}, {"out": 40}, {"p": 18}, {"w": 18}, {"p": 17, "dt": BF16}):
        with pytest.raises(RuntimeError, match="aligned"):
            call(**kw)
    for fac in (1, 3, 16, 0):
        with pytest.raises(NotImplementedError, match="up factor"):
            call(fac=fac)
    with pytest.raises(NotImplementedError, match="32-bit"):
        call(shp=(64, 256, 256, 256))
    for st in (_C.EINVAL, _C.EUNSUPPORTED):
        assert st != _C.OK


# ------------------------------------------------------------------ fuse_ida_up: what it matches
def _state_bytes(model):
    buf = io.BytesIO()
    torch.save(model.state_dict(), buf)
    return buf.getvalue()


def test_counts_the_dla34_neck_and_leaves_look_alikes_alone():
    neck = Neck()
    before = _state_bytes(neck)
    assert I.fuse_ida_up(neck) == 8
    assert _state_bytes(neck) == before
    assert I.fuse_ida_up(neck) == 8                                      # idempotent
    fwd = neck.ida_up.forward
    assert I.fuse_ida_up(neck) == 8 and neck.ida_up.forward is fwd       # not wrapped twice
    assert _state_bytes(neck) == before
    for other in (Dlav0IDAUp(), nn.Sequential(nn.Conv2d(3, 8, 3), nn.ConvTranspose2d(8, 8, 4, 2, 1, groups=8)),
                  ConvIDAUp()):
        assert I.fuse_ida_up(other) == 0 and "forward" not in other.__dict__


@pytest.mark.parametrize("change", ["bias", "f3", "dense", "padding", "output_padding", "gap", "proj_0"])
def test_steps_outside_the_pattern_leave_the_module_alone(change):
    m = IDAUp(16, [16, 32, 32], [1, 2, 2])
    if change == "bias":
        m.up_2 = nn.ConvTranspose2d(16, 16, 4, stride=2, padding=1, groups=16, bias=True)
    elif change == "f3":
        m.up_2 = nn.ConvTranspose2d(16, 16, 6, stride=3, padding=1, groups=16, bias=False)
    elif change == "dense":
        m.up_2 = nn.ConvTranspose2d(16, 16, 4, stride=2, padding=1, bias=False)
    elif change == "padding":
        m.up_2 = nn.ConvTranspose2d(16, 16, 4, stride=2, padding=2, groups=16, bias=False)
    elif change == "output_padding":
        m.up_2 = nn.ConvTranspose2d(16, 16, 4, stride=2, padding=1, output_padding=1, groups=16, bias=False)
    elif change == "gap":
        del m.node_1
    else:
        m.proj_0 = DeformConv(16, 16)
    assert I.fuse_ida_up(m) == 0 and "forward" not in m.__dict__
    assert I.fuse_ida_up(IDAUp(16, [16, 32, 32], [1, 2, 4])) == 2


# ------------------------------------------------------------------ which path a step takes
class FakeCuda(torch.Tensor):
    """A CPU tensor that reports itself as CUDA, so a step takes its GPU branch into the stubbed C module."""

    @property
    def is_cuda(self):
        return True


def _fake(x):
    return torch.Tensor._make_subclass(FakeCuda, x, x.requires_grad)


class StubC:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return getattr(_C, name)

    def ida_up_add(self, *a):
        self.calls.append(a)


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(I, "_F2_MIN_OUT", 0)          # the small maps below would take the original step
    s = StubC()
    monkeypatch.setattr(I, "C", s)
    monkeypatch.setattr(I, "stream_ptr", lambda t: 0)
    return s


class Recorder(nn.Module):
    """Stands in for a proj / node: passes its input through and records it."""

    def __init__(self):
        super().__init__()
        self.seen = []

    def forward(self, x):
        self.seen.append(x)
        return x


def _step_module(o=16, f=2, dtype=torch.float32):
    """A one-step IDAUp whose proj and node are DeformConvs (so it matches) and then run as recorders."""
    m = IDAUp(o, [o, o], [1, f]).to(dtype)
    m.up_1.weight = nn.Parameter(_fake(m.up_1.weight.detach()))        # a weight that reports itself as CUDA
    assert I.fuse_ida_up(m) == 1
    proj, node = Recorder(), Recorder()
    m.proj_1.forward = proj.forward
    m.node_1.forward = node.forward
    return m, proj, node


def _layers(o=16, f=2, hp=3, wp=5, dtype=torch.float32, skip_cl=False, grad=False, fake=True):
    g = torch.Generator().manual_seed(0)
    skip = torch.randn(2, o, f * hp, f * wp, generator=g).to(dtype)
    p = torch.randn(2, o, hp, wp, generator=g).to(dtype)
    if skip_cl:
        skip = skip.contiguous(memory_format=torch.channels_last)
    if grad:
        p.requires_grad_(True)
    return [_fake(skip), _fake(p)] if fake else [skip, p]


def test_fused_step_passes_the_layouts_and_shapes(stub):
    for dtype, skip_cl, want_out_cl in ((torch.float32, False, 0), (torch.float32, True, 1), (BF, False, 0),
                                        (BF, True, 1)):
        stub.calls.clear()
        m, _, node = _step_module(dtype=dtype)
        layers = _layers(dtype=dtype, skip_cl=skip_cl)
        with torch.no_grad():
            m(layers, 0, 2)
        assert len(stub.calls) == 1
        a = stub.calls[0]
        assert a[1] == (_C.DTYPE_BF16 if dtype == BF else _C.DTYPE_F32) and a[2] == 0 and a[4] == 2
        assert a[6] == int(skip_cl) and a[8] == want_out_cl and a[9:13] == (2, 16, 3, 5)
        y = node.seen[-1]
        assert y.shape == (2, 16, 6, 10) and y.dtype == dtype
        assert y.is_contiguous(memory_format=torch.channels_last if want_out_cl else torch.contiguous_format)
        assert layers[1] is y                                            # the node's output replaces layers[1]


def _fall_back_cases(monkeypatch):
    def grad(m, layers):                       # grad mode, parameters requiring grad
        with torch.enable_grad():
            return m(layers, 0, 2)

    def grad_input(m, layers):                 # grad mode, an input requiring grad
        for p in m.parameters():
            p.requires_grad_(False)
        layers[1] = _fake(layers[1].detach().requires_grad_(True))
        with torch.enable_grad():
            return m(layers, 0, 2)

    def cpu(m, layers):
        layers[:] = [t.as_subclass(torch.Tensor) for t in layers]
        with torch.no_grad():
            return m(layers, 0, 2)

    def float64(m, layers):
        m.double()
        layers[:] = [_fake(t.double()) for t in layers]
        with torch.no_grad():
            return m(layers, 0, 2)

    def mixed(m, layers):                      # bf16 p, fp32 skip
        m.to(BF)
        layers[1] = _fake(layers[1].to(BF))
        with torch.no_grad():
            return m(layers, 0, 2)

    def weight_dtype(m, layers):               # the original conv raises its dtype error
        m.to(BF)
        with torch.no_grad(), pytest.raises(RuntimeError):
            m(layers, 0, 2)

    def autocast_f16(m, layers):
        monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
        monkeypatch.setattr(torch, "get_autocast_dtype", lambda *a: torch.float16)
        m.to(BF)
        layers[:] = [_fake(t.to(BF)) for t in layers]
        with torch.no_grad():
            return m(layers, 0, 2)

    def autocast_fp32_inputs(m, layers):
        monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
        monkeypatch.setattr(torch, "get_autocast_dtype", lambda *a: BF)
        with torch.no_grad():
            return m(layers, 0, 2)

    def shape(m, layers):                      # skip of the wrong size: the add's own error
        layers[0] = _fake(layers[0][..., :-1].contiguous())
        with torch.no_grad(), pytest.raises(RuntimeError, match="size"):
            m(layers, 0, 2)

    return {"grad": grad, "grad_input": grad_input, "cpu": cpu, "float64": float64, "mixed_dtypes": mixed,
            "weight_dtype": weight_dtype, "autocast_f16": autocast_f16,
            "autocast_bf16_fp32_inputs": autocast_fp32_inputs, "shape": shape}


@pytest.mark.parametrize("case", ["grad", "grad_input", "cpu", "float64", "mixed_dtypes", "weight_dtype",
                                  "autocast_f16", "autocast_bf16_fp32_inputs", "shape"])
def test_every_fall_back_runs_the_original_step(stub, monkeypatch, case):
    fn = _fall_back_cases(monkeypatch)[case]
    m, proj, node = _step_module()
    layers = _layers()
    fn(m, layers)
    assert stub.calls == []
    if node.seen:                               # the node got exactly up(p) + skip
        with torch.no_grad():
            want = m.up_1(proj.seen[-1]) + layers[0]
        assert torch.equal(node.seen[-1].detach(), want) and layers[1] is node.seen[-1]


def test_fall_back_output_equals_the_original_step(stub):
    m, _, node = _step_module()
    layers = _layers(fake=False)
    skip, p = layers
    m(layers, 0, 2)                                                      # CPU, grad mode: the original step
    with torch.no_grad():
        want = m.up_1(p) + skip
    assert stub.calls == [] and torch.equal(node.seen[-1].detach(), want)


def test_bf16_autocast_on_bf16_inputs_fuses_with_bf16_weights(stub, monkeypatch):
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
    monkeypatch.setattr(torch, "get_autocast_dtype", lambda *a: BF)
    m, _, node = _step_module()                                          # fp32 weights
    with torch.no_grad():
        m.up_1.weight.add_(1e-3)                                         # not representable in bf16
    layers = [_fake(t.to(BF)) for t in _layers()]
    with torch.no_grad():
        m(layers, 0, 2)
    assert len(stub.calls) == 1 and stub.calls[0][1] == _C.DTYPE_BF16
    w = m.up_1.__dict__["_cnb_ida_w"][3]
    assert w.dtype == torch.float32 and torch.equal(w, m.up_1.weight.detach().to(BF).float())


def test_grad_mode_without_anything_requiring_grad_fuses(stub):
    m, _, node = _step_module()
    for p in m.parameters():
        p.requires_grad_(False)
    with torch.enable_grad():
        m(_layers(), 0, 2)
    assert len(stub.calls) == 1


def test_weight_cache_follows_the_weight(stub):
    m, _, _ = _step_module(dtype=BF)                                    # bf16 weight: the cache holds a copy
    with torch.no_grad():
        m(_layers(dtype=BF), 0, 2)
        w0 = m.up_1.__dict__["_cnb_ida_w"][3]
        assert w0.dtype == torch.float32 and torch.equal(w0, m.up_1.weight.float())
        m(_layers(dtype=BF), 0, 2)
        assert m.up_1.__dict__["_cnb_ida_w"][3] is w0
        m.up_1.weight.mul_(2.0)                                          # in place: the version moves
        m(_layers(dtype=BF), 0, 2)
        assert torch.equal(m.up_1.__dict__["_cnb_ida_w"][3], w0 * 2)


def test_functional_form_validates_its_inputs():
    p, skip, w = torch.randn(1, 4, 3, 3), torch.randn(1, 4, 6, 6), torch.randn(4, 1, 4, 4)
    with pytest.raises(NotImplementedError, match="CUDA"):
        I.ida_up_add(p, w, 2, skip)
    fp, fs, fw = _fake(p), _fake(skip), _fake(w)
    with pytest.raises(TypeError, match="float32"):
        I.ida_up_add(_fake(p.double()), fw, 2, _fake(skip.double()))
    with pytest.raises(TypeError, match="float32"):
        I.ida_up_add(_fake(p.to(BF)), fw, 2, fs)
    with pytest.raises(ValueError, match="skip"):
        I.ida_up_add(fp, fw, 4, fs)
    with pytest.raises(ValueError, match="weight"):
        I.ida_up_add(fp, _fake(torch.randn(4, 1, 3, 3)), 2, fs)
    with pytest.raises(ValueError, match="p must"):
        I.ida_up_add(_fake(p[0]), fw, 2, fs)


def test_small_f2_steps_take_the_original_step(stub, monkeypatch):
    monkeypatch.setattr(I, "_F2_MIN_OUT", 2 * 16 * 6 * 10 + 1)
    m, _, node = _step_module()
    with torch.no_grad():
        m(_layers(), 0, 2)
    assert stub.calls == []
    monkeypatch.setattr(I, "_F2_MIN_OUT", 2 * 16 * 6 * 10)
    with torch.no_grad():
        m(_layers(), 0, 2)
    assert len(stub.calls) == 1
    stub.calls.clear()
    monkeypatch.setattr(I, "_F2_MIN_OUT", 1 << 30)
    m4, _, _ = _step_module(f=4)                       # f = 4 always fuses
    with torch.no_grad():
        m4(_layers(f=4), 0, 2)
    assert len(stub.calls) == 1 and stub.calls[0][4] == 4

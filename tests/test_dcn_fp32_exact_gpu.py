"""GPU: the default fp32 DCNv2 paths, bit for bit against the fp64 oracle on exact grids.

Paths: the 3xTF32 tensor-core forward (DCNv2Function on NCHW and channels_last input, cnb_dcnv2_forward with a
workspace), the fp32 CUDA-core forward (cnb_dcnv2_forward without one), the fused inference form (offset/mask glue in
the sampler, BN + ReLU in the epilogue), the tensor-core backward (default and deterministic mode, NCHW and the
channels_last _ex form) and the fp32 CUDA-core backward (no workspace, anisotropic stride/pad/dilation, dW above
Cout 256).

1. Exact grids.  x and dY in {0, +-1/2, +-1}, W in {0, +-1/16, +-1/8}, half-integer offsets (so the corner weights are
   in {0, 1/4, 1/2, 1}), mask in {1/4, 1/2, 1}, bias on the 1/8 grid below 1.  Every value has at most 6 significant
   bits, so its TF32 hi part is itself and its lo part 0: each 3xTF32 product is the exact product.  The largest case
   has Cin <= 256, Cout <= 272, 9 taps and B*Ho*Wo <= 2^12; there
     column value  sum_q w_q x_q m          lies on a 2^-5 grid, |.| <= 1                          ( 6 bits)
     output        b + sum_{c,t} W col      on a 2^-9 grid, |.| <= 1 + 256 * 9 / 8 = 289 < 2^9        (18 bits)
     dcol          sum_o W dY               on a 2^-5 grid, |.| <= 272 / 8 = 34 < 2^6               (11 bits)
     dW            sum_p dY col             on a 2^-6 grid, |.| <= B Ho Wo <= 2^12                  (18 bits)
     dMask         sum_c dcol val           on a 2^-8 grid (val on 2^-3), |.| <= 256 * 34 < 2^14    (22 bits)
     dOffset       sum_c dcol m cw          on a 2^-9 grid (cw, the corner difference, on 2^-2, |cw| <= 2),
                                            |.| <= 256 * 34 * 2 < 2^15                              (24 bits)
     dX            sum_{t,p} dcol m w_q     on a 2^-9 grid; with |offset| <= 3.5 a sample reaches an input
                                            element from at most 9 x 9 output pixels per tap, so
                                            |.| <= 34 * 9 * 81 < 2^15                               (24 bits)
     dBias         sum_p dY                 on a 2^-1 grid, |.| <= 2^12                             (13 bits)
   Every partial sum of these, in any order, is bounded by the sum of the magnitudes of its terms, so it is exact in
   fp32 too: the kernels must EQUAL the fp64 autograd of the oracle, in default mode as well (exact float atomics
   commute) and with the 64-bit fixed-point dX of deterministic mode.  The raw C ABI backward accumulates into its
   gradient buffers: they are pre-filled with G in {0, +-1/2, +-1}, which keeps every partial sum on its grid and below
   2^15 + 1, and must come back as G + oracle.  Each test first asserts that the fp64 answers are fp32 values.
   The fused form takes the raw conv_offset_mask output: mask logits 0 and 100 (sigmoid exactly 1/2 and 1), BN scale
   in {1/2, 1, 2} and shift on the 1/8 grid keep it exact (on a 2^-10 grid below 2^10).
2. Sampling boundaries.  For every tap, 100 output pixels sample exactly at h and w in {-1.5, -1, -0.5, 0, H-1,
   H-0.5, H, H+0.5, -40, H+40} (W for w), every combination; the other pixels keep the grid's offsets.  The cases
   have Cout <= 8 (dcol <= 1): however many samples fall by one input element, |dX| <= 9 * Ho * Wo <= 2^11, on the
   2^-9 grid (20 bits).  The other budgets of 1. are unchanged.  -1 and H sit just outside the open sampling box:
   the value there is 0 under either comparison, but dOffset at h = -1 is x[0] - 0 under `>=` and 0 under `>`.
3. Random data (offsets rounded to 2^-16, so fp32 and fp64 sample at the same points) against derived bounds; see
   test_random_within_derived_bound.
4. Anisotropic stride/pad/dilation through the C ABI: the CUDA-core kernels, exact grid; deterministic mode refuses
   them."""
import pytest
import torch

from oracle.dcn_ref import dcn_v2_forward
from test_bf16_bwd_gpu import NAMES, oracle_grads

pytestmark = pytest.mark.gpu


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def out_hw(H, W, kh, kw, stride, pad, dil):
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(pad), _pair(dil)
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil, seed=0):
    """The exact grid of 1. (stride / pad / dil may be (h, w) pairs)."""
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = out_hw(H, W, kh, kw, stride, pad, dil)
    kt = kh * kw
    x = torch.randint(-2, 3, (B, Ci, H, W), generator=g).float() / 2
    off = torch.randint(-7, 8, (B, 2 * kt * dg, Ho, Wo), generator=g).float() / 2
    m = torch.tensor([0.25, 0.5, 1.0])[torch.randint(0, 3, (B, kt * dg, Ho, Wo), generator=g)]
    w = torch.randint(-2, 3, (Co, Ci, kh, kw), generator=g).float() / 16
    b = torch.randint(-8, 9, (Co,), generator=g).float() / 8
    go = torch.randint(-2, 3, (B, Co, Ho, Wo), generator=g).float() / 2
    return x, off, m, w, b, go


def boundary_offsets(off, H, W, kh, kw, stride, pad, dil, dg):
    """Offsets that put the samples of output pixels 0..99 of every tap at each (h, w) of the boundary sets."""
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(pad), _pair(dil)
    B, _, Ho, Wo = off.shape
    assert Ho * Wo >= 100
    hs = (-1.5, -1.0, -0.5, 0.0, H - 1.0, H - 0.5, float(H), H + 0.5, -40.0, H + 40.0)
    ws = (-1.5, -1.0, -0.5, 0.0, W - 1.0, W - 0.5, float(W), W + 0.5, -40.0, W + 40.0)
    off = off.clone()
    kt = kh * kw
    for g in range(dg):
        for t in range(kt):
            i, j = t // kw, t % kw
            for p in range(100):
                ho, wo = p // Wo, p % Wo
                th, tw = hs[(p + t) % 10], ws[(p // 10 + 3 * t + g) % 10]
                off[:, g * 2 * kt + 2 * t, ho, wo] = th - (ho * sh - ph + i * dh)
                off[:, g * 2 * kt + 2 * t + 1, ho, wo] = tw - (wo * sw - pw + j * dw)
    return off


def _exact32(t):
    t32 = t.float()
    assert torch.equal(t32.double(), t), "the grid's fp64 answer is not an fp32 value"
    return t32


def _G(t, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-2, 3, t.shape, generator=g).float() / 2


def _ws(n, dev="cuda"):
    from centernet_b200._lib import workspace
    return workspace(n, dev)


def raw_forward(x, off, m, w, b, stride, pad, dil, dg, with_ws):
    from centernet_b200._lib import C, ptr, stream_ptr
    B, Ci, H, W = x.shape
    Co, _, kh, kw = w.shape
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(pad), _pair(dil)
    Ho, Wo = out_hw(H, W, kh, kw, stride, pad, dil)
    out = torch.full((B, Co, Ho, Wo), float("nan"), device=x.device)      # every element must be written
    ws, wsb = None, 0
    if with_ws:
        wsb = C.dcnv2_workspace_bytes(B, Ci, Co, H, W, kh, kw, sh, ph, dh, dg)
        assert wsb > 0
        ws = _ws(wsb)
    C.dcnv2_forward(ptr(x), ptr(off), ptr(m), ptr(w), ptr(b), ptr(out), B, Ci, H, W, Co, kh, kw, sh, sw, ph, pw, dh, dw,
                    dg, ptr(ws), wsb, stream_ptr(x))
    return out


def raw_backward(x, off, m, w, go, stride, pad, dil, dg, mode, which=NAMES, x_cl=False, seed=7):
    """One cnb_dcnv2_backward (mode "fp32": no workspace; "tc": with one) or, with x_cl, cnb_dcnv2_backward_ex on a
    channels_last input and grad_input.  The requested gradients start at G (returned too) and are accumulated into."""
    from centernet_b200._lib import C, ptr, stream_ptr
    B, Ci, H, W = x.shape
    Co, _, kh, kw = w.shape
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(pad), _pair(dil)
    shapes = {"input": x.shape, "offset": off.shape, "mask": m.shape, "weight": w.shape, "bias": (Co,)}
    G = {n: _G(torch.empty(shapes[n]), seed + k) for k, n in enumerate(NAMES) if n in which}
    buf = {n: t.cuda() for n, t in G.items()}
    xin = x
    if x_cl:
        xin = x.contiguous(memory_format=torch.channels_last)
        if "input" in buf:
            buf["input"] = buf["input"].contiguous(memory_format=torch.channels_last)
    ws, wsb = None, 0
    if mode == "tc":
        wsb = C.dcnv2_backward_workspace_bytes(B, Ci, Co, H, W, kh, kw, sh, ph, dh, dg)
        assert wsb > 0
        ws = _ws(wsb)
    gp = [ptr(buf.get(n)) for n in NAMES]
    if x_cl:
        C.dcnv2_backward_ex(ptr(xin), 1, ptr(off), ptr(m), ptr(w), ptr(go), gp[0], 1, *gp[1:], B, Ci, H, W, Co, kh, kw,
                            sh, ph, dh, dg, ptr(ws), wsb, stream_ptr(x))
    else:
        C.dcnv2_backward(ptr(xin), ptr(off), ptr(m), ptr(w), ptr(go), *gp, B, Ci, H, W, Co, kh, kw, sh, sw, ph, pw, dh,
                         dw, dg, ptr(ws), wsb, stream_ptr(x))
    if x_cl and "input" in buf:
        assert buf["input"].is_contiguous(memory_format=torch.channels_last)
    return [buf.get(n) for n in NAMES], [G.get(n) for n in NAMES]


def autograd(f, x, off, m, w, b, go):
    leaves = [None if t is None else t.detach().clone().requires_grad_(True) for t in (x, off, m, w, b)]
    f(*leaves).backward(go)
    return [None if t is None else t.grad for t in leaves]


def _det(on):
    from centernet_b200._lib import C
    torch.use_deterministic_algorithms(on)
    C.dcnv2_set_deterministic(int(on))


def check_forward(x, off, m, w, b, stride, pad, dil, dg):
    """Every fp32 forward path == the oracle (and the fused form == the oracle's BN + ReLU)."""
    from centernet_b200.dcn_v2_func import DCNv2Function, dcn_fused_inference
    Ci, Co = x.shape[1], w.shape[0]
    want = _exact32(dcn_v2_forward(x, off, m, w, b, stride, pad, dil, dg))
    xc, offc, mc, wc, bc = [t.cuda() for t in (x, off, m, w, b)]
    xcl = xc.contiguous(memory_format=torch.channels_last)
    f = DCNv2Function(stride, pad, dil, dg)
    for xin in (xc, xcl):            # channels_last with whole 32-channel blocks is sampled in place
        y = f(xin, offc, mc, wc, bc)
        assert y.dtype == torch.float32 and y.is_contiguous()
        assert torch.equal(y.cpu(), want), ("DCNv2Function", xin.is_contiguous())
    assert torch.equal(raw_forward(xc, offc, mc, wc, bc, stride, pad, dil, dg, True).cpu(), want), "ABI, workspace"
    assert torch.equal(raw_forward(xc, offc, mc, wc, bc, stride, pad, dil, dg, False).cpu(), want), "ABI, CUDA cores"
    want_nb = _exact32(dcn_v2_forward(x, off, m, w, None, stride, pad, dil, dg))
    assert torch.equal(f(xc, offc, mc, wc, None).cpu(), want_nb), "bias=None"
    assert torch.equal(raw_forward(xc, offc, mc, wc, None, stride, pad, dil, dg, False).cpu(), want_nb)

    g = torch.Generator().manual_seed(1)
    m2 = torch.where(m == 1.0, 1.0, 0.5)
    om = torch.cat([off, torch.where(m2 == 1.0, 100.0, 0.0)], dim=1).cuda()
    sc = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (Co,), generator=g)]
    sh = torch.randint(-8, 9, (Co,), generator=g).float() / 8
    y64 = dcn_v2_forward(x, off, m2, w, b, stride, pad, dil, dg)
    want_plain = _exact32(y64)
    want_bn = _exact32(torch.relu(y64 * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)))
    for xin in (xc, xcl):
        y = dcn_fused_inference(xin, om, wc, bc, stride, pad, dil, dg, bn_scale=sc.cuda(), bn_shift=sh.cuda(), relu=True)
        assert torch.equal(y.cpu(), want_bn), ("fused BN + ReLU", xin.is_contiguous())
        y = dcn_fused_inference(xin, om, wc, bc, stride, pad, dil, dg)
        assert torch.equal(y.cpu(), want_plain), ("fused", xin.is_contiguous())


def _expect(got, want, G, what):
    for name, a, ref, g0 in zip(NAMES, got, want, G):
        if a is None:
            continue
        exp = ref if g0 is None else _exact32(g0.double() + ref.double())
        assert torch.equal(a.cpu(), exp), (name,) + tuple(what)


def check_backward(x, off, m, w, b, go, stride, pad, dil, dg):
    """All five gradients of every fp32 backward path == the oracle's (G + the oracle's for the raw ABI)."""
    from centernet_b200._lib import C
    from centernet_b200.dcn_v2_func import DCNv2Function
    B, Ci, H, W = x.shape
    Co, _, kh, kw = w.shape
    want = [_exact32(t) for t in oracle_grads(x, off, m, w, b, go, stride, pad, dil, dg)]
    xc, offc, mc, wc, bc, goc = [t.cuda() for t in (x, off, m, w, b, go)]
    xcl = xc.contiguous(memory_format=torch.channels_last)
    cl_ok = (Ci // dg) % 32 == 0 and Co <= 256
    f = DCNv2Function(stride, pad, dil, dg)
    subsets = (NAMES, ("weight", "bias"), ("input", "offset", "mask"))
    try:
        for det in (False, True):
            _det(det)
            for xin in (xc, xcl):
                got = autograd(f, xin, offc, mc, wc, bc, goc)
                _expect(got, want, [None] * 5, ("autograd", det, xin is xcl))
            got = autograd(f, xc, offc, mc, wc, None, goc)
            assert got[4] is None
            _expect(got, want, [None] * 5, ("autograd, bias=None", det))
            for which in subsets:
                got, G = raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "tc", which)
                _expect(got, want, G, ("ABI, tensor cores", det, which))
                if cl_ok:
                    got, G = raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "tc", which, x_cl=True)
                    _expect(got, want, G, ("ABI _ex, channels_last", det, which))
                else:        # channels-last tensors need whole 32-channel blocks and the tensor-core dW (Cout <= 256)
                    with pytest.raises(NotImplementedError):
                        raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "tc", which, x_cl=True)
            _det(False)
            for which in subsets:                 # the CUDA-core kernels (default mode only)
                got, G = raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "fp32", which)
                _expect(got, want, G, ("ABI, CUDA cores", which))
        _det(True)
        with pytest.raises(NotImplementedError):   # deterministic mode needs the tensor-core backward
            raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "fp32")
    finally:
        _det(False)
    assert C.dcnv2_get_deterministic() == 0


CASES = [
    # B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil
    (2, 64, 20, 24, 64, 1, 3, 3, 1, 1, 1),      # dla_34 64 -> 64
    (2, 80, 17, 19, 40, 2, 3, 3, 1, 1, 1),      # 40 channels a group: ragged 32-channel blocks, two groups
    (2, 12, 9, 11, 5, 2, 3, 3, 1, 1, 1),        # 6 channels a group
    (1, 6, 10, 14, 7, 1, 3, 3, 2, 1, 1),        # Cin 6, stride 2
    (2, 64, 21, 23, 72, 2, 3, 3, 2, 1, 1),      # stride 2, two groups of 32
    (1, 32, 22, 20, 32, 1, 3, 3, 3, 1, 1),      # stride 3
    (1, 32, 18, 18, 32, 1, 3, 3, 1, 2, 2),      # dilation 2, pad 2
    (1, 32, 17, 19, 24, 1, 3, 3, 1, 1, 3),      # dilation 3, pad 1
    (2, 32, 14, 15, 16, 1, 3, 3, 1, 0, 1),      # pad 0
    (1, 32, 13, 12, 16, 1, 3, 3, 1, 2, 1),      # pad 2, dilation 1
    (2, 64, 16, 16, 48, 1, 1, 1, 1, 0, 1),      # 1x1
    (2, 64, 16, 20, 64, 1, 1, 3, 1, 1, 1),      # 1x3
    (1, 32, 15, 13, 40, 1, 3, 1, 1, 1, 1),      # 3x1
    (2, 32, 12, 12, 24, 1, 2, 2, 1, 0, 1),      # 2x2, pad 0
    (2, 32, 17, 16, 32, 1, 3, 2, 2, 1, 1),      # 3x2, stride 2
    (2, 32, 24, 9, 32, 1, 3, 3, 1, 1, 1),       # Wo 9 < 12: 16 x 8 pixel tiles
    (1, 32, 10, 12, 32, 1, 3, 3, 1, 1, 1),      # Wo 12: 8 x 16 tiles
    (3, 32, 7, 9, 32, 1, 3, 3, 1, 1, 1),        # Ho * Wo = 63 < 128: one partial tile; B = 3
    (1, 256, 8, 8, 272, 1, 3, 3, 1, 1, 1),      # small map, Cin 256: split-K; Cout 272: three tiles, fp32 dW
    (2, 32, 12, 12, 1, 1, 3, 3, 1, 1, 1),       # Cout 1
    (1, 64, 14, 14, 65, 1, 3, 3, 1, 1, 1),      # Cout 65: one 128-wide tile with a tail
]


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil", CASES)
def test_exact_grid_forward(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    x, off, m, w, b, _ = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil)
    check_forward(x, off, m, w, b, stride, pad, dil, dg)


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil", CASES)
def test_exact_grid_backward(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    x, off, m, w, b, go = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil)
    check_backward(x, off, m, w, b, go, stride, pad, dil, dg)


BOUNDARY = [
    # B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil
    (2, 64, 12, 12, 8, 1, 3, 3, 1, 1, 1),
    (1, 80, 11, 13, 8, 2, 3, 3, 1, 1, 1),       # ragged blocks, two groups
    (2, 32, 10, 13, 6, 1, 1, 3, 1, 1, 1),       # 1x3
    (1, 32, 24, 24, 4, 1, 3, 3, 2, 2, 2),       # stride 2, dilation 2
    (1, 12, 13, 11, 3, 1, 2, 2, 1, 0, 1),       # 2x2, Cin 12
]


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil", BOUNDARY)
def test_sampling_boundaries(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    x, off, m, w, b, go = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil, seed=3)
    off = boundary_offsets(off, H, W, kh, kw, stride, pad, dil, dg)
    check_forward(x, off, m, w, b, stride, pad, dil, dg)
    check_backward(x, off, m, w, b, go, stride, pad, dil, dg)


ANISO = [
    # B, Ci, H, W, Co, dg, kh, kw, (sh, sw), (ph, pw), (dh, dw)
    (2, 16, 13, 17, 12, 1, 3, 3, (1, 2), (1, 0), (2, 1)),
    (1, 24, 15, 11, 8, 2, 2, 3, (2, 1), (0, 2), (1, 2)),
]


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil", ANISO)
def test_anisotropic_abi(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    """Anisotropic stride/pad/dilation: the C ABI runs the CUDA-core kernels, a workspace or not."""
    from centernet_b200._lib import C
    x, off, m, w, b, go = grid_inputs(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil, seed=5)
    want = _exact32(dcn_v2_forward(x, off, m, w, b, stride, pad, dil, dg))
    xc, offc, mc, wc, bc, goc = [t.cuda() for t in (x, off, m, w, b, go)]
    assert torch.equal(raw_forward(xc, offc, mc, wc, bc, stride, pad, dil, dg, False).cpu(), want)
    grads = [_exact32(t) for t in oracle_grads(x, off, m, w, b, go, stride, pad, dil, dg)]
    for which in (NAMES, ("weight", "bias"), ("input", "offset", "mask")):
        got, G = raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "fp32", which)
        _expect(got, grads, G, ("anisotropic", which))
    try:
        _det(True)
        with pytest.raises(NotImplementedError):
            raw_backward(xc, offc, mc, wc, goc, stride, pad, dil, dg, "fp32")
    finally:
        _det(False)
    assert C.dcnv2_get_deterministic() == 0


# ---------------------------------------------------------------- 3. random data against derived bounds
PREC = [
    # B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil
    (2, 64, 32, 32, 64, 1, 3, 3, 1, 1, 1),      # dla_34 64 -> 64
    (2, 128, 24, 24, 128, 1, 3, 3, 1, 1, 1),    # dla_34 128 -> 128
    (2, 12, 9, 11, 5, 2, 3, 3, 1, 1, 1),
    (2, 64, 16, 20, 64, 1, 1, 3, 1, 1, 1),
    (2, 32, 21, 23, 40, 1, 3, 3, 2, 1, 1),
]


def _tf32(t):
    """Truncation to TF32 (the low 13 mantissa bits dropped), as tf32_hi in the kernels."""
    return (t.float().view(torch.int32) & -8192).view(torch.float32)


@pytest.mark.parametrize("B,Ci,H,W,Co,dg,kh,kw,stride,pad,dil", PREC)
def test_random_within_derived_bound(B, Ci, H, W, Co, dg, kh, kw, stride, pad, dil):
    """Random x, W, dY; offsets within +-3.5 px on a 2^-16 grid (every sampling position is exact in fp32); S = the
    oracle at |x|, |W| (and |dY|), which bounds the sum of magnitudes behind each output and gradient element.

    Products.  3xTF32 splits v = hi + lo, hi = v with its low 13 mantissa bits cleared, so |lo| < 2^-10 |v|; the tensor
    core reads lo as TF32 as well, dropping its lowest 2 bits (< 2^-21 |v|).  hi.hi + hi.lo + lo.hi then misses
    lo.lo (< 2^-20 |xw|) and the two dropped lo bits (< 2 * 2^-21 |xw|): e_prod <= 2^-19.  The column value (four
    corner weights times values, mask folded in) carries at most 8 fp32 roundings of its magnitude: + 8 * 2^-24.
    Sums.  Each of the n terms of a contraction adds at most one rounding of the running magnitude (<= S): n * 2^-24.
      output:  n = Cin * taps (plus the split-K partials and the bias, 8 more)        (e_prod + (n + 8) 2^-24) S
      dW:      n = B * Ho * Wo pixels                                                 same form, S_w
      dX:      dcol = sum over Cout (3xTF32), then at most taps * 9 * 9 scattered contributions per element
               (|offset| <= 3.5): n = Cout + taps * 81 + 8                             S_x
      dMask:   n = Cout + Cin / dg + 8 (the channel sum of dcol * value)              S_m
      dOffset: as dMask, against sum_c |dcol| m * 2 max|x| (the corner difference |cw| <= 2 max|x|)
      dBias:   n = B * Ho * Wo fp32 adds of dY                                        sum |dY|
    The bound has teeth: a 1xTF32 forward (the oracle at TF32-truncated x and W, dropping the correction terms) and
    a 1xTF32 column gradient (at TF32-truncated W and dY) both exceed it on the same data."""
    from centernet_b200.dcn_v2_func import DCNv2Function
    g = torch.Generator().manual_seed(21)
    Ho, Wo = out_hw(H, W, kh, kw, stride, pad, dil)
    kt = kh * kw
    x = torch.randn(B, Ci, H, W, generator=g)
    off = torch.round((torch.randn(B, 2 * kt * dg, Ho, Wo, generator=g) * 2).clamp(-3.5, 3.5) * 2.0 ** 16) / 2.0 ** 16
    m = torch.sigmoid(torch.randn(B, kt * dg, Ho, Wo, generator=g))
    w = torch.randn(Co, Ci, kh, kw, generator=g) / (Ci * kt) ** 0.5
    b = torch.randn(Co, generator=g)
    go = torch.randn(B, Co, Ho, Wo, generator=g)
    e_prod = 2.0 ** -19 + 8 * 2.0 ** -24
    u = 2.0 ** -24
    npix = B * Ho * Wo

    y64 = dcn_v2_forward(x, off, m, w, b, stride, pad, dil, dg)
    S = dcn_v2_forward(x.abs(), off, m, w.abs(), None, stride, pad, dil, dg)
    bound = (e_prod + (Ci * kt + 8) * u) * S + u * y64.abs()
    f = DCNv2Function(stride, pad, dil, dg)
    xc, offc, mc, wc, bc, goc = [t.cuda() for t in (x, off, m, w, b, go)]
    for xin in (xc, xc.contiguous(memory_format=torch.channels_last)):
        err = (f(xin, offc, mc, wc, bc).double().cpu() - y64).abs()
        assert (err <= bound).all(), ("output", (err / bound).max().item())
    y1 = dcn_v2_forward(_tf32(x), off, m, _tf32(w), b, stride, pad, dil, dg)
    assert ((y1 - y64).abs() > bound).any(), "the forward bound does not see 1xTF32"

    ref = oracle_grads(x, off, m, w, b, go, stride, pad, dil, dg)
    Sg = oracle_grads(x.abs(), off, m, w.abs(), None, go.abs(), stride, pad, dil, dg)
    # sum over the channels of each group of |dcol| = |W|^T |dY|, times the mask: the scale of dOffset's sum
    dcol = torch.einsum("ock,bop->bckp", w.abs().double().reshape(Co, Ci, kt), go.abs().double().reshape(B, Co, -1))
    dsum = dcol.reshape(B, dg, Ci // dg, kt, Ho, Wo).sum(2).reshape(B, dg * kt, Ho, Wo) * m.double()
    s_off = (2 * x.abs().max().item()) * dsum.repeat_interleave(2, dim=1)
    bounds = {"input": (e_prod + (Co + kt * 81 + 8) * u) * Sg[0],
              "offset": (e_prod + (Co + Ci // dg + 8) * u) * s_off,
              "mask": (e_prod + (Co + Ci // dg + 8) * u) * Sg[2],
              "weight": (e_prod + (npix + 8) * u) * Sg[3],
              "bias": (npix * u) * go.abs().double().sum((0, 2, 3))}
    for det in (False, True):
        try:
            _det(det)
            got = autograd(f, xc, offc, mc, wc, bc, goc)
        finally:
            _det(False)
        for name, a, r in zip(NAMES, got, ref):
            err = (a.double().cpu() - r).abs()
            assert (err <= bounds[name]).all(), (name, det, (err - bounds[name]).max().item())
    e = oracle_grads(x, off, m, _tf32(w), b, _tf32(go), stride, pad, dil, dg)
    assert ((e[0] - ref[0]).abs() > bounds["input"]).any(), "the dX bound does not see a 1xTF32 column gradient"

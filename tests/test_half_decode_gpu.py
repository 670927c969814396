"""bf16 / fp16 heads decoded in place: every call returns, bit for bit, what it returns for the .float() upcast of
the same tensors (the fp32 path is pinned against the reference in test_decode_gpu.py / test_logits_gpu.py)."""
import numpy as np
import pytest
import torch

from helpers import assert_dets_equal

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]


def _up(t):
    return None if t is None else t.float()


def _check(heat, wh, reg=None, K=100, cat=False, logits=False):
    """new(x) == today(x.float()) for ctdet_decode (or _from_logits); inputs untouched."""
    from centernet_b200 import decode as D
    fn = D.ctdet_decode_from_logits if logits else D.ctdet_decode
    keep = [None if t is None else t.clone() for t in (heat, wh, reg)]
    got = fn(heat, wh, reg=reg, cat_spec_wh=cat, K=K)
    want = fn(_up(heat), _up(wh), reg=_up(reg), cat_spec_wh=cat, K=K)
    for t, k in zip((heat, wh, reg), keep):
        assert t is None or torch.equal(t, k), "input modified"
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert torch.equal(got, want)
    return got


def _bench(B, dt, seed=317, C=80, H=128, W=128, logits=False):
    """bench.py's synthetic heads (heat = sigmoid(randn - 2.19), wh = rand * 32, reg = rand), rounded to dt."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, C, H, W, device="cuda", generator=g) - 2.19
    heat = x if logits else torch.sigmoid(x)
    wh = torch.rand(B, 2, H, W, device="cuda", generator=g) * 32
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g)
    return heat.to(dt), wh.to(dt), reg.to(dt)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("logits", [False, True], ids=["heat", "logits"])
@pytest.mark.parametrize("B", [1, 2, 8, 64, 150])
def test_batch_sizes(B, logits, dt):
    heat, wh, reg = _bench(B, dt, seed=317 + B, logits=logits)
    _check(heat, wh, reg, logits=logits)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("logits", [False, True], ids=["heat", "logits"])
@pytest.mark.parametrize("K", [1, 100, 256, 1000])
def test_k(K, logits, dt):
    heat, wh, reg = _bench(3, dt, seed=K, logits=logits)
    _check(heat, wh, reg, K=K, logits=logits)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("logits", [False, True], ids=["heat", "logits"])
def test_cat_spec_wh_and_no_reg(logits, dt):
    B, C = 2, 80
    heat, _, reg = _bench(B, dt, seed=5, logits=logits)
    g = torch.Generator(device="cuda").manual_seed(6)
    wh = (torch.rand(B, 2 * C, 128, 128, device="cuda", generator=g) * 16).to(dt)
    _check(heat, wh, reg, cat=True, logits=logits)
    _check(heat, wh[:, :2].contiguous(), None, logits=logits)
    _check(heat, wh, None, K=7, cat=True, logits=logits)


def _blobs(B, C, H, W, g):
    """Gaussian blobs (plateaus where they saturate and overlap, < K peaks in most classes) on a low noise floor."""
    yy = torch.arange(H, device="cuda").view(1, H, 1).float()
    xx = torch.arange(W, device="cuda").view(1, 1, W).float()
    heat = 0.01 * torch.rand(B, C, H, W, device="cuda", generator=g)
    for b in range(B):
        n = 40
        cls = torch.randint(0, C, (n,), device="cuda", generator=g)
        cy = torch.randint(0, H, (n,), device="cuda", generator=g).float().view(n, 1, 1)
        cx = torch.randint(0, W, (n,), device="cuda", generator=g).float().view(n, 1, 1)
        r = torch.randint(1, 14, (n,), device="cuda", generator=g).float().view(n, 1, 1)
        blob = torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * (r / 3) ** 2)).clamp(max=0.9 + 0.1 * (r > 8))
        for i in range(n):
            heat[b, cls[i]] = torch.maximum(heat[b, cls[i]], blob[i])
    return heat


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_distributions(dt):
    B, C, H, W = 4, 80, 128, 128
    g = torch.Generator(device="cuda").manual_seed(41)
    wh = (torch.rand(B, 2, H, W, device="cuda", generator=g) * 32).to(dt)
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g).to(dt)
    _check(_blobs(B, C, H, W, g).to(dt), wh, reg)
    quant = torch.randint(0, 9, (B, C, H, W), device="cuda", generator=g).float() / 8      # plateaus of ties
    _check(quant.to(dt), wh, reg)
    _check(quant.to(dt), wh, reg, K=256)
    _check((quant * 12 - 6).to(dt), wh, reg, logits=True)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_degenerate_maps(dt):
    B, C, H, W = 2, 80, 128, 128
    g = torch.Generator(device="cuda").manual_seed(43)
    wh = (torch.rand(B, 2, H, W, device="cuda", generator=g) * 32).to(dt)
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g).to(dt)
    zero = torch.zeros(B, C, H, W, device="cuda", dtype=dt)
    _check(zero, wh, reg)
    _check(-torch.rand(B, C, H, W, device="cuda", generator=g).to(dt) - 0.01, wh, reg)     # all negative
    few = torch.zeros(B, C, H, W, device="cuda")
    few[0, 3, 10, 20] = 0.7
    few[0, 7, 100, 5] = 0.2
    few[1, 79, 127, 127] = 0.9
    few[1, 0, 0, 0] = -0.5
    _check(few.to(dt), wh, reg)                                                              # fewer than K peaks
    _check(torch.ones(B, C, H, W, device="cuda", dtype=dt), wh, reg)                        # saturated
    sat = torch.rand(B, C, H, W, device="cuda", generator=g)
    sat[sat > 0.5] = 1.0
    _check(sat.to(dt), wh, reg)


def test_fp16_subnormals_and_infinities():
    B, C, H, W = 2, 80, 128, 128
    g = torch.Generator(device="cuda").manual_seed(47)
    wh = (torch.rand(B, 2, H, W, device="cuda", generator=g) * 32).half()
    reg = torch.rand(B, 2, H, W, device="cuda", generator=g).half()
    sub = (torch.rand(B, C, H, W, device="cuda", generator=g) * 6e-5).half()                # mostly fp16 subnormals
    assert bool(((sub > 0) & (sub < 6.1e-5)).any())
    _check(sub, wh, reg)
    _check(sub, wh, reg, K=1000)
    inf = torch.sigmoid(torch.randn(B, C, H, W, device="cuda", generator=g) - 2.19).half()
    inf[0, 5, 64, 64] = float("inf")
    inf[0, 5, 64, 65] = float("inf")
    inf[1, 9, 0, 127] = float("inf")
    inf[1, 2, 30:40, 30:40] = float("-inf")
    _check(inf, wh, reg)
    lg = (torch.randn(B, C, H, W, device="cuda", generator=g) * 2 - 2).half()
    lg[0, 1, 3, 4] = float("inf")
    lg[1, 1, 50:60, 50:60] = float("-inf")
    _check(lg, wh, reg, logits=True)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_extreme_logits(dt):
    B, C, H, W = 2, 80, 128, 128
    g = torch.Generator(device="cuda").manual_seed(53)
    wh = (torch.rand(B, 2, H, W, device="cuda", generator=g) * 32).to(dt)
    x = torch.randn(B, C, H, W, device="cuda", generator=g) * 3 - 2
    x[0, :4] = 100.0
    x[1, 10:12] = -100.0
    x[0, 20, 5, 5] = float("inf")
    x[1, 21, 6, 6] = float("-inf")
    _check(x.to(dt), wh, None, logits=True)
    _check(torch.full((B, C, H, W), -100.0, device="cuda").to(dt), wh, None, logits=True)
    _check(torch.full((B, C, H, W), 100.0, device="cuda").to(dt), wh, None, logits=True)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("logits", [False, True], ids=["heat", "logits"])
def test_overflow_rescan_ramp(logits, dt):
    """Every plane brighter than the ones before: stale threshold, key-buffer overflow, exact rebuild from the
    16-bit map (test_decode_gpu.py::test_hot_kernel_overflow_rescan on half heads)."""
    B, C, H, W = 4, 80, 128, 128
    g = torch.Generator(device="cuda").manual_seed(99 + B)
    base = torch.rand(B, C, H, W, device="cuda", generator=g)
    if logits:
        x = base * 0.05 + torch.linspace(-6, 4, C, device="cuda").view(1, C, 1, 1)
    else:
        x = base * 0.01 + torch.linspace(0.01, 0.99, C, device="cuda").view(1, C, 1, 1)
    wh = (torch.rand(B, 2, H, W, device="cuda", generator=g) * 8).to(dt)
    _check(x.to(dt).contiguous(), wh, None, logits=logits)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("logits", [False, True], ids=["heat", "logits"])
@pytest.mark.parametrize("HW", [(96, 320), (30, 30), (200, 152)])
def test_other_geometries(HW, logits, dt):
    H, W = HW
    heat, wh, reg = _bench(3, dt, seed=H * W, H=H, W=W, logits=logits)
    _check(heat, wh, reg, K=min(100, H * W), logits=logits)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("logits", [False, True], ids=["heat", "logits"])
def test_misaligned_view(logits, dt):
    B, C, H, W = 2, 80, 128, 128
    heat, wh, reg = _bench(B, dt, seed=61, logits=logits)
    buf = torch.empty(heat.numel() + 1, device="cuda", dtype=dt)
    buf[1:] = heat.reshape(-1)
    mis = buf[1:].view(B, C, H, W)
    assert mis.data_ptr() % 16 != 0 and mis.storage_offset() == 1
    got = _check(mis, wh, reg, logits=logits)
    from centernet_b200 import decode as D
    fn = D.ctdet_decode_from_logits if logits else D.ctdet_decode
    assert torch.equal(got, fn(heat, wh, reg=reg))                      # same dets as the aligned, in-place read


@pytest.mark.parametrize("logits", [False, True], ids=["heat", "logits"])
def test_mixed_dtypes(logits):
    B = 3
    heat, wh, reg = _bench(B, torch.float32, seed=67, logits=logits)
    combos = [(torch.bfloat16, torch.float32, torch.float16), (torch.float16, torch.bfloat16, torch.float32),
              (torch.float32, torch.float16, torch.bfloat16), (torch.bfloat16, torch.bfloat16, None),
              (torch.float32, torch.float32, torch.float16), (torch.float16, torch.float16, torch.bfloat16)]
    for hd, wd, rd in combos:
        _check(heat.to(hd), wh.to(wd), None if rd is None else reg.to(rd), logits=logits)
    # non-hot geometry with mixed heads: the widened map + 16-bit gathers
    h2, w2, r2 = _bench(2, torch.float32, seed=71, H=96, W=320, logits=logits)
    _check(h2.half(), w2.bfloat16(), r2, logits=logits)
    # float64 / integer heads keep the upcast
    _check(heat.to(torch.float64), wh.half(), reg.bfloat16(), logits=logits)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_flip_merge_modes(dt):
    from centernet_b200 import decode as D
    g = torch.Generator(device="cuda").manual_seed(73)
    flip_idx = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
    hm = (torch.randn(4, 6, 12, 20, device="cuda", generator=g) * 3).to(dt)
    hps = torch.randn(4, 34, 12, 20, device="cuda", generator=g).to(dt)
    hm_hp = (torch.randn(4, 17, 12, 20, device="cuda", generator=g) * 2).to(dt)
    for x, kw in ((hm, dict(sigmoid=True)), (hm, {}), (hps, {}), (hps, dict(flip_idx=flip_idx, offsets=True)),
                  (hm_hp, dict(sigmoid=True, flip_idx=flip_idx))):
        keep = x.clone()
        got = D.flip_merge(x, **kw)
        assert torch.equal(x, keep)
        assert got.dtype == torch.float32
        assert torch.equal(got, D.flip_merge(x.float(), **kw))


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_flip_wrappers(dt):
    from centernet_b200 import decode as D
    g = torch.Generator(device="cuda").manual_seed(79)
    n, C, H, W = 2, 80, 128, 128
    hm = (torch.randn(2 * n, C, H, W, device="cuda", generator=g) - 2.19).to(dt)
    wh = (torch.rand(2 * n, 2, H, W, device="cuda", generator=g) * 32).to(dt)
    reg = torch.rand(2 * n, 2, H, W, device="cuda", generator=g).to(dt)
    assert torch.equal(D.ctdet_decode_flip_from_logits(hm, wh, reg=reg),
                       D.ctdet_decode_flip_from_logits(hm.float(), wh.float(), reg=reg.float()))
    flip_idx = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
    hmp = (torch.randn(2 * n, 1, 64, 64, device="cuda", generator=g) - 2).to(dt)
    whp = (torch.rand(2 * n, 2, 64, 64, device="cuda", generator=g) * 16).to(dt)
    hps = torch.randn(2 * n, 34, 64, 64, device="cuda", generator=g).to(dt)
    regp = torch.rand(2 * n, 2, 64, 64, device="cuda", generator=g).to(dt)
    hm_hp = (torch.randn(2 * n, 17, 64, 64, device="cuda", generator=g) - 2).to(dt)
    hp_off = torch.rand(2 * n, 2, 64, 64, device="cuda", generator=g).to(dt)
    args = dict(reg=regp, hm_hp=hm_hp, hp_offset=hp_off, flip_idx=flip_idx, K=20)
    got = D.multi_pose_decode_flip_from_logits(hmp, whp, hps, **args)
    want = D.multi_pose_decode_flip_from_logits(hmp.float(), whp.float(), hps.float(),
                                                **{k: (v.float() if torch.is_tensor(v) else v) for k, v in args.items()})
    assert torch.equal(got, want)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_from_host_stages_half(dt):
    from centernet_b200 import decode as D
    B = 20
    heat, wh, reg = [t.cpu().pin_memory() for t in _bench(B, dt, seed=83)]
    got = D.ctdet_decode_from_host(heat, wh, reg=reg, K=100, chunk=8)
    ctx = next(iter(D._HOST_TLS.ctx.values()))
    assert ctx["heat"][0].dtype == dt and ctx["wh"][0].dtype == dt and ctx["reg"][0].dtype == dt
    want = D.ctdet_decode_from_host(heat.float(), wh.float(), reg=reg.float(), K=100, chunk=8)
    ctx = next(iter(D._HOST_TLS.ctx.values()))
    assert ctx["heat"][0].dtype == torch.float32
    assert not got.is_cuda and torch.equal(got, want)
    assert torch.equal(got, D.ctdet_decode(heat.cuda(), wh.cuda(), reg=reg.cuda()).cpu())
    # mixed host dtypes, no reg
    got2 = D.ctdet_decode_from_host(heat, wh.float(), K=50, chunk=8)
    assert torch.equal(got2, D.ctdet_decode(heat.float().cuda(), wh.float().cuda(), K=50).cpu())


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_non_default_stream(dt):
    from centernet_b200 import decode as D
    heat, wh, reg = _bench(8, dt, seed=89)
    lg, _, _ = _bench(8, dt, seed=90, logits=True)
    want = D.ctdet_decode(heat.float(), wh.float(), reg=reg.float())
    want_l = D.ctdet_decode_from_logits(lg.float(), wh.float(), reg=reg.float())
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = D.ctdet_decode(heat, wh, reg=reg)
        got_l = D.ctdet_decode_from_logits(lg, wh, reg=reg)
    s.synchronize()
    assert torch.equal(got, want) and torch.equal(got_l, want_l)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_batch_shard_invariance(dt):
    from centernet_b200 import decode as D
    heat, wh, reg = _bench(64, dt, seed=97)
    full = D.ctdet_decode(heat, wh, reg=reg)
    for shard in (1, 8, 13):
        parts = [D.ctdet_decode(heat[s:s + shard], wh[s:s + shard], reg=reg[s:s + shard]) for s in range(0, 64, shard)]
        assert torch.equal(torch.cat(parts), full)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_matches_reference_ops_on_half_cuda_tensors(dt):
    """The reference op sequence run on the half CUDA tensors (it promotes to fp32) equals our dets up to the order
    of tied scores, which ties at the K-th score make routine here."""
    from centernet_b200 import decode as D
    from oracle import torch_port as TP
    heat, wh, reg = _bench(4, dt, seed=317)
    want = TP.ctdet_decode(heat, wh, reg=reg, K=100)
    got = D.ctdet_decode(heat, wh, reg=reg, K=100)
    assert want.dtype == torch.float32
    assert_dets_equal(want.cpu().numpy(), got.cpu().numpy(), what=str(dt))
    s = got[:, :, 4].cpu().numpy()
    # the defined order inside a tie: flat index (class * H * W + y * W + x) ascending
    for b in range(s.shape[0]):
        for k in range(s.shape[1] - 1):
            if s[b, k] == s[b, k + 1]:
                d0, d1 = got[b, k].cpu().numpy(), got[b, k + 1].cpu().numpy()
                assert d0[5] <= d1[5]
    assert np.isfinite(s).all()

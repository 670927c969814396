"""Secondary measurements of bench.py (rank 0, N=1): every other kernel of the hot path on the BASELINE
config geometries, each with its own roofline sub-dict, plus the "reference on the GPU" bars of BASELINE.md
section 2 (the reference's ATen-op decode on CUDA tensors; the reference's DCNv2 kernels, oracle/_ref).
All times are CUDA events on the launching stream after warm-up; inputs are synthetic (seed 317).
Algorithmic bytes / FLOPs per unit follow SURVEY.md section 8(d)."""
import json
import os

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
H = W = 128


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        j = json.load(open(p))
        return float(j["hbm_gbs"]), float(j["bf16_tflops"]), "measured"
    except Exception:
        return 3350.0, 989.0, "fallback (H100 SXM data sheet: 3.35 TB/s HBM3, 989 TFLOP/s dense BF16)"


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _hbm(ms, alg_bytes, peak, src, **extra):
    ach = alg_bytes / (ms * 1e-3) / 1e9
    d = {"ms": round(ms, 5), "roofline": {"bound": "hbm", "achieved": round(ach, 1), "peak": peak, "unit": "GB/s",
                                          "frac": round(ach / peak, 4), "alg_bytes": int(alg_bytes), "peak_source": src}}
    d.update(extra)
    return d


def _tensor(ms, flops, peak_tf, src, **extra):
    # 3xTF32 emulation of the reference's fp32 SGEMM: three tf32 MMAs per product, tf32 peak = bf16 peak / 2,
    # so the ceiling for fp32-accurate useful FLOPs is bf16_peak / 6
    ceil_tf = peak_tf / 6.0
    ach = flops / (ms * 1e-3) / 1e12
    d = {"ms": round(ms, 5), "roofline": {"bound": "tensor", "achieved": round(ach, 2), "peak": round(ceil_tf, 1),
                                          "unit": "TFLOP/s", "frac": round(ach / ceil_tf, 4), "flops": int(flops),
                                          "peak_source": src + " bf16_tflops / 6 (3xTF32 at half the bf16 rate)"}}
    d.update(extra)
    return d


def blob_heat(B, C, dev, g):
    """Second input set of SURVEY 8(d): class-sparse Gaussian blobs (the library's own splat) x 0.9 + 0.01 noise:
    plateaus, < K peaks per class."""
    from centernet_b200 import losses as L
    M = 40
    cls = torch.randint(0, C, (B, M), device=dev, generator=g)
    cx = torch.randint(0, W, (B, M), device=dev, generator=g)
    cy = torch.randint(0, H, (B, M), device=dev, generator=g)
    rad = torch.randint(1, 14, (B, M), device=dev, generator=g)
    val = torch.ones(B, M, dtype=torch.uint8, device=dev)
    hm = L.splat_gaussian(cls, cx, cy, rad, val, C, H, W)
    return hm * 0.9 + 0.01 * torch.rand(B, C, H, W, device=dev, generator=g)


def run(dev, batches, K=100, steps=20):
    from centernet_b200 import decode as D, losses as L
    from centernet_b200.dcn_v2_func import DCNv2Function
    hbm, tf, src = _peaks()
    g = torch.Generator(device=dev).manual_seed(317)
    C = 80
    out = {}
    img_bytes = C * H * W * 4 + K * 16 + K * 24

    def guarded(name, fn):
        try:
            out[name] = fn()
        except Exception as e:   # a secondary number never takes the headline down
            out[name] = {"failed": str(e)[:160]}
        torch.cuda.synchronize()

    # ---- ctdet decode: the plateau / blob input set, and the small batches the reference's test.py uses
    def ctdet_blobs():
        bb = [(blob_heat(64, C, dev, g), batches[i][1], batches[i][2]) for i in range(3)]
        i = [0]

        def f():
            h, w_, r = bb[i[0] % 3]; i[0] += 1
            D.ctdet_decode(h, w_, reg=r, K=K)
        ms = timeit(f, steps)
        return _hbm(ms, 64 * img_bytes, hbm, src, value=64 / ms * 1e3, unit="images/s",
                    config="64 img x 80x128x128 Gaussian-blob/plateau heat (SURVEY 8d second set), K=100")
    guarded("ctdet_decode_blobs", ctdet_blobs)

    for b in (1, 2, 8):
        def small(b=b):
            h, w_, r = [t[:b].contiguous() for t in batches[0]]
            ms = timeit(lambda: D.ctdet_decode(h, w_, reg=r, K=K), 50, 5)
            return _hbm(ms, b * img_bytes, hbm, src, value=b / ms * 1e3, unit="images/s", latency_us=round(ms * 1e3, 2),
                        config="B=%d x 80x128x128, K=100 (L2-warm: the same batch every call)" % b)
        guarded("ctdet_decode_b%d" % b, small)

    # ---- multi_pose decode (config 3: heads hm 1, hps 34, hm_hp 17; 64 -> 8 per GPU)
    for b in (8, 64):
        def mp(b=b):
            h1 = torch.sigmoid(torch.randn(b, 1, H, W, device=dev, generator=g) - 2.19)
            wh = torch.rand(b, 2, H, W, device=dev, generator=g) * 32
            kps = torch.randn(b, 34, H, W, device=dev, generator=g) * 6
            reg = torch.rand(b, 2, H, W, device=dev, generator=g)
            hm_hp = torch.sigmoid(torch.randn(b, 17, H, W, device=dev, generator=g) - 1.0)
            hpo = torch.rand(b, 2, H, W, device=dev, generator=g)
            ms = timeit(lambda: D.multi_pose_decode(h1, wh, kps, reg=reg, hm_hp=hm_hp, hp_offset=hpo, K=K), steps)
            return _hbm(ms, b * 1224448, hbm, src, value=b / ms * 1e3, unit="images/s",
                        config="multi_pose_decode B=%d (1+17 maps of 128x128, K=100)" % b)
        guarded("multi_pose_decode_b%d" % b, mp)

    # ---- exct decode (config 5): K=40 (signature default) and K=100 (what detectors/exdet.py passes)
    def exct(k, b, aggr, iters):
        maps = [torch.sigmoid(torch.randn(b, C, H, W, device=dev, generator=g) - 2.19) for _ in range(5)]
        regs = [torch.rand(b, 2, H, W, device=dev, generator=g) for _ in range(4)]
        ms = timeit(lambda: D.exct_decode(*maps, *regs, K=k, num_dets=1000, aggr_weight=aggr), iters, 1)
        alg = b * (5 * C * H * W * 4 + 4 * k * 8 + 1000 * 14 * 4)
        return _hbm(ms, alg, hbm, src, value=b / ms * 1e3, unit="images/s", tuples_per_image=k ** 4,
                    config="exct_decode B=%d 5x80x128x128, K=%d, aggr_weight=%g, num_dets=1000" % (b, k, aggr))
    guarded("exct_decode_k40", lambda: exct(40, 8, 0.0, 5))
    guarded("exct_decode_k40_aggr", lambda: exct(40, 8, 0.1, 5))
    guarded("exct_decode_k100", lambda: exct(100, 2, 0.0, 2))

    # ---- edge aggregation ("corner_pool" of BASELINE.json), B=32
    heat = batches[0][0][:32].contiguous()
    n = heat.numel()
    guarded("h_aggregate", lambda: _hbm(timeit(lambda: D._h_aggregate(heat, 0.1), steps), 2 * n * 4, hbm, src,
                                        config="_h_aggregate 32x80x128x128"))
    guarded("v_aggregate", lambda: _hbm(timeit(lambda: D._v_aggregate(heat, 0.1), steps), 2 * n * 4, hbm, src,
                                        config="_v_aggregate 32x80x128x128"))

    # ---- focal loss + target splat, forward + gradient, B=32, 128 objects per image
    def focal():
        B, M = 32, 128
        pred = torch.clamp(batches[1][0][:B], 1e-4, 1 - 1e-4).contiguous().requires_grad_(True)
        cls = torch.randint(0, C, (B, M), device=dev, generator=g)
        cx = torch.randint(0, W, (B, M), device=dev, generator=g)
        cy = torch.randint(0, H, (B, M), device=dev, generator=g)
        rad = torch.randint(0, 12, (B, M), device=dev, generator=g)
        val = torch.ones(B, M, dtype=torch.uint8, device=dev)
        crit = L.FocalSplatLoss()
        ms = timeit(lambda: crit(pred, cls, cx, cy, rad, val), steps)
        r = _hbm(ms, 2 * pred.numel() * 4, hbm, src, value=B / ms * 1e3, unit="images/s",
                 config="FocalSplatLoss fwd+grad 32x80x128x128, 128 objects/image (target never materialised)")
        gt = L.splat_gaussian(cls, cx, cy, rad, val, C, H, W)
        ms2 = timeit(lambda: L._neg_loss(pred, gt), steps)
        r["dense_target_variant"] = _hbm(ms2, 3 * pred.numel() * 4, hbm, src, config="_neg_loss fwd+grad with a dense gt map")
        ms3 = timeit(lambda: L.splat_gaussian(cls, cx, cy, rad, val, C, H, W), steps)
        r["splat_only"] = _hbm(ms3, pred.numel() * 4, hbm, src, config="splat_gaussian 32x80x128x128")
        return r
    guarded("focal_splat", focal)

    # ---- DCNv2 on the dla_34 layer shapes (B=16): forward and forward+backward, next to the reference kernels
    try:
        from oracle import ref_gpu
        have_ref = ref_gpu.available()
    except Exception:
        have_ref = False
    for (b, ci, hh, co) in ((16, 64, 128, 64), (16, 128, 64, 128), (16, 256, 32, 256), (16, 512, 16, 256),
                            (64, 64, 128, 64)):
        def dcn(b=b, ci=ci, hh=hh, co=co):
            x = torch.randn(b, ci, hh, hh, device=dev, generator=g)
            off = torch.randn(b, 18, hh, hh, device=dev, generator=g) * 2
            msk = torch.sigmoid(torch.randn(b, 9, hh, hh, device=dev, generator=g))
            w = torch.randn(co, ci, 3, 3, device=dev, generator=g) / (3 * ci ** 0.5)
            bias = torch.randn(co, device=dev, generator=g)
            fn = DCNv2Function(1, 1, 1, 1)
            flops = 2.0 * co * ci * 9 * hh * hh * b
            ms = timeit(lambda: fn(x, off, msk, w, bias), steps)
            r = _tensor(ms, flops, tf, src, config="DCNv2 forward B=%d %d@%dx%d->%d (wgmma, 3xTF32)" % (b, ci, hh, hh, co))
            alg = b * ((ci + 27) * hh * hh * 4 + co * hh * hh * 4) + co * ci * 36
            r["hbm_frac"] = round(alg / (ms * 1e-3) / 1e9 / hbm, 4)
            leaves = [t.clone().requires_grad_(True) for t in (x, off, msk, w, bias)]

            def fb():
                for t in leaves:
                    t.grad = None
                fn(*leaves).sum().backward()
            r["fwd_bwd_ms"] = round(timeit(fb, max(5, steps // 4), 2), 5)
            # the backward alone (wgmma: column-gradient GEMM + weight-gradient GEMM = twice the forward's flops)
            bwd_ms = max(r["fwd_bwd_ms"] - ms, 1e-6)
            r["backward"] = _tensor(bwd_ms, 2.0 * flops, tf, src,
                                    config="DCNv2 backward (fwd_bwd_ms - forward; dX by 16-byte vector reductions, the other "
                                           "four gradients bit-identical run to run)")
            r["fwd_bwd_over_fwd"] = round(r["fwd_bwd_ms"] / ms, 2)
            try:   # deterministic dX (cnb_dcnv2_set_deterministic): offsets held inside the gather window
                from centernet_b200._lib import C as _C
                leaves_d = [t.clone().requires_grad_(True) for t in (x, off.clamp(-1.9, 1.9), msk, w, bias)]

                def fbd():
                    for t in leaves_d:
                        t.grad = None
                    fn(*leaves_d).sum().backward()
                import centernet_b200.dcn_v2_func as _f
                prev = _f._DETERMINISTIC
                _f._DETERMINISTIC = True
                try:
                    r["fwd_bwd_deterministic_ms"] = round(timeit(fbd, 3, 1), 5)
                finally:
                    _f._DETERMINISTIC = prev
                    _C.dcnv2_set_deterministic(0)
            except Exception as e:   # noqa: BLE001
                r["fwd_bwd_deterministic_ms"] = "failed: %r" % (e,)
            if have_ref:
                r["reference_gpu_fwd_ms"] = round(timeit(lambda: ref_gpu.dcn_v2_forward(x, off, msk, w, bias), 5, 2), 5)
                go = torch.ones(b, co, hh, hh, device=dev)

                def rfb():
                    ref_gpu.dcn_v2_forward(x, off, msk, w, bias)
                    ref_gpu.dcn_v2_backward(x, off, msk, w, bias, go)
                r["reference_gpu_fwd_bwd_ms"] = round(timeit(rfb, 3, 1), 5)
                r["reference_gpu"] = "oracle/_ref: the reference's dcn_v2_im2col_cuda.cu compiled unmodified + cuBLAS SGEMM"
            try:   # third-party bar of BASELINE.md section 2(c): the same algorithm as shipped by torchvision
                from torchvision.ops import deform_conv2d
                r["torchvision_fwd_ms"] = round(timeit(lambda: deform_conv2d(x, off, w, bias, padding=1, mask=msk), 5, 2), 5)

                def tvfb():
                    for t in leaves:
                        t.grad = None
                    deform_conv2d(leaves[0], leaves[1], leaves[3], leaves[4], padding=1, mask=leaves[2]).sum().backward()
                r["torchvision_fwd_bwd_ms"] = round(timeit(tvfb, 3, 1), 5)
            except Exception:
                pass
            return r
        guarded("dcnv2_b%d_%dx%d_%dto%d" % (b, hh, hh, ci, co), dcn)

    # ---- the reference's ATen-op decode on CUDA tensors (BASELINE.md section 2 "reference on GPU" bar)
    def ref_decode_gpu():
        from oracle import torch_port
        h, w_, r = batches[0]
        ms = timeit(lambda: torch_port.ctdet_decode(h, w_, reg=r, K=K), 10, 3)
        return {"ms": round(ms, 4), "value": 64 / ms * 1e3, "unit": "images/s",
                "config": "reference op sequence (max_pool2d + 2x topk + gathers, oracle/torch_port.py) on CUDA tensors, "
                          "64 img x 80x128x128, K=100"}
    guarded("reference_gpu_ctdet_decode", ref_decode_gpu)
    return out


def run_allreduce(dev, world, rank, steps=10):
    """E2 (training side, N > 1; called on EVERY rank): the per-step gradient exchange of a DLA-34-sized model
    (19.7 M fp32 = 78.7 MB, trains/base_trainer.py:31-35 / models/data_parallel.py) through
    centernet_b200.data_parallel.GradientAllReducer -- bucketed NCCL all-reduce launched from autograd hooks.
    Three timings of one optimiser step of a 20-layer stack with that many parameters: no exchange, exchange
    after the backward (sequential), exchange overlapped with the backward (the shim)."""
    import torch.distributed as dist
    from torch import nn
    from centernet_b200.data_parallel import GradientAllReducer
    torch.manual_seed(1 + rank)
    width, layers, batch = 992, 20, 2048                      # 20 x (992 x 992 + 992) = 19.70 M parameters
    model = nn.Sequential(*[m for _ in range(layers) for m in (nn.Linear(width, width), nn.ReLU())]).to(dev)
    nparam = sum(p.numel() for p in model.parameters())
    x = torch.randn(batch, width, device=dev)
    opt = torch.optim.SGD(model.parameters(), lr=1e-4)

    def step(reduce_after=None):
        model.zero_grad(set_to_none=False)
        model(x).square().mean().backward()
        if reduce_after is not None:
            for p in model.parameters():
                reduce_after.append(dist.all_reduce(p.grad, op=dist.ReduceOp.AVG, async_op=True))
            for h in reduce_after:
                h.wait()
            reduce_after.clear()
        opt.step()

    def timed(fn):
        for _ in range(3):
            fn()
        dist.barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        dist.barrier(); torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / steps], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    ms_none = timed(lambda: step(None))
    ms_seq = timed(lambda: step([]))
    red = GradientAllReducer(model.parameters(), bucket_mb=25.0)
    ms_ovl = timed(lambda: step(None))                        # hooks launch the bucket all-reduces during backward
    n_buckets = len(red.buckets)
    # the exchange alone: the flat buckets, back to back
    def only():
        hs = [dist.all_reduce(b["flat"], op=dist.ReduceOp.AVG, async_op=True) for b in red.buckets]
        for h in hs:
            h.wait()
    ms_ar = timed(only)
    red.remove()
    nbytes = nparam * 4
    busbw = 2.0 * (world - 1) / world * nbytes / (ms_ar * 1e-3) / 1e9
    return {"grad_allreduce_dla34": {
        "bytes": nbytes, "params": nparam, "buckets": n_buckets, "allreduce_ms": round(ms_ar, 4),
        "bus_bandwidth_gbs": round(busbw, 1),
        "note": "a 78.7 MB message in 4 buckets is latency-dominated",
        "step_ms_no_exchange": round(ms_none, 4), "step_ms_exchange_after_backward": round(ms_seq, 4),
        "step_ms_overlapped": round(ms_ovl, 4),
        "exposed_exchange_ms": round(ms_ovl - ms_none, 4),
        "config": "20 x Linear(992, 992) + ReLU, batch 2048/GPU, SGD; gradients averaged over %d ranks (max over ranks, "
                  "CUDA events)" % world}}

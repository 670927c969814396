"""Times one training step of the losses on bf16 / fp16 heads read in place against the fp32 losses and against what
a half head cost before (an explicit .float() upcast in front of the fp32 loss, autograd casting the gradient back),
with CUDA events after warm-up.  A step is what a trainer does: (0.1 * loss).backward(), the gradient landing in
pred.grad.

  f32           fp32 pred through the fp32 path
  upcast_bf16   bf16 pred, loss(pred.float()): the cast, the fp32 kernel, grad * grad_out, the cast back (all timed)
  native_bf16   bf16 pred read in place: the loss pass, then the gradient pass writing bf16 (FocalSplatLoss: the
                loss pass stores its fp32 gradient, then a scale-and-round pass writes bf16)
  native_fp16   the same for fp16

Workloads (seed 317): the bench_secondary.py focal set (80 x 128 x 128, 128 objects per image, radii 0-11) at B = 32
and 64 through _neg_loss (dense target, clamped sigmoid input), _neg_loss_from_logits and
FocalSplatLoss(from_logits=True); RegL1Loss on [B,2,128,128] and [B,34,128,128] with M = 128.

The arms of a group are alternated (the order rotates every repeat); each is timed over windows of at least --window
seconds, --repeats times, and the best window is reported with the spread.  In every timed configuration the native
arms' loss and gradient are compared bit for bit with the upcast arm of the same dtype.  Reported per arm: ms per step,
images/s, the bytes per step its design moves through HBM, computed from the shapes (bytes_per_step below), and the
share of the H100 SXM data-sheet bandwidth (3.35 TB/s) that this is: a whole-step figure, not a kernel's.  After the
timing, in a pass of its own, torch.profiler lists the kernels of one step of every arm at B = 64.  The card's name and
power limit are read in the same call.  Writes DIR/loss_half_time.json and DIR/loss_half_profile.json.  GPU only."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from centernet_b200 import losses as L  # noqa: E402

C_, H_, W_, M_ = 80, 128, 128, 128
HBM_GBS = 3350.0   # H100 SXM data sheet
ARMS = ("f32", "upcast_bf16", "native_bf16", "native_fp16")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001 - the numbers are still worth having without the card name
        return torch.cuda.get_device_name(), "unknown (%s)" % e


def bytes_per_step(arm, n, kind):
    """HBM bytes of one forward + backward over a map of n elements, by the design of each arm.
    f32:     the kernel reads pred 4, writes grad 4; grad * grad_out reads 4, writes 4                       = 16 n
    upcast:  .float() reads 2, writes 4; the f32 arm's 16; the cast back reads 4, writes 2                   = 28 n
    native, dense target: the loss pass reads 2; the gradient pass reads 2, writes 2                         =  6 n
    native, fused splat:  the loss pass reads 2, stores the fp32 gradient 4; scale-and-round reads 4, writes 2 = 12 n
    a dense fp32 gt adds its reads: counting pass 4 + loss pass 4 (f32, upcast), + gradient pass 4 (native).
    reg (the gathered values are noise): f32 zero map 4 + scale 8 = 12 n; upcast 6 + 12 + 6 = 24 n; native fill 2 n."""
    arm = arm.split("_")[0]
    if kind == "reg":
        return {"f32": 12, "upcast": 24, "native": 2}[arm] * n
    if kind == "splat":
        return {"f32": 16, "upcast": 28, "native": 12}[arm] * n
    return {"f32": 16 + 8, "upcast": 28 + 8, "native": 6 + 12}[arm] * n


def window(fn, min_s):
    """ms per call over one window of >= min_s seconds (CUDA events on the current stream)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        fn()
    e1.record()
    torch.cuda.synchronize()
    n = max(3, int(min_s * 1e3 / max(e0.elapsed_time(e1) / 3, 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def time_group(steps, warmup, repeats, min_s):
    names = list(steps)
    for n in names:
        for _ in range(warmup):
            steps[n]()
    torch.cuda.synchronize()
    runs = {n: [] for n in names}
    for r in range(repeats):
        for n in names[r % len(names):] + names[:r % len(names)]:
            runs[n].append(window(steps[n], min_s))
    return runs


def make_step(loss_fn, pred, upcast, keep):
    """One trainer step on pred (a leaf that requires grad); keeps the last loss and leaves the gradient in pred.grad."""
    def step():
        pred.grad = None
        loss = loss_fn(pred.float() if upcast else pred)
        (0.1 * loss).backward()
        keep["loss"] = loss.detach()
    return step


def arms_for(loss_fn, pred32):
    """name -> (step, pred, kept).  The half arms hold pred32 rounded to their dtype; upcast_fp16 is only the oracle of
    native_fp16 and is not timed."""
    arms = {}
    for name, dtype, upcast in (("f32", torch.float32, False), ("upcast_bf16", torch.bfloat16, True),
                                ("native_bf16", torch.bfloat16, False), ("native_fp16", torch.float16, False),
                                ("upcast_fp16", torch.float16, True)):
        pred = pred32.to(dtype).clone().requires_grad_(True)
        keep = {}
        arms[name] = (make_step(loss_fn, pred, upcast, keep), pred, keep)
    return arms


def identical(arms):
    """Bit equality of the loss and of pred.grad as the timed steps left them, native against upcast, per dtype."""
    torch.cuda.synchronize()
    same = {}
    for dt in ("bf16", "fp16"):
        (_, pn, kn), (_, pu, ku) = arms["native_" + dt], arms["upcast_" + dt]
        assert pn.grad.dtype == pu.grad.dtype == pn.dtype
        same[dt] = bool(torch.equal(kn["loss"].view(torch.int32), ku["loss"].view(torch.int32))
                        and torch.equal(pn.grad.view(torch.int16), pu.grad.view(torch.int16)))
    return same


def profile_step(step):
    from torch.profiler import ProfilerActivity, profile as tprofile
    step()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            rows.append({"kernel": ev.key[:110], "us": round(t, 2), "calls": ev.count})
    return sorted(rows, key=lambda r: -r["us"])


def workloads(B, dev):
    """name -> (loss_fn, fp32 pred, kind of bytes_per_step)."""
    g = torch.Generator(device=dev).manual_seed(317)
    logits = torch.randn(B, C_, H_, W_, device=dev, generator=g) - 2.19
    cls = torch.randint(0, C_, (B, M_), device=dev, generator=g)
    cx = torch.randint(0, W_, (B, M_), device=dev, generator=g)
    cy = torch.randint(0, H_, (B, M_), device=dev, generator=g)
    rad = torch.randint(0, 12, (B, M_), device=dev, generator=g)
    val = torch.ones(B, M_, dtype=torch.uint8, device=dev)
    gt = L.splat_gaussian(cls, cx, cy, rad, val, C_, H_, W_)
    splat = L.FocalSplatLoss(from_logits=True)
    out = {"neg_loss": (lambda p: L._neg_loss(p, gt), torch.clamp(torch.sigmoid(logits), 1e-4, 1 - 1e-4), "dense"),
           "neg_loss_from_logits": (lambda p: L._neg_loss_from_logits(p, gt), logits, "dense"),
           "focal_splat_from_logits": (lambda p: splat(p, cls, cx, cy, rad, val), logits, "splat")}
    ind = cy * W_ + cx
    mask = torch.ones(B, M_, device=dev)
    reg = L.RegL1Loss()
    for d in (2, 34):
        target = torch.rand(B, M_, d, device=dev, generator=g) * 32
        pred = torch.rand(B, d, H_, W_, device=dev, generator=g) * 32
        out["reg_l1_D%d" % d] = ((lambda p, t=target: reg(p, mask, ind, t)), pred, "reg")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for loss_half_time.json (created if missing)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0, help="seconds per timed window")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("loss_half_time: needs a CUDA device")
    name, power = card()
    result = {"card": name, "power_limit": power, "hbm_peak_gbs": HBM_GBS,
              "hbm_peak_source": "H100 SXM data sheet (3.35 TB/s)",
              "workload": "seed 317, %dx%dx%d, %d objects per image, radii 0-11; step = (0.1 * loss).backward()"
                          % (C_, H_, W_, M_), "groups": {}}
    profiles = {"card": name, "power_limit": power, "groups": {}}
    for B in (32, 64):
        for wname, (loss_fn, pred32, kind) in workloads(B, "cuda").items():
            arms = arms_for(loss_fn, pred32)
            n = pred32.numel()
            del pred32
            arms["upcast_fp16"][0]()   # the oracle of native_fp16
            runs = time_group({a: arms[a][0] for a in ARMS}, args.warmup, args.repeats, args.window)
            same = identical(arms)
            gname = "%s_B%d" % (wname, B)
            assert all(same.values()), "%s: native differs from its upcast: %s" % (gname, same)
            rows = {}
            for a, ms in runs.items():
                best = min(ms)
                nbytes = bytes_per_step(a, n, kind)
                rows[a] = {"ms_runs": [round(m, 5) for m in ms], "ms": round(best, 5),
                           "spread": round((max(ms) - min(ms)) / best, 4), "images_per_s": round(B / (best * 1e-3), 1),
                           "bytes_per_step": nbytes,
                           "share_of_3.35TBs": round(nbytes / (best * 1e-3) / (HBM_GBS * 1e9), 4)}
            g = {"B": B, "arms": rows, "native_equals_upcast_bitwise": same,
                 "native_bf16_vs_upcast_bf16": round(rows["upcast_bf16"]["ms"] / rows["native_bf16"]["ms"], 3),
                 "native_bf16_vs_f32": round(rows["f32"]["ms"] / rows["native_bf16"]["ms"], 3),
                 "native_fp16_vs_f32": round(rows["f32"]["ms"] / rows["native_fp16"]["ms"], 3)}
            result["groups"][gname] = g
            print("%-30s " % gname + "  ".join("%s %.4f ms" % (a, v["ms"]) for a, v in rows.items())
                  + "  native/upcast x%.2f" % g["native_bf16_vs_upcast_bf16"], flush=True)
            if B == 64:   # tracing slows the host: after the timed windows, never inside them
                profiles["groups"][gname] = {a: profile_step(arms[a][0]) for a in ARMS}
            del arms
            torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    for fname, obj in (("loss_half_time.json", result), ("loss_half_profile.json", profiles)):
        with open(os.path.join(args.out, fname), "w") as f:
            json.dump(obj, f, indent=1)
    print("card: %s, power limit %s; wrote %s" % (name, power, os.path.join(args.out, "loss_half_time.json")))


if __name__ == "__main__":
    main()

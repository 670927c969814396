"""Times the fused bf16 output heads (centernet_b200.heads.fuse_heads) against the unfused heads under
torch.autocast(bfloat16), per task head set of dla_34 (Cin = 64, head_conv = 256), at B = 1, 8 and 64:

  ctdet       hm 80, wh 2, reg 2                                  128 x 128
  multi_pose  hm 1, wh 2, hps 34, reg 2, hm_hp 17, hp_offset 2     128 x 128
  ddd         hm 3, dep 1, rot 8, dim 3, wh 2, reg 2              96 x 320
  exdet       hm_t/l/b/r/ct 80 each, reg_t/l/b/r 2 each           128 x 128

Arms, each running every head of the set on one bf16 input (what an autocast network hands its heads):
  autocast_nchw / autocast_cl   the unfused Sequential under autocast, NCHW / channels_last input
  fused_nchw / fused_cl         the same heads after fuse_heads, under no_grad

The arms alternate within one call: every round times each arm once over a window of at least --seconds with CUDA
events, and the best round counts.  Before timing, every arm's outputs are checked against the fp64 oracle bound of
tests/test_heads_gpu.py on the first two images.  A separate torch.profiler pass (B = 8) gives each arm's kernel time
and the achieved TFLOP/s from shapes.  The card name and power limit are read in the same call.  Writes
heads_time.json into --out.  GPU only."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centernet_b200.heads import fuse_heads  # noqa: E402

TASKS = {
    "ctdet": ({"hm": 80, "wh": 2, "reg": 2}, 128, 128),
    "multi_pose": ({"hm": 1, "wh": 2, "hps": 34, "reg": 2, "hm_hp": 17, "hp_offset": 2}, 128, 128),
    "ddd": ({"hm": 3, "dep": 1, "rot": 8, "dim": 3, "wh": 2, "reg": 2}, 96, 320),
    "exdet": (dict([("hm_" + s, 80) for s in "tlbr"] + [("hm_ct", 80)] + [("reg_" + s, 2) for s in "tlbr"]), 128,
              128),
}
CIN, HEAD_CONV = 64, 256
BF = torch.bfloat16
BF16_PEAK_TFLOPS = 989.0     # H100 SXM dense bf16 (data sheet)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001 - the numbers are still worth having without the card name
        return torch.cuda.get_device_name(), "unknown (%s)" % e


class Heads(nn.Module):
    def __init__(self, heads):
        super().__init__()
        self.heads = heads
        for name, c in heads.items():
            fc = nn.Sequential(nn.Conv2d(CIN, HEAD_CONV, 3, padding=1, bias=True), nn.ReLU(inplace=True),
                               nn.Conv2d(HEAD_CONV, c, 1, stride=1, padding=0, bias=True))
            if "hm" in name:
                fc[-1].bias.data.fill_(-2.19)
            self.__setattr__(name, fc)

    def forward(self, y):
        return {h: self.__getattr__(h)(y) for h in self.heads}


def flops(heads, B, h, w):
    return sum(2.0 * B * h * w * (9 * CIN * HEAD_CONV + HEAD_CONV * c) for c in heads.values())


def bound_check(net, x, outs):
    """max over heads of |y - y64| / bound on the first two images (bf16 output bound of tests/test_heads_gpu.py)."""
    worst = 0.0
    xb = x[:2].double()
    for name in net.heads:
        m = getattr(net, name)
        w1, b1 = m[0].weight.to(BF).double(), m[0].bias.double()
        w2, b2 = m[2].weight.to(BF).double(), m[2].bias.double()
        mid64 = F.conv2d(xb, w1, b1, padding=1)
        e1 = 9 * CIN * 2.0 ** -22 * F.conv2d(xb.abs(), w1.abs(), b1.abs(), padding=1)
        dmid = e1 + 2.0 ** -7 * (mid64.clamp_min(0) + e1)
        midr = mid64.clamp_min(0).float().to(BF).double()
        out64 = F.conv2d(midr, w2, b2)
        bound = F.conv2d(dmid, w2.abs()) + HEAD_CONV * 2.0 ** -22 * F.conv2d(midr + dmid, w2.abs(), b2.abs())
        bound = bound + 2.0 ** -8 * (out64.abs() + bound) + 1e-6
        worst = max(worst, ((outs[name][:2].double() - out64).abs() / bound).max().item())
    return worst


def window(fn, seconds):
    """Calls fn back to back for at least `seconds` (CUDA events); returns ms per call."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, total = 0, 0.0
    while total < seconds * 1e3:
        k = max(1, n)
        e0.record()
        for _ in range(k):
            fn()
        e1.record()
        torch.cuda.synchronize()
        total += e0.elapsed_time(e1)
        n += k
    return total / n


def profile(arms, out_dir, tag):
    from torch.profiler import ProfilerActivity, profile as tprofile
    res = {}
    for name, fn in arms.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0:
                kern[ev.key] = t / 5.0
        res[name] = {"kernel_us_per_call": sum(kern.values()),
                     "top": sorted(kern.items(), key=lambda kv: -kv[1])[:6]}
    with open(os.path.join(out_dir, "heads_profile_%s.json" % tag), "w") as f:
        json.dump(res, f, indent=1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for heads_time.json (created if missing)")
    ap.add_argument("--tasks", default="ctdet,multi_pose,ddd,exdet")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "heads_time.py needs a GPU"
    os.makedirs(args.out, exist_ok=True)
    name, power = card()
    result = {"card": name, "power_limit": power, "window_s": args.seconds, "rounds": args.rounds, "rows": []}
    print("card: %s, power limit %s" % (name, power))
    torch.manual_seed(0)
    for task in args.tasks.split(","):
        heads, h, w = TASKS[task]
        net = Heads(heads).cuda().eval()
        fused = Heads(heads).cuda().eval()
        fused.load_state_dict(net.state_dict())
        assert fuse_heads(fused) == len(heads)
        for B in [int(b) for b in args.batches.split(",")]:
            x = (torch.randn(B, CIN, h, w, device="cuda") * 0.5).to(BF)
            xc = x.contiguous(memory_format=torch.channels_last)

            def ac(inp):
                with torch.no_grad(), torch.autocast("cuda", dtype=BF):
                    return net(inp)

            def fu(inp):
                with torch.no_grad():
                    return fused(inp)

            arms = {"autocast_nchw": lambda: ac(x), "autocast_cl": lambda: ac(xc),
                    "fused_nchw": lambda: fu(x), "fused_cl": lambda: fu(xc)}
            checks = {}
            for an, fn in arms.items():
                outs = fn()
                assert all(o.dtype == BF for o in outs.values()), an
                checks[an] = bound_check(net, x, outs)
                assert checks[an] <= 1.0, (task, B, an, checks[an])
            for fn in arms.values():   # warm-up: module loads, cuDNN algorithm choice
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            best = {an: float("inf") for an in arms}
            for _ in range(args.rounds):
                for an, fn in arms.items():
                    best[an] = min(best[an], window(fn, args.seconds))
            fl = flops(heads, B, h, w)
            row = {"task": task, "B": B, "H": h, "W": w, "gflop": fl / 1e9, "ms": best, "bound_ratio": checks,
                   "tflops": {an: fl / (ms * 1e-3) / 1e12 for an, ms in best.items()},
                   "speedup_cl": best["autocast_cl"] / best["fused_cl"],
                   "speedup_nchw": best["autocast_nchw"] / best["fused_nchw"]}
            result["rows"].append(row)
            print("%-10s B=%-3d  ac_nchw %8.3f  ac_cl %8.3f  fu_nchw %8.3f  fu_cl %8.3f ms   fused_cl %6.1f TFLOP/s  "
                  "x%.2f (cl) x%.2f (nchw)" % (task, B, best["autocast_nchw"], best["autocast_cl"], best["fused_nchw"],
                                               best["fused_cl"], row["tflops"]["fused_cl"], row["speedup_cl"],
                                               row["speedup_nchw"]), flush=True)
            if B == 8:
                prof = profile(arms, args.out, "%s_B%d" % (task, B))
                row["profile_kernel_us"] = {an: p["kernel_us_per_call"] for an, p in prof.items()}
                row["profile_tflops"] = {an: fl / (p["kernel_us_per_call"] * 1e-6) / 1e12
                                         for an, p in prof.items() if p["kernel_us_per_call"] > 0}
                row["profile_share_of_peak"] = {an: v / BF16_PEAK_TFLOPS for an, v in row["profile_tflops"].items()}
                print("           profiler kernel us/call: %s" % {an: round(v, 1) for an, v in
                                                                   row["profile_kernel_us"].items()}, flush=True)
            del x, xc
            torch.cuda.empty_cache()
    name2, power2 = card()
    result["card_after"], result["power_limit_after"] = name2, power2
    path = os.path.join(args.out, "heads_time.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("card: %s, power limit %s; wrote %s (%s)" % (name, power, path, time.strftime("%H:%M:%S")))


if __name__ == "__main__":
    main()

"""Times DCNv2 forward + backward through DCNv2Function on the 16 DCN layers of dla_34 at 512x512 (the 7 distinct
shapes of SURVEY 3.2, weighted by how often they occur), at B = 16 and 64, for three paths:

  fp32        the default (3xTF32 forward and backward), fp32 input of the same values
  bf16        compute_dtype=torch.bfloat16: bf16 forward, fp32 backward at the upcast operands
  bf16_bwd16  compute_dtype=backward_dtype=torch.bfloat16: bf16 forward and bf16 backward

with offsets randn * 1.5 (on a 2^-16 grid), the activation bf16 (fp32 for the fp32 path) in channels_last and in
NCHW layout, and the gradient of the output in the output's dtype.  The three paths of a (layer, layout) run in
alternation: 3 windows of at least 1 s each per path, best window reported with the spread (max - min) / min of the
three.  The gradients of
the timed bf16_bwd16 calls are checked against the bounds of tests/test_bf16_bwd_gpu.py with the float64 DCNv2 (FP64
tensor cores) at the bf16 operands (dBias: the depth of its fixed summation tree times 2^-24 sum |dY|); each
gradient's largest |error| / bound is reported.  The offsets are rounded to a 2^-16 grid so that every sampling position
is exact in fp32 and the fp64 reference samples the same points.
A torch.profiler per-kernel table of the two bf16 paths for 64@128^2->64 and 256@32^2->256 (B = 16, channels_last)
is taken in a phase of its own after the timing, and for every layer where bf16_bwd16 is slower than bf16.  The card
name and power limit are read in the same call.  Writes dcn_bf16_bwd_time.json into --out.  GPU only."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centernet_b200.dcn_v2_func import DCNv2Function  # noqa: E402

BF = torch.bfloat16
# (Cin, H = W, Cout, layers of this shape in dla_34)
LAYERS = [(512, 16, 256, 1), (256, 32, 256, 1), (256, 32, 128, 2), (128, 64, 128, 2), (128, 64, 64, 4),
          (64, 128, 64, 5), (256, 32, 64, 1)]
PATHS = {"fp32": DCNv2Function(1, 1), "bf16": DCNv2Function(1, 1, compute_dtype=BF),
         "bf16_bwd16": DCNv2Function(1, 1, compute_dtype=BF, backward_dtype=BF)}
PROFILED = [(64, 128, 64), (256, 32, 256)]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001 - the numbers are still worth having without the card name
        return torch.cuda.get_device_name(), "unknown (%s)" % e


def layer_case(B, Ci, HW, Co, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, Ci, HW, HW, device="cuda", generator=g).to(BF)
    off = torch.round(torch.randn(B, 18, HW, HW, device="cuda", generator=g) * 1.5 * 2.0 ** 16) / 2.0 ** 16
    m = torch.sigmoid(torch.randn(B, 9, HW, HW, device="cuda", generator=g))
    w = torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) / (3.0 * Ci ** 0.5)
    b = torch.randn(Co, device="cuda", generator=g)
    go = torch.randn(B, Co, HW, HW, device="cuda", generator=g).to(BF)
    return x, off, m, w, b, go


def step(path, x, off, m, w, b, go):
    """One forward + backward; the gradients are returned, not accumulated."""
    f = PATHS[path]
    xin = x.float() if path == "fp32" else x          # the same values; .float() keeps the memory format
    leaves = [t.detach().requires_grad_(True) for t in (xin, off, m, w, b)]
    y = f(*leaves)
    return torch.autograd.grad(y, leaves, go.to(y.dtype))


def window(fn, seconds):
    """ms per call over a window of at least `seconds` (host clock around work that ends in a synchronise)."""
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        if n % 4 == 0:
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if dt >= seconds:
                return dt * 1e3 / n


def check(x, off, m, w, b, go, grads):
    """max over the five gradients of |g - g64| / bound, the bounds of tests/test_bf16_bwd_gpu.py::
    test_random_within_bound (g64 and S: the float64 DCNv2 at the bf16 operands and at their magnitudes)."""
    f64 = DCNv2Function(1, 1)

    def g64(xx, ww, bb, gg):
        leaves = [t.detach().double().requires_grad_(True) for t in (xx, off, m, ww, bb)]
        y = f64(*leaves)
        return torch.autograd.grad(y, leaves, gg.double())

    wb = w.to(BF)
    ref = g64(x, wb, b, go)
    S = g64(x.abs(), wb.abs(), b, go.abs())
    Ci, Co = x.shape[1], w.shape[0]
    gam = (Co + Ci + 9 * 81 + 16) * 2.0 ** -24
    B, HW = x.shape[0], x.shape[2] * x.shape[3]
    depth = 13 + (B * ((HW + 31) // 32) + 255) // 256      # dBias: 32-pixel shuffle tree, strided sums, 256-way tree
    bounds = [gam * S[0] + 1e-6 + 2.0 ** -8 * ref[0].abs(),        # grad_input is returned in bf16
              2.0 ** -12 * ref[1].abs().max() + 1e-6, gam * S[2] + 1e-6, (2.0 ** -8 + 2.0 ** -12) * S[3] + 1e-6,
              depth * 2.0 ** -24 * go.double().abs().sum((0, 2, 3)) + 1e-6]
    return {n: ((g.double() - r).abs() / bd).max().item()
            for n, g, r, bd in zip(("input", "offset", "mask", "weight", "bias"), grads, ref, bounds)}


def profile(fn, reps=5):
    from torch.profiler import ProfilerActivity, profile as tprofile
    fn()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            rows.append({"kernel": ev.key[:120], "us_per_step": t / reps, "calls_per_step": ev.count / reps})
    return sorted(rows, key=lambda r: -r["us_per_step"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for dcn_bf16_bwd_time.json (created if missing)")
    ap.add_argument("--batches", type=int, nargs="*", default=[16, 64])
    ap.add_argument("--seconds", type=float, default=1.0, help="least length of one timing window")
    ap.add_argument("--windows", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    result = {"card": name, "power_limit": power, "windows": args.windows, "window_s": args.seconds, "layers": [],
              "dla34_sum_ms": {}, "profiles": []}
    slower = []
    for B in args.batches:
        sums = {}
        for Ci, HW, Co, count in LAYERS:
            x, off, m, w, b, go = layer_case(B, Ci, HW, Co)
            for layout in ("channels_last", "nchw"):
                xl = x.contiguous(memory_format=torch.channels_last) if layout == "channels_last" else x.contiguous()
                fns = {p: (lambda p=p: step(p, xl, off, m, w, b, go)) for p in PATHS}
                for fn in fns.values():       # warm-up: module load, weight tiles, allocator
                    for _ in range(3):
                        fn()
                times = {p: [] for p in PATHS}
                for _ in range(args.windows):
                    for p, fn in fns.items():
                        times[p].append(window(fn, args.seconds))
                row = {"B": B, "cin": Ci, "hw": HW, "cout": Co, "count": count, "layout": layout, "paths": {}}
                for p, ts in times.items():
                    row["paths"][p] = {"ms": min(ts), "spread": (max(ts) - min(ts)) / min(ts), "windows_ms": ts}
                    sums.setdefault(layout, {}).setdefault(p, 0.0)
                    sums[layout][p] += count * min(ts)
                row["speedup_vs_bf16"] = row["paths"]["bf16"]["ms"] / row["paths"]["bf16_bwd16"]["ms"]
                row["err_over_bound"] = check(xl, off, m, w, b, go, fns["bf16_bwd16"]())
                if row["speedup_vs_bf16"] < 1.0:
                    slower.append((B, Ci, HW, Co, layout))
                result["layers"].append(row)
                print("B%-3d %3d@%3dx%-3d->%3d x%d %-13s " % (B, Ci, HW, HW, Co, count, layout) +
                      "  ".join("%s %.3f ms (+-%.1f%%)" % (p, v["ms"], 100 * v["spread"])
                                for p, v in row["paths"].items()) +
                      "  bwd16 vs bf16 %.2fx  err/bound %s" % (row["speedup_vs_bf16"], " ".join(
                          "%s %.3f" % kv for kv in row["err_over_bound"].items())),
                      flush=True)
                del fns, xl
            del x, off, m, w, b, go
            torch.cuda.empty_cache()
        result["dla34_sum_ms"]["B%d" % B] = sums
        for layout, s in sums.items():
            print("B%d dla_34 DCN fwd+bwd sum (%s): " % (B, layout) +
                  "  ".join("%s %.3f ms" % kv for kv in s.items()) +
                  "  bwd16 vs bf16 %.3fx" % (s["bf16"] / s["bf16_bwd16"]), flush=True)

    # profiles, with the timing done: the two named shapes, and every layer where the bf16 backward was slower
    todo = [(16, Ci, HW, Co, "channels_last") for Ci, HW, Co in PROFILED] + [t for t in slower if t[0] == 16]
    for B, Ci, HW, Co, layout in todo:
        x, off, m, w, b, go = layer_case(B, Ci, HW, Co)
        xl = x.contiguous(memory_format=torch.channels_last) if layout == "channels_last" else x.contiguous()
        entry = {"B": B, "cin": Ci, "hw": HW, "cout": Co, "layout": layout}
        for p in ("bf16", "bf16_bwd16"):
            entry[p] = profile(lambda p=p: step(p, xl, off, m, w, b, go))
        result["profiles"].append(entry)
        for p in ("bf16", "bf16_bwd16"):
            print("profile B%d %d@%d->%d %s %s:" % (B, Ci, HW, Co, layout, p))
            for r in entry[p][:14]:
                print("   %9.1f us  x%.0f  %s" % (r["us_per_step"], r["calls_per_step"], r["kernel"][:90]))
        del x, off, m, w, b, go, xl
        torch.cuda.empty_cache()
    name2, power2 = card()
    result["card_after"], result["power_limit_after"] = name2, power2
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "dcn_bf16_bwd_time.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("card: %s, power limit %s; wrote %s" % (name, power, path))


if __name__ == "__main__":
    main()

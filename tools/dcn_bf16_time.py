"""Times the bf16 DCNv2 forward against the fp32 (3xTF32) forward on the 16 DCN layers of dla_34 at 512x512 (the 7
distinct shapes of SURVEY 3.2, weighted by how often they occur), at B = 16 and 64, with CUDA events after warm-up:

  fp32_nchw      cnb_dcnv2_forward_prepared, fp32 NCHW input (one re-layout pass)
  fp32_cl        cnb_dcnv2_forward_prepared, fp32 channels_last input (sampled in place)
  bf16_cl        cnb_dcnv2_forward_bf16, bf16 channels_last input (sampled in place), bf16 output
  fp32_fused     cnb_dcnv2_forward_fused + BN + ReLU, fp32 channels_last input
  bf16_fused     cnb_dcnv2_forward_fused_bf16 + BN + ReLU, bf16 channels_last input, bf16 output

Per layer: ms, TFLOP/s, share of the 989 TFLOP/s dense bf16 data-sheet peak (H100 SXM), the compute and bytes bounds
and which one applies, and the largest |y - y64| / bound of tests/test_bf16_gpu.py (bound = 2^-7 S + 2^-8 |y64| +
1e-5, y64 and S from the float64 DCNv2 kernels on two images).  Also the summed DCN forward time of a 64-image
dla_34 batch per mode, and the card and its power limit.  A layer where bf16 is not faster than fp32 gets a
torch.profiler kernel table.  Writes one JSON file into --out.  GPU only."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centernet_b200._lib import C, ptr, stream_ptr, workspace  # noqa: E402
from centernet_b200.dcn_v2_func import DCNv2Function  # noqa: E402

# (Cin, H = W, Cout, layers of this shape in dla_34)
LAYERS = [(512, 16, 256, 1), (256, 32, 256, 1), (256, 32, 128, 2), (128, 64, 128, 2), (128, 64, 64, 4),
          (64, 128, 64, 5), (256, 32, 64, 1)]
BF16_PEAK_TFLOPS = 989.0     # H100 SXM dense bf16 (data sheet)
TF32X3_PEAK_TFLOPS = BF16_PEAK_TFLOPS / 6   # 3 TF32 MMAs (half the bf16 rate each) per product
HBM_TBPS = 3.35              # H100 SXM HBM3 (data sheet)


def timeit(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


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
    x = torch.randn(B, Ci, HW, HW, device="cuda", generator=g)
    off = torch.randn(B, 18, HW, HW, device="cuda", generator=g) * 1.5
    m = torch.sigmoid(torch.randn(B, 9, HW, HW, device="cuda", generator=g))
    w = torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) / (3.0 * Ci ** 0.5)
    b = torch.randn(Co, device="cuda", generator=g)
    sc = torch.rand(Co, device="cuda", generator=g) + 0.5
    sh = torch.randn(Co, device="cuda", generator=g) * 0.2
    return x, off, m, w, b, sc, sh


def calls(B, Ci, HW, Co, x, off, m, w, b, sc, sh):
    """The five forwards as argument-ready closures on preallocated buffers (no allocation in the timed loop)."""
    cfg = (B, Ci, HW, HW, Co, 3, 3)
    wt32 = workspace(C.dcnv2_wtiles_bytes(Ci, Co, 3, 3, 1), x.device)
    C.dcnv2_prepare_weights(ptr(w), Ci, Co, 3, 3, 1, ptr(wt32), wt32.numel(), stream_ptr(w))
    wt16 = workspace(C.dcnv2_wtiles_bf16_bytes(Ci, Co, 3, 3, 1), x.device)
    C.dcnv2_prepare_weights_bf16(ptr(w), Ci, Co, 3, 3, 1, ptr(wt16), wt16.numel(), stream_ptr(w))
    query = (B, Ci, Co, HW, HW, 3, 3, 1, 1, 1, 1)   # the queries take cout before h, w
    ws32 = workspace(C.dcnv2_prepared_workspace_bytes(*query), x.device)
    ws16 = workspace(C.dcnv2_bf16_workspace_bytes(*query), x.device)
    xcl = x.contiguous(memory_format=torch.channels_last)
    x16 = xcl.to(torch.bfloat16)
    om = torch.cat([off, torch.logit(m)], dim=1).contiguous()
    y32 = torch.empty(B, Co, HW, HW, device="cuda")
    y16 = torch.empty(B, Co, HW, HW, device="cuda", dtype=torch.bfloat16)
    s = stream_ptr(x)
    BF16 = C.DTYPE_BF16

    def fp32(xin, cl):
        return lambda: C.dcnv2_forward_prepared(ptr(xin), cl, ptr(off), ptr(m), ptr(wt32), ptr(b), ptr(y32), *cfg,
                                                1, 1, 1, 1, 1, 1, 1, ptr(ws32), ws32.numel(), s)
    return {
        "fp32_nchw": (fp32(x, 0), y32),
        "fp32_cl": (fp32(xcl, 1), y32),
        "bf16_cl": (lambda: C.dcnv2_forward_bf16(ptr(x16), BF16, 1, ptr(off), ptr(m), ptr(wt16), ptr(b), ptr(y16),
                                                 BF16, *cfg, 1, 1, 1, 1, ptr(ws16), ws16.numel(), s), y16),
        "fp32_fused": (lambda: C.dcnv2_forward_fused(ptr(xcl), 1, ptr(om), ptr(wt32), ptr(b), ptr(sc), ptr(sh), 1,
                                                     ptr(y32), *cfg, 1, 1, 1, 1, ptr(ws32), ws32.numel(), s), y32),
        "bf16_fused": (lambda: C.dcnv2_forward_fused_bf16(ptr(x16), BF16, 1, ptr(om), ptr(wt16), ptr(b), ptr(sc),
                                                          ptr(sh), 1, ptr(y16), BF16, *cfg, 1, 1, 1, 1, ptr(ws16),
                                                          ws16.numel(), s), y16),
    }


def bound_ratio(x, off, m, w, b, n_img=2):
    """max |y - y64| / (2^-7 S + 2^-8 |y64| + 1e-5) of the bf16 forward (bf16 channels_last in, bf16 out)."""
    x, off, m = x[:n_img], off[:n_img], m[:n_img]
    xb, wb = x.to(torch.bfloat16).double(), w.to(torch.bfloat16).double()
    f64 = DCNv2Function(1, 1)
    y64 = f64(xb, off.double(), m.double(), w.double(), b.double())
    S = f64(xb.abs(), off.double(), m.double(), wb.abs(), None)
    y = DCNv2Function(1, 1, compute_dtype=torch.bfloat16)(
        x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last), off, m, w, b)
    return ((y.double() - y64).abs() / (2.0 ** -7 * S + 2.0 ** -8 * y64.abs() + 1e-5)).max().item()


def profile(fn):
    from torch.profiler import ProfilerActivity, profile as tprofile
    fn()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            rows.append({"kernel": ev.key[:120], "us_per_call": t / 5.0, "calls_per_step": ev.count / 5.0})
    return sorted(rows, key=lambda r: -r["us_per_call"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for dcn_bf16_time.json (created if missing)")
    ap.add_argument("--batches", type=int, nargs="*", default=[16, 64])
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, power = card()
    result = {"card": name, "power_limit": power, "bf16_peak_tflops": BF16_PEAK_TFLOPS,
              "tf32x3_peak_tflops": TF32X3_PEAK_TFLOPS, "hbm_tbps": HBM_TBPS, "layers": [], "dla34_sum_ms": {}}
    for B in args.batches:
        sums = {}
        for Ci, HW, Co, count in LAYERS:
            x, off, m, w, b, sc, sh = layer_case(B, Ci, HW, Co)
            fns = calls(B, Ci, HW, Co, x, off, m, w, b, sc, sh)
            flop = 2.0 * B * Co * Ci * 9 * HW * HW
            row = {"B": B, "cin": Ci, "hw": HW, "cout": Co, "count": count, "gflop": flop / 1e9, "modes": {}}
            for mode, (fn, _) in fns.items():
                ms = timeit(fn, args.warmup, args.iters)
                bf = mode.startswith("bf16")
                # bytes a pass must move at least: input, offsets + mask (fp32), weights, output
                act = 2 if bf else 4
                nbytes = B * HW * HW * (Ci * act + 27 * 4 + Co * act) + Co * Ci * 9 * act
                t_compute = flop / ((BF16_PEAK_TFLOPS if bf else TF32X3_PEAK_TFLOPS) * 1e12) * 1e3
                t_bytes = nbytes / (HBM_TBPS * 1e12) * 1e3
                tflops = flop / (ms * 1e-3) / 1e12
                row["modes"][mode] = {
                    "ms": ms, "tflops": tflops, "share_of_bf16_peak": tflops / BF16_PEAK_TFLOPS,
                    "compute_bound_ms": t_compute, "bytes_bound_ms": t_bytes,
                    "bound": "compute" if t_compute >= t_bytes else "bytes",
                    "share_of_bound": max(t_compute, t_bytes) / ms}
                sums[mode] = sums.get(mode, 0.0) + count * ms
            row["bf16_speedup_plain"] = row["modes"]["fp32_cl"]["ms"] / row["modes"]["bf16_cl"]["ms"]
            row["bf16_speedup_fused"] = row["modes"]["fp32_fused"]["ms"] / row["modes"]["bf16_fused"]["ms"]
            row["max_err_over_bound"] = bound_ratio(x, off, m, w, b)
            if row["bf16_speedup_plain"] <= 1.0 or row["bf16_speedup_fused"] <= 1.0:
                row["profile"] = {k: profile(fns[k][0]) for k in ("fp32_cl", "bf16_cl", "fp32_fused", "bf16_fused")}
            result["layers"].append(row)
            print("B%-3d %3d@%3dx%-3d->%3d x%d  " % (B, Ci, HW, HW, Co, count) +
                  "  ".join("%s %.3f ms (%.0f TF/s)" % (k, v["ms"], v["tflops"]) for k, v in row["modes"].items()) +
                  "  speed-up %.2fx / fused %.2fx  err/bound %.3f" % (row["bf16_speedup_plain"],
                                                                      row["bf16_speedup_fused"],
                                                                      row["max_err_over_bound"]), flush=True)
            del x, off, m, w, b, sc, sh, fns
            torch.cuda.empty_cache()
        result["dla34_sum_ms"]["B%d" % B] = sums
        print("B%d dla_34 DCN forward sum: " % B + "  ".join("%s %.3f ms" % kv for kv in sums.items()), flush=True)
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "dcn_bf16_time.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("card: %s, power limit %s; wrote %s" % (name, power, path))


if __name__ == "__main__":
    main()

"""Times the DCN block kernel (cnb_dcnv2_forward_block_bf16: conv_offset_mask inside the bf16 DCN kernel) against
today's bf16 inference path on the 16 DCN layers of dla_34 at 512x512 (the 7 distinct shapes of LAYERS in
tools/dcn_bf16_time.py, weighted by how often they occur), at B = 1, 16 and 64.  Each layer is a DeformConv (DCN, then
BatchNorm + ReLU) in bf16, channels_last, in eval mode under no_grad:

  today   set_compute_dtype(bf16) + fuse_dcn_bn_relu: cuDNN bf16 conv_offset_mask, the fp32 copy of its output and
          cnb_dcnv2_forward_fused_bf16 with BN + ReLU in the epilogue
  block   the same module after fuse_offset_conv: one cnb_dcnv2_forward_block_bf16

The two arms alternate in one run (--reps rounds), each timed with CUDA events over a window of at least --window
seconds after warm-up; the median round is reported.  Per layer: ms of both arms and the speed-up, TFLOP/s and GB/s
of the block kernel (FLOPs of the offset conv and the DCN contraction; bytes of the bf16 input and output and the
weights) against the larger of the bf16 compute bound and the HBM bound, and the largest |y - y64| / bound of
tests/test_dcn_block_gpu.py on two images.  Then the 16-layer sums, the card and its power limit.  Writes one JSON
file into --out.  GPU only."""
import argparse
import json
import os
import statistics
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from centernet_b200.dcn_v2 import DCN, fuse_dcn_bn_relu, fuse_offset_conv, set_compute_dtype  # noqa: E402
from centernet_b200.dcn_v2_func import dcn_block_inference  # noqa: E402
from dcn_bf16_time import BF16_PEAK_TFLOPS, HBM_TBPS, LAYERS, card  # noqa: E402

BF = torch.bfloat16


class DeformConv(nn.Module):
    """pose_dla_dcn.DeformConv"""

    def __init__(self, chi, cho):
        super().__init__()
        self.actf = nn.Sequential(nn.BatchNorm2d(cho, momentum=0.1), nn.ReLU(inplace=True))
        self.conv = DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)

    def forward(self, x):
        return self.actf(self.conv(x))


def layer(Ci, Co, seed=0):
    torch.manual_seed(seed)
    m = DeformConv(Ci, Co)
    m.conv.conv_offset_mask.weight.data.normal_(0, 0.3 / Ci ** 0.5)    # offsets of a few pixels, as a trained model
    m.conv.conv_offset_mask.bias.data.normal_(0, 1.0)
    bn = m.actf[0]
    bn.running_mean.uniform_(-0.5, 0.5)
    bn.running_var.uniform_(0.5, 2.0)
    m = m.cuda().to(BF).to(memory_format=torch.channels_last).eval()
    set_compute_dtype(m, BF)
    fuse_dcn_bn_relu(m)
    fuse_offset_conv(m)       # the arms below switch the flag it sets
    return m


def window(fn, seconds, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 1
    while True:
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= seconds * 1e3:
            return ms / n
        n = max(n * 2, int(n * seconds * 1.1e3 / max(ms, 1e-3)))


def bound_ratio(m, Ci, HW):
    """largest |block - y64| / bound on two images (tests/test_dcn_block_gpu.block_bound; no BN)"""
    from test_dcn_block_gpu import block_bound
    c = m.conv
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, Ci, HW, HW, generator=g).to(BF)
    w_om, b_om = c.conv_offset_mask.weight.float().cpu(), c.conv_offset_mask.bias.float().cpu()
    w, b = c.weight.float().cpu(), c.bias.float().cpu()
    y64, bound = block_bound(x.float(), w_om, b_om, w, b)
    y = dcn_block_inference(x.cuda().contiguous(memory_format=torch.channels_last), c.conv_offset_mask.weight,
                            c.conv_offset_mask.bias, c.weight, c.bias, 1, 1, 1, 1)
    lim = bound + 2.0 ** -8 * y64.abs()
    return ((y.double().cpu() - y64).abs() / lim).max().item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for dcn_block_time.json (created if missing)")
    ap.add_argument("--batches", type=int, nargs="*", default=[1, 16, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dcn_block_time.py needs a GPU"
    name, power = card()
    rows = []
    for Ci, HW, Co, count in LAYERS:
        m = layer(Ci, Co)
        ratio = bound_ratio(m, Ci, HW)
        for B in args.batches:
            x = torch.randn(B, Ci, HW, HW, device="cuda").to(BF).contiguous(memory_format=torch.channels_last)

            def today():
                m.conv.offset_conv_fused = False
                return m(x)

            def block():
                m.conv.offset_conv_fused = True
                return m(x)

            with torch.no_grad():
                assert torch.equal(block(), block())
                times = {"today": [], "block": []}
                for _ in range(args.reps):
                    for arm, fn in (("today", today), ("block", block)):
                        times[arm].append(window(fn, args.window, args.warmup))
            arms = {k: statistics.median(v) for k, v in times.items()}
            flop = 2.0 * B * HW * HW * 9 * Ci * (Co + 27)
            nbytes = 2.0 * (B * HW * HW * (Ci + Co) + 9 * Ci * (Co + 27))
            t_min = max(flop / (BF16_PEAK_TFLOPS * 1e12), nbytes / (HBM_TBPS * 1e12)) * 1e3
            bound_by = "bf16" if flop / BF16_PEAK_TFLOPS > nbytes / HBM_TBPS else "hbm"
            t = arms["block"]
            row = {"B": B, "cin": Ci, "hw": HW, "cout": Co, "count": count, "ms_today": arms["today"],
                   "ms_block": t, "speedup": arms["today"] / t, "tflops_block": flop / t / 1e9,
                   "gbps_block": nbytes / t / 1e6, "bound": bound_by, "share_of_bound": t_min / t,
                   "err_over_bound": ratio, "all_ms": times}
            rows.append(row)
            print("B=%-3d %4d@%-3d -> %-3d x%d  today %8.4f ms  block %8.4f ms  x%.2f  %6.1f TFLOP/s %7.1f GB/s  "
                  "%.1f%% of the %s bound  err/bound %.3f" % (B, Ci, HW, Co, count, arms["today"], t,
                                                               arms["today"] / t, flop / t / 1e9, nbytes / t / 1e6,
                                                               100 * t_min / t, bound_by, ratio), flush=True)
    sums = {}
    for B in args.batches:
        rs = [r for r in rows if r["B"] == B]
        sums[B] = {"ms_today": sum(r["ms_today"] * r["count"] for r in rs),
                   "ms_block": sum(r["ms_block"] * r["count"] for r in rs)}
        sums[B]["speedup"] = sums[B]["ms_today"] / sums[B]["ms_block"]
        print("B=%-3d 16 layers: today %.3f ms, block %.3f ms, x%.3f" % (B, sums[B]["ms_today"], sums[B]["ms_block"],
                                                                       sums[B]["speedup"]))
    print("card: %s, power limit %s" % (name, power))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "dcn_block_time.json"), "w") as f:
        json.dump({"card": name, "power_limit": power, "rows": rows, "sums": sums}, f, indent=1)


if __name__ == "__main__":
    main()

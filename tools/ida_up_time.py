"""Times the fused IDA up-sampling step (cnb_ida_up_add) against the unfused one on the 8 up layers of dla_34 at
512x512 (the 4 distinct shapes of UPS, weighted by how often they occur), at B = 1, 16 and 64.

Per up shape, for fp32 and bf16 and for NCHW and channels_last inputs (p and skip in the same layout):

  unfused   up(p) + skip: cuDNN's depthwise ConvTranspose2d (TF32 allowed, as by default), then one ATen add
  fused     the step as fuse_ida_up runs it where it fuses (ida._fused_step with the routing of small f = 2 steps
            turned off: the cached fp32 weight, one kernel, output in skip's layout), so both sides of that rule show

Then the whole IDA chain of the dla_34 neck (8 steps: proj + up + add + node, all 16 DeformConvs on the bf16 DCN block
kernel through set_compute_dtype + fuse_offset_conv + fuse_dcn_bn_relu), in bf16 at 512x512 input, in three arms:

  unfused   the neck as it is
  fused     after fuse_ida_up: each step writes skip's layout (NCHW here), which the node's kernel converts first
  fused_cl  after fuse_ida_up, with each step writing channels_last, which the node's kernel reads in place

The arms alternate in one run (--reps rounds), each timed with CUDA events over a window of at least --window seconds
after warm-up; the median round is reported.  Per shape: ms of both arms, the speed-up, the algorithmic bytes
(p + skip + out) and the achieved bytes/s of each arm beside the H100 SXM data-sheet HBM3 bandwidth (a reference, not
a target), and the largest |y - y64| / bound of every arm against the fp64 oracle (fused: the bound of
tests/test_ida_gpu.py; unfused: two roundings of its dtype, TF32 in fp32).  The card and its power limit are read in
the same run.  Writes ida_up_time.json into --out.  GPU only."""
import argparse
import copy
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests"))
from centernet_b200 import ida as I  # noqa: E402
from centernet_b200.dcn_v2 import fuse_dcn_bn_relu, fuse_offset_conv, set_compute_dtype  # noqa: E402
from dcn_bf16_time import HBM_TBPS, card  # noqa: E402
from dcn_block_time import window  # noqa: E402
from test_ida_abi import Neck, neck_inputs  # noqa: E402

BF = torch.bfloat16
U32, U16, UTF32 = 2.0 ** -24, 2.0 ** -8, 2.0 ** -11
# (channels o, low-resolution side, up factor f, up layers of this shape in dla_34 at 512x512)
UPS = [(256, 16, 2, 1), (128, 32, 2, 2), (64, 64, 2, 4), (64, 32, 4, 1)]


def check(y, p, w, f, skip, u):
    """max |y - y64| / (u * (sum |w p| + |skip|)), in fp64 on the GPU."""
    pd, wd, sd = p.double(), w.double(), skip.double()
    want = F.conv_transpose2d(pd, wd, stride=f, padding=f // 2, groups=p.shape[1]) + sd
    S = F.conv_transpose2d(pd.abs(), wd.abs(), stride=f, padding=f // 2, groups=p.shape[1]) + sd.abs()
    return ((y.double() - want).abs() / (u * S).clamp_min(1e-300)).max().item()


def up_rows(args):
    rows = []
    min_out, I._F2_MIN_OUT = I._F2_MIN_OUT, 0
    for B in args.batches:
        for o, hp, f, count in UPS:
            for dtype in (torch.float32, BF):
                for cl in (False, True):
                    fmt = torch.channels_last if cl else torch.contiguous_format
                    g = torch.Generator(device="cuda").manual_seed(B + o + f)
                    p = torch.randn(B, o, hp, hp, device="cuda", generator=g).to(dtype).contiguous(memory_format=fmt)
                    skip = torch.randn(B, o, f * hp, f * hp, device="cuda", generator=g).to(dtype) \
                        .contiguous(memory_format=fmt)
                    up = torch.nn.ConvTranspose2d(o, o, 2 * f, stride=f, padding=f // 2, groups=o, bias=False)
                    up = up.to(device="cuda", dtype=dtype).eval()
                    w = up.weight.detach()
                    arms = {"unfused": lambda: up(p) + skip, "fused": lambda: I._fused_step(up, p, skip)}
                    err = {}
                    with torch.no_grad():
                        for name, fn in arms.items():
                            u = (6 * U32 + U16) if dtype == BF else 6 * U32
                            if name == "unfused":
                                u = 6 * U32 + 2 * U16 + U16 * U16 if dtype == BF else 6 * U32 + 2 * UTF32
                            err[name] = check(fn(), p, w, f, skip, u)
                        times = {k: [] for k in arms}
                        for _ in range(args.reps):
                            for name, fn in arms.items():
                                times[name].append(window(fn, args.window, args.warmup))
                    ms = {k: statistics.median(v) for k, v in times.items()}
                    esz = 4 if dtype == torch.float32 else 2
                    nbytes = (B * o * hp * hp + 2 * B * o * (f * hp) ** 2) * esz
                    row = {"B": B, "o": o, "p": hp, "f": f, "count": count, "dtype": str(dtype).split(".")[-1],
                           "layout": "channels_last" if cl else "nchw", "ms_unfused": ms["unfused"],
                           "ms_fused": ms["fused"], "speedup": ms["unfused"] / ms["fused"], "bytes": nbytes,
                           "tbps_fused": nbytes / ms["fused"] * 1e-9, "tbps_unfused": nbytes / ms["unfused"] * 1e-9,
                           "err_over_bound": err}
                    rows.append(row)
                    print("B%-3d o%-4d %3d^2 f%d %-5s %-13s unfused %.4f ms  fused %.4f ms  x%.2f  fused %.2f TB/s "
                          "(data sheet %.2f)  err/bound %s" % (B, o, hp, f, row["dtype"], row["layout"],
                                                              ms["unfused"], ms["fused"], row["speedup"],
                                                              row["tbps_fused"], HBM_TBPS,
                                                              {k: round(v, 3) for k, v in err.items()}), flush=True)
                    assert max(err.values()) <= 1.0, "an arm is outside its error bound"
    I._F2_MIN_OUT = min_out
    return rows


def neck(seed=0):
    torch.manual_seed(seed)
    m = Neck()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.uniform_(-0.2, 0.2)
            mod.running_var.uniform_(0.5, 2.0)
        if hasattr(mod, "conv_offset_mask"):
            mod.conv_offset_mask.weight.data.normal_(0, 0.01)
            mod.conv_offset_mask.bias.data.normal_(0, 0.3)
    m = m.cuda().to(BF).eval()
    set_compute_dtype(m, BF)
    fuse_offset_conv(m)
    fuse_dcn_bn_relu(m)
    return m


def chain_rows(args):
    rows = []
    base = neck()
    fused = copy.deepcopy(base)
    for m in fused.modules():          # deepcopy keeps the instance forwards of base bound to base's modules
        m.__dict__.pop("forward", None)
    set_compute_dtype(fused, BF)
    fuse_offset_conv(fused)
    fuse_dcn_bn_relu(fused)
    assert I.fuse_ida_up(fused) == 8
    layout = {"out_cl": None}
    orig = I.ida_up_add

    def ida_up_add(p, weight, f, skip, channels_last=None):
        return orig(p, weight, f, skip, channels_last=layout["out_cl"] if layout["out_cl"] is not None else
                    channels_last)

    I.ida_up_add = ida_up_add
    try:
        for B in args.batches:
            x = neck_inputs(B, 128, dtype=BF, device="cuda")
            ref = None

            def arm(model, out_cl):
                def run():
                    layout["out_cl"] = out_cl
                    return model(x)
                return run

            arms = {"unfused": arm(base, None), "fused": arm(fused, None), "fused_cl": arm(fused, True)}
            err = {}
            with torch.no_grad():
                ref = arms["unfused"]()
                scale = ref.float().abs().max().item()
                for k, fn in arms.items():
                    err[k] = (fn().float() - ref.float()).abs().max().item() / scale
                times = {k: [] for k in arms}
                for _ in range(args.reps):
                    for k, fn in arms.items():
                        times[k].append(window(fn, args.window, args.warmup))
            ms = {k: statistics.median(v) for k, v in times.items()}
            row = {"B": B, "ms": ms, "speedup": ms["unfused"] / ms["fused"],
                   "speedup_cl": ms["unfused"] / ms["fused_cl"], "max_rel_diff_to_unfused": err}
            rows.append(row)
            print("chain B%-3d unfused %.3f ms  fused (skip layout) %.3f ms  x%.3f  fused (channels_last) %.3f ms  "
                  "x%.3f  max |diff| / max |y| %s" % (B, ms["unfused"], ms["fused"], row["speedup"],
                                                     ms["fused_cl"], row["speedup_cl"],
                                                     {k: "%.2e" % v for k, v in err.items()}), flush=True)
            assert max(err.values()) <= 2 ** -5
    finally:
        I.ida_up_add = orig
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for ida_up_time.json (created if missing)")
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16, 64])
    ap.add_argument("--window", type=float, default=1.0, help="seconds of each timed window")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-chain", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ida_up_time.py times the GPU; there is nothing to measure without one"
    name, power = card()
    print("card: %s, power limit %s" % (name, power), flush=True)
    result = {"card": name, "power_limit": power, "hbm_tbps_datasheet": HBM_TBPS, "ups": up_rows(args)}
    if not args.skip_chain:
        result["chain"] = chain_rows(args)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "ida_up_time.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

"""Times the ctdet decode on bf16 / fp16 heads read in place against the fp32 decode and against today's way of
decoding half heads (.float() casts, then the fp32 decode), with CUDA events after warm-up:

  f32            ctdet_decode on fp32 heads
  upcast_<dt>    ctdet_decode(heat.float(), wh.float(), reg.float()) on dt heads (the casts are timed)
  native_<dt>    ctdet_decode on dt heads (read in place)

for the bench workload (seed 317, B = 64, 80 x 128 x 128, K = 100, 3 rotating batches) as heat maps and as logits
(ctdet_decode_from_logits), for the class-sparse blob set of bench_secondary.py, at B = 1 and B = 8 (latency), and
ctdet_decode_from_host from pinned fp32 and pinned bf16 host buffers (B = 64).  The arms of a group are
alternated; each is timed over windows of at least --window seconds, --repeats times, to show the spread.  Reports
images/s, algorithmic bytes per image (80*128*128*s + 100*4*s + 100*24, s the element size of the heads) and the
share of the HBM peak (MEASURED_PEAKS.json, else 3.35 TB/s), asserts that the half and upcast arms' timed outputs
are bit-identical, and records the card and its power limit.  If native half is less than 1.5x faster than fp32
device-resident, a torch.profiler kernel table is added.  Writes DIR/decode_half_time.json.  GPU only."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from centernet_b200 import decode as D  # noqa: E402

C_, H_, W_, K_ = 80, 128, 128, 100
HALF = {"bf16": torch.bfloat16, "fp16": torch.float16}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001 - the numbers are still worth having without the card name
        return torch.cuda.get_device_name(), "unknown (%s)" % e


def hbm_peak_gbs():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]), "MEASURED_PEAKS.json"
    except Exception:  # noqa: BLE001
        return 3350.0, "H100 SXM data sheet (3.35 TB/s)"


def alg_bytes(s):
    """Bytes per image a decode must move at least: the heat map, the K gathered wh / reg pairs, the dets."""
    return C_ * H_ * W_ * s + K_ * 4 * s + K_ * 24


def synth(B, seed, device="cuda"):
    """bench.py's inputs: x = randn - 2.19 (the logits), heat = sigmoid(x), wh = rand * 32, reg = rand."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(B, C_, H_, W_, device=device, generator=g) - 2.19
    wh = torch.rand(B, 2, H_, W_, device=device, generator=g) * 32
    reg = torch.rand(B, 2, H_, W_, device=device, generator=g)
    return x, wh, reg


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


def time_group(arms, warmup, repeats, min_s):
    """arms: name -> callable.  Alternates the arms (rotating the order every repeat)."""
    names = list(arms)
    for n in names:
        for _ in range(warmup):
            arms[n]()
    torch.cuda.synchronize()
    runs = {n: [] for n in names}
    for r in range(repeats):
        for n in names[r % len(names):] + names[:r % len(names)]:
            runs[n].append(window(arms[n], min_s))
    return runs


def rotating(fn, batches, outs):
    """Closure that decodes the next batch of the rotation and keeps its (timed) output."""
    state = {"i": 0}

    def call():
        i = state["i"]
        outs[i] = fn(*batches[i])
        state["i"] = (i + 1) % len(batches)
    return call


def summarise(runs, B, elem, peak):
    out = {}
    for n, ms in runs.items():
        s = elem[n]
        best = min(ms)
        ips = B / (best * 1e-3)
        out[n] = {"ms_runs": [round(m, 5) for m in ms], "ms": round(best, 5),
                  "spread": round((max(ms) - min(ms)) / best, 4), "images_per_s": round(ips, 1),
                  "alg_bytes_per_image": alg_bytes(s), "hbm_share": round(ips * alg_bytes(s) / (peak * 1e9), 4)}
    return out


def arm_sets(batches32):
    """f32 / upcast / native arms over the same rounded values: the f32 arm decodes the fp32 originals."""
    sets = {"f32": batches32}
    for dt, tdt in HALF.items():
        half = [tuple(t.to(tdt) for t in b) for b in batches32]
        sets["upcast_" + dt] = half
        sets["native_" + dt] = half
    return sets


def arm_fn(fn, arm):
    """The decode an arm times: upcast arms cast every head to fp32 first."""
    if arm.startswith("upcast"):
        return lambda *t: fn(*[x.float() for x in t])
    return fn


def run_device(name, fn, sets, B, args, peak):
    outs = {n: [None] * len(b) for n, b in sets.items()}
    arms = {n: rotating(arm_fn(fn, n), b, outs[n]) for n, b in sets.items()}
    runs = time_group(arms, args.warmup, args.repeats, args.window)
    torch.cuda.synchronize()
    ident = {}
    for dt in HALF:
        same = all(torch.equal(a, b) for a, b in zip(outs["native_" + dt], outs["upcast_" + dt]))
        assert same, "%s: native %s differs from its upcast" % (name, dt)
        ident[dt] = same
    elem = {n: (4 if n == "f32" else 2) for n in sets}
    a = summarise(runs, B, elem, peak)
    res = {"B": B, "arms": a, "half_equals_upcast_bitwise": ident}
    for dt in HALF:
        res["speedup_%s_vs_f32" % dt] = round(a["f32"]["ms"] / a["native_" + dt]["ms"], 3)
        res["speedup_%s_vs_upcast" % dt] = round(a["upcast_" + dt]["ms"] / a["native_" + dt]["ms"], 3)
    print("%-10s B=%-3d " % (name, B) + "  ".join("%s %.3f ms (%.0f img/s, %.0f%% HBM)" % (
        n, v["ms"], v["images_per_s"], 100 * v["hbm_share"]) for n, v in a.items()), flush=True)
    return res, arms


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
    ap.add_argument("--out", required=True, help="directory for decode_half_time.json (created if missing)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0, help="seconds per timed window")
    args = ap.parse_args()
    name, power = card()
    peak, peak_src = hbm_peak_gbs()
    result = {"card": name, "power_limit": power, "hbm_peak_gbs": peak, "hbm_peak_source": peak_src,
              "workload": "seed 317, B=64, %dx%dx%d, K=%d, 3 rotating batches" % (C_, H_, W_, K_), "groups": {}}
    G = result["groups"]
    B = 64
    raw = [synth(B, 317 + i) for i in range(3)]
    heat32 = [(torch.sigmoid(x), wh, reg) for x, wh, reg in raw]
    G["heat"], arms_heat = run_device("heat", D.ctdet_decode, arm_sets(heat32), B, args, peak)
    G["logits"], _ = run_device("logits", D.ctdet_decode_from_logits, arm_sets(raw), B, args, peak)
    del raw
    from bench_secondary import blob_heat
    g = torch.Generator(device="cuda").manual_seed(317)
    blobs = [(blob_heat(B, C_, "cuda", g), heat32[0][1], heat32[0][2])]
    G["blobs"], _ = run_device("blobs", D.ctdet_decode, arm_sets(blobs), B, args, peak)
    del blobs
    for b in (1, 8):
        small = [tuple(t[i * b:(i + 1) * b].contiguous() for t in heat32[0]) for i in range(3)]
        G["latency_B%d" % b], _ = run_device("latency", D.ctdet_decode, arm_sets(small), b, args, peak)
    # host buffers (PCIe-bound): pinned fp32 vs pinned bf16, dets back in host memory
    host = {"f32": [tuple(t.cpu().pin_memory() for t in heat32[0])]}
    host["native_bf16"] = [tuple(t.to(torch.bfloat16).cpu().pin_memory() for t in heat32[0])]
    outs = {n: [None] for n in host}
    arms = {n: rotating(D.ctdet_decode_from_host, b, outs[n]) for n, b in host.items()}
    runs = time_group(arms, args.warmup, args.repeats, args.window)
    a = summarise(runs, B, {"f32": 4, "native_bf16": 2}, peak)
    for n in a:
        a[n].pop("hbm_share")
        a[n]["pcie_bytes_per_image"] = (C_ + 4) * H_ * W_ * (4 if n == "f32" else 2) + K_ * 24
    ref = D.ctdet_decode(*[t.to(torch.bfloat16) for t in heat32[0]]).cpu()
    assert torch.equal(outs["native_bf16"][0], ref)
    G["host_e2e"] = {"B": B, "arms": a, "half_equals_device_decode_bitwise": True,
                     "speedup_bf16_vs_f32": round(a["f32"]["ms"] / a["native_bf16"]["ms"], 3)}
    print("host_e2e   B=%-3d " % B + "  ".join("%s %.3f ms (%.0f img/s)" % (n, v["ms"], v["images_per_s"])
                                             for n, v in a.items()), flush=True)
    sp = min(G["heat"]["speedup_bf16_vs_f32"], G["heat"]["speedup_fp16_vs_f32"])
    if sp < 1.5:
        result["profile_heat_B64"] = {n: profile(arms_heat[n]) for n in ("f32", "native_bf16", "native_fp16")}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "decode_half_time.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("card: %s, power limit %s; wrote %s" % (name, power, path))


if __name__ == "__main__":
    main()

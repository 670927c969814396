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
device-resident, a torch.profiler kernel table is added.  Writes DIR/decode_half_time.json.  GPU only.

--task multi_pose (128 x 128, 17 joints, K = 100) and --task ddd (96 x 320, C = 3, K = 100) time, at B = 1, 8 and 64
(3 rotating batches of synthetic heads, seed 317):

  detector_f32         today's detector path on fp32 logits: torch's sigmoid of hm (and hm_hp; for ddd also the
                       depth transform 1. / (dep.sigmoid() + 1e-6) - 1.), then the fp32 decode
  logits_f32           *_decode_from_logits on the fp32 logits
  upcast_<dt>          a dt model today: the .float() casts of every head, then the detector path (casts timed)
  native_<dt>_logits   *_decode_from_logits on the dt heads, read in place
  heat_f32             the fp32 decode on fp32 heat maps (sigmoid / depth transform already applied)
  native_<dt>_heat     the decode on those heat maps rounded to dt, read in place

asserts that detector_f32 == logits_f32, upcast_<dt> == native_<dt>_logits and native_<dt>_heat == the decode of
its .float() upcast bit for bit in every timed call, and adds a torch.profiler kernel table at B = 64 and at every
batch size where a new arm is slower than the arm it replaces.  Writes DIR/decode_half_time_<task>.json.

--task exdet times exct_decode and agnex_ct_decode on five 80 x 128 x 128 maps and four regression maps (3 rotating
batches, seed 317, logits randn - 2.19) at K = 40 (B = 1 and 8) and K = 100 (B = 2), aggr_weight 0 and 0.1, with the
same six arms (detector_f32: torch's sigmoid of the five maps, detectors/exdet.py:32-36, then the fp32 decode; the
*_logits arms call *_decode_from_logits; the upcast arms cast all nine tensors), the same bit-identity asserts, the
algorithmic bytes per image (the five maps at s bytes each, plus, with aggregation, the four fp32 aggregated maps
written and read once) and their share of the HBM peak at K = 40, and a torch.profiler kernel table wherever a new arm
is slower than the arm it replaces.  Writes DIR/decode_half_time_exdet.json."""
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


POSE_J, DDD_C, HEAD_K = 17, 3, 100


def task_heads(task, B, seed, device="cuda"):
    """Synthetic raw head outputs: logits randn - 2.19 for the heat maps (as bench.py), uniform regressions."""
    g = torch.Generator(device=device).manual_seed(seed)

    def r(c, h, w, scale=1.0, shift=0.0):
        return torch.rand(B, c, h, w, device=device, generator=g) * scale + shift
    if task == "multi_pose":
        H, W, J = H_, W_, POSE_J
        hm = torch.randn(B, 1, H, W, device=device, generator=g) - 2.19
        wh, hps, reg = r(2, H, W, 40), r(2 * J, H, W, 24, -12), r(2, H, W)
        hm_hp = torch.randn(B, J, H, W, device=device, generator=g) - 2.19
        return [hm, wh, hps, reg, hm_hp, r(2, H, W)]
    H, W = 96, 320
    hm = torch.randn(B, DDD_C, H, W, device=device, generator=g) - 2.19
    rot = torch.randn(B, 8, H, W, device=device, generator=g)
    dep = torch.randn(B, 1, H, W, device=device, generator=g) * 2
    return [hm, rot, dep, r(3, H, W, 4), r(2, H, W, 60), r(2, H, W)]


def task_alg_bytes(task, s):
    """Bytes per image the decode must move at least: the score maps, the K gathered rows (multi_pose: wh, reg, kps and
    hp_offset at every (joint, candidate)), the dets.  multi_pose at s = 4 is DESIGN 4.2's 1,224,448 B."""
    if task == "multi_pose":
        return (1 + POSE_J) * H_ * W_ * s + HEAD_K * (72 * s + 4 * (6 + 2 * POSE_J))
    return DDD_C * 96 * 320 * s + HEAD_K * (16 * s + 4 * 18)


def task_fns(task):
    """(decode on heat maps, decode from logits, the detector's glue from logits to heat maps)."""
    if task == "multi_pose":
        def dec(hm, wh, hps, reg, hm_hp, off):
            return D.multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=off, K=HEAD_K)

        def dec_logits(hm, wh, hps, reg, hm_hp, off):
            return D.multi_pose_decode_from_logits(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=off, K=HEAD_K)

        def glue(hm, wh, hps, reg, hm_hp, off):   # detectors/multi_pose.py:33-35 (out of place: inputs are reused)
            return [hm.sigmoid(), wh, hps, reg, hm_hp.sigmoid(), off]
        return dec, dec_logits, glue

    def dec(hm, rot, dep, dim, wh, reg):
        return D.ddd_decode(hm, rot, dep, dim, wh=wh, reg=reg, K=HEAD_K)

    def dec_logits(hm, rot, dep, dim, wh, reg):
        return D.ddd_decode_from_logits(hm, rot, dep, dim, wh=wh, reg=reg, K=HEAD_K)

    def glue(hm, rot, dep, dim, wh, reg):         # detectors/ddd.py:61-62
        return [hm.sigmoid(), rot, 1. / (dep.sigmoid() + 1e-6) - 1., dim, wh, reg]
    return dec, dec_logits, glue


def run_task(task, args):
    name, power = card()
    peak, peak_src = hbm_peak_gbs()
    geom = ("%d joints, %dx%d" % (POSE_J, H_, W_)) if task == "multi_pose" else "C=%d, 96x320" % DDD_C
    result = {"card": name, "power_limit": power, "hbm_peak_gbs": peak, "hbm_peak_source": peak_src,
              "workload": "%s, seed 317, %s, K=%d, 3 rotating batches" % (task, geom, HEAD_K), "groups": {}}
    dec, dec_logits, glue = task_fns(task)
    for B in (1, 8, 64):
        raw = [task_heads(task, B, 317 + i) for i in range(3)]
        heat = [glue(*b) for b in raw]
        sets = {"detector_f32": raw, "logits_f32": raw, "heat_f32": heat}
        fns = {"detector_f32": lambda *t: dec(*glue(*t)), "logits_f32": dec_logits, "heat_f32": dec}
        elem = {"detector_f32": 4, "logits_f32": 4, "heat_f32": 4}
        for dt, tdt in HALF.items():
            half = [[t.to(tdt) for t in b] for b in raw]
            sets["upcast_" + dt] = half
            fns["upcast_" + dt] = lambda *t: dec(*glue(*[x.float() for x in t]))
            sets["native_%s_logits" % dt] = half
            fns["native_%s_logits" % dt] = dec_logits
            sets["native_%s_heat" % dt] = [[t.to(tdt) for t in b] for b in heat]
            fns["native_%s_heat" % dt] = dec
            elem.update({"upcast_" + dt: 2, "native_%s_logits" % dt: 2, "native_%s_heat" % dt: 2})
        outs = {n: [None] * 3 for n in sets}
        arms = {n: rotating(fns[n], sets[n], outs[n]) for n in sets}
        runs = time_group(arms, args.warmup, args.repeats, args.window)
        torch.cuda.synchronize()
        same = {"logits_f32 == detector_f32": all(map(torch.equal, outs["logits_f32"], outs["detector_f32"]))}
        for dt in HALF:
            same["native_%s_logits == upcast_%s" % (dt, dt)] = all(
                map(torch.equal, outs["native_%s_logits" % dt], outs["upcast_" + dt]))
            same["native_%s_heat == decode of its upcast" % dt] = all(
                torch.equal(o, dec(*[t.float() for t in b])) for o, b in zip(outs["native_%s_heat" % dt],
                                                                            sets["native_%s_heat" % dt]))
        assert all(same.values()), "%s B=%d: timed outputs differ: %s" % (task, B, same)
        a = {}
        for n, ms in runs.items():
            best = min(ms)
            ips = B / (best * 1e-3)
            a[n] = {"ms_runs": [round(m, 5) for m in ms], "ms": round(best, 5),
                    "spread": round((max(ms) - min(ms)) / best, 4), "images_per_s": round(ips, 1),
                    "alg_bytes_per_image": task_alg_bytes(task, elem[n]),
                    "hbm_share": round(ips * task_alg_bytes(task, elem[n]) / (peak * 1e9), 4)}
        # each new arm against the arm it replaces
        vs = {"logits_f32": "detector_f32", "heat_f32": None}
        for dt in HALF:
            vs.update({"native_%s_logits" % dt: "detector_f32", "upcast_" + dt: None,
                       "native_%s_heat" % dt: "heat_f32"})
        speed = {"%s vs %s" % (n, o): round(a[o]["ms"] / a[n]["ms"], 3) for n, o in vs.items() if o}
        speed.update({"native_%s_logits vs upcast_%s" % (dt, dt): round(a["upcast_" + dt]["ms"]
                                                                          / a["native_%s_logits" % dt]["ms"], 3)
                      for dt in HALF})
        g = {"B": B, "arms": a, "bitwise_identical": same, "speedups": speed}
        slower = [k.split(" vs ")[0] for k, v in speed.items() if v < 1.0]
        if B == 64 or slower:
            prof = set(slower) | {"detector_f32", "logits_f32", "native_bf16_logits", "upcast_bf16"}
            g["profile"] = {n: profile(arms[n]) for n in sorted(prof)}
        result["groups"]["B%d" % B] = g
        print("%-10s B=%-3d " % (task, B) + "  ".join("%s %.4f ms" % (n, v["ms"]) for n, v in a.items()), flush=True)
        print("           speedups: %s" % speed, flush=True)
        del raw, heat, sets, outs, arms
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "decode_half_time_%s.json" % task)
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("card: %s, power limit %s; wrote %s" % (name, power, path))


EX_C = 80


def exdet_inputs(B, seed, device="cuda"):
    """Logits of the t, l, b, r and centre maps (randn - 2.19, as bench.py's heat) and four uniform regressions."""
    g = torch.Generator(device=device).manual_seed(seed)
    maps = [torch.randn(B, EX_C, H_, W_, device=device, generator=g) - 2.19 for _ in range(5)]
    regs = [torch.rand(B, 2, H_, W_, device=device, generator=g) for _ in range(4)]
    return maps + regs


def exdet_alg_bytes(s, aggr):
    maps = EX_C * H_ * W_
    return 5 * maps * s + (4 * maps * 8 if aggr else 0) + 1000 * 14 * 4


def run_exdet(args):
    name, power = card()
    peak, peak_src = hbm_peak_gbs()
    result = {"card": name, "power_limit": power, "hbm_peak_gbs": peak, "hbm_peak_source": peak_src,
              "workload": "exdet, seed 317, 5 x %dx%dx%d maps + 4 regressions, num_dets=1000, 3 rotating batches"
                          % (EX_C, H_, W_), "groups": {}}
    for K, B in ((40, 1), (40, 8), (100, 2)):
        raw = [exdet_inputs(B, 317 + i) for i in range(3)]
        heat = [[torch.sigmoid(t) for t in b[:5]] + b[5:] for b in raw]
        for agnostic in (False, True):
            dec0 = D.agnex_ct_decode if agnostic else D.exct_decode
            dec0_logits = D.agnex_ct_decode_from_logits if agnostic else D.exct_decode_from_logits
            for aggr in (0.0, 0.1):
                kw = dict(K=K, aggr_weight=aggr)

                def dec(*t, _f=dec0, _kw=kw):
                    return _f(*t, **_kw)

                def dec_logits(*t, _f=dec0_logits, _kw=kw):
                    return _f(*t, **_kw)

                def detector(*t, _dec=dec):   # detectors/exdet.py:32-36 (out of place: the inputs are reused)
                    return _dec(*[torch.sigmoid(x) for x in t[:5]], *t[5:])
                sets = {"detector_f32": raw, "logits_f32": raw, "heat_f32": heat}
                fns = {"detector_f32": detector, "logits_f32": dec_logits, "heat_f32": dec}
                elem = {"detector_f32": 4, "logits_f32": 4, "heat_f32": 4}
                for dt, tdt in HALF.items():
                    half = [[t.to(tdt) for t in b] for b in raw]
                    sets["upcast_" + dt] = half
                    fns["upcast_" + dt] = lambda *t, _d=detector: _d(*[x.float() for x in t])
                    sets["native_%s_logits" % dt] = half
                    fns["native_%s_logits" % dt] = dec_logits
                    sets["native_%s_heat" % dt] = [[t.to(tdt) for t in b] for b in heat]
                    fns["native_%s_heat" % dt] = dec
                    elem.update({"upcast_" + dt: 2, "native_%s_logits" % dt: 2, "native_%s_heat" % dt: 2})
                outs = {n: [None] * 3 for n in sets}
                arms = {n: rotating(fns[n], sets[n], outs[n]) for n in sets}
                runs = time_group(arms, args.warmup, args.repeats, args.window)
                torch.cuda.synchronize()
                same = {"logits_f32 == detector_f32": all(map(torch.equal, outs["logits_f32"], outs["detector_f32"]))}
                for dt in HALF:
                    same["native_%s_logits == upcast_%s" % (dt, dt)] = all(
                        map(torch.equal, outs["native_%s_logits" % dt], outs["upcast_" + dt]))
                    same["native_%s_heat == decode of its upcast" % dt] = all(
                        torch.equal(o, dec(*[t.float() for t in b])) for o, b in zip(outs["native_%s_heat" % dt],
                                                                                    sets["native_%s_heat" % dt]))
                gname = "%s_K%d_B%d_aggr%g" % ("agnex" if agnostic else "exct", K, B, aggr)
                assert all(same.values()), "%s: timed outputs differ: %s" % (gname, same)
                a = {}
                for n, ms in runs.items():
                    best = min(ms)
                    ips = B / (best * 1e-3)
                    a[n] = {"ms_runs": [round(m, 5) for m in ms], "ms": round(best, 5),
                            "spread": round((max(ms) - min(ms)) / best, 4), "images_per_s": round(ips, 1),
                            "alg_bytes_per_image": exdet_alg_bytes(elem[n], aggr)}
                    if K == 40:   # memory-bound; at K = 100 the K^4 tuple stage dominates
                        a[n]["hbm_share"] = round(ips * exdet_alg_bytes(elem[n], aggr) / (peak * 1e9), 4)
                vs = {"logits_f32": "detector_f32"}
                for dt in HALF:
                    vs.update({"native_%s_logits" % dt: "detector_f32", "native_%s_heat" % dt: "heat_f32"})
                speed = {"%s vs %s" % (n, o): round(a[o]["ms"] / a[n]["ms"], 3) for n, o in vs.items()}
                speed.update({"native_%s_logits vs upcast_%s" % (dt, dt): round(
                    a["upcast_" + dt]["ms"] / a["native_%s_logits" % dt]["ms"], 3) for dt in HALF})
                g = {"K": K, "B": B, "aggr_weight": aggr, "agnostic": agnostic, "arms": a,
                     "bitwise_identical": same, "speedups": speed}
                slower = sorted({k.split(" vs ")[0] for k, v in speed.items() if v < 1.0})
                if slower:   # each slower arm and the arms it replaces
                    prof = set(slower) | {vs[n] for n in slower if n in vs}
                    prof |= {"upcast_" + n.split("_")[1] for n in slower if n.endswith("_logits")}
                    g["profile"] = {n: profile(arms[n]) for n in sorted(prof)}
                result["groups"][gname] = g
                print("%-24s " % gname + "  ".join("%s %.4f ms" % (n, v["ms"]) for n, v in a.items()), flush=True)
                print("           speedups: %s" % speed, flush=True)
                del sets, outs, arms
        del raw, heat
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "decode_half_time_exdet.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("card: %s, power limit %s; wrote %s" % (name, power, path))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for decode_half_time.json (created if missing)")
    ap.add_argument("--task", choices=("ctdet", "multi_pose", "ddd", "exdet"), default="ctdet")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0, help="seconds per timed window")
    args = ap.parse_args()
    if args.task == "exdet":
        return run_exdet(args)
    if args.task != "ctdet":
        return run_task(args.task, args)
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

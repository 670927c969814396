"""Times the device tails of the exdet and multi_pose detectors against the host tails they replace, on one GPU:

  device   exdet_merge_device / multi_pose_merge_device (one device->host copy)
  host     what detectors/exdet.py:85-122 and detectors/multi_pose.py:62-81 do: per image and scale the D2H copy of
           the decode output and post_process, then merge_outputs -- restated by tests/detector_tails_np.py, with the
           reference's compiled Cython soft_nms / soft_nms_39 from oracle/_ref (python -m oracle.build_ref)

Workloads (seed 317): exdet at B = 1 and B = 32, flip test, 1 and 5 test scales (0.5 - 1.5), exct_decode outputs
(num_dets 1000, K 40) of 80-class maps at 128 x 128 x scale; multi_pose at B = 64, one scale, K = 100, with and
without --nms.  Both tails start from the same decode outputs on the device; every timed pair of results is checked
to be equal bit for bit.  Also times the two top-K cuts (k_topk_keep's sort, k_topk_keep_wide's radix select) at
<= 4096 rows per image.  Prints per-image ms (median of --repeats calls after --warmup), the card name and its
power limit, and with --out DIR writes DIR/detector_tail_time.json.  GPU only.

--task ddd times the ddd tail instead: ddd_merge_device against what detectors/ddd.py:75-88 does per image (the D2H
copy of the decode output, ddd_post_process and merge_outputs), restated row by row by tests/ddd_tail_np.py, from the
same ddd_decode_from_logits outputs (seed 317, 3-class 96 x 320 heads, K = 100) at B = 1 and B = 32, KITTI metas
and one calibration per image; every timed pair of results is checked (bit for bit but alpha and rot_y, which must
agree within 2.5e-6 rad)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from centernet_b200 import decode as D  # noqa: E402
from centernet_b200 import post_process as P  # noqa: E402
from centernet_b200._lib import C, ptr, stream_ptr  # noqa: E402
from oracle import build_ref  # noqa: E402
import ddd_tail_cases as DC  # noqa: E402
import ddd_tail_np as DO  # noqa: E402
import detector_tails_np as O  # noqa: E402

F32 = np.float32


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        limit = "unknown (%s)" % e
    return name, limit


def metas_for(B, scales, seed):
    rng = np.random.default_rng(seed)
    c = [np.array([rng.uniform(200, 400), rng.uniform(150, 300)], F32) for _ in range(B)]
    s = [F32(rng.uniform(500, 700)) for _ in range(B)]
    return [{"c": [ci * F32(sc) for ci in c], "s": [F32(si * sc) for si in s], "out_height": int(128 * sc),
             "out_width": int(128 * sc), "scale": float(sc)} for sc in scales]


def host_exdet(dets, metas, nc, flip):
    p = 2 if flip else 1
    out = []
    for i in range(dets[0].shape[0] // p):
        per_scale = []
        for d, m in zip(dets, metas):
            h = d[p * i:p * i + p].cpu().numpy()             # the per-image, per-scale copy of detectors/exdet.py:87
            per_scale.append(O.exdet_post_process(h, {"c": m["c"][i], "s": m["s"][i], "out_width": m["out_width"],
                                                      "out_height": m["out_height"]}, m["scale"]))
        out.append(O.exdet_merge_outputs(per_scale, nc, 100))
    return out


def host_multi_pose(dets, metas, nms):
    out = []
    for i in range(dets[0].shape[0]):
        per_scale = []
        for d, m in zip(dets, metas):
            h = d[i].cpu().numpy()                           # the per-image, per-scale copy of multi_pose.py:63
            size = (m["out_width"], m["out_height"])
            bbox = O.affine_points(h[:, :4].reshape(-1, 2), m["c"][i], m["s"][i], size).reshape(-1, 4)
            pts = O.affine_points(h[:, 5:39].reshape(-1, 2), m["c"][i], m["s"][i], size).reshape(-1, 34)
            r = np.concatenate([bbox, h[:, 4:5], pts], axis=1).astype(F32)
            r[:, :4] /= F32(m["scale"]); r[:, 5:] /= F32(m["scale"])
            per_scale.append({1: r})
        out.append({1: O.multi_pose_merge_outputs(per_scale, nms or len(dets) > 1)[1].tolist()})
    return out


def same_exdet(a, b, nc):
    for x, y in zip(a, b):
        for j in range(1, nc + 1):
            u, v = np.asarray(x[j], F32), np.asarray(y[j], F32)
            if u.shape != v.shape or not np.array_equal(u, v, equal_nan=True):
                return False
    return len(a) == len(b)


def timed(fn, warmup, repeats):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, r


def exdet_dets(B, scales, flip, seed=317):
    g = torch.Generator().manual_seed(seed)
    out = []
    for sc in scales:
        h = w = int(128 * sc)
        n = (2 if flip else 1) * B
        maps = [torch.sigmoid(torch.randn(n, 80, h, w, generator=g) - 2.19).cuda() for _ in range(4)]
        ct = torch.sigmoid(torch.randn(n, 80, h, w, generator=g) - 2.19).cuda()
        out.append(D.exct_decode(*maps, ct, K=40, num_dets=1000))
        del maps, ct
    return out


def cut_times(warmup, repeats):
    """k_topk_keep (bitonic sort in shared memory) against k_topk_keep_wide (radix select) at <= 4096 rows."""
    res = []
    for n in (512, 2048, 4096):
        B, nc = 32, 80
        rng = np.random.default_rng(n)
        rows = torch.from_numpy(rng.uniform(0, 1, (B, n, 5)).astype(F32)).cuda()
        offs = torch.from_numpy(np.tile(np.linspace(0, n, nc + 1).astype(np.int32), (B, 1))).cuda()
        keeps = [torch.empty((B, n), dtype=torch.uint8, device="cuda") for _ in range(2)]
        arms = {"sort": lambda: C.topk_keep(ptr(rows), B, n, 5, ptr(offs), nc, 100, ptr(keeps[0]), 0, stream_ptr(rows)),
                "radix": lambda: C.topk_keep_wide(ptr(rows), B, n, 5, ptr(offs), nc, 100, ptr(keeps[1]), 0,
                                                  stream_ptr(rows))}
        row = {"rows": n, "images": B}
        for name, fn in arms.items():
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(repeats * 10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            row[name + "_us"] = e0.elapsed_time(e1) * 1e3 / (repeats * 10)
        assert torch.equal(keeps[0], keeps[1]), "the two cuts disagree at %d rows" % n
        res.append(row)
        print("cut %5d rows x %d images: sort %.1f us, radix %.1f us" % (n, B, row["sort_us"], row["radix_us"]))
    return res


def ddd_times(warmup, repeats):
    """ddd_merge_device against the per-image host tail, from the same decode outputs."""
    res = []
    for B in (1, 32):
        g = torch.Generator().manual_seed(317)
        H, W = DC.INPUT_HW[0] // 4, DC.INPUT_HW[1] // 4
        heads = [torch.randn(B, ch, H, W, generator=g).cuda() for ch in (DC.NUM_CLASSES, 8, 1, 3, 2, 2)]
        heads[3] = heads[3] * 0.3 + 1.5                                  # dims
        heads[4] = heads[4].abs() * 20                                   # wh
        dets = D.ddd_decode_from_logits(*heads, K=100)
        base = np.array([[707.0493, 0, 604.0814, 45.75831], [0, 707.0493, 180.5066, -0.3454157],
                         [0, 0, 1., 0.004981016]], F32)
        meta = {"c": [np.array([621.0, 187.5], F32)] * B, "s": [np.array([1242, 375], np.int32)] * B,
                "calib": [base + F32(i) * F32(0.25) for i in range(B)], "out_height": H, "out_width": W}

        def host():
            out = []
            for i in range(B):
                h = dets[i:i + 1].cpu().numpy()                  # the per-image copy of detectors/ddd.py:76
                r = DO.ddd_post_process(h, [meta["c"][i]], [meta["s"][i]], [meta["calib"][i]], W, H, DC.NUM_CLASSES)
                out.append(DO.merge_outputs(r[0], DC.NUM_CLASSES, DC.PEAK_THRESH))
            return out

        td, rd = timed(lambda: P.ddd_merge_device(dets, meta, DC.NUM_CLASSES, DC.PEAK_THRESH), warmup, repeats)
        th, rh = timed(host, min(warmup, 1), max(1, repeats // 2))
        DC.assert_ddd_equal(DC.flatten(rd), DC.flatten(rh), "ddd B=%d" % B)
        n = int(sum(len(r[j]) for r in rd for j in r))
        row = {"B": B, "K": 100, "rows_kept": n, "device_ms_per_image": td / B, "host_ms_per_image": th / B,
               "equal": True}
        res.append(row)
        print("ddd B=%d K=100: device %.3f ms/image, host %.3f ms/image, %d rows kept, equal True"
              % (B, td / B, th / B, n))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for detector_tail_time.json (default: print only)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--task", choices=("exdet_multi_pose", "ddd"), default="exdet_multi_pose")
    a = ap.parse_args()
    if a.task == "ddd":
        torch.cuda.set_device(0)
        name, limit = card()
        print("card: %s, power limit %s" % (name, limit))
        results = {"card": name, "power_limit": limit, "ddd": ddd_times(a.warmup, a.repeats)}
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "detector_tail_time_ddd.json"), "w") as f:
                json.dump(results, f, indent=1)
        return
    nms = build_ref.load_nms()
    if nms is None:
        sys.exit("oracle/_ref has no compiled reference soft_nms: run python -m oracle.build_ref where the reference "
                 "sources are")
    # the host tail runs the reference's compiled soft-NMS, as the detectors do
    O.soft_nms = lambda b, sigma=0.5, Nt=0.3, threshold=0.001, method=0, ncols_swap=0: \
        (nms.soft_nms_39 if ncols_swap else nms.soft_nms)(b, sigma=sigma, Nt=Nt, threshold=threshold, method=method)
    torch.cuda.set_device(0)
    name, limit = card()
    print("card: %s, power limit %s" % (name, limit))
    results = {"card": name, "power_limit": limit, "exdet": [], "multi_pose": []}
    for B, scales in ((1, (1.0,)), (1, (0.5, 0.75, 1.0, 1.25, 1.5)), (32, (1.0,)), (32, (0.5, 0.75, 1.0, 1.25, 1.5))):
        dets = exdet_dets(B, scales, True)
        metas = metas_for(B, scales, 7)
        td, rd = timed(lambda: P.exdet_merge_device(dets, metas, 80, flip=True), a.warmup, a.repeats)
        th, rh = timed(lambda: host_exdet(dets, metas, 80, True), min(a.warmup, 1), max(1, a.repeats // 2))
        ok = same_exdet(rd, rh, 80)
        row = {"B": B, "scales": len(scales), "flip": True, "rows_per_image": sum(2 * int(d.shape[1]) for d in dets),
               "device_ms_per_image": td / B, "host_ms_per_image": th / B, "equal": ok}
        results["exdet"].append(row)
        print("exdet B=%d S=%d flip: device %.3f ms/image, host %.3f ms/image, equal %s"
              % (B, len(scales), td / B, th / B, ok))
        assert ok, "device and host exdet tails differ"
        del dets
    g = torch.Generator().manual_seed(317)
    B = 64
    heat = torch.sigmoid(torch.randn(B, 1, 128, 128, generator=g) - 2.19).cuda()
    wh = (torch.rand(B, 2, 128, 128, generator=g) * 32).cuda()
    kps = (torch.randn(B, 34, 128, 128, generator=g) * 8).cuda()
    dets = [D.multi_pose_decode(heat, wh, kps, K=100)]
    metas = metas_for(B, (1.0,), 9)
    for use_nms in (False, True):
        td, rd = timed(lambda: P.multi_pose_merge_device(dets, metas, nms=use_nms), a.warmup, a.repeats)
        th, rh = timed(lambda: host_multi_pose(dets, metas, use_nms), min(a.warmup, 1), max(1, a.repeats // 2))
        ok = all(np.array_equal(np.asarray(x[1], F32), np.asarray(y[1], F32), equal_nan=True) for x, y in zip(rd, rh))
        results["multi_pose"].append({"B": B, "nms": use_nms, "device_ms_per_image": td / B,
                                      "host_ms_per_image": th / B, "equal": ok})
        print("multi_pose B=%d nms=%s: device %.3f ms/image, host %.3f ms/image, equal %s"
              % (B, use_nms, td / B, th / B, ok))
        assert ok, "device and host multi_pose tails differ"
    results["cut"] = cut_times(a.warmup, a.repeats)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "detector_tail_time.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

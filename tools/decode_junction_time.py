"""Where the fp32 bench call spends time outside its plane stream: per-CTA global-clock timestamps of k_select_hot over
back-to-back ctdet_decode calls on the bench workload (B = 64, 80x128x128, K = 100, 3 rotating batches).

Needs a library built with the statistics compiled in (they are NOT in the production build):
    CNB_NVCC_DEFINES=-DCNB_SELECT_STATS python centernet_b200/build.py --force
    python tools/decode_junction_time.py --out DIR

Every CTA records %globaltimer at entry, when its first stage is ready, when its last plane is swept and at exit
(after its closing flush / finalize).  Per call i (kernel i = the CTAs of launch i):
  call_us      entry(i+1) - entry(i), first CTA entry to first CTA entry: the steady-state period
  kernel_us    last CTA exit - first CTA entry
  gap_us       entry(i+1) - exit(i): idle stream between two kernels (negative: the launches overlap)
  ready_med_us / ready_max_us   per-CTA first-stage-ready time after its own entry (median, max)
  ready_spread_us               last CTA's first stage ready - first CTA entry
  tail_us      first CTA exit -> last CTA exit of kernel i (the window in which SMs of kernel i stop streaming)
  streaming_at_tail_start       CTAs of kernel i still sweeping planes when its first CTA exits
  tail_streaming_mean           CTAs sweeping planes (of kernel i, or of kernel i+1 once entered), averaged over
                                the tail window; the grid has n_cta (132) CTAs, so n_cta means no SM lost its stream
When consecutive launches overlap (programmatic dependent launch), call i+1's CTAs enter while call i still runs, so
gap_us is negative and kernel_us / tail_us span the wait of early CTAs for the previous call; call_us and the
streaming counts stay comparable.
Writes DIR/junction.json (medians + every call) and prints the median table.  %globaltimer ticks in steps of
`timer_step_ns` (reported); differences below that step are not resolved."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import B_PER_GPU, K, N_ROT, synth  # noqa: E402
import centernet_b200  # noqa: E402
from centernet_b200 import decode as D  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        return q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi failed: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=48, help="timed back-to-back calls (<= timestamp ring - 2)")
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    lib = ctypes.CDLL(os.path.join(os.path.dirname(centernet_b200.__file__), "lib", "libcenternet_b200.so"))
    if not hasattr(lib, "cnb_debug_select_times"):
        raise SystemExit("decode_junction_time: the library was built without -DCNB_SELECT_STATS")
    n_calls, ring, max_cta = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    lib.cnb_debug_select_times(None, ctypes.byref(n_calls), ctypes.byref(ring), ctypes.byref(max_cta))
    assert args.calls + 2 <= ring.value, "--calls exceeds the timestamp ring (%d)" % ring.value

    dev = torch.device("cuda", 0)
    batches = [synth(B_PER_GPU, dev, 317 + i) for i in range(N_ROT)]
    for i in range(6):
        D.ctdet_decode(*batches[i % N_ROT][:2], reg=batches[i % N_ROT][2], K=K)
    torch.cuda.synchronize()
    lib.cnb_debug_select_times(None, ctypes.byref(n_calls), ctypes.byref(ring), ctypes.byref(max_cta))
    first = n_calls.value
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.calls):
        D.ctdet_decode(*batches[i % N_ROT][:2], reg=batches[i % N_ROT][2], K=K)
    e1.record()
    torch.cuda.synchronize()
    ev_ms = e0.elapsed_time(e1) / args.calls
    buf = np.zeros((ring.value, max_cta.value, 4), np.uint64)
    assert lib.cnb_debug_select_times(buf.ctypes.data_as(ctypes.c_void_p), ctypes.byref(n_calls),
                                      ctypes.byref(ring), ctypes.byref(max_cta)) == 0
    assert n_calls.value - first == args.calls, "other hot launches ran in the timed window"
    plan = (ctypes.c_int * 9)()
    assert lib.cnb_select_plan_info(ctypes.c_void_p(batches[0][0].data_ptr()), B_PER_GPU, 80, 128, 128, K, 1, 4,
                                    plan, 9) == 0
    n_cta = plan[1]
    t = [buf[(first + i) % ring.value, :n_cta].astype(np.int64) for i in range(args.calls)]
    base = min(int(x[:, 0].min()) for x in t)
    t = [x - base for x in t]
    steps = np.diff(np.unique(np.concatenate([x.ravel() for x in t])))
    timer_step = int(steps[steps > 0].min()) if (steps > 0).any() else 0

    rows = []
    for i in range(args.calls - 1):
        a, b = t[i], t[i + 1]
        entry, ready, swept, exit_ = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
        t_in, t_out, t_first_out = entry.min(), exit_.max(), exit_.min()
        grid = np.linspace(t_first_out, t_out, 201)
        busy = ((grid[None, :] <= swept[:, None]).sum(0) +
                ((grid[None, :] >= b[:, 0][:, None]) & (grid[None, :] <= b[:, 2][:, None])).sum(0))
        rows.append({
            "call_us": (b[:, 0].min() - t_in) / 1e3,
            "kernel_us": (t_out - t_in) / 1e3,
            "gap_us": (b[:, 0].min() - t_out) / 1e3,
            "ready_med_us": float(np.median(ready - entry)) / 1e3,
            "ready_max_us": float((ready - entry).max()) / 1e3,
            "ready_spread_us": (ready.max() - t_in) / 1e3,
            "tail_us": (t_out - t_first_out) / 1e3,
            "streaming_at_tail_start": int((swept > t_first_out).sum()),
            "tail_streaming_mean": float(busy.mean()),
        })
    med = {k: float(np.median([r[k] for r in rows])) for k in rows[0]}
    res = {"label": args.label, "card": card(), "n_cta": n_cta, "calls": args.calls, "event_ms_per_call": ev_ms,
           "timer_step_ns": timer_step, "median": med, "per_call": [{k: float(v) for k, v in r.items()} for r in rows]}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "junction%s.json" % ("_" + args.label if args.label else "")), "w") as f:
        json.dump(res, f, indent=1)
    print("%s | %s | n_cta %d | events %.4f ms/call | globaltimer step %d ns" % (args.label, res["card"], n_cta, ev_ms,
                                                                                   timer_step))
    print("| " + " | ".join(med) + " |")
    print("| " + " | ".join("%.2f" % v for v in med.values()) + " |")


if __name__ == "__main__":
    main()

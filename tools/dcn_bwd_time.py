"""Times cnb_dcnv2_backward on the dla_34 DCN layer shapes (B=16): tensor-core path (with workspace) vs the fp32
CUDA-core path (workspace = NULL), checks the two against each other and that dOffset / dMask / dW of the
tensor-core path are bit-identical run to run.  GPU only."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centernet_b200._lib import C, ptr, stream_ptr, workspace

LAYERS = [(16, 64, 128, 128, 64), (16, 128, 64, 64, 128), (16, 256, 32, 32, 256), (16, 512, 16, 16, 256),
          (16, 128, 64, 64, 64), (16, 256, 32, 32, 128)]


def run(x, off, m, w, go, tc, want_dx=True):
    """tc=False: the fp32 CUDA-core path, which has no deterministic mode: the switch is off for that call."""
    det = C.dcnv2_get_deterministic()
    if not tc:
        C.dcnv2_set_deterministic(0)
    try:
        return _run(x, off, m, w, go, tc, want_dx)
    finally:
        C.dcnv2_set_deterministic(det)


def _run(x, off, m, w, go, tc, want_dx):
    B, Ci, H, W = x.shape
    Co = w.shape[0]
    gx = torch.zeros_like(x); goff = torch.zeros_like(off); gm = torch.zeros_like(m)
    gw = torch.zeros_like(w); gb = torch.zeros(Co, device=x.device)
    ws, wsb = 0, 0
    if tc:
        wsb = C.dcnv2_backward_workspace_bytes(B, Ci, Co, H, W, 3, 3, 1, 1, 1, 1)
        wsbuf = workspace(wsb, x.device); ws = ptr(wsbuf)
    C.dcnv2_backward(ptr(x), ptr(off), ptr(m), ptr(w), ptr(go), ptr(gx) if want_dx else 0, ptr(goff), ptr(gm), ptr(gw), ptr(gb),
                     B, Ci, H, W, Co, 3, 3, 1, 1, 1, 1, 1, 1, 1, ws, wsb, stream_ptr(x))
    return gx, goff, gm, gw, gb


def run_cl(xcl, off, m, w, go):
    """cnb_dcnv2_backward_ex: input and grad_input channels-last (no layout passes)."""
    B, Ci, H, W = xcl.shape
    Co = w.shape[0]
    gx = torch.zeros_like(xcl); goff = torch.zeros_like(off); gm = torch.zeros_like(m)
    gw = torch.zeros_like(w); gb = torch.zeros(Co, device=xcl.device)
    wsb = C.dcnv2_backward_workspace_bytes(B, Ci, Co, H, W, 3, 3, 1, 1, 1, 1)
    wsbuf = workspace(wsb, xcl.device)
    C.dcnv2_backward_ex(ptr(xcl), 1, ptr(off), ptr(m), ptr(w), ptr(go), ptr(gx), 1, ptr(goff), ptr(gm), ptr(gw), ptr(gb),
                        B, Ci, H, W, Co, 3, 3, 1, 1, 1, 1, ptr(wsbuf), wsb, stream_ptr(xcl))
    return gx, goff, gm, gw, gb


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, nargs="*", default=None, help="indices into LAYERS (default: all)")
    ap.add_argument("--quick", action="store_true", help="tensor-core path only, one call per layer (for ncu)")
    ap.add_argument("--deterministic", action="store_true", help="cnb_dcnv2_set_deterministic(1): fixed-point (order-independent) dX")
    ap.add_argument("--off-scale", type=float, default=1.5)
    ap.add_argument("--off-clamp", type=float, default=0.0, help="clamp the offsets to +-this (0 = no clamp)")
    args = ap.parse_args()
    torch.manual_seed(0)
    C.dcnv2_set_deterministic(int(args.deterministic))
    for li, (B, Ci, H, W, Co) in enumerate(LAYERS):
        if args.layers is not None and li not in args.layers:
            continue
        x = torch.randn(B, Ci, H, W, device="cuda")
        off = torch.randn(B, 18, H, W, device="cuda") * args.off_scale
        if args.off_clamp > 0:
            off = off.clamp(-args.off_clamp, args.off_clamp)
        m = torch.sigmoid(torch.randn(B, 9, H, W, device="cuda"))
        w = torch.randn(Co, Ci, 3, 3, device="cuda") / (3.0 * Ci ** 0.5)
        go = torch.randn(B, Co, H, W, device="cuda")
        a = run(x, off, m, w, go, True)
        if args.quick:
            torch.cuda.synchronize()
            continue
        a2 = run(x, off, m, w, go, True)
        r = run(x, off, m, w, go, False)
        torch.cuda.synchronize()
        errs = []
        for name, u, v in zip(("dx", "doff", "dmask", "dw", "db"), a, r):
            errs.append("%s %.2e/%.1f" % (name, (u - v).abs().max().item(), v.abs().max().item()))
        det = [bool((u == v).all().item()) for u, v in zip(a, a2)]
        t_tc = timeit(lambda: run(x, off, m, w, go, True))
        t_nodx = timeit(lambda: run(x, off, m, w, go, True, False))
        t_cl = float("nan")
        if Ci % 32 == 0:
            xcl = x.contiguous(memory_format=torch.channels_last)
            c = run_cl(xcl, off, m, w, go)
            errs.append("cl-dx %.2e" % (c[0] - r[0]).abs().max().item())
            t_cl = timeit(lambda: run_cl(xcl, off, m, w, go))
        t_fp = timeit(lambda: run(x, off, m, w, go, False), 3)
        print("B%d %d@%dx%d->%d  tc %.3f ms (without dX %.3f, channels-last %.3f)  fp32 %.3f ms | %s | bit-identical dx,doff,dmask,dw,db: %s"
              % (B, Ci, H, W, Co, t_tc, t_nodx, t_cl, t_fp, "  ".join(errs), det), flush=True)


if __name__ == "__main__":
    main()

"""Generates tests/golden/ref_gpu.npz: outputs of the UNMODIFIED reference DCNv2 / deformable-PSROI CUDA kernels
(oracle/_ref, built by `python -m oracle.build_ref` where the reference sources exist) for every case of
tests/test_ref_gpu.py.  Needs a GPU and oracle/_ref; the tests only read the .npz.

The inputs are rebuilt by the test from CPU seeds, so only reference outputs are stored: tensors of up to
SAMPLE elements whole, larger ones as a fixed, seeded sample of SAMPLE flat positions, plus the tensor's
max |value| (the scale the backward tolerances use).

    python tests/golden/make_golden_ref_gpu.py [OUT.npz]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import test_ref_gpu as T  # noqa: E402
from oracle import ref_gpu  # noqa: E402

SAMPLE = 1024


def put(store, key, t):
    a = t.detach().float().cpu().numpy().ravel()
    if a.size <= SAMPLE:
        idx = np.arange(a.size, dtype=np.int32)
    else:
        idx = np.sort(np.random.default_rng(len(store)).choice(a.size, SAMPLE, replace=False)).astype(np.int32)
    store[key + "/idx"] = idx
    store[key + "/val"] = a[idx]
    store[key + "/absmax"] = np.float32(np.abs(a).max() if a.size else 0.0)
    store[key + "/shape"] = np.array(t.shape, dtype=np.int64)


def main(path):
    store = {}
    torch.manual_seed(0)
    x = T.kat_input()
    N, C, H, W = x.shape
    w = torch.zeros(C, C, 3, 3)
    for i in range(C):
        w[i, i, 1, 1] = 1.0
    put(store, "kat", ref_gpu.dcn_v2_forward(x.cuda(), torch.zeros(N, 18, H, W, device="cuda"),
                                             torch.full((N, 9, H, W), 0.5, device="cuda"), w.cuda(),
                                             torch.zeros(C, device="cuda")) * 2)
    for case in T.LAYERS:
        cu = [t.cuda() for t in T.make(*case)]
        put(store, T.key("fwd", case), ref_gpu.dcn_v2_forward(*cu, case[-1], 1, 1, case[-2]))
    for case in T.FP32_LAYERS:
        cu = [t.cuda() for t in T.make(*case, seed=5)]
        put(store, T.key("fp32", case), ref_gpu.dcn_v2_forward(*cu, case[-1], 1, 1, case[-2]))
    for case in T.BWD_LAYERS:
        x, off, m, w, b, go = T.make_bwd(*case)
        cu = [t.cuda() for t in (x, off, m, w, b)]
        grads = ref_gpu.dcn_v2_backward(*cu, go.cuda(), case[-1], 1, 1, case[-2])
        for name, g in zip(T.GRAD_NAMES, grads):
            put(store, T.key("bwd_" + name, case), g)
    for case in T.PS_CASES:
        data, rois, trans, cfg = T._case(*case)
        d = torch.from_numpy(data).cuda(); r = torch.from_numpy(rois).cuda()
        t = torch.zeros(1, device="cuda") if trans is None else torch.from_numpy(trans).cuda()
        kw = T.ps_kwargs(cfg)
        out, cnt = ref_gpu.psroi_forward(d, r, t, **kw)
        go = torch.from_numpy(T.ps_grad(tuple(out.shape))).cuda()
        gi, gt = ref_gpu.psroi_backward(go, d, r, t, cnt, **kw)
        for name, v in (("out", out), ("cnt", cnt), ("gi", gi), ("gt", gt)):
            put(store, T.key("ps_" + name, case[:1]), v)
    torch.cuda.synchronize()
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes,", len(store) // 4, "tensors")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ref_gpu.npz"))

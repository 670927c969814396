"""Generates tests/golden/ref_gpu_f64.npz: outputs of the UNMODIFIED reference float64 DCNv2 / deformable-PSROI
CUDA kernels (the dcn_v2_double build; oracle/_ref/libdcnv2_ref_f64.so, built by `python -m oracle.build_ref_f64`
where the reference sources exist) for the float64 cases of tests/test_f64_gpu.py.  Needs a GPU and oracle/_ref;
the tests only read the .npz.

Same format as ref_gpu.npz, stored as float64: tensors of up to SAMPLE elements whole, larger ones as a fixed,
seeded sample of SAMPLE flat positions, plus the tensor's max |value| (the scale of the tolerances).

    python tests/golden/make_golden_ref_gpu_f64.py [OUT.npz]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import test_f64_gpu as T  # noqa: E402
from oracle import ref_gpu_f64  # noqa: E402

SAMPLE = 1024


def put(store, key, t):
    a = t.detach().double().cpu().numpy().ravel()
    if a.size <= SAMPLE:
        idx = np.arange(a.size, dtype=np.int32)
    else:
        idx = np.sort(np.random.default_rng(len(store)).choice(a.size, SAMPLE, replace=False)).astype(np.int32)
    store[key + "/idx"] = idx
    store[key + "/val"] = a[idx]
    store[key + "/absmax"] = np.float64(np.abs(a).max() if a.size else 0.0)
    store[key + "/shape"] = np.array(t.shape, dtype=np.int64)


def main(path):
    store = {}
    x, off, mask, w, b = [t.cuda() for t in T.kat_inputs()]
    put(store, "kat", ref_gpu_f64.dcn_v2_forward(x, off, mask, w, b) * 2)
    for case in T.LAYERS:
        cu = [t.cuda() for t in T._layer(*case, seed=0)]
        put(store, T.key("fwd", case), ref_gpu_f64.dcn_v2_forward(*cu, case[-1], 1, 1, case[-2]))
    for case in T.BWD_LAYERS:
        x, off, m, w, b, go = T.bwd_inputs(case)
        grads = ref_gpu_f64.dcn_v2_backward(*[t.cuda() for t in (x, off, m, w, b)], go.cuda(), case[-1], 1, 1,
                                            case[-2])
        for name, g in zip(T.GRAD_NAMES, grads):
            put(store, T.key("bwd_" + name, case), g)
    for case in T.PS_CASES:
        data, rois, trans, cfg = T._ps_case(*case)
        d = torch.from_numpy(data).cuda(); r = torch.from_numpy(rois).cuda()
        t = torch.zeros(1, device="cuda", dtype=torch.float64) if trans is None else torch.from_numpy(trans).cuda()
        kw = dict(spatial_scale=cfg["spatial_scale"], pooled_size=cfg["pooled_size"], output_dim=cfg["output_dim"],
                  no_trans=cfg["no_trans"], group_size=cfg["group_size"], part_size=cfg["part_size"],
                  sample_per_part=cfg["sample_per_part"], trans_std=cfg["trans_std"])
        out, cnt = ref_gpu_f64.psroi_forward(d, r, t, **kw)
        go = torch.from_numpy(T.ps_grad(tuple(out.shape))).cuda()
        gi, gt = ref_gpu_f64.psroi_backward(go, d, r, t, cnt, **kw)
        # the reference only prints a failed launch: an all-zero count means its kernels did not run
        assert cnt.max().item() > 0, "reference float64 PSROI kernels did not run"
        for name, v in (("out", out), ("cnt", cnt), ("gi", gi), ("gt", gt)):
            put(store, T.key("ps_" + name, case[:1]), v)
    torch.cuda.synchronize()
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes,", len(store) // 4, "tensors")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ref_gpu_f64.npz"))

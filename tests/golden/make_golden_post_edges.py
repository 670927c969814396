"""Generates tests/golden/post_edges.npz: the UNMODIFIED reference soft-NMS (src/lib/external/nms.pyx, compiled by
oracle/build_ref.py into oracle/_ref/) and post-processing (utils/post_process.py imported from the reference tree)
at the edges where the device kernels of csrc/post.cu branch: list lengths around the warp width, the 256-row
chunks of k_group_by_class and the former 1536-row shared-memory list size, up to 4096 rows; ties, exact-threshold
scores and overlaps, touching and degenerate boxes, +-inf / NaN scores and NaN coordinates; multi-scale merges
(detectors/ctdet.py:47-92) with per-image centres / scales, a class list over 1536 rows and 4096 rows per image.
Build container only; tests read the .npz.

    python tests/golden/make_golden_post_edges.py

Layout: `nms_names` lists the soft-NMS cases; case `k` has `k_in` (float32 [N, 5 or 39]), `k_out` (the whole
array as the reference leaves it in place, stale rows included), `k_n` (len(keep)) and `k_cfg` (float32 sigma,
Nt, threshold, method).  `merge_names` lists the merges; case `m` has `m_dets` (float32 [S, B, K, 6] decode
outputs), `m_c` (float32 [S, B, 2]), `m_s` (float32 [S, B, 2]; `m_s_scalar` [B] marks images whose scale is the
scalar m_s[..., 0]), `m_scales` (float64 [S]), `m_hw` (int [S, 2] output height, width), `m_cfg` (int:
num_classes, max_per_image, nms flag) and `m_out` (float32 [R, 7]: image, class id, x1, y1, x2, y2, score, in
image / class order).
"""
import os
import sys

import numpy as np

REF = "/root/reference/src/lib"
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from utils import post_process as P  # noqa: E402
from oracle import build_ref  # noqa: E402

nms = build_ref.load_nms()
assert nms is not None, "oracle/_ref nms module not built (python -m oracle.build_ref, where the reference exists)"

F32 = np.float32
NAN_NEG = np.array([0xffc00000], np.uint32).view(F32)[0]    # the x86 default NaN (sign bit set)
NAN_POS = np.array([0x7fc00000], np.uint32).view(F32)[0]


def clustered(rng, n, extra=0, size=512.0, grid=0.5):
    """Boxes on a `grid` lattice (compressible, exact differences), a quarter of them in clusters of three so that
    decays and discards both happen; scores in (0.0005, 1)."""
    x = rng.uniform(0, size - 40, n); y = rng.uniform(0, size - 40, n)
    k = n // 4
    x[:k * 3] = np.repeat(x[:k], 3) + rng.uniform(-6, 6, k * 3)
    y[:k * 3] = np.repeat(y[:k], 3) + rng.uniform(-6, 6, k * 3)
    w = rng.uniform(8, 120, n); h = rng.uniform(8, 120, n)
    q = lambda v: np.round(v / grid) * grid
    x, y, w, h = q(x), q(y), q(w), q(h)
    s = rng.uniform(0.0005, 1.0, n)
    cols = [x, y, x + w, y + h, s] + [np.round(rng.uniform(0, size, n)) for _ in range(extra)]
    return np.stack(cols, 1).astype(F32)


def nms_cases(rng):
    """(name, boxes, sigma, Nt, threshold, method)."""
    cases = []
    short = (1, 2, 31, 32, 33, 64, 65, 255, 256, 257)
    for n in short:                                      # every method at every short length
        for method, Nt in ((0, 0.3), (1, 0.3), (2, 0.5)):
            cases.append(("len%d_m%d" % (n, method), clustered(rng, n), 0.5, Nt, 0.001, method))
    for n, method, Nt in ((1535, 2, 0.5), (1536, 1, 0.3), (1537, 0, 0.3), (2048, 2, 0.5), (4096, 2, 0.5)):
        cases.append(("len%d_m%d" % (n, method), clustered(rng, n), 0.5, Nt, 0.001, method))
    # non-default sigma / threshold, threshold 0 (a weight of 0 leaves a score of 0, which is kept)
    cases.append(("sigma_thr", clustered(rng, 200), 0.1, 0.5, 0.05, 2))
    b = clustered(rng, 120); b[::7, 4] *= -1                 # negative scores next to threshold 0
    for method in (0, 1, 2):
        cases.append(("thr0_m%d" % method, b.copy(), 0.5, 0.3, 0.0, method))
    # equal scores split across lanes: ten levels, so every arg-max has ties in several lanes
    b = clustered(rng, 200); b[:, 4] = (rng.integers(1, 11, 200) / 10).astype(F32)
    for method in (0, 2):
        cases.append(("ties_m%d" % method, b.copy(), 0.5, 0.3, 0.001, method))
    b = clustered(rng, 70); b[:, 4] = F32(0.5)
    for method in (0, 1, 2):
        cases.append(("alleq_m%d" % method, b.copy(), 0.5, 0.3, 0.001, method))
    # duplicates: 40 boxes repeated 2-5 times (IoU 1), so discards copy in rows that are discarded in turn
    base = clustered(rng, 40)
    b = np.repeat(base, rng.integers(2, 6, 40), axis=0)
    b = b[rng.permutation(len(b))]; b[:, 4] = rng.uniform(0.01, 1, len(b)).astype(F32)
    for method in (0, 1, 2):
        cases.append(("dups_m%d" % method, b.copy(), 0.5, 0.3, 0.001, method))
    # touching boxes: 10-wide cells on a 10 grid give iw = 0 / ih = 0 exactly; every third cell grows by one (iw 1)
    gx, gy = np.meshgrid(np.arange(8) * 10.0, np.arange(8) * 10.0)
    x1, y1 = gx.ravel(), gy.ravel()
    grow = (np.arange(64) % 3 == 0).astype(np.float64)
    b = np.stack([x1, y1, x1 + 9 + grow, y1 + 9 + grow[::-1], rng.uniform(0.1, 1, 64)], 1).astype(F32)
    for method in (0, 1):
        cases.append(("touch_m%d" % method, b.copy(), 0.5, 0.3, 0.001, method))
    # overlap exactly Nt: A = [0,0,9,9] (area 100) against B = [0,0,9,19] (IoU 100/200 = 0.5) and against
    # C = [5,0,14,9] (IoU 50/150, the float32 of 1/3 as Nt is)
    rows = []
    for k in range(12):
        ox, oy = 40.0 * k, 0.0
        rows += [[ox, oy, ox + 9, oy + 9, 0.9 - 0.01 * k], [ox, oy, ox + 9, oy + 19, 0.8 - 0.01 * k],
                 [ox + 5, oy + 30, ox + 14, oy + 39, 0.7], [ox, oy + 30, ox + 9, oy + 39, 0.75]]
    b = np.array(rows, F32)
    for method, Nt in ((0, 0.5), (1, 0.5), (0, 1.0 / 3.0), (1, 1.0 / 3.0)):
        cases.append(("ovnt_m%d_%s" % (method, "half" if Nt == 0.5 else "third"), b.copy(), 0.5, Nt, 0.001, method))
    # score exactly at the threshold: IoU 0.5 > Nt 0.3 under method 1 halves 0.5 to 0.25 (kept at threshold
    # 0.25) and 0.49 to 0.245 (dropped); untouched scores of exactly 0.25 stay
    rows = []
    for k in range(10):
        ox = 40.0 * k
        rows += [[ox, 0, ox + 9, 9, 0.95], [ox, 0, ox + 9, 19, 0.5 if k % 2 else 0.49], [ox, 100, ox + 9, 109, 0.25]]
    cases.append(("thr_exact", np.array(rows, F32), 0.5, 0.3, 0.25, 1))
    # degenerate boxes (x2 < x1 and / or y2 < y1)
    b = clustered(rng, 100)
    f = rng.random(100) < 0.3; b[f, 0], b[f, 2] = b[f, 2].copy(), b[f, 0].copy()
    f = rng.random(100) < 0.3; b[f, 1], b[f, 3] = b[f, 3].copy(), b[f, 1].copy()
    for method in (0, 2):
        cases.append(("degen_m%d" % method, b.copy(), 0.5, 0.3, 0.001, method))
    # +-inf scores: inf * weight 0 is NaN (kept: NaN < threshold is false)
    b = clustered(rng, 60); b[[3, 17, 40], 4] = np.inf; b[[5, 33], 4] = -np.inf
    for method in (0, 1, 2):
        cases.append(("inf_m%d" % method, b.copy(), 0.5, 0.3, 0.001, method))
    # NaN scores: never chosen as the pivot, except where the scan starts on one
    b = clustered(rng, 50); b[[7, 20, 41], 4] = NAN_NEG
    cases.append(("nanscore_m2", b.copy(), 0.5, 0.5, 0.001, 2))
    b2 = b.copy(); b2[0, 4] = NAN_POS; b2[30, 4] = np.inf
    for method in (0, 1):
        cases.append(("nanscore0_m%d" % method, b2.copy(), 0.5, 0.3, 0.001, method))
    # NaN coordinates: min(a, NaN) is NaN in nms.pyx, so the pair does not overlap
    b = np.array([[10, 10, 60, 60, 0.9], [12, 11, 61, np.nan, 0.8], [11, np.nan, 59, 62, 0.7], [9, 12, 58, 59, 0.6]], F32)
    cases.append(("nancoord4_m2", b, 0.5, 0.5, 0.001, 2))
    b = clustered(rng, 48)
    for col in range(4):
        b[rng.choice(48, 3, replace=False), col] = NAN_NEG
    for method in (0, 2):
        cases.append(("nancoord_m%d" % method, b.copy(), 0.5, 0.3, 0.001, method))
    # soft_nms_39: many discards, so swapped extra columns and copied box columns part ways
    cases.append(("s39_hard", clustered(rng, 160, extra=34, size=256.0), 0.5, 0.3, 0.001, 0))
    cases.append(("s39_gauss", clustered(rng, 96, extra=34, size=256.0), 0.5, 0.5, 0.3, 2))
    return cases


def decode_like(rng, B, K, num_classes, out_hw, levels=None, disjoint=False):
    """[B, K, 6] ctdet_decode-shaped detections on the output grid: scores descending, integer class ids."""
    oh, ow = out_hw
    d = np.zeros((B, K, 6), F32)
    if disjoint:      # cells of a lattice that never overlap, so soft-NMS leaves every score alone
        side = int(np.ceil(np.sqrt(K)))
        cell = np.arange(K)
        d[..., 0] = (cell % side) * 4.0; d[..., 1] = (cell // side) * 4.0
        d[..., 2] = d[..., 0] + 1.5; d[..., 3] = d[..., 1] + 1.5
    else:
        d[..., 0] = rng.uniform(-2, ow, (B, K)); d[..., 1] = rng.uniform(-2, oh, (B, K))
        k = K // 3
        d[:, :k * 2, 0] = np.repeat(d[:, :k, 0], 2, axis=1) + rng.uniform(-1, 1, (B, 2 * k))
        d[:, :k * 2, 1] = np.repeat(d[:, :k, 1], 2, axis=1) + rng.uniform(-1, 1, (B, 2 * k))
        d[..., 2] = d[..., 0] + rng.uniform(1, 24, (B, K)); d[..., 3] = d[..., 1] + rng.uniform(1, 24, (B, K))
    if levels is None:
        sc = rng.uniform(0.0, 1.0, (B, K))
    else:
        sc = rng.integers(1, levels + 1, (B, K)) / levels
    d[..., 4] = np.sort(sc, axis=1)[:, ::-1]
    d[..., 5] = rng.integers(0, num_classes, (B, K))
    return d


def ref_merge(dets, c, s, s_scalar, scales, hw, num_classes, max_per_image, run_nms):
    """detectors/ctdet.py:47-58 (post_process) per image and scale, then :76-92 (merge_outputs) with the compiled
    reference soft_nms.  Returns the flat [R, 7] rows."""
    S, B = dets.shape[0], dets.shape[1]
    flat = []
    for i in range(B):
        detections = []
        for k in range(S):
            si = F32(s[k, i, 0]) if s_scalar[i] else s[k, i].copy()
            r = P.ctdet_post_process(dets[k, i:i + 1].copy(), [c[k, i]], [si], int(hw[k, 0]), int(hw[k, 1]),
                                     num_classes)[0]
            for j in range(1, num_classes + 1):
                r[j] = np.array(r[j], dtype=F32).reshape(-1, 5)
                r[j][:, :4] /= float(scales[k])
            detections.append(r)
        results = {}
        for j in range(1, num_classes + 1):
            results[j] = np.concatenate([d[j] for d in detections], axis=0).astype(F32)
            if run_nms:
                nms.soft_nms(results[j], Nt=0.5, method=2)
        scores = np.hstack([results[j][:, 4] for j in range(1, num_classes + 1)])
        if len(scores) > max_per_image:
            kth = len(scores) - max_per_image
            thresh = np.partition(scores, kth)[kth]
            for j in range(1, num_classes + 1):
                results[j] = results[j][results[j][:, 4] >= thresh]
        for j in range(1, num_classes + 1):
            a = results[j]
            flat.append(np.concatenate([np.full((len(a), 1), i, F32), np.full((len(a), 1), j, F32), a], 1))
    return np.concatenate(flat, 0)


def merge_cases(rng):
    """(name, scales, B, K, num_classes, max_per_image, nms, levels, disjoint)."""
    return [("scales5", (0.5, 0.75, 1.0, 1.25, 1.5), 3, 100, 80, 100, 1, None, False),
            ("nc1_long", (1.0, 1.25), 2, 800, 1, 100, 1, None, False),       # one class list of 1600 rows
            ("n4096", (0.5, 0.75, 1.0, 1.25), 1, 1024, 2, 100, 1, None, False),
            ("ties", (0.75, 1.0), 3, 100, 80, 100, 1, 8, True),             # ties at the max_per_image cut
            ("ties_nonms", (1.0,), 3, 300, 80, 100, 0, 6, False)]


def main():
    rng = np.random.default_rng(20261016)
    out = {}
    names = []
    for name, b, sigma, Nt, thr, method in nms_cases(rng):
        a = b.copy()
        fn = nms.soft_nms_39 if b.shape[1] == 39 else nms.soft_nms
        keep = fn(a, sigma=sigma, Nt=Nt, threshold=thr, method=method)
        out[name + "_in"] = b; out[name + "_out"] = a; out[name + "_n"] = np.int64(len(keep))
        out[name + "_cfg"] = np.array([sigma, Nt, thr, method], F32)
        names.append(name)
    out["nms_names"] = np.array(names)
    mnames = []
    for name, scales, B, K, nc, mpi, run_nms, levels, disjoint in merge_cases(rng):
        S = len(scales)
        base_c = np.stack([rng.uniform(150, 400, B), rng.uniform(100, 300, B)], 1)
        base_s = np.stack([rng.uniform(480, 800, B), rng.uniform(360, 640, B)], 1)
        s_scalar = np.arange(B) % 2 == 0                 # scalar max(h, w) scales and --keep_res vector scales
        base_s[s_scalar, 1] = base_s[s_scalar, 0]
        hw = np.array([[int(round(128 * sc)), int(round(128 * sc)) + 32] for sc in scales], np.int64)
        c = np.stack([base_c * sc for sc in scales], 0).astype(F32)
        s = np.stack([base_s * sc for sc in scales], 0).astype(F32)
        dets = np.stack([decode_like(rng, B, K, nc, hw[k], levels, disjoint) for k in range(S)], 0)
        res = ref_merge(dets, c, s, s_scalar, scales, hw, nc, mpi, run_nms)
        out.update({name + "_dets": dets, name + "_c": c, name + "_s": s, name + "_s_scalar": s_scalar,
                    name + "_scales": np.array(scales, np.float64), name + "_hw": hw,
                    name + "_cfg": np.array([nc, mpi, run_nms], np.int64), name + "_out": res})
        mnames.append(name)
    out["merge_names"] = np.array(mnames)
    path = os.path.join(HERE, "post_edges.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(names), "soft-NMS lists,", len(mnames), "merges")


if __name__ == "__main__":
    main()

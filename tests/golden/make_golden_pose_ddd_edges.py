"""Generates tests/golden/pose_ddd_edges.npz by running the UNMODIFIED reference's models/decode.py
(multi_pose_decode, ddd_decode) on CPU torch, on small hand-built maps that each sit on one branch of the
keypoint assembly (decode.py:527-567) or of the ddd gathers (:426-462).

Run in the build container only:  python tests/golden/make_golden_pose_ddd_edges.py
The GPU box has no /root/reference; tests read the committed .npz.

multi_pose cases (16x16 maps, one image, the "subject" detection at pixel (8, 8)):
* joint score exactly float32(0.1) and one ulp either side (the `> 0.1` mask and the `< 0.1` reject);
* a candidate exactly on each box edge, and one ulp outside it (the four strict box tests);
* min_dist exactly equal to fl(fl(max(b - t, r - l)) * 0.3f) and one ulp either side, with a 3-4-5 distance
  scaled by a power of two and the box width searched in float32;
* equidistant candidates (the first one in top-K order must win) and masked candidates that all sit at
  (-10000, -10000);
* a zero-size box with the candidate at distance 0, and a box of negative size;
* every joint below the threshold, K larger than the number of joint peaks, K = 1;
* all six valid combinations of the optional heads reg, hm_hp and hp_offset;
* NaN, +inf and -inf, one per case, in the kps x / y, wh w / h and reg x / y of the subject, and in the
  hp_offset x of an above-threshold and of a below-threshold joint candidate.
ddd cases: C = 1 and 3, with and without wh / reg, every pixel selected (K = H*W), NaN and inf in rot, depth,
dim, wh and reg (gathered unchanged).

Every case is checked here: its centre and joint scores are tie-free among the positive ones, and the centre map
has at least K positive peaks, so the detections do not depend on torch.topk's order of equal scores (the zero
joint fillers all become the identical candidate (-1, -10000, -10000)).  The one exception is the ddd cases that
select every pixel: their zero-score rows are a fixed set whose order is open, so tests compare them tie-aware.
"""
import os
import sys

import numpy as np
import torch

REF = "/root/reference/src/lib"
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))

from models import decode as R  # noqa: E402

F32 = np.float32
U32 = np.uint32
HW = 16
DECOYS = [(1, x) for x in (1, 4, 7, 10, 13)] + [(14, x) for x in (1, 4, 7, 10, 13)]
OUT = {}


def up(x):
    return np.nextafter(F32(x), F32(np.inf))


def dn(x):
    return np.nextafter(F32(x), F32(-np.inf))


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def positive_peaks(m):
    """[N, C, H, W] -> per (n, c) plane, the positive values of the reference's _nms."""
    n = R._nms(t(m)).numpy()
    return [p[p > 0] for p in n.reshape(-1, n.shape[2] * n.shape[3])]


def check_tie_free(m, what):
    for p in positive_peaks(m):
        assert len(np.unique(p)) == len(p), "ties in " + what


def store(name, arrays, dets):
    for k, v in arrays.items():
        if v is not None:
            OUT[name + "__" + k] = np.asarray(v)
    OUT[name + "__dets"] = dets


class Pose(object):
    def __init__(self, J=1):
        self.J = J
        self.heat = np.zeros((1, 1, HW, HW), F32)
        self.wh = np.zeros((1, 2, HW, HW), F32)
        self.kps = np.zeros((1, 2 * J, HW, HW), F32)
        self.reg = np.zeros((1, 2, HW, HW), F32)
        self.hm_hp = np.zeros((1, J, HW, HW), F32)
        self.off = np.zeros((1, 2, HW, HW), F32)

    def det(self, y, x, score, wh=(6.0, 5.0), reg=(0.25, 0.25), kps=None):
        """A centre peak; kps are the regressed joint locations (x, y) (decode.py:506-509 adds the integer centre)."""
        self.heat[0, 0, y, x] = score
        self.wh[0, :, y, x] = wh
        self.reg[0, :, y, x] = reg
        for j in range(self.J):
            kx, ky = kps[j] if kps else (x, y)
            self.kps[0, 2 * j, y, x] = F32(kx) - F32(x)
            self.kps[0, 2 * j + 1, y, x] = F32(ky) - F32(y)
            assert self.kps[0, 2 * j, y, x] + F32(x) == F32(kx) and self.kps[0, 2 * j + 1, y, x] + F32(y) == F32(ky)

    def decoys(self, n):
        for i, (y, x) in enumerate(DECOYS[:n]):
            self.det(y, x, F32(0.3 - 0.01 * i), wh=(2.0, 2.0), reg=(0.5, 0.5))

    def cand(self, j, xy, score):
        """A joint peak whose hp_offset puts the candidate exactly at xy."""
        x, y = F32(xy[0]), F32(xy[1])
        px, py = int(np.floor(x)), int(np.floor(y))
        self.hm_hp[0, j, py, px] = score
        self.off[0, :, py, px] = (x - F32(px), y - F32(py))
        assert F32(px) + self.off[0, 0, py, px] == x and F32(py) + self.off[0, 1, py, px] == y
        return py, px

    def finish(self, name, K, reg=True, hp=True, off=True):
        assert not off or hp
        check_tie_free(self.heat, name + " heat")
        assert sum(len(p) for p in positive_peaks(self.heat)) >= K, name + ": fewer than K centre peaks"
        if hp:
            check_tie_free(self.hm_hp, name + " hm_hp")
        heads = dict(heat=self.heat, wh=self.wh, kps=self.kps, reg=self.reg if reg else None,
                     hm_hp=self.hm_hp if hp else None, hp_offset=self.off if off and hp else None)
        with torch.no_grad():
            dets = R.multi_pose_decode(t(self.heat), t(self.wh), t(self.kps.copy()),
                                       reg=t(self.reg) if reg else None, hm_hp=t(self.hm_hp) if hp else None,
                                       hp_offset=t(self.off) if off and hp else None, K=K).numpy()
        store(name, heads, dets)
        OUT[name + "__K"] = np.int64(K)
        return dets


def subject_box():
    """The subject's box in float32, as decode.py:519-522 computes it: reg (0.25, 0.25), wh (6, 5)."""
    xs, ys = F32(8) + F32(0.25), F32(8) + F32(0.25)
    return xs - F32(3), ys - F32(2.5), xs + F32(3), ys + F32(2.5)   # 5.25, 5.75, 11.25, 10.75


def pose_cases():
    names = []

    def add(name, p, K, **kw):
        p.finish(name, K, **kw)
        names.append(name)
        return name

    # ---- the two thresholds (:544 mask = hm_score > 0.1, :564 hm_score < 0.1)
    for tag, s in (("eq", F32(0.1)), ("up", up(0.1)), ("dn", dn(0.1))):
        p = Pose()
        p.det(8, 8, 0.9, kps=[(8.75, 8.5)])
        p.decoys(2)
        p.cand(0, (8.5, 8.5), s)
        add("thr_" + tag, p, 3)

    # ---- box edges: on the edge is inside (strict tests), one ulp outside is not
    l, tp, r, b = subject_box()
    edges = {"l": ((l, F32(8.25)), (l + F32(0.5), F32(8.25)), (dn(l), F32(8.25))),
             "r": ((r, F32(8.25)), (r - F32(0.5), F32(8.25)), (up(r), F32(8.25))),
             "t": ((F32(8.25), tp), (F32(8.25), tp + F32(0.5)), (F32(8.25), dn(tp))),
             "b": ((F32(8.25), b), (F32(8.25), b - F32(0.5)), (F32(8.25), up(b)))}
    for e, (on, kp, out) in edges.items():
        for tag, c in (("on", on), ("out", out)):
            p = Pose()
            p.det(8, 8, 0.9, kps=[kp])
            p.decoys(2)
            p.cand(0, c, 0.5)
            add("box_%s_%s" % (e, tag), p, 3)

    # ---- the distance limit: dist = 5 exactly (dx = 3, dy = 4) against limit = fl(fl(r - l) * 0.3f), w searched
    # in float32 (the product steps by about 1.2 ulps, so the box centre is chosen where D and both neighbours occur)
    D = F32(5.0)
    xs = ys = F32(7.0)                                          # subject at pixel (7, 7), reg (0, 0)
    h = F32(2.0)
    ws = np.arange(F32(16.0).view(U32), F32(17.2).view(U32), dtype=U32).view(F32)
    half = ws / F32(2)
    ext = np.maximum((ys + h / F32(2)) - (ys - h / F32(2)), (xs + half) - (xs - half))
    lim = ext * F32(0.3)
    lim_mut = ext * up(0.3)                                     # the limit were 0.3f one ulp larger
    picks = {"eq": ws[lim == D][0], "above": ws[lim == up(D)][0],
             "below": ws[(lim == dn(D)) & (lim_mut >= D)][0]}   # a larger constant would accept it
    for tag, w in picks.items():
        p = Pose()
        p.det(7, 7, 0.9, wh=(w, h), reg=(0.0, 0.0), kps=[(4.0, 3.0)])
        p.decoys(2)
        p.cand(0, (7.0, 7.0), 0.5)
        add("dist_lim_" + tag, p, 3)
    # the same with the height as the larger side
    ext = np.maximum((ys + half) - (ys - half), (xs + h / F32(2)) - (xs - h / F32(2)))
    w = ws[ext * F32(0.3) == D][0]
    p = Pose()
    p.det(7, 7, 0.9, wh=(h, w), reg=(0.0, 0.0), kps=[(3.0, 4.0)])
    p.decoys(2)
    p.cand(0, (7.0, 7.0), 0.5)
    add("dist_lim_eq_h", p, 3)

    # ---- equal distances: the first candidate in top-K order (higher score, higher pixel index) must win
    for tag, a, b_ in (("x", (7.25, 8.25), (9.25, 8.25)), ("y", (8.25, 7.25), (8.25, 9.25))):
        p = Pose()
        p.det(8, 8, 0.9, wh=(8.0, 8.0), kps=[(8.25, 8.25)])
        p.decoys(2)
        p.cand(0, a, 0.5)
        p.cand(0, b_, 0.6)
        add("dist_tie_" + tag, p, 3)

    # ---- degenerate boxes
    p = Pose()
    p.det(8, 8, 0.9, wh=(0.0, 0.0), kps=[(8.25, 8.25)])
    p.decoys(2)
    p.cand(0, (8.25, 8.25), 0.5)
    add("box_zero", p, 3)
    p = Pose()
    p.det(8, 8, 0.9, wh=(-2.0, -2.0), kps=[(8.5, 8.25)])
    p.decoys(2)
    p.cand(0, (8.25, 8.25), 0.5)
    add("box_negative", p, 3)

    # ---- every joint below the threshold: all candidates masked to (-10000, -10000), all distances tie
    p = Pose(J=3)
    p.det(8, 8, 0.9, kps=[(8.5, 8.5), (7.5, 9.5), (9.5, 7.5)])
    p.decoys(3)
    for j in range(3):
        p.cand(j, (8.5 + j, 8.5 - j), F32(0.09 - 0.01 * j))
        p.cand(j, (6.5 + j, 10.5), F32(0.05 - 0.01 * j))
    add("all_below", p, 4)

    # ---- K larger than the number of joint peaks (zero fillers), and K = 1
    p = Pose(J=2)
    p.det(8, 8, 0.9, kps=[(8.75, 8.5), (6.0, 10.0)])
    p.decoys(7)
    p.cand(0, (8.5, 8.5), 0.6)
    p.cand(0, (10.5, 6.5), 0.4)
    p.cand(1, (6.5, 10.5), 0.7)
    add("k_gt_peaks", p, 8)
    p = Pose(J=2)
    p.det(8, 8, 0.9, kps=[(8.75, 8.5), (6.0, 10.0)])
    p.decoys(3)
    p.cand(0, (8.5, 8.5), 0.6)      # the only candidate of joint 0: snaps
    p.cand(0, (10.5, 6.5), 0.4)
    p.cand(1, (3.5, 12.5), 0.7)     # the only candidate of joint 1: outside the box
    p.cand(1, (6.5, 10.5), 0.3)
    add("k1", p, 1)

    # ---- the optional heads: a seeded scene with values on a 1/8 grid, J = 3, K = 6
    rng = np.random.default_rng(317)
    lattice = [(y, x) for y in range(1, HW, 3) for x in range(1, HW, 3)]
    base = Pose(J=3)
    cen = rng.permutation(len(lattice))[:6]
    cs = rng.permutation(np.arange(20, 90))[:6] / F32(100)
    for s, i in zip(cs, cen):
        y, x = lattice[i]
        kp = [(x + rng.integers(-24, 25) / 8, y + rng.integers(-24, 25) / 8) for _ in range(3)]
        base.det(y, x, F32(s), wh=(rng.integers(8, 96) / 8, rng.integers(8, 96) / 8),
                 reg=(rng.integers(0, 8) / 8, rng.integers(0, 8) / 8), kps=kp)
    shifted = [(y + 1, x + 1) for y, x in lattice if y + 1 < HW and x + 1 < HW]
    for j in range(3):
        for s, i in zip(rng.permutation(np.arange(3, 60))[:5] / F32(100), rng.permutation(len(shifted))[:5]):
            y, x = shifted[i]
            base.hm_hp[0, j, y, x] = F32(s)
    base.off[:] = rng.integers(0, 8, base.off.shape) / F32(8)
    for reg in (True, False):
        for hp, off in ((False, False), (True, False), (True, True)):
            add("heads_%s_%s" % ("reg" if reg else "noreg", "off" if off else ("hp" if hp else "nohp")), base, 6,
                reg=reg, hp=hp, off=off)

    # ---- non-finite regression values, one per case
    def nf_scene():
        p = Pose(J=2)
        p.det(8, 8, 0.9, kps=[(6.5, 8.5), (10.0, 10.5)])
        p.decoys(3)
        a = p.cand(0, (9.0, 8.5), 0.6)        # nearest to joint 0 and inside the box, but 2.5 > 0.3 * max(5, 6)
        p.cand(0, (12.5, 3.5), 0.4)
        lo = p.cand(0, (11.5, 6.5), 0.05)     # below the threshold
        p.cand(0, (3.5, 12.5), 0.3)
        for i, xy in enumerate(((10.25, 10.25), (4.5, 4.5), (12.5, 12.5), (2.5, 9.5))):
            p.cand(1, xy, F32(0.7 - 0.1 * i))
        return p, a, lo

    for vname, v in (("nan", np.nan), ("pinf", np.inf), ("ninf", -np.inf)):
        for where in ("kps_x", "kps_y", "wh_w", "wh_h", "reg_x", "reg_y", "off_above", "off_below"):
            p, a, lo = nf_scene()
            if where.startswith("kps"):
                p.kps[0, 0 if where == "kps_x" else 1, 8, 8] = v
            elif where.startswith("wh"):
                p.wh[0, 0 if where == "wh_w" else 1, 8, 8] = v
            elif where.startswith("reg"):
                p.reg[0, 0 if where == "reg_x" else 1, 8, 8] = v
            else:
                py, px = a if where == "off_above" else lo
                p.off[0, 0, py, px] = v
            add("nf_%s_%s" % (where, vname), p, 4)
    return names


def ddd_cases():
    rng = np.random.default_rng(2024)
    names = []

    def add(name, heat, K, wh_reg, nonfinite=None):
        B, C, H, W = heat.shape
        check_tie_free(heat, name)
        if K > sum(len(p) for p in positive_peaks(heat)):
            assert K == H * W and C == 1, name   # every pixel selected: the set is fixed, only its order is open
        rot = rng.standard_normal((B, 8, H, W)).astype(F32)
        dep = rng.standard_normal((B, 1, H, W)).astype(F32) * F32(20)
        dim = rng.random((B, 3, H, W), dtype=F32) * F32(4)
        wh = rng.random((B, 2, H, W), dtype=F32) * F32(60) if wh_reg else None
        reg = rng.random((B, 2, H, W), dtype=F32) if wh_reg else None
        heads = dict(rot=rot, depth=dep, dim=dim, wh=wh, reg=reg)
        if nonfinite:
            m = heads[nonfinite]
            for i, v in enumerate((np.nan, np.inf, -np.inf)):
                m[0, i % m.shape[1], (2 * i + 1) % H, (3 * i + 2) % W] = v
        with torch.no_grad():
            dets = R.ddd_decode(t(heat), t(rot), t(dep), t(dim), wh=None if wh is None else t(wh),
                                reg=None if reg is None else t(reg), K=K).numpy()
        store(name, dict(heat=heat, **heads), dets)
        OUT[name + "__K"] = np.int64(K)
        names.append(name)

    def noise(C, H, W):
        return (rng.permutation(C * H * W).reshape(1, C, H, W) + 1).astype(F32) / F32(C * H * W + 1)

    strip = np.zeros((1, 3, 1, 8), F32)                        # 4 peaks per class, 12 >= K = H*W = 8
    strip[0, :, 0, ::2] = (rng.permutation(12) + 1).reshape(3, 4) / F32(16)
    lattice = np.zeros((1, 3, 7, 7), F32)                      # 9 peaks per class
    lattice[0, :, ::3, ::3] = (rng.permutation(27) + 1).reshape(3, 3, 3) / F32(32)
    for wh_reg in (True, False):
        tag = "full" if wh_reg else "min"
        add("ddd_c1_all_" + tag, noise(1, 5, 7), 35, wh_reg)
        add("ddd_c3_strip_" + tag, strip, 8, wh_reg)
        add("ddd_c3_lattice_" + tag, lattice, 20, wh_reg)
    for head in ("rot", "depth", "dim", "wh", "reg"):
        add("ddd_nf_" + head, noise(1, 5, 7), 35, True, nonfinite=head)
    return names


def main():
    pose = pose_cases()
    ddd = ddd_cases()
    OUT["pose_cases"] = np.array(pose)
    OUT["ddd_cases"] = np.array(ddd)
    np.savez_compressed(os.path.join(HERE, "pose_ddd_edges.npz"), **OUT)
    print("wrote pose_ddd_edges: %d multi_pose cases, %d ddd cases" % (len(pose), len(ddd)))


if __name__ == "__main__":
    main()

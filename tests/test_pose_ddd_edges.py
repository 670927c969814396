"""CPU: the numpy oracle of multi_pose_decode and ddd_decode against the UNMODIFIED reference on the edge cases of
tests/golden/pose_ddd_edges.npz (made by tests/golden/make_golden_pose_ddd_edges.py), bit for bit.

nonfinite="reference" must reproduce every golden.  nonfinite="library" (the keypoint assembly's defined rule,
DESIGN.md "Non-finite scores") must reproduce every golden except the cases its two deviations change, and must
change exactly those."""
import numpy as np
import pytest

from helpers import assert_dets_bits, canonical_bits, golden
from oracle import decode_np as O

G = golden("pose_ddd_edges")
POSE = [str(n) for n in G["pose_cases"]]
DDD = [str(n) for n in G["ddd_cases"]]

# Where the library's rule gives another answer than the reference: (a) a below-threshold candidate whose
# hp_offset is not finite stays at (-10000, -10000) instead of turning NaN, (b) a NaN distance is not a minimum.
LIBRARY_CHANGES = {"nf_off_above_nan", "nf_off_below_nan", "nf_off_below_pinf", "nf_off_below_ninf"}

# What the subject detection's joint 0 must do in the cases built for one branch: take the heat-map candidate
# ("snap") or keep its regressed location ("keep").  (box_zero is not listed: its candidate sits on the regressed
# location, so the two answers have the same bits.)
BRANCH = {"thr_eq": "keep", "thr_up": "snap", "thr_dn": "keep",
          "box_l_on": "snap", "box_l_out": "keep", "box_r_on": "snap", "box_r_out": "keep",
          "box_t_on": "snap", "box_t_out": "keep", "box_b_on": "snap", "box_b_out": "keep",
          "dist_lim_eq": "snap", "dist_lim_above": "snap", "dist_lim_below": "keep", "dist_lim_eq_h": "snap",
          "dist_tie_x": "snap", "dist_tie_y": "snap", "box_negative": "keep",
          "all_below": "keep", "nf_wh_w_nan": "snap", "nf_wh_h_nan": "snap", "nf_reg_x_nan": "snap"}


def pose_heads(name):
    return [G.get(name + "__" + k) for k in ("heat", "wh", "kps", "reg", "hm_hp", "hp_offset")]


def ddd_heads(name):
    return [G.get(name + "__" + k) for k in ("heat", "rot", "depth", "dim", "wh", "reg")]


def K_of(name):
    return int(G[name + "__K"])


@pytest.mark.parametrize("name", POSE)
def test_multi_pose_reference_mode(name):
    got = O.multi_pose_decode(*pose_heads(name), K=K_of(name), nonfinite="reference")
    assert_dets_bits(G[name + "__dets"], got, what=name)


@pytest.mark.parametrize("name", POSE)
def test_multi_pose_library_mode(name):
    got = O.multi_pose_decode(*pose_heads(name), K=K_of(name), nonfinite="library")
    if name in LIBRARY_CHANGES:
        assert not np.array_equal(canonical_bits(got), canonical_bits(G[name + "__dets"])), name
        assert np.isfinite(got[..., 5:-1]).all() or not name.startswith("nf_off_below"), name
    else:
        assert_dets_bits(G[name + "__dets"], got, what=name)


def test_library_changes_are_cases():
    assert LIBRARY_CHANGES <= set(POSE) and set(BRANCH) <= set(POSE)


@pytest.mark.parametrize("name", sorted(BRANCH))
def test_cases_sit_on_their_branch(name):
    heat, kps = G[name + "__heat"], G[name + "__kps"]
    y, x = np.unravel_index(np.argmax(heat[0, 0]), heat.shape[2:])
    regressed = np.array([kps[0, 0, y, x] + np.float32(x), kps[0, 1, y, x] + np.float32(y)], np.float32)
    row = G[name + "__dets"][0, 0]
    assert row[4] == heat[0, 0, y, x]
    assert np.array_equal(row[5:7], regressed) == (BRANCH[name] == "keep"), (name, row[5:7], regressed)


@pytest.mark.parametrize("name", DDD)
def test_ddd(name):
    got = O.ddd_decode(*ddd_heads(name)[:4], wh=ddd_heads(name)[4], reg=ddd_heads(name)[5], K=K_of(name))
    assert_dets_bits(G[name + "__dets"], got, score_col=2, what=name)

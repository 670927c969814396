"""numpy restatement of the exdet training sampler's targets given its drawn parameters
(datasets/sample/exdet.py:95-135), written from the numeric contract of DESIGN.md section 4.12 and pinned by
tests/golden/train_exdet.npz (the unmodified EXDetDataset.__getitem__ on seeded images).  The float32 affine map and
the image are those of tests/train_np.py."""
import numpy as np

from oracle import image_np
from train_np import affine_f32

F32 = np.float32
PARTS = ('t', 'l', 'b', 'r')


def exdet_points(pts, flip, width, trans_output, out_res):
    """One object's extreme points [4, 2] (t, l, b, r) after the flip (x -> width - x - 1 in float32, l <-> r) and
    the float32 affine map: (unclipped, clipped to [0, R - 1] by np.clip)."""
    p = np.array(pts, F32).reshape(4, 2)
    if flip:
        p[:, 0] = (F32(width) - p[:, 0] - F32(1)).astype(F32)
        p = p[[0, 3, 2, 1]]
    raw = np.array([affine_f32(trans_output, x, y) for x, y in p], F32)
    return raw, np.clip(raw, F32(0), F32(out_res - 1))


def exdet_targets(pts, cls, flip, width, trans_output, max_objs, out_res, agnostic_ex):
    """exdet.py:95-129 for one image: pts [n, 4, 2] float32, cls [n] -> dict of reg_t/l/b/r [M, 2] f32, ind_t/l/b/r
    [M] i64, reg_mask [M] u8, the centre lists obj_cls / obj_cx / obj_cy / obj_radius (int32) and obj_valid (uint8)
    [M], and the extreme lists ex_cls / ex_cx / ex_cy / ex_radius / ex_valid [4, M].  An object counts when h > 0
    and w > 0 after the clip; its radius is ctdet's float64 gaussian_radius of the sides rounded up; float32 -
    int32 is one rounding of the exact difference."""
    m, R = max_objs, out_res
    r = {'reg_mask': np.zeros(m, np.uint8)}
    for p in PARTS:
        r['reg_' + p], r['ind_' + p] = np.zeros((m, 2), F32), np.zeros(m, np.int64)
    for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius'):
        r[k] = np.zeros(m, np.int32)
    r['obj_valid'] = np.zeros(m, np.uint8)
    for k in ('ex_cls', 'ex_cx', 'ex_cy', 'ex_radius'):
        r[k] = np.zeros((4, m), np.int32)
    r['ex_valid'] = np.zeros((4, m), np.uint8)
    for k in range(min(len(pts), m)):
        _, q = exdet_points(pts[k], flip, width, trans_output, R)
        h, w = F32(q[2, 1] - q[0, 1]), F32(q[3, 0] - q[1, 0])
        if not (h > 0 and w > 0):
            continue
        rad = max(0, int(image_np.gaussian_radius((int(np.ceil(h)), int(np.ceil(w))))))
        qi = q.astype(np.int32)
        c = int(cls[k])
        for j, p in enumerate(PARTS):
            r['reg_' + p][k] = (q[j].astype(np.float64) - qi[j]).astype(F32)
            r['ind_' + p][k] = int(qi[j, 1]) * R + int(qi[j, 0])
            r['ex_cls'][j, k] = 0 if agnostic_ex else c
            r['ex_cx'][j, k], r['ex_cy'][j, k], r['ex_radius'][j, k], r['ex_valid'][j, k] = qi[j, 0], qi[j, 1], rad, 1
        r['reg_mask'][k] = 1
        r['obj_cls'][k], r['obj_radius'][k], r['obj_valid'][k] = c, rad, 1
        r['obj_cx'][k] = int(F32(q[3, 0] + q[1, 0]) / F32(2))
        r['obj_cy'][k] = int(F32(q[0, 1] + q[2, 1]) / F32(2))
    return r


def exdet_maps(t, num_classes, out_res, agnostic_ex):
    """hm_t / hm_l / hm_b / hm_r [num_hm, R, R] and hm_c [C, R, R] of one image from exdet_targets' lists:
    draw_umich_gaussian of every listed point."""
    num_hm = 1 if agnostic_ex else num_classes
    keys = ('ex_cls', 'ex_cx', 'ex_cy', 'ex_radius', 'ex_valid')
    ex = image_np.splat_objects(*[t[k] for k in keys], num_hm, out_res, out_res)
    out = {'hm_' + p: ex[j] for j, p in enumerate(PARTS)}
    lists = [t[k][None] for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid')]
    out['hm_c'] = image_np.splat_objects(*lists, num_classes, out_res, out_res)[0]
    return out

"""numpy restatement of the multi_pose training sampler's targets given its drawn parameters
(datasets/sample/multi_pose.py:104-160), written from the numeric contract of DESIGN.md section 4.10 and pinned by
tests/golden/train_multi_pose.npz (the unmodified MultiPoseDataset.__getitem__ on seeded images).  The box half,
the float32 affine map and the image are those of tests/train_np.py."""
import numpy as np

from oracle import image_np
from train_np import affine_f32

F32 = np.float32


def multi_pose_targets(boxes, cls, kps, flip, width, perm, rotated, trans_output, trans_output_rot, max_objs,
                       out_res):
    """multi_pose.py:104-160 for one image: boxes [n, 4] float32 corners, cls [n], kps [n, J, 3] float32, the
    flip permutation perm (new joint j = old joint perm[j]) -> dict of wh, ind, reg, reg_mask, hps, hps_mask,
    hp_offset, hp_ind, hp_mask, the centre lists (obj_*, [M]) and the joint lists (hp_cx, hp_cy, hp_radius,
    hp_valid, [J, M]).  A slot gets targets when (h > 0 and w > 0) or rotated; reg_mask also needs a non-zero
    visibility; a joint counts when visible and mapped into [0, R) x [0, R); float32 - int32 is one rounding of the
    exact difference; rotated images keep everything but reg_mask and hps_mask."""
    m, nj, R = max_objs, len(perm), out_res
    r = {'wh': np.zeros((m, 2), F32), 'reg': np.zeros((m, 2), F32), 'ind': np.zeros(m, np.int64),
         'reg_mask': np.zeros(m, np.uint8), 'hps': np.zeros((m, 2 * nj), F32),
         'hps_mask': np.zeros((m, 2 * nj), np.uint8), 'hp_offset': np.zeros((m * nj, 2), F32),
         'hp_ind': np.zeros(m * nj, np.int64), 'hp_mask': np.zeros(m * nj, np.int64)}
    for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius'):
        r[k] = np.zeros(m, np.int32)
    r['obj_valid'] = np.zeros(m, np.uint8)
    for k in ('hp_cx', 'hp_cy', 'hp_radius'):
        r[k] = np.zeros((nj, m), np.int32)
    r['hp_valid'] = np.zeros((nj, m), np.uint8)
    for k in range(min(len(boxes), m)):
        x0, y0, x1, y1 = [F32(v) for v in boxes[k]]
        pts = np.array(kps[k], F32).reshape(nj, 3)
        if flip:
            x0, x1 = F32(F32(F32(width) - x1) - F32(1)), F32(F32(F32(width) - x0) - F32(1))
            pts[:, 0] = (F32(width) - pts[:, 0] - F32(1)).astype(F32)
            pts = pts[np.asarray(perm)]
        x0, y0 = affine_f32(trans_output, x0, y0)
        x1, y1 = affine_f32(trans_output, x1, y1)
        x0, x1, y0, y1 = [F32(min(max(v, F32(0)), F32(R - 1))) for v in (x0, x1, y0, y1)]
        h, w = F32(y1 - y0), F32(x1 - x0)
        if not ((h > 0 and w > 0) or rotated):
            continue
        rad = max(0, int(image_np.gaussian_radius((int(np.ceil(h)), int(np.ceil(w))))))
        ct = np.array([(x0 + x1) / F32(2), (y0 + y1) / F32(2)], F32)
        ci = ct.astype(np.int32)
        r['wh'][k] = w, h
        r['ind'][k] = int(ci[1]) * R + int(ci[0])
        r['reg'][k] = ct - ci.astype(F32)
        r['reg_mask'][k] = 0 if rotated or not (pts[:, 2] != 0).any() else 1
        r['obj_cls'][k], r['obj_cx'][k], r['obj_cy'][k], r['obj_radius'][k] = int(cls[k]), ci[0], ci[1], rad
        r['obj_valid'][k] = 1
        for j in range(nj):
            if not pts[j, 2] > 0:
                continue
            px, py = affine_f32(trans_output_rot, pts[j, 0], pts[j, 1])
            if not (0 <= px < R and 0 <= py < R):
                continue
            pi = np.array([px, py], F32).astype(np.int32)
            r['hps'][k, 2 * j:2 * j + 2] = F32(px - F32(ci[0])), F32(py - F32(ci[1]))
            r['hps_mask'][k, 2 * j:2 * j + 2] = 0 if rotated else 1
            r['hp_offset'][k * nj + j] = F32(px - F32(pi[0])), F32(py - F32(pi[1]))
            r['hp_ind'][k * nj + j] = int(pi[1]) * R + int(pi[0])
            r['hp_mask'][k * nj + j] = 1
            r['hp_cx'][j, k], r['hp_cy'][j, k], r['hp_radius'][j, k], r['hp_valid'][j, k] = pi[0], pi[1], rad, 1
    return r


def multi_pose_maps(t, num_classes, out_res, rotated):
    """hm [C, R, R] and hm_hp [J, R, R] of one image from multi_pose_targets' lists: draw_umich_gaussian of every
    listed centre / joint, hm the constant f32(0.9999) when rotated."""
    lists = [t[k][None] for k in ('obj_cls', 'obj_cx', 'obj_cy', 'obj_radius', 'obj_valid')]
    hm = image_np.splat_objects(*lists, num_classes, out_res, out_res)[0]
    if rotated:
        hm[:] = F32(0.9999)
    nj = t['hp_cx'].shape[0]
    hp = [np.zeros_like(t['hp_cx'])] + [t[k] for k in ('hp_cx', 'hp_cy', 'hp_radius', 'hp_valid')]
    hm_hp = image_np.splat_objects(*hp, 1, out_res, out_res).reshape(nj, out_res, out_res)
    return hm, hm_hp

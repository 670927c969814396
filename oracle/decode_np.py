"""numpy restatement of the reference heat-map decode family (TEST INFRASTRUCTURE).

Every function cites the reference lines it follows (paths relative to
``/root/reference/src/lib``).  All arithmetic is done in float32 in the same
operation order as the reference so float outputs agree to the last bit on
tie-free inputs.

One thing is *defined* here that the reference leaves to ``torch.topk``'s
implementation: the order of equal scores.  The oracle (and the CUDA path)
use the total order  (score descending, flat index ascending)  where the flat
index is ``cls*H*W + y*W + x`` and non-peaks carry score 0 exactly as
``heat * keep`` does in ``models/decode.py:15``.  A per-class top-K followed by
a cross-class top-K (decode.py:103-119) under that order is identical to one
global top-K, which is what makes a single fused GPU selection legal.
"""
import numpy as np

F32 = np.float32


# --------------------------------------------------------------------------- A1
def nms(heat, kernel=3):
    """models/decode.py:9-15  (_nms): 3x3/stride-1 max-pool with -inf padding,
    keep = (hmax == heat), return heat * keep."""
    assert kernel == 3
    heat = np.asarray(heat, dtype=F32)
    B, C, H, W = heat.shape
    pad = np.full((B, C, H + 2, W + 2), -np.inf, dtype=F32)
    pad[:, :, 1:-1, 1:-1] = heat
    hmax = pad[:, :, 1:-1, 1:-1].copy()
    for dy in range(3):
        for dx in range(3):
            np.maximum(hmax, pad[:, :, dy:dy + H, dx:dx + W], out=hmax)
    keep = (hmax == heat).astype(F32)
    return heat * keep


def _stable_topk(flat, K):
    """Top-K of the last axis under (value desc, index asc)."""
    order = np.argsort(-flat, axis=-1, kind="stable")[..., :K]
    return np.take_along_axis(flat, order, axis=-1), order.astype(np.int64)


# --------------------------------------------------------------------------- A3
def topk_channel(scores, K=40):
    """models/decode.py:92-101 (_topk_channel)."""
    B, C, H, W = scores.shape
    s, inds = _stable_topk(scores.reshape(B, C, H * W), K)
    inds = inds % (H * W)
    ys = (inds // W).astype(F32)          # (inds / width).int().float()
    xs = (inds % W).astype(F32)
    return s, inds, ys, xs


# --------------------------------------------------------------------------- A2
def topk(scores, K=40):
    """models/decode.py:103-119 (_topk): per-class top-K then cross-class top-K."""
    B, C, H, W = scores.shape
    s1, inds, ys, xs = topk_channel(scores, K)
    s2, ind2 = _stable_topk(s1.reshape(B, C * K), K)
    clses = (ind2 // K).astype(np.int32)
    pick = lambda a: np.take_along_axis(a.reshape(B, C * K), ind2, axis=1)
    return s2, pick(inds), clses, pick(ys), pick(xs)


# --------------------------------------------------------------------------- A4
def gather_feat(feat, ind):
    """models/utils.py:12-20 (_gather_feat, mask=None): feat[B,N,D], ind[B,M] -> [B,M,D]."""
    return np.take_along_axis(feat, ind[:, :, None].astype(np.int64), axis=1)


def transpose_and_gather_feat(feat, ind):
    """models/utils.py:22-26: NCHW -> [B,HW,C] then gather rows ``ind``."""
    B, C, H, W = feat.shape
    f = np.ascontiguousarray(np.transpose(feat, (0, 2, 3, 1))).reshape(B, H * W, C)
    return gather_feat(f, ind)


# --------------------------------------------------------------------------- A5
def ctdet_decode(heat, wh, reg=None, cat_spec_wh=False, K=100):
    """models/decode.py:464-495."""
    heat = np.asarray(heat, F32); wh = np.asarray(wh, F32)
    B, C, H, W = heat.shape
    scores, inds, clses, ys, xs = topk(nms(heat), K)
    if reg is not None:
        r = transpose_and_gather_feat(np.asarray(reg, F32), inds)
        xs = xs[..., None] + r[:, :, 0:1]
        ys = ys[..., None] + r[:, :, 1:2]
    else:
        xs = xs[..., None] + F32(0.5)
        ys = ys[..., None] + F32(0.5)
    w = transpose_and_gather_feat(wh, inds)
    if cat_spec_wh:
        w = w.reshape(B, K, C, 2)
        ci = clses.astype(np.int64)[:, :, None, None].repeat(2, axis=3)
        w = np.take_along_axis(w, ci, axis=2).reshape(B, K, 2)
    half_w = w[..., 0:1] / F32(2)
    half_h = w[..., 1:2] / F32(2)
    boxes = np.concatenate([xs - half_w, ys - half_h, xs + half_w, ys + half_h], axis=2)
    return np.concatenate([boxes, scores[..., None], clses.astype(F32)[..., None]], axis=2).astype(F32)


# --------------------------------------------------------------------------- A9
def ddd_decode(heat, rot, depth, dim, wh=None, reg=None, K=40):
    """models/decode.py:426-462."""
    heat = np.asarray(heat, F32)
    scores, inds, clses, ys, xs = topk(nms(heat), K)
    if reg is not None:
        r = transpose_and_gather_feat(np.asarray(reg, F32), inds)
        xs = xs[..., None] + r[:, :, 0:1]
        ys = ys[..., None] + r[:, :, 1:2]
    else:
        xs = xs[..., None] + F32(0.5)
        ys = ys[..., None] + F32(0.5)
    cols = [xs, ys, scores[..., None],
            transpose_and_gather_feat(np.asarray(rot, F32), inds),
            transpose_and_gather_feat(np.asarray(depth, F32), inds),
            transpose_and_gather_feat(np.asarray(dim, F32), inds)]
    if wh is not None:
        cols.append(transpose_and_gather_feat(np.asarray(wh, F32), inds))
    cols.append(clses.astype(F32)[..., None])
    return np.concatenate(cols, axis=2).astype(F32)


# --------------------------------------------------------------------------- A6
def multi_pose_decode(heat, wh, kps, reg=None, hm_hp=None, hp_offset=None, K=100, nonfinite="reference"):
    """models/decode.py:497-571.

    ``nonfinite="reference"`` is the reference's arithmetic, NaN and inf included.  ``"library"`` is the keypoint
    assembly's defined rule (DESIGN.md, "Non-finite scores"): the same arithmetic with two deviations, both where one
    non-finite value would otherwise reach every detection of the image:
    (a) a joint candidate at or below the threshold is exactly (score -1, x -10000, y -10000), whatever its offset
        (the reference's ``-10000 + 0 * off`` is NaN for a non-finite offset);
    (b) the nearest candidate is the first minimum over the non-NaN distances, candidate 0 when all are NaN (the
        reference's ``torch.min`` picks the first NaN).
    Heat-map scores are assumed finite (their rule is the selection's, ``oracle/select_torch.py``)."""
    if nonfinite not in ("reference", "library"):
        raise ValueError("nonfinite must be 'reference' or 'library'")
    with np.errstate(invalid="ignore", over="ignore"):
        return _multi_pose_decode(heat, wh, kps, reg, hm_hp, hp_offset, K, nonfinite == "library")


def _first_min_skip_nan(dist):
    """Index of the first minimum along the last axis, NaN skipped; 0 where every entry is NaN."""
    nan = np.isnan(dist)
    key = np.where(nan, F32(np.inf), dist)
    hit = (key == key.min(axis=-1, keepdims=True)) & ~nan
    return hit.argmax(axis=-1)


def _multi_pose_decode(heat, wh, kps, reg, hm_hp, hp_offset, K, library):
    heat = np.asarray(heat, F32); wh = np.asarray(wh, F32); kps = np.asarray(kps, F32)
    B, C, H, W = heat.shape
    J = kps.shape[1] // 2
    scores, inds, clses, ys, xs = topk(nms(heat), K)
    kp = transpose_and_gather_feat(kps, inds).reshape(B, K, J * 2).copy()
    kp[..., 0::2] += xs[..., None]              # integer xs/ys, before reg (:508-509)
    kp[..., 1::2] += ys[..., None]
    if reg is not None:
        r = transpose_and_gather_feat(np.asarray(reg, F32), inds)
        xs = xs[..., None] + r[:, :, 0:1]
        ys = ys[..., None] + r[:, :, 1:2]
    else:
        xs = xs[..., None] + F32(0.5)
        ys = ys[..., None] + F32(0.5)
    w = transpose_and_gather_feat(wh, inds)
    half_w = w[..., 0:1] / F32(2)
    half_h = w[..., 1:2] / F32(2)
    boxes = np.concatenate([xs - half_w, ys - half_h, xs + half_w, ys + half_h], axis=2)
    if hm_hp is not None:
        thresh = F32(0.1)
        hm = nms(np.asarray(hm_hp, F32))
        reg_kps = kp.reshape(B, K, J, 2).transpose(0, 2, 1, 3)            # B,J,K,2
        hs, hinds, hys, hxs = topk_channel(hm, K)                          # B,J,K
        if hp_offset is not None:
            off = transpose_and_gather_feat(np.asarray(hp_offset, F32), hinds.reshape(B, -1))
            off = off.reshape(B, J, K, 2)
            hxs = hxs + off[..., 0]
            hys = hys + off[..., 1]
        else:
            hxs = hxs + F32(0.5)
            hys = hys + F32(0.5)
        keep = hs > thresh
        if library:                                                        # rule (a)
            hs = np.where(keep, hs, F32(-1))
            hys = np.where(keep, hys, F32(-10000))
            hxs = np.where(keep, hxs, F32(-10000))
        else:
            m = keep.astype(F32)
            hs = (F32(1) - m) * F32(-1) + m * hs
            hys = (F32(1) - m) * F32(-10000) + m * hys
            hxs = (F32(1) - m) * F32(-10000) + m * hxs
        hm_kps = np.stack([hxs, hys], axis=-1)                             # B,J,K,2
        d = reg_kps[:, :, :, None, :] - hm_kps[:, :, None, :, :]           # B,J,K(det),K(cand),2
        dist = np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]).astype(F32)).astype(F32)
        # first minimum; np.argmin, like torch.min, takes the first NaN if there is one; rule (b) skips NaN
        min_ind = _first_min_skip_nan(dist) if library else dist.argmin(axis=3)
        min_dist = np.take_along_axis(dist, min_ind[..., None], axis=3)    # B,J,K,1
        sel_s = np.take_along_axis(hs, min_ind, axis=2)[..., None]
        sel_kp = np.take_along_axis(hm_kps, min_ind[..., None].repeat(2, axis=-1), axis=2)
        l = boxes[:, None, :, 0:1]; t = boxes[:, None, :, 1:2]
        r_ = boxes[:, None, :, 2:3]; b_ = boxes[:, None, :, 3:4]
        bad = ((sel_kp[..., 0:1] < l) | (sel_kp[..., 0:1] > r_) |
               (sel_kp[..., 1:2] < t) | (sel_kp[..., 1:2] > b_) |
               (sel_s < thresh) | (min_dist > np.maximum(b_ - t, r_ - l) * F32(0.3)))   # np.maximum keeps NaN
        m = np.broadcast_to(bad, sel_kp.shape).astype(F32)
        out_kp = (F32(1) - m) * sel_kp + m * reg_kps                       # the reference's blend (:566)
        kp = out_kp.transpose(0, 2, 1, 3).reshape(B, K, J * 2)
    return np.concatenate([boxes, scores[..., None], kp, clses.astype(F32)[..., None]],
                          axis=2).astype(F32)


# --------------------------------------------------------------------------- A7
def _run_sum(heat2d_last_axis, reverse):
    """ret[i] = heat[i] + ret[i-1]*[heat[i] >= heat[i-1]] along the LAST axis, strictly
    sequential fp32 adds (decode.py:25-27 / :38-40), returns ret - heat (:28)."""
    h = heat2d_last_axis
    ret = h.copy()
    n = h.shape[-1]
    rng = range(n - 2, -1, -1) if reverse else range(1, n)
    step = 1 if reverse else -1
    for i in rng:
        ge = (h[..., i] >= h[..., i + step]).astype(F32)
        ret[..., i] = ret[..., i] + ret[..., i + step] * ge
    return ret - h


def left_aggregate(heat):   # decode.py:17-28
    return _run_sum(np.asarray(heat, F32), reverse=False)


def right_aggregate(heat):  # decode.py:30-41
    return _run_sum(np.asarray(heat, F32), reverse=True)


def top_aggregate(heat):    # decode.py:43-55
    return _run_sum(np.asarray(heat, F32).swapaxes(2, 3), reverse=False).swapaxes(2, 3)


def bottom_aggregate(heat):  # decode.py:57-69
    return _run_sum(np.asarray(heat, F32).swapaxes(2, 3), reverse=True).swapaxes(2, 3)


def h_aggregate(heat, aggr_weight=0.1):
    """decode.py:71-73:  w*left + w*right + heat  (fp32, that operation order)."""
    w = F32(aggr_weight)
    return np.ascontiguousarray(w * left_aggregate(heat) + w * right_aggregate(heat) + heat)


def v_aggregate(heat, aggr_weight=0.1):
    """decode.py:75-77."""
    w = F32(aggr_weight)
    return np.ascontiguousarray(w * top_aggregate(heat) + w * bottom_aggregate(heat) + heat)


# --------------------------------------------------------------------------- A8
def _exct_core(t_heat, l_heat, b_heat, r_heat, ct_heat, regs, K, scores_thresh,
               center_thresh, aggr_weight, num_dets, agnostic):
    t_heat, l_heat, b_heat, r_heat, ct_heat = [np.asarray(a, F32) for a in
                                               (t_heat, l_heat, b_heat, r_heat, ct_heat)]
    B, C, H, W = t_heat.shape
    if aggr_weight > 0:                                   # decode.py:287-291
        t_heat = h_aggregate(t_heat, aggr_weight); l_heat = v_aggregate(l_heat, aggr_weight)
        b_heat = h_aggregate(b_heat, aggr_weight); r_heat = v_aggregate(r_heat, aggr_weight)
    ext = []
    for hmap in (t_heat, l_heat, b_heat, r_heat):         # :294-307
        n = nms(hmap)
        n[n > 1] = 1
        ext.append(topk(n, K))
    (ts, ti, tc, ty, tx), (ls, li, lc, ly, lx), (bs, bi, bc, by, bx), (rs, ri, rc, ry, rx) = ext
    if agnostic:                                                       # :159,175-180
        agn = ct_heat.max(axis=1); agn_cls = ct_heat.argmax(axis=1)
    bidx = np.arange(B).reshape(B, 1, 1, 1, 1)

    def slab(t0, t1):
        """Scores and classes of the tuples whose t index lies in [t0, t1): [B, (t1-t0)*K^3] each.
        The reference materialises all K^4 at once (:309-360); slabs keep the oracle inside a few
        hundred MB at K=100 without changing a single per-tuple operation."""
        n = t1 - t0
        sh = lambda a, ax: a.reshape([B] + [(n if ax == 0 else K) if i == ax else 1 for i in range(4)])
        ty_, tx_, ts_, tc_ = [sh(a[:, t0:t1], 0) for a in (ty, tx, ts, tc)]
        ly_, lx_, ls_, lc_ = sh(ly, 1), sh(lx, 1), sh(ls, 1), sh(lc, 1)
        by_, bx_, bs_, bc_ = sh(by, 2), sh(bx, 2), sh(bs, 2), sh(bc, 2)
        ry_, rx_, rs_, rc_ = sh(ry, 3), sh(rx, 3), sh(rs, 3), sh(rc, 3)
        full = (B, n, K, K, K)
        cx = ((lx_ + rx_ + F32(0.5)) / F32(2)).astype(np.int64)          # :322-323
        cy = ((ty_ + by_ + F32(0.5)) / F32(2)).astype(np.int64)
        cx = np.broadcast_to(cx, full); cy = np.broadcast_to(cy, full)
        if agnostic:
            ct = agn[bidx, cy, cx]
            clses = agn_cls[bidx, cy, cx].astype(F32)
        else:                                                              # :324-327
            tcl = np.broadcast_to(tc_.astype(np.int64), full)
            ct = ct_heat[bidx, tcl, cy, cx]
            clses = np.broadcast_to(tc_.astype(F32), full)
        scores = ((((ts_ + ls_) + bs_) + rs_) + F32(2) * ct) / F32(6)      # :333 / :192
        sc_bad = ((ts_ < F32(scores_thresh)) | (ls_ < F32(scores_thresh)) |
                  (bs_ < F32(scores_thresh)) | (rs_ < F32(scores_thresh)) |
                  (ct < F32(center_thresh)))
        top_bad = (ty_ > ly_) | (ty_ > by_) | (ty_ > ry_)
        left_bad = (lx_ > tx_) | (lx_ > bx_) | (lx_ > rx_)
        bot_bad = (by_ < ty_) | (by_ < ly_) | (by_ < ry_)
        right_bad = (rx_ < tx_) | (rx_ < lx_) | (rx_ < bx_)
        scores = scores - np.broadcast_to(sc_bad, full).astype(F32)
        if not agnostic:
            cls_bad = (tc_ != lc_) | (tc_ != bc_) | (tc_ != rc_)
            scores = scores - np.broadcast_to(cls_bad, full).astype(F32)
        for bad in (top_bad, left_bad, bot_bad, right_bad):
            scores = scores - np.broadcast_to(bad, full).astype(F32)
        return scores.reshape(B, -1), np.asarray(clses).reshape(B, -1)

    # topk(num_dets) over all K^4 tuples (:362-364) = top of the union of per-slab tops; slabs are
    # visited in ascending tuple index, so the stable final sort keeps (score desc, index asc).
    step = max(1, min(K, (4 << 20) // (K * K * K)))
    cs, ci, cc = [], [], []
    for t0 in range(0, K, step):
        s_, c_ = slab(t0, min(K, t0 + step))
        v, o = _stable_topk(s_, min(num_dets, s_.shape[1]))
        o = np.sort(o, axis=1)                                         # back to index order inside the slab
        cs.append(np.take_along_axis(s_, o, axis=1)); cc.append(np.take_along_axis(c_, o, axis=1))
        ci.append(o + t0 * K * K * K)
    cs, ci, cc = np.concatenate(cs, 1), np.concatenate(ci, 1), np.concatenate(cc, 1)
    scores, pick = _stable_topk(cs, num_dets)
    sel = np.take_along_axis(ci, pick, axis=1)
    clses_sel = np.take_along_axis(cc, pick, axis=1)
    if all(r is not None for r in regs):                                # :366-384
        tr, lr, br, rr = [transpose_and_gather_feat(np.asarray(r, F32), i)
                          for r, i in zip(regs, (ti, li, bi, ri))]
        tx2, ty2 = tx + tr[..., 0], ty + tr[..., 1]
        lx2, ly2 = lx + lr[..., 0], ly + lr[..., 1]
        bx2, by2 = bx + br[..., 0], by + br[..., 1]
        rx2, ry2 = rx + rr[..., 0], ry + rr[..., 1]
    else:                                                               # :385-393
        h = F32(0.5)
        tx2, ty2, lx2, ly2 = tx + h, ty + h, lx + h, ly + h
        bx2, by2, rx2, ry2 = bx + h, by + h, rx + h, ry + h
    i_t = sel // (K * K * K); i_l = (sel // (K * K)) % K; i_b = (sel // K) % K; i_r = sel % K
    g = lambda a, i: np.take_along_axis(a, i, axis=1)
    clses = clses_sel
    cols = [g(lx2, i_l), g(ty2, i_t), g(rx2, i_r), g(by2, i_b), scores,
            g(tx2, i_t), g(ty2, i_t), g(lx2, i_l), g(ly2, i_l),
            g(bx2, i_b), g(by2, i_b), g(rx2, i_r), g(ry2, i_r), clses]
    return np.stack(cols, axis=2).astype(F32)


def exct_decode(t_heat, l_heat, b_heat, r_heat, ct_heat, t_regr=None, l_regr=None,
                b_regr=None, r_regr=None, K=40, scores_thresh=0.1, center_thresh=0.1,
                aggr_weight=0.0, num_dets=1000):
    """models/decode.py:273-424."""
    return _exct_core(t_heat, l_heat, b_heat, r_heat, ct_heat,
                      (t_regr, l_regr, b_regr, r_regr), K, scores_thresh, center_thresh,
                      aggr_weight, num_dets, agnostic=False)


def agnex_ct_decode(t_heat, l_heat, b_heat, r_heat, ct_heat, t_regr=None, l_regr=None,
                    b_regr=None, r_regr=None, K=40, scores_thresh=0.1, center_thresh=0.1,
                    aggr_weight=0.0, num_dets=1000):
    """models/decode.py:122-271 (class-agnostic extreme maps, centre = max over classes)."""
    return _exct_core(t_heat, l_heat, b_heat, r_heat, ct_heat,
                      (t_regr, l_regr, b_regr, r_regr), K, scores_thresh, center_thresh,
                      aggr_weight, num_dets, agnostic=True)

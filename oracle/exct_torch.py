"""torch restatement of exct_decode / agnex_ct_decode (models/decode.py:122-424) (TEST INFRASTRUCTURE).

Runs on CPU and on CUDA tensors, so the kernel's large cases (B ~ 300 images, K = 100, one K = 255 image) get an
independent answer in seconds.  It follows the reference operation by operation:

* aggregation (aggr_weight > 0): ``decode_np``'s h / v aggregation, pinned bit for bit to the reference;
* the four selections: ``select_torch.nms(nonfinite="library")``, the clamp to 1 (:299-302), ``select_torch.topk``;
* the centre map: agnostic, ``torch.max(dim=1)`` semantics (NaN propagates, its class is the first NaN class, ties
  take the first class); per class, a raw gather at ``t_cls * H*W + cy*W + cx``;
* the tuple score ``((((t + l) + b) + r) + 2*ct) / 6`` in fp32, then the six penalty subtractions in :355-360 order,
  the centre ``((l_x + r_x + 0.5) / 2).long()``;
* the cut (torch.topk over the K^4 tuples, :362-364): one stable descending sort per image, visited in chunks of
  the top index and merged, after folding -0 to +0 and every NaN, whatever its sign, into one NaN that sorts first.
  This is the library's order, which the reference leaves to torch.topk: score descending, tuple index
  ``((i*K + j)*K + k)*K + m`` ascending.  The score column returns the folded values, as the kernel does, so it
  deliberately differs from the reference's in two ways: a -0 score comes out as +0, and every NaN as one
  positive NaN (DESIGN.md, "non-finite scores");
* each regression column one fp32 add (or ``+ 0.5`` without regression).

Division by 6.  torch on CUDA turns ``tensor / 6`` (a Python scalar divisor) into a multiplication by fp32(1/6),
which is not correctly rounded; the reference on CPU, the numpy oracle and the kernel divide.  Here the fp32 sum is
divided in float64 and rounded once to fp32, which equals the correctly rounded fp32 quotient (a 53-bit quotient
of two 24-bit operands never double-rounds).  ``div6`` is that step; ``tests/test_exct_oracle.py`` checks it
against numpy's float32 division.
"""
import torch

from oracle import decode_np as O
from oracle import select_torch as ST


def div6(x):
    """fp32 x / 6, correctly rounded on any device."""
    return (x.double() / 6.0).float()


def _aggregate(heat, aggr_weight, horizontal):
    f = O.h_aggregate if horizontal else O.v_aggregate
    return torch.from_numpy(f(heat.cpu().numpy(), aggr_weight)).to(heat.device)


def centre_max(ct):
    """torch.max(ct, dim=1) of an [B, CC, H, W] map: (values, classes int64), each [B, H, W].  NaN wins over every
    number and the first NaN class is taken; among equal values, the first class."""
    v = torch.amax(ct, dim=1, keepdim=True)                       # NaN if any class is NaN
    hit = (ct == v) | torch.isnan(ct)                             # no NaN in ct unless v is NaN
    cls = torch.argmax(hit.to(torch.uint8), dim=1, keepdim=True)  # argmax returns the first maximal index
    return torch.gather(ct, 1, cls)[:, 0], cls[:, 0]


def _sort_key(s):
    """Scores as sorted: -0 -> +0 and one NaN for every NaN (torch.sort puts it first in descending order)."""
    s = s + 0.0
    return torch.where(torch.isnan(s), torch.full_like(s, float("nan")), s)


def _core(maps, ct, regs, K, scores_thresh, center_thresh, aggr_weight, num_dets, agnostic, chunk_elems):
    maps = [m.float() for m in maps]
    ct = ct.float()
    B, C, H, W = maps[0].shape
    HW = H * W
    dev = maps[0].device
    if aggr_weight > 0:                                           # :287-291: t, b horizontal; l, r vertical
        maps = [_aggregate(m, aggr_weight, h) for m, h in zip(maps, (True, False, True, False))]
    lists = []
    for m in maps:                                                # :294-307
        n = ST.nms(m, "library")
        n = torch.where(n > 1, torch.ones_like(n), n)
        lists.append(ST.topk(n, K))                               # (scores, inds, clses, ys, xs), each [B, K]
    (ts, ti, tc, ty, tx), (ls, li, lc, ly, lx), (bs, bi, bc, by, bx), (rs, ri, rc, ry, rx) = lists
    if agnostic:
        agn, agn_cls = centre_max(ct)
        ct_flat, cls_flat = agn.reshape(B, HW), agn_cls.reshape(B, HW)
    else:
        ct_flat = ct.reshape(B, -1)
    st, cth = torch.tensor(scores_thresh, dtype=torch.float32), torch.tensor(center_thresh, dtype=torch.float32)
    st, cth = st.to(dev), cth.to(dev)

    def scores_of(t0, t1):
        """[B, (t1-t0)*K^3] scores of the tuples whose top index lies in [t0, t1), in tuple-index order."""
        n = t1 - t0
        sh = lambda a, ax: a.reshape([B] + [(n if ax == 0 else K) if i == ax else 1 for i in range(4)])
        ty_, tx_, ts_, tc_ = [sh(a[:, t0:t1], 0) for a in (ty, tx, ts, tc)]
        ly_, lx_, ls_, lc_ = [sh(a, 1) for a in (ly, lx, ls, lc)]
        by_, bx_, bs_, bc_ = [sh(a, 2) for a in (by, bx, bs, bc)]
        ry_, rx_, rs_, rc_ = [sh(a, 3) for a in (ry, rx, rs, rc)]
        full = (B, n, K, K, K)
        cx = ((lx_ + rx_ + 0.5) / 2).long()                      # :322-323
        cy = ((ty_ + by_ + 0.5) / 2).long()
        sp = (cy * W + cx).expand(full)
        if agnostic:
            idx = sp
        else:                                                     # :324-327
            idx = tc_.long() * HW + sp
        ctv = torch.gather(ct_flat, 1, idx.reshape(B, -1)).reshape(full)
        s = div6(((((ts_ + ls_) + bs_) + rs_) + 2 * ctv))         # :334
        sc_bad = (ts_ < st) | (ls_ < st) | (bs_ < st) | (rs_ < st) | (ctv < cth)
        pen = [sc_bad]
        if not agnostic:
            pen.append((tc_ != lc_) | (tc_ != bc_) | (tc_ != rc_))
        pen += [(ty_ > ly_) | (ty_ > by_) | (ty_ > ry_),          # :341-348
                (lx_ > tx_) | (lx_ > bx_) | (lx_ > rx_),
                (by_ < ty_) | (by_ < ly_) | (by_ < ry_),
                (rx_ < tx_) | (rx_ < lx_) | (rx_ < bx_)]
        for p in pen:                                             # :355-360
            s = s - p.expand(full).float()
        return s.reshape(B, -1)

    K3 = K * K * K
    step = max(1, min(K, chunk_elems // max(1, B * K3)))
    vals, inds = [], []
    for t0 in range(0, K, step):
        s = _sort_key(scores_of(t0, min(K, t0 + step)))
        v, o = torch.sort(s, dim=1, descending=True, stable=True)
        keep = min(num_dets, s.shape[1])
        vals.append(v[:, :keep]); inds.append(o[:, :keep] + t0 * K3)
    # chunks in ascending tuple index: the stable sort of their tops keeps equal keys in index order
    v, o = torch.sort(torch.cat(vals, 1), dim=1, descending=True, stable=True)
    scores = v[:, :num_dets]
    sel = torch.gather(torch.cat(inds, 1), 1, o[:, :num_dets])
    return _rows(scores, sel, lists, regs, K, W, agnostic, cls_flat if agnostic else None)


def _rows(scores, sel, lists, regs, K, W, agnostic, cls_flat):
    """The 14 columns of the selected tuples (:395-421)."""
    (_, ti, tc, ty, tx), (_, li, _, ly, lx), (_, bi, _, by, bx), (_, ri, _, ry, rx) = lists
    xy = [[tx, ty], [lx, ly], [bx, by], [rx, ry]]
    if all(r is not None for r in regs):                          # :366-384: the head at each list's peaks
        for q, (r, sp) in enumerate(zip(regs, (ti, li, bi, ri))):
            rr = ST._gather(r.float(), sp)                        # [B, K, 2]
            xy[q] = [xy[q][0] + rr[..., 0], xy[q][1] + rr[..., 1]]
    else:                                                         # :385-393
        xy = [[x + 0.5, y + 0.5] for x, y in xy]
    pick = (sel // (K * K * K), (sel // (K * K)) % K, (sel // K) % K, sel % K)
    (tx2, ty2), (lx2, ly2), (bx2, by2), (rx2, ry2) = [[torch.gather(a, 1, i) for a in p] for p, i in zip(xy, pick)]
    if agnostic:                                                  # the class at the tuple's centre
        g = lambda a, i: torch.gather(a, 1, i)
        cx = ((g(lx, pick[1]) + g(rx, pick[3]) + 0.5) / 2).long()
        cy = ((g(ty, pick[0]) + g(by, pick[2]) + 0.5) / 2).long()
        cls = torch.gather(cls_flat, 1, cy * W + cx).float()
    else:
        cls = torch.gather(tc, 1, pick[0]).float()
    return torch.stack([lx2, ty2, rx2, by2, scores, tx2, ty2, lx2, ly2, bx2, by2, rx2, ry2, cls], dim=2)


def exct_decode(t_heat, l_heat, b_heat, r_heat, ct_heat, t_regr=None, l_regr=None, b_regr=None, r_regr=None, K=40,
                scores_thresh=0.1, center_thresh=0.1, aggr_weight=0.0, num_dets=1000, chunk_elems=1 << 24):
    """models/decode.py:273-424 -> dets [B, num_dets, 14] float32, on the device of the inputs.  Every input is
    widened exactly to fp32.  chunk_elems bounds the tuples scored at once (at least one top index per chunk)."""
    return _core((t_heat, l_heat, b_heat, r_heat), ct_heat, (t_regr, l_regr, b_regr, r_regr), K, scores_thresh,
                 center_thresh, aggr_weight, num_dets, False, chunk_elems)


def agnex_ct_decode(t_heat, l_heat, b_heat, r_heat, ct_heat, t_regr=None, l_regr=None, b_regr=None, r_regr=None,
                    K=40, scores_thresh=0.1, center_thresh=0.1, aggr_weight=0.0, num_dets=1000, chunk_elems=1 << 24):
    """models/decode.py:122-271: class-agnostic extreme maps, centre = max over the centre map's classes."""
    return _core((t_heat, l_heat, b_heat, r_heat), ct_heat, (t_regr, l_regr, b_regr, r_regr), K, scores_thresh,
                 center_thresh, aggr_weight, num_dets, True, chunk_elems)

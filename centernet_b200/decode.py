"""Mirror of src/lib/models/decode.py: same names, signatures, defaults and outputs.

Every function takes fp32 CUDA tensors (NCHW; heat maps already sigmoided by the
caller, as in detectors/ctdet.py:31,40), does not mutate its inputs, and returns a new
fp32 tensor on the same device, enqueued on the current stream.  Other dtypes are upcast
to fp32 first, except in ctdet_decode, multi_pose_decode, ddd_decode, exct_decode,
agnex_ct_decode, their *_from_logits forms, the edge aggregation helpers (_h_aggregate,
_v_aggregate, _left/_right/_top/_bottom_aggregate), flip_merge (and so the *_flip_from_logits
wrappers) and ctdet_decode_from_host: they read bf16 and fp16 heads in place, and return, bit
for bit, what they return for the .float() upcast.  The work is done by
the hand-written sm_90a kernels behind ``include/centernet_b200.h``; there is no
CPU path (non-CUDA inputs raise NotImplementedError).

Tie order, which the reference leaves to torch.topk, is defined here as
(score desc, flat index cls*H*W + y*W + x asc).
"""
import torch

from ._lib import C, dtype_code, f32c, floatc, ptr, require_cuda, stream_ptr, workspace
from .utils import _gather_feat, _transpose_and_gather_feat  # noqa: F401  (re-exported like the reference)


def _dims(t):
    b, c, h, w = t.shape
    return int(b), int(c), int(h), int(w)


# ------------------------------------------------------------------ decode.py:9-15
def _nms(heat, kernel=3):
    if kernel != 3:
        raise NotImplementedError("_nms: only the 3x3 kernel the reference uses is implemented")
    require_cuda(heat, what="_nms")
    heat = f32c(heat)
    b, c, h, w = _dims(heat)
    out = torch.empty_like(heat)
    if heat.numel():
        C.nms(ptr(heat), ptr(out), b, c, h, w, stream_ptr(heat))
    return out


# ------------------------------------------------------------------ decode.py:17-77
def _aggregate(heat, aggr_weight, horizontal):
    require_cuda(heat, what="_aggregate")
    heat = floatc(heat)
    b, c, h, w = _dims(heat)
    out = torch.empty(heat.shape, dtype=torch.float32, device=heat.device)
    if heat.dtype == torch.float32:
        C.edge_aggregate(ptr(heat), ptr(out), b, c, h, w, float(aggr_weight), int(horizontal), stream_ptr(heat))
    else:  # a bf16 / fp16 map is read in place; the fp32 result equals that of its .float() upcast
        C.edge_aggregate_ex(ptr(heat), dtype_code(heat), 0, ptr(out), b, c, h, w, float(aggr_weight), int(horizontal),
                            stream_ptr(heat))
    return out


def _h_aggregate(heat, aggr_weight=0.1):
    """decode.py:71-73: aggr_weight*left + aggr_weight*right + heat (one fused scan kernel)."""
    return _aggregate(heat, aggr_weight, True)


def _v_aggregate(heat, aggr_weight=0.1):
    """decode.py:75-77."""
    return _aggregate(heat, aggr_weight, False)


def _left_aggregate(heat):
    """decode.py:17-28.  Derived from the fused kernel's directional outputs."""
    return _directional(heat, 0)


def _right_aggregate(heat):
    """decode.py:30-41."""
    return _directional(heat, 1)


def _top_aggregate(heat):
    """decode.py:43-55."""
    return _directional(heat, 2)


def _bottom_aggregate(heat):
    """decode.py:57-69."""
    return _directional(heat, 3)


def _directional(heat, direction):
    # weight=1 with the opposite direction disabled is encoded as horizontal = 2 + direction
    return _aggregate(heat, 1.0, 2 + direction)


# ------------------------------------------------------------------ decode.py:92-119
def _topk_channel(scores, K=40):
    require_cuda(scores, what="_topk_channel")
    scores = f32c(scores)
    b, c, h, w = _dims(scores)
    dev = scores.device
    s = torch.empty((b, c, K), dtype=torch.float32, device=dev)
    inds = torch.empty((b, c, K), dtype=torch.int64, device=dev)
    ys = torch.empty((b, c, K), dtype=torch.float32, device=dev)
    xs = torch.empty((b, c, K), dtype=torch.float32, device=dev)
    nb = C.topk_workspace_bytes(b * c, 1, h, w, K)
    ws = workspace(nb, dev)
    C.topk_channel(ptr(scores), b, c, h, w, K, 0, ptr(s), ptr(inds), ptr(ys), ptr(xs), ptr(ws), ws.numel(),
                   stream_ptr(scores))
    return s, inds, ys, xs


def _topk(scores, K=40):
    require_cuda(scores, what="_topk")
    scores = f32c(scores)
    b, c, h, w = _dims(scores)
    dev = scores.device
    s = torch.empty((b, K), dtype=torch.float32, device=dev)
    inds = torch.empty((b, K), dtype=torch.int64, device=dev)
    clses = torch.empty((b, K), dtype=torch.int32, device=dev)
    ys = torch.empty((b, K), dtype=torch.float32, device=dev)
    xs = torch.empty((b, K), dtype=torch.float32, device=dev)
    nb = C.topk_workspace_bytes(b, c, h, w, K)
    ws = workspace(nb, dev)
    C.topk(ptr(scores), b, c, h, w, K, 0, ptr(s), ptr(inds), ptr(clses), ptr(ys), ptr(xs), ptr(ws), ws.numel(),
           stream_ptr(scores))
    return s, inds, clses, ys, xs


# ------------------------------------------------------------------ decode.py:464-495
def _all_f32(*tensors):
    return all(t is None or t.dtype == torch.float32 for t in tensors)


def _decode_ex(heat, wh, reg, cat_spec_wh, K, logits, dets):
    """cnb_ctdet_decode_ex: heat / wh / reg each fp32, fp16 or bf16."""
    b, c, h, w = _dims(heat)
    ws = workspace(C.ctdet_decode_ex_workspace_bytes(ptr(heat), dtype_code(heat), logits, b, c, h, w, K), heat.device)
    C.ctdet_decode_ex(ptr(heat), dtype_code(heat), logits, ptr(wh), dtype_code(wh), ptr(reg), dtype_code(reg),
                      int(bool(cat_spec_wh)), b, c, h, w, K, ptr(dets), ptr(ws), ws.numel(), stream_ptr(heat))
    return dets


def ctdet_decode(heat, wh, reg=None, cat_spec_wh=False, K=100):
    """bf16 / fp16 heat, wh and reg (each its own dtype) are read in place: the dets equal, bit for bit, those of
    the .float() upcast."""
    require_cuda(heat, wh, reg, what="ctdet_decode")
    heat, wh, reg = floatc(heat), floatc(wh), floatc(reg)
    b, c, h, w = _dims(heat)
    want = 2 * c if cat_spec_wh else 2
    if wh.shape[0] != b or wh.shape[1] != want or tuple(wh.shape[2:]) != (h, w):
        raise RuntimeError("ctdet_decode: wh must be [%d, %d, %d, %d], got %s" % (b, want, h, w, tuple(wh.shape)))
    if reg is not None and tuple(reg.shape) != (b, 2, h, w):
        raise RuntimeError("ctdet_decode: reg must be [%d, 2, %d, %d], got %s" % (b, h, w, tuple(reg.shape)))
    dets = torch.empty((b, K, 6), dtype=torch.float32, device=heat.device)
    if not _all_f32(heat, wh, reg):
        return _decode_ex(heat, wh, reg, cat_spec_wh, K, 0, dets)
    ws = workspace(C.topk_workspace_bytes(b, c, h, w, K), heat.device)
    C.ctdet_decode(ptr(heat), ptr(wh), ptr(reg), int(bool(cat_spec_wh)), b, c, h, w, K, ptr(dets), ptr(ws),
                   ws.numel(), stream_ptr(heat))
    return dets


def ctdet_decode_from_logits(hm, wh, reg=None, cat_spec_wh=False, K=100):
    """`ctdet_decode(hm.sigmoid_(), wh, reg, ...)` (detectors/ctdet.py:30-45) in one launch, reading the
    head's raw logits: the selection runs in logit space (the sigmoid is monotone) and only the
    candidates are pushed through 1/(1+exp(-x)).  Scores are bit-identical to torch's CUDA sigmoid,
    indices / classes / boxes identical to ctdet_decode on that heat map; `hm` is not modified.
    bf16 / fp16 logits (and wh / reg) are read in place and scored with the fp32 sigmoid of the widened logit, so
    the dets equal those of the .float() upcast (the reference's `hm.sigmoid_()` on a half tensor would round the
    scores to half precision first)."""
    require_cuda(hm, wh, reg, what="ctdet_decode_from_logits")
    hm, wh, reg = floatc(hm), floatc(wh), floatc(reg)
    b, c, h, w = _dims(hm)
    want = 2 * c if cat_spec_wh else 2
    if wh.shape[0] != b or wh.shape[1] != want or tuple(wh.shape[2:]) != (h, w):
        raise RuntimeError("ctdet_decode_from_logits: wh must be [%d, %d, %d, %d], got %s" % (b, want, h, w, tuple(wh.shape)))
    if reg is not None and tuple(reg.shape) != (b, 2, h, w):
        raise RuntimeError("ctdet_decode_from_logits: reg must be [%d, 2, %d, %d], got %s" % (b, h, w, tuple(reg.shape)))
    dets = torch.empty((b, K, 6), dtype=torch.float32, device=hm.device)
    if not _all_f32(hm, wh, reg):
        return _decode_ex(hm, wh, reg, cat_spec_wh, K, 1, dets)
    ws = workspace(C.ctdet_logits_workspace_bytes(ptr(hm), b, c, h, w, K), hm.device)
    C.ctdet_decode_logits(ptr(hm), ptr(wh), ptr(reg), int(bool(cat_spec_wh)), b, c, h, w, K, ptr(dets), ptr(ws),
                          ws.numel(), stream_ptr(hm))
    return dets


def sigmoid(x):
    """Bare sigmoid (detectors/ctdet.py:31) through the library's own kernel; returns a new tensor."""
    require_cuda(x, what="sigmoid")
    x = f32c(x)
    out = torch.empty_like(x)
    C.sigmoid(ptr(x), ptr(out), x.numel(), stream_ptr(x))
    return out


# ------------------------------------------------------------------ flip test (detectors/*.py), N1
def flip_merge(x, sigmoid=False, flip_idx=None, offsets=False):
    """(f(x[:n]) + flip(f(x[n:]))) / 2 for a batch x [2n, C, H, W] = n images followed by their mirrored copies
    (base_detector.py:63-64).  flip: flip_tensor; with `flip_idx` the joint channels are swapped as in flip_lr
    (models/utils.py:33-39), with `offsets` as in flip_lr_off (:41-50: C = 2 x joints, x offsets negated).
    One kernel, no host round trip (the reference's flip_lr / flip_lr_off go through numpy).  A bf16 / fp16 x is
    read in place (widened exactly); the result is fp32 either way."""
    require_cuda(x, what="flip_merge")
    x = floatc(x)
    b2, c, h, w = _dims(x)
    if b2 % 2:
        raise RuntimeError("flip_merge: batch must hold image / mirrored-image pairs")
    n = b2 // 2
    perm = sign = None
    if flip_idx is not None:
        if offsets:
            j = c // 2
            p = list(range(j))
            for a, b_ in flip_idx:
                p[a], p[b_] = p[b_], p[a]
            perm = torch.tensor([2 * p[ch // 2] + (ch & 1) for ch in range(c)], dtype=torch.int32, device=x.device)
            sign = torch.tensor([-1.0 if (ch & 1) == 0 else 1.0 for ch in range(c)], dtype=torch.float32, device=x.device)
        else:
            p = list(range(c))
            for a, b_ in flip_idx:
                p[a], p[b_] = p[b_], p[a]
            perm = torch.tensor(p, dtype=torch.int32, device=x.device)
    out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    if x.dtype == torch.float32:
        C.flip_merge(ptr(x), ptr(out), n, c, h, w, int(bool(sigmoid)), ptr(perm), ptr(sign), stream_ptr(x))
    else:
        C.flip_merge_ex(ptr(x), dtype_code(x), ptr(out), n, c, h, w, int(bool(sigmoid)), ptr(perm), ptr(sign),
                        stream_ptr(x))
    return out


def ctdet_decode_flip_from_logits(hm, wh, reg=None, cat_spec_wh=False, K=100):
    """detectors/ctdet.py:30-45 with --flip_test: hm/wh/reg [2n, ...] (images then mirrored images) ->
    dets [n, K, 6].  Two launches (merge of hm + wh, fused decode) instead of ~10 ATen ops + the decode."""
    heat = flip_merge(hm, sigmoid=True)
    whm = flip_merge(wh)
    n = heat.shape[0]
    return ctdet_decode(heat, whm, reg=None if reg is None else reg[:n], cat_spec_wh=cat_spec_wh, K=K)


def multi_pose_decode_flip_from_logits(hm, wh, hps, reg=None, hm_hp=None, hp_offset=None, flip_idx=(), K=100):
    """detectors/multi_pose.py:29-55 with --flip_test (hm and hm_hp given as logits)."""
    heat = flip_merge(hm, sigmoid=True)
    n = heat.shape[0]
    hm_hp_m = None if hm_hp is None else flip_merge(hm_hp, sigmoid=True, flip_idx=flip_idx)
    return multi_pose_decode(heat, flip_merge(wh), flip_merge(hps, flip_idx=flip_idx, offsets=True),
                             reg=None if reg is None else reg[:n], hm_hp=hm_hp_m,
                             hp_offset=None if hp_offset is None else hp_offset[:n], K=K)


# ------------------------------------------------------------------ decode.py:426-462
def _ddd_heads(what, heat, rot, depth, dim, wh, reg):
    require_cuda(heat, rot, depth, dim, wh, reg, what=what)
    heads = [floatc(t) for t in (heat, rot, depth, dim, wh, reg)]
    b, c, h, w = _dims(heads[0])
    for name, t, ch in zip(("rot", "depth", "dim", "wh", "reg"), heads[1:], (8, 1, 3, 2, 2)):
        if t is not None and tuple(t.shape) != (b, ch, h, w):
            raise RuntimeError("%s: %s must be [%d, %d, %d, %d], got %s" % (what, name, b, ch, h, w, tuple(t.shape)))
    return heads


def _ddd_ex(heat, rot, depth, dim, wh, reg, K, logits):
    """cnb_ddd_decode_ex: every head fp32, fp16 or bf16."""
    b, c, h, w = _dims(heat)
    dets = torch.empty((b, K, 18 if wh is not None else 16), dtype=torch.float32, device=heat.device)
    ws = workspace(C.ddd_decode_ex_workspace_bytes(ptr(heat), dtype_code(heat), logits, b, c, h, w, K), heat.device)
    C.ddd_decode_ex(ptr(heat), dtype_code(heat), logits, ptr(rot), dtype_code(rot), ptr(depth), dtype_code(depth),
                    ptr(dim), dtype_code(dim), ptr(wh), dtype_code(wh), ptr(reg), dtype_code(reg), b, c, h, w, K,
                    ptr(dets), ptr(ws), ws.numel(), stream_ptr(heat))
    return dets


def ddd_decode(heat, rot, depth, dim, wh=None, reg=None, K=40):
    """bf16 / fp16 heads (each its own dtype) are read in place: the dets equal, bit for bit, those of the .float()
    upcast."""
    heat, rot, depth, dim, wh, reg = _ddd_heads("ddd_decode", heat, rot, depth, dim, wh, reg)
    if not _all_f32(heat, rot, depth, dim, wh, reg):
        return _ddd_ex(heat, rot, depth, dim, wh, reg, K, 0)
    b, c, h, w = _dims(heat)
    dets = torch.empty((b, K, 18 if wh is not None else 16), dtype=torch.float32, device=heat.device)
    ws = workspace(C.topk_workspace_bytes(b, c, h, w, K), heat.device)
    C.ddd_decode(ptr(heat), ptr(rot), ptr(depth), ptr(dim), ptr(wh), ptr(reg), b, c, h, w, K, ptr(dets), ptr(ws),
                 ws.numel(), stream_ptr(heat))
    return dets


def ddd_decode_from_logits(hm, rot, dep, dim, wh=None, reg=None, K=40):
    """`ddd_decode(hm.sigmoid_(), rot, 1. / (dep.sigmoid() + 1e-6) - 1., dim, wh, reg, K)` (detectors/ddd.py:61-68)
    on the heads' raw outputs: hm is selected through its sigmoid, and the depth transform runs, in torch's op order,
    at the K selected positions only.  The dets equal, bit for bit, those of ddd_decode on torch's CUDA sigmoid of hm
    and torch's transform of dep; no input is modified.  bf16 / fp16 heads are read in place, widened exactly and
    processed as fp32 (the reference's ops on a half tensor would round every step to half precision)."""
    hm, rot, dep, dim, wh, reg = _ddd_heads("ddd_decode_from_logits", hm, rot, dep, dim, wh, reg)
    return _ddd_ex(hm, rot, dep, dim, wh, reg, K, 1)


# ------------------------------------------------------------------ decode.py:497-571
def _pose_heads(what, heat, wh, kps, reg, hm_hp, hp_offset):
    require_cuda(heat, wh, kps, reg, hm_hp, hp_offset, what=what)
    heads = [floatc(t) for t in (heat, wh, kps, reg, hm_hp, hp_offset)]
    b, c, h, w = _dims(heads[0])
    j = int(heads[2].shape[1]) // 2
    for name, t, ch in zip(("wh", "kps", "reg", "hm_hp", "hp_offset"), heads[1:], (2, 2 * j, 2, j, 2)):
        if t is not None and tuple(t.shape) != (b, ch, h, w):
            raise RuntimeError("%s: %s must be [%d, %d, %d, %d], got %s" % (what, name, b, ch, h, w, tuple(t.shape)))
    return heads


def _multi_pose_ex(heat, wh, kps, reg, hm_hp, hp_offset, K, logits):
    """cnb_multi_pose_decode_ex: every head fp32, fp16 or bf16."""
    b, c, h, w = _dims(heat)
    j = int(kps.shape[1]) // 2
    dets = torch.empty((b, K, 4 + 1 + 2 * j + 1), dtype=torch.float32, device=heat.device)
    nb = C.multi_pose_decode_ex_workspace_bytes(ptr(heat), dtype_code(heat), ptr(hm_hp), dtype_code(hm_hp), logits,
                                                b, c, j, h, w, K)
    ws = workspace(nb, heat.device)
    C.multi_pose_decode_ex(ptr(heat), dtype_code(heat), logits, ptr(wh), dtype_code(wh), ptr(kps), dtype_code(kps),
                           ptr(reg), dtype_code(reg), ptr(hm_hp), dtype_code(hm_hp), ptr(hp_offset),
                           dtype_code(hp_offset), b, c, j, h, w, K, ptr(dets), ptr(ws), ws.numel(), stream_ptr(heat))
    return dets


def multi_pose_decode(heat, wh, kps, reg=None, hm_hp=None, hp_offset=None, K=100):
    """bf16 / fp16 heads (each its own dtype) are read in place: the dets equal, bit for bit, those of the .float()
    upcast."""
    heat, wh, kps, reg, hm_hp, hp_offset = _pose_heads("multi_pose_decode", heat, wh, kps, reg, hm_hp, hp_offset)
    if not _all_f32(heat, wh, kps, reg, hm_hp, hp_offset):
        return _multi_pose_ex(heat, wh, kps, reg, hm_hp, hp_offset, K, 0)
    b, c, h, w = _dims(heat)
    j = int(kps.shape[1]) // 2
    dets = torch.empty((b, K, 4 + 1 + 2 * j + 1), dtype=torch.float32, device=heat.device)
    ws = workspace(C.multi_pose_workspace_bytes(b, c, j, h, w, K), heat.device)
    C.multi_pose_decode(ptr(heat), ptr(wh), ptr(kps), ptr(reg), ptr(hm_hp), ptr(hp_offset), b, c, j, h, w, K,
                        ptr(dets), ptr(ws), ws.numel(), stream_ptr(heat))
    return dets


def multi_pose_decode_from_logits(hm, wh, hps, reg=None, hm_hp=None, hp_offset=None, K=100):
    """`multi_pose_decode(hm.sigmoid_(), wh, hps, reg, hm_hp.sigmoid_(), hp_offset, K)` (detectors/multi_pose.py:
    33-35,53) on the raw logits of hm and hm_hp, without the two full-map sigmoid passes: in the hot geometry both
    selections run in logit space and only the candidates go through the sigmoid.  The dets equal, bit for bit, those
    of multi_pose_decode on torch's CUDA sigmoid of hm and hm_hp; no input is modified.  bf16 / fp16 heads are read in
    place, widened exactly and processed as fp32 (the reference's `sigmoid_()` on a half tensor would round the scores
    to half precision first)."""
    heads = _pose_heads("multi_pose_decode_from_logits", hm, wh, hps, reg, hm_hp, hp_offset)
    return _multi_pose_ex(*heads, K, 1)


# ------------------------------------------------------------------ decode.py:122-424
def _exct(t_heat, l_heat, b_heat, r_heat, ct_heat, regs, K, scores_thresh, center_thresh, aggr_weight, num_dets,
          agnostic, name, logits=0):
    require_cuda(t_heat, l_heat, b_heat, r_heat, ct_heat, *regs, what=name)
    t_heat, l_heat, b_heat, r_heat, ct_heat = [floatc(t) for t in (t_heat, l_heat, b_heat, r_heat, ct_heat)]
    b, c, h, w = _dims(t_heat)
    cc = int(ct_heat.shape[1])
    for t in (l_heat, b_heat, r_heat):
        if tuple(t.shape) != (b, c, h, w):
            raise RuntimeError("%s: extreme-point heat maps must share one shape" % name)
    if all(r is not None for r in regs):  # decode.py:366-367: all four or none
        regs = [floatc(r) for r in regs]
    else:
        regs = [None] * 4
    dets = torch.empty((b, num_dets, 14), dtype=torch.float32, device=t_heat.device)
    maps = (t_heat, l_heat, b_heat, r_heat)
    if logits or not _all_f32(*maps, ct_heat, *regs):  # cnb_exct_decode_ex: each input its own dtype
        inputs = maps + (ct_heat,) + tuple(regs)
        codes = [dtype_code(t) for t in inputs]
        nb = C.exct_decode_ex_workspace_bytes(*[ptr(t) for t in maps], *codes, int(logits), b, c, cc, h, w, K,
                                              float(aggr_weight), int(num_dets), int(agnostic))
        ws = workspace(nb, t_heat.device)
        C.exct_decode_ex(*[a for t, dt in zip(inputs, codes) for a in (ptr(t), dt)], int(logits), b, c, cc, h, w, K,
                         float(scores_thresh), float(center_thresh), float(aggr_weight), int(num_dets), int(agnostic),
                         ptr(dets), ptr(ws), ws.numel(), stream_ptr(t_heat))
        return dets
    ws = workspace(C.exct_workspace_bytes(b, c, cc, h, w, K, num_dets), t_heat.device)
    C.exct_decode(ptr(t_heat), ptr(l_heat), ptr(b_heat), ptr(r_heat), ptr(ct_heat), ptr(regs[0]), ptr(regs[1]),
                  ptr(regs[2]), ptr(regs[3]), b, c, cc, h, w, K, float(scores_thresh), float(center_thresh),
                  float(aggr_weight), int(num_dets), int(agnostic), ptr(dets), ptr(ws), ws.numel(),
                  stream_ptr(t_heat))
    return dets


def agnex_ct_decode(t_heat, l_heat, b_heat, r_heat, ct_heat, t_regr=None, l_regr=None, b_regr=None, r_regr=None,
                    K=40, scores_thresh=0.1, center_thresh=0.1, aggr_weight=0.0, num_dets=1000):
    """bf16 / fp16 maps and regression heads (each its own dtype) are read in place: the dets equal, bit for bit,
    those of the .float() upcast."""
    return _exct(t_heat, l_heat, b_heat, r_heat, ct_heat, (t_regr, l_regr, b_regr, r_regr), K, scores_thresh,
                 center_thresh, aggr_weight, num_dets, True, "agnex_ct_decode")


def exct_decode(t_heat, l_heat, b_heat, r_heat, ct_heat, t_regr=None, l_regr=None, b_regr=None, r_regr=None,
                K=40, scores_thresh=0.1, center_thresh=0.1, aggr_weight=0.0, num_dets=1000):
    """bf16 / fp16 maps and regression heads (each its own dtype) are read in place: the dets equal, bit for bit,
    those of the .float() upcast."""
    return _exct(t_heat, l_heat, b_heat, r_heat, ct_heat, (t_regr, l_regr, b_regr, r_regr), K, scores_thresh,
                 center_thresh, aggr_weight, num_dets, False, "exct_decode")


def agnex_ct_decode_from_logits(t, l, b, r, ct, t_regr=None, l_regr=None, b_regr=None, r_regr=None, K=40,
                                scores_thresh=0.1, center_thresh=0.1, aggr_weight=0.0, num_dets=1000):
    """`agnex_ct_decode` on torch's sigmoid of the five maps, read as raw logits; see exct_decode_from_logits."""
    return _exct(t, l, b, r, ct, (t_regr, l_regr, b_regr, r_regr), K, scores_thresh, center_thresh, aggr_weight,
                 num_dets, True, "agnex_ct_decode_from_logits", logits=1)


def exct_decode_from_logits(t, l, b, r, ct, t_regr=None, l_regr=None, b_regr=None, r_regr=None, K=40,
                            scores_thresh=0.1, center_thresh=0.1, aggr_weight=0.0, num_dets=1000):
    """`exct_decode(t.sigmoid_(), l.sigmoid_(), b.sigmoid_(), r.sigmoid_(), ct.sigmoid_(), ...)` (detectors/exdet.py:
    32-36) on the raw logits of the five maps, without the five full-map sigmoid passes: in the hot geometry the four
    selections run in logit space, and the edge aggregation and the centre map apply the sigmoid as they load.  The
    dets equal, bit for bit and filler rows included, those of exct_decode on torch's CUDA sigmoid of the five maps;
    no input is modified.  bf16 / fp16 inputs are read in place, widened exactly and processed as fp32 (the
    reference's `sigmoid_()` on a half tensor would round the scores to half precision first)."""
    return _exct(t, l, b, r, ct, (t_regr, l_regr, b_regr, r_regr), K, scores_thresh, center_thresh, aggr_weight,
                 num_dets, False, "exct_decode_from_logits", logits=1)


# ------------------------------------------------------------------ host-buffer entry (end-to-end path)
import threading

_HOST_TLS = threading.local()   # staging buffers, events and the copy stream are PER THREAD (one thread per GPU
                                # in DataParallel-style callers): nothing here is shared between threads


def ctdet_decode_from_host(heat, wh, reg=None, cat_spec_wh=False, K=100, chunk=8, device=None):
    """ctdet_decode for HOST tensors (pinned memory recommended): the batch is cut into
    `chunk`-image pieces whose H2D copies run on a side stream, double-buffered against the
    decode kernels of the previous piece; the [B, K, 6] detections come back in pinned host
    memory.  This is the call a detector makes when the heat maps are produced off-device
    (and what bench.py times as `e2e`).  Same semantics as ctdet_decode: the result is a FRESH host
    tensor the caller owns (the pinned staging buffer is copied out, 2.4 KB per image).  bf16 / fp16 host
    tensors are staged in their own dtype (no CPU-side conversion, half the bytes over PCIe) and decoded in
    place."""
    if heat.is_cuda:
        return ctdet_decode(heat, wh, reg=reg, cat_spec_wh=cat_spec_wh, K=K).cpu()
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    heat, wh, reg = floatc(heat), floatc(wh), floatc(reg)
    b, c, h, w = _dims(heat)
    chunk = max(1, min(chunk, b))
    native = _all_f32(heat, wh, reg)
    key = (dev.index, c, h, w, int(wh.shape[1]), reg is not None, chunk, b, K, heat.dtype, wh.dtype,
           None if reg is None else reg.dtype)
    cache = getattr(_HOST_TLS, "ctx", None)
    if cache is None:
        cache = _HOST_TLS.ctx = {}
    ctx = cache.get(key)
    if ctx is None:
        ctx = {
            "copy": torch.cuda.Stream(device=dev),
            "heat": [torch.empty((chunk, c, h, w), dtype=heat.dtype, device=dev) for _ in range(2)],
            "wh": [torch.empty((chunk, int(wh.shape[1]), h, w), dtype=wh.dtype, device=dev) for _ in range(2)],
            "reg": [torch.empty((chunk, 2, h, w), dtype=reg.dtype, device=dev) for _ in range(2)]
                   if reg is not None else [None, None],
            "dets": torch.empty((b, K, 6), dtype=torch.float32, device=dev),
            "out": torch.empty((b, K, 6), dtype=torch.float32).pin_memory(),
            "free": [torch.cuda.Event(), torch.cuda.Event()],
            "ready": [torch.cuda.Event(), torch.cuda.Event()],
        }
        if native:
            ctx["ws"] = workspace(C.topk_workspace_bytes(chunk, c, h, w, K), dev)
        else:  # the staging buffers are fresh allocations: both slots share one alignment and so one path
            hp = ptr(ctx["heat"][0])
            ctx["ws"] = workspace(max(C.ctdet_decode_ex_workspace_bytes(hp, dtype_code(heat), 0, n, c, h, w, K)
                                      for n in {chunk, b % chunk or chunk}), dev)
        cache.clear()  # keep one geometry resident per thread
        cache[key] = ctx
    main = torch.cuda.current_stream(dev)
    copy = ctx["copy"]
    copy.wait_stream(main)
    for i, s in enumerate(range(0, b, chunk)):
        n = min(chunk, b - s)
        slot = i & 1
        with torch.cuda.stream(copy):
            if i >= 2:
                copy.wait_event(ctx["free"][slot])
            ctx["heat"][slot][:n].copy_(heat[s:s + n], non_blocking=True)
            ctx["wh"][slot][:n].copy_(wh[s:s + n], non_blocking=True)
            if reg is not None:
                ctx["reg"][slot][:n].copy_(reg[s:s + n], non_blocking=True)
            ctx["ready"][slot].record(copy)
        main.wait_event(ctx["ready"][slot])
        dets = ctx["dets"][s:s + n]
        if native:
            C.ctdet_decode(ptr(ctx["heat"][slot]), ptr(ctx["wh"][slot]), ptr(ctx["reg"][slot]),
                           int(bool(cat_spec_wh)), n, c, h, w, K, ptr(dets), ptr(ctx["ws"]), ctx["ws"].numel(),
                           main.cuda_stream)
        else:
            C.ctdet_decode_ex(ptr(ctx["heat"][slot]), dtype_code(heat), 0, ptr(ctx["wh"][slot]), dtype_code(wh),
                              ptr(ctx["reg"][slot]), dtype_code(reg), int(bool(cat_spec_wh)), n, c, h, w, K,
                              ptr(dets), ptr(ctx["ws"]), ctx["ws"].numel(), main.cuda_stream)
        ctx["free"][slot].record(main)
    ctx["out"].copy_(ctx["dets"], non_blocking=True)
    main.synchronize()
    return ctx["out"].clone()

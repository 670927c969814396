"""torch restatement of the heat-map selection: _nms + _topk + the ctdet epilogue (TEST INFRASTRUCTURE).

Runs on CPU and on CUDA tensors, so the large-batch cases of the selection tests (B=64, C=80 at 128x128 and up)
get an independent answer in milliseconds where the numpy oracle would take minutes.  It follows
``oracle/decode_np.py`` (and through it ``models/decode.py:9-15, 92-119, 464-495``):

* ``_nms``: ``max_pool2d(3, 1, 1)`` (-inf padding), ``keep = hmax == heat``, ``heat * keep``;
* ``_topk``: ONE stable descending sort of each image's flattened ``C*H*W`` map.  Stability gives the tie rule the
  library defines (score desc, flat index ``cls*H*W + y*W + x`` asc), and under that total order the reference's
  per-class top-K followed by the top-K of the ``C*K`` survivors is the same as one global top-K;
* ``-0.0`` is canonicalised to ``+0.0`` before the sort: a radix sort on the float bits would put ``+0`` before
  ``-0``, while the reference, the numpy oracle and the kernel treat the two as one value ordered by index;
* the ctdet box columns use the reference's own operations (``xs + reg``, ``wh / 2``, ``xs - half_w``), each one
  fp32 rounding, so they agree bit for bit with any implementation that performs the same operations.

Non-finite scores.  The reference's answer is not usable (``max_pool2d`` propagates NaN, ``-inf * 0`` is NaN, and
``torch.topk`` then ranks NaN first), so the library defines its own rule (DESIGN.md, "Non-finite scores"), which
``nonfinite="library"`` applies:

* a NaN pixel scores 0 (a zero filler, in index order) and is left out of its neighbours' 3x3 maximum;
* a ``-inf`` that is not a 3x3 peak scores 0; a ``-inf`` peak scores ``-inf``;
* ``+inf`` peaks (and ``+inf`` plateaus) score ``+inf``, ties by index like any other value.

``nonfinite="reference"`` (the default) is the reference's arithmetic, meant for finite maps.
"""
import torch
import torch.nn.functional as F


def nms(heat, nonfinite="reference"):
    """heat * keep of models/decode.py:9-15 for an [N, C, H, W] float32 tensor."""
    heat = heat.float()
    if nonfinite == "reference":
        hmax = F.max_pool2d(heat, 3, stride=1, padding=1)
        return heat * (hmax == heat).float()
    if nonfinite != "library":
        raise ValueError("nonfinite must be 'reference' or 'library'")
    nan = torch.isnan(heat)
    hmax = F.max_pool2d(heat.masked_fill(nan, float("-inf")), 3, stride=1, padding=1)
    keep = (hmax == heat) & ~nan
    return torch.where(keep, heat, torch.zeros_like(heat))


def _select(flat, K):
    """Top-K of the last axis under (value desc, index asc); returns (values, indices)."""
    flat = flat + 0.0                                    # -0.0 -> +0.0 (and a copy)
    vals, order = torch.sort(flat, dim=-1, descending=True, stable=True)
    return vals[..., :K].contiguous(), order[..., :K].contiguous()


def topk(scores, K):
    """models/decode.py:103-119 (_topk) on an already NMS'd [B, C, H, W] map:
    (scores, inds = y*W + x, clses int32, ys, xs)."""
    B, C, H, W = scores.shape
    s, flat = _select(scores.reshape(B, C * H * W), K)
    inds = flat % (H * W)
    return s, inds, (flat // (H * W)).int(), (inds // W).float(), (inds % W).float()


def topk_channel(scores, K):
    """models/decode.py:92-101 (_topk_channel): (scores, inds, ys, xs), each [B, C, K]."""
    B, C, H, W = scores.shape
    s, inds = _select(scores.reshape(B, C, H * W), K)
    return s, inds, (inds // W).float(), (inds % W).float()


def _gather(feat, sp):
    """feat[b, ch, sp[b, k]] for every channel: [B, ch, HW] x [B, K] -> [B, K, ch]."""
    B, D = feat.shape[:2]
    f = feat.reshape(B, D, -1)
    return torch.gather(f, 2, sp[:, None, :].expand(B, D, sp.shape[1])).transpose(1, 2)


def ctdet_decode(heat, wh, reg=None, cat_spec_wh=False, K=100, nonfinite="reference"):
    """models/decode.py:464-495 -> dets [B, K, 6] = x1, y1, x2, y2, score, class (float32).
    heat / wh / reg may be fp32, fp16 or bf16; each is widened exactly to fp32 first."""
    heat = heat.float()
    B, C, H, W = heat.shape
    scores, inds, clses, ys, xs = topk(nms(heat, nonfinite), K)
    if reg is not None:
        r = _gather(reg.float(), inds)
        xs = xs + r[..., 0]
        ys = ys + r[..., 1]
    else:
        xs = xs + 0.5
        ys = ys + 0.5
    w = _gather(wh.float(), inds)                        # [B, K, 2] or [B, K, 2C]
    if cat_spec_wh:
        c = clses.long()
        w = torch.stack([torch.gather(w, 2, (2 * c)[..., None])[..., 0],
                         torch.gather(w, 2, (2 * c + 1)[..., None])[..., 0]], dim=-1)
    half_w = w[..., 0] / 2
    half_h = w[..., 1] / 2
    return torch.stack([xs - half_w, ys - half_h, xs + half_w, ys + half_h, scores, clses.float()], dim=-1)

"""Shared test helpers: golden loading, bit and tie-aware detection comparison, and the training samplers' stubs."""
import os
import random
import zlib

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    return {k: z[k] for k in z.files}


def assert_dets_equal(ref, got, score_col=4, atol=0.0, positive_only=False, what=""):
    """Detections [B, K, D] sorted by score desc.  Rows are compared as multisets inside
    every run of equal scores (torch.topk leaves that order open).  With positive_only
    rows whose reference score is <= 0 (non-peak fillers) are only required to have the
    same score."""
    ref = np.asarray(ref); got = np.asarray(got)
    assert ref.shape == got.shape, (what, ref.shape, got.shape)
    for b in range(ref.shape[0]):
        rs, gs = ref[b, :, score_col], got[b, :, score_col]
        np.testing.assert_array_equal(rs, gs, err_msg="%s: scores differ (image %d)" % (what, b))
        k = 0
        K = ref.shape[1]
        while k < K:
            e = k
            while e + 1 < K and rs[e + 1] == rs[k]:
                e += 1
            if positive_only and rs[k] <= 0:
                k = e + 1
                continue
            a = ref[b, k:e + 1]; c = got[b, k:e + 1]
            if e > k:  # tie group: order-free
                a = a[np.lexsort(a.T[::-1])]; c = c[np.lexsort(c.T[::-1])]
            if atol == 0.0:
                np.testing.assert_array_equal(a, c, err_msg="%s: rows %d..%d image %d" % (what, k, e, b))
            else:
                np.testing.assert_allclose(a, c, rtol=0, atol=atol, err_msg="%s: rows %d..%d image %d" % (what, k, e, b))
            k = e + 1


def canonical_bits(a):
    """float32 -> its uint32 bits, with every NaN (any sign, any payload) mapped to the one NaN 0x7fc00000."""
    a = np.asarray(a, np.float32)
    u = np.ascontiguousarray(a).view(np.uint32).copy()
    u[np.isnan(a)] = 0x7fc00000
    return u


def assert_dets_bits(ref, got, score_col=4, what=""):
    """assert_dets_equal without any tolerance at the bit level: every float equal as canonical_bits (so -0 differs
    from +0 and NaN matches NaN); rows compared as multisets inside every run of equal scores."""
    ref, got = canonical_bits(ref), canonical_bits(got)
    assert ref.shape == got.shape, (what, ref.shape, got.shape)
    for b in range(ref.shape[0]):
        rs = ref[b, :, score_col]
        np.testing.assert_array_equal(got[b, :, score_col], rs, err_msg="%s: scores differ (image %d)" % (what, b))
        k, K = 0, ref.shape[1]
        while k < K:
            e = k
            while e + 1 < K and rs[e + 1] == rs[k]:
                e += 1
            a, c = ref[b, k:e + 1], got[b, k:e + 1]
            if e > k:
                a = a[np.lexsort(a.T[::-1])]; c = c[np.lexsort(c.T[::-1])]
            if not np.array_equal(a, c):
                i = np.argwhere(a != c)[0]
                raise AssertionError("%s: image %d rows %d..%d differ, first at row %d column %d: got %r, want %r"
                                     % (what, b, k, e, k + i[0], i[1], c[tuple(i)].view(np.float32),
                                        a[tuple(i)].view(np.float32)))
            k = e + 1


def assert_same_bits(got, want, what=""):
    """float32 arrays equal bit for bit (the sign of zero included); NaN matches NaN of any sign or payload (the
    device's canonical NaN and x86's default NaN differ in their bits, not in what they mean)."""
    got = np.asarray(got, np.float32); want = np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    bad = (gn != wn) | (~gn & ~wn & (got.view(np.uint32) != want.view(np.uint32)))
    if bad.any():
        idx = np.argwhere(bad)
        i = tuple(idx[0])
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r, want %r"
                             % (what, len(idx), bad.size, i, got[i], want[i]))


def assert_bits(got, want, what):
    """Same dtype, same shape and the same bytes (NaN payloads and the sign of zero included)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, got.shape, want.dtype, want.shape)
    u = np.dtype("u%d" % got.itemsize)
    bad = np.ascontiguousarray(got).view(u) != np.ascontiguousarray(want).view(u)
    assert not bad.any(), "%s: %d of %d values differ, first at %s" % (what, bad.sum(), bad.size,
                                                                         np.argwhere(bad)[0])


def state_crcs(data_rng):
    """CRCs of the three generators a training sampler draws from: np.random, random and the dataset's data_rng."""
    k, pos = np.random.get_state()[1:3]
    c_np = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    c_py = zlib.crc32(np.asarray(random.getstate()[1], np.uint64).tobytes())
    k, pos = data_rng.get_state()[1:3]
    c_dr = zlib.crc32(np.asarray(k, np.uint32).tobytes() + np.int64(pos).tobytes())
    return np.array([c_np, c_py, c_dr], np.uint32)


class StubCOCO(object):
    """The pycocotools calls the training datasets make, over {image id: file name} and {image id: [annotation]}."""

    def __init__(self, files, anns):
        self.files, self.anns = files, anns

    def loadImgs(self, ids):
        return [{'file_name': self.files[ids[0]]}]

    def getAnnIds(self, imgIds):
        return [(imgIds[0], k) for k in range(len(self.anns[imgIds[0]]))]

    def loadAnns(self, ids):
        return [self.anns[i][k] for i, k in ids]


def flat_results(res, num_classes):
    """Per-image {class id: [n, 5]} results -> [R, 7] rows (image, class id, x1, y1, x2, y2, score)."""
    rows = []
    for i, r in enumerate(res):
        for j in range(1, num_classes + 1):
            a = np.asarray(r[j], np.float32).reshape(-1, 5)
            rows.append(np.concatenate([np.full((len(a), 1), i, np.float32), np.full((len(a), 1), j, np.float32), a], 1))
    return np.concatenate(rows, 0)


def edge_merge_case(g, name):
    """Inputs of the merge `name` of tests/golden/post_edges.npz: per-scale [B, K, 6] detections, the per-scale
    metas of ctdet_merge_device (per-image centre and scalar or vector scale), num_classes, max_per_image, nms."""
    dets, c, s, scalar = g[name + "_dets"], g[name + "_c"], g[name + "_s"], g[name + "_s_scalar"]
    scales, hw = g[name + "_scales"], g[name + "_hw"]
    nc, mpi, run_nms = (int(v) for v in g[name + "_cfg"])
    S, B = dets.shape[0], dets.shape[1]
    metas = [{"c": [c[k, i] for i in range(B)],
              "s": [np.float32(s[k, i, 0]) if scalar[i] else s[k, i] for i in range(B)],
              "out_height": int(hw[k, 0]), "out_width": int(hw[k, 1]), "scale": float(scales[k])} for k in range(S)]
    return [dets[k] for k in range(S)], metas, nc, mpi, bool(run_nms)

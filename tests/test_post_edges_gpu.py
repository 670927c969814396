"""The device post-processing of csrc/post.cu at its edges, bit for bit:
  * k_soft_nms (drop-in soft_nms / soft_nms_39) on every list of tests/golden/post_edges.npz, the reference's
    compiled routine's output: the whole in-place array, stale rows included, and the keep length;
  * ctdet_merge_device (k_post_transform, k_group_by_class, k_soft_nms, k_topk_keep) on every merge of that
    golden: five test scales, per-image centres and scales, a class list over 1536 rows, 4096 rows per image;
  * k_group_by_class against boolean-mask grouping across its 256-row chunks, with class ids that are out of
    range, negative, non-integer, -0.0 and NaN;
  * k_topk_keep against np.partition (merge_outputs) with ties, +-0, +-inf and NaN of both signs;
  * ctdet_post_process / multi_pose_post_process on five images with their own centres and scales."""
import numpy as np
import pytest
import torch

from helpers import assert_same_bits, edge_merge_case, flat_results, golden
from oracle import post_np as O

pytestmark = pytest.mark.gpu

EDGES = golden("post_edges")
NMS_NAMES = [str(n) for n in EDGES["nms_names"]]
MERGE_NAMES = [str(n) for n in EDGES["merge_names"]]
NAN_NEG = np.array([0xffc00000], np.uint32).view(np.float32)[0]
NAN_POS = np.array([0x7fc00000], np.uint32).view(np.float32)[0]


@pytest.fixture(scope="module")
def P():
    from centernet_b200 import post_process
    return post_process


@pytest.mark.parametrize("name", NMS_NAMES)
def test_soft_nms_edges(P, name):
    a = EDGES[name + "_in"].copy()
    sigma, Nt, thr, method = (float(v) for v in EDGES[name + "_cfg"])
    fn = P.soft_nms_39 if a.shape[1] == 39 else P.soft_nms
    keep = fn(a, sigma=sigma, Nt=Nt, threshold=thr, method=int(method))
    assert keep == list(range(int(EDGES[name + "_n"])))
    assert_same_bits(a, EDGES[name + "_out"], name)


@pytest.mark.parametrize("name", MERGE_NAMES)
def test_merge_edges(P, name):
    dets, metas, nc, mpi, run_nms = edge_merge_case(EDGES, name)
    res = P.ctdet_merge_device([torch.from_numpy(d).cuda() for d in dets], metas, nc, max_per_image=mpi, nms=run_nms)
    assert_same_bits(flat_results(res, nc), EDGES[name + "_out"], name)


def _class_ids(rng, shape, nc):
    """Mostly valid ids, with ids that the reference's `classes == j` mask never matches (out of range,
    negative, non-integer, NaN, inf) and -0.0, which matches class 0."""
    c = rng.integers(0, nc, shape).astype(np.float32)
    odd = np.array([nc, nc + 3, 1e9, 2.0 ** 31, -1, -7, 0.5, nc - 0.5, np.nan, NAN_NEG, np.inf, -np.inf, -0.0],
                   np.float32)
    pick = rng.random(shape) < 0.15
    c[pick] = odd[rng.integers(0, len(odd), int(pick.sum()))]
    return c


@pytest.mark.parametrize("nc", [1, 80, 8192])
@pytest.mark.parametrize("n", [255, 256, 257, 1000, 4096])
def test_group_by_class(n, nc):
    from centernet_b200._lib import C, ptr, stream_ptr
    rng = np.random.default_rng(1000 * n + nc)
    B = 2
    dets = rng.uniform(-50, 600, (B, n, 6)).astype(np.float32)
    dets[:, ::37, 0] = NAN_NEG                 # payload bits travel untouched
    dets[..., 5] = _class_ids(rng, (B, n), nc)
    d = torch.from_numpy(dets).cuda()
    rows = torch.full((B, n, 5), 12345.0, dtype=torch.float32, device="cuda")
    offs = torch.empty((B, nc + 1), dtype=torch.int32, device="cuda")
    C.group_by_class(ptr(d), B, n, nc, ptr(rows), ptr(offs), stream_ptr(d))
    rows, offs = rows.cpu().numpy(), offs.cpu().numpy()
    for i in range(B):
        cls = dets[i, :, 5]
        want = [dets[i, cls == j, :5] for j in range(nc)]          # utils/post_process.py:93-97, input order kept
        counts = np.array([len(w) for w in want])
        np.testing.assert_array_equal(offs[i], np.concatenate([[0], np.cumsum(counts)]))
        got, want = rows[i, :offs[i, nc]], np.concatenate(want, 0)
        assert_same_bits(got, want, "n=%d nc=%d image %d" % (n, nc, i))
        assert (got.view(np.uint32) == want.view(np.uint32)).all()      # rows are copied: NaN payloads kept too
    assert int(offs[:, nc].sum()) < B * n                               # some ids were dropped


def _scores(rng, kind, shape):
    if kind == "rand":
        return rng.uniform(0, 1, shape).astype(np.float32)
    if kind == "ties":                                # few levels: the threshold value is shared by many rows
        return (rng.integers(1, 6, shape) / 5).astype(np.float32)
    if kind == "zeros":                               # +0 / -0 at the threshold
        s = np.where(rng.random(shape) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
        s[rng.random(shape) < 0.2] = 0.5
        return s
    vals = np.array([0.25, 0.5, 0.0, -0.0, np.inf, -np.inf, NAN_POS, NAN_NEG, -0.25], np.float32)
    p = {"specials": [0.3, 0.3, 0.05, 0.05, 0.05, 0.05, 0.05, 0.1, 0.05],
         "nans": [0.1, 0.1, 0.0, 0.0, 0.05, 0.05, 0.3, 0.4, 0.0]}[kind]   # "nans": the threshold itself is NaN
    return vals[rng.choice(len(vals), shape, p=p)]


TOPK_CASES = [(100, 100, "rand", 80), (101, 100, "rand", 80), (128, 100, "ties", 80), (256, 100, "specials", 80),
              (512, 100, "zeros", 80), (1024, 100, "ties", 80), (2048, 100, "specials", 1), (4096, 100, "specials", 80),
              (4096, 4095, "ties", 80), (4096, 1, "specials", 80), (2, 1, "specials", 1), (101, 100, "nans", 80),
              (300, 100, "nans", 3)]


@pytest.mark.parametrize("n,mpi,kind,nc", TOPK_CASES)
def test_topk_keep_vs_partition(P, n, mpi, kind, nc):
    """ctdet_merge_device on one scale without soft-NMS: the cut is merge_outputs' np.partition threshold."""
    rng = np.random.default_rng(n * 7 + mpi)
    B = 2
    d = np.zeros((B, n, 6), np.float32)
    d[..., 0] = rng.uniform(0, 100, (B, n)); d[..., 1] = rng.uniform(0, 100, (B, n))
    d[..., 2] = d[..., 0] + 4; d[..., 3] = d[..., 1] + 4
    d[..., 4] = _scores(rng, kind, (B, n))
    d[..., 5] = rng.integers(0, nc, (B, n))
    meta = {"c": [np.array([64.0, 48.0], np.float32)] * B, "s": [128.0, np.array([128.0, 96.0], np.float32)],
            "out_height": 96, "out_width": 128}
    got = P.ctdet_merge_device([torch.from_numpy(d).cuda()], [meta], nc, max_per_image=mpi)
    for i in range(B):
        r = O.ctdet_post_process(d[i:i + 1], meta["c"][i:i + 1], meta["s"][i:i + 1], 96, 128, nc)[0]
        want = O.merge_outputs([r], nc, mpi, run_nms=False)
        assert_same_bits(flat_results([got[i]], nc), flat_results([want], nc), "%s n=%d image %d" % (kind, n, i))


def test_post_process_per_image_centres_and_scales(P):
    """Five images, each with its own centre and a scalar or vector scale, against the oracle."""
    rng = np.random.default_rng(55)
    B, K, nc, h, w = 5, 100, 80, 96, 160
    c = [np.array([rng.uniform(100, 500), rng.uniform(80, 300)], np.float32) for _ in range(B)]
    s = [512.0, np.array([640.0, 384.0], np.float32), np.float32(777.5), np.array([320.0, 480.0], np.float32), 1024]
    dets = np.zeros((B, K, 6), np.float32)
    dets[..., 0] = rng.uniform(-4, w, (B, K)); dets[..., 1] = rng.uniform(-4, h, (B, K))
    dets[..., 2] = dets[..., 0] + rng.uniform(0, 40, (B, K)); dets[..., 3] = dets[..., 1] + rng.uniform(0, 40, (B, K))
    dets[..., 4] = np.sort(rng.uniform(0, 1, (B, K)), axis=1)[:, ::-1]
    dets[..., 5] = rng.integers(0, nc, (B, K))
    for src in (dets, torch.from_numpy(dets).cuda()):
        got = P.ctdet_post_process(src, c, s, h, w, nc)
        assert_same_bits(flat_results(got, nc), flat_results(O.ctdet_post_process(dets, c, s, h, w, nc), nc), "ctdet")
    mp = np.zeros((B, K, 40), np.float32)
    mp[..., :5] = dets[..., :5]
    mp[..., 5:39] = rng.uniform(-10, w + 10, (B, K, 34))
    got = P.multi_pose_post_process(torch.from_numpy(mp).cuda(), c, s, h, w)
    want = O.multi_pose_post_process(mp, c, s, h, w)
    assert_same_bits(np.stack([np.asarray(got[i][1], np.float32) for i in range(B)]),
                     np.stack([want[i][1] for i in range(B)]), "multi_pose")

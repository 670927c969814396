"""The numpy soft-NMS / merge oracle (oracle/post_np.py) against the reference's compiled soft_nms and
post-processing at the edges of tests/golden/post_edges.npz (tests/golden/make_golden_post_edges.py): list lengths
around 32 / 256 / 1536 / 4096, ties, exact thresholds and overlaps, touching and degenerate boxes, +-inf / NaN
scores and NaN coordinates, multi-scale merges.  The oracle is plain Python, O(N^2): it is run live on lists of at
most 300 rows; longer lists are checked against the stored reference output on the GPU only
(tests/test_post_edges_gpu.py)."""
import numpy as np
import pytest

from helpers import assert_same_bits, edge_merge_case, flat_results, golden
from oracle import post_np as O

EDGES = golden("post_edges")
LIVE_ROWS = 300
NMS_NAMES = [str(n) for n in EDGES["nms_names"]]
MERGE_NAMES = [str(n) for n in EDGES["merge_names"]]


def test_golden_covers_the_edges():
    """The golden keeps the list lengths and edge cases the GPU tests rely on."""
    lengths = {len(EDGES[n + "_in"]) for n in NMS_NAMES}
    assert {1, 2, 31, 32, 33, 64, 65, 255, 256, 257, 1535, 1536, 1537, 2048, 4096} <= lengths
    assert {int(EDGES[n + "_cfg"][3]) for n in NMS_NAMES} == {0, 1, 2}
    assert any(EDGES[n + "_cfg"][2] == 0 for n in NMS_NAMES)
    nan_scores = [n for n in NMS_NAMES if np.isnan(EDGES[n + "_in"][:, 4]).any()]
    nan_coords = [n for n in NMS_NAMES if np.isnan(EDGES[n + "_in"][:, :4]).any()]
    assert nan_scores and nan_coords
    assert any(EDGES[n + "_in"].shape[1] == 39 for n in NMS_NAMES)
    longest_list, most_rows = 0, 0
    for m in MERGE_NAMES:
        dets, _, nc, _, _ = edge_merge_case(EDGES, m)
        most_rows = max(most_rows, sum(d.shape[1] for d in dets))
        for j in range(nc):        # rows of class j in one image, over every scale
            longest_list = max(longest_list, int(max(sum((d[i, :, 5] == j).sum() for d in dets)
                                                     for i in range(dets[0].shape[0]))))
    assert longest_list > 1536       # a class list longer than the former fixed shared-memory list size
    assert most_rows == 4096


@pytest.mark.parametrize("name", [n for n in NMS_NAMES if len(EDGES[n + "_in"]) <= LIVE_ROWS])
def test_oracle_soft_nms_edges(name):
    """The whole in-place array and the keep length, bit for bit (NaN where the reference has NaN).  The NaN cases
    pin the pivot scan (a NaN score is never picked, and a NaN at row i stays there) and nms.pyx's own min / max
    (a NaN second operand wins)."""
    b = EDGES[name + "_in"]
    sigma, Nt, thr, method = EDGES[name + "_cfg"]
    a = b.copy()
    n = O.soft_nms(a, sigma=sigma, Nt=Nt, threshold=thr, method=int(method), ncols_swap=b.shape[1] - 5)
    assert n == int(EDGES[name + "_n"])
    assert_same_bits(a, EDGES[name + "_out"], name)


@pytest.mark.parametrize("name", MERGE_NAMES)
def test_oracle_merge_edges(name):
    """ctdet_post_process of every image and scale, the division by the scale and merge_outputs, against the
    reference, where every class list stays within the live-oracle length."""
    dets, metas, nc, mpi, run_nms = edge_merge_case(EDGES, name)
    if sum(d.shape[1] for d in dets) > LIVE_ROWS and nc < 80:
        pytest.skip("class lists longer than %d rows: checked against the stored reference on the GPU" % LIVE_ROWS)
    B = dets[0].shape[0]
    res = []
    for i in range(B):
        per_scale = []
        for d, m in zip(dets, metas):
            r = O.ctdet_post_process(d[i:i + 1], m["c"][i:i + 1], m["s"][i:i + 1], m["out_height"], m["out_width"], nc)[0]
            for j in r:
                r[j] = np.asarray(r[j], np.float32).reshape(-1, 5)
                r[j][:, :4] /= m["scale"]
            per_scale.append(r)
        res.append(O.merge_outputs(per_scale, nc, mpi, run_nms=run_nms or len(dets) > 1))
    assert_same_bits(flat_results(res, nc), EDGES[name + "_out"], name)


def test_soft_nms_length_limit_without_gpu():
    """Lists longer than 4096 rows are refused before anything reaches the device (drop-in and C ABI)."""
    from centernet_b200 import _C
    from centernet_b200 import post_process as P
    with pytest.raises(NotImplementedError, match="4096"):
        P.soft_nms(np.zeros((4097, 5), np.float32))
    with pytest.raises(RuntimeError, match="4096"):
        _C.soft_nms(16, 16, 16, 1, 1, 4097, 5, 0.5, 0.3, 0.001, 0, 0, 0)
